// int8.cuh -- the LLM.int8() output arithmetic shared by the int8 wgmma GEMM (gemm_wgmma.cu) and the int8 GEMV
// (int8.cu), so that both paths produce the same bits.  The contract (bitsandbytes Linear8bitLt, threshold 6.0,
// restated in tests/int8_ref.py):
//   base = fp16(((float)acc * 6.200012e-05f) * SCA[m] * SCB[n])          acc = sum_k CA[m,k] CB[n,k], int32
//   corr = fp16(sum_{j in O, ascending} A[m,j] * fp16(CB[n,j] * SCB[n] / 127))   fp32 accumulation
//   y    = O empty ? base : fp16(base + corr)
#pragma once

#include <cuda_fp16.h>
#include <stdint.h>

namespace sb {

constexpr float INT8_DEQUANT = 6.200012e-05f;   // bitsandbytes MM_DEQUANT_CONST, 1 / 127^2

__device__ __forceinline__ float int8_base(int acc, float sca, float scb) {
  return __half2float(__float2half_rn(((float)acc * INT8_DEQUANT) * sca * scb));
}

// The outlier correction of output (m, n) added to its base, by the 32 lanes of a warp (the int8 GEMV): a_row = fp16
// activations of row m, cb_row = int8 weight row n, ol[0..cnt) = the outlier columns in ascending order.  Each lane
// loads and multiplies one column of a 32-column chunk (the fp16 x fp16 products are exact in fp32), then the sum is
// taken in ascending column order through shuffles.  Every lane returns y.
template <typename Idx>
__device__ __forceinline__ __half int8_finish_warp(float base, const __half* a_row, const int8_t* cb_row, float scb,
                                                   const Idx* ol, int cnt, int lane) {
  if (cnt == 0) return __float2half_rn(base);
  float c = 0.0f;
  for (int t0 = 0; t0 < cnt; t0 += 32) {
    float p = 0.0f;
    if (t0 + lane < cnt) {
      const int j = ol[t0 + lane];
      p = __half2float(a_row[j]) * __half2float(__float2half_rn((float)cb_row[j] * scb / 127.0f));
    }
    const int n = min(32, cnt - t0);
    for (int i = 0; i < n; ++i) c += __shfl_sync(0xffffffffu, p, i);
  }
  return __float2half_rn(base + __half2float(__float2half_rn(c)));
}

// base plus a precomputed fp16 correction (the GEMM path's int8_correction kernel)
__device__ __forceinline__ __half int8_add_corr(float base, __half corr) {
  return __float2half_rn(base + __half2float(corr));
}

// SiLU-gate on fp16-rounded gate and up values, the arithmetic of the fp16 wgmma GEMM's mode-1 epilogue
__device__ __forceinline__ __half int8_silu_mul(__half gate, __half up) {
  const float g = __half2float(gate);
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * g));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  const float s = __half2float(__float2half_rn(g * r));
  return __float2half_rn(s * __half2float(up));
}

}  // namespace sb
