// quant4.cu -- bitsandbytes 4-bit weights (transformers load_in_4bit=True, Linear4bit; FP4 or NF4, blocks of 64):
//   quantize_4bit    fp16 W [N,K] -> packed codes uint8 [N, K/2] + absmax fp32 [N, K/64], once per weight at load,
//                    optionally into a fused row layout (the LLaMA handle's q|k|v and 128-row gate|up blocks)
//   dequantize_4bit  packed codes + absmax -> fp16 W' [N,K]: the prefill path's weight (0.5625 bytes read and 2
//                    bytes written per weight)
// The 4-bit GEMV is the fp16 GEMV's kernel with a weight-format parameter (misc.cu).  The arithmetic is stated in
// include/seedb200.h.
#include "common.cuh"
#include "ops.h"
#include "quant4.cuh"

namespace sb {

// code of the normalised value n: NF4 = the number of the 15 midpoints of the NF4 table that n exceeds; FP4 = sign
// bit 8 for n < 0 and the magnitude bucket of |n| among 7 pivots, mapped to the 3-bit code of that value.  NaN
// exceeds nothing and is not negative: code 0.
__device__ __forceinline__ uint32_t q4_code(int type, float n, const float* nf4_thr) {
  if (type == SEEDB200_Q4_NF4) {
    uint32_t c = 0;
#pragma unroll
    for (int i = 0; i < 15; ++i) c += n > nf4_thr[i] ? 1u : 0u;
    return c;
  }
  const float a = fabsf(n);
  uint32_t b = 0;
  b += a > 0.00260417f; b += a > 0.0859375f; b += a > 0.20833333f; b += a > 0.29166667f;
  b += a > 0.4166667f; b += a > 0.583333f; b += a > 0.8333333f;
  constexpr uint32_t kBucketCode = 0x32547610u;   // bucket i -> nibble i: 0, 1, 6, 7, 4, 5, 2, 3
  return ((kBucketCode >> (4 * b)) & 7u) | (n < 0.0f ? 8u : 0u);
}

// one thread per 8 consecutive weights (one 16-byte load), 8 threads per block of 64; row n of W goes to row
// (n / grp) * gstride + n % grp + off of packed / absmax
__global__ void __launch_bounds__(256)
quantize_4bit_kernel(const __half* __restrict__ W, long long ldw, int N, int K, int type, uint8_t* __restrict__ packed,
                     float* __restrict__ absmax, int grp, int gstride, int off) {
  __shared__ float thr[15];
  if (threadIdx.x < 15)   // NF4 thresholds: fp32 midpoints of adjacent table values
    thr[threadIdx.x] = __fmul_rn(__fadd_rn(kQ4Value[1][threadIdx.x], kQ4Value[1][threadIdx.x + 1]), 0.5f);
  __syncthreads();
  const int gpr = K / 8;
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const bool valid = g < (long long)N * gpr;           // whole blocks of 64 are valid or not together
  const int n = valid ? (int)(g / gpr) : 0, c = valid ? (int)(g % gpr) : 0;
  uint4 raw = make_uint4(0, 0, 0, 0);
  if (valid) raw = *reinterpret_cast<const uint4*>(W + (long long)n * ldw + (long long)c * 8);
  const __half* h = reinterpret_cast<const __half*>(&raw);
  float v[8], mx = 0.0f;
#pragma unroll
  for (int j = 0; j < 8; ++j) { v[j] = __half2float(h[j]); mx = fmaxf(mx, fabsf(v[j])); }
#pragma unroll
  for (int s = 1; s < 8; s <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
  if (!valid) return;
  const float r = __frcp_rn(mx);
  uint32_t p = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) p |= q4_code(type, __fmul_rn(v[j], r), thr) << (8 * (j / 2) + ((j & 1) ? 0 : 4));
  const long long row = (long long)(n / grp) * gstride + n % grp + off;
  *reinterpret_cast<uint32_t*>(packed + row * (K / 2) + (long long)c * 4) = p;
  if ((c & 7) == 0) absmax[row * (K / Q4_BLOCK) + c / 8] = mx;
}

__global__ void __launch_bounds__(256)
dequantize_4bit_kernel(const uint8_t* __restrict__ packed, const float* __restrict__ absmax, int N, int K, int type,
                       __half* __restrict__ out, long long ldo) {
  __shared__ float tab[16];
  if (threadIdx.x < 16) tab[threadIdx.x] = kQ4Value[type][threadIdx.x];
  __syncthreads();
  const int gpr = K / 8;
  const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (g >= (long long)N * gpr) return;
  const long long n = g / gpr;
  const int c = (int)(g % gpr);
  const uint32_t p = __ldg(reinterpret_cast<const uint32_t*>(packed + n * (K / 2)) + c);
  const float a = __ldg(absmax + n * (K / Q4_BLOCK) + c / 8);
  *reinterpret_cast<uint4*>(out + n * ldo + (long long)c * 8) = q4_deq8(p, a, tab);
}

int q4_check(const char* who, int type, int N, int K) {
  SB_REQUIRE(type == SEEDB200_Q4_FP4 || type == SEEDB200_Q4_NF4, "%s: quant_type %d is neither FP4 (0) nor NF4 (1)",
             who, type);
  SB_REQUIRE(N > 0 && K > 0, "%s: bad shape N=%d K=%d", who, N, K);
  SB_REQUIRE(K % Q4_BLOCK == 0, "%s: K=%d is not a multiple of the 4-bit blocksize %d", who, K, Q4_BLOCK);
  return 0;
}

int quantize_4bit_rows(const void* W, int64_t ldw, int N, int K, int type, void* packed, void* absmax, int grp,
                       int gstride, int off, cudaStream_t stream) {
  SB_PROPAGATE(q4_check("quantize_4bit", type, N, K));
  if (ldw == 0) ldw = K;
  SB_REQUIRE(W && packed && absmax && grp > 0, "quantize_4bit: null operand");
  SB_REQUIRE(ldw >= K && ldw % 8 == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
             "quantize_4bit: W must be 16-byte aligned with ldw (%lld) >= K (%d) a multiple of 8", (long long)ldw, K);
  const long long threads = (long long)N * (K / 8);
  quantize_4bit_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(
      static_cast<const __half*>(W), ldw, N, K, type, static_cast<uint8_t*>(packed), static_cast<float*>(absmax), grp,
      gstride, off);
  SB_LAUNCH_CHECK();
  return 0;
}

int dequantize_4bit(const void* packed, const void* absmax, int N, int K, int type, void* out, int64_t ldo,
                    cudaStream_t stream) {
  SB_PROPAGATE(q4_check("dequantize_4bit", type, N, K));
  if (ldo == 0) ldo = K;
  SB_REQUIRE(packed && absmax && out, "dequantize_4bit: null operand");
  SB_REQUIRE(ldo >= K && ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(packed) & 3) == 0,
             "dequantize_4bit: out must be 16-byte aligned with ldo (%lld) >= K (%d) a multiple of 8", (long long)ldo, K);
  const long long threads = (long long)N * (K / 8);
  dequantize_4bit_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(
      static_cast<const uint8_t*>(packed), static_cast<const float*>(absmax), N, K, type, static_cast<__half*>(out),
      ldo);
  SB_LAUNCH_CHECK();
  return 0;
}

}  // namespace sb

extern "C" {

int seedb200_quantize_4bit(const void* W, int64_t ldw, int N, int K, int quant_type, void* packed, void* absmax,
                           void* stream) {
  return sb::quantize_4bit_rows(W, ldw, N, K, quant_type, packed, absmax, N > 0 ? N : 1, 0, 0,
                                static_cast<cudaStream_t>(stream));
}

int seedb200_dequantize_4bit(const void* packed, const void* absmax, int N, int K, int quant_type, void* out,
                             int64_t ldo, void* stream) {
  return sb::dequantize_4bit(packed, absmax, N, K, quant_type, out, ldo, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
