// lora.cu -- unmerged PEFT LoRA on the fp16 decoder linears (include/seedb200.h states the arithmetic):
//   shrink   T = fp16(X . A_cat^T) for the A matrices that share an input (q|k|v, o, gate|up, down); more than 4
//            rows go to the wgmma GEMM with N = r_tot
//   expand   y = fp16(base + fp16(fp16(B . t) * s)), then the linear's own epilogue step (residual add or SiLU gate)
//   merge    W = fp16(W + fp16(fp16(B . A) * s)) in place, PEFT's merge
// Decode (<= 4 rows): the expand runs in the GEMV's epilogue (misc.cu).  More rows: the base product comes from the
// unchanged wgmma GEMM (mode 0, no residual) and the expand kernel below reads it back, so the GEMM and its rounding
// stay exactly as without an adapter.
#include "common.cuh"
#include "ops.h"

namespace sb {

// ----------------------------------------------------------------------------
// shrink, M <= 4 rows (decode): one CTA per column j of A_cat [r_tot, K], 256 threads spread over K.  With norm_w the
// rows are RMS-normalised while staged, with gemv_kernel's arithmetic and reduction order (misc.cu), so t is computed
// from exactly the activations the fused-norm GEMV multiplies.
// ----------------------------------------------------------------------------
template <int M, bool NORM>
__global__ void __launch_bounds__(256)
lora_shrink_rows_kernel(const __half* __restrict__ x, const __half* __restrict__ norm_w, float eps,
                        const __half* __restrict__ A, int K, __half* __restrict__ T, long long ldt) {
  __shared__ float red[8];
  __shared__ float part[8][M];
  const int nvec = K / 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5, nthr = blockDim.x;
  const int j = blockIdx.x;
  pdl_trigger();
  pdl_wait();
  float rstd[M];
#pragma unroll
  for (int m = 0; m < M; ++m) rstd[m] = 1.0f;
  if constexpr (NORM) {
#pragma unroll 1
    for (int m = 0; m < M; ++m) {
      float ss = 0.0f;
      for (int i = threadIdx.x; i < nvec; i += nthr) {
        const uint4 raw = reinterpret_cast<const uint4*>(x)[m * nvec + i];
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int q = 0; q < 4; ++q) { const float2 f = __half22float2(h[q]); ss += f.x * f.x; ss += f.y * f.y; }
      }
      ss = warp_sum(ss);
      __syncthreads();
      if (lane == 0) red[warp] = ss;
      __syncthreads();
      float tot = 0.0f;
      for (int i = 0; i < nw; ++i) tot += red[i];
      rstd[m] = rsqrtf(tot * (1.0f / (float)K) + eps);
    }
  }
  float acc[M];
#pragma unroll
  for (int m = 0; m < M; ++m) acc[m] = 0.0f;
  const uint4* arow = reinterpret_cast<const uint4*>(A + (long long)j * K);
  for (int i = threadIdx.x; i < nvec; i += nthr) {
    const uint4 av = __ldg(arow + i);
    const __half* ah = reinterpret_cast<const __half*>(&av);
    uint4 wraw = make_uint4(0, 0, 0, 0);
    if constexpr (NORM) wraw = __ldg(reinterpret_cast<const uint4*>(norm_w) + i);
    const __half* wh = reinterpret_cast<const __half*>(&wraw);
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const uint4 raw = reinterpret_cast<const uint4*>(x)[m * nvec + i];
      const __half* h = reinterpret_cast<const __half*>(&raw);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        float v = __half2float(h[q]);
        if constexpr (NORM) {
          const __half n16 = __float2half_rn(v * rstd[m]);
          v = __half2float(__float2half_rn(__half2float(n16) * __half2float(wh[q])));
        }
        acc[m] = fmaf(__half2float(ah[q]), v, acc[m]);
      }
    }
  }
#pragma unroll
  for (int m = 0; m < M; ++m) {
    const float s = warp_sum(acc[m]);
    if (lane == 0) part[warp][m] = s;
  }
  __syncthreads();
  if (threadIdx.x < M) {
    float tot = 0.0f;
    for (int w = 0; w < nw; ++w) tot += part[w][threadIdx.x];
    T[(long long)threadIdx.x * ldt + j] = __float2half_rn(tot);
  }
}

int lora_shrink(const void* x, int64_t ldx, const void* norm_w, float eps, const void* A, int M, int K, int rtot,
                void* T, int64_t ldt, cudaStream_t stream) {
  SB_REQUIRE(M >= 1 && K >= 8 && K % 8 == 0, "lora_shrink: M=%d K=%d (K must be a positive multiple of 8)", M, K);
  SB_REQUIRE(rtot >= 1 && rtot <= LORA_MAX_RTOT, "lora_shrink: r_tot %d outside [1,%d]", rtot, LORA_MAX_RTOT);
  SB_REQUIRE(ldt >= rtot, "lora_shrink: ldt %lld < r_tot %d", (long long)ldt, rtot);
  const __half* xp = static_cast<const __half*>(x);
  const __half* ap = static_cast<const __half*>(A);
  const __half* np = static_cast<const __half*>(norm_w);
  __half* tp = static_cast<__half*>(T);
  if (M <= 4) {
    SB_REQUIRE(ldx == K, "lora_shrink: rows of <= 4 must be dense (ldx %lld != K %d)", (long long)ldx, K);
#define SB_SHRINK(M_)                                                                                        \
    if (M == M_) {                                                                                           \
      if (np) SB_CHECK_CUDA(launch_chain(lora_shrink_rows_kernel<M_, true>, dim3(rtot), dim3(256), 0, stream,   \
                                         xp, np, eps, ap, K, tp, (long long)ldt));                          \
      else SB_CHECK_CUDA(launch_chain(lora_shrink_rows_kernel<M_, false>, dim3(rtot), dim3(256), 0, stream,     \
                                      xp, np, eps, ap, K, tp, (long long)ldt));                             \
    }
    SB_SHRINK(1) SB_SHRINK(2) SB_SHRINK(3) SB_SHRINK(4)
#undef SB_SHRINK
    SB_LAUNCH_CHECK();
    return 0;
  }
  // more rows: the wgmma GEMM with N = r_tot (fp32 accumulation on the tensor cores, one rounding to fp16)
  SB_REQUIRE(norm_w == nullptr, "lora_shrink: norm_w is only folded for <= 4 rows");
  SB_REQUIRE(ldx >= K && ldx % 8 == 0, "lora_shrink: ldx %lld must be >= K %d and a multiple of 8", (long long)ldx, K);
  seedb200_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.M = M; d.N = rtot; d.K = K; d.A = x; d.lda = ldx; d.W = A; d.ldw = K; d.out = T; d.ldo = ldt;
  return gemm(d, stream);
}

// ----------------------------------------------------------------------------
// expand: a thread owns one output row n of the fused layout (two in mode 1: gate n and up n + 128) and keeps its B
// row(s) in registers across EX_ROWS activation rows, whose t rows are staged in shared memory.  Row n reads the r
// columns ((n / grp) % nsub) * r of t; a sub-block without an adapter (mask bit clear) passes base through.  RB = r
// rounded up to 8, 16, 32 or 64: lanes j >= r multiply zeros staged here, never a t value.
// GEMV_SILU picks the SiLU of the kernel that made `base` (the GEMV's __expf and IEEE divide, or the GEMM epilogue's
// ex2 / rcp approximations), so that a zero B reproduces the base model bit for bit.
// ----------------------------------------------------------------------------
constexpr int EX_ROWS = 16;

__device__ __forceinline__ float rcp_approx_f(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx_f(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

template <int RB>
struct LoraRow {
  float b[RB];
  int sub;
  bool on;
  __device__ __forceinline__ void load(const __half* __restrict__ Bw, int n, int r, int grp, int nsub, unsigned mask) {
    sub = (n / grp) % nsub;
    on = (mask >> sub) & 1u;
#pragma unroll
    for (int j = 0; j < RB; ++j) b[j] = j < r ? __half2float(Bw[(long long)n * r + j]) : 0.0f;
  }
  // y = fp16(base + fp16(fp16(B t) * s))
  __device__ __forceinline__ __half y(__half base, const float* t, float s) const {
    if (!on) return base;
    const float* ts = t + sub * RB;
    float acc = 0.0f;
#pragma unroll
    for (int j = 0; j < RB; ++j) acc = fmaf(b[j], ts[j], acc);
    const __half u = __float2half_rn(acc);
    const __half c = __float2half_rn(__half2float(u) * s);
    return __float2half_rn(__half2float(base) + __half2float(c));
  }
};

template <int MODE, bool GEMV_SILU, int RB>
__global__ void __launch_bounds__(256)
lora_expand_kernel(const __half* base, long long ldb, const __half* __restrict__ T, long long ldt,
                   const __half* __restrict__ Bw, int r, int grp, int nsub, unsigned mask, float s, int M, int N,
                   const __half* residual, long long ldr, __half* out, long long ldo) {
  __shared__ float ts[EX_ROWS][3 * RB];
  const int m0 = blockIdx.y * EX_ROWS;
  const int rows = min(EX_ROWS, M - m0);
  pdl_trigger();
  pdl_wait();
  for (int i = threadIdx.x; i < EX_ROWS * 3 * RB; i += blockDim.x) {
    const int mm = i / (3 * RB), sb = (i % (3 * RB)) / RB, j = i % RB;
    ts[mm][sb * RB + j] = (mm < rows && sb < nsub && j < r) ? __half2float(T[(long long)(m0 + mm) * ldt + sb * r + j])
                                                           : 0.0f;
  }
  __syncthreads();
  const int task = blockIdx.x * blockDim.x + threadIdx.x;
  if (MODE == 1) {
    if (task >= N / 2) return;
    const int n0 = (task / 128) * 256 + task % 128, n1 = n0 + 128;
    LoraRow<RB> g, u;
    g.load(Bw, n0, r, grp, nsub, mask);
    u.load(Bw, n1, r, grp, nsub, mask);
    for (int mm = 0; mm < rows; ++mm) {
      const long long m = m0 + mm;
      const float gv = __half2float(g.y(base[m * ldb + n0], ts[mm], s));
      const float uv = __half2float(u.y(base[m * ldb + n1], ts[mm], s));
      float sg;
      if (GEMV_SILU) sg = __half2float(__float2half_rn(gv / (1.0f + __expf(-gv))));
      else sg = __half2float(__float2half_rn(gv * rcp_approx_f(1.0f + ex2_approx_f(-1.4426950408889634f * gv))));
      out[m * ldo + task] = __float2half_rn(sg * uv);
    }
  } else {
    if (task >= N) return;
    LoraRow<RB> w;
    w.load(Bw, task, r, grp, nsub, mask);
    for (int mm = 0; mm < rows; ++mm) {
      const long long m = m0 + mm;
      __half y = w.y(base[m * ldb + task], ts[mm], s);
      if (residual != nullptr) y = __float2half_rn(__half2float(y) + __half2float(residual[m * ldr + task]));
      out[m * ldo + task] = y;
    }
  }
}

static int lora_check(const seedb200_lora_operand& lo, int N, int mode) {
  SB_REQUIRE(lo.T && lo.B, "lora: null T or B");
  SB_REQUIRE(lo.r >= 1 && lo.r <= LORA_MAX_R, "lora: r %d outside [1,%d]", lo.r, LORA_MAX_R);
  SB_REQUIRE(lo.nsub >= 1 && lo.nsub <= 3 && lo.grp >= 1, "lora: nsub %d / grp %d", lo.nsub, lo.grp);
  SB_REQUIRE(lo.ldt >= (int64_t)lo.r * lo.nsub, "lora: ldt %lld < r * nsub", (long long)lo.ldt);
  SB_REQUIRE(mode == 0 || mode == 1, "lora: unknown mode %d", mode);
  SB_REQUIRE(mode == 0 || N % 256 == 0, "lora: mode 1 needs N %% 256 == 0 (N=%d)", N);
  return 0;
}

int lora_expand(const void* base, int64_t ldb, const seedb200_lora_operand& lo, int M, int N, int mode,
                bool gemv_silu, const void* residual, int64_t ldr, void* out, int64_t ldo, cudaStream_t stream) {
  SB_PROPAGATE(lora_check(lo, N, mode));
  SB_REQUIRE(M >= 1 && N >= 1, "lora_expand: M %d / N %d", M, N);
  const int tasks = mode == 1 ? N / 2 : N;
  const dim3 grid((tasks + 255) / 256, (M + EX_ROWS - 1) / EX_ROWS);
  const __half* bp = static_cast<const __half*>(base);
  const __half* tp = static_cast<const __half*>(lo.T);
  const __half* wp = static_cast<const __half*>(lo.B);
  const __half* rp = static_cast<const __half*>(residual);
  __half* op = static_cast<__half*>(out);
  const long long a1 = ldb, a3 = lo.ldt, a11 = ldr, a13 = ldo;
#define SB_EXPAND(MD_, GS_, RB_)                                                                              \
  SB_CHECK_CUDA(launch_chain(lora_expand_kernel<MD_, GS_, RB_>, grid, dim3(256), 0, stream, bp, a1, tp, a3, wp,    \
                             lo.r, lo.grp, lo.nsub, lo.mask, lo.scale, M, N, rp, a11, op, a13))
#define SB_EXPAND_R(MD_, GS_)                                                                                 \
  if (lo.r <= 8) SB_EXPAND(MD_, GS_, 8); else if (lo.r <= 16) SB_EXPAND(MD_, GS_, 16);                      \
  else if (lo.r <= 32) SB_EXPAND(MD_, GS_, 32); else SB_EXPAND(MD_, GS_, 64);
  if (mode == 1) {
    if (gemv_silu) { SB_EXPAND_R(1, true) } else { SB_EXPAND_R(1, false) }
  } else {
    SB_EXPAND_R(0, false)
  }
#undef SB_EXPAND_R
#undef SB_EXPAND
  SB_LAUNCH_CHECK();
  return 0;
}

// the base product goes to lo.workspace (or straight to out when mode 0 has no residual), then the expand kernel
int gemm_lora(const seedb200_gemm_desc& d, const seedb200_lora_operand& lo, cudaStream_t stream) {
  SB_PROPAGATE(lora_check(lo, d.N, d.mode));
  SB_REQUIRE(!d.bias && d.act == SEEDB200_ACT_NONE && !d.ln_stats && !d.row_moments && d.row_group == 0 &&
                 d.res_mod == 0,
             "gemm_lora: only the plain, residual and SiLU-gate epilogues take a LoRA operand");
  const bool in_place = d.mode == 0 && d.residual == nullptr && lo.workspace == nullptr;
  SB_REQUIRE(in_place || lo.workspace, "gemm_lora: a workspace of [M, N] fp16 is needed for this epilogue");
  seedb200_gemm_desc b = d;
  b.mode = 0; b.residual = nullptr; b.ldr = 0;
  b.out = in_place ? d.out : lo.workspace;
  b.ldo = in_place ? (d.ldo ? d.ldo : d.N) : d.N;
  if (d.mode == 1 && b.bn == 0) b.bn = 256;     // the SiLU-gate GEMM's tile: the same k order per output
  SB_PROPAGATE(gemm(b, stream));
  const int64_t ldo = d.ldo ? d.ldo : (d.mode == 1 ? d.N / 2 : d.N);
  return lora_expand(b.out, b.ldo, lo, d.M, d.N, d.mode, false, d.residual, d.ldr ? d.ldr : ldo, d.out, ldo, stream);
}

// decode: the expand runs in the GEMV's epilogue (misc.cu); no workspace, no second launch
int gemv_lora(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w, float eps,
              int M, int N, int K, int mode, const seedb200_lora_operand& lo, cudaStream_t stream, int64_t ldo) {
  SB_PROPAGATE(lora_check(lo, N, mode));
  return gemv(x, W, ldw, out, residual, norm_w, eps, M, N, K, mode, stream, ldo, &lo);
}

// ----------------------------------------------------------------------------
// merge: W[n, k] (fused layout, row stride K) += fp16(fp16(sum_j B[n, j] A[sub r + j, k]) * s)
// ----------------------------------------------------------------------------
__global__ void lora_merge_kernel(__half* W, const __half* __restrict__ A, const __half* __restrict__ Bw, int N, int K,
                                  int r, int grp, int nsub, unsigned mask, float s) {
  const long long n = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int sub = (int)((n / grp) % nsub);
  if (k >= K || !((mask >> sub) & 1u)) return;
  float acc = 0.0f;
  for (int j = 0; j < r; ++j) acc = fmaf(__half2float(Bw[n * r + j]), __half2float(A[(long long)(sub * r + j) * K + k]), acc);
  const __half d = __float2half_rn(__half2float(__float2half_rn(acc)) * s);
  W[n * K + k] = __float2half_rn(__half2float(W[n * K + k]) + __half2float(d));
}

int lora_merge(void* W, const void* A, const seedb200_lora_operand& lo, int N, int K, cudaStream_t stream) {
  SB_PROPAGATE(lora_check(lo, N, 0));
  SB_REQUIRE(N >= 1 && N <= 65535 && K >= 1, "lora_merge: N %d outside [1,65535] or K %d < 1", N, K);
  lora_merge_kernel<<<dim3((K + 255) / 256, N), 256, 0, stream>>>(
      static_cast<__half*>(W), static_cast<const __half*>(A), static_cast<const __half*>(lo.B), N, K, lo.r, lo.grp,
      lo.nsub, lo.mask, lo.scale);
  SB_LAUNCH_CHECK();
  return 0;
}

}  // namespace sb

extern "C" {

int seedb200_lora_shrink(const void* x, int64_t ldx, const void* norm_w, float eps, const void* A, int M, int K,
                         int r_tot, void* T, int64_t ldt, void* stream) {
  SB_REQUIRE(x && A && T, "seedb200_lora_shrink: null operand");
  return sb::lora_shrink(x, ldx, norm_w, eps, A, M, K, r_tot, T, ldt, static_cast<cudaStream_t>(stream));
}

int seedb200_gemm_lora(const seedb200_gemm_lora_desc* d, void* stream) {
  SB_REQUIRE(d != nullptr, "seedb200_gemm_lora: null descriptor");
  return sb::gemm_lora(d->gemm, d->lora, static_cast<cudaStream_t>(stream));
}

int seedb200_gemv_lora(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w,
                       float eps, int M, int N, int K, int mode, const seedb200_lora_operand* lora, void* stream) {
  SB_REQUIRE(x && W && out && lora, "seedb200_gemv_lora: null operand");
  return sb::gemv_lora(x, W, ldw, out, residual, norm_w, eps, M, N, K, mode, *lora, static_cast<cudaStream_t>(stream),
                       0);
}

}  // extern "C"
