// int8.cu -- LLM.int8() (transformers load_in_8bit=True, bitsandbytes Linear8bitLt with has_fp16_weights=False):
//   int8_quantize_weight  fp16 W -> int8 CB + fp32 SCB, once per weight at load
//   int8_quantize_act     fp16 A -> int8 CA + fp32 SCA + ascending outlier columns, per call, no host synchronisation
//   gemv_int8             M <= 4 rows (the decode step): quantises (and optionally RMS-normalises) the activation rows
//                         while staging them, streams the int8 weights once and accumulates with dp4a
// The arithmetic is stated in include/seedb200.h; the output rounding is shared with the int8 wgmma GEMM (int8.cuh).
#include "common.cuh"
#include "int8.cuh"
#include "ops.h"

namespace sb {

int get_option(const char* key);

__device__ __forceinline__ float block_max_256(float v, float* red) {
  v = warp_max(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float m = 0.0f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
  return m;
}

__device__ __forceinline__ int8_t quant8(float x, float inv) { return (int8_t)__float2int_rn(x * inv); }

// ---- weights: one block per row ----
// row n of W goes to row (n / grp) * gstride + n % grp + off of CB / SCB (the LLaMA handle's fused layouts)
__global__ void __launch_bounds__(256)
int8_quantize_weight_kernel(const __half* __restrict__ W, long long ldw, int K, int8_t* __restrict__ CB,
                            float* __restrict__ SCB, int grp, int gstride, int off) {
  __shared__ float red[8];
  const int n = blockIdx.x;
  const long long r = (long long)(n / grp) * gstride + n % grp + off;
  const __half* row = W + (long long)n * ldw;
  float mx = 0.0f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) mx = fmaxf(mx, fabsf(__half2float(row[k])));
  mx = block_max_256(mx, red);
  if (threadIdx.x == 0) SCB[r] = mx;
  const float inv = 127.0f / mx;
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    CB[r * K + k] = mx == 0.0f ? (int8_t)0 : quant8(__half2float(row[k]), inv);
}

int int8_quantize_weight_rows(const void* W, int64_t ldw, int N, int K, void* CB, void* SCB, int grp, int gstride,
                              int off, cudaStream_t stream) {
  if (ldw == 0) ldw = K;
  SB_REQUIRE(W && CB && SCB && N > 0 && K > 0 && ldw >= K && grp > 0, "int8_quantize_weight: bad arguments (N=%d K=%d "
             "ldw=%lld)", N, K, (long long)ldw);
  int8_quantize_weight_kernel<<<N, 256, 0, stream>>>(static_cast<const __half*>(W), ldw, K, static_cast<int8_t*>(CB),
                                                     static_cast<float*>(SCB), grp, gstride, off);
  SB_LAUNCH_CHECK();
  return 0;
}

int int8_quantize_weight(const void* W, int64_t ldw, int N, int K, void* CB, void* SCB, cudaStream_t stream) {
  return int8_quantize_weight_rows(W, ldw, N, K, CB, SCB, N > 0 ? N : 1, 0, 0, stream);
}

// ---- activations: (1) per row, SCA and the outlier flags of its columns (flags live in the outlier list buffer,
// zeroed before); (2) per row, CA with the flagged columns zeroed; (3) one block turns the flags into the ascending
// list in place and writes the count ----
__global__ void __launch_bounds__(256)
int8_act_scan_kernel(const __half* __restrict__ A, long long lda, int K, float thr, float* __restrict__ SCA,
                     int* __restrict__ flags) {
  __shared__ float red[8];
  const int m = blockIdx.x;
  const __half* row = A + (long long)m * lda;
  float mx = 0.0f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float a = fabsf(__half2float(row[k]));
    if (!(a < thr)) flags[k] = 1;
    else mx = fmaxf(mx, a);
  }
  mx = block_max_256(mx, red);
  if (threadIdx.x == 0) SCA[m] = mx;
}

__global__ void __launch_bounds__(256)
int8_act_quant_kernel(const __half* __restrict__ A, long long lda, int K, const float* __restrict__ SCA,
                      const int* __restrict__ flags, int8_t* __restrict__ CA) {
  const int m = blockIdx.x;
  const __half* row = A + (long long)m * lda;
  const float s = SCA[m];
  const float inv = 127.0f / s;
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    CA[(long long)m * K + k] = (flags[k] != 0 || s == 0.0f) ? (int8_t)0 : quant8(__half2float(row[k]), inv);
}

__global__ void __launch_bounds__(1024) int8_act_compact_kernel(int* list, int K, int* count) {
  __shared__ int wtot[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int base = 0;
  for (int c = 0; c < K; c += 1024) {
    const int k = c + threadIdx.x;
    const bool f = k < K && list[k] != 0;
    const unsigned b = __ballot_sync(0xffffffffu, f);
    if (lane == 0) wtot[warp] = __popc(b);
    __syncthreads();                  // every flag of this chunk is read before any index is written
    int off = 0, tot = 0;
    for (int w = 0; w < 32; ++w) {
      if (w < warp) off += wtot[w];
      tot += wtot[w];
    }
    if (f) list[base + off + __popc(b & ((1u << lane) - 1u))] = k;   // position <= k: never a flag still unread
    base += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = base;
}

int int8_quantize_act(const void* A, int64_t lda, int M, int K, float threshold, void* CA, void* SCA, int* outliers,
                      int* n_outliers, cudaStream_t stream) {
  if (lda == 0) lda = K;
  SB_REQUIRE(A && CA && SCA && outliers && n_outliers && M > 0 && K > 0 && lda >= K,
             "int8_quantize_act: bad arguments (M=%d K=%d lda=%lld)", M, K, (long long)lda);
  const __half* a = static_cast<const __half*>(A);
  SB_CHECK_CUDA(cudaMemsetAsync(outliers, 0, (size_t)K * sizeof(int), stream));
  int8_act_scan_kernel<<<M, 256, 0, stream>>>(a, lda, K, threshold, static_cast<float*>(SCA), outliers);
  SB_LAUNCH_CHECK();
  int8_act_quant_kernel<<<M, 256, 0, stream>>>(a, lda, K, static_cast<const float*>(SCA), outliers,
                                               static_cast<int8_t*>(CA));
  SB_LAUNCH_CHECK();
  int8_act_compact_kernel<<<1, 1024, 0, stream>>>(outliers, K, n_outliers);
  SB_LAUNCH_CHECK();
  return 0;
}

// ---- outlier correction of the GEMM path: corr[m,n] = fp16(sum_{t ascending} A[m,O_t] * subB[n,O_t]) ----
// A dense product over the gathered outlier columns: 64 x 64 outputs per CTA, 4 x 4 per thread, the columns staged
// 32 at a time in shared memory (A gathered from its outlier columns, subB = fp16(CB * SCB / 127) made on the way).
// Each output is one fp32 chain in ascending column order, so the result is the contract's bits.  Nothing is
// written when there are no outliers (the GEMM epilogue does not read corr then).
constexpr int CORR_T = 64, CORR_KC = 32;
__global__ void __launch_bounds__(256)
int8_correction_kernel(const __half* __restrict__ A, long long lda, const int8_t* __restrict__ W, long long ldw,
                       const float* __restrict__ SCB, const int* __restrict__ ol, const int* __restrict__ n_ol, int M,
                       int N, __half* __restrict__ corr, long long ldc) {
  const int cnt = *n_ol;
  if (cnt == 0) return;
  __shared__ float as[CORR_KC][CORR_T + 1], bs[CORR_KC][CORR_T + 1];
  __shared__ int js[CORR_KC];
  const int m0 = blockIdx.y * CORR_T, n0 = blockIdx.x * CORR_T;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  for (int c = 0; c < cnt; c += CORR_KC) {
    const int kc = min(CORR_KC, cnt - c);
    __syncthreads();
    if (threadIdx.x < kc) js[threadIdx.x] = ol[c + threadIdx.x];
    __syncthreads();
    for (int e = threadIdx.x; e < CORR_KC * CORR_T; e += 256) {
      const int t = e / CORR_T, r = e % CORR_T;
      float av = 0.0f, bv = 0.0f;
      if (t < kc) {
        const int j = js[t];
        if (m0 + r < M) av = __half2float(A[(long long)(m0 + r) * lda + j]);
        if (n0 + r < N) {
          const float sb = SCB[n0 + r];
          bv = __half2float(__float2half_rn((float)W[(long long)(n0 + r) * ldw + j] * sb / 127.0f));
        }
      }
      as[t][r] = av;
      bs[t][r] = bv;
    }
    __syncthreads();
    for (int t = 0; t < kc; ++t) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = as[t][ty + 16 * i]; b[i] = bs[t][tx + 16 * i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);   // exact products, ordered sums
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty + 16 * i, n = n0 + tx + 16 * j;
      if (m < M && n < N) corr[(long long)m * ldc + n] = __float2half_rn(acc[i][j]);
    }
}

int int8_correction(const void* A16, int64_t lda, const void* W, int64_t ldw, const void* SCB, const int* outliers,
                    const int* n_outliers, int M, int N, void* corr, cudaStream_t stream) {
  dim3 grid((N + CORR_T - 1) / CORR_T, (M + CORR_T - 1) / CORR_T);
  int8_correction_kernel<<<grid, 256, 0, stream>>>(static_cast<const __half*>(A16), lda, static_cast<const int8_t*>(W),
                                                   ldw, static_cast<const float*>(SCB), outliers, n_outliers, M, N,
                                                   static_cast<__half*>(corr), N);
  SB_LAUNCH_CHECK();
  return 0;
}

// ---- GEMV (M <= 4) ----
// Every CTA stages the M activation rows in shared memory (RMS-normalised as seedb200_gemv does when norm_w is
// given), finds the outlier columns and the row scales, quantises the rows, and builds the ascending outlier list.
// Then each warp owns a pair of weight rows, streams them with 16-byte ld.global.nc.L1::no_allocate loads and
// accumulates 4 int8 products per dp4a.  Shared memory: fp16 rows [M][K], int8 rows [M][K], flags [K], list [K]
// (uint16).
constexpr int GEMV8_U = 4;   // 16-byte vectors per weight row a lane keeps in flight

__device__ __forceinline__ uint4 ldw_na(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ int dot16(const uint4& w, const uint4& x, int acc) {
  acc = __dp4a((int)w.x, (int)x.x, acc);
  acc = __dp4a((int)w.y, (int)x.y, acc);
  acc = __dp4a((int)w.z, (int)x.z, acc);
  return __dp4a((int)w.w, (int)x.w, acc);
}

template <int M, int MODE, bool NORM>
__global__ void __launch_bounds__(256)
gemv_int8_kernel(const __half* __restrict__ x, const __half* __restrict__ norm_w, float eps, float thr,
                 const int8_t* __restrict__ W, const float* __restrict__ SCB, __half* __restrict__ out,
                 const __half* __restrict__ residual, int N, int K, int iters) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __half* xs = reinterpret_cast<__half*>(smem_raw);                            // [M][K]
  int8_t* cs = reinterpret_cast<int8_t*>(smem_raw + (size_t)M * K * 2);         // [M][K]
  uint8_t* flags = reinterpret_cast<uint8_t*>(smem_raw + (size_t)M * K * 3);    // [K]
  uint16_t* ol = reinterpret_cast<uint16_t*>(smem_raw + (size_t)M * K * 3 + ((K + 15) / 16) * 16);   // [K]
  __shared__ float red[8];
  __shared__ float sca[M];
  __shared__ int n_ol;
  const int nvec = K / 8, nv16 = K / 16;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5, nthr = blockDim.x;
  const int n_out = MODE == 1 ? N / 2 : N;
  const int n_tasks = MODE == 1 ? N / 2 : (N + 1) / 2;
  pdl_trigger();
  pdl_wait();
  uint4* xv = reinterpret_cast<uint4*>(xs);
  if constexpr (NORM) {    // seedb200_gemv's staging, operation for operation
#pragma unroll 1
    for (int m = 0; m < M; ++m) {
      float ss = 0.0f;
      for (int i = threadIdx.x; i < nvec; i += nthr) {
        const uint4 raw = reinterpret_cast<const uint4*>(x)[m * nvec + i];
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); ss += f.x * f.x; ss += f.y * f.y; }
      }
      ss = warp_sum(ss);
      __syncthreads();
      if (lane == 0) red[warp] = ss;
      __syncthreads();
      float tot = 0.0f;
      for (int i = 0; i < nw; ++i) tot += red[i];
      const float rstd = rsqrtf(tot * (1.0f / (float)K) + eps);
      for (int i = threadIdx.x; i < nvec; i += nthr) {
        const uint4 raw = reinterpret_cast<const uint4*>(x)[m * nvec + i];
        const uint4 wraw = __ldg(reinterpret_cast<const uint4*>(norm_w) + i);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        const __half* wh = reinterpret_cast<const __half*>(&wraw);
        uint4 o;
        __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const __half n16 = __float2half_rn(__half2float(h[j]) * rstd);
          oh[j] = __float2half_rn(__half2float(n16) * __half2float(wh[j]));
        }
        xv[m * nvec + i] = o;
      }
    }
  } else {
    for (int i = threadIdx.x; i < M * nvec; i += nthr) xv[i] = reinterpret_cast<const uint4*>(x)[i];
  }
  for (int k = threadIdx.x; k < K; k += nthr) flags[k] = 0;
  __syncthreads();
  // outlier columns and row scales
#pragma unroll 1
  for (int m = 0; m < M; ++m) {
    float mx = 0.0f;
    for (int k = threadIdx.x; k < K; k += nthr) {
      const float a = fabsf(__half2float(xs[m * K + k]));
      if (!(a < thr)) flags[k] = 1;
      else mx = fmaxf(mx, a);
    }
    mx = block_max_256(mx, red);
    if (threadIdx.x == 0) sca[m] = mx;
  }
  __syncthreads();
  // int8 rows; warp 0 also builds the ascending outlier list
#pragma unroll 1
  for (int m = 0; m < M; ++m) {
    const float s = sca[m], inv = 127.0f / s;
    for (int k = threadIdx.x; k < K; k += nthr)
      cs[m * K + k] = (flags[k] != 0 || s == 0.0f) ? (int8_t)0 : quant8(__half2float(xs[m * K + k]), inv);
  }
  if (warp == 0) {
    int base = 0;
    for (int c = 0; c < K; c += 32) {
      const bool f = c + lane < K && flags[c + lane] != 0;
      const unsigned b = __ballot_sync(0xffffffffu, f);
      if (f) ol[base + __popc(b & ((1u << lane) - 1u))] = (uint16_t)(c + lane);
      base += __popc(b);
    }
    if (lane == 0) n_ol = base;
  }
  __syncthreads();
  const int cnt = n_ol;
  const uint4* cv = reinterpret_cast<const uint4*>(cs);

  for (int it = 0; it < iters; ++it) {
    const int t = (blockIdx.x + it * gridDim.x) * nw + warp;
    if (t >= n_tasks) break;           // no barrier below this point
    long long r0, r1;
    if (MODE == 1) { r0 = (long long)(t / 128) * 256 + (t % 128); r1 = r0 + 128; }
    else { r0 = 2LL * t; r1 = min(r0 + 1, (long long)N - 1); }
    const uint4* w0 = reinterpret_cast<const uint4*>(W + r0 * K);
    const uint4* w1 = reinterpret_cast<const uint4*>(W + r1 * K);
    int a0[M], a1[M];
#pragma unroll
    for (int m = 0; m < M; ++m) { a0[m] = 0; a1[m] = 0; }
    for (int v = lane; v < nv16; v += 32 * GEMV8_U) {
      uint4 wa[GEMV8_U], wb[GEMV8_U];
#pragma unroll
      for (int u = 0; u < GEMV8_U; ++u) {
        const int vi = v + u * 32;
        if (vi < nv16) { wa[u] = ldw_na(w0 + vi); wb[u] = ldw_na(w1 + vi); }
      }
#pragma unroll
      for (int u = 0; u < GEMV8_U; ++u) {
        const int vi = v + u * 32;
        if (vi < nv16) {
#pragma unroll
          for (int m = 0; m < M; ++m) {
            const uint4 q = cv[m * nv16 + vi];
            a0[m] = dot16(wa[u], q, a0[m]);
            a1[m] = dot16(wb[u], q, a1[m]);
          }
        }
      }
    }
#pragma unroll
    for (int m = 0; m < M; ++m) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        a0[m] += __shfl_xor_sync(0xffffffffu, a0[m], o);
        a1[m] += __shfl_xor_sync(0xffffffffu, a1[m], o);
      }
    }
    // epilogue: the whole warp evaluates each output's outlier correction (int8_finish_warp), lane 0 stores
#pragma unroll
    for (int m = 0; m < M; ++m) {
      const __half* xrow = xs + m * K;
      if (MODE == 1) {
        const float sg = SCB[r0], su = SCB[r1];
        const __half g = int8_finish_warp(int8_base(a0[m], sca[m], sg), xrow, W + r0 * K, sg, ol, cnt, lane);
        const __half u = int8_finish_warp(int8_base(a1[m], sca[m], su), xrow, W + r1 * K, su, ol, cnt, lane);
        if (lane == 0) out[(long long)m * n_out + t] = int8_silu_mul(g, u);
      } else {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          if (r == 1 && r1 == r0) continue;
          const long long n = r == 0 ? r0 : r1;
          const float sb = SCB[n];
          __half y = int8_finish_warp(int8_base(r == 0 ? a0[m] : a1[m], sca[m], sb), xrow, W + n * K, sb, ol, cnt,
                                      lane);
          if (lane == 0) {
            if (residual != nullptr) y = __float2half_rn(__half2float(y) + __half2float(residual[(long long)m * n_out + n]));
            out[(long long)m * n_out + n] = y;
          }
        }
      }
    }
  }
}

int gemv_int8(const void* x, const void* norm_w, float eps, float threshold, const void* W, const void* SCB, void* out,
              const void* residual, int M, int N, int K, int mode, cudaStream_t stream) {
  SB_REQUIRE(x && W && SCB && out, "gemv_int8: null operand");
  SB_REQUIRE(M >= 1 && M <= 4, "gemv_int8: M=%d outside [1,4]", M);
  SB_REQUIRE(N > 0 && K > 0 && K % 16 == 0 && K <= 65536, "gemv_int8: K=%d must be a positive multiple of 16 (<= 65536)", K);
  SB_REQUIRE(mode == 0 || (mode == 1 && N % 256 == 0 && residual == nullptr), "gemv_int8: bad mode/shape");
  const size_t smem = (size_t)M * K * 3 + (size_t)((K + 15) / 16) * 16 + (size_t)K * 2;
  SB_REQUIRE(smem <= 220 * 1024, "gemv_int8: activation rows do not fit shared memory (M=%d K=%d)", M, K);
  const int n_tasks = mode == 1 ? N / 2 : (N + 1) / 2;
  const __half* xp = static_cast<const __half*>(x);
  const __half* np = static_cast<const __half*>(norm_w);
  const int8_t* wp = static_cast<const int8_t*>(W);
  const float* sp = static_cast<const float*>(SCB);
  __half* op = static_cast<__half*>(out);
  const __half* rp = static_cast<const __half*>(residual);
#define SB_GEMV8_LAUNCH(M_, MD_, NM_)                                                                       \
  {                                                                                                         \
    auto kern = gemv_int8_kernel<M_, MD_, NM_>;                                                             \
    const int threads = 256;                                                                                \
    static size_t attr_smem_dev[SB_MAX_DEVICES] = {};                                                      \
    const int dev_ = cur_device();                                                                          \
    size_t& attr_smem = attr_smem_dev[dev_];                                                                \
    if (attr_smem == 0) attr_smem = 48 * 1024;                                                              \
    if (smem > attr_smem) {                                                                                 \
      SB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
      attr_smem = smem;                                                                                     \
    }                                                                                                       \
    int occ = 0;                                                                                            \
    SB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));                \
    if (occ < 1) occ = 1;                                                                                   \
    const int tpi = threads / 32;                                                                           \
    int blocks = (n_tasks + tpi - 1) / tpi;                                                                 \
    if (blocks > num_sms() * occ) blocks = num_sms() * occ;                                                 \
    const int iters = (n_tasks + blocks * tpi - 1) / (blocks * tpi);                                        \
    SB_CHECK_CUDA(launch_chain(kern, dim3(blocks), dim3(threads), smem, stream, xp, np, eps, threshold, wp, sp, op, \
                               rp, N, K, iters));                                                           \
    SB_LAUNCH_CHECK();                                                                                      \
    return 0;                                                                                               \
  }
#define SB_GEMV8(M_, MD_)                                                                                   \
  if (M == M_ && mode == MD_) {                                                                             \
    if (norm_w != nullptr) SB_GEMV8_LAUNCH(M_, MD_, true)                                                   \
    SB_GEMV8_LAUNCH(M_, MD_, false)                                                                         \
  }
  SB_GEMV8(1, 0) SB_GEMV8(2, 0) SB_GEMV8(3, 0) SB_GEMV8(4, 0)
  SB_GEMV8(1, 1) SB_GEMV8(2, 1) SB_GEMV8(3, 1) SB_GEMV8(4, 1)
#undef SB_GEMV8
#undef SB_GEMV8_LAUNCH
  set_error("gemv_int8: unsupported configuration");
  return SEEDB200_ERR_UNSUPPORTED;
}

}  // namespace sb

extern "C" {

int seedb200_int8_quantize_weight(const void* W, int64_t ldw, int N, int K, void* CB, void* SCB, void* stream) {
  return sb::int8_quantize_weight(W, ldw, N, K, CB, SCB, static_cast<cudaStream_t>(stream));
}

int seedb200_int8_quantize_act(const void* A, int64_t lda, int M, int K, float threshold, void* CA, void* SCA,
                               int32_t* outliers, int32_t* n_outliers, void* stream) {
  return sb::int8_quantize_act(A, lda, M, K, threshold, CA, SCA, outliers, n_outliers,
                               static_cast<cudaStream_t>(stream));
}

int seedb200_gemv_int8(const void* x, const void* norm_w, float eps, float threshold, const void* W, const void* SCB,
                       void* out, const void* residual, int M, int N, int K, int mode, void* stream) {
  return sb::gemv_int8(x, norm_w, eps, threshold, W, SCB, out, residual, M, N, K, mode,
                       static_cast<cudaStream_t>(stream));
}

}  // extern "C"
