// misc.cu -- small-M kernels of the LLaMA decode step (HBM-bound: every weight byte is read once per
// token, llama_xformer.py:745-776 generation loop) and a row-wise add used at handle creation.
//   gemv              y[m,:] = x[m,:] . W^T for m <= 4 rows: the batch-1 decode form of every nn.Linear in
//                     LlamaDecoderLayer (llama_xformer.py:186,223-225,258) and lm_head (:718)
//   decode_attention  one query token against the KV cache (llama_xformer.py:240-256 with attn_bias=None),
//                     split over the key axis so that B*H*splits CTAs cover the SMs
#include <type_traits>

#include "common.cuh"
#include "ops.h"
#include "quant4.cuh"

namespace sb {

int get_option(const char* key);

__global__ void add_rows_kernel(const __half* a, const __half* b, __half* out, int rows, int cols, int b_rows) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)rows * cols) return;
  const int r = (int)(i / cols), c = (int)(i % cols);
  out[i] = __float2half_rn(__half2float(a[i]) + __half2float(b[(long long)(r % b_rows) * cols + c]));
}

int add_rows(const void* a, const void* b, void* out, int rows, int cols, int b_rows, cudaStream_t stream) {
  const long long n = (long long)rows * cols;
  add_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(static_cast<const __half*>(a),
                                                                  static_cast<const __half*>(b),
                                                                  static_cast<__half*>(out), rows, cols, b_rows);
  SB_LAUNCH_CHECK();
  return 0;
}

// ----------------------------------------------------------------------------
// GEMV (M <= 4 activation rows): the batch-1 decode form of every nn.Linear.  HBM-bound: every weight byte is
// read exactly once.  Each warp owns a PAIR of weight rows and streams both with 16-byte loads (2 rows x 4
// vectors = 128 bytes in flight per lane; one row per warp left the HBM pipe half empty: 4.4 vs 6.4 TB/s).  The
// first batch of weight loads is issued before the activations are staged (weights do not depend on them).
// mode 0: rows (2t, 2t+1) -> out[m, 2t], out[m, 2t+1] (+ residual).
// mode 1: W rows are [128 gate | 128 up] blocks and out[m,j] = silu(gate_j) * up_j (same rounding points
// as the GEMM epilogue, llama_xformer.py:186).
// NORM: the staged activations are RMS-normalised on the way into shared memory (LlamaRMSNorm,
// llama_xformer.py:105-113: fp32 x * rsqrt(mean(x^2) + eps) -> fp16 -> * weight -> fp16), which removes the
// separate norm launch in front of the QKV and gate/up projections of the decode step.
// (A variant that staged the weights through per-warp rings of 1-D cp.async.bulk copies was measured at
// ~17 B/clk/SM -- 5.0 TB/s chip-wide regardless of ring depth -- and dropped: profiles/r01_summary.md.)
// ----------------------------------------------------------------------------
constexpr int GEMV_MAXM = 4;

__device__ __forceinline__ void dot8(const uint4& w, const uint4& x, float& acc) {
  const __half2* wh = reinterpret_cast<const __half2*>(&w);
  const __half2* xh = reinterpret_cast<const __half2*>(&x);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 a = __half22float2(wh[j]), b = __half22float2(xh[j]);
    acc = fmaf(a.x, b.x, acc);
    acc = fmaf(a.y, b.y, acc);
  }
}

// U: 16-byte vectors per weight row a lane keeps in flight (4 = 128 bytes per lane).  Measured and dropped (r02,
// profiles/r02_decode_ab.json): U = 8 on 128-thread CTAs for the short-N projections (4.98 -> 5.37 ms/token) and a cap on
// the CTAs per SM so that the next kernel of the programmatic-launch chain is co-resident early (5.08 / 6.13 ms/token).
// NA: the weight stream is loaded with ld.global.nc.L1::no_allocate -- every weight byte is used exactly once, so it should
// not displace anything in L1 on its way through (13B decode step 4.87 -> 4.80 ms/token; an added L2::256B prefetch-size hint
// and 256-bit ld.global.v8.b32 loads measured equal or slower, profiles/r02_gemv_load_policy_ab.txt)
template <bool NA>
__device__ __forceinline__ uint4 gemv_ldw(const uint4* p) {
  if constexpr (!NA) {
    return __ldg(p);
  } else {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p));
    return v;
  }
}
template <bool NA>
__device__ __forceinline__ uint32_t gemv_ldw(const uint32_t* p) {
  if constexpr (!NA) {
    return __ldg(p);
  } else {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
  }
}

// WF: the weight format.  0 = fp16 W [N, ldw halves], one 16-byte vector per group of 8 weights.  1 + quant type
// (SEEDB200_Q4_FP4 / SEEDB200_Q4_NF4) = bitsandbytes 4-bit codes [N, ldw bytes] with absmax [N, K/64]: 4 packed
// bytes per group, dequantised in registers to the halves the fp16 GEMV would read from dequantize_4bit(W) and then
// summed exactly like them (same lane -> group mapping, same dot8 order), so the output is bit-identical.
template <int WF>
using GemvVec = std::conditional_t<WF == 0, uint4, uint32_t>;
template <int WF>
constexpr int kGemvVecsPerLine = WF == 0 ? 8 : 32;     // vectors per 128-byte line

template <int WF>
__device__ __forceinline__ const GemvVec<WF>* gemv_row(const __half* W, long long r, long long ldw) {
  if constexpr (WF == 0) return reinterpret_cast<const uint4*>(W + r * ldw);
  else return reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint8_t*>(W) + r * ldw);
}

// the dequantisation table of a 4-bit instantiation (the fp16 ones declare no shared table)
template <int WF>
__device__ __forceinline__ float* gemv_q4_table() {
  __shared__ float tab[16];
  return tab;
}

template <int WF>
__device__ __forceinline__ uint4 gemv_wvec(const GemvVec<WF>& w, float absmax, const float* tab) {
  if constexpr (WF == 0) return w;
  else return q4_deq8(w, absmax, tab);
}

// LORA: the LoRA expand of include/seedb200.h in the epilogue (lo.T staged in shared memory; ksplit must be 1).  Lane
// 2 m + i of the warp that owns a row pair finishes output row r_i of activation row m: y = fp16(fp16(acc) + c), then
// the residual add or (mode 1, gate and up exchanged between the two lanes) the SiLU gate.  Without LORA the code is
// the plain GEMV.
template <int M, int MODE, bool NORM, int U, bool NA, bool LORA, int WF>
__global__ void __launch_bounds__(256)
gemv_kernel(const __half* __restrict__ x, const __half* __restrict__ W, long long ldw, __half* __restrict__ out,
            const __half* __restrict__ residual, const __half* __restrict__ norm_w, float eps, int N, int K,
            int ksplit, int iters, long long ldo, int pf_lines, seedb200_lora_operand lo,
            const float* __restrict__ absmax) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float lts[LORA ? M * LORA_MAX_RTOT : 1];
  uint4* xs = reinterpret_cast<uint4*>(smem_raw);     // [M][K/8]
  __shared__ float red[8];
  __shared__ float part[2][8][M][2];                  // [iteration parity][warp][row m][row of the pair]
  const int nvec = K / 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_out = (MODE == 1) ? N / 2 : N;
  const int n_tasks = (MODE == 1) ? N / 2 : (N + 1) / 2;
  // the 8 warps of a CTA work on 8/ksplit row pairs at a time; warp = (pair, K slice).  Short-N projections
  // (o_proj, down_proj: 2560 row pairs for ~3500 resident warps) would otherwise be one long dependent chain of
  // load batches per warp.
  const int nw = blockDim.x >> 5, nthr = blockDim.x;
  const int tpi = nw / ksplit;                        // row pairs per CTA iteration
  const int slice = warp % ksplit, tin = warp / ksplit;
  const int vps = (((nvec + ksplit - 1) / ksplit) + 31) / 32 * 32;
  const int v0 = slice * vps, v1 = min(nvec, v0 + vps);
  auto rows_of = [&](int t, long long& r0, long long& r1) {
    if (MODE == 1) { r0 = (long long)(t / 128) * 256 + (t % 128); r1 = r0 + 128; }
    else { r0 = 2LL * t; r1 = min(r0 + 1, (long long)N - 1); }
  };
  const int nblk = K / Q4_BLOCK;                      // 4-bit: absmax entries per row
  // first batch of this warp's first task: in flight while the activations are staged
  GemvVec<WF> wa[U], wb[U];
  float sa[WF ? U : 1], sb[WF ? U : 1];               // 4-bit: absmax of each vector's block
  const int t_first = blockIdx.x * tpi + tin;
  if (t_first < n_tasks) {
    long long r0, r1;
    rows_of(t_first, r0, r1);
    const GemvVec<WF>* w0 = gemv_row<WF>(W, r0, ldw);
    const GemvVec<WF>* w1 = gemv_row<WF>(W, r1, ldw);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int vi = v0 + lane + u * 32;
      if (vi < v1) {
        wa[u] = gemv_ldw<NA>(w0 + vi); wb[u] = gemv_ldw<NA>(w1 + vi);
        if constexpr (WF != 0) { sa[u] = __ldg(absmax + r0 * nblk + vi / 8); sb[u] = __ldg(absmax + r1 * nblk + vi / 8); }
      }
    }
    // ... and the next pf_lines 128-byte lines of both rows go to L2: with programmatic dependent launch this CTA is
    // resident long before its predecessor has finished, and the dependency wait + activation staging below would
    // otherwise leave HBM idle (weights never depend on the predecessor).  Sized by the host to ~24 MB per launch.
    for (int l = lane; l < pf_lines; l += 32) {
      const int vi = v0 + 32 * U + l * kGemvVecsPerLine<WF>;
      if (vi < v1) { prefetch_l2(w0 + vi); prefetch_l2(w1 + vi); }
    }
  }
  pdl_trigger();
  pdl_wait();
  if constexpr (NORM) {
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
        xs[m * nvec + i] = o;
      }
    }
  } else {
    for (int i = threadIdx.x; i < M * nvec; i += nthr) xs[i] = reinterpret_cast<const uint4*>(x)[i];
  }
  if constexpr (WF != 0) {
    if (threadIdx.x < 16) gemv_q4_table<WF>()[threadIdx.x] = kQ4Value[WF - 1][threadIdx.x];
  }
  if constexpr (LORA) {
    const int rt = lo.r * lo.nsub;
    for (int i = threadIdx.x; i < M * rt; i += nthr)
      lts[(i / rt) * LORA_MAX_RTOT + i % rt] = __half2float(static_cast<const __half*>(lo.T)[(long long)(i / rt) * lo.ldt + i % rt]);
  }
  __syncthreads();

  for (int it = 0; it < iters; ++it) {                // trip count is uniform over the CTA (barriers inside)
    const int t = (blockIdx.x + it * gridDim.x) * tpi + tin;
    const bool valid = t < n_tasks;
    long long r0 = 0, r1 = 0;
    float a0[M], a1[M];
#pragma unroll
    for (int m = 0; m < M; ++m) { a0[m] = 0.0f; a1[m] = 0.0f; }
    if (valid) {
      rows_of(t, r0, r1);
      const GemvVec<WF>* w0 = gemv_row<WF>(W, r0, ldw);
      const GemvVec<WF>* w1 = gemv_row<WF>(W, r1, ldw);
      for (int v = v0 + lane; v < v1; v += 32 * U) {
        if (it != 0 || v != v0 + lane) {    // the very first batch is already in registers
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int vi = v + u * 32;
            if (vi < v1) {
              wa[u] = gemv_ldw<NA>(w0 + vi); wb[u] = gemv_ldw<NA>(w1 + vi);
              if constexpr (WF != 0) {
                sa[u] = __ldg(absmax + r0 * nblk + vi / 8); sb[u] = __ldg(absmax + r1 * nblk + vi / 8);
              }
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int vi = v + u * 32;
          if (vi < v1) {
            const float* tab = nullptr;
            if constexpr (WF != 0) tab = gemv_q4_table<WF>();
            const uint4 da = gemv_wvec<WF>(wa[u], sa[WF ? u : 0], tab);
            const uint4 db = gemv_wvec<WF>(wb[u], sb[WF ? u : 0], tab);
#pragma unroll
            for (int m = 0; m < M; ++m) {
              const uint4 xv = xs[m * nvec + vi];
              dot8(da, xv, a0[m]);
              dot8(db, xv, a1[m]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int m = 0; m < M; ++m) {
      a0[m] = warp_sum(a0[m]);
      a1[m] = warp_sum(a1[m]);
    }
    if (ksplit > 1) {
      // fold the K slices in slice order (deterministic); double-buffered so one barrier per iteration is enough
      if (lane == 0) {
#pragma unroll
        for (int m = 0; m < M; ++m) { part[it & 1][warp][m][0] = a0[m]; part[it & 1][warp][m][1] = a1[m]; }
      }
      __syncthreads();
      if (slice == 0 && lane == 0) {
#pragma unroll
        for (int m = 0; m < M; ++m) {
          float s0 = 0.0f, s1 = 0.0f;
          for (int k = 0; k < ksplit; ++k) { s0 += part[it & 1][warp + k][m][0]; s1 += part[it & 1][warp + k][m][1]; }
          a0[m] = s0; a1[m] = s1;
        }
      }
    }
    if constexpr (LORA) {
      if (valid) {                                     // warp-uniform; every lane holds the warp sums (ksplit == 1)
        const int m = lane < 2 * M ? lane >> 1 : 0, which = lane & 1;
        float acc = 0.0f;
#pragma unroll
        for (int mm = 0; mm < M; ++mm)
          if (mm == m) acc = which ? a1[mm] : a0[mm];
        const long long rr = which ? r1 : r0;
        __half y = __float2half_rn(acc);
        const int sub = (int)((rr / lo.grp) % lo.nsub);
        if ((lo.mask >> sub) & 1u) {
          const __half* brow = static_cast<const __half*>(lo.B) + rr * lo.r;
          const float* tr = lts + m * LORA_MAX_RTOT + sub * lo.r;
          float ua = 0.0f;
          for (int j = 0; j < lo.r; ++j) ua = fmaf(__half2float(brow[j]), tr[j], ua);
          const __half c = __float2half_rn(__half2float(__float2half_rn(ua)) * lo.scale);
          y = __float2half_rn(__half2float(y) + __half2float(c));
        }
        if (MODE == 1) {
          const float yf = __half2float(y), other = __shfl_xor_sync(0xffffffffu, yf, 1);
          if (lane < 2 * M && which == 0) {
            const float sg = __half2float(__float2half_rn(yf / (1.0f + __expf(-yf))));
            out[(long long)m * ldo + t] = __float2half_rn(sg * other);
          }
        } else if (lane < 2 * M && (which == 0 || r1 != r0)) {
          if (residual != nullptr) y = __float2half_rn(__half2float(y) + __half2float(residual[(long long)m * n_out + rr]));
          out[(long long)m * ldo + rr] = y;
        }
      }
    } else if (valid && slice == 0 && lane == 0) {
#pragma unroll
      for (int m = 0; m < M; ++m) {
        if (MODE == 1) {
          const float g = __half2float(__float2half_rn(a0[m]));
          const float u = __half2float(__float2half_rn(a1[m]));
          const float s = __half2float(__float2half_rn(g / (1.0f + __expf(-g))));
          out[(long long)m * ldo + t] = __float2half_rn(s * u);
        } else {
          __half h0 = __float2half_rn(a0[m]), h1 = __float2half_rn(a1[m]);
          if (residual != nullptr) {
            h0 = __float2half_rn(__half2float(h0) + __half2float(residual[(long long)m * n_out + r0]));
            h1 = __float2half_rn(__half2float(h1) + __half2float(residual[(long long)m * n_out + r1]));
          }
          out[(long long)m * ldo + r0] = h0;
          if (r1 != r0) out[(long long)m * ldo + r1] = h1;
        }
      }
    }
  }
}

// U of the 4-bit instantiations: 16 groups per row in flight (64 bytes of codes per lane and row, the fp16 GEMV's
// bytes in flight per lane); -Xptxas -v shows no spills
constexpr int GEMV_U_Q4 = 16;

// WF as in gemv_kernel; 4-bit: W = packed codes (ldw in bytes), absmax, no LoRA, no-allocate weight loads
template <int WF>
static int gemv_impl(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w,
                     float eps, int M, int N, int K, int mode, cudaStream_t stream, int64_t ldo,
                     const seedb200_lora_operand* lora, const float* absmax) {
  if (ldo <= 0) ldo = mode == 1 ? N / 2 : N;
  seedb200_lora_operand lo;
  memset(&lo, 0, sizeof(lo));
  if (lora != nullptr) {
    lo = *lora;
    SB_REQUIRE(lo.T && lo.B && lo.r >= 1 && lo.r <= LORA_MAX_R && lo.nsub >= 1 && lo.nsub <= 3 && lo.grp >= 1 &&
                   lo.ldt >= (int64_t)lo.r * lo.nsub,
               "gemv: bad LoRA operand (r %d, nsub %d, grp %d, ldt %lld)", lo.r, lo.nsub, lo.grp, (long long)lo.ldt);
  }
  SB_REQUIRE(M >= 1 && M <= GEMV_MAXM, "gemv: M=%d outside [1,%d]", M, GEMV_MAXM);
  SB_REQUIRE(K % 8 == 0 && ldw % 8 == 0, "gemv: K and ldw must be multiples of 8");
  SB_REQUIRE(aligned16(x) && aligned16(W) && (norm_w == nullptr || aligned16(norm_w)),
             "gemv: x, W and norm_w must be 16-byte aligned");
  SB_REQUIRE(mode == 0 || (mode == 1 && N % 256 == 0 && residual == nullptr), "gemv: bad mode/shape");
  if constexpr (WF != 0) SB_REQUIRE(lora == nullptr && absmax != nullptr, "gemv_4bit: bad operands");
  const size_t smem = (size_t)M * K * 2;
  SB_REQUIRE(smem <= 200 * 1024, "gemv: activation rows do not fit shared memory (M=%d K=%d)", M, K);
  const int n_tasks = mode == 1 ? N / 2 : (N + 1) / 2;
  const int force_split = get_option("gemv_ksplit");
  const bool no_alloc = get_option("gemv_no_allocate") != 0;
  const __half* xp = static_cast<const __half*>(x);
  const __half* wp = static_cast<const __half*>(W);
  const __half* rp = static_cast<const __half*>(residual);
  const __half* np = static_cast<const __half*>(norm_w);
  __half* op = static_cast<__half*>(out);
#define SB_GEMV_LAUNCH(M_, MD_, NM_, U_, NA_, LO_)                                                         \
  {                                                                                                        \
    auto kern = gemv_kernel<M_, MD_, NM_, U_, NA_, LO_, WF>;                                               \
    const int threads = 256;                                                                               \
    static size_t attr_smem_dev[SB_MAX_DEVICES] = {};   /* per device: cudaFuncSetAttribute is */          \
    const int dev_ = cur_device();                                                                         \
    size_t& attr_smem = attr_smem_dev[dev_];                                                               \
    if (attr_smem == 0) attr_smem = 48 * 1024;                                                             \
    if (smem > attr_smem) {                                                                                \
      SB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
      attr_smem = smem;                                                                                    \
    }                                                                                                      \
    /* one full wave: grid = SMs x resident CTAs (a partial second wave costs a whole task time) */        \
    static int occ_dev[SB_MAX_DEVICES] = {}; static size_t occ_smem_dev[SB_MAX_DEVICES] = {};              \
    int& occ = occ_dev[dev_]; size_t& occ_smem = occ_smem_dev[dev_];                                       \
    if (occ == 0) occ_smem = (size_t)-1;                                                                   \
    if (occ_smem != smem) {                                                                                \
      SB_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));             \
      occ_smem = smem;                                                                                     \
      if (occ < 1) occ = 1;                                                                                \
    }                                                                                                      \
    const int resident = num_sms() * occ;                                                                  \
    /* K can be split over 2 or 4 warps per row pair (option gemv_ksplit); measured on the 13B decode step it  */ \
    /* loses (5.19 ms/token unsplit, 5.44 / 5.62 with 2 / 4 slices), so the default stays one warp per pair */ \
    int ksplit = 1;                                                                                        \
    if (!(LO_) && (force_split == 1 || force_split == 2 || force_split == 4)) ksplit = force_split;        \
    const int tpi = (threads / 32) / ksplit;                                                               \
    int blocks = (n_tasks + tpi - 1) / tpi;                                                                \
    if (blocks > resident) blocks = resident;                                                              \
    const int iters = (n_tasks + blocks * tpi - 1) / (blocks * tpi);                                       \
    /* L2 prefetch ahead of the dependency wait: ~24 MB per launch, spread over the tasks' first lines */    \
    int pf_lines = get_option("gemv_prefetch_mb") > 0                                                       \
                       ? (int)(((long long)get_option("gemv_prefetch_mb") << 20) / (2LL * n_tasks * 128)) : 0; \
    const int row_bytes = WF ? K / 2 : K * 2;                                                              \
    if (pf_lines > (row_bytes / ksplit) / 128) pf_lines = (row_bytes / ksplit) / 128;                       \
    SB_CHECK_CUDA(launch_chain(kern, dim3(blocks), dim3(threads), smem, stream, xp, wp, (long long)ldw, op, rp, np, eps, N, K, \
                               ksplit, iters, (long long)ldo, pf_lines, lo, absmax));                      \
    SB_LAUNCH_CHECK();                                                                                     \
    return 0;                                                                                              \
  }
#define SB_GEMV(M_, MD_)                                                                                   \
  if (M == M_ && mode == MD_) {                                                                            \
    if constexpr (WF != 0) {                                                                               \
      if (norm_w != nullptr) SB_GEMV_LAUNCH(M_, MD_, true, GEMV_U_Q4, true, false)                         \
      SB_GEMV_LAUNCH(M_, MD_, false, GEMV_U_Q4, true, false)                                               \
    } else {                                                                                               \
      if (lora != nullptr) {                                                                               \
        if (norm_w != nullptr) SB_GEMV_LAUNCH(M_, MD_, true, 4, true, true)                                \
        SB_GEMV_LAUNCH(M_, MD_, false, 4, true, true)                                                      \
      }                                                                                                    \
      if (no_alloc) {                                                                                      \
        if (norm_w != nullptr) SB_GEMV_LAUNCH(M_, MD_, true, 4, true, false)                               \
        SB_GEMV_LAUNCH(M_, MD_, false, 4, true, false)                                                     \
      }                                                                                                    \
      if (norm_w != nullptr) SB_GEMV_LAUNCH(M_, MD_, true, 4, false, false)                                \
      SB_GEMV_LAUNCH(M_, MD_, false, 4, false, false)                                                      \
    }                                                                                                      \
  }
  SB_GEMV(1, 0) SB_GEMV(2, 0) SB_GEMV(3, 0) SB_GEMV(4, 0)
  SB_GEMV(1, 1) SB_GEMV(2, 1) SB_GEMV(3, 1) SB_GEMV(4, 1)
#undef SB_GEMV
#undef SB_GEMV_LAUNCH
  set_error("gemv: unsupported configuration");
  return SEEDB200_ERR_UNSUPPORTED;
}

int gemv(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w, float eps,
         int M, int N, int K, int mode, cudaStream_t stream, int64_t ldo, const seedb200_lora_operand* lora) {
  return gemv_impl<0>(x, W, ldw, out, residual, norm_w, eps, M, N, K, mode, stream, ldo, lora, nullptr);
}

int gemv_4bit(const void* x, const void* norm_w, float eps, const void* packed, const float* absmax, int type,
              void* out, const void* residual, int M, int N, int K, int mode, cudaStream_t stream) {
  SB_PROPAGATE(q4_check("gemv_4bit", type, N, K));
  SB_REQUIRE(x && packed && absmax && out, "gemv_4bit: null operand");
  SB_REQUIRE((reinterpret_cast<uintptr_t>(packed) & 15) == 0, "gemv_4bit: packed codes must be 16-byte aligned");
  if (type == SEEDB200_Q4_FP4)
    return gemv_impl<1 + SEEDB200_Q4_FP4>(x, packed, K / 2, out, residual, norm_w, eps, M, N, K, mode, stream, 0,
                                          nullptr, absmax);
  return gemv_impl<1 + SEEDB200_Q4_NF4>(x, packed, K / 2, out, residual, norm_w, eps, M, N, K, mode, stream, 0,
                                        nullptr, absmax);
}

// ----------------------------------------------------------------------------
// Decode attention: q [B,H,D] (one token), caches [B,H,max_seq,D], D = 128.
// Kernel 1: CTA (split, h, b) of 128 threads walks its keys in blocks of 128.  Scores: one key per thread (the
// whole 256-byte K row in 16 independent 16-byte loads, q broadcast from shared memory -- no shuffles and one
// memory latency per block instead of one per key).  P.V: thread (g, c) = (key group of 8, 16-byte dim chunk)
// loads its 16 V vectors up front, then the 8 key groups are folded through shared memory.  Online softmax
// across blocks; partial (m, l, o[128]) per split.
// Kernel 2: merge the splits.
// ----------------------------------------------------------------------------
constexpr int DA_D = 128;
constexpr int DA_BLK = 128;
constexpr int DA_MAX_SPLITS = 64;

// key-axis split of a cache of kv_len keys: whole 128-key blocks per split, at most DA_MAX_SPLITS, no empty split
__host__ __device__ inline void da_split(int kv_len, int& nsplit, int& chunk) {
  nsplit = (kv_len + DA_BLK - 1) / DA_BLK;
  if (nsplit > DA_MAX_SPLITS) nsplit = DA_MAX_SPLITS;
  chunk = ((kv_len + nsplit - 1) / nsplit + DA_BLK - 1) / DA_BLK * DA_BLK;
  nsplit = (kv_len + chunk - 1) / chunk;
}

// Lineage (LIN): cached key / value p of row b is read from row slot[b * max_seq + p] of the caches instead of row b
// (beam search: beams share the prefix they inherited without copying it).  Only the addresses change.
template <bool LIN>
__device__ __forceinline__ long long da_row(const int* __restrict__ slot, long long base, int b, int H, int h,
                                            int max_seq, int p) {
  if (!LIN) return base + (long long)p * DA_D;
  const long long r = slot[(long long)b * max_seq + p];
  return ((r * H + h) * max_seq + p) * DA_D;
}

template <bool LIN>
__global__ void __launch_bounds__(128)
decode_attn_partial(const __half* __restrict__ q, const __half* __restrict__ kc, const __half* __restrict__ vc,
                    float* __restrict__ ws, int H, int kv_len, int max_seq, int chunk, float scale_log2,
                    const int* __restrict__ dyn, int* __restrict__ tickets, __half* __restrict__ out,
                    const int* __restrict__ slot) {
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  int nsplit = gridDim.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  __shared__ __align__(16) float s_q[DA_D];
  __shared__ float s_p[DA_BLK];
  __shared__ float s_red[2][4];
  __shared__ __align__(16) float s_o[8][DA_D];
  pdl_trigger();
  pdl_wait();
  if (dyn != nullptr) {
    // graph-replayed decode step: the cache length lives in device memory (dyn[0] = tokens already cached, this
    // step's token has just been appended); the grid was sized for max_seq keys, surplus splits exit.  Clamped to
    // the cache like the append kernels clamp their row.
    kv_len = min(dyn[0] + 1, max_seq);
    da_split(kv_len, nsplit, chunk);
    if (split >= nsplit) return;
  }
  s_q[tid] = __half2float(q[((long long)b * H + h) * DA_D + tid]);
  const long long base = ((long long)b * H + h) * max_seq * DA_D;
  const int k0 = split * chunk, k1 = min(kv_len, k0 + chunk);
  const int g = tid >> 4, c = tid & 15;            // P.V role: key group (8 groups), 8-dim chunk
  float m_run = -INFINITY, l_run = 0.0f, o_run = 0.0f;     // o_run: dim `tid`
  __syncthreads();
  for (int kb = k0; kb < k1; kb += DA_BLK) {
    const int cnt = min(DA_BLK, k1 - kb);
    // V vectors of this thread: keys g, g+8, ... (16 of them), dims c*8..c*8+7 -- issued before the score math
    uint4 vv[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int t = g + 8 * i;
      vv[i] = t < cnt ? __ldg(reinterpret_cast<const uint4*>(vc + da_row<LIN>(slot, base, b, H, h, max_seq, kb + t)) + c)
                      : make_uint4(0, 0, 0, 0);
    }
    float s = -INFINITY;
    if (tid < cnt) {
      const uint4* kr = reinterpret_cast<const uint4*>(kc + da_row<LIN>(slot, base, b, H, h, max_seq, kb + tid));
      uint4 kk[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) kk[i] = __ldg(kr + i);
      float acc = 0.0f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 qa = *reinterpret_cast<const float4*>(s_q + i * 8);
        const float4 qb = *reinterpret_cast<const float4*>(s_q + i * 8 + 4);
        const __half2* kh = reinterpret_cast<const __half2*>(&kk[i]);
        const float2 f0 = __half22float2(kh[0]), f1 = __half22float2(kh[1]);
        const float2 f2 = __half22float2(kh[2]), f3 = __half22float2(kh[3]);
        acc = fmaf(qa.x, f0.x, acc); acc = fmaf(qa.y, f0.y, acc); acc = fmaf(qa.z, f1.x, acc); acc = fmaf(qa.w, f1.y, acc);
        acc = fmaf(qb.x, f2.x, acc); acc = fmaf(qb.y, f2.y, acc); acc = fmaf(qb.z, f3.x, acc); acc = fmaf(qb.w, f3.y, acc);
      }
      s = acc * scale_log2;
    }
    const float wm = warp_max(s);
    if (lane == 0) s_red[0][warp] = wm;
    __syncthreads();
    const float bm = fmaxf(fmaxf(s_red[0][0], s_red[0][1]), fmaxf(s_red[0][2], s_red[0][3]));
    const float m_new = fmaxf(m_run, bm);                   // finite: every block has at least one key
    const float corr = exp2f(m_run - m_new);                // 0 on the first block
    const float p = exp2f(s - m_new);                       // 0 for absent keys
    s_p[tid] = p;
    const float ws_ = warp_sum(p);
    if (lane == 0) s_red[1][warp] = ws_;
    __syncthreads();
    l_run = l_run * corr + (s_red[1][0] + s_red[1][1] + s_red[1][2] + s_red[1][3]);
    m_run = m_new;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float pk = s_p[g + 8 * i];
      const __half2* vh = reinterpret_cast<const __half2*>(&vv[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(vh[j]);
        acc[2 * j] = fmaf(pk, f.x, acc[2 * j]);
        acc[2 * j + 1] = fmaf(pk, f.y, acc[2 * j + 1]);
      }
    }
    *reinterpret_cast<float4*>(&s_o[g][c * 8]) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(&s_o[g][c * 8 + 4]) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    __syncthreads();
    float od = 0.0f;
#pragma unroll
    for (int gg = 0; gg < 8; ++gg) od += s_o[gg][tid];
    o_run = o_run * corr + od;
    __syncthreads();                                        // s_p / s_o / s_red are rewritten by the next block
  }
  float* dst = ws + (((long long)b * H + h) * nsplit + split) * (DA_D + 2);
  if (tid == 0) { dst[0] = m_run; dst[1] = l_run; }
  dst[2 + tid] = o_run;
  if (tickets == nullptr) return;              // two-kernel form: decode_attn_merge follows
  // fused merge: the split that finishes last for this (b, h) combines all of them (one launch less per layer)
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int t = atomicAdd(&tickets[b * H + h], 1);
    s_last = (t == nsplit - 1);
    if (s_last) tickets[b * H + h] = 0;        // self-resetting: zero again for the next launch
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* src = ws + ((long long)b * H + h) * nsplit * (DA_D + 2);
  float mm = -INFINITY;
  for (int sidx = 0; sidx < nsplit; ++sidx) mm = fmaxf(mm, __ldcg(src + sidx * (DA_D + 2)));
  const float mu = (mm == -INFINITY) ? 0.0f : mm;
  float ll = 0.0f, acc = 0.0f;
  for (int sidx = 0; sidx < nsplit; ++sidx) {
    const float c = exp2f(__ldcg(src + sidx * (DA_D + 2)) - mu);
    ll += __ldcg(src + sidx * (DA_D + 2) + 1) * c;
    acc += __ldcg(src + sidx * (DA_D + 2) + 2 + tid) * c;
  }
  // ll is 0 only without keys; a NaN score makes it NaN, and the output NaN as torch's softmax does
  out[((long long)b * H + h) * DA_D + tid] = __float2half_rn(ll != 0.0f ? acc / ll : 0.0f);
}

__global__ void __launch_bounds__(DA_D)
decode_attn_merge(const float* __restrict__ ws, __half* __restrict__ out, int nsplit, const int* __restrict__ dyn) {
  const long long bh = blockIdx.x;
  const int d = threadIdx.x;
  pdl_trigger();
  pdl_wait();
  if (dyn != nullptr) { int chunk; da_split(dyn[0] + 1, nsplit, chunk); }
  const float* src = ws + bh * nsplit * (DA_D + 2);
  float mm = -INFINITY;
  for (int s = 0; s < nsplit; ++s) mm = fmaxf(mm, src[s * (DA_D + 2)]);
  const float mu = (mm == -INFINITY) ? 0.0f : mm;
  float ll = 0.0f, acc = 0.0f;
  for (int s = 0; s < nsplit; ++s) {
    const float c = exp2f(src[s * (DA_D + 2)] - mu);
    ll += src[s * (DA_D + 2) + 1] * c;
    acc += src[s * (DA_D + 2) + 2 + d] * c;
  }
  out[bh * DA_D + d] = __float2half_rn(ll != 0.0f ? acc / ll : 0.0f);
}

// ----------------------------------------------------------------------------
// Fused decode attention: apply_rotary_pos_emb on the new token's q / k (llama_xformer.py:152-161), the KV-cache append
// (:234-239) and the attention of that one query against the cache (:240-256) in ONE launch per layer: CTA (h, b) of
// ng x 128 threads.  Thread group g walks the 128-key blocks g, g + ng, ... exactly like decode_attn_partial walks a
// split (same arithmetic per block, so for caches of <= ng*128 keys the result is bit-identical to
// rope_kv_kernel -> decode_attn_partial -> merge); the groups' (m, l, o) meet in shared memory instead of a global
// workspace + ticket.  The new key / value never make a round trip through HBM: the group that owns cache row
// `past_len` takes them from shared memory (they are also written to the caches for the following steps).
// Used for max_seq <= 2048 (the decode step is latency-bound there: 2 launches, a global partial buffer and an atomic
// ticket per layer become 1 launch); longer caches keep the split-KV kernels, which spread a head over more SMs.
// ----------------------------------------------------------------------------
constexpr int DAF_MAX_GROUPS = 4;

template <bool LIN>
__global__ void __launch_bounds__(DAF_MAX_GROUPS * 128)
decode_attn_rope_kernel(const __half* __restrict__ qkv, const long long* __restrict__ positions,
                        const __half* __restrict__ cos_t, const __half* __restrict__ sin_t, int max_pos,
                        __half* __restrict__ kc, __half* __restrict__ vc, int H, int past_len, int max_seq,
                        float scale_log2, const int* __restrict__ dyn, __half* __restrict__ out,
                        const int* __restrict__ slot) {
  const int h = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, grp = tid >> 7, gt = tid & 127, ng = blockDim.x >> 7;
  const int warp = gt >> 5, lane = tid & 31;
  __shared__ __align__(16) float s_q[DA_D];
  __shared__ __align__(16) __half s_kn[DA_D];
  __shared__ __align__(16) __half s_vn[DA_D];
  __shared__ float s_p[DAF_MAX_GROUPS][DA_BLK];
  __shared__ float s_red[DAF_MAX_GROUPS][2][4];
  __shared__ __align__(16) float s_o[DAF_MAX_GROUPS][8][DA_D];
  __shared__ float s_ml[DAF_MAX_GROUPS][2];
  __shared__ float s_part[DAF_MAX_GROUPS][DA_D];
  pdl_trigger();
  pdl_wait();
  if (dyn != nullptr) past_len = dyn[0];      // graph-replayed decode step: the cache length lives in device memory
  int crow = past_len;
  if (crow >= max_seq) crow = max_seq - 1;    // only reachable through dyn (host-checked otherwise)
  const int kv_len = crow + 1;
  const long long HD = (long long)H * DA_D;
  const __half* row = qkv + (long long)b * 3 * HD + (long long)h * DA_D;
  const long long base = ((long long)b * H + h) * max_seq * DA_D;
  const long long cache_row = base + (long long)crow * DA_D;
  for (int i = tid; i < 2 * DA_D; i += blockDim.x) {
    if (i < DA_D) {
      // q (i < 64) and k (i >= 64): dims (j, j + 64) of the rotate-half pair, every op rounded to fp16 like rope_kv_kernel
      const int which = i >> 6, j = i & 63;
      long long pos = positions ? positions[b] : (long long)past_len;
      if (pos < 0) pos = 0;
      if (pos >= max_pos) pos = max_pos - 1;
      const float c = __half2float(cos_t[pos * (DA_D / 2) + j]), sn = __half2float(sin_t[pos * (DA_D / 2) + j]);
      const float xl = __half2float(row[which * HD + j]), xh = __half2float(row[which * HD + DA_D / 2 + j]);
      const float a_lo = __half2float(__float2half_rn(xl * c));
      const float b_lo = __half2float(__float2half_rn(-xh * sn));
      const float a_hi = __half2float(__float2half_rn(xh * c));
      const float b_hi = __half2float(__float2half_rn(xl * sn));
      const __half olo = __float2half_rn(a_lo + b_lo), ohi = __float2half_rn(a_hi + b_hi);
      if (which == 0) {
        s_q[j] = __half2float(olo); s_q[j + DA_D / 2] = __half2float(ohi);
      } else {
        s_kn[j] = olo; s_kn[j + DA_D / 2] = ohi;
        kc[cache_row + j] = olo; kc[cache_row + DA_D / 2 + j] = ohi;
      }
    } else {
      const int j = i - DA_D;
      const __half v = row[2 * HD + j];
      s_vn[j] = v;
      vc[cache_row + j] = v;
    }
  }
  __syncthreads();
  const int g = gt >> 4, c = gt & 15;              // P.V role inside the group: key group (8 groups), 8-dim chunk
  const int bar_id = 1 + grp;                       // the groups run different trip counts: one named barrier each
  float m_run = -INFINITY, l_run = 0.0f, o_run = 0.0f;     // o_run: dim `gt`
  for (int kb = grp * DA_BLK; kb < kv_len; kb += ng * DA_BLK) {
    const int cnt = min(DA_BLK, kv_len - kb);
    uint4 vv[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int t = g + 8 * i;
      if (t >= cnt) vv[i] = make_uint4(0, 0, 0, 0);
      else if (kb + t == crow) vv[i] = *(reinterpret_cast<const uint4*>(s_vn) + c);
      else vv[i] = __ldg(reinterpret_cast<const uint4*>(vc + da_row<LIN>(slot, base, b, H, h, max_seq, kb + t)) + c);
    }
    float s = -INFINITY;
    if (gt < cnt) {
      const bool fresh = (kb + gt == crow);
      const uint4* kr = fresh ? reinterpret_cast<const uint4*>(s_kn)
                              : reinterpret_cast<const uint4*>(kc + da_row<LIN>(slot, base, b, H, h, max_seq, kb + gt));
      uint4 kk[16];
      if (fresh) {
#pragma unroll
        for (int i = 0; i < 16; ++i) kk[i] = kr[i];
      } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) kk[i] = __ldg(kr + i);
      }
      float acc = 0.0f;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float4 qa = *reinterpret_cast<const float4*>(s_q + i * 8);
        const float4 qb = *reinterpret_cast<const float4*>(s_q + i * 8 + 4);
        const __half2* kh = reinterpret_cast<const __half2*>(&kk[i]);
        const float2 f0 = __half22float2(kh[0]), f1 = __half22float2(kh[1]);
        const float2 f2 = __half22float2(kh[2]), f3 = __half22float2(kh[3]);
        acc = fmaf(qa.x, f0.x, acc); acc = fmaf(qa.y, f0.y, acc); acc = fmaf(qa.z, f1.x, acc); acc = fmaf(qa.w, f1.y, acc);
        acc = fmaf(qb.x, f2.x, acc); acc = fmaf(qb.y, f2.y, acc); acc = fmaf(qb.z, f3.x, acc); acc = fmaf(qb.w, f3.y, acc);
      }
      s = acc * scale_log2;
    }
    const float wm = warp_max(s);
    if (lane == 0) s_red[grp][0][warp] = wm;
    asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
    const float bm = fmaxf(fmaxf(s_red[grp][0][0], s_red[grp][0][1]), fmaxf(s_red[grp][0][2], s_red[grp][0][3]));
    const float m_new = fmaxf(m_run, bm);
    const float corr = exp2f(m_run - m_new);
    const float p = exp2f(s - m_new);
    s_p[grp][gt] = p;
    const float ws_ = warp_sum(p);
    if (lane == 0) s_red[grp][1][warp] = ws_;
    asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
    l_run = l_run * corr + (s_red[grp][1][0] + s_red[grp][1][1] + s_red[grp][1][2] + s_red[grp][1][3]);
    m_run = m_new;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0f;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float pk = s_p[grp][g + 8 * i];
      const __half2* vh = reinterpret_cast<const __half2*>(&vv[i]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(vh[j]);
        acc[2 * j] = fmaf(pk, f.x, acc[2 * j]);
        acc[2 * j + 1] = fmaf(pk, f.y, acc[2 * j + 1]);
      }
    }
    *reinterpret_cast<float4*>(&s_o[grp][g][c * 8]) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(&s_o[grp][g][c * 8 + 4]) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
    float od = 0.0f;
#pragma unroll
    for (int gg = 0; gg < 8; ++gg) od += s_o[grp][gg][gt];
    o_run = o_run * corr + od;
    asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");   // s_p / s_o / s_red are rewritten by the next block
  }
  if (gt == 0) { s_ml[grp][0] = m_run; s_ml[grp][1] = l_run; }
  s_part[grp][gt] = o_run;
  __syncthreads();
  if (grp != 0) return;
  // merge the groups in index order: the arithmetic of decode_attn_merge over the non-empty "splits"
  const int nsplit = min(ng, (kv_len + DA_BLK - 1) / DA_BLK);
  float mm = -INFINITY;
  for (int sidx = 0; sidx < nsplit; ++sidx) mm = fmaxf(mm, s_ml[sidx][0]);
  const float mu = (mm == -INFINITY) ? 0.0f : mm;
  float ll = 0.0f, acc = 0.0f;
  for (int sidx = 0; sidx < nsplit; ++sidx) {
    const float cc = exp2f(s_ml[sidx][0] - mu);
    ll += s_ml[sidx][1] * cc;
    acc += s_part[sidx][gt] * cc;
  }
  out[((long long)b * H + h) * DA_D + gt] = __float2half_rn(ll != 0.0f ? acc / ll : 0.0f);
}

bool decode_attention_rope_supported(int D, int max_seq) {
  return D == DA_D && max_seq >= 1 && (max_seq + DA_BLK - 1) / DA_BLK <= 4 * DAF_MAX_GROUPS;
}

// qkv [B, 3*H*D] (one new token per sequence: q | k | v), positions [B] or NULL (= past_len); appends K (post-RoPE) and
// V at cache row past_len (dyn: dyn[0]) of caches [B,H,max_seq,D] and writes the attention output out [B, H*D].
// The thread-group count depends on max_seq only, so eager launches and the captured decode step run the same code.
int decode_attention_rope(const void* qkv, const int64_t* positions, int B, int H, int D, int past_len, int max_seq,
                          int max_pos, const void* cos_t, const void* sin_t, void* k_cache, void* v_cache, void* out,
                          float scale, cudaStream_t stream, const int* dyn, const int* slot) {
  SB_REQUIRE(qkv && k_cache && v_cache && out && cos_t && sin_t, "decode_attention_rope: null operand");
  SB_REQUIRE(aligned16(qkv) && aligned16(k_cache) && aligned16(v_cache),
             "decode_attention_rope: qkv and the caches must be 16-byte aligned");
  SB_REQUIRE(decode_attention_rope_supported(D, max_seq),
             "decode_attention_rope: head_dim %d / max_seq %d unsupported (head_dim 128, max_seq <= %d)", D, max_seq,
             4 * DAF_MAX_GROUPS * DA_BLK);
  SB_REQUIRE(dyn != nullptr || (past_len >= 0 && past_len < max_seq), "decode_attention_rope: past_len %d outside [0,%d)",
             past_len, max_seq);
  int ng = (max_seq + DA_BLK - 1) / DA_BLK;
  if (ng > DAF_MAX_GROUPS) ng = DAF_MAX_GROUPS;
  SB_CHECK_CUDA(launch_chain(slot ? decode_attn_rope_kernel<true> : decode_attn_rope_kernel<false>, dim3(H, B),
                             dim3(ng * 128), 0, stream,
                             static_cast<const __half*>(qkv), reinterpret_cast<const long long*>(positions),
                             static_cast<const __half*>(cos_t), static_cast<const __half*>(sin_t), max_pos,
                             static_cast<__half*>(k_cache), static_cast<__half*>(v_cache), H, past_len, max_seq,
                             scale * 1.4426950408889634f, dyn, static_cast<__half*>(out), slot));
  SB_LAUNCH_CHECK();
  return 0;
}

// the most splits any kv_len <= max_seq takes.  da_split is not monotone in kv_len (8192 keys: 64 splits of 128,
// 8193 keys: 33 splits of 256), so da_split(max_seq) itself is not a bound; ceil(kv_len / 128) capped at
// DA_MAX_SPLITS is (every chunk holds at least one 128-key block).
int decode_attention_max_splits(int max_seq) {
  const int n = ((max_seq < 1 ? 1 : max_seq) + DA_BLK - 1) / DA_BLK;
  return n > DA_MAX_SPLITS ? DA_MAX_SPLITS : n;
}

// workspace: [B*H*max_splits*(D+2)] floats of partials (+ [B*H] int tickets when `tickets` is NULL: zeroed here on
// every call).  tickets != NULL: a caller-owned [>= B*H] int array that is zero on entry -- the kernel leaves it zero,
// so a handle zeroes it once at create and never again.
int decode_attention(const void* q, const void* k_cache, const void* v_cache, void* out, int B, int H, int D,
                     int kv_len, int max_seq, float scale, void* workspace, cudaStream_t stream, const int* dyn,
                     int* tickets, const int* slot) {
  SB_REQUIRE(D == DA_D, "decode_attention: head_dim %d unsupported (LLaMA uses 128)", D);
  SB_REQUIRE(dyn != nullptr || (kv_len >= 1 && kv_len <= max_seq), "decode_attention: kv_len %d outside [1,%d]", kv_len, max_seq);
  SB_REQUIRE(aligned16(q) && aligned16(k_cache) && aligned16(v_cache),
             "decode_attention: q and the caches must be 16-byte aligned");
  // dyn: the grid covers the split count of every cache length up to max_seq (surplus splits exit in-kernel, and
  // the kernel derives its chunk from dyn)
  int nsplit = decode_attention_max_splits(max_seq), chunk = 0;
  if (dyn == nullptr) da_split(kv_len, nsplit, chunk);
  if (tickets == nullptr) {
    tickets = reinterpret_cast<int*>(static_cast<float*>(workspace) +
                                     (size_t)B * H * decode_attention_max_splits(max_seq) * (DA_D + 2));
    SB_CHECK_CUDA(cudaMemsetAsync(tickets, 0, (size_t)B * H * sizeof(int), stream));
  }
  dim3 grid(nsplit, H, B);
  SB_CHECK_CUDA(launch_chain(slot ? decode_attn_partial<true> : decode_attn_partial<false>, grid, dim3(128), 0, stream,
                             static_cast<const __half*>(q),
                             static_cast<const __half*>(k_cache), static_cast<const __half*>(v_cache),
                             static_cast<float*>(workspace), H, kv_len, max_seq, chunk, scale * 1.4426950408889634f, dyn,
                             tickets, static_cast<__half*>(out), slot));
  SB_LAUNCH_CHECK();
  return 0;
}

}  // namespace sb

extern "C" {

/* y[m,:] = epilogue(x[m,:] . W^T) for M <= 4 rows (the decode form of nn.Linear, llama_xformer.py:186,223-225,258,718) */
int seedb200_gemv(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w,
                  float eps, int M, int N, int K, int mode, void* stream) {
  SB_REQUIRE(x && W && out, "seedb200_gemv: null operand");
  return sb::gemv(x, W, ldw, out, residual, norm_w, eps, M, N, K, mode, static_cast<cudaStream_t>(stream));
}

int seedb200_gemv_4bit(const void* x, const void* norm_w, float eps, const void* packed, const void* absmax,
                       int quant_type, void* out, const void* residual, int M, int N, int K, int mode, void* stream) {
  return sb::gemv_4bit(x, norm_w, eps, packed, static_cast<const float*>(absmax), quant_type, out, residual, M, N, K,
                       mode, static_cast<cudaStream_t>(stream));
}

int64_t seedb200_decode_attention_workspace_bytes(int B, int H, int max_seq) {
  return (int64_t)B * H * sb::decode_attention_max_splits(max_seq) * (sb::DA_D + 2) * (int64_t)sizeof(float) +
         (int64_t)B * H * (int64_t)sizeof(int);
}

int seedb200_decode_attention(const void* q, const void* k_cache, const void* v_cache, void* out, int B, int H, int D,
                              int kv_len, int max_seq, float scale, void* workspace, void* stream) {
  SB_REQUIRE(q && k_cache && v_cache && out && workspace, "seedb200_decode_attention: null operand");
  return sb::decode_attention(q, k_cache, v_cache, out, B, H, D, kv_len, max_seq, scale, workspace,
                              static_cast<cudaStream_t>(stream));
}

int seedb200_decode_attention_lineage(const void* q, const void* k_cache, const void* v_cache, const int32_t* slot,
                                      void* out, int B, int H, int D, int kv_len, int max_seq, float scale,
                                      void* workspace, void* stream) {
  SB_REQUIRE(q && k_cache && v_cache && slot && out && workspace, "seedb200_decode_attention_lineage: null operand");
  return sb::decode_attention(q, k_cache, v_cache, out, B, H, D, kv_len, max_seq, scale, workspace,
                              static_cast<cudaStream_t>(stream), nullptr, nullptr, slot);
}

}  // extern "C"
