// attention.cu -- softmax(scale * Q K^T [+causal]) V over strided [batch, head, token, dim] views.
//
// Replaces, with one kernel family:
//   eva_vit.py:139-156         ViT-g attention, 257 x 257, 16 heads x 88   (SURVEY 2.4 row E5)
//   qformer_causual.py:189-236 Q-Former self (32 x 32, causal -10000 mask) and
//                              cross attention (32 x 257, 12 heads x 64)   (rows E10, E13)
//   vit.py:93-103              de-tokenizer blocks (32 x 32, 12 x 64)       (row D2)
//   llama_xformer.py:240-256   xops.memory_efficient_attention, causal prefill, d = 128 (row L7)
//
// Two kernels:
//   * vit_attn_kernel (non-causal, head_dim 88, at most 272 keys: the ViT-g shape) -- persistent CTAs over the
//     (image, head) items, TMA-fed, S = Q K^T and O = P V on wgmma with the whole key row in registers and the softmax
//     arithmetic of attn_fwd_kernel (same output bits); see the comment above it.
//   * attn_fwd_kernel (every other shape: the Q-Former, the LLaMA prefill, causal head_dim 88, longer key rows) --
//     flash-attention style: one CTA per (batch, head, query tile); K/V tiles of 64 keys stream through a
//     double-buffered cp.async ring; S = Q K^T and O += P V run on mma.sync m16n8k16 (fp16 in, fp32
//     accumulate); softmax statistics stay in fp32 registers (the reference runs softmax in fp32 under
//     autocast, eva_vit.py:154 / SURVEY 8a precision table).  head_dim 88 is zero-padded to 96 in shared
//     memory only.  The additive -10000 causal mask of the Q-Former underflows to exactly 0 after exp in
//     fp32, so it is implemented as a hard mask.  A wgmma version of it (online softmax over long key rows)
//     is the next step for the LLaMA prefill path.
#include "common.cuh"
#include "wgmma.cuh"

namespace sb {

struct AttnParams {
  const __half* q; const __half* k; const __half* v; __half* o;
  long long q_bs, q_hs, q_ts, k_bs, k_hs, k_ts, v_bs, v_hs, v_ts, o_bs, o_hs, o_ts;
  int nq, nk, head_dim, causal;
  float scale_log2;   // scale * log2(e)
};

__device__ __forceinline__ void ldsm_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ float fast_exp2(float x) {   // ex2.approx: -inf -> +0, 2 ulp
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

constexpr int ATT_BK = 64;

// Load `rows` rows x head_dim halves (row stride ts elements) into smem rows of LDS halves; rows >= valid
// are zero-filled; columns [head_dim, DPAD) were zeroed once at kernel start.
template <int LDS>
__device__ __forceinline__ void load_tile_async(uint32_t smem, const __half* gbase, long long ts, int row0,
                                                int rows, int valid_rows, int chunks, int tid, int nthreads) {
  const int total = rows * chunks;
  for (int i = tid; i < total; i += nthreads) {
    const int r = i / chunks, c = i - r * chunks;
    const int gr = row0 + r;
    const bool ok = gr < valid_rows;
    const __half* src = gbase + (long long)(ok ? gr : 0) * ts + c * 8;
    cp_async16(smem + (uint32_t)(r * LDS + c * 8) * 2u, src, ok ? 16 : 0);
  }
}

template <int DPAD, int NW>
__global__ void __launch_bounds__(NW * 32, (NW * 32 <= 288 && DPAD <= 96) ? 2 : 1)
attn_fwd_kernel(const AttnParams p) {
  constexpr int BQ = NW * 16;
  constexpr int LDS = DPAD + 8;            // padded row stride (halves): conflict-free ldmatrix
  constexpr int KSTEPS = DPAD / 16;
  constexpr int NTHREADS = NW * 32;

  extern __shared__ __align__(16) uint8_t smem_raw[];
  __half* sQ = reinterpret_cast<__half*>(smem_raw);
  __half* sK = sQ + BQ * LDS;              // [2][ATT_BK][LDS]
  __half* sV = sK + 2 * ATT_BK * LDS;      // [2][ATT_BK][LDS]
  const uint32_t sQ_a = smem_u32(sQ), sK_a = smem_u32(sK), sV_a = smem_u32(sV);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * BQ;
  const int head = blockIdx.y, b = blockIdx.z;
  const __half* qg = p.q + b * p.q_bs + head * p.q_hs;
  const __half* kg = p.k + b * p.k_bs + head * p.k_hs;
  const __half* vg = p.v + b * p.v_bs + head * p.v_hs;
  const int chunks = p.head_dim / 8;

  // zero the padding columns (and the 8-half row pad) of every buffer once
  if (p.head_dim < LDS) {
    const int padc = LDS - p.head_dim;
    const int rows_total = BQ + 4 * ATT_BK;
    for (int i = tid; i < rows_total * padc; i += NTHREADS) {
      const int r = i / padc, c = p.head_dim + (i - r * padc);
      sQ[r * LDS + c] = __float2half(0.0f);
    }
  }

  const int causal_off = p.nk - p.nq;
  int nk_eff = p.nk;
  if (p.causal) {
    const int last_row = min(q0 + BQ, p.nq) - 1;
    nk_eff = min(p.nk, last_row + causal_off + 1);
  }
  const int n_ktiles = (nk_eff + ATT_BK - 1) / ATT_BK;

  load_tile_async<LDS>(sQ_a, qg, p.q_ts, q0, BQ, p.nq, chunks, tid, NTHREADS);
  if (n_ktiles > 0) {
    load_tile_async<LDS>(sK_a, kg, p.k_ts, 0, ATT_BK, p.nk, chunks, tid, NTHREADS);
    load_tile_async<LDS>(sV_a, vg, p.v_ts, 0, ATT_BK, p.nk, chunks, tid, NTHREADS);
  }
  cp_async_commit();

  float o_acc[DPAD / 8][4];
#pragma unroll
  for (int i = 0; i < DPAD / 8; ++i) { o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.0f; }
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_run[2] = {0.0f, 0.0f};

  const int row_lo = q0 + warp * 16 + (lane >> 2);   // this thread's two query rows
  const int row_hi = row_lo + 8;
  const int warp_row_max = q0 + warp * 16 + 15;
  const uint32_t q_frag_addr = sQ_a + (uint32_t)((warp * 16 + (lane & 15)) * LDS + (lane >> 4) * 8) * 2u;

  for (int kt = 0; kt < n_ktiles; ++kt) {
    const int buf = kt & 1;
    // one barrier per tile: tile kt has landed and is visible, and every warp is done with tile kt-1, whose
    // buffer is refilled right below while tile kt is being consumed
    cp_async_wait<0>();
    __syncthreads();
    if (kt + 1 < n_ktiles) {
      const int nb = buf ^ 1;
      load_tile_async<LDS>(sK_a + nb * ATT_BK * LDS * 2, kg, p.k_ts, (kt + 1) * ATT_BK, ATT_BK, p.nk, chunks, tid,
                           NTHREADS);
      load_tile_async<LDS>(sV_a + nb * ATT_BK * LDS * 2, vg, p.v_ts, (kt + 1) * ATT_BK, ATT_BK, p.nk, chunks, tid,
                           NTHREADS);
      cp_async_commit();
    }

    // keys of this tile that exist / that this warp may see (a ragged last tile only pays for what it holds:
    // 257 keys = 4 full tiles + 1 key, not 5 tiles)
    const int key0 = kt * ATT_BK;
    int valid = min(ATT_BK, p.nk - key0);
    if (p.causal) valid = min(valid, warp_row_max + causal_off + 1 - key0);
    if (valid <= 0) continue;                         // warp-uniform
    const int npairs = (valid + 15) >> 4;             // 16-key groups to compute (1..4)
    const bool need_mask = (valid < ATT_BK) || (p.causal && key0 + ATT_BK - 1 > q0 + warp * 16 + causal_off);

    // ---- S = Q K^T for this warp's 16 rows x 64 keys ----
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.0f; }
    const uint32_t kbase = sK_a + buf * ATT_BK * LDS * 2;
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
      uint32_t qf[4];
      ldsm_x4(qf[0], qf[1], qf[2], qf[3], q_frag_addr + ks * 32);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        if (np < npairs) {
          const int mi = lane >> 3;
          const int key = np * 16 + (mi >> 1) * 8 + (lane & 7);
          const int dcol = ks * 16 + (mi & 1) * 8;
          uint32_t b0, b1, b2, b3;
          ldsm_x4(b0, b1, b2, b3, kbase + (uint32_t)(key * LDS + dcol) * 2u);
          mma16816(s[2 * np], qf, b0, b1);
          mma16816(s[2 * np + 1], qf, b2, b3);
        }
      }
    }

    // ---- scale, mask, online softmax ----
    float mx[2] = {-INFINITY, -INFINITY};
    if (need_mask) {
      const int kcol0 = key0 + (lane & 3) * 2;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = kcol0 + nt * 8 + (e & 1);
          const int row = (e < 2) ? row_lo : row_hi;
          const bool masked = (col >= p.nk) || (p.causal && col > row + causal_off);
          const float val = masked ? -INFINITY : s[nt][e] * p.scale_log2;
          s[nt][e] = val;
          mx[e >> 1] = fmaxf(mx[e >> 1], val);
        }
      }
    } else {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float val = s[nt][e] * p.scale_log2;
          s[nt][e] = val;
          mx[e >> 1] = fmaxf(mx[e >> 1], val);
        }
      }
    }
    float corr[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = (m_new == -INFINITY) ? 0.0f : m_new;
      corr[r] = fast_exp2(m_run[r] - m_use[r]);     // m_run = -inf -> 0
      m_run[r] = m_new;
      l_run[r] *= corr[r];
    }
    float rs[2] = {0.0f, 0.0f};
    uint32_t pf[4][4];   // P as A fragments for 4 key-steps of 16
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = fast_exp2(s[nt][0] - m_use[0]);
      const float p1 = fast_exp2(s[nt][1] - m_use[0]);
      const float p2 = fast_exp2(s[nt][2] - m_use[1]);
      const float p3 = fast_exp2(s[nt][3] - m_use[1]);
      // the reference rounds the probabilities to fp16 before P.V (autocast, eva_vit.py:155-156);
      // accumulate the row sum from the rounded values so that sum(P)/l is consistent
      const __half2 h01 = __floats2half2_rn(p0, p1);
      const __half2 h23 = __floats2half2_rn(p2, p3);
      const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
      rs[0] += f01.x + f01.y;
      rs[1] += f23.x + f23.y;
      const int ks2 = nt >> 1;
      if ((nt & 1) == 0) {
        pf[ks2][0] = *reinterpret_cast<const uint32_t*>(&h01);
        pf[ks2][1] = *reinterpret_cast<const uint32_t*>(&h23);
      } else {
        pf[ks2][2] = *reinterpret_cast<const uint32_t*>(&h01);
        pf[ks2][3] = *reinterpret_cast<const uint32_t*>(&h23);
      }
    }
    l_run[0] += rs[0];
    l_run[1] += rs[1];
#pragma unroll
    for (int dt = 0; dt < DPAD / 8; ++dt) {
      o_acc[dt][0] *= corr[0]; o_acc[dt][1] *= corr[0];
      o_acc[dt][2] *= corr[1]; o_acc[dt][3] *= corr[1];
    }

    // ---- O += P V ----
    const uint32_t vbase = sV_a + buf * ATT_BK * LDS * 2;
#pragma unroll
    for (int ks2 = 0; ks2 < 4; ++ks2) {
      if (ks2 < npairs) {
#pragma unroll
        for (int dp = 0; dp < DPAD / 16; ++dp) {
          const int mi = lane >> 3;
          const int key = ks2 * 16 + (mi & 1) * 8 + (lane & 7);
          const int dcol = dp * 16 + (mi >> 1) * 8;
          uint32_t b0, b1, b2, b3;
          ldsm_x4_t(b0, b1, b2, b3, vbase + (uint32_t)(key * LDS + dcol) * 2u);
          mma16816(o_acc[2 * dp], pf[ks2], b0, b1);
          mma16816(o_acc[2 * dp + 1], pf[ks2], b2, b3);
        }
      }
    }
  }

  // ---- finalize: quad-reduce the row sums, normalise, store ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv0 = l_run[0] > 0.0f ? 1.0f / l_run[0] : 0.0f;
  const float inv1 = l_run[1] > 0.0f ? 1.0f / l_run[1] : 0.0f;
  __half* og = p.o + b * p.o_bs + head * p.o_hs;
#pragma unroll
  for (int dt = 0; dt < DPAD / 8; ++dt) {
    const int col = dt * 8 + (lane & 3) * 2;
    if (col < p.head_dim) {
      if (row_lo < p.nq)
        *reinterpret_cast<uint32_t*>(og + (long long)row_lo * p.o_ts + col) =
            pack_half2(o_acc[dt][0] * inv0, o_acc[dt][1] * inv0);
      if (row_hi < p.nq)
        *reinterpret_cast<uint32_t*>(og + (long long)row_hi * p.o_ts + col) =
            pack_half2(o_acc[dt][2] * inv1, o_acc[dt][3] * inv1);
    }
  }
}

template <int DPAD, int NW>
static int launch_attn(const seedb200_attn_desc& d, cudaStream_t stream) {
  constexpr int BQ = NW * 16, LDS = DPAD + 8;
  constexpr int smem = (BQ + 4 * ATT_BK) * LDS * 2;
  auto kern = attn_fwd_kernel<DPAD, NW>;
  static bool attr_set_dev[SB_MAX_DEVICES] = {};   // cudaFuncSetAttribute is per device
  bool& attr_set = attr_set_dev[cur_device()];
  if (!attr_set) {
    SB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    // ask for the full shared-memory carve-out so that two CTAs of the 83 KB ViT tile are co-resident
    SB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    attr_set = true;
  }
  AttnParams p;
  p.q = static_cast<const __half*>(d.q); p.k = static_cast<const __half*>(d.k);
  p.v = static_cast<const __half*>(d.v); p.o = static_cast<__half*>(d.o);
  p.q_bs = d.q_bs; p.q_hs = d.q_hs; p.q_ts = d.q_ts;
  p.k_bs = d.k_bs; p.k_hs = d.k_hs; p.k_ts = d.k_ts;
  p.v_bs = d.v_bs; p.v_hs = d.v_hs; p.v_ts = d.v_ts;
  p.o_bs = d.o_bs; p.o_hs = d.o_hs; p.o_ts = d.o_ts;
  p.nq = d.nq; p.nk = d.nk; p.head_dim = d.head_dim; p.causal = d.causal;
  p.scale_log2 = d.scale * 1.4426950408889634f;
  dim3 grid((d.nq + BQ - 1) / BQ, d.heads, d.batch);
  profile_mark_begin(1, stream);
  kern<<<grid, NW * 32, smem, stream>>>(p);
  profile_mark_end(1, stream, 4.0 * (double)d.batch * d.heads * (double)d.nq * d.nk * d.head_dim * (d.causal ? 0.5 : 1.0));
  SB_LAUNCH_CHECK();
  return 0;
}

// ============================================================================
// ViT attention on wgmma: non-causal, head_dim 88, at most VA_NK keys (the ViT-g's 257 x 257 x 88, eva_vit.py:139-156)
// ============================================================================
//
// Persistent CTAs walk the (image, head) items; warpgroup 0 is the TMA producer (one thread), warpgroups 1 and 2 take
// alternate 64-row query tiles of the items' tile sequence.  Per tile the whole key row is held in registers:
// S = Q K^T is one m64n256 + one m64n16 wgmma chain (fp32).  The softmax statistics and O = P V then follow
// attn_fwd_kernel's arithmetic block by block of 64 keys (running max, fp16 P, O rescaled before each block's P V),
// so this kernel gives the mma.sync kernel's output bit for bit; with every score already in registers that costs
// one wgmma wait per key block, not a reload.  P V runs with P from registers (fp16, the RS form) and V read in its
// natural d-contiguous layout (transposed-B descriptor).
//
// Operands arrive by TMA through 4-D tensor maps whose extents are exactly (88 head dims, n tokens, heads, batch), so
// the zero fill of TMA supplies head dims 88..95 and the key / query rows past nk / nq (V rows past nk must be zero,
// not only masked in S: 0 * NaN = NaN in P V).  The 96 head dims of a row are stored as two parts, dims 0..63
// (128-byte rows, 128-byte swizzle) and dims 64..95 (64-byte rows, 64-byte swizzle); each wgmma k-step of S and each
// n-part of O takes the descriptor of its own part.
//
// Shared memory: K double-buffered (the next item's K streams in while this item's tiles run), V single-buffered (the
// next item's V streams in while the next item's S-GEMMs run), and a ring of VA_QST query tiles.
//
// Rounding contract (as the mma.sync kernel): fp32 scores, P = exp2(s * scale * log2 e - running max) rounded to fp16,
// the row sum taken from the rounded values, one division at the end.
constexpr int VA_NK = 272;                       // keys: one n256 chunk + one n16 chunk
constexpr int VA_BLOCKS = 5;                     // softmax blocks of 64 keys (the last one: 16)
constexpr int VA_KBOX = VA_NK / 2;               // key rows per TMA box (a box dimension is at most 256)
constexpr int VA_KV_LO = VA_NK * 128;            // head dims 0..63 of K or V
constexpr int VA_KV_HI = VA_NK * 64;             // head dims 64..95
constexpr int VA_KV_BYTES = VA_KV_LO + VA_KV_HI;
constexpr int VA_Q_LO = 64 * 128, VA_Q_HI = 64 * 64, VA_Q_BYTES = VA_Q_LO + VA_Q_HI;
constexpr int VA_KST = 2;                        // K buffers
constexpr int VA_QST = 6;                        // query tile ring (even: a slot always serves the same warpgroup)
constexpr int VA_THREADS = 384;
constexpr int VA_SMEM = 1024 /*align slack*/ + (VA_KST + 1) * VA_KV_BYTES + VA_QST * VA_Q_BYTES +
                        (2 * VA_QST + 2 * VA_KST + 2) * 8;
static_assert(VA_SMEM <= 227 * 1024, "shared memory budget");
static_assert(VA_KV_LO % 1024 == 0 && VA_KV_HI % 1024 == 0 && VA_Q_BYTES % 1024 == 0 && (VA_KBOX * 64) % 512 == 0,
              "swizzle atoms must stay aligned");

struct VitAttnMaps { CUtensorMap q_lo, q_hi, k_lo, k_hi, v_lo, v_hi; };

// K-major operand (S = Q K^T), head dims 64..95: 64-byte rows, 8-row groups 512 B apart
__device__ __forceinline__ uint64_t wgmma_desc_sw64(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(512 >> 4) << 32;
  d |= static_cast<uint64_t>(2) << 62;                      // SWIZZLE_64B
  return d;
}
// V as the transposed (N-major) B operand of O = P V: rows of `row_bytes` (one swizzle atom wide, 64 or 32 head
// dims), 8-key groups 8 * row_bytes apart.  The n-extent of each wgmma is one atom, so only the 8-key group stride is
// used; it is written to both offset fields.
__device__ __forceinline__ uint64_t wgmma_desc_vt(uint32_t smem_addr, uint32_t row_bytes) {
  const uint64_t grp = (8 * row_bytes) >> 4;
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= grp << 16;
  d |= grp << 32;
  d |= static_cast<uint64_t>(row_bytes == 128 ? 1 : 2) << 62;
  return d;
}

// D[64 x N] += A[64 x 16] . B[16 x N], A from registers (fp16 pairs, the m16n8k16 A-fragment layout per warp), B N-major
// in shared memory
template <int N>
__device__ __forceinline__ void wgmma_f16_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b);
template <> __device__ __forceinline__ void wgmma_f16_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}
template <> __device__ __forceinline__ void wgmma_f16_rs<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t b) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 1;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));
}

__global__ void __launch_bounds__(VA_THREADS, 1)
vit_attn_kernel(const __grid_constant__ VitAttnMaps tm, const AttnParams p, int items, int heads, int m_tiles) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sK = base;                                  // [VA_KST][lo | hi]
  const uint32_t sV = sK + VA_KST * VA_KV_BYTES;             // lo | hi
  const uint32_t sQ = sV + VA_KV_BYTES;                      // [VA_QST][lo | hi]
  const uint32_t q_full = sQ + VA_QST * VA_Q_BYTES;          // [VA_QST]
  const uint32_t q_empty = q_full + 8 * VA_QST;              // [VA_QST]
  const uint32_t k_full = q_empty + 8 * VA_QST;              // [VA_KST]
  const uint32_t k_empty = k_full + 8 * VA_KST;              // [VA_KST]
  const uint32_t v_full = k_empty + 8 * VA_KST;
  const uint32_t v_empty = v_full + 8;

  const int wg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7), 0);
  const int lane = threadIdx.x & 31;
  // a single query tile per item goes to warpgroup 1 only: with alternate tiles, a warpgroup that skips whole items
  // could fall two phases behind the single V buffer's barrier
  const int n_wg = m_tiles > 1 ? 2 : 1;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm.q_lo); tma_prefetch_desc(&tm.q_hi);
    tma_prefetch_desc(&tm.k_lo); tma_prefetch_desc(&tm.k_hi);
    tma_prefetch_desc(&tm.v_lo); tma_prefetch_desc(&tm.v_hi);
    for (int s = 0; s < VA_QST; ++s) {
      mbar_init(q_full + 8 * s, 1);                // the producer's arrive.expect_tx
      mbar_init(q_empty + 8 * s, 4);               // one arrive per warp of the tile's warpgroup
    }
    for (int s = 0; s < VA_KST; ++s) {
      mbar_init(k_full + 8 * s, 1);
      mbar_init(k_empty + 8 * s, 4 * m_tiles);     // one arrive per warp and query tile of the item
    }
    mbar_init(v_full, 1);
    mbar_init(v_empty, 4 * m_tiles);
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int g = 0;                                   // query tile counter, in the consumers' order
      for (int j = 0, item = blockIdx.x; item < items; ++j, item += gridDim.x) {
        const int b = item / heads, h = item - b * heads;
        const int ks = j % VA_KST;
        const uint32_t kbar = k_full + 8 * ks, kdst = sK + ks * VA_KV_BYTES;
        mbar_wait_relaxed_nocall(k_empty + 8 * ks, ((j / VA_KST) & 1) ^ 1);
        mbar_arrive_expect_tx(kbar, VA_KV_BYTES);
        tma_load_4d(kdst, &tm.k_lo, kbar, 0, 0, h, b);
        tma_load_4d(kdst + VA_KBOX * 128, &tm.k_lo, kbar, 0, VA_KBOX, h, b);
        tma_load_4d(kdst + VA_KV_LO, &tm.k_hi, kbar, 64, 0, h, b);
        tma_load_4d(kdst + VA_KV_LO + VA_KBOX * 64, &tm.k_hi, kbar, 64, VA_KBOX, h, b);
        // V goes after the query tiles that fit the ring, before any tile whose slot this item's own earlier tiles
        // release: their warpgroups may be waiting for this V in their P V
        auto load_v = [&]() {
          mbar_wait_relaxed_nocall(v_empty, (j & 1) ^ 1);
          mbar_arrive_expect_tx(v_full, VA_KV_BYTES);
          tma_load_4d(sV, &tm.v_lo, v_full, 0, 0, h, b);
          tma_load_4d(sV + VA_KBOX * 128, &tm.v_lo, v_full, 0, VA_KBOX, h, b);
          tma_load_4d(sV + VA_KV_LO, &tm.v_hi, v_full, 64, 0, h, b);
          tma_load_4d(sV + VA_KV_LO + VA_KBOX * 64, &tm.v_hi, v_full, 64, VA_KBOX, h, b);
        };
        for (int mt = 0; mt < m_tiles; ++mt, ++g) {
          if (mt == VA_QST) load_v();
          const int qs = g % VA_QST;
          const uint32_t qbar = q_full + 8 * qs, qdst = sQ + qs * VA_Q_BYTES;
          mbar_wait_relaxed_nocall(q_empty + 8 * qs, ((g / VA_QST) & 1) ^ 1);
          mbar_arrive_expect_tx(qbar, VA_Q_BYTES);
          tma_load_4d(qdst, &tm.q_lo, qbar, 0, mt * 64, h, b);
          tma_load_4d(qdst + VA_Q_LO, &tm.q_hi, qbar, 64, mt * 64, h, b);
        }
        if (m_tiles <= VA_QST) load_v();
      }
    }
    return;
  }

  // ===================== consumers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int w = wg - 1;
  if (w >= n_wg) return;
  const int warp = (threadIdx.x >> 5) & 3;
  const int quad = lane & 3;
  int g = 0;
  for (int j = 0, item = blockIdx.x; item < items; ++j, item += gridDim.x) {
    const int b = item / heads, h = item - b * heads;
    const int ks = j % VA_KST;
    const uint32_t kbuf = sK + ks * VA_KV_BYTES;
    for (int mt = 0; mt < m_tiles; ++mt, ++g) {
      if (g % n_wg != w) continue;
      const int qs = g % VA_QST;
      const uint32_t qbuf = sQ + qs * VA_Q_BYTES;

      // ---- S = Q K^T over all VA_NK keys: 6 k-steps of 16 head dims ----
      float s0[128], s1[8];
#pragma unroll
      for (int i = 0; i < 128; ++i) s0[i] = 0.0f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s1[i] = 0.0f;
      mbar_wait_nocall(k_full + 8 * ks, (j / VA_KST) & 1);
      mbar_wait_nocall(q_full + 8 * qs, (g / VA_QST) & 1);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {             // head dims 0..63: +32 bytes per k-step inside the 128-byte atom
        const uint64_t a = wgmma_desc_sw128(qbuf) + 2 * kk;
        wgmma_f16<256>(s0, a, wgmma_desc_sw128(kbuf) + 2 * kk);
        wgmma_f16<16>(s1, a, wgmma_desc_sw128(kbuf + 256 * 128) + 2 * kk);
      }
#pragma unroll
      for (int kk = 0; kk < 2; ++kk) {             // head dims 64..95
        const uint64_t a = wgmma_desc_sw64(qbuf + VA_Q_LO) + 2 * kk;
        wgmma_f16<256>(s0, a, wgmma_desc_sw64(kbuf + VA_KV_LO) + 2 * kk);
        wgmma_f16<16>(s1, a, wgmma_desc_sw64(kbuf + VA_KV_LO + 256 * 64) + 2 * kk);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(s0);
      acc_fence(s1);
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(q_empty + 8 * qs);
        mbar_arrive(k_empty + 8 * ks);
      }

      // ---- softmax with the statistics of attn_fwd_kernel, block by block of 64 keys (the last block is the n16
      //      chunk): running max, P = fp16(exp2(s - running max)), l = l * corr + rowsum(P).  Every key is already
      //      in registers, so this is the same arithmetic in the same order as the mma.sync kernel, and the output is
      //      the one it gives.  A block past nk is all -inf: corr = 1 and P = 0 leave l and O as they are.
      //      P as A fragments of 17 k-steps of 16 keys.
      const int row0 = mt * 64 + warp * 16;        // this warp's first query row
      // Every warp runs it, also one whose rows are all past nq (zero queries: finite scores): wgmma operands written
      // or accumulators read on a divergent path make ptxas serialise the wgmma instructions.  Such warps skip the
      // stores only.
      uint32_t pf[VA_NK / 16][4];
      float corr[VA_BLOCKS][2];
      float l_run[2] = {0.0f, 0.0f};
      {
        float m_run[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int blk = 0; blk < VA_BLOCKS; ++blk) {
          float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
          for (int cc = 0; cc < 8; ++cc) {           // this block's n8 chunks (the last block: 2)
            const int c = 8 * blk + cc;
            if (c >= VA_NK / 8) break;
            float* e = c < 32 ? &s0[4 * c] : &s1[4 * (c - 32)];
            const int col = 8 * c + 2 * quad;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float val = (col + (i & 1) < p.nk) ? e[i] * p.scale_log2 : -INFINITY;
              e[i] = val;
              mx[i >> 1] = fmaxf(mx[i >> 1], val);
            }
          }
          float m_use[2];
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float m_new = fmaxf(m_run[r], mx[r]);
            m_use[r] = (m_new == -INFINITY) ? 0.0f : m_new;
            corr[blk][r] = fast_exp2(m_run[r] - m_use[r]);   // m_run = -inf -> 0
            m_run[r] = m_new;
            l_run[r] *= corr[blk][r];
          }
          float rs[2] = {0.0f, 0.0f};
#pragma unroll
          for (int cc = 0; cc < 8; ++cc) {
            const int c = 8 * blk + cc;
            if (c >= VA_NK / 8) break;
            const float* e = c < 32 ? &s0[4 * c] : &s1[4 * (c - 32)];
            // the reference rounds the probabilities to fp16 before P V; the row sum is taken from the rounded values
            const __half2 h01 = __floats2half2_rn(fast_exp2(e[0] - m_use[0]), fast_exp2(e[1] - m_use[0]));
            const __half2 h23 = __floats2half2_rn(fast_exp2(e[2] - m_use[1]), fast_exp2(e[3] - m_use[1]));
            const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
            rs[0] += f01.x + f01.y;
            rs[1] += f23.x + f23.y;
            pf[c >> 1][2 * (c & 1)] = *reinterpret_cast<const uint32_t*>(&h01);
            pf[c >> 1][2 * (c & 1) + 1] = *reinterpret_cast<const uint32_t*>(&h23);
          }
          l_run[0] += rs[0];
          l_run[1] += rs[1];
        }
      }

      // ---- O = P V block by block, O rescaled by the block's corr before its P V (as attn_fwd_kernel): head dims
      //      0..63 (n64) and 64..95 (n32) ----
      float o0[32], o1[16];
#pragma unroll
      for (int i = 0; i < 32; ++i) o0[i] = 0.0f;
#pragma unroll
      for (int i = 0; i < 16; ++i) o1[i] = 0.0f;
      mbar_wait_nocall(v_full, j & 1);
#pragma unroll
      for (int blk = 0; blk < VA_BLOCKS; ++blk) {
        if (blk > 0) {                             // block 0: corr = 0 on O = 0
          wgmma_wait<0>();
          acc_fence(o0);
          acc_fence(o1);
#pragma unroll
          for (int i = 0; i < 32; i += 4) {
            o0[i] *= corr[blk][0]; o0[i + 1] *= corr[blk][0]; o0[i + 2] *= corr[blk][1]; o0[i + 3] *= corr[blk][1];
          }
#pragma unroll
          for (int i = 0; i < 16; i += 4) {
            o1[i] *= corr[blk][0]; o1[i + 1] *= corr[blk][0]; o1[i + 2] *= corr[blk][1]; o1[i + 3] *= corr[blk][1];
          }
        }
        wgmma_fence();
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int kk = 4 * blk + t;
          if (kk >= VA_NK / 16) break;
          wgmma_f16_rs<64>(o0, pf[kk], wgmma_desc_vt(sV + kk * 16 * 128, 128));
          wgmma_f16_rs<32>(o1, pf[kk], wgmma_desc_vt(sV + VA_KV_LO + kk * 16 * 64, 64));
        }
        wgmma_commit();
      }
      wgmma_wait<0>();
      acc_fence(o0);
      acc_fence(o1);
      __syncwarp();
      if (lane == 0) mbar_arrive(v_empty);

      // ---- normalise (outside any branch: the accumulators of a wgmma are read on a converged path) and store
      //      this warp's rows, head dims 0..87 ----
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
      }
      const float inv0 = l_run[0] > 0.0f ? 1.0f / l_run[0] : 0.0f;
      const float inv1 = l_run[1] > 0.0f ? 1.0f / l_run[1] : 0.0f;
      uint32_t out_lo[11], out_hi[11];             // 11 column blocks of 8 = 88 head dims
#pragma unroll
      for (int c = 0; c < 11; ++c) {
        const float* e = c < 8 ? &o0[4 * c] : &o1[4 * (c - 8)];
        out_lo[c] = pack_half2(e[0] * inv0, e[1] * inv0);
        out_hi[c] = pack_half2(e[2] * inv1, e[3] * inv1);
      }
      const int r_lo = row0 + (lane >> 2), r_hi = r_lo + 8;
      __half* og = p.o + b * p.o_bs + h * p.o_hs + 2 * quad;
      if (r_lo < p.nq) {
#pragma unroll
        for (int c = 0; c < 11; ++c) *reinterpret_cast<uint32_t*>(og + (long long)r_lo * p.o_ts + 8 * c) = out_lo[c];
      }
      if (r_hi < p.nq) {
#pragma unroll
        for (int c = 0; c < 11; ++c) *reinterpret_cast<uint32_t*>(og + (long long)r_hi * p.o_ts + 8 * c) = out_hi[c];
      }
    }
  }
}

// [batch, heads, n, 88] view with element strides (bs, hs, ts) -> tensor map of (box_cols x box_rows) boxes starting
// at any head-dim column; everything outside the 88 x n x heads x batch extents reads as zero
static int make_head_tmap(CUtensorMap* tm, const void* ptr, int batch, int heads, int n, int64_t bs, int64_t hs,
                          int64_t ts, int box_cols, int box_rows, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) {
    set_error("cuTensorMapEncodeTiled entry point not available (no CUDA driver?)");
    return SEEDB200_ERR_CUDA;
  }
  // a stride of an extent-1 dimension is never applied; TMA wants every stride to be a positive multiple of 16 bytes
  cuuint64_t gdim[4] = {88, (cuuint64_t)n, (cuuint64_t)heads, (cuuint64_t)batch};
  cuuint64_t gstr[3] = {(cuuint64_t)(n > 1 ? ts * 2 : 16), (cuuint64_t)(heads > 1 ? hs * 2 : 16),
                        (cuuint64_t)(batch > 1 ? bs * 2 : 16)};
  cuuint32_t box[4] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("attention: cuTensorMapEncodeTiled failed with CUresult %d (n=%d heads=%d batch=%d strides %lld %lld %lld)",
              (int)r, n, heads, batch, (long long)bs, (long long)hs, (long long)ts);
    return SEEDB200_ERR_CUDA;
  }
  return 0;
}

// the wgmma kernel's inputs: non-causal head_dim 88 with at most VA_NK keys, q / k / v strides positive wherever the
// extent is above 1 (TMA addresses by positive strides only)
static bool vit_attn_fits(const seedb200_attn_desc& d) {
  if (d.head_dim != 88 || d.causal || d.nk > VA_NK || (int64_t)d.batch * d.heads > INT32_MAX) return false;
  const int64_t st[3][3] = {{d.q_bs, d.q_hs, d.q_ts}, {d.k_bs, d.k_hs, d.k_ts}, {d.v_bs, d.v_hs, d.v_ts}};
  const int ext[3][3] = {{d.batch, d.heads, d.nq}, {d.batch, d.heads, d.nk}, {d.batch, d.heads, d.nk}};
  for (int t = 0; t < 3; ++t)
    for (int i = 0; i < 3; ++i)
      if (ext[t][i] > 1 && st[t][i] <= 0) return false;
  return true;
}

static int launch_vit_attn(const seedb200_attn_desc& d, cudaStream_t stream) {
  static bool attr_set_dev[SB_MAX_DEVICES] = {};   // cudaFuncSetAttribute is per device
  bool& attr_set = attr_set_dev[cur_device()];
  if (!attr_set) {
    SB_CHECK_CUDA(cudaFuncSetAttribute(vit_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, VA_SMEM));
    attr_set = true;
  }
  VitAttnMaps tm;
  const CUtensorMapSwizzle lo = CU_TENSOR_MAP_SWIZZLE_128B, hi = CU_TENSOR_MAP_SWIZZLE_64B;
  SB_PROPAGATE(make_head_tmap(&tm.q_lo, d.q, d.batch, d.heads, d.nq, d.q_bs, d.q_hs, d.q_ts, 64, 64, lo));
  SB_PROPAGATE(make_head_tmap(&tm.q_hi, d.q, d.batch, d.heads, d.nq, d.q_bs, d.q_hs, d.q_ts, 32, 64, hi));
  SB_PROPAGATE(make_head_tmap(&tm.k_lo, d.k, d.batch, d.heads, d.nk, d.k_bs, d.k_hs, d.k_ts, 64, VA_KBOX, lo));
  SB_PROPAGATE(make_head_tmap(&tm.k_hi, d.k, d.batch, d.heads, d.nk, d.k_bs, d.k_hs, d.k_ts, 32, VA_KBOX, hi));
  SB_PROPAGATE(make_head_tmap(&tm.v_lo, d.v, d.batch, d.heads, d.nk, d.v_bs, d.v_hs, d.v_ts, 64, VA_KBOX, lo));
  SB_PROPAGATE(make_head_tmap(&tm.v_hi, d.v, d.batch, d.heads, d.nk, d.v_bs, d.v_hs, d.v_ts, 32, VA_KBOX, hi));
  AttnParams p = {};
  p.o = static_cast<__half*>(d.o);
  p.o_bs = d.o_bs; p.o_hs = d.o_hs; p.o_ts = d.o_ts;
  p.nq = d.nq; p.nk = d.nk; p.head_dim = d.head_dim; p.causal = 0;
  p.scale_log2 = d.scale * 1.4426950408889634f;
  const int items = d.batch * d.heads;
  const int m_tiles = (d.nq + 63) / 64;
  const int grid = items < num_sms() ? items : num_sms();
  profile_mark_begin(1, stream);
  vit_attn_kernel<<<grid, VA_THREADS, VA_SMEM, stream>>>(tm, p, items, d.heads, m_tiles);
  profile_mark_end(1, stream, 4.0 * (double)d.batch * d.heads * (double)d.nq * d.nk * d.head_dim);
  SB_LAUNCH_CHECK();
  return 0;
}

int attention(const seedb200_attn_desc& d, cudaStream_t stream) {
  SB_REQUIRE(d.q && d.k && d.v && d.o, "attention: null operand");
  SB_REQUIRE(d.batch > 0 && d.heads > 0 && d.nq > 0 && d.nk > 0, "attention: empty problem");
  SB_REQUIRE(d.head_dim == 64 || d.head_dim == 88 || d.head_dim == 128,
             "attention: head_dim %d not in {64, 88, 128}", d.head_dim);
  SB_REQUIRE(d.batch <= 65535 && d.heads <= 65535, "attention: batch/heads exceed grid limits");
  const int64_t strides[] = {d.q_bs, d.q_hs, d.q_ts, d.k_bs, d.k_hs, d.k_ts, d.v_bs, d.v_hs, d.v_ts,
                             d.o_bs, d.o_hs, d.o_ts};
  for (int i = 0; i < 9; ++i)
    SB_REQUIRE(strides[i] % 8 == 0, "attention: q/k/v strides must be multiples of 8 elements (16-byte cp.async)");
  for (int i = 9; i < 12; ++i) SB_REQUIRE(strides[i] % 2 == 0, "attention: o strides must be even");
  SB_REQUIRE(((uintptr_t)d.q % 16 == 0) && ((uintptr_t)d.k % 16 == 0) && ((uintptr_t)d.v % 16 == 0) &&
                 ((uintptr_t)d.o % 4 == 0),
             "attention: misaligned pointer");
  if (d.head_dim == 64) {
    if (d.nq <= 32) return launch_attn<64, 2>(d, stream);
    return launch_attn<64, 4>(d, stream);
  }
  if (vit_attn_fits(d)) return launch_vit_attn(d, stream);
  if (d.head_dim == 88) {
    if (d.nq > 64 && d.nq <= 288) return launch_attn<96, 9>(d, stream);   // 257 tokens -> 2 x 144-row tiles
    return launch_attn<96, 4>(d, stream);
  }
  if (d.nq <= 64) return launch_attn<128, 4>(d, stream);
  return launch_attn<128, 8>(d, stream);
}

}  // namespace sb

extern "C" int seedb200_attention(const seedb200_attn_desc* d, void* stream) {
  if (d == nullptr) {
    sb::set_error("seedb200_attention: null descriptor");
    return SEEDB200_ERR_INVALID;
  }
  return sb::attention(*d, static_cast<cudaStream_t>(stream));
}
