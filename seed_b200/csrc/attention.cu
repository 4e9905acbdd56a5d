// attention.cu -- softmax(scale * Q K^T [+causal]) V over strided [batch, head, token, dim] views.
//
// Replaces, with one kernel family:
//   eva_vit.py:139-156         ViT-g attention, 257 x 257, 16 heads x 88   (SURVEY 2.4 row E5)
//   qformer_causual.py:189-236 Q-Former self (32 x 32, causal -10000 mask) and
//                              cross attention (32 x 257, 12 heads x 64)   (rows E10, E13)
//   vit.py:93-103              de-tokenizer blocks (32 x 32, 12 x 64)       (row D2)
//   llama_xformer.py:240-256   xops.memory_efficient_attention, causal prefill, d = 128 (row L7)
//
// Flash-attention style: one CTA per (batch, head, query tile); K/V tiles of 64 keys stream through a
// double-buffered cp.async ring; S = Q K^T and O += P V run on mma.sync m16n8k16 (fp16 in, fp32
// accumulate); softmax statistics stay in fp32 registers (the reference runs softmax in fp32 under
// autocast, eva_vit.py:154 / SURVEY 8a precision table).  head_dim 88 is zero-padded to 96 in shared
// memory only.  The additive -10000 causal mask of the Q-Former underflows to exactly 0 after exp in
// fp32, so it is implemented as a hard mask.
//
// This is ~3% of the encode FLOPs; the tensor-core budget went to the GEMM first.  A wgmma version of
// this kernel is the next step for the LLaMA prefill path.
#include "common.cuh"

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
