// sampler.cu -- the token side of the generation loop, on the device (SURVEY.md 8f rows 2 and 3).
//
//   sample_kernel          next-token selection from fp16 logits, one CTA per sequence.  Replaces what the reference
//                          gets from HF GenerationMixin.sample / greedy_search at its call site
//                          scripts/seed_llama_inference_8B.py:33 (temperature=1.0, top_p=0.5, do_sample=True):
//                          TemperatureLogitsWarper (logits / T), TopPLogitsWarper (drop the ascending-sorted tokens whose
//                          cumulative probability is <= 1 - top_p, keep at least one), softmax, multinomial.
//                          Sort-free: the nucleus is {i : mass of tokens more probable than i < top_p}, which is a
//                          threshold on p found by bisection over the float bit pattern (31 block reductions); the draw
//                          inverts the CDF of the kept tokens in index order with one Philox4x32-10 uniform per
//                          (sequence, step).  Greedy = argmax with ties to the lowest id (torch.argmax).
//   image_ids_to_tokens    [n,32] codebook ids -> `<img> <img_xxxxx>*32 </img>` token ids by arithmetic
//                          (scripts/seed_llama_inference_8B.py:16-23,60,98-100 build them through a string round trip).
#include <string.h>

#include "common.cuh"
#include "ops.h"

namespace sb {

constexpr int SAMP_THREADS = 1024;

// ---- Philox4x32-10 (Salmon et al., SC'11) -- same constants as cuRAND / torch's Philox -----------------------------
__host__ __device__ inline void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint64_t p0 = (uint64_t)0xD2511F53u * c[0];
  const uint64_t p1 = (uint64_t)0xCD9E8D57u * c[2];
  const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
  const uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
// first output word of Philox4x32-10 for counter (offset_lo, offset_hi, row, word3), key = seed
__host__ __device__ inline uint32_t philox_word(uint64_t seed, uint64_t offset, uint32_t row, uint32_t word3) {
  uint32_t c[4] = {(uint32_t)offset, (uint32_t)(offset >> 32), row, word3};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c[0];
}
// uniform in (0, 1]: counter = (offset_lo, offset_hi, row, 0), key = seed; first output word, cuRAND's conversion
__host__ __device__ inline float philox_uniform(uint64_t seed, uint64_t offset, uint32_t row) {
  return (float)philox_word(seed, offset, row, 0u) * 2.3283064365386963e-10f + 1.1641532182693481e-10f;   // (x + 0.5) / 2^32
}
// uniform strictly inside (0, 1) of the beam sampler's Gumbel keys: counter (offset_lo, offset_hi, row, 1 + j).
// ((x >> 9) + 0.5) * 2^-23 is exact in fp32 (24 significant bits), so it never rounds to 1.
__host__ __device__ inline float philox_open_uniform(uint64_t seed, uint64_t offset, uint32_t row, uint32_t j) {
  return ((float)(philox_word(seed, offset, row, 1u + j) >> 9) + 0.5f) * 1.1920928955078125e-07f;
}

struct SampleArgs {
  const __half* logits; long long ld; int V;
  GenParams gp;                        // sampling parameters + eos/pad by value, or ...
  const GenParams* gp_dev;             // ... read from device memory when non-null (graph replay)
  unsigned long long step;             // Philox offset of this call = sp.offset + step, or ...
  int* state;                          // ... state[1] when non-null: device counters {cache length, step, arrive,
                                       //     valid steps, any-unfinished flag}, advanced by the last CTA to finish
  int advance_cache;                   // also bump state[0] (a decode forward consumed the previous token)
  long long* tokens;                   // [B] next token per sequence (also the next step's input ids)
  long long* out; long long out_ld;    // optional [B, out_ld] history: out[b, step] = token
  int* finished;                       // optional [B]: sequences that already produced eos emit pad (HF semantics)
  int B;
};

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (threadIdx.x < SAMP_THREADS / 32) ? red[threadIdx.x] : 0.0f;
  if (warp == 0) {
    t = warp_sum(t);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

// nucleus threshold (TopPLogitsWarper in threshold form): the smallest t with mass{p > t} < target, found by bisection
// over the float bit pattern of p in (0, 1] (31 block reductions); kept = {p >= t}.  prob(i) is this thread's p_i over
// its elements [i0, i1).
template <typename Prob>
__device__ float nucleus_threshold(const Prob& prob, int i0, int i1, float target, float* red) {
  uint32_t lo = 0u, hi = 0x3F800000u;        // mass{p > 1} = 0 < target, so hi always qualifies
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    const float t = __uint_as_float(mid);
    float m = 0.0f;
    for (int i = i0; i < i1; ++i) { const float p = prob(i); m += p > t ? p : 0.0f; }
    m = block_sum(m, red);
    if (m < target) hi = mid; else lo = mid + 1;
  }
  return __uint_as_float(lo);
}

__global__ void __launch_bounds__(SAMP_THREADS)
sample_kernel(const SampleArgs a) {
  __shared__ float red[SAMP_THREADS / 32];
  __shared__ float red_v[SAMP_THREADS / 32];
  __shared__ int red_i[SAMP_THREADS / 32];
  __shared__ float scan[SAMP_THREADS];
  __shared__ int s_pick;
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_trigger();
  pdl_wait();
  const GenParams gp = a.gp_dev ? *a.gp_dev : a.gp;
  const seedb200_sample_params sp = gp.sp;
  const unsigned long long step = a.state ? (unsigned long long)a.state[1] : a.step;
  const __half* row = a.logits + (long long)b * a.ld;
  const int V = a.V;
  // contiguous chunk per thread (the CDF inversion below walks tokens in index order)
  const int per = (V + SAMP_THREADS - 1) / SAMP_THREADS;
  const int i0 = min(V, tid * per), i1 = min(V, i0 + per);

  // ---- argmax (ties -> lowest index), also the softmax max ----
  float mx = -INFINITY; int mi = 0x7fffffff;
  for (int i = i0; i < i1; ++i) {
    const float x = __half2float(row[i]);
    if (x > mx || (x == mx && i < mi)) { mx = x; mi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
    if (ov > mx || (ov == mx && oi < mi)) { mx = ov; mi = oi; }
  }
  if (lane == 0) { red_v[warp] = mx; red_i[warp] = mi; }
  __syncthreads();
  if (warp == 0) {
    mx = red_v[lane]; mi = red_i[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, mx, o);
      const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
      if (ov > mx || (ov == mx && oi < mi)) { mx = ov; mi = oi; }
    }
    if (lane == 0) { red_v[0] = mx; red_i[0] = mi; }
  }
  __syncthreads();
  mx = red_v[0]; mi = red_i[0];
  if (mi == 0x7fffffff) mi = 0;
  int pick = mi;

  if (sp.do_sample != 0) {
    // p_i = exp((x_i - max) / T)  (unnormalised; TemperatureLogitsWarper then softmax)
    const float inv_t = 1.0f / fmaxf(sp.temperature, 1e-6f);
    const float kk = inv_t * 1.4426950408889634f;
    auto prob = [&](int i) { return exp2f((__half2float(row[i]) - mx) * kk); };
    float z = 0.0f;
    for (int i = i0; i < i1; ++i) z += prob(i);
    const float Z = block_sum(z, red);
    // nucleus threshold: smallest t with mass{p > t} < top_p * Z; kept = {p >= t}.  top_p >= 1 keeps everything.
    float thr = 0.0f;
    if (sp.top_p < 1.0f) thr = nucleus_threshold(prob, i0, i1, sp.top_p * Z, red);
    // inverse CDF over the kept tokens in index order
    float k = 0.0f;
    for (int i = i0; i < i1; ++i) { const float p = prob(i); k += p >= thr ? p : 0.0f; }
    scan[tid] = k;
    __syncthreads();
    // inclusive scan of the 1024 per-thread masses (Hillis-Steele in shared memory)
    for (int o = 1; o < SAMP_THREADS; o <<= 1) {
      const float add = tid >= o ? scan[tid - o] : 0.0f;
      __syncthreads();
      scan[tid] += add;
      __syncthreads();
    }
    const float K = scan[SAMP_THREADS - 1];
    const float u = philox_uniform(sp.seed, sp.offset + step, (uint32_t)b) * K;     // (0, K]
    if (tid == 0) s_pick = -1;
    __syncthreads();
    const float before = tid > 0 ? scan[tid - 1] : 0.0f;
    if (k > 0.0f && u > before && u <= scan[tid]) {
      // exactly one chunk holds the draw (the scan is monotone and u <= K); walk it in index order.  If rounding
      // leaves the running sum a hair under u at the end of the chunk, the chunk's last kept token is the answer.
      float c = before; int sel = -1;
      for (int i = i0; i < i1; ++i) {
        const float p = prob(i);
        if (p >= thr) { c += p; sel = i; if (c >= u) break; }
      }
      s_pick = sel;
    }
    __syncthreads();
    pick = s_pick >= 0 ? s_pick : mi;          // numerically empty nucleus cannot happen (argmax is always kept)
  }

  if (tid == 0) {
    long long tok = pick;
    bool was_unfinished = true;
    if (a.finished != nullptr) {
      was_unfinished = a.finished[b] == 0;
      if (!was_unfinished) tok = gp.pad;                       // HF: next_tokens * unfinished + pad * (1 - unfinished)
      else if (gp.eos >= 0 && tok == gp.eos) a.finished[b] = 1;
    }
    a.tokens[b] = tok;
    if (a.out != nullptr) a.out[(long long)b * a.out_ld + (long long)step] = tok;
    if (a.state != nullptr) {
      if (was_unfinished) atomicOr(&a.state[4], 1);
      __threadfence();
      if (atomicAdd(&a.state[2], 1) == a.B - 1) {       // last sequence of this step: publish the new position
        if (atomicOr(&a.state[4], 0) != 0) a.state[3] = (int)step + 1;   // steps HF would have kept (it stops once all finished)
        a.state[4] = 0;
        a.state[2] = 0;
        a.state[1] = (int)step + 1;
        if (a.advance_cache) a.state[0] += 1;
        __threadfence();
      }
    }
  }
}

int sample(const void* logits, int64_t ld, int B, int V, const GenParams* gp, const GenParams* gp_dev, uint64_t step,
           int* state, int advance_cache, int64_t* tokens, int64_t* out, int64_t out_ld, int* finished,
           cudaStream_t stream) {
  SB_REQUIRE(logits && tokens && B >= 1 && V >= 1 && ld >= V, "sample: bad arguments");
  SB_REQUIRE(gp != nullptr || gp_dev != nullptr, "sample: no sampling parameters");
  SampleArgs a;
  a.logits = static_cast<const __half*>(logits); a.ld = ld; a.V = V;
  if (gp) a.gp = *gp;
  else { a.gp.sp.do_sample = 0; a.gp.sp.temperature = 1.0f; a.gp.sp.top_p = 1.0f; a.gp.sp.seed = 0; a.gp.sp.offset = 0; a.gp.eos = -1; a.gp.pad = 0; }
  a.gp_dev = gp_dev; a.step = step; a.state = state; a.advance_cache = advance_cache;
  a.tokens = reinterpret_cast<long long*>(tokens);
  a.out = reinterpret_cast<long long*>(out); a.out_ld = out_ld;
  a.finished = finished; a.B = B;
  SB_CHECK_CUDA(launch_chain(sample_kernel, dim3(B), dim3(SAMP_THREADS), 0, stream, a));
  SB_LAUNCH_CHECK();
  return 0;
}

// ---- beam search candidates (transformers 4.30.2 beam_search / beam_sample, include/seedb200.h) ------------------
// Two launches.  beam_row_stats_kernel, one CTA per (beam row, sequence): max and second max, the fp32 log-sum-exp, so
// that lp = fp16((x - max) - logZ) (log_softmax in the logits' dtype) and s = lp + beam_score in fp32; when sampling,
// w = s / T and the TopP threshold on w (min_tokens_to_keep = 2, threshold form).  beam_select_kernel, one CTA per
// sequence over its k rows: key = s (greedy) or w + Gumbel(u) / -inf (sampling); each thread keeps its own best NC
// (key, flat index) pairs, and 2k block-wide rounds then pop the best head.
struct BeamSelectArgs {
  const __half* logits; long long seq_ld, beam_ld; int V;
  const float* beam_scores;            // [B*k]
  BeamParams bp; const BeamParams* bp_dev;
  unsigned long long step; const int* state;
  float* row_stats;                    // [B*k, 5]: max, logZ, beam score, max w, nucleus threshold
  float* cand_score; int* cand_idx;    // [B, 2k]
};

__device__ __forceinline__ bool cand_better(float a, int ia, float b, int ib) { return a > b || (a == b && ia < ib); }

__device__ __forceinline__ void top2_merge(float& m1, float& m2, float o1, float o2) {
  const float n2 = fmaxf(fminf(m1, o1), fmaxf(m2, o2));
  m1 = fmaxf(m1, o1);
  m2 = n2;
}

// one CTA per (beam row j, sequence i): the row's statistics, so that the k rows of a sequence run on k SMs
__global__ void __launch_bounds__(SAMP_THREADS)
beam_row_stats_kernel(const BeamSelectArgs a) {
  __shared__ float red[SAMP_THREADS / 32];
  __shared__ float red2[SAMP_THREADS / 32];
  const int j = blockIdx.x, sq = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_trigger();
  pdl_wait();
  const BeamParams bp = a.bp_dev ? *a.bp_dev : a.bp;
  const int k = bp.k, V = a.V;
  if (j >= k) return;
  const float T = bp.temperature;
  const int per = (V + SAMP_THREADS - 1) / SAMP_THREADS;
  const int i0 = min(V, tid * per), i1 = min(V, i0 + per);
  const __half* row = a.logits + (long long)sq * a.seq_ld + (long long)j * a.beam_ld;
  float m1 = -INFINITY, m2 = -INFINITY;
  for (int i = i0; i < i1; ++i) top2_merge(m1, m2, __half2float(row[i]), -INFINITY);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    top2_merge(m1, m2, __shfl_xor_sync(0xffffffffu, m1, o), __shfl_xor_sync(0xffffffffu, m2, o));
  if (lane == 0) { red[warp] = m1; red2[warp] = m2; }
  __syncthreads();
  if (warp == 0) {
    m1 = red[lane]; m2 = red2[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      top2_merge(m1, m2, __shfl_xor_sync(0xffffffffu, m1, o), __shfl_xor_sync(0xffffffffu, m2, o));
    if (lane == 0) { red[0] = m1; red2[0] = m2; }
  }
  __syncthreads();
  m1 = red[0]; m2 = red2[0];
  float z = 0.0f;
  for (int i = i0; i < i1; ++i) z += expf(__half2float(row[i]) - m1);
  const float lz = logf(block_sum(z, red));
  const float bsc = a.beam_scores[sq * k + j];
  // s = float(fp16 log_softmax) + beam score, fp32
  auto score = [&](float x) { return __half2float(__float2half_rn((x - m1) - lz)) + bsc; };
  float mxw = 0.0f, thr = 0.0f;
  if (bp.do_sample != 0) {
    mxw = score(m1) / T;                   // every step is monotone in x: the largest x gives the largest w
    auto prob = [&](int i) { return exp2f((score(__half2float(row[i])) / T - mxw) * 1.4426950408889634f); };
    if (bp.top_p < 1.0f) {
      float zp = 0.0f;
      for (int i = i0; i < i1; ++i) zp += prob(i);
      const float Zp = block_sum(zp, red);
      thr = nucleus_threshold(prob, i0, i1, bp.top_p * Zp, red);
      // min_tokens_to_keep = 2: the two most probable tokens stay (and every token tied with them)
      const float p2 = m2 == -INFINITY ? 0.0f : exp2f((score(m2) / T - mxw) * 1.4426950408889634f);
      thr = fminf(thr, p2);
    }
  }
  if (tid == 0) {
    float* o = a.row_stats + (long long)(sq * k + j) * 5;
    o[0] = m1; o[1] = lz; o[2] = bsc; o[3] = mxw; o[4] = thr;
  }
}

template <int NC>
__global__ void __launch_bounds__(SAMP_THREADS)
beam_select_kernel(const BeamSelectArgs a) {
  __shared__ float red[SAMP_THREADS / 32];
  __shared__ int redi[SAMP_THREADS / 32];
  __shared__ float s_mx[BEAM_MAX], s_lz[BEAM_MAX], s_bs[BEAM_MAX], s_mxw[BEAM_MAX], s_thr[BEAM_MAX];
  __shared__ float s_key[2 * BEAM_MAX];
  __shared__ int s_idx[2 * BEAM_MAX];
  const int sq = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_trigger();
  pdl_wait();
  const BeamParams bp = a.bp_dev ? *a.bp_dev : a.bp;
  const unsigned long long step = a.state ? (unsigned long long)a.state[1] : a.step;
  const int k = bp.k, n2 = 2 * k, V = a.V;
  const bool samp = bp.do_sample != 0;
  const float T = bp.temperature;
  auto rowp = [&](int j) { return a.logits + (long long)sq * a.seq_ld + (long long)j * a.beam_ld; };
  auto score = [&](int j, float x) {      // s = float(fp16 log_softmax) + beam score, fp32
    return __half2float(__float2half_rn((x - s_mx[j]) - s_lz[j])) + s_bs[j];
  };
  if (tid < k) {
    const float* st = a.row_stats + (long long)(sq * k + tid) * 5;
    s_mx[tid] = st[0]; s_lz[tid] = st[1]; s_bs[tid] = st[2]; s_mxw[tid] = st[3]; s_thr[tid] = st[4];
  }
  __syncthreads();
  // ---- per-thread best NC candidates, flat index f = j * V + t in increasing order ----
  float kv[NC];
  int ki[NC];
#pragma unroll
  for (int q = 0; q < NC; ++q) { kv[q] = -INFINITY; ki[q] = 0x7fffffff; }
  for (int j = 0; j < k; ++j) {
    const __half* row = rowp(j);
    for (int t = tid; t < V; t += SAMP_THREADS) {
      const float sc = score(j, __half2float(row[t]));
      const int f = j * V + t;
      float key = sc;
      if (samp) {
        const float w = sc / T;
        const float p = exp2f((w - s_mxw[j]) * 1.4426950408889634f);
        key = -INFINITY;
        if (p >= s_thr[j]) {
          const float u = philox_open_uniform(bp.seed, bp.offset + step, (uint32_t)sq, (uint32_t)f);
          key = w + (-logf(-logf(u)));
        }
      }
      float ck = key;
      int ci = f;
#pragma unroll
      for (int q = 0; q < NC; ++q) {
        if (cand_better(ck, ci, kv[q], ki[q])) {
          const float tk = kv[q]; const int ti = ki[q];
          kv[q] = ck; ki[q] = ci; ck = tk; ci = ti;
        }
      }
    }
  }
  // ---- 2k rounds: the best head of all threads wins and is popped ----
  for (int r = 0; r < n2; ++r) {
    float bk = kv[0];
    int bi = ki[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ok = __shfl_xor_sync(0xffffffffu, bk, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (cand_better(ok, oi, bk, bi)) { bk = ok; bi = oi; }
    }
    __syncthreads();
    if (lane == 0) { red[warp] = bk; redi[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      bk = red[lane]; bi = redi[lane];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ok = __shfl_xor_sync(0xffffffffu, bk, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (cand_better(ok, oi, bk, bi)) { bk = ok; bi = oi; }
      }
      if (lane == 0) { s_key[r] = bk; s_idx[r] = bi; }
    }
    __syncthreads();
    if (ki[0] == s_idx[r] && ki[0] != 0x7fffffff) {
#pragma unroll
      for (int q = 0; q + 1 < NC; ++q) { kv[q] = kv[q + 1]; ki[q] = ki[q + 1]; }
      kv[NC - 1] = -INFINITY; ki[NC - 1] = 0x7fffffff;
    }
  }
  if (tid != 0) return;
  // the scorer receives s (greedy) or w (sampling), the draws sorted by w descending, ties to the lowest index
  float sc[2 * BEAM_MAX];
  int ix[2 * BEAM_MAX];
  for (int r = 0; r < n2; ++r) {
    int f = s_idx[r];
    if (f < 0 || f >= k * V) f = 0;      // unreachable with k * V >= 2k entries
    const int j = f / V;
    const float v = score(j, __half2float(rowp(j)[f - j * V]));
    float w = samp ? v / T : v;
    int q = r;
    while (q > 0 && cand_better(w, f, sc[q - 1], ix[q - 1])) { sc[q] = sc[q - 1]; ix[q] = ix[q - 1]; --q; }
    sc[q] = w; ix[q] = f;
  }
  for (int r = 0; r < n2; ++r) {
    a.cand_score[(long long)sq * n2 + r] = sc[r];
    a.cand_idx[(long long)sq * n2 + r] = ix[r];
  }
}

int beam_select(const void* logits, int64_t seq_ld, int64_t beam_ld, int B, int k, int V, const float* beam_scores,
                const BeamParams* bp, const BeamParams* bp_dev, uint64_t step, const int* state, float* row_stats,
                float* cand_score, int* cand_idx, cudaStream_t stream) {
  SB_REQUIRE(logits && beam_scores && row_stats && cand_score && cand_idx && (bp || bp_dev), "beam_select: null operand");
  SB_REQUIRE(B >= 1 && k >= 1 && k <= BEAM_MAX && V >= 2 && (int64_t)k * V < 0x7fffffff,
             "beam_select: bad sizes (B %d, k %d in [1,%d], V %d >= 2)", B, k, BEAM_MAX, V);
  SB_REQUIRE(seq_ld >= 0 && beam_ld >= 0, "beam_select: negative row stride");
  if (bp) {
    SB_REQUIRE(bp->k == k, "beam_select: params.num_beams %d != k %d", bp->k, k);
    SB_REQUIRE(!bp->do_sample || (bp->temperature > 0.0f && bp->top_p > 0.0f),
               "beam_select: temperature and top_p must be > 0 when sampling");
  }
  BeamSelectArgs a;
  memset(&a, 0, sizeof(a));
  a.logits = static_cast<const __half*>(logits); a.seq_ld = seq_ld; a.beam_ld = beam_ld; a.V = V;
  a.beam_scores = beam_scores;
  if (bp) a.bp = *bp;
  a.bp_dev = bp_dev; a.step = step; a.state = state; a.row_stats = row_stats;
  a.cand_score = cand_score; a.cand_idx = cand_idx;
  SB_CHECK_CUDA(launch_chain(beam_row_stats_kernel, dim3(k, B), dim3(SAMP_THREADS), 0, stream, a));
  SB_LAUNCH_CHECK();
  const int n2 = 2 * k;
  auto kern = n2 <= 4 ? beam_select_kernel<4> : (n2 <= 8 ? beam_select_kernel<8> : beam_select_kernel<16>);
  SB_CHECK_CUDA(launch_chain(kern, dim3(B), dim3(SAMP_THREADS), 0, stream, a));
  SB_LAUNCH_CHECK();
  return 0;
}

// ---- codebook ids -> LLaMA token ids -----------------------------------------------------------------------------
__global__ void image_ids_to_tokens_kernel(const long long* __restrict__ ids, int n, long long shift, long long boi,
                                           long long eoi, long long* __restrict__ out, long long out_stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 34) return;
  const int img = i / 34, j = i - img * 34;
  long long t;
  if (j == 0) t = boi;
  else if (j == 33) t = eoi;
  else t = ids[(long long)img * 32 + (j - 1)] + shift;
  out[(long long)img * out_stride + j] = t;
}

int image_ids_to_tokens(const int64_t* ids, int n, int64_t shift, int64_t boi, int64_t eoi, int64_t* out,
                        int64_t out_stride, cudaStream_t stream) {
  SB_REQUIRE(ids && out && n >= 1 && out_stride >= 34, "image_ids_to_tokens: bad arguments");
  const int total = n * 34;
  image_ids_to_tokens_kernel<<<(total + 255) / 256, 256, 0, stream>>>(
      reinterpret_cast<const long long*>(ids), n, shift, boi, eoi, reinterpret_cast<long long*>(out), out_stride);
  SB_LAUNCH_CHECK();
  return 0;
}

}  // namespace sb

extern "C" {

int seedb200_sample(const void* logits, int64_t ld, int B, int V, const seedb200_sample_params* sp, uint64_t step,
                    int64_t* tokens_out, void* stream) {
  SB_REQUIRE(sp != nullptr, "seedb200_sample: null parameters");
  sb::GenParams gp;
  gp.sp = *sp; gp.eos = -1; gp.pad = 0;
  return sb::sample(logits, ld, B, V, &gp, nullptr, step, nullptr, 0, tokens_out, nullptr, 0, nullptr,
                    static_cast<cudaStream_t>(stream));
}

float seedb200_philox_uniform(uint64_t seed, uint64_t offset, uint32_t row) {
  return sb::philox_uniform(seed, offset, row);
}

int seedb200_beam_select(const void* logits, int64_t seq_ld, int64_t beam_ld, int B, int V, const float* beam_scores,
                         const seedb200_beam_params* bp, uint64_t step, float* cand_score, int32_t* cand_idx,
                         void* stream) {
  SB_REQUIRE(bp != nullptr, "seedb200_beam_select: null parameters");
  SB_REQUIRE(bp->num_beams >= 1 && bp->num_beams <= sb::BEAM_MAX && B >= 1,
             "seedb200_beam_select: bad sizes (B %d, k %d in [1,%d])", B, bp->num_beams, sb::BEAM_MAX);
  sb::BeamParams p = sb::beam_params(*bp, -1, 0, 0, 0, B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* row_stats = nullptr;     // per-call scratch of the row statistics (the handle path keeps its own)
  SB_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&row_stats), (size_t)B * bp->num_beams * 5 * sizeof(float), st));
  const int s = sb::beam_select(logits, seq_ld, beam_ld, B, bp->num_beams, V, beam_scores, &p, nullptr, step, nullptr,
                                row_stats, cand_score, cand_idx, st);
  cudaFreeAsync(row_stats, st);
  return s;
}

int seedb200_image_ids_to_tokens(const int64_t* ids, int n, int64_t image_id_shift, int64_t boi, int64_t eoi,
                                 int64_t* tokens_out, int64_t out_stride, void* stream) {
  return sb::image_ids_to_tokens(ids, n, image_id_shift, boi, eoi, tokens_out, out_stride,
                                 static_cast<cudaStream_t>(stream));
}

}  // extern "C"
