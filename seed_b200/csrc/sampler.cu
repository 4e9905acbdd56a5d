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
#include "select.cuh"

namespace sb {

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
  int* state;                          // ... state[GS_STEP] when non-null: the GenSlot counters, advanced by the last
                                       //     CTA to finish
  int advance_cache;                   // also bump the cache length (a decode forward consumed the previous token)
  long long* tokens;                   // [B] next token per sequence (also the next step's input ids)
  long long* out; long long out_ld;    // optional [B, out_ld] history: out[b, gp.proc.S + step] = token (columns
                                       //     [0, S) hold the prompt when a history control reads it)
  int* finished;                       // optional [B]: sequences that already produced eos emit pad (HF semantics)
  int B;
};

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

// fp16 <-> a 16-bit key in the same order (larger value, larger key; -0 sorts just below +0)
__device__ __forceinline__ uint32_t half_key(__half h) {
  const uint32_t u = __half_as_ushort(h);
  return (u & 0x8000u) ? (~u & 0xFFFFu) : (u | 0x8000u);
}
__device__ __forceinline__ float key_half(uint32_t k) {
  return __half2float(__ushort_as_half((unsigned short)((k & 0x8000u) ? (k & 0x7FFFu) : (~k & 0xFFFFu))));
}

// the kk-th largest (1-based) of the fp16 values val(i) of the block's elements (this thread: [i0, i1)): two passes of
// a 256-bin histogram, high byte then low byte.  Every thread returns it.
template <typename Val>
__device__ float kth_largest(const Val& val, int i0, int i1, int kk, unsigned* hist, int* sel) {
  uint32_t prefix = 0u;
  int rem = kk;
  for (int pass = 0; pass < 2; ++pass) {
    for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0u;
    __syncthreads();
    for (int i = i0; i < i1; ++i) {
      const uint32_t key = half_key(val(i));
      if (pass == 0) atomicAdd(&hist[key >> 8], 1u);
      else if ((key >> 8) == prefix) atomicAdd(&hist[key & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int r = rem, b = 255;
      for (; b > 0 && (int)hist[b] < r; --b) r -= (int)hist[b];
      sel[0] = b; sel[1] = r;
    }
    __syncthreads();
    prefix = pass == 0 ? (uint32_t)sel[0] : (prefix << 8) | (uint32_t)sel[0];
    rem = sel[1];
    __syncthreads();
  }
  return key_half(prefix);
}

// ---- history processors (seedb200_logits_params), in place, one CTA per row ------------------------------------
template <typename Tok>
struct ProcArgs {
  __half* logits; long long seq_ld, beam_ld; int V;
  LogitsProc p; const LogitsProc* p_dev;
  const int* state;
  const Tok* hist; long long hist_ld; int hist_rows, hist_len;
  int log_softmax;
};

template <typename Tok>
__global__ void __launch_bounds__(SEL_THREADS)
logits_process_kernel(const ProcArgs<Tok> a) {
  extern __shared__ uint32_t s_seen[];       // one bit per vocabulary id: the row's distinct history tokens
  __shared__ float red[SEL_WARPS];
  const int j = blockIdx.x, sq = blockIdx.y, tid = threadIdx.x;
  pdl_trigger();
  pdl_wait();
  const LogitsProc p = a.p_dev ? *a.p_dev : a.p;
  const int V = a.V;
  __half* row = a.logits + (long long)sq * a.seq_ld + (long long)j * a.beam_ld;
  const Tok* h = a.hist + ((long long)sq * a.hist_rows + j) * a.hist_ld;
  const int L = a.state ? p.S + a.state[GS_STEP] : a.hist_len;
  if (a.log_softmax) {
    // lp = fp16((x - max) - logZ): beam_row_stats_kernel's arithmetic (same chunks, same reduction order)
    const int per = (V + SEL_THREADS - 1) / SEL_THREADS;
    const int i0 = min(V, tid * per), i1 = min(V, i0 + per);
    float m = -INFINITY;
    for (int i = i0; i < i1; ++i) m = fmaxf(m, __half2float(row[i]));
    m = block_max(m, red);
    const float lz = logf(block_exp_sum(row, i0, i1, m, red));
    for (int i = i0; i < i1; ++i) row[i] = __float2half_rn((__half2float(row[i]) - m) - lz);
  }
  const int nw = (V + 31) >> 5;
  const float pen = p.lp.repetition_penalty;
  if (pen != 1.0f) {
    for (int w = tid; w < nw; w += SEL_THREADS) s_seen[w] = 0u;
    __syncthreads();
    for (int t = tid; t < L; t += SEL_THREADS) {
      const long long tok = (long long)h[t];
      if (tok >= 0 && tok < V) atomicOr(&s_seen[tok >> 5], 1u << (tok & 31));
    }
    __syncthreads();
    const float inv = 1.0f / pen;            // torch: fp16 tensor / Python scalar = x * fp32 reciprocal
    for (int w = tid; w < nw; w += SEL_THREADS) {
      uint32_t bits = s_seen[w];
      while (bits) {
        const int t = (w << 5) + __ffs(bits) - 1;
        bits &= bits - 1u;
        const float v = __half2float(row[t]);
        row[t] = __float2half_rn(v < 0.0f ? v * pen : v * inv);
      }
    }
  }
  __syncthreads();                           // the bans below overwrite penalised entries
  const int n = p.lp.no_repeat_ngram_size;
  if (n > 0 && L + 1 >= n) {
    for (int i = tid; i <= L - n; i += SEL_THREADS) {
      bool match = true;
      for (int q = 0; q + 1 < n && match; ++q) match = h[i + q] == h[L - n + 1 + q];
      const long long tok = (long long)h[i + n - 1];
      if (match && tok >= 0 && tok < V) row[tok] = __float2half_rn(-INFINITY);
    }
  }
  if (tid == 0 && p.eos >= 0 && p.eos < V && (L < p.lp.min_length || L - p.S < p.lp.min_new_tokens))
    row[p.eos] = __float2half_rn(-INFINITY);
}

template <typename Tok>
int logits_process(void* logits, int64_t seq_ld, int64_t beam_ld, int B, int beams, int V, const LogitsProc* p,
                   const LogitsProc* p_dev, const int* state, const Tok* hist, int64_t hist_ld, int hist_rows,
                   int hist_len, bool log_softmax, cudaStream_t stream) {
  const size_t smem = (size_t)((V + 31) >> 5) * 4;
  SB_REQUIRE(logits && hist && (p || p_dev) && B >= 1 && beams >= 1 && V >= 1 && hist_ld >= 0 && hist_len >= 0,
             "logits_process: bad arguments");
  SB_REQUIRE(smem <= 48 * 1024, "logits_process: vocabulary %d above %d", V, 48 * 1024 * 8);
  ProcArgs<Tok> a;
  memset(&a, 0, sizeof(a));
  a.logits = static_cast<__half*>(logits); a.seq_ld = seq_ld; a.beam_ld = beam_ld; a.V = V;
  if (p) a.p = *p;
  a.p_dev = p_dev; a.state = state; a.hist = hist; a.hist_ld = hist_ld; a.hist_rows = hist_rows;
  a.hist_len = hist_len; a.log_softmax = log_softmax ? 1 : 0;
  SB_CHECK_CUDA(launch_chain(logits_process_kernel<Tok>, dim3(beams, B), dim3(SEL_THREADS), smem, stream, a));
  SB_LAUNCH_CHECK();
  return 0;
}
template int logits_process<int64_t>(void*, int64_t, int64_t, int, int, int, const LogitsProc*, const LogitsProc*,
                                     const int*, const int64_t*, int64_t, int, int, bool, cudaStream_t);
template int logits_process<int>(void*, int64_t, int64_t, int, int, int, const LogitsProc*, const LogitsProc*,
                                 const int*, const int*, int64_t, int, int, bool, cudaStream_t);

int logits_params_check(const char* who, const seedb200_logits_params* p) {
  if (p == nullptr) return 0;
  SB_REQUIRE(p->top_k >= 0, "%s: top_k %d < 0", who, p->top_k);
  SB_REQUIRE(isfinite(p->repetition_penalty) && p->repetition_penalty > 0.0f,
             "%s: repetition_penalty %g must be finite and > 0", who, (double)p->repetition_penalty);
  SB_REQUIRE(p->no_repeat_ngram_size >= 0 && p->min_length >= 0 && p->min_new_tokens >= 0,
             "%s: no_repeat_ngram_size %d, min_length %d and min_new_tokens %d must be >= 0", who,
             p->no_repeat_ngram_size, p->min_length, p->min_new_tokens);
  return 0;
}

__global__ void __launch_bounds__(SEL_THREADS)
sample_kernel(const SampleArgs a) {
  __shared__ float red[SEL_WARPS];
  __shared__ int red_i[SEL_WARPS];
  __shared__ float scan[SEL_THREADS];
  __shared__ unsigned s_hist[256];
  __shared__ int s_sel[2];
  __shared__ int s_pick;
  const int b = blockIdx.x, tid = threadIdx.x;
  pdl_trigger();
  pdl_wait();
  const GenParams gp = a.gp_dev ? *a.gp_dev : a.gp;
  const seedb200_sample_params sp = gp.sp;
  const unsigned long long step = a.state ? (unsigned long long)a.state[GS_STEP] : a.step;
  const __half* row = a.logits + (long long)b * a.ld;
  const int V = a.V;
  // contiguous chunk per thread (the CDF inversion below walks tokens in index order)
  const int per = (V + SEL_THREADS - 1) / SEL_THREADS;
  const int i0 = min(V, tid * per), i1 = min(V, i0 + per);

  // ---- argmax (ties -> lowest index), also the softmax max ----
  float mx = -INFINITY; int mi = 0x7fffffff;
  for (int i = i0; i < i1; ++i) {
    const float x = __half2float(row[i]);
    if (key_better(x, i, mx, mi)) { mx = x; mi = i; }
  }
  block_best(mx, mi, red, red_i, &red[0], &red_i[0]);
  mx = red[0]; mi = red_i[0];
  if (mi == 0x7fffffff) mi = 0;
  int pick = mi;
  // this step's scores row of sequence b (seedb200_gen_outputs), formed where it is written
  auto scores_row = [&]() { return gp.scores + (long long)step * gp.scores_step + (long long)b * gp.scores_pitch; };

  if (sp.do_sample == 0 && gp.scores != nullptr) {     // greedy_search's scores: the processed row, no warpers
    __half* srow = scores_row();
    for (int i = tid; i < V; i += SEL_THREADS) srow[i] = row[i];
  }
  if (sp.do_sample != 0) {
    // p_i = exp((x_i - max) / T)  (unnormalised; TemperatureLogitsWarper then softmax)
    const float inv_t = 1.0f / fmaxf(sp.temperature, 1e-6f);
    const float kk = inv_t * 1.4426950408889634f;
    // top_k: keep the tokens whose tempered fp16 logit (HF: fp16 logits / T, skipped at T == 1) is >= the k'-th
    // largest.  The tempered value is monotone in x, so that is x >= xmin, the least fp16 x whose tempered value
    // reaches the tempered k'-th largest x (-inf: every token).
    float xmin = -INFINITY;
    const int top_k = min(max(gp.proc.lp.top_k, 1), V);
    if (gp.proc.lp.top_k > 0 && top_k < V) {
      const float xk = kth_largest([&](int i) { return row[i]; }, i0, i1, top_k, s_hist, s_sel);
      if (sp.temperature == 1.0f) {
        xmin = xk;
      } else {
        const float inv_tk = 1.0f / sp.temperature;
        auto tk = [&](float x) { return __half2float(__float2half_rn(x * inv_tk)); };
        const float kth = tk(xk);
        uint32_t lo = 0u, hi = half_key(__float2half_rn(xk));      // smallest key with tk(value) >= kth
        while (lo < hi) {
          const uint32_t mid = (lo + hi) >> 1;
          if (tk(key_half(mid)) >= kth) hi = mid; else lo = mid + 1;
        }
        xmin = key_half(lo);
      }
    }
    auto prob = [&](int i) {
      const float x = __half2float(row[i]);
      const float p = exp2f((x - mx) * kk);
      return x < xmin ? 0.0f : p;
    };
    float z = 0.0f;
    for (int i = i0; i < i1; ++i) z += prob(i);
    const float Z = block_sum(z, red);
    // nucleus threshold: smallest t with mass{p > t} < top_p * Z; kept = {p >= t}.  top_p >= 1 keeps everything.
    float thr = 0.0f;
    if (sp.top_p < 1.0f) thr = nucleus_threshold(prob, i0, i1, sp.top_p * Z, red);
    // sample's scores (4.30.2 generation/utils.py sample: next_token_scores after the warpers): the tempered fp16 logit
    // on the kept set the draw below uses, -inf elsewhere (the filter value of TopK / TopP)
    if (gp.scores != nullptr) {
      __half* srow = scores_row();
      const float inv_tk = 1.0f / sp.temperature;
      for (int i = tid; i < V; i += SEL_THREADS) {
        const float x = __half2float(row[i]);
        const __half v = sp.temperature == 1.0f ? row[i] : __float2half_rn(x * inv_tk);
        srow[i] = (x >= xmin && prob(i) >= thr) ? v : __float2half_rn(-INFINITY);
      }
    }
    // inverse CDF over the kept tokens in index order
    float k = 0.0f;
    for (int i = i0; i < i1; ++i) { const float p = prob(i); k += p >= thr ? p : 0.0f; }
    scan[tid] = k;
    __syncthreads();
    // inclusive scan of the 1024 per-thread masses (Hillis-Steele in shared memory)
    for (int o = 1; o < SEL_THREADS; o <<= 1) {
      const float add = tid >= o ? scan[tid - o] : 0.0f;
      __syncthreads();
      scan[tid] += add;
      __syncthreads();
    }
    const float K = scan[SEL_THREADS - 1];
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
    bool was_unfinished;
    a.tokens[b] = emit_token(pick, b, (long long)step, gp, a.finished, a.out, a.out_ld, &was_unfinished);
    if (a.state != nullptr) seq_arrive(a.state, a.B, (int)step, a.advance_cache != 0, was_unfinished);
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
  else {
    a.gp.sp.do_sample = 0; a.gp.sp.temperature = 1.0f; a.gp.sp.top_p = 1.0f; a.gp.sp.seed = 0; a.gp.sp.offset = 0;
    a.gp.eos = -1; a.gp.pad = 0; a.gp.proc = logits_proc(nullptr, -1, 0);
    a.gp.scores = nullptr; a.gp.scores_pitch = 0; a.gp.scores_step = 0;
  }
  a.gp_dev = gp_dev; a.step = step; a.state = state; a.advance_cache = advance_cache;
  a.tokens = reinterpret_cast<long long*>(tokens);
  a.out = reinterpret_cast<long long*>(out); a.out_ld = out_ld;
  a.finished = finished; a.B = B;
  SB_CHECK_CUDA(launch_chain(sample_kernel, dim3(B), dim3(SEL_THREADS), 0, stream, a));
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
  float* row_stats;                    // [B*k, 5]: max, logZ (0 for processed rows), top-k threshold on w (-inf:
                                       // none), max w, nucleus threshold; the beam score is read from beam_scores
  float* cand_score; int* cand_idx;    // [B, 2k]
};

// s = float(fp16 log_softmax(x)) + beam score; a processed row already holds the fp16 log_softmax
__device__ __forceinline__ float beam_s(bool processed, float x, float mx, float lz, float bs) {
  return processed ? x + bs : __half2float(__float2half_rn((x - mx) - lz)) + bs;
}

__device__ __forceinline__ void top2_merge(float& m1, float& m2, float o1, float o2) {
  const float n2 = fmaxf(fminf(m1, o1), fmaxf(m2, o2));
  m1 = fmaxf(m1, o1);
  m2 = n2;
}

// one CTA per (beam row j, sequence i): the row's statistics, so that the k rows of a sequence run on k SMs
__global__ void __launch_bounds__(SEL_THREADS)
beam_row_stats_kernel(const BeamSelectArgs a) {
  __shared__ float red[SEL_WARPS];
  __shared__ float red2[SEL_WARPS];
  const int j = blockIdx.x, sq = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_trigger();
  pdl_wait();
  const BeamParams bp = a.bp_dev ? *a.bp_dev : a.bp;
  const int k = bp.k, V = a.V;
  if (j >= k) return;
  const float T = bp.temperature;
  const int per = (V + SEL_THREADS - 1) / SEL_THREADS;
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
  const bool processed = bp.processed != 0;
  float lz = 0.0f;
  if (!processed) lz = logf(block_exp_sum(row, i0, i1, m1, red));
  // beam_search's scores (4.30.2 generation/utils.py: scores += (next_token_scores_processed,)): the processed fp16
  // log_softmax, before the beam score.  At step 0 every beam row reads its sequence's one row (beam_ld 0), so the k
  // rows of a sequence are identical.
  if (bp.scores != nullptr) {
    const long long step = a.state ? a.state[GS_STEP] : (long long)a.step;
    __half* srow = bp.scores + step * bp.scores_step + (long long)(sq * k + j) * bp.scores_pitch;
    for (int i = tid; i < V; i += SEL_THREADS)
      srow[i] = processed ? row[i] : __float2half_rn((__half2float(row[i]) - m1) - lz);
  }
  const float bsc = a.beam_scores[sq * k + j];
  // s = float(fp16 log_softmax) + beam score, fp32 (processed rows hold the fp16 log_softmax already)
  auto score = [&](float x) { return beam_s(processed, x, m1, lz, bsc); };
  float mxw = 0.0f, thr = 0.0f, wk = -INFINITY;
  if (bp.do_sample != 0) {
    mxw = score(m1) / T;                   // every step is monotone in x: the largest x gives the largest w
    // top_k on w (min_tokens_to_keep 2): w is monotone in the row value, so the k'-th largest w is w(k'-th value)
    const int top_k = min(max(bp.proc.lp.top_k, 2), V);
    if (bp.proc.lp.top_k > 0 && top_k < V) {
      __shared__ unsigned s_hist[256];
      __shared__ int s_sel[2];
      wk = score(kth_largest([&](int i) { return row[i]; }, i0, i1, top_k, s_hist, s_sel)) / T;
    }
    const bool use_k = wk != -INFINITY;
    auto prob = [&](int i) {
      const float w = score(__half2float(row[i])) / T;
      const float p = exp2f((w - mxw) * 1.4426950408889634f);
      return (use_k && w < wk) ? 0.0f : p;
    };
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
    o[0] = m1; o[1] = lz; o[2] = wk; o[3] = mxw; o[4] = thr;
  }
}

template <int NC>
__global__ void __launch_bounds__(SEL_THREADS)
beam_select_kernel(const BeamSelectArgs a) {
  __shared__ float red[SEL_WARPS];
  __shared__ int redi[SEL_WARPS];
  __shared__ float s_mx[BEAM_MAX], s_lz[BEAM_MAX], s_bs[BEAM_MAX], s_mxw[BEAM_MAX], s_thr[BEAM_MAX], s_wk[BEAM_MAX];
  __shared__ float s_key[2 * BEAM_MAX];
  __shared__ int s_idx[2 * BEAM_MAX];
  const int sq = blockIdx.x, tid = threadIdx.x;
  pdl_trigger();
  pdl_wait();
  const BeamParams bp = a.bp_dev ? *a.bp_dev : a.bp;
  const unsigned long long step = a.state ? (unsigned long long)a.state[GS_STEP] : a.step;
  const int k = bp.k, n2 = 2 * k, V = a.V;
  const bool samp = bp.do_sample != 0, processed = bp.processed != 0;
  const float T = bp.temperature;
  auto rowp = [&](int j) { return a.logits + (long long)sq * a.seq_ld + (long long)j * a.beam_ld; };
  auto score = [&](int j, float x) { return beam_s(processed, x, s_mx[j], s_lz[j], s_bs[j]); };
  if (tid < k) {
    const float* st = a.row_stats + (long long)(sq * k + tid) * 5;
    s_mx[tid] = st[0]; s_lz[tid] = st[1]; s_wk[tid] = st[2]; s_mxw[tid] = st[3]; s_thr[tid] = st[4];
    s_bs[tid] = a.beam_scores[sq * k + tid];
  }
  __syncthreads();
  // ---- per-thread best NC candidates, flat index f = j * V + t in increasing order ----
  BestList<NC> best;
  for (int j = 0; j < k; ++j) {
    const __half* row = rowp(j);
    for (int t = tid; t < V; t += SEL_THREADS) {
      const float sc = score(j, __half2float(row[t]));
      const int f = j * V + t;
      float key = sc;
      if (samp) {
        const float w = sc / T;
        const float p = exp2f((w - s_mxw[j]) * 1.4426950408889634f);
        key = -INFINITY;
        if (p >= s_thr[j] && !(s_wk[j] != -INFINITY && w < s_wk[j])) {
          const float u = philox_open_uniform(bp.seed, bp.offset + step, (uint32_t)sq, (uint32_t)f);
          key = w + (-logf(-logf(u)));
        }
      }
      best.insert(key, f);
    }
  }
  best.pop_rounds(n2, red, redi, s_key, s_idx);     // 2k rounds: the best head of all threads wins and is popped
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
    while (q > 0 && key_better(w, f, sc[q - 1], ix[q - 1])) { sc[q] = sc[q - 1]; ix[q] = ix[q - 1]; --q; }
    sc[q] = w; ix[q] = f;
  }
  for (int r = 0; r < n2; ++r) {
    a.cand_score[(long long)sq * n2 + r] = sc[r];
    a.cand_idx[(long long)sq * n2 + r] = ix[r];
  }
}

// beam_sample's scores (4.30.2 generation/utils.py: scores += (logits_warper(input_ids,
// next_token_scores_processed),)): the warpers on the processed fp16 row, without the beam score, in place on the rows
// beam_row_stats_kernel wrote.  One CTA per (beam row j, sequence).  Temperature v = fp16(x * fp32(1 / T)) (x at
// T == 1); TopK keeps v >= the k'-th largest v, k' = min(max(top_k, 2), V); TopP keeps p = exp(v - max) >= the nucleus
// threshold of the TopK-kept tokens, lowered to the second largest v's p (min_tokens_to_keep 2).  Removed: -inf.
__global__ void __launch_bounds__(SEL_THREADS)
beam_scores_warp_kernel(const BeamSelectArgs a) {
  __shared__ float red[SEL_WARPS];
  __shared__ unsigned s_hist[256];
  __shared__ int s_sel[2];
  const int j = blockIdx.x, sq = blockIdx.y, tid = threadIdx.x;
  pdl_trigger();
  pdl_wait();
  const BeamParams bp = a.bp_dev ? *a.bp_dev : a.bp;
  const int k = bp.k, V = a.V;
  if (j >= k || bp.scores == nullptr) return;
  const long long step = a.state ? a.state[GS_STEP] : (long long)a.step;
  __half* row = bp.scores + step * bp.scores_step + (long long)(sq * k + j) * bp.scores_pitch;
  const int per = (V + SEL_THREADS - 1) / SEL_THREADS;
  const int i0 = min(V, tid * per), i1 = min(V, i0 + per);
  const float T = bp.temperature, inv = 1.0f / T;
  auto val = [&](int i) { return T == 1.0f ? row[i] : __float2half_rn(__half2float(row[i]) * inv); };
  const float vmax = kth_largest(val, i0, i1, 1, s_hist, s_sel);
  float vk = -INFINITY;
  const int top_k = min(max(bp.proc.lp.top_k, 2), V);
  if (bp.proc.lp.top_k > 0 && top_k < V) vk = kth_largest(val, i0, i1, top_k, s_hist, s_sel);
  auto prob = [&](int i) {
    const float v = __half2float(val(i));
    return v < vk ? 0.0f : exp2f((v - vmax) * 1.4426950408889634f);
  };
  float thr = 0.0f;
  if (bp.top_p < 1.0f) {
    float z = 0.0f;
    for (int i = i0; i < i1; ++i) z += prob(i);
    const float Z = block_sum(z, red);
    const float v2 = kth_largest(val, i0, i1, 2, s_hist, s_sel);
    thr = fminf(nucleus_threshold(prob, i0, i1, bp.top_p * Z, red),
                v2 == -INFINITY ? 0.0f : exp2f((v2 - vmax) * 1.4426950408889634f));
  }
  // every reduction above has completed (each ends in a block barrier); each element is read and written by one thread
  for (int i = tid; i < V; i += SEL_THREADS) {
    const __half v = val(i);
    row[i] = (__half2float(v) >= vk && prob(i) >= thr) ? v : __float2half_rn(-INFINITY);
  }
}

int beam_select(const void* logits, int64_t seq_ld, int64_t beam_ld, int B, int k, int V, const float* beam_scores,
                const BeamParams* bp, const BeamParams* bp_dev, uint64_t step, const int* state, float* row_stats,
                float* cand_score, int* cand_idx, cudaStream_t stream, bool warp_scores) {
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
  SB_CHECK_CUDA(launch_chain(beam_row_stats_kernel, dim3(k, B), dim3(SEL_THREADS), 0, stream, a));
  SB_LAUNCH_CHECK();
  if (warp_scores) {
    SB_CHECK_CUDA(launch_chain(beam_scores_warp_kernel, dim3(k, B), dim3(SEL_THREADS), 0, stream, a));
    SB_LAUNCH_CHECK();
  }
  const int n2 = 2 * k;
  auto kern = n2 <= 4 ? beam_select_kernel<4> : (n2 <= 8 ? beam_select_kernel<8> : beam_select_kernel<16>);
  SB_CHECK_CUDA(launch_chain(kern, dim3(B), dim3(SEL_THREADS), 0, stream, a));
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
  return seedb200_sample_processed(const_cast<void*>(logits), ld, B, V, sp, step, tokens_out, stream, nullptr, nullptr,
                                   0, 0, 0, -1);
}

int seedb200_sample_processed(void* logits, int64_t ld, int B, int V, const seedb200_sample_params* sp, uint64_t step,
                              int64_t* tokens_out, void* stream, const seedb200_logits_params* lp,
                              const int64_t* history, int64_t hist_ld, int hist_len, int prompt_len, int64_t eos_id) {
  return seedb200_sample_scores(logits, ld, B, V, sp, step, tokens_out, stream, lp, history, hist_ld, hist_len,
                                prompt_len, eos_id, nullptr, 0);
}

int seedb200_sample_scores(void* logits, int64_t ld, int B, int V, const seedb200_sample_params* sp, uint64_t step,
                           int64_t* tokens_out, void* stream, const seedb200_logits_params* lp,
                           const int64_t* history, int64_t hist_ld, int hist_len, int prompt_len, int64_t eos_id,
                           void* scores_out, int64_t scores_ld) {
  SB_REQUIRE(sp != nullptr, "seedb200_sample: null parameters");
  SB_PROPAGATE(sb::logits_params_check("seedb200_sample_processed", lp));
  SB_REQUIRE(scores_out == nullptr || (scores_ld >= V && scores_ld % 8 == 0 && (uintptr_t)scores_out % 16 == 0),
             "seedb200_sample_scores: scores rows need a pitch >= V %d that is a multiple of 8 (got %lld) and a "
             "16-byte aligned base", V, (long long)scores_ld);
  sb::GenParams gp;
  gp.sp = *sp; gp.eos = -1; gp.pad = 0;
  gp.proc = sb::logits_proc(lp, eos_id, prompt_len);
  gp.scores = static_cast<__half*>(scores_out); gp.scores_pitch = scores_ld; gp.scores_step = 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (sb::logits_history_active(gp.proc)) {
    SB_REQUIRE(history != nullptr && hist_len >= 0 && hist_ld >= hist_len && prompt_len >= 0 && prompt_len <= hist_len,
               "seedb200_sample_processed: a history control needs history [B, >= hist_len %d] and prompt_len %d <= it",
               hist_len, prompt_len);
    SB_REQUIRE(logits && B >= 1 && V >= 1 && ld >= V, "sample: bad arguments");
    SB_PROPAGATE(sb::logits_process<int64_t>(logits, ld, 0, B, 1, V, &gp.proc, nullptr, nullptr, history, hist_ld, 1,
                                             hist_len, false, st));
  }
  return sb::sample(logits, ld, B, V, &gp, nullptr, step, nullptr, 0, tokens_out, nullptr, 0, nullptr, st);
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
