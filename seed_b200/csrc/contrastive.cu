// contrastive.cu -- contrastive search on the device (transformers 4.30.2 GenerationMixin.contrastive_search with
// _ranking_fast, stated in include/seedb200.h next to seedb200_contrastive_params).
//
//   contrastive_candidates_kernel  one CTA per sequence: fp16 softmax of the (processed) logits row, then the top k
//                                  probabilities (descending, ties to the lower id).  Each thread keeps its own best k
//                                  in registers over a contiguous chunk; k block-wide rounds pop the best head.  Points
//                                  the lineage entry of every candidate row at position p to the row itself, where
//                                  the candidate forward appends its K/V.
//   contrastive_rank_kernel        (CTAs, sequence): every CTA streams a slice of the sequence's normalised context once
//                                  and dots each row with the k normalised candidates staged in shared memory; per-CTA
//                                  maxima go to a workspace.  The last CTA to arrive (a ticket per sequence) scores the
//                                  candidates, appends n(h_sel) to the context and, in the generation loop, makes the
//                                  selected candidate the sequence's own: logits row, lineage entry at p, output token,
//                                  finished flag and the device counters.
//   contrastive_context_init_kernel  normalises the prompt's final hidden states into the context and points every
//                                  candidate row's lineage at the prefill row of its sequence for positions < S.
#include <string.h>

#include "common.cuh"
#include "ops.h"
#include "select.cuh"

namespace sb {

constexpr int RANK_THREADS = 256;
constexpr int RANK_WARPS = RANK_THREADS / 32;
static_assert(RANK_WARPS >= CONTRAST_MAX_K, "one warp per candidate");
constexpr int RANK_MIN_ROWS = 16;        // context rows per CTA at least: below that, staging the candidates dominates
constexpr int RANK_MAX_SMEM = 200 * 1024;   // k * hidden fp16: 8 candidates up to hidden 12800

// torch.max: NaN propagates
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fffffff) : fmaxf(a, b); }

// n(x) = fp16(float(x) / float(fp16(sqrt(sum of float(x)^2)))), one warp per row of H halves (H % 8 == 0, 16-byte rows)
__device__ void normalise_row(const __half* __restrict__ src, __half* __restrict__ dst, int H, int lane) {
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  uint4* d4 = reinterpret_cast<uint4*>(dst);
  float ss = 0.0f;
#pragma unroll 4
  for (int c = lane; c < H / 8; c += 32) {
    const uint4 u = s4[c];
    const __half* x = reinterpret_cast<const __half*>(&u);
#pragma unroll
    for (int e = 0; e < 8; ++e) { const float f = __half2float(x[e]); ss += f * f; }
  }
  ss = warp_sum(ss);
  const float nrm = __half2float(__float2half_rn(sqrtf(ss)));
#pragma unroll 4
  for (int c = lane; c < H / 8; c += 32) {
    const uint4 u = s4[c];
    const __half* x = reinterpret_cast<const __half*>(&u);
    uint4 o;
    __half* y = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] = __float2half_rn(__half2float(x[e]) / nrm);
    d4[c] = o;
  }
}

// ---- candidates ---------------------------------------------------------------------------------------------------
struct CandArgs {
  const __half* logits; long long ld; int V;
  ContrastParams p; const ContrastParams* p_dev;
  const int* state; int pos;           // candidates' position p: state[GS_CACHE_LEN] when state is given
  int* slot; int max_seq;              // optional lineage table [B*k, max_seq]
  long long* ids; __half* probs;       // [B*k]
  const GenParams* gp_dev;             // optional (with state): the loop's parameters, whose scores buffer receives
                                       // the row the candidates are taken from
};

__global__ void __launch_bounds__(SEL_THREADS) contrastive_candidates_kernel(const CandArgs a) {
  __shared__ float red[SEL_WARPS];
  __shared__ int redi[SEL_WARPS];
  __shared__ float s_key[CONTRAST_MAX_K];
  __shared__ int s_idx[CONTRAST_MAX_K];
  const int b = blockIdx.x, tid = threadIdx.x;
  pdl_trigger();
  pdl_wait();
  const int k = a.p_dev ? a.p_dev->k : a.p.k;
  const int V = a.V;
  const __half* row = a.logits + (long long)b * a.ld;
  const int per = (V + SEL_THREADS - 1) / SEL_THREADS;
  const int i0 = min(V, tid * per), i1 = min(V, i0 + per);
  // contrastive_search's scores (4.30.2 generation/utils.py: scores += (logit_for_next_step,)): the processed row
  if (a.gp_dev != nullptr && a.state != nullptr && a.gp_dev->scores != nullptr) {
    __half* srow = a.gp_dev->scores + (long long)a.state[GS_STEP] * a.gp_dev->scores_step +
                   (long long)b * a.gp_dev->scores_pitch;
    for (int i = tid; i < V; i += SEL_THREADS) srow[i] = row[i];
  }
  float mx = -INFINITY;
  for (int i = i0; i < i1; ++i) mx = fmaxf(mx, __half2float(row[i]));
  mx = block_max(mx, red);
  const float inv = 1.0f / block_exp_sum(row, i0, i1, mx, red);
  // softmax in fp16: torch's CUDA epilogue exp(x - max) * fp32(1 / sum), one rounding
  BestList<CONTRAST_MAX_K> best;
  for (int i = i0; i < i1; ++i) best.insert(__half2float(__float2half_rn(expf(__half2float(row[i]) - mx) * inv)), i);
  best.pop_rounds(k, red, redi, s_key, s_idx);
  if (tid < k) {
    const int r = b * k + tid;
    a.ids[r] = s_idx[tid];
    a.probs[r] = __float2half_rn(s_key[tid]);
    const int pos = a.state ? a.state[GS_CACHE_LEN] : a.pos;
    if (a.slot != nullptr && pos < a.max_seq) a.slot[(long long)r * a.max_seq + pos] = r;
  }
}

int contrastive_candidates(const void* logits, int64_t ld, int B, int V, const ContrastParams* p,
                           const ContrastParams* p_dev, const int* state, int pos, int* slot, int max_seq,
                           int64_t* ids, void* probs, cudaStream_t stream, const GenParams* gp_dev) {
  SB_REQUIRE(logits && ids && probs && (p || p_dev) && B >= 1 && V >= CONTRAST_MAX_K && ld >= V,
             "contrastive_candidates: bad arguments (B %d, V %d >= %d, ld %lld)", B, V, CONTRAST_MAX_K, (long long)ld);
  CandArgs a;
  memset(&a, 0, sizeof(a));
  a.logits = static_cast<const __half*>(logits); a.ld = ld; a.V = V;
  if (p) a.p = *p;
  a.p_dev = p_dev; a.state = state; a.pos = pos; a.slot = slot; a.max_seq = max_seq;
  a.ids = reinterpret_cast<long long*>(ids); a.probs = static_cast<__half*>(probs);
  a.gp_dev = gp_dev;
  SB_CHECK_CUDA(launch_chain(contrastive_candidates_kernel, dim3(B), dim3(SEL_THREADS), 0, stream, a));
  SB_LAUNCH_CHECK();
  return 0;
}

// ---- rank + select ------------------------------------------------------------------------------------------------
struct RankArgs {
  __half* ctx; long long ctx_ld;       // context row i of sequence b: ctx + b * ctx_ld + i * H (normalised)
  int ctx_rows;                        // n(h_sel) is appended at row p when p < ctx_rows
  int H;
  const __half* h;                     // [B*k, H] candidates' final hidden states
  const __half* probs;                 // [B*k]
  ContrastParams p; const ContrastParams* p_dev;
  int* state; int pos;                 // p = context rows: state[GS_CACHE_LEN] when state is given (the loop's counters)
  float* part; int* tickets; int G;    // [B, G, CONTRAST_MAX_K] per-CTA maxima; [B] arrival counters, left 0
  int* sel; float* score;              // optional [B], [B*k]
  // the generation loop's bookkeeping (state != NULL)
  const long long* cand_ids;           // [B*k]
  const __half* cand_logits; __half* seq_logits; long long vpad;   // row b*k+sel -> row b
  int* slot; int max_seq;
  const GenParams* gp;                 // eos, pad, prompt length
  long long* out; long long out_ld;    // out[b, S + step] = token
  int* finished;
  int B;
};

__global__ void __launch_bounds__(RANK_THREADS) contrastive_rank_kernel(const RankArgs a) {
  extern __shared__ __align__(16) __half s_h[];       // [k, H] normalised candidates
  __shared__ float s_max[RANK_WARPS][CONTRAST_MAX_K];
  __shared__ float s_pen[CONTRAST_MAX_K];
  __shared__ int s_last, s_sel;
  const int b = blockIdx.y, cta = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_trigger();
  pdl_wait();
  const ContrastParams cp = a.p_dev ? *a.p_dev : a.p;
  const int k = cp.k, H = a.H;
  const int P = a.state ? a.state[GS_CACHE_LEN] : a.pos;
  const int rpc = max(RANK_MIN_ROWS, (P + a.G - 1) / a.G);
  const int r0 = cta * rpc, r1 = min(P, r0 + rpc);
  const bool active = r0 < r1;
  auto stage = [&]() {
    for (int j = warp; j < k; j += RANK_WARPS)
      normalise_row(a.h + (long long)(b * k + j) * H, s_h + (long long)j * H, H, lane);
    __syncthreads();
  };
  float mxj[CONTRAST_MAX_K];
#pragma unroll
  for (int j = 0; j < CONTRAST_MAX_K; ++j) mxj[j] = -INFINITY;
  if (active) {
    stage();
    const uint4* sh4 = reinterpret_cast<const uint4*>(s_h);
    const int H8 = H / 8;
    for (int r = r0 + warp; r < r1; r += RANK_WARPS) {
      const uint4* crow = reinterpret_cast<const uint4*>(a.ctx + (long long)b * a.ctx_ld + (long long)r * H);
      float acc[CONTRAST_MAX_K];
#pragma unroll
      for (int j = 0; j < CONTRAST_MAX_K; ++j) acc[j] = 0.0f;
#pragma unroll 2
      for (int c = lane; c < H8; c += 32) {
        const uint4 u = crow[c];
        const __half2* x = reinterpret_cast<const __half2*>(&u);
        float2 xf[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) xf[e] = __half22float2(x[e]);
#pragma unroll
        for (int j = 0; j < CONTRAST_MAX_K; ++j) {
          if (j < k) {
            const uint4 w = sh4[j * H8 + c];
            const __half2* y = reinterpret_cast<const __half2*>(&w);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 yf = __half22float2(y[e]);
              acc[j] = fmaf(xf[e].x, yf.x, acc[j]);
              acc[j] = fmaf(xf[e].y, yf.y, acc[j]);
            }
          }
        }
      }
#pragma unroll
      for (int j = 0; j < CONTRAST_MAX_K; ++j)
        if (j < k) mxj[j] = nan_max(mxj[j], __half2float(__float2half_rn(warp_sum(acc[j]))));
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < CONTRAST_MAX_K; ++j) s_max[warp][j] = mxj[j];
  }
  __syncthreads();
  if (tid < k) {
    float m = -INFINITY;
    for (int w = 0; w < RANK_WARPS; ++w) m = nan_max(m, s_max[w][tid]);
    a.part[((long long)b * a.G + cta) * CONTRAST_MAX_K + tid] = m;
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(&a.tickets[b], 1) == a.G - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (!active) stage();                                // the append needs n(h_sel)
  if (warp < k) {                                      // warp j: pen_j over the CTAs' maxima (k <= RANK_WARPS)
    float pen = -INFINITY;
    for (int c = lane; c < a.G; c += 32)
      pen = nan_max(pen, __ldcg(a.part + ((long long)b * a.G + c) * CONTRAST_MAX_K + warp));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) pen = nan_max(pen, __shfl_xor_sync(0xffffffffu, pen, o));
    if (lane == 0) s_pen[warp] = pen;
  }
  __syncthreads();
  if (tid == 0) {
    a.tickets[b] = 0;
    int best = 0;
    float bs = 0.0f;
    for (int j = 0; j < k; ++j) {
      const float pen = s_pen[j];
      const float q = __half2float(a.probs[b * k + j]);
      const float t1 = __half2float(__float2half_rn(cp.c_prob * q));
      const float t2 = __half2float(__float2half_rn(cp.c_pen * pen));
      const float sc = __half2float(__float2half_rn(t1 - t2));
      if (a.score) a.score[b * k + j] = sc;
      // argmax, ties to the lower j; the first NaN wins (torch.max)
      if (j == 0 || (bs == bs && (sc != sc || sc > bs))) { best = j; bs = sc; }
    }
    s_sel = best;
    if (a.sel) a.sel[b] = best;
  }
  __syncthreads();
  const int sel = s_sel;
  if (P < a.ctx_rows) {
    const uint4* src = reinterpret_cast<const uint4*>(s_h + (long long)sel * H);
    uint4* dst = reinterpret_cast<uint4*>(a.ctx + (long long)b * a.ctx_ld + (long long)P * H);
    for (int c = tid; c < H / 8; c += RANK_THREADS) dst[c] = src[c];
  }
  if (a.state == nullptr) return;
  const int r = b * k + sel;
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.cand_logits + (long long)r * a.vpad);
    uint4* dst = reinterpret_cast<uint4*>(a.seq_logits + (long long)b * a.vpad);
    for (long long c = tid; c < a.vpad / 8; c += RANK_THREADS) dst[c] = src[c];
  }
  if (tid < k && P < a.max_seq) a.slot[(long long)(b * k + tid) * a.max_seq + P] = r;
  if (tid == 0) {
    const int step = a.state[GS_STEP];
    bool was_unfinished;
    emit_token(a.cand_ids[r], b, step, *a.gp, a.finished, a.out, a.out_ld, &was_unfinished);
    seq_arrive(a.state, a.B, step, true, was_unfinished);
  }
}

int contrastive_rank_ctas(int max_rows, int B) {
  int g = (max_rows + RANK_MIN_ROWS - 1) / RANK_MIN_ROWS;
  const int cap = (2 * num_sms() + B - 1) / B;
  if (g > cap) g = cap;
  if (g > CONTRAST_MAX_CTAS) g = CONTRAST_MAX_CTAS;
  return g < 1 ? 1 : g;
}

int contrastive_rank(const ContrastRank& r, cudaStream_t stream) {
  const int k = r.k;
  SB_REQUIRE(r.ctx && r.h && r.probs && r.part && r.tickets && (r.p || r.p_dev) && r.B >= 1 && k >= 2 &&
             k <= CONTRAST_MAX_K && r.H >= 8 && r.H % 8 == 0 && r.G >= 1 && r.G <= CONTRAST_MAX_CTAS,
             "contrastive_rank: bad arguments (B %d, k %d, hidden %d, ctas %d)", r.B, k, r.H, r.G);
  SB_REQUIRE(aligned16(r.ctx) && aligned16(r.h) && r.ctx_ld % 8 == 0, "contrastive_rank: context and hidden states "
             "must be 16-byte aligned with a row stride that is a multiple of 8");
  RankArgs a;
  memset(&a, 0, sizeof(a));
  a.ctx = r.ctx; a.ctx_ld = r.ctx_ld; a.ctx_rows = r.ctx_rows; a.H = r.H; a.h = r.h; a.probs = r.probs;
  if (r.p) a.p = *r.p;
  a.p_dev = r.p_dev; a.state = r.state; a.pos = r.pos; a.part = r.part; a.tickets = r.tickets; a.G = r.G;
  a.sel = r.sel; a.score = r.score; a.cand_ids = r.cand_ids; a.cand_logits = r.cand_logits;
  a.seq_logits = r.seq_logits; a.vpad = r.vpad; a.slot = r.slot; a.max_seq = r.max_seq; a.gp = r.gp; a.out = r.out;
  a.out_ld = r.out_ld; a.finished = r.finished; a.B = r.B;
  const size_t smem = (size_t)k * r.H * 2;
  SB_REQUIRE(smem <= RANK_MAX_SMEM, "contrastive_rank: %d candidates of hidden %d exceed shared memory", k, r.H);
  static bool attr_set_dev[SB_MAX_DEVICES] = {};   // cudaFuncSetAttribute is per device
  bool& attr_set = attr_set_dev[cur_device()];
  if (!attr_set) {
    SB_CHECK_CUDA(cudaFuncSetAttribute(contrastive_rank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       RANK_MAX_SMEM));
    attr_set = true;
  }
  SB_CHECK_CUDA(launch_chain(contrastive_rank_kernel, dim3(r.G, r.B), dim3(RANK_THREADS), smem, stream, a));
  SB_LAUNCH_CHECK();
  return 0;
}

// ---- context init -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(RANK_THREADS)
contrastive_context_init_kernel(const __half* __restrict__ hs, int S, int H, __half* __restrict__ ctx, long long ctx_ld,
                                int* slot, int k, int max_seq, ContrastParams p, ContrastParams* p_out) {
  const int b = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * RANK_WARPS + warp;
  if (i < S) normalise_row(hs + ((long long)b * S + i) * H, ctx + (long long)b * ctx_ld + (long long)i * H, H, lane);
  if (slot != nullptr && blockIdx.x == 0)
    for (int e = threadIdx.x; e < k * S; e += RANK_THREADS)
      slot[(long long)(b * k + e / S) * max_seq + e % S] = b;
  if (p_out != nullptr && b == 0 && blockIdx.x == 0 && threadIdx.x == 0) *p_out = p;
}

int contrastive_context_init(const void* hidden_states, int B, int S, int H, void* ctx, int64_t ctx_ld, int* slot,
                             int k, int max_seq, const ContrastParams& p, ContrastParams* p_out, cudaStream_t stream) {
  SB_REQUIRE(hidden_states && ctx && B >= 1 && S >= 1 && H >= 8 && H % 8 == 0 && ctx_ld >= (int64_t)S * H &&
             ctx_ld % 8 == 0, "contrastive_context_init: bad arguments (B %d, S %d, hidden %d, ctx_ld %lld)", B, S, H,
             (long long)ctx_ld);
  SB_REQUIRE(aligned16(hidden_states) && aligned16(ctx), "contrastive_context_init: operands must be 16-byte aligned");
  SB_REQUIRE(slot == nullptr || (S <= max_seq && k >= 1 && k <= CONTRAST_MAX_K), "contrastive_context_init: bad lineage");
  contrastive_context_init_kernel<<<dim3((S + RANK_WARPS - 1) / RANK_WARPS, B), RANK_THREADS, 0, stream>>>(
      static_cast<const __half*>(hidden_states), S, H, static_cast<__half*>(ctx), ctx_ld, slot, k, max_seq, p, p_out);
  SB_LAUNCH_CHECK();
  return 0;
}

int contrastive_params_check(const char* who, const seedb200_contrastive_params* cp) {
  SB_REQUIRE(cp != nullptr, "%s: null contrastive parameters", who);
  SB_REQUIRE(cp->top_k >= 2 && cp->top_k <= CONTRAST_MAX_K, "%s: top_k %d outside [2,%d]", who, cp->top_k,
             CONTRAST_MAX_K);
  SB_REQUIRE(isfinite(cp->penalty_alpha) && cp->penalty_alpha > 0.0, "%s: penalty_alpha %g must be finite and > 0",
             who, cp->penalty_alpha);
  return 0;
}

ContrastParams contrast_params(const seedb200_contrastive_params& cp) {
  ContrastParams p;
  p.k = cp.top_k;
  p.c_prob = (float)(1.0 - cp.penalty_alpha);      // Python's 1.0 - alpha in double, an fp32 scalar of the fp16 op
  p.c_pen = (float)cp.penalty_alpha;
  return p;
}

}  // namespace sb

extern "C" {

int seedb200_contrastive_candidates(const void* logits, int64_t ld, int B, int V, int top_k, int64_t* ids_out,
                                    void* probs_out, void* stream) {
  SB_REQUIRE(top_k >= 2 && top_k <= sb::CONTRAST_MAX_K, "seedb200_contrastive_candidates: top_k %d outside [2,%d]",
             top_k, sb::CONTRAST_MAX_K);
  sb::ContrastParams p;
  p.k = top_k; p.c_prob = 0.0f; p.c_pen = 0.0f;
  return sb::contrastive_candidates(logits, ld, B, V, &p, nullptr, nullptr, 0, nullptr, 0, ids_out, probs_out,
                                    static_cast<cudaStream_t>(stream));
}

int seedb200_contrastive_rank(void* context, int64_t ctx_ld, int ctx_rows, int p, int hidden, const void* cand_hidden,
                              const void* cand_probs, int B, const seedb200_contrastive_params* cp, int32_t* sel_out,
                              float* scores_out, void* stream) {
  SB_PROPAGATE(sb::contrastive_params_check("seedb200_contrastive_rank", cp));
  SB_REQUIRE(context && cand_hidden && cand_probs && B >= 1 && hidden >= 8 && p >= 1 && p <= ctx_rows &&
             ctx_ld >= (int64_t)ctx_rows * hidden, "seedb200_contrastive_rank: bad arguments (B %d, p %d, rows %d, "
             "hidden %d, ctx_ld %lld)", B, p, ctx_rows, hidden, (long long)ctx_ld);
  const sb::ContrastParams cpar = sb::contrast_params(*cp);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int G = sb::contrastive_rank_ctas(p, B);
  // per-call workspace: the maxima and the zeroed tickets (the handle path keeps its own)
  void* ws = nullptr;
  const size_t part_bytes = (size_t)B * G * sb::CONTRAST_MAX_K * sizeof(float);
  SB_CHECK_CUDA(cudaMallocAsync(&ws, part_bytes + (size_t)B * sizeof(int), st));
  int* tickets = reinterpret_cast<int*>(static_cast<char*>(ws) + part_bytes);
  int s = cudaMemsetAsync(tickets, 0, (size_t)B * sizeof(int), st) == cudaSuccess ? 0 : SEEDB200_ERR_CUDA;
  if (s != 0) sb::set_error("seedb200_contrastive_rank: cudaMemsetAsync failed");
  if (s == 0) {
    sb::ContrastRank r;
    memset(&r, 0, sizeof(r));
    r.ctx = static_cast<__half*>(context); r.ctx_ld = ctx_ld; r.ctx_rows = ctx_rows; r.H = hidden;
    r.h = static_cast<const __half*>(cand_hidden); r.probs = static_cast<const __half*>(cand_probs);
    r.p = &cpar; r.k = cpar.k; r.pos = p; r.part = static_cast<float*>(ws); r.tickets = tickets; r.G = G;
    r.sel = sel_out; r.score = scores_out; r.B = B;
    s = sb::contrastive_rank(r, st);
  }
  cudaFreeAsync(ws, st);
  return s;
}

int seedb200_contrastive_context_init(const void* hidden_states, int B, int S, int hidden, void* context,
                                      int64_t ctx_ld, void* stream) {
  sb::ContrastParams p;
  memset(&p, 0, sizeof(p));
  return sb::contrastive_context_init(hidden_states, B, S, hidden, context, ctx_ld, nullptr, 0, 0, p, nullptr,
                                      static_cast<cudaStream_t>(stream));
}

}  // extern "C"
