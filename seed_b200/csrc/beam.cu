// beam.cu -- the bookkeeping side of beam search / beam sampling on the device (transformers 4.30.2
// BeamSearchScorer.process / BeamHypotheses / finalize, stated in include/seedb200.h next to seedb200_beam_params).
//
//   beam_init_kernel      beam scores (0 / -1e9), hypotheses, counters, and the lineage table of the prompt: every beam
//                         of sequence i reads cache row i for positions < S (the prompt is prefilled once, at B rows)
//   beam_score_kernel     one CTA per sequence: thread 0 walks the 2k candidates (process + is_done), then the CTA
//                         gathers the parents' lineage rows and points position `pos` of every beam at its own row,
//                         where the next decode step appends its K/V
//   beam_finalize_kernel  adds the running beams of unfinished sequences, picks the best hypothesis and writes the
//                         generated tokens by walking the (token, parent) history back
#include "common.cuh"
#include "ops.h"

namespace sb {

// BeamHypotheses of one sequence: at most k entries in insertion order (4.30.2 BeamHypotheses.add)
struct Hyps {
  double score[BEAM_MAX + 1];
  int len[BEAM_MAX + 1], beam[BEAM_MAX + 1], step[BEAM_MAX + 1];
  int n;
  double worst;
};

__device__ void hyps_load(const BeamState& s, int i, int k, Hyps& h) {
  h.n = s.hyp_n[i];
  h.worst = s.worst[i];
  for (int q = 0; q < h.n; ++q) {
    h.score[q] = s.hyp_score[i * k + q]; h.len[q] = s.hyp_len[i * k + q];
    h.beam[q] = s.hyp_beam[i * k + q]; h.step[q] = s.hyp_step[i * k + q];
  }
}

__device__ void hyps_store(const BeamState& s, int i, int k, const Hyps& h) {
  s.hyp_n[i] = h.n;
  s.worst[i] = h.worst;
  for (int q = 0; q < h.n; ++q) {
    s.hyp_score[i * k + q] = h.score[q]; s.hyp_len[i * k + q] = h.len[q];
    s.hyp_beam[i * k + q] = h.beam[q]; s.hyp_step[i * k + q] = h.step[q];
  }
}

__device__ void hyps_add(Hyps& h, int k, double lp, double sum_logprobs, int len, int beam, int step) {
  const double score = sum_logprobs / pow((double)len, lp);
  if (h.n < k || score > h.worst) {
    h.score[h.n] = score; h.len[h.n] = len; h.beam[h.n] = beam; h.step[h.n] = step;
    ++h.n;
    if (h.n > k) {
      // sorted((s, idx)): drop the lowest (ties: lowest idx), worst = the second entry of that order
      int lo = 0;
      for (int q = 1; q < h.n; ++q) if (h.score[q] < h.score[lo]) lo = q;
      int second = -1;
      for (int q = 0; q < h.n; ++q)
        if (q != lo && (second < 0 || h.score[q] < h.score[second])) second = q;
      h.worst = h.score[second];
      for (int q = lo; q + 1 < h.n; ++q) {
        h.score[q] = h.score[q + 1]; h.len[q] = h.len[q + 1]; h.beam[q] = h.beam[q + 1]; h.step[q] = h.step[q + 1];
      }
      --h.n;
    } else {
      h.worst = fmin(score, h.worst);
    }
  }
}

__device__ bool hyps_done(const Hyps& h, const BeamParams& bp, double best, int cur_len) {
  if (h.n < bp.k) return false;
  if (bp.early_stopping == 1) return true;
  double denom = pow((double)cur_len, bp.length_penalty);
  if (bp.early_stopping == 2 && bp.length_penalty > 0.0) denom = pow((double)(bp.S + bp.max_new), bp.length_penalty);
  return h.worst >= best / denom;
}

__global__ void beam_init_kernel(BeamParams bp, BeamState s) {
  const int rows = bp.B * bp.k;
  const int g = blockIdx.x * blockDim.x + threadIdx.x, n = gridDim.x * blockDim.x;
  if (g == 0) {
    *s.params = bp;
    s.state[0] = bp.S; s.state[1] = 0; s.state[2] = 0; s.state[3] = 0; s.state[4] = 0; s.state[5] = 0;
  }
  for (int e = g; e < rows; e += n) s.beam_scores[e] = e % bp.k == 0 ? 0.0f : -1e9f;
  for (int e = g; e < bp.B; e += n) { s.done[e] = 0; s.hyp_n[e] = 0; s.worst[e] = 1e9; }
  for (long long e = g; e < (long long)rows * bp.S; e += n) {
    const int b = (int)(e / bp.S), p = (int)(e % bp.S);
    s.slot[(long long)b * s.max_seq + p] = b / bp.k;
  }
}

int beam_init(const BeamState& st, const BeamParams& bp, cudaStream_t stream) {
  long long work = (long long)bp.B * bp.k * bp.S;
  int blocks = (int)((work + 255) / 256);
  if (blocks < 1) blocks = 1;
  if (blocks > 1024) blocks = 1024;
  beam_init_kernel<<<blocks, 256, 0, stream>>>(bp, st);
  SB_LAUNCH_CHECK();
  return 0;
}

__global__ void __launch_bounds__(256) beam_score_kernel(const BeamState s, int V, int advance_cache) {
  __shared__ int s_par[BEAM_MAX];
  const int i = blockIdx.x, tid = threadIdx.x;
  pdl_trigger();
  pdl_wait();
  const BeamParams bp = *s.params;
  const int k = bp.k, n2 = 2 * k, rows = bp.B * k;
  const int step = s.state[1];
  const int cur_len = bp.S + step;                        // input_ids.shape[-1] before this step's append
  const int pos = advance_cache ? s.state[0] + 1 : s.state[0];   // where the next decode step appends
  if (tid == 0) {
    float nbs[BEAM_MAX];
    long long ntok[BEAM_MAX];
    int npar[BEAM_MAX];
    if (s.done[i]) {                                       // finished: pad (4.30.2 process)
      for (int j = 0; j < k; ++j) { nbs[j] = 0.0f; ntok[j] = bp.pad; npar[j] = j; }
    } else {
      Hyps h;
      hyps_load(s, i, k, h);
      int bi = 0;
      double best = -INFINITY;
      for (int r = 0; r < n2; ++r) best = fmax(best, (double)s.cand_score[i * n2 + r]);
      for (int r = 0; r < n2 && bi < k; ++r) {
        const float sc = s.cand_score[i * n2 + r];
        const int f = s.cand_idx[i * n2 + r];
        const int beam = f / V;
        const long long tok = f - beam * V;
        if (bp.eos >= 0 && tok == bp.eos) {
          if (r >= k) continue;                              // not among the top k: not a hypothesis
          hyps_add(h, k, bp.length_penalty, (double)sc, cur_len, beam, step - 1);
        } else {
          nbs[bi] = sc; ntok[bi] = tok; npar[bi] = beam;
          ++bi;
        }
      }
      for (; bi < k; ++bi) { nbs[bi] = 0.0f; ntok[bi] = bp.pad; npar[bi] = bi; }   // unreachable with one eos id
      const bool done = hyps_done(h, bp, best, cur_len);
      hyps_store(s, i, k, h);
      if (done) s.done[i] = 1;
    }
    for (int j = 0; j < k; ++j) {
      const int b = i * k + j;
      s.beam_scores[b] = nbs[j];
      s.tokens[b] = ntok[j];
      s.hist_tok[(long long)step * rows + b] = ntok[j];
      s.hist_par[(long long)step * rows + b] = npar[j];
      s_par[j] = npar[j];
    }
  }
  __syncthreads();
  // lineage: new beam j inherits its parent's positions [0, pos); position pos is its own row
  const int np = pos < s.max_seq ? pos : s.max_seq;
  const int total = k * np;
  for (int e = tid; e < total; e += blockDim.x) {
    const int j = e / np, p = e - j * np;
    s.slot_tmp[(long long)(i * k + j) * s.max_seq + p] = s.slot[(long long)(i * k + s_par[j]) * s.max_seq + p];
  }
  __syncthreads();
  for (int e = tid; e < total; e += blockDim.x) {
    const int j = e / np, p = e - j * np;
    s.slot[(long long)(i * k + j) * s.max_seq + p] = s.slot_tmp[(long long)(i * k + j) * s.max_seq + p];
  }
  if (pos < s.max_seq && tid < k) s.slot[(long long)(i * k + tid) * s.max_seq + pos] = i * k + tid;
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(&s.state[2], 1) == bp.B - 1) {          // last sequence of this step: advance the counters
      int all = 1;
      for (int q = 0; q < bp.B; ++q) all &= (__ldcg(s.done + q) != 0);
      s.state[5] = all;
      s.state[2] = 0;
      s.state[1] = step + 1;
      if (advance_cache) s.state[0] += 1;
      __threadfence();
    }
  }
}

int beam_score(const BeamState& st, int B, int k, int V, int advance_cache, cudaStream_t stream) {
  SB_REQUIRE(B >= 1 && k >= 1 && k <= BEAM_MAX, "beam_score: bad sizes");
  SB_CHECK_CUDA(launch_chain(beam_score_kernel, dim3(B), dim3(256), 0, stream, st, V, advance_cache));
  SB_LAUNCH_CHECK();
  return 0;
}

__global__ void __launch_bounds__(1024)
beam_finalize_kernel(const BeamState s, long long* __restrict__ out, long long ld, float* __restrict__ best_scores) {
  __shared__ int s_maxlen;
  const int i = threadIdx.x;
  const BeamParams bp = *s.params;
  const int k = bp.k, rows = bp.B * k, steps = s.state[1];
  if (i == 0) s_maxlen = 0;
  __syncthreads();
  int len = 0, beam = 0, step = -1;
  if (i < bp.B) {
    Hyps h;
    hyps_load(s, i, k, h);
    if (!s.done[i])
      for (int j = 0; j < k; ++j)
        hyps_add(h, k, bp.length_penalty, (double)s.beam_scores[i * k + j], bp.S + steps, j, steps - 1);
    int best = 0;
    for (int q = 1; q < h.n; ++q) if (h.score[q] >= h.score[best]) best = q;
    len = h.len[best]; beam = h.beam[best]; step = h.step[best];
    if (best_scores) best_scores[i] = (float)h.score[best];
    atomicMax(&s_maxlen, len);
  }
  __syncthreads();
  const int width = min(s_maxlen + 1, bp.S + bp.max_new);
  if (i == 0) *s.n_out = width - bp.S;
  if (i >= bp.B) return;
  long long* row = out + (long long)i * ld;
  for (int t = step; t >= 0; --t) {
    const int b = i * k + beam;
    row[t] = s.hist_tok[(long long)t * rows + b];
    beam = s.hist_par[(long long)t * rows + b];
  }
  for (int c = len - bp.S; c < bp.max_new; ++c)
    row[c] = (c == len - bp.S && len < width && bp.eos >= 0) ? bp.eos : bp.pad;
}

int beam_finalize(const BeamState& st, int B, int64_t* tokens_out, int64_t ld, float* best_scores, cudaStream_t stream) {
  SB_REQUIRE(B >= 1 && B <= 1024, "beam_finalize: batch %d outside [1,1024]", B);
  beam_finalize_kernel<<<1, (B + 31) / 32 * 32, 0, stream>>>(st, reinterpret_cast<long long*>(tokens_out), ld,
                                                              best_scores);
  SB_LAUNCH_CHECK();
  return 0;
}

}  // namespace sb
