// ops.h -- internal C++ entry points of the kernels (one launch each), used by the handle-level
// orchestration in encoder.cu / llama.cu and re-exported 1:1 through the C ABI.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/seedb200.h"

namespace sb {

int gemm(const seedb200_gemm_desc& d, cudaStream_t stream);
int attention(const seedb200_attn_desc& d, cudaStream_t stream);
int layernorm(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy, int rows, int cols,
              float eps, cudaStream_t stream);
int row_stats(const void* x, int64_t ldx, int rows, int cols, float eps, void* stats, cudaStream_t stream);
int row_stats_from_moments(const void* moments, int rows, int cols, float eps, void* stats, cudaStream_t stream);
int ln_fold_weights(const void* W, int64_t ldw, const void* gamma, const void* beta, const void* bias, int N, int K,
                    void* W_out, void* c_out, void* b_out, cudaStream_t stream);
int rmsnorm(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy, int rows, int cols, float eps,
            cudaStream_t stream);
int patchify(const void* images, int B, void* cols, int kpad, cudaStream_t stream);
int broadcast_rows(const void* src, int src_rows, int cols, void* dst, int64_t ldd, int64_t group_stride_rows,
                   int groups, cudaStream_t stream);
int embedding(const void* table, int64_t ld, const int64_t* ids, int n, int cols, void* out, int64_t ldo,
              int64_t n_rows, cudaStream_t stream);
int vq_argmin(const void* z, const void* codebook, int n, int n_codes, int dim, int mode, int64_t* ids,
              cudaStream_t stream);
// dyn (optional, device): dyn[0] overrides past_len at run time (graph-replayed decode step)
int rope_kv_append_tables(const void* qkv, const int64_t* positions, int B, int S, int H, int D, int past_len,
                          int max_seq, int max_pos, const void* cos_t, const void* sin_t, void* q_out,
                          void* k_cache, void* v_cache, cudaStream_t stream, const int* dyn = nullptr);
int build_rope_tables(void* cos_t, void* sin_t, int max_pos, int D, float base, cudaStream_t stream);
int get_rope_tables(int D, float base, int min_pos, const void** cos_t, const void** sin_t, int* max_pos,
                    cudaStream_t stream);
// elementwise helpers (misc.cu)
int add_rows(const void* a, const void* b, void* out, int rows, int cols, int b_rows, cudaStream_t stream);
int gemv(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w, float eps,
         int M, int N, int K, int mode, cudaStream_t stream, int64_t ldo = 0);   // ldo 0 = dense output rows
// dyn (optional, device): kv_len = dyn[0] + 1 at run time; the grid is then sized for max_seq keys
int decode_attention(const void* q, const void* k_cache, const void* v_cache, void* out, int B, int H, int D,
                     int kv_len, int max_seq, float scale, void* workspace, cudaStream_t stream,
                     const int* dyn = nullptr, int* tickets = nullptr, const int* slot = nullptr);
int decode_attention_max_splits(int max_seq);
// RoPE of the new token's q / k + KV append + attention in one launch (max_seq <= 2048); dyn as above (past_len = dyn[0])
bool decode_attention_rope_supported(int D, int max_seq);
int decode_attention_rope(const void* qkv, const int64_t* positions, int B, int H, int D, int past_len, int max_seq,
                          int max_pos, const void* cos_t, const void* sin_t, void* k_cache, void* v_cache, void* out,
                          float scale, cudaStream_t stream, const int* dyn = nullptr, const int* slot = nullptr);
// slot (optional, device) [B, max_seq] int32: cached key / value p of row b lives in cache row slot[b*max_seq + p]
// (beam lineage); NULL = row b.  The new token is still appended at row b.
// sampler.cu
struct GenParams { seedb200_sample_params sp; long long eos, pad; };
// gp (host, by value) or gp_dev (device, read at run time); state (device, optional) = {cache length, step, arrive,
// valid steps, flag}: the step index comes from state[1] and the last CTA advances the counters.
int sample(const void* logits, int64_t ld, int B, int V, const GenParams* gp, const GenParams* gp_dev, uint64_t step,
           int* state, int advance_cache, int64_t* tokens, int64_t* out, int64_t out_ld, int* finished,
           cudaStream_t stream);
// beam search (sampler.cu: candidates; beam.cu: scorer, bookkeeping, finalize)
constexpr int BEAM_MAX = 8;
struct BeamParams {                    // read by the beam kernels at run time (graph replay)
  int k, do_sample, early_stopping, S, max_new, B;
  float temperature, top_p;
  double length_penalty;
  unsigned long long seed, offset;
  long long eos, pad;
};
inline BeamParams beam_params(const seedb200_beam_params& p, long long eos, long long pad, int S, int max_new, int B) {
  BeamParams b;
  b.k = p.num_beams; b.do_sample = p.do_sample; b.early_stopping = p.early_stopping; b.S = S; b.max_new = max_new;
  b.B = B; b.temperature = p.temperature; b.top_p = p.top_p; b.length_penalty = p.length_penalty;
  b.seed = p.seed; b.offset = p.offset; b.eos = eos; b.pad = pad;
  return b;
}
// logits row of (sequence i, beam j) = logits + i * seq_ld + j * beam_ld; -> cand_score / cand_idx [B, 2k]
int beam_select(const void* logits, int64_t seq_ld, int64_t beam_ld, int B, int k, int V, const float* beam_scores,
                const BeamParams* bp, const BeamParams* bp_dev, uint64_t step, const int* state, float* row_stats,
                float* cand_score, int* cand_idx, cudaStream_t stream);   // row_stats: [B*k, 5] scratch
// the device state of one beam-search run (rows = B * k <= max_batch; hyps: k per sequence)
struct BeamState {
  BeamParams* params;
  int* state;            // {cache length, step, arrive counter, -, -, all sequences done}
  float* beam_scores;    // [rows]
  float* row_stats;      // [rows, 5] per-row statistics of the candidate kernel
  float* cand_score;     // [rows * 2]
  int* cand_idx;         // [rows * 2]
  long long* tokens;     // [rows] next decode input
  int* slot;             // [rows, max_seq] lineage table
  int* slot_tmp;         // [rows, max_seq]
  long long* hist_tok;   // [max_seq, rows] token chosen at step t by beam b
  int* hist_par;         // [max_seq, rows] its parent beam (within the sequence)
  double* hyp_score;     // [rows]: k finished hypotheses per sequence, in insertion order
  int* hyp_len;          // [rows] length including the prompt
  int* hyp_beam;         // [rows] beam whose sequence after step hyp_step it is
  int* hyp_step;         // [rows]
  int* hyp_n;            // [rows] (first B used)
  double* worst;         // [rows]
  int* done;             // [rows]
  int* n_out;            // [1]
  int max_seq;
};
int beam_init(const BeamState& st, const BeamParams& bp, cudaStream_t stream);
int beam_score(const BeamState& st, int B, int k, int V, int advance_cache, cudaStream_t stream);
int beam_finalize(const BeamState& st, int B, int64_t* tokens_out, int64_t ld, float* best_scores, cudaStream_t stream);
int image_ids_to_tokens(const int64_t* ids, int n, int64_t shift, int64_t boi, int64_t eoi, int64_t* out,
                        int64_t out_stride, cudaStream_t stream);
int cur_device();
// LLM.int8() (int8.cu, gemm_wgmma.cu)
int int8_quantize_weight(const void* W, int64_t ldw, int N, int K, void* CB, void* SCB, cudaStream_t stream);
// the same into a fused layout: row n -> (n / grp) * gstride + n % grp + off
int int8_quantize_weight_rows(const void* W, int64_t ldw, int N, int K, void* CB, void* SCB, int grp, int gstride,
                              int off, cudaStream_t stream);
int int8_quantize_act(const void* A, int64_t lda, int M, int K, float threshold, void* CA, void* SCA, int* outliers,
                      int* n_outliers, cudaStream_t stream);
int gemm_int8(const seedb200_gemm_int8_desc& d, cudaStream_t stream);
// corr [M,N] fp16 = the outlier correction of every output (written only when *n_outliers > 0)
int int8_correction(const void* A16, int64_t lda, const void* W, int64_t ldw, const void* SCB, const int* outliers,
                    const int* n_outliers, int M, int N, void* corr, cudaStream_t stream);
int gemv_int8(const void* x, const void* norm_w, float eps, float threshold, const void* W, const void* SCB, void* out,
              const void* residual, int M, int N, int K, int mode, cudaStream_t stream);

}  // namespace sb
