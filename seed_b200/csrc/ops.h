// ops.h -- internal C++ entry points of the kernels (one launch each), used by the handle-level
// orchestration in encoder.cu / llama.cu and re-exported 1:1 through the C ABI.
#pragma once

#include <cuda_fp16.h>
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
// ldo 0 = dense output rows; lora (optional): the LoRA expand fused into the epilogue (include/seedb200.h)
int gemv(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w, float eps,
         int M, int N, int K, int mode, cudaStream_t stream, int64_t ldo = 0,
         const seedb200_lora_operand* lora = nullptr);
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
// The device counters of a generation run: int[GS_SLOTS], one array per LLaMA handle.  Every kernel of a decode unit
// reads them at run time, which is what lets one captured graph replay every step.  The run's first launch
// (gen_reset_kernel, beam_init_kernel) sets GS_CACHE_LEN to the prompt length and zeroes the other slots; after that
// they change only through the arrival at the end of each step (step_arrive / seq_arrive in select.cuh).
//   GS_CACHE_LEN   K/V positions in the cache
//   GS_STEP        the step being generated
//   GS_ARRIVE      sequences that have ended the current step
//   GS_VALID       steps HF keeps: last step with an unfinished sequence + 1 (sampler and contrastive loops); in the
//                  beam loop the step at which every search became done + 1 (0: not done)
//   GS_UNFINISHED  some sequence was unfinished at the current step (sampler and contrastive loops)
//   GS_ALL_DONE    every sequence's beam search is done (beam loop)
enum GenSlot { GS_CACHE_LEN, GS_STEP, GS_ARRIVE, GS_VALID, GS_UNFINISHED, GS_ALL_DONE, GS_SLOTS };
static_assert(GS_CACHE_LEN == 0, "the decode forward reads the cache length as dyn[0]");
// sampler.cu
// logits processors (seedb200_logits_params) with the eos id they mask and the prompt length S: the history of a
// row is its first L tokens, L = S + state[GS_STEP] in the device loops (the prompt, then one token per step)
struct LogitsProc { seedb200_logits_params lp; long long eos; int S; };
inline LogitsProc logits_proc(const seedb200_logits_params* p, long long eos, int S) {
  LogitsProc r;
  r.lp.top_k = 0; r.lp.repetition_penalty = 1.0f; r.lp.no_repeat_ngram_size = 0; r.lp.min_length = 0;
  r.lp.min_new_tokens = 0;
  if (p) r.lp = *p;
  r.eos = eos; r.S = S;
  return r;
}
// a control that reads the history or the length: the processing launch runs only then
inline bool logits_history_active(const LogitsProc& p) {
  return p.lp.repetition_penalty != 1.0f || p.lp.no_repeat_ngram_size > 0 ||
         (p.eos >= 0 && (p.lp.min_length > 0 || p.lp.min_new_tokens > 0));
}
int logits_params_check(const char* who, const seedb200_logits_params* p);   // NULL passes
// out[b, proc.S + step] = token (the device loop keeps the prompt in out[b, 0:S]).  scores (NULL: none): the step's
// scores row of row b goes to scores + step * scores_step + b * scores_pitch (seedb200_gen_outputs); it lives here,
// in the device-resident parameters each call rewrites, so that a replayed graph writes into this call's buffer.
struct GenParams {
  seedb200_sample_params sp; long long eos, pad; LogitsProc proc;
  __half* scores; long long scores_pitch, scores_step;
};
// gp (host, by value) or gp_dev (device, read at run time); state (device, optional): the GenSlot counters, which
// give the step and which the last CTA advances.
int sample(const void* logits, int64_t ld, int B, int V, const GenParams* gp, const GenParams* gp_dev, uint64_t step,
           int* state, int advance_cache, int64_t* tokens, int64_t* out, int64_t out_ld, int* finished,
           cudaStream_t stream);
// the history processors, in place on fp16 rows, one CTA per row.  Row (sequence i, beam j) = logits + i * seq_ld +
// j * beam_ld, its history = hist + (i * hist_rows + j) * hist_ld, j < beams.  log_softmax: the row holds logits and
// is first replaced by fp16 log_softmax (beam search).  p (host) or p_dev (device); L = p.S + state[GS_STEP] when
// state is given, else hist_len.  Tok = int64 (sampler) or int32 (beam token table).
template <typename Tok>
int logits_process(void* logits, int64_t seq_ld, int64_t beam_ld, int B, int beams, int V, const LogitsProc* p,
                   const LogitsProc* p_dev, const int* state, const Tok* hist, int64_t hist_ld, int hist_rows,
                   int hist_len, bool log_softmax, cudaStream_t stream);
// beam search (sampler.cu: candidates; beam.cu: scorer, bookkeeping, finalize)
constexpr int BEAM_MAX = 8;
struct BeamParams {                    // read by the beam kernels at run time (graph replay)
  int k, do_sample, early_stopping, S, max_new, B;
  int gpp;                             // sequences per prompt: sequence i searches prompt row i / gpp
  float temperature, top_p;
  double length_penalty;
  unsigned long long seed, offset;
  long long eos, pad;
  LogitsProc proc;                     // top_k (beam sampling) and the history processors
  int processed;                       // 1: the rows already hold the processed fp16 log_softmax (logits_process)
  // outputs (seedb200_gen_outputs; NULL: none), here so that a replayed graph writes into this call's buffers: the
  // scores row of (step t, beam row r) at scores + t * scores_step + r * scores_pitch; beam_indices [B, bi_ld]
  __half* scores; long long scores_pitch, scores_step;
  long long* beam_indices; long long bi_ld;
};
inline BeamParams beam_params(const seedb200_beam_params& p, long long eos, long long pad, int S, int max_new, int B,
                              const seedb200_logits_params* lp = nullptr, int gpp = 1) {
  BeamParams b;
  b.k = p.num_beams; b.do_sample = p.do_sample; b.early_stopping = p.early_stopping; b.S = S; b.max_new = max_new;
  b.B = B; b.gpp = gpp; b.temperature = p.temperature; b.top_p = p.top_p; b.length_penalty = p.length_penalty;
  b.seed = p.seed; b.offset = p.offset; b.eos = eos; b.pad = pad;
  b.proc = logits_proc(lp, eos, S);
  b.processed = logits_history_active(b.proc) ? 1 : 0;
  b.scores = nullptr; b.scores_pitch = 0; b.scores_step = 0; b.beam_indices = nullptr; b.bi_ld = 0;
  return b;
}
// logits row of (sequence i, beam j) = logits + i * seq_ld + j * beam_ld; -> cand_score / cand_idx [B, 2k].  With a
// scores buffer in the parameters the row statistics launch also writes each beam row's fp16 log_softmax there;
// warp_scores (beam sampling with scores) adds one launch that warps those rows in place.
int beam_select(const void* logits, int64_t seq_ld, int64_t beam_ld, int B, int k, int V, const float* beam_scores,
                const BeamParams* bp, const BeamParams* bp_dev, uint64_t step, const int* state, float* row_stats,
                float* cand_score, int* cand_idx, cudaStream_t stream,
                bool warp_scores = false);   // row_stats: [B*k, 5] scratch
// the device state of one beam-search run (rows = B * k <= max_batch; hyps: k per sequence)
struct BeamState {
  BeamParams* params;
  int* state;            // the GenSlot counters
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
  int* tok;              // [rows, max_seq] each beam row's tokens (prompt, then its own), or NULL: allocated by
                         // the first run with a history control and maintained only while params->processed
  int max_seq;
};
// prompt [B / bp.gpp, S] int64 (device): prompt row i / gpp is the prefix of every beam of sequence i, in the lineage
// table and (when bp.processed) in `tok`
int beam_init(const BeamState& st, const BeamParams& bp, const int64_t* prompt, cudaStream_t stream);
int beam_score(const BeamState& st, int B, int k, int V, int advance_cache, cudaStream_t stream);
int beam_finalize(const BeamState& st, int B, int64_t* tokens_out, int64_t ld, float* best_scores, cudaStream_t stream);
int image_ids_to_tokens(const int64_t* ids, int n, int64_t shift, int64_t boi, int64_t eoi, int64_t* out,
                        int64_t out_stride, cudaStream_t stream);
// contrastive search (contrastive.cu)
constexpr int CONTRAST_MAX_K = 8, CONTRAST_MAX_CTAS = 512;
struct ContrastParams { int k; float c_prob, c_pen; };   // c_prob = fp32(1 - alpha), c_pen = fp32(alpha)
int contrastive_params_check(const char* who, const seedb200_contrastive_params* cp);   // NULL is refused
ContrastParams contrast_params(const seedb200_contrastive_params& cp);
// candidates of B rows (logits + b * ld): ids / probs [B*k]; p (host) or p_dev (device); slot (optional)
// [B*k, max_seq] gets slot[r, pos] = r with pos = state[GS_CACHE_LEN] when state is given; gp_dev (optional, with
// state): each row is also copied to gp_dev's scores buffer at step state[GS_STEP] when it has one
int contrastive_candidates(const void* logits, int64_t ld, int B, int V, const ContrastParams* p,
                           const ContrastParams* p_dev, const int* state, int pos, int* slot, int max_seq,
                           int64_t* ids, void* probs, cudaStream_t stream, const GenParams* gp_dev = nullptr);
// one rank + select launch (see RankArgs in contrastive.cu); the loop fields are NULL in the standalone entry point
struct ContrastRank {
  __half* ctx; int64_t ctx_ld; int ctx_rows, H;
  const __half* h; const __half* probs;
  const ContrastParams* p; const ContrastParams* p_dev; int k;
  int* state; int pos;
  float* part; int* tickets; int G;
  int* sel; float* score;
  const long long* cand_ids; const __half* cand_logits; __half* seq_logits; int64_t vpad;
  int* slot; int max_seq;
  const GenParams* gp; long long* out; int64_t out_ld; int* finished;
  int B;
};
int contrastive_rank_ctas(int max_rows, int B);   // the rank kernel's CTAs per sequence for contexts of max_rows
int contrastive_rank(const ContrastRank& r, cudaStream_t stream);
// hidden_states [B*S, H] -> ctx rows [0, S) of each sequence; slot (optional) [B*k, max_seq]: positions < S of every
// candidate row read the prefill row b; p_out (optional, device) receives p
int contrastive_context_init(const void* hidden_states, int B, int S, int H, void* ctx, int64_t ctx_ld, int* slot,
                             int k, int max_seq, const ContrastParams& p, ContrastParams* p_out, cudaStream_t stream);
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
// bitsandbytes 4-bit weights (quant4.cu; the GEMV in misc.cu).  type: SEEDB200_Q4_FP4 / SEEDB200_Q4_NF4
int q4_check(const char* who, int type, int N, int K);   // quant type and K % 64, reported through set_error
// row n of W -> row (n / grp) * gstride + n % grp + off of packed [*, K/2] / absmax [*, K/64]
int quantize_4bit_rows(const void* W, int64_t ldw, int N, int K, int type, void* packed, void* absmax, int grp,
                       int gstride, int off, cudaStream_t stream);
int dequantize_4bit(const void* packed, const void* absmax, int N, int K, int type, void* out, int64_t ldo,
                    cudaStream_t stream);
// seedb200_gemv on dequantize_4bit(packed, absmax), bit for bit, without materialising it
int gemv_4bit(const void* x, const void* norm_w, float eps, const void* packed, const float* absmax, int type,
              void* out, const void* residual, int M, int N, int K, int mode, cudaStream_t stream);
// LoRA (lora.cu)
constexpr int LORA_MAX_R = 64, LORA_MAX_RTOT = 3 * LORA_MAX_R;
int lora_shrink(const void* x, int64_t ldx, const void* norm_w, float eps, const void* A, int M, int K, int rtot,
                void* T, int64_t ldt, cudaStream_t stream);
// gemv_silu: the SiLU of the GEMV (base made by gemv) instead of the GEMM epilogue's
int lora_expand(const void* base, int64_t ldb, const seedb200_lora_operand& lo, int M, int N, int mode,
                bool gemv_silu, const void* residual, int64_t ldr, void* out, int64_t ldo, cudaStream_t stream);
int gemm_lora(const seedb200_gemm_desc& d, const seedb200_lora_operand& lo, cudaStream_t stream);
int gemv_lora(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w, float eps,
              int M, int N, int K, int mode, const seedb200_lora_operand& lo, cudaStream_t stream, int64_t ldo = 0);
int lora_merge(void* W, const void* A, const seedb200_lora_operand& lo, int N, int K, cudaStream_t stream);

}  // namespace sb
