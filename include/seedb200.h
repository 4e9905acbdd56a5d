/*
 * seedb200.h -- C ABI of libseedb200.so: the H100 (sm_90a) replacement for the
 * SEED visual-tokenizer encode path and the llama_xformer forward path.
 *
 * The reference (AILab-CVC/SEED) has no FFI of its own: its "plugin interface"
 * for this path is a set of Python methods (SURVEY.md section 8b).  Every entry
 * point below names the reference function it replaces (file:line relative to
 * /root/reference).  The Python mirror in seed_b200/ binds these with ctypes
 * (see INTEGRATION.md for the exact stub a reference maintainer would add).
 *
 * Conventions
 *   - plain C types only; `stream` is a cudaStream_t passed as void*;
 *   - unless a name ends in _host, every data pointer is a DEVICE pointer;
 *   - fp16 tensors are IEEE binary16, row-major, innermost dimension contiguous;
 *   - every call returns 0 on success, non-zero on failure, and never throws;
 *     seedb200_last_error() returns a thread-local message for the last failure;
 *   - all work is enqueued on the caller's stream, no hidden synchronisation and
 *     no allocation after *_create (so an encode / forward call is CUDA-graph
 *     capturable);
 *   - handles are not thread-safe; distinct handles are independent.
 */
#ifndef SEEDB200_H
#define SEEDB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SEEDB200_VERSION 200

enum seedb200_status {
  SEEDB200_OK = 0,
  SEEDB200_ERR_INVALID = 1,   /* bad argument / shape / missing weight            */
  SEEDB200_ERR_CUDA = 2,      /* a CUDA runtime or driver call failed             */
  SEEDB200_ERR_UNSUPPORTED = 3
};

enum seedb200_dtype { SEEDB200_F16 = 0, SEEDB200_F32 = 1, SEEDB200_I64 = 2, SEEDB200_I32 = 3, SEEDB200_I8 = 4 };

enum seedb200_act { SEEDB200_ACT_NONE = 0, SEEDB200_ACT_GELU = 1, SEEDB200_ACT_TANH = 2, SEEDB200_ACT_RELU = 3 };

/* VQ distance arithmetic (SURVEY 8a/a10 rounding contract):
 *   FP16: every term rounded to binary16 exactly where torch rounds it when the
 *         reference runs its fp16 GPU mode (configs/tokenizer/..._hf.yaml:3);
 *   FP32: distances evaluated in binary32 (the reference's fp16=False mode).   */
enum seedb200_vq_mode { SEEDB200_VQ_FP16 = 0, SEEDB200_VQ_FP32 = 1 };

int seedb200_version(void);
const char* seedb200_last_error(void);
/* number of kernels launched by this library on the calling thread since the
 * last reset (bench.py's "gpu_launches"). */
int64_t seedb200_launch_count(void);
void seedb200_reset_launch_count(void);
/* Optional per-kernel timing for bench.py's roofline: between begin and end every GEMM / attention launch of
 * the calling thread is bracketed by CUDA events on its stream.  end() synchronises, then reports for
 * kind 0 (wgmma GEMM) and kind 1 (attention): launches, summed device milliseconds and, for the GEMM, the
 * summed algorithmic FLOPs (2*M*N*K per launch).  out[kind*3 + {0,1,2}] = {launches, ms, flops}. */
/* Process-wide switches (tests / A-B measurements).
 * "decode_pdl": 1 (default) launches the kernels of the cached decode step (q_len 1) with programmatic stream
 * serialization (each starts while its predecessor drains and waits on griddepcontrol before reading activations).
 * "decode_fused_attention": 1 (default) = the cached decode step runs RoPE + KV append + attention as one kernel per
 * layer when max_seq <= 2048 (seedb200_decode_attention_rope), 0 = rope_kv_append + split-KV decode attention.
 * "gemv_no_allocate": 1 (default) = the decode GEMVs stream their weights with ld.global.nc.L1::no_allocate, 0 = ld.global.nc.
 * "gemm_sched": 1 (default) = a GEMM of a short LLaMA prompt (M <= 256) picks its tile width from a busy-SM
 * model (seedb200_gemm_plan), 0 = the fixed heuristics, 2 = balanced-tail tile order with an explicit bn.
 * "encoder_ln_fold" (read by seedb200_encoder_create): 1 (default) = norm1 / norm2 of the ViT blocks are folded
 * into the qkv / fc1 GEMMs (seedb200_gemm_desc.ln_stats), 0 = standalone LayerNorm kernels.                    */
int seedb200_set_option(const char* key, int value);
int seedb200_profile_begin(void);
int seedb200_profile_end(double* out6);

/* A named tensor handed to *_create.  Pointers are borrowed DEVICE pointers to
 * contiguous fp16 data; the caller keeps them alive for the handle's lifetime.
 * Names are the reference state-dict keys (qformer_quantizer.py:366-374 for the
 * tokenizer, HF LLaMA names for llama_xformer.py). */
typedef struct seedb200_tensor {
  const char* name;
  const void* data;
  int32_t dtype;      /* seedb200_dtype; weights must be SEEDB200_F16 */
  int32_t ndim;
  int64_t shape[4];
} seedb200_tensor;

/* ------------------------------------------------------------------------- */
/* Per-op entry points (unit tests, ncu).  Each is one kernel launch.         */
/* ------------------------------------------------------------------------- */

/* out = epilogue(A[M,K] . W[N,K]^T): torch.nn.functional.linear as used at
 * eva_vit.py:133-135/:157/:60-65, qformer_causual.py:176-181/:251-255/:320-337,
 * llama_xformer.py:186/:223-225/:258/:718.  wgmma + TMA kernel.               */
typedef struct seedb200_gemm_desc {
  int32_t M, N, K;
  const void* A;  int64_t lda;        /* fp16 [M,K]                              */
  const void* W;  int64_t ldw;        /* fp16 [N,K] (nn.Linear.weight layout)    */
  void* out;      int64_t ldo;        /* fp16 [rows, N] (N/2 columns in mode 1)  */
  const void* bias;                   /* fp16 [N] or NULL                        */
  const void* residual; int64_t ldr;  /* fp16, added after bias/act, or NULL     */
  /* leading dimensions in elements; 0 = packed rows (K for lda / ldw, the output width for ldo / ldr).  A nonzero
   * value below that width is refused (SEEDB200_ERR_INVALID), as is a residual in mode 1.                          */
  int32_t act;                        /* seedb200_act                            */
  int32_t mode;                       /* 0 linear; 1 SiLU-gate: W rows are blocks
                                         of [128 gate | 128 up], out[m,j] =
                                         silu(gate_j) * up_j (llama_xformer.py:186) */
  /* optional output-row remap: out_row = (m / row_group) * row_stride +
   * (m % row_group) + row_offset when row_group > 0, else out_row = m.
   * residual row = (m % res_mod) + res_offset when res_mod > 0 else out_row.
   * Used to write patch tokens behind the cls token and add pos_embed
   * (eva_vit.py:373-377).                                                      */
  int32_t row_group, row_stride, row_offset;
  int32_t res_mod, res_offset;
  int32_t bn;                         /* tile-N hint, 0 = auto                   */
  int32_t ctas;                       /* 0, 1 or 2: accepted; single-CTA tiles    */
  /* LayerNorm folded into the GEMM (eva_vit.py:201-202: x + attn(norm1(x)), x + mlp(norm2(x))): with
   * W' = W diag(gamma) as the W operand and A = the UN-normalised rows x,
   *   linear(LayerNorm(x), W, bias) = rstd_m * (acc_mn - mean_m * c_n) + b'_n,
   *   c_n = sum_k W'[n,k],  b'_n = sum_k W[n,k] beta_k + bias_n        (seedb200_ln_fold_weights)
   * ln_stats: float2 (mean, rstd) per row of A (seedb200_row_stats); ln_c, ln_b: fp32 [N].  All NULL = plain GEMM.
   * The normalised activations are never materialised (no LN kernel, no fp16 LN tensor in HBM); the reference's
   * rounding of LN(x) to fp16 is replaced by the rounding of W gamma to fp16 -- same order, bounded in the tests. */
  const void* ln_stats; const void* ln_c; const void* ln_b;
  /* optional: float2 [M, N/64] -- (sum, sum of squares) of every 64-column group of the OUTPUT row as stored (after
   * bias / activation / residual, rounded to fp16); every group holds its own sums.  seedb200_row_stats_from_moments turns the groups into the (mean, rstd) of the next
   * LayerNorm-folded GEMM, so the residual stream is not re-read for its statistics (eva_vit.py:201-202: the output of
   * x + attn(..) / x + mlp(..) is what norm2 / the next block's norm1 normalise).  Needs mode 0, N % 64 == 0, no row
   * remap and a tile width that is a multiple of 64; otherwise SEEDB200_ERR_UNSUPPORTED.                          */
  void* row_moments;
} seedb200_gemm_desc;
int seedb200_gemm(const seedb200_gemm_desc* d, void* stream);
/* Host-only views of the GEMM's persistent tile schedule (no GPU needed; tests/test_capi_cpu.py checks that every
 * tile is handed out exactly once).  gemm_plan: what seedb200_gemm would pick for `d` on a device with `sms` SMs --
 * out9 = {bn, ctas, sched, ksub, m_tiles, n_tiles, units, tile_shift, tail_w} (ctas = ksub = 1, tile_shift = tail_w = 0
 * on H100); pointers in `d` are not dereferenced.
 * gemm_schedule_tile: the tile (mt * n_tiles + nt) of unit `unit`'s round-th iteration, m_tiles * n_tiles when the
 * unit is done.  sched 0 = rotated round robin (default), 1 = balanced tail (full-width tiles round robin, then the
 * units that got one fewer take the last-column tiles; option "gemm_sched" = 2).                                    */
int seedb200_gemm_plan(const seedb200_gemm_desc* d, int sms, int32_t* out9);
int seedb200_gemm_schedule_tile(int sched, int round, int unit, int units, int m_tiles, int n_tiles, int tile_shift);

/* The two helpers of the LayerNorm-folded GEMM (seedb200_gemm_desc.ln_stats):
 * row_stats: (mean, rstd = 1/sqrt(var + eps)) of every row of x [rows, cols] fp16, two-pass in fp32 exactly like
 * seedb200_layernorm (torch.nn.LayerNorm's statistics); stats_out: float2 [rows].
 * ln_fold_weights: W [N,K], gamma/beta [K], bias [N] or NULL (fp16) -> W' [N,K] fp16 = W diag(gamma) rounded once,
 * c [N] fp32 = row sums of the ROUNDED W' (so that acc - mean*c is exact for the operand the MMA really reads),
 * b' [N] fp32 = W beta + bias.                                                                                   */
int seedb200_row_stats(const void* x, int64_t ldx, int rows, int cols, float eps, void* stats_out, void* stream);
/* (mean, rstd) per row from the 64-column moments a GEMM epilogue left (seedb200_gemm_desc.row_moments): groups are
 * summed in index order in fp32, mean and variance (E[x^2] - mean^2) finished in fp64; cols = the row length N.     */
int seedb200_row_stats_from_moments(const void* moments, int rows, int cols, float eps, void* stats_out, void* stream);
int seedb200_ln_fold_weights(const void* W, int64_t ldw, const void* gamma, const void* beta, const void* bias, int N,
                             int K, void* W_out, void* c_out, void* b_out, void* stream);

/* y = LayerNorm(x) * w + b, statistics in fp32 (eva_vit.py:201-202 norm1/norm2,
 * blip2.py:179-184 ln_vision, qformer_causual.py:96/:254/:336).               */
int seedb200_layernorm(const void* x, int64_t ldx, const void* w, const void* b, void* y, int64_t ldy,
                       int rows, int cols, float eps, void* stream);
/* LlamaRMSNorm.forward (llama_xformer.py:105-113): fp32 normalise, round to
 * fp16, multiply by the fp16 weight.                                           */
int seedb200_rmsnorm(const void* x, int64_t ldx, const void* w, void* y, int64_t ldy,
                     int rows, int cols, float eps, void* stream);

/* softmax(scale * Q K^T [+ causal]) V for strided [batch, head, token, dim]
 * views.  Replaces eva_vit.py:139-156, qformer_causual.py:189-236, vit.py:93-103
 * and xops.memory_efficient_attention at llama_xformer.py:240-256.
 * Strides are in elements; head_dim in {64, 88, 128}.  causal != 0 masks key j
 * for query i when j > i + (nk - nq).                                          */
typedef struct seedb200_attn_desc {
  const void* q; const void* k; const void* v; void* o;
  int64_t q_bs, q_hs, q_ts;   /* batch / head / token strides of q              */
  int64_t k_bs, k_hs, k_ts;
  int64_t v_bs, v_hs, v_ts;
  int64_t o_bs, o_hs, o_ts;
  int32_t batch, heads, nq, nk, head_dim;
  int32_t causal;
  float scale;
} seedb200_attn_desc;
int seedb200_attention(const seedb200_attn_desc* d, void* stream);

/* VectorQuantizer2.forward (qformer_quantizer.py:94-98): nearest codebook row
 * under squared L2, ties -> lowest index, int64 ids.  z [n,dim], codebook
 * [n_codes,dim] fp16; dim must be 32.                                          */
int seedb200_vq_argmin(const void* z, const void* codebook, int n, int n_codes, int dim,
                       int mode, int64_t* ids, void* stream);

/* PatchEmbed unfold (eva_vit.py:222,229 conv k14 s14 as a GEMM): images
 * [B,3,224,224] fp16 -> rows [B*256, kpad] fp16 (column = c*196 + dy*14 + dx,
 * zero padded to kpad), plus the cls rows of x: x[b,0,:] = cls + pos[0]
 * (eva_vit.py:373-377).                                                        */
int seedb200_patchify(const void* images, int B, void* cols, int kpad, void* stream);

/* apply_rotary_pos_emb (llama_xformer.py:152-161) fused with the KV-cache append
 * (llama_xformer.py:234-239).  qkv [T, 3*H*D] (q | k | v per token), positions
 * [T] int64; writes q_out [T, H*D] and appends K (post-RoPE) and V at cache row
 * past_len + t of caches laid out [B, H, max_seq, D].                          */
int seedb200_rope_kv_append(const void* qkv, const int64_t* positions, int B, int S, int H, int D,
                            int past_len, int max_seq, void* q_out, void* k_cache, void* v_cache,
                            void* stream);

/* embedding gather (llama_xformer.py:544; qformer_quantizer.py:133).           */
int seedb200_embedding(const void* table, int64_t ld, const int64_t* ids, int n, int cols,
                       void* out, int64_t ldo, int64_t n_rows, void* stream);

/* y[m,:] = x[m,:] . W^T for M <= 4 activation rows: the batch-1 decode form of every nn.Linear of
 * LlamaDecoderLayer (llama_xformer.py:186,223-225,258) and of lm_head (:718); HBM-bound, every weight byte read
 * once.  x [M,K], W [N,K] (row stride ldw), out [M,N] fp16.  mode 0: plain (+ residual [M,N] when non-NULL);
 * mode 1: W rows are blocks of [128 gate | 128 up] and out [M,N/2] = silu(gate) * up (llama_xformer.py:186).
 * norm_w != NULL: x is RMS-normalised while it is staged (LlamaRMSNorm, llama_xformer.py:105-113, eps).        */
int seedb200_gemv(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w,
                  float eps, int M, int N, int K, int mode, void* stream);

/* ---- LLM.int8() linear layers (transformers load_in_8bit=True: bitsandbytes Linear8bitLt, has_fp16_weights=False) ----
 * Weights are quantised once:  SCB[n] = max_k |W[n,k]| (fp32),  CB[n,k] = rint(W[n,k] * (127 / SCB[n])) (int8,
 * half to even; 0 for a row with SCB 0).  Activations per call: element (m,k) is an outlier when !(|A[m,k]| <
 * threshold) (NaN and inf are outliers); the outlier set O is every column holding an outlier in any row;
 * SCA[m] = max |A[m,k]| over the row's non-outlier elements; CA[m,k] = rint(A[m,k] * (127 / SCA[m])), 0 for k in O
 * and when SCA[m] == 0.  Output, with acc = sum_k CA[m,k] CB[n,k] in int32:
 *   base = fp16(((float)acc * 6.200012e-05f) * SCA[m] * SCB[n])
 *   y    = O empty ? base : fp16(base + fp16(sum_{j in O ascending} A[m,j] * fp16(CB[n,j] * SCB[n] / 127)))
 * then mode 0 adds the residual (fp16(y + r)) and mode 1 applies SiLU-gate to the fp16 gate and up values.
 * The GEMM (any M) and the GEMV (M <= 4) produce the same bits.                                                   */
/* W fp16 [N,K] (row stride ldw elements) -> CB int8 [N,K] packed, SCB fp32 [N].  One block per row.              */
int seedb200_int8_quantize_weight(const void* W, int64_t ldw, int N, int K, void* CB, void* SCB, void* stream);
/* A fp16 [M,K] (row stride lda) -> CA int8 [M,K] packed, SCA fp32 [M], outliers int32 [K] (capacity K: the outlier
 * columns in ascending order) and *n_outliers (device int32).  No host synchronisation: graph capturable.  K % 8 == 0. */
int seedb200_int8_quantize_act(const void* A, int64_t lda, int M, int K, float threshold, void* CA, void* SCA,
                               int32_t* outliers, int32_t* n_outliers, void* stream);
/* out = epilogue(linear8(A, W)) by the int8 wgmma GEMM: CA / SCA / outliers / n_outliers as quantize_act left them,
 * A16 the fp16 activations they came from (read at the outlier columns), W = CB and SCB of quantize_weight.
 * Leading dimensions in elements, 0 = packed.  K % 16 == 0; mode 1 needs N % 256 == 0 (W rows in blocks of
 * [128 gate | 128 up]) and no residual.  bn: tile width 64, 128 or 256, 0 = auto.  Two launches: the outlier
 * correction as a dense product over the gathered outlier columns (into workspace), then the GEMM.              */
typedef struct seedb200_gemm_int8_desc {
  int32_t M, N, K;
  const void* A;   int64_t lda;       /* int8 CA [M,K]                             */
  const void* SCA;                    /* fp32 [M]                                  */
  const void* A16; int64_t lda16;     /* fp16 [M,K]                                */
  const int32_t* outliers;            /* ascending outlier columns                 */
  const int32_t* n_outliers;          /* device int32: how many                    */
  const void* W;   int64_t ldw;       /* int8 CB [N,K]                             */
  const void* SCB;                    /* fp32 [N]                                  */
  void* out;       int64_t ldo;       /* fp16 [M, N] (N/2 columns in mode 1)       */
  const void* residual; int64_t ldr;  /* fp16 or NULL, mode 0 only                 */
  int32_t mode;
  int32_t bn;
  void* workspace;                    /* fp16 [M,N]: the outlier corrections   */
} seedb200_gemm_int8_desc;
int seedb200_gemm_int8(const seedb200_gemm_int8_desc* d, void* stream);
/* The same for M <= 4 rows from fp16 x [M,K] (packed): the activation quantisation (and, with norm_w, the RMSNorm of
 * seedb200_gemv) happens while the rows are staged in shared memory; W = CB [N,K] packed, SCB [N]; out [M,N] packed
 * ([M,N/2] in mode 1), residual [M,N] or NULL.  K % 16 == 0.                                                    */
int seedb200_gemv_int8(const void* x, const void* norm_w, float eps, float threshold, const void* W, const void* SCB,
                       void* out, const void* residual, int M, int N, int K, int mode, void* stream);

/* LlamaAttention.forward with q_len == 1 (llama_xformer.py:240-256, attn_bias=None): q [B,H,D] against the first
 * kv_len rows of caches laid out [B,H,max_seq,D]; out [B,H*D] fp16; D must be 128.  workspace: at least
 * seedb200_decode_attention_workspace_bytes(B, H, max_seq) bytes of device memory (split-KV partials).          */
int64_t seedb200_decode_attention_workspace_bytes(int B, int H, int max_seq);
int seedb200_decode_attention(const void* q, const void* k_cache, const void* v_cache, void* out, int B, int H, int D,
                              int kv_len, int max_seq, float scale, void* workspace, void* stream);

/* The same step fused with what precedes it in the decode form of LlamaAttention.forward: apply_rotary_pos_emb on
 * the new token's q / k (llama_xformer.py:152-161), the KV-cache append (:234-239) and the attention (:240-256) in one
 * launch.  qkv [B, 3*H*D] (q | k | v of ONE new token per sequence), positions [B] int64 or NULL (= past_len); K (post-
 * RoPE) and V are appended at cache row past_len of caches [B,H,max_seq,D]; out [B, H*D] fp16.  D = 128 and
 * max_seq <= 2048 (longer caches: seedb200_rope_kv_append + seedb200_decode_attention); for caches of at most 512 keys
 * the result is bit-identical to that pair.                                                                       */
int seedb200_decode_attention_rope(const void* qkv, const int64_t* positions, int B, int H, int D, int past_len,
                                   int max_seq, void* k_cache, void* v_cache, void* out, float scale, void* stream);

/* Next-token selection, on the device.  Replaces what the reference gets from HF GenerationMixin at its call
 * site scripts/seed_llama_inference_8B.py:33 / gradio_demo/seed_llama_flask.py:172 (temperature, top_p,
 * do_sample, num_beams=1): logits / temperature (TemperatureLogitsWarper), nucleus filtering (TopPLogitsWarper,
 * min_tokens_to_keep = 1), softmax, one multinomial draw; do_sample = 0 is argmax with ties to the lowest id
 * (torch.argmax).  The draw for (sequence b, step t) uses one Philox4x32-10 uniform with key = seed and counter
 * (offset + t, b), inverting the CDF of the kept tokens in index order -- reproducible, and independent of how
 * the steps are batched or replayed.  Sampled ids are not comparable with torch's RNG stream; logits are the
 * parity contract (SURVEY 8c), the sampler is checked against its own restatement (oracle/sampler_oracle.py). */
typedef struct seedb200_sample_params {
  int32_t do_sample;
  float temperature;
  float top_p;
  uint64_t seed;
  uint64_t offset;
} seedb200_sample_params;
/* logits [B, ld] fp16 (first V columns valid) -> tokens_out [B] int64. */
int seedb200_sample(const void* logits, int64_t ld, int B, int V, const seedb200_sample_params* sp, uint64_t step,
                    int64_t* tokens_out, void* stream);
/* the uniform in (0,1] the sampler draws for (seed, offset + step, row) -- host function, for tests */
float seedb200_philox_uniform(uint64_t seed, uint64_t offset, uint32_t row);

/* Beam search and beam sampling (num_beams > 1), transformers 4.30.2 GenerationMixin.beam_search / beam_sample with
 * BeamSearchScorer(num_beam_hyps_to_keep = 1), the arithmetic the reference pins (requirements.txt:8):
 *   init       beam_scores fp32 = 0 for beam 0 and -1e9 for beams 1..k-1 of every sequence (the prompt is expanded k
 *              times, so all beams see the same first logits)
 *   step       lp = log_softmax(logits) rounded to fp16 (the logits' dtype); s = float(lp) + beam_score in fp32
 *   greedy     the top 2k of s over the sequence's [k * V] flat entries, descending, ties to the lowest flat index;
 *              beam = j / V, token = j % V
 *   sampling   w = s / temperature (fp32); TopP on each beam row of w with min_tokens_to_keep = 2 in threshold form
 *              (every token tied with the least kept one stays, as seedb200_sample); 2k draws without replacement
 *              from softmax(w) over [k * V] by Gumbel-top-k: key_j = w_j + (-log(-log u_j)) in fp32, filtered
 *              entries -inf, the top 2k keys (ties to the lowest j; non-finite keys fill the last ranks by index).
 *              u_j = ((x >> 9) + 0.5) * 2^-23 with x the first word of Philox4x32-10, key = seed, counter =
 *              (offset + step lo, hi, sequence, 1 + j): strictly inside (0, 1), and word 3 != 0 keeps this stream
 *              apart from seedb200_sample's.  The draws are sorted by w descending (ties to the lowest index) and
 *              the scorer receives w, so running beam scores accumulate temperature-scaled sums (4.30.2's quirk).
 *   scorer     candidates in rank order: an eos candidate at rank < k adds the hypothesis "parent's sequence" with
 *              score = (double)s / len ** length_penalty, len = prompt + generated tokens before the append; at rank
 *              >= k it is skipped; other candidates become the next beams until k are chosen.  At most k hypotheses
 *              are kept: on overflow the lowest score goes (ties: the earliest added), worst_score as BeamHypotheses.
 *              Done (early_stopping 0 = False: k hypotheses and worst >= best / cur_len ** lp; 1 = True: k
 *              hypotheses; 2 = "never": worst >= best / max_length ** lp when lp > 0, else as False).  A finished
 *              sequence emits pad.  The loop ends when every sequence is done or after max_new_tokens steps.
 *   finalize   unfinished sequences add their k running beams; the best hypothesis is the last of a stable ascending
 *              sort by score (ties to the latest added); output width = min(longest + 1, S + max_new_tokens),
 *              eos_id right after every shorter hypothesis and pad after that.                                   */
typedef struct seedb200_beam_params {
  int32_t num_beams;          /* k, 1..8 */
  int32_t do_sample;          /* 0 = beam_search, 1 = beam_sample */
  float temperature, top_p;
  double length_penalty;
  int32_t early_stopping;     /* 0 = False, 1 = True, 2 = "never" */
  uint64_t seed, offset;
} seedb200_beam_params;
/* logits row of (sequence i, beam j) = logits + i * seq_ld + j * beam_ld (fp16, V valid columns; beam_ld = 0 reads
 * one row for every beam, as after the prefill); beam_scores [B * k] fp32 -> cand_score [B, 2k] fp32 (s or w) and
 * cand_idx [B, 2k] int32 flat indices (beam * V + token), in the scorer's order.  step: the Philox step.          */
int seedb200_beam_select(const void* logits, int64_t seq_ld, int64_t beam_ld, int B, int V, const float* beam_scores,
                         const seedb200_beam_params* bp, uint64_t step, float* cand_score, int32_t* cand_idx,
                         void* stream);

/* Codebook ids -> LLaMA token ids without the '<img_%05d>' string round trip of
 * scripts/seed_llama_inference_8B.py:16-23,60,98-100 and gradio_demo/seed_llama_flask.py:144-150:
 * ids [n,32] int64 -> tokens_out[i*out_stride + 0..33] = boi, image_id_shift + id (x32), eoi.  out_stride >= 34
 * lets the spans land directly inside a prompt buffer.                                                         */
int seedb200_image_ids_to_tokens(const int64_t* ids, int n, int64_t image_id_shift, int64_t boi, int64_t eoi,
                                 int64_t* tokens_out, int64_t out_stride, void* stream);

/* ------------------------------------------------------------------------- */
/* Image tokenizer: Blip2QformerQuantizer (qformer_quantizer.py:143-338)       */
/* ------------------------------------------------------------------------- */
typedef struct seedb200_encoder seedb200_encoder;

typedef struct seedb200_encoder_config {
  int32_t vit_depth;        /* 39  (eva_vit.py:466)                              */
  int32_t qformer_layers;   /* 12  (BertConfig default, blip2.py:54)             */
  int32_t detok_depth;      /* 4   (qformer_quantizer.py:176), 0 = no de-tokenizer head */
  int32_t n_codes;          /* 8192                                              */
  int32_t max_batch;        /* workspace is sized for this many images per call  */
  int32_t vq_mode;          /* seedb200_vq_mode                                  */
  int32_t gemm_ctas;        /* 0, 1, 2: passed to the GEMMs' ctas field          */
} seedb200_encoder_config;

int seedb200_encoder_create(const seedb200_encoder_config* cfg, const seedb200_tensor* weights, int n_weights,
                            seedb200_encoder** out);
void seedb200_encoder_destroy(seedb200_encoder* enc);

/* Blip2QformerQuantizer.get_codebook_indices (qformer_quantizer.py:288-307) as
 * called by ImageTokenizer.encode (seed_llama_tokenizer.py:75-90):
 * images [B,3,224,224] fp16 -> ids [B,32] int64.  Optional outputs (NULL to
 * skip): z [B*32,32] fp16 (encode_task_layer output, the VQ input) and
 * query_up [B,32,768] fp16 (decode_task_layer(quant), the 2nd return value).   */
int seedb200_encoder_encode(seedb200_encoder* enc, const void* images, int B, int64_t* ids,
                            void* z_out, void* query_up_out, void* stream);
/* Same, with pinned HOST buffers; copies ride the same stream (bench e2e).     */
int seedb200_encoder_encode_host(seedb200_encoder* enc, const void* images_host, int B,
                                 int64_t* ids_host, void* stream);
/* encode fused with the id -> token arithmetic of seedb200_image_ids_to_tokens: images [B,3,224,224] fp16 ->
 * tokens_out[i*out_stride + 0..33] = boi, image_id_shift + id (x32), eoi, ready to be spliced into a LLaMA prompt
 * (scripts/seed_llama_inference_8B.py:98-100) without leaving the device.  ids_out [B,32] optional.            */
int seedb200_encoder_encode_tokens(seedb200_encoder* enc, const void* images, int B, int64_t image_id_shift, int64_t boi,
                                   int64_t eoi, int64_t* tokens_out, int64_t out_stride, int64_t* ids_out, void* stream);
/* Blip2QformerQuantizer.get_codebook_entry (qformer_quantizer.py:309-338):
 * ids [B,32] int64 -> image_embeds [B,1024] fp16.                              */
int seedb200_encoder_detokenize(seedb200_encoder* enc, const int64_t* ids, int B, void* embeds_out,
                                void* stream);
/* Debug / parity taps: copy an internal activation of the last encode call.
 * what: 0 = ViT output before ln_vision [B*257,1408]; 1 = Q-Former output
 * [B*32,768]; 2 = ln_vision output [B*257,1408].  Returns element count.       */
int64_t seedb200_encoder_tap(seedb200_encoder* enc, int what, void* dst, int64_t max_elems, void* stream);

/* ------------------------------------------------------------------------- */
/* LLaMA: models/llama_xformer.py LlamaForCausalLM                              */
/* ------------------------------------------------------------------------- */
typedef struct seedb200_llama seedb200_llama;

typedef struct seedb200_llama_config {
  int32_t hidden, layers, heads, head_dim, ffn, vocab;
  int32_t max_batch, max_seq;   /* KV cache [layers][2][max_batch, heads, max_seq, head_dim] */
  float rms_eps;
  float rope_base;              /* 10000 (llama_xformer.py:118)                  */
  int32_t gemm_ctas;
} seedb200_llama_config;

int seedb200_llama_create(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights,
                          seedb200_llama** out);
/* The same model with LLM.int8() decoder linears (transformers LlamaForCausalLM.from_pretrained(load_in_8bit=True)):
 * q/k/v/o_proj and gate/up/down_proj of every layer come as "<name>.weight" SEEDB200_I8 [N,K] (CB) plus
 * "<name>.SCB" SEEDB200_F32 [N] (bitsandbytes' state-dict names, seedb200_int8_quantize_weight's output); every other
 * tensor is fp16 as for seedb200_llama_create.  The int8 weights and scales are copied into the handle (the caller
 * may free them after this call); the fp16 tensors are borrowed.  threshold: the outlier threshold (6.0).
 * A linear given with neither tensor is loaded later with seedb200_llama_int8_load_weight.                     */
int seedb200_llama_create_int8(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights,
                               float threshold, seedb200_llama** out);
/* Quantises the fp16 weight `name` (a decoder linear, e.g. "model.layers.3.mlp.up_proj.weight", [N,K] with row
 * stride ldw elements, 0 = K) straight into the handle's fused int8 layout.  create_int8 accepts a linear with
 * neither "<name>.weight" nor "<name>.SCB"; it must then be loaded this way before the first forward / generate
 * (which refuse otherwise).  Loading one fp16 tensor at a time keeps device memory at the int8 model plus that
 * tensor.  Enqueued on `stream`; W may be freed once the stream has passed this call.                          */
int seedb200_llama_int8_load_weight(seedb200_llama* llm, const char* name, const void* W, int64_t ldw, void* stream);
void seedb200_llama_destroy(seedb200_llama* llm);

/* LlamaForCausalLM.forward (llama_xformer.py:661-743).  input_ids [B,S] int64
 * (or inputs_embeds [B,S,hidden] fp16 when input_ids is NULL), position_ids
 * [B,S] int64 (NULL = past_len + arange(S), llama_xformer.py:530-539).  The
 * internal KV cache must already hold past_len tokens.  logits_out is
 * [B,S,vocab] fp16 (logits_mode 0, the reference contract) or [B,1,vocab]
 * (logits_mode 1: last position only, the generate() fast path).
 * Attention is causal over past+new, except S == 1 where the reference passes
 * attn_bias=None (llama_xformer.py:255).                                        */
int seedb200_llama_forward(seedb200_llama* llm, const int64_t* input_ids, const void* inputs_embeds,
                           const int64_t* position_ids, int B, int S, int past_len, int logits_mode,
                           void* logits_out, void* stream);
/* Same with an explicit row stride for the logits (elements, >= vocab): a stride that is a multiple of 8 lets
 * the lm_head epilogue use 16-byte stores when vocab (40194) is not; the caller views [..., :vocab].           */
int seedb200_llama_forward_ld(seedb200_llama* llm, const int64_t* input_ids, const void* inputs_embeds,
                              const int64_t* position_ids, int B, int S, int past_len, int logits_mode,
                              void* logits_out, int64_t logits_ld, void* stream);

/* The generation loop of scripts/seed_llama_inference_8B.py:26-38 (model.generate -> HF sample / greedy_search with
 * llama_xformer.py:745-776 prepare_inputs_for_generation) as ONE call that never leaves the device: prefill of
 * prompt_ids [B,S] (device int64, cache reset), then max_new_tokens x (sampler -> cached q_len-1 forward).  The
 * cache position and the step counter live in device memory, so the decode step is position independent: it is
 * captured once per batch size into a CUDA graph (use_graph != 0) and replayed; use_graph == 0 enqueues the same
 * launches eagerly.  Sequences that emitted eos_id (>= 0) produce pad_id afterwards (HF semantics).  With an
 * eos_id the call synchronises the stream every 32 steps to stop early once every sequence has finished;
 * without one it only enqueues.  tokens_out [B, max_new_tokens] int64 (device); *n_generated_host (may be NULL)
 * receives the number of valid columns.  Returns an error when B > 4 (the decode step uses the <= 4-row GEMV). */
int seedb200_llama_generate(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                            const seedb200_sample_params* sp, int64_t eos_id, int64_t pad_id, int use_graph,
                            int64_t* tokens_out, int* n_generated_host, void* stream);
/* 1 when the last generate() replayed a captured graph, 0 when it ran eagerly, -1 before any call */
int seedb200_llama_generate_used_graph(seedb200_llama* llm);
/* Beam search / beam sampling (see seedb200_beam_params) of prompt_ids [B,S] (device int64): prefill at B cache rows,
 * then per step candidates -> scorer -> one cached forward of B * k rows whose attention reads each beam's past
 * through a lineage table (no cache copies).  The decode step is captured once per (B, k) into a CUDA graph when
 * use_graph != 0.  eos_id < 0: no eos (fixed length).  B * k <= max_batch (see seedb200_llama_reserve_rows).
 * tokens_out [B, max_new_tokens] int64 (device): the generated part of the output; *n_out_host receives its valid
 * width (output width - S); best_scores_out [B] fp32 (device, may be NULL): the chosen hypotheses' scores.
 * Synchronises the stream (every 32 steps with an eos id, and once at the end).                                  */
int seedb200_llama_beam_generate(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                                 const seedb200_beam_params* bp, int64_t eos_id, int64_t pad_id, int use_graph,
                                 int64_t* tokens_out, int* n_out_host, float* best_scores_out, void* stream);
/* Grows every buffer sized by max_batch (KV caches, activations, int8 workspaces, generation state) to `rows`
 * rows; no-op when rows <= max_batch.  The cache contents and the captured graphs are dropped.  Synchronises the
 * device.  Bytes added per row: see INTEGRATION.md "C4. Beam search".                                           */
int seedb200_llama_reserve_rows(seedb200_llama* llm, int rows);
/* Decode attention through a lineage table: cached key / value p of row b is read from cache row
 * slot[b * max_seq + p] (slot [B, max_seq] int32, device); otherwise seedb200_decode_attention. */
int seedb200_decode_attention_lineage(const void* q, const void* k_cache, const void* v_cache, const int32_t* slot,
                                      void* out, int B, int H, int D, int kv_len, int max_seq, float scale,
                                      void* workspace, void* stream);
/* seedb200_decode_attention_rope through a lineage table (max_seq <= 2048): the new K/V are appended at row b,
 * position past_len, which slot[b * max_seq + past_len] must name (= b); earlier positions are read from
 * slot[b * max_seq + p].                                                                                         */
int seedb200_decode_attention_rope_lineage(const void* qkv, const int64_t* positions, const int32_t* slot, int B, int H,
                                           int D, int past_len, int max_seq, void* k_cache, void* v_cache, void* out,
                                           float scale, void* stream);

/* Views of the KV cache of one layer: [max_batch, heads, max_seq, head_dim]
 * fp16; the first past_len+S rows per (batch, head) are valid.  Used to build
 * the past_key_values tuple the reference returns (llama_xformer.py:239).      */
int seedb200_llama_kv_ptrs(seedb200_llama* llm, int layer, void** k, void** v);
/* Load an externally supplied past (past_key_values argument) into the cache:  */
int seedb200_llama_kv_load(seedb200_llama* llm, int layer, const void* k, const void* v, int B, int past_len,
                           void* stream);
/* tap: final hidden states (after model.norm) of the last forward [B*S,hidden] */
int64_t seedb200_llama_tap(seedb200_llama* llm, int what, void* dst, int64_t max_elems, void* stream);

/* ---- image preprocessing (SURVEY.md 8f row 1: the caller side of encode) -------------------------------------
 * Replaces the CPU pipeline in front of the tokenizer, bit for bit:
 *   models/transforms.py:4-19             Resize((S,S)) [PIL BILINEAR = filter 2] -> ToTensor -> Normalize(CLIP)
 *   models/seed_llama_tokenizer.py:50-56  Resize((S,S), interpolation=3) [PIL BICUBIC = filter 3] -> ToTensor -> Normalize
 * plus the .half() of ImageTokenizer.encode (:84-85).  Input: n RGB images of one size, uint8 [n,in_h,in_w,3]
 * (interleaved, as np.asarray(pil_image)) in device memory; output fp16 [n,3,S,S] ready for
 * seedb200_encoder_encode.  The resize is Pillow's 8-bit two-pass fixed-point resampling (weights built on the
 * host in double exactly as Pillow does, 22 fractional bits, 8-bit intermediate image); the normalisation is
 * IEEE fp32 ((v/255 - mean)/std), so the result equals torchvision's on the same bytes.
 * A plan owns the weight tables and the intermediate buffer for one (in_h, in_w, S, filter); run() allocates
 * nothing and only enqueues on `stream`.                                                                        */
typedef struct seedb200_preprocess seedb200_preprocess;
int seedb200_preprocess_create(int in_h, int in_w, int out_size, int filter, int max_batch,
                               seedb200_preprocess** out);
/* keep_ratio=True of models/transforms.py:6-9 (the reference default): Resize(S) [shorter side -> S, the other
 * int(S * long / short)] -> CenterCrop(S).  The caller passes the resize size and the crop origin exactly as
 * torchvision computes them; only the crop window of the resample is evaluated.  create() is create_ex() with
 * resize = out_size x out_size and no crop.                                                                     */
int seedb200_preprocess_create_ex(int in_h, int in_w, int resize_h, int resize_w, int crop_top, int crop_left,
                                  int out_size, int filter, int max_batch, seedb200_preprocess** out);
void seedb200_preprocess_destroy(seedb200_preprocess* plan);
int seedb200_preprocess_run(seedb200_preprocess* plan, const void* images_u8, int n, void* out_f16, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SEEDB200_H */
