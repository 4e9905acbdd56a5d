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
  /* consumer-warpgroup schedule hint, 0 = auto (the planner's choice, seedb200_gemm_plan_schedule): 1 = cooperative
   * (both consumer warpgroups on one 128 x bn tile), 2 = ping-pong (mode 0 only: one 128 x 128 tile per warpgroup,
   * one warpgroup's epilogue under the other's MMAs; a bn hint other than 0 or 128 is SEEDB200_ERR_UNSUPPORTED).
   * Both give bit-identical results.                                                                            */
  int32_t wg_schedule;
} seedb200_gemm_desc;
enum seedb200_gemm_schedule { SEEDB200_GEMM_COOPERATIVE = 1, SEEDB200_GEMM_PINGPONG = 2 };
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
/* Host-only: the consumer schedule seedb200_gemm runs `d` with on a device with `sms` SMs (*schedule =
 * SEEDB200_GEMM_COOPERATIVE or SEEDB200_GEMM_PINGPONG); pointers in `d` are only tested against NULL.           */
int seedb200_gemm_plan_schedule(const seedb200_gemm_desc* d, int sms, int32_t* schedule);

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
 * kv_len rows of caches laid out [B,H,max_seq,D]; out [B,H*D] fp16; D must be 128.  q and the caches must be
 * 16-byte aligned.  workspace: at least seedb200_decode_attention_workspace_bytes(B, H, max_seq) bytes of device
 * memory: split-KV partials for the largest split count of any kv_len <= max_seq (min(64, ceil(max_seq / 128))
 * splits per head; the split count is not monotone in kv_len), then B*H int tickets.                            */
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

/* Further generation controls, transformers 4.30.2's logits processors and TopK warper on fp16 logits, as the
 * reference runs them on CUDA.  Neutral values (all 0, repetition_penalty 1) change nothing and launch nothing.
 * The processors run first, in this order, on a row whose current length L includes the prompt (S tokens):
 *   repetition_penalty p   every distinct token t among the row's history (prompt + generated tokens): v = score[t]
 *                          becomes fp16(v * p) when v < 0, else fp16(v * fp32(1 / p)) -- torch's CUDA division of an
 *                          fp16 tensor by a Python scalar multiplies by the fp32 reciprocal.  Duplicates count once.
 *   no_repeat_ngram_size n nothing when L + 1 < n; else for every i <= L - n with x[i : i+n-1] == x[L-n+1 : L],
 *                          x[i+n-1] is set to -inf
 *   min_length m           eos is -inf while L < m
 *   min_new_tokens m       eos is -inf while L - S < m (both length rules need an eos id >= 0)
 * then the warpers, when sampling: temperature, top_k, top_p.  top_k k keeps every token whose compared value is >=
 * the k'-th largest, k' = min(max(k, min_keep), V), ties kept (the threshold form of TopP).  Sampling (min_keep 1)
 * compares the tempered fp16 logit fp16(x * fp32(1 / T)), or x when T == 1 (no temperature warper); TopP then runs
 * on the kept tokens.  Greedy decoding and beam search apply the processors only.
 * Beam search / sampling: the processors act on lp = fp16 log_softmax(logits) of each beam row, with that row's own
 * tokens as history, before s = lp + beam_score; beam sampling compares w = s / T for top_k (min_keep 2), then TopP.
 * Refused with SEEDB200_ERR_INVALID before any device work: top_k < 0, a repetition_penalty that is not finite and
 * > 0, or a negative no_repeat_ngram_size / min_length / min_new_tokens.                                          */
typedef struct seedb200_logits_params {
  int32_t top_k;                 /* 0 = off */
  float repetition_penalty;      /* 1 = off */
  int32_t no_repeat_ngram_size;  /* 0 = off */
  int32_t min_length;            /* 0 = off */
  int32_t min_new_tokens;        /* 0 = off */
} seedb200_logits_params;
/* seedb200_sample with the controls above; lp NULL is seedb200_sample.  history [B, hist_ld] int64 (device): row b's
 * first hist_len tokens (prompt_len of them the prompt) are its input ids; needed when a history control is active.
 * When one is, the processors rewrite the logits rows in place before the selection.  eos_id < 0: none.          */
int seedb200_sample_processed(void* logits, int64_t ld, int B, int V, const seedb200_sample_params* sp, uint64_t step,
                              int64_t* tokens_out, void* stream, const seedb200_logits_params* lp,
                              const int64_t* history, int64_t hist_ld, int hist_len, int prompt_len, int64_t eos_id);
/* seedb200_sample_processed that also writes each row's generation score (see seedb200_gen_outputs) to
 * scores_out + b * scores_ld (fp16 [B, scores_ld], V valid columns); scores_out NULL is seedb200_sample_processed.
 * Refused with SEEDB200_ERR_INVALID before any device work: scores_ld < V or not a multiple of 8, or a base that is
 * not 16-byte aligned. */
int seedb200_sample_scores(void* logits, int64_t ld, int B, int V, const seedb200_sample_params* sp, uint64_t step,
                           int64_t* tokens_out, void* stream, const seedb200_logits_params* lp,
                           const int64_t* history, int64_t hist_ld, int hist_len, int prompt_len, int64_t eos_id,
                           void* scores_out, int64_t scores_ld);

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

/* ---- bitsandbytes 4-bit linear layers (transformers load_in_4bit=True: Linear4bit, blocksize 64) ----------------
 * Follows bitsandbytes 0.39-0.41 quantize_4bit / dequantize_4bit / MatMul4Bit (restated in tests/quant4_ref.py; not
 * checked against bitsandbytes itself).  W fp16 [N,K], K % 64 == 0, is cut row-major into blocks of 64 weights
 * (blocks never cross rows):
 *   absmax[n, b] = max |W| over the block (fp32, fmaxf: NaN dropped)
 *   v            = fp32(w) * (1.0f / absmax)          (correctly rounded reciprocal; an all-zero block gives NaN)
 *   NF4 code     = the number of the 15 fp32 midpoints (a + b) * 0.5f of adjacent NF4 values (table below) that v
 *                  strictly exceeds: a value on a midpoint takes the lower code, NaN takes code 0
 *   FP4 code     = 8 if v < 0 (-0 and NaN: no sign bit) | the 3-bit code of the bucket of |v| among the pivots
 *                  0.00260417, 0.0859375, 0.20833333, 0.29166667, 0.4166667, 0.583333, 0.8333333 (strict >); the
 *                  buckets in ascending order have the codes 0, 1, 6, 7, 4, 5, 2, 3
 *   packed       = uint8 [N, K/2], two codes per byte, the even-index element in the HIGH nibble; absmax fp32 [N, K/64]
 *   W'           = fp16_rn(value[code] * absmax) with the fp32 values
 *                  FP4 codes 0..7: 0, 0.005208333333, 0.66666667, 1, 0.33333333, 0.5, 0.16666667, 0.25 (bit 8: negated)
 *                  NF4 codes 0..15: -1, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453,
 *                  -0.28444138169288635, -0.18477343022823334, -0.09105003625154495, 0, 0.07958029955625534,
 *                  0.16093020141124725, 0.24611230194568634, 0.33791524171829224, 0.44070982933044434,
 *                  0.5626170039176941, 0.7229568362236023, 1
 *   linear4(x)   = fp16(x . W'^T) with fp32 accumulation (MatMul4Bit's dequantise-then-linear form, exact for an fp32
 *                  or fp16 compute dtype; bitsandbytes >= 0.40's one-token gemv_4bit kernel may sum and round
 *                  differently and is not the contract).  seedb200_gemv_4bit equals seedb200_gemv on W' bit for bit.
 * Double quantisation and a bf16 compute dtype are not supported.                                                   */
enum seedb200_quant4 { SEEDB200_Q4_FP4 = 0, SEEDB200_Q4_NF4 = 1 };
/* W fp16 [N,K] (row stride ldw elements, 0 = K; 16-byte aligned rows) -> packed uint8 [N, K/2], absmax fp32 [N, K/64] */
int seedb200_quantize_4bit(const void* W, int64_t ldw, int N, int K, int quant_type, void* packed, void* absmax,
                           void* stream);
/* packed + absmax -> W' fp16 [N,K] (row stride ldo elements, 0 = K)                                                  */
int seedb200_dequantize_4bit(const void* packed, const void* absmax, int N, int K, int quant_type, void* out,
                             int64_t ldo, void* stream);
/* out = epilogue(linear4(x)) for M <= 4 rows: seedb200_gemv's modes (0 with optional residual; 1 = SiLU gate over
 * [128 gate | 128 up] row blocks) and norm_w (RMSNorm folded into the staging); packed / absmax dense.               */
int seedb200_gemv_4bit(const void* x, const void* norm_w, float eps, const void* packed, const void* absmax,
                       int quant_type, void* out, const void* residual, int M, int N, int K, int mode, void* stream);

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
/* The same model with bitsandbytes 4-bit decoder linears (from_pretrained(load_in_4bit=True), see seedb200_quant4):
 * `weights` holds the fp16 tensors other than the seven decoder linears (which are refused here); every linear is
 * then quantised into the handle by seedb200_llama_4bit_load_weight, and forward / generate refuse to run until all
 * are.  The handle also owns an fp16 scratch of 2 * ffn * hidden elements: more than 4 rows (prefill, or a decode
 * step of more than 4 rows) dequantise each fused linear into it and run the fp16 GEMM, as MatMul4Bit does, so the
 * logits equal an fp16 model holding W'.  Up to 4 rows use seedb200_gemv_4bit.  LoRA adapters are refused.          */
int seedb200_llama_create_4bit(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights,
                               int quant_type, seedb200_llama** out);
/* Quantises the fp16 decoder linear `name` ([N,K], row stride ldw elements, 0 = K) into the 4-bit handle's fused
 * layout (q|k|v concatenated, gate|up in 128-row blocks).  Enqueued on `stream`; W may be freed once the stream has
 * passed this call.                                                                                                  */
int seedb200_llama_4bit_load_weight(seedb200_llama* llm, const char* name, const void* W, int64_t ldw, void* stream);
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
 * receives the number of valid columns.  B <= max_batch (see seedb200_llama_reserve_rows); a call is
 * seedb200_llama_generate_n with num_return_sequences = 1. */
int seedb200_llama_generate(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                            const seedb200_sample_params* sp, int64_t eos_id, int64_t pad_id, int use_graph,
                            int64_t* tokens_out, int* n_generated_host, void* stream);
/* seedb200_llama_generate with the controls of seedb200_logits_params; lp NULL is seedb200_llama_generate.  They live
 * in device memory like the sampling parameters, so new values replay the captured decode step; a history control
 * adds one launch per step and its own captured graph. */
int seedb200_llama_generate_processed(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                      int max_new_tokens, const seedb200_sample_params* sp, int64_t eos_id,
                                      int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host,
                                      void* stream, const seedb200_logits_params* lp);
/* num_return_sequences = n samples per prompt (transformers 4.30.2 generate(do_sample=True, num_return_sequences=n),
 * which expands the inputs n times): R = B * n rows, prompt-major, row b * n + j is sample j of prompt b.  Each
 * prompt is prefilled once, at cache row b; row r reads prompt r / n's K/V through the lineage table and appends its
 * own from position S on, so the prompt's K/V are written once per prompt.  Every row samples on its own: Philox row
 * r, its own eos / pad state and its own history for the controls, so the tokens equal those of a call on
 * prompt_ids.repeat_interleave(n, 0) with n = 1.  n = 1 issues the launches of seedb200_llama_generate.
 * tokens_out [R, max_new_tokens].  Refused with SEEDB200_ERR_INVALID before any device work: n < 1, R > max_batch,
 * R > 1024.  With n > 1 the cache rows hold lineages afterwards (as after beam search).                            */
int seedb200_llama_generate_n(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                              int num_return_sequences, const seedb200_sample_params* sp, int64_t eos_id,
                              int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host, void* stream);
int seedb200_llama_generate_n_processed(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                        int max_new_tokens, int num_return_sequences,
                                        const seedb200_sample_params* sp, int64_t eos_id, int64_t pad_id,
                                        int use_graph, int64_t* tokens_out, int* n_generated_host, void* stream,
                                        const seedb200_logits_params* lp);
/* Generation scores, transformers 4.30.2 generate(output_scores=True, return_dict_in_generate=True): one fp16 row of
 * V scores per generated row and step, written by the kernel that already holds the row (no extra pass).  The row of
 * step t and row r is scores + (t * R + r) * scores_pitch (halves), R the call's row count; the caller allocates
 * max_new_tokens * R * scores_pitch halves.  What a row holds:
 *   greedy     the processed logits: the controls of seedb200_logits_params other than top_k, no warpers
 *              (4.30.2 greedy_search: next_tokens_scores = logits_processor(input_ids, next_token_logits))
 *   sampling   the warped row (4.30.2 sample: next_token_scores = logits_warper(...)): fp16(x * fp32(1 / T)), or x
 *              when T == 1, on the tokens the draw kept (top_k, then top_p, in the threshold form of
 *              seedb200_sample) and -inf elsewhere
 *   contrastive the processed logits the candidates are taken from (4.30.2 contrastive_search:
 *              scores += (logit_for_next_step,), no warpers)
 *   beam search   (4.30.2 beam_search: scores += (next_token_scores_processed,)) R = G * k beam rows, row g * k + j:
 *              lp = fp16((x - max) - logZ) of beam j, the processors applied, before the beam score is added.  At step
 *              0 the k rows of a search are identical (every beam reads the prefill's row).
 *   beam sampling (4.30.2 beam_sample: scores += (logits_warper(input_ids, next_token_scores_processed),)) the warpers
 *              on the processed lp row without the beam score: v = fp16(lp * fp32(1 / T)) (lp when T == 1), TopK keeps
 *              v >= the k'-th largest, k' = min(max(top_k, 2), V), TopP keeps p = exp(v - max v) >= its threshold, at
 *              least the two largest (min_tokens_to_keep = 2); removed tokens are -inf.  This is not the w = s / T the
 *              draws use; it costs one more launch per step.
 * n_steps_out receives the number of entries transformers returns.  Sampling, greedy and contrastive: the valid width
 * of tokens_out (the loop stops once every row has finished).  Beams: the number of BeamSearchScorer.process calls, the
 * step at which every search became done + 1, or max_new_tokens; the device records that step, and it may exceed the
 * valid width.  Rows of later steps may hold scores of steps the early-stop poll ran past; they are not counted.
 * beam_indices (beam entry point only, optional; NULL elsewhere): int64 [G, S + max_new_tokens], row g written in
 * full: entry t is the flat beam row in [0, G * k) whose scores row produced token t of the returned hypothesis (4.30.2
 * BeamSearchScorer: beam_indices[beam_idx] + (beam_idx,)); a hypothesis closed by an eos candidate has one entry more,
 * the eos step's parent row; -1 after that.
 * Refused with SEEDB200_ERR_INVALID before any device work: a NULL scores, a scores_pitch < V or not a multiple of 8,
 * a base that is not 16-byte aligned, a non-NULL beam_indices outside the beam entry point.  The pointers reach the
 * captured decode step through the device-resident parameters each call rewrites (GenParams, BeamParams), so
 * consecutive calls may pass different buffers. */
typedef struct seedb200_gen_outputs {
  void* scores;              /* fp16, device */
  int64_t scores_pitch;      /* halves between rows, >= V, a multiple of 8 */
  int64_t* beam_indices;     /* beams: int64 [G, S + max_new_tokens] (device), optional, and NULL elsewhere */
  int32_t n_steps_out;       /* written by the call */
} seedb200_gen_outputs;
/* seedb200_llama_generate_n_processed with optional outputs (NULL: none, the launches of the call without them). */
int seedb200_llama_generate_ex(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                               int num_return_sequences, const seedb200_sample_params* sp, int64_t eos_id,
                               int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host, void* stream,
                               const seedb200_logits_params* lp, seedb200_gen_outputs* outputs);
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
/* seedb200_llama_beam_generate with the controls of seedb200_logits_params; lp NULL is seedb200_llama_beam_generate.
 * The first call with a history control allocates a [max_batch, max_seq] int32 token table (4 * max_seq bytes per
 * row), kept until seedb200_llama_reserve_rows reallocates the rows. */
int seedb200_llama_beam_generate_processed(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                           int max_new_tokens, const seedb200_beam_params* bp, int64_t eos_id,
                                           int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_out_host,
                                           float* best_scores_out, void* stream, const seedb200_logits_params* lp);
/* Beam sampling with num_return_sequences = n, as transformers 4.30.2 runs it: BeamSearchScorer(batch_size = B * n,
 * num_beams = k) keeping one hypothesis per search, and inputs expanded k * n times.  So each prompt gets n
 * independent beam-sample searches and each returns its best hypothesis; n may exceed k.  (Later transformers
 * releases return the top n hypotheses of one search instead; that is not what this computes.)  Search g = b * n + j
 * (prompt-major) reads prompt b, prefilled once at cache row b, through the lineage table, and draws from Philox
 * sequence g, so the tokens equal those of a call on prompt_ids.repeat_interleave(n, 0) with n = 1.
 * tokens_out [B * n, max_new_tokens], best_scores_out [B * n].  B * n * k <= max_batch.  Refused with
 * SEEDB200_ERR_INVALID before any device work: n < 1, n > 1 with bp->do_sample == 0 (beam search keeps refusing it),
 * rows above max_batch, B * n > 1024.  n = 1 is seedb200_llama_beam_generate{,_processed}.                       */
int seedb200_llama_beam_generate_n(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                                   int num_return_sequences, const seedb200_beam_params* bp, int64_t eos_id,
                                   int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_out_host,
                                   float* best_scores_out, void* stream);
int seedb200_llama_beam_generate_n_processed(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                             int max_new_tokens, int num_return_sequences,
                                             const seedb200_beam_params* bp, int64_t eos_id, int64_t pad_id,
                                             int use_graph, int64_t* tokens_out, int* n_out_host,
                                             float* best_scores_out, void* stream, const seedb200_logits_params* lp);
/* seedb200_llama_beam_generate_n_processed with optional outputs (seedb200_gen_outputs; NULL: none, the launches of
 * the call without them).  R = B * n * k beam rows; best_scores_out holds transformers' sequences_scores.  With
 * outputs and bp->do_sample the decode step has one more launch (the warp of the scores rows) and its own graph. */
int seedb200_llama_beam_generate_ex(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                                    int num_return_sequences, const seedb200_beam_params* bp, int64_t eos_id,
                                    int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_out_host,
                                    float* best_scores_out, void* stream, const seedb200_logits_params* lp,
                                    seedb200_gen_outputs* outputs);
/* Contrastive search (generate(penalty_alpha > 0, top_k = k > 1), num_beams 1, no sampling): transformers 4.30.2
 * GenerationMixin.contrastive_search with _ranking_fast, as the reference runs them on CUDA in fp16.  Per sequence b
 * and step t, at position p = S + t:
 *   logits     fp16 [V]: t = 0 the prefill's last-position logits, later the selected candidate's logits of step t-1,
 *              after the history processors of seedb200_logits_params, and no warpers: top_k is the
 *              candidate count
 *   probs      softmax in fp16: fp16(exp(x - max) * fp32(1 / sum)), max and sum in fp32 (torch's CUDA epilogue
 *              multiplies by the reciprocal; tests/test_contrastive_gpu.py pins it against the installed torch)
 *   candidates (q_j, id_j), j < k: the k largest probs, descending, ties to the lower token id
 *   forward    k rows, token id_j at position p, each attending to the prompt + the selected history through the
 *              lineage table (no KV copies) -> logits_j, h_j = the row's final RMSNorm output (hidden_states[-1])
 *   context    c_i, i < p: h of position i -- the prefill's rows for i < S, then each step's selected h
 *   n(x)       fp16(float(x) / float(fp16(sqrt(fp32 sum of float(x)^2))))  (torch's fp16 vector_norm; any sum order)
 *   cos_ij     fp16(sum_d n(c_i)[d] * n(h_j)[d]), fp32 accumulation in any order (cuBLAS in HF)
 *   pen_j      max_i cos_ij (a NaN propagates)
 *   score_j    fp16(fp16(fp32(1 - alpha) * q_j) - fp16(fp32(alpha) * pen_j)); 1 - alpha is computed in double, as
 *              Python does, then rounded to fp32 (not 1 - fp32(alpha))
 *   sel        argmax_j score_j, ties to the lower j; the first NaN wins (torch.max)
 *   token      id_sel, or pad_id once the sequence has finished; the selected candidate's K/V, h and logits carry
 *              the sequence on either way.  The sequence finishes on eos_id; the loop stops when all have.
 * The context is stored once per position, already normalised (n depends on its row only), instead of being
 * renormalised every step: the bits are the same.  top_k in [2, 8]; penalty_alpha finite and > 0.              */
typedef struct seedb200_contrastive_params {
  int32_t top_k;          /* k: candidates per step, [2, 8]                                                      */
  double penalty_alpha;   /* alpha, finite and > 0; double so that fp32(1 - alpha) is the scalar torch uses     */
} seedb200_contrastive_params;
/* Contrastive search of prompt_ids [B,S] (device int64): prefill at B rows, the prompt's normalised hidden states
 * into the context, then max_new_tokens x (history processors when lp has one -> candidates -> one cached forward of
 * B * k rows through the lineage table -> rank + select).  The step is captured once per (B, k, processors) into a
 * CUDA graph when use_graph != 0 (contrastive units never replay a sampler or beam graph).  B * k <= max_batch (see
 * seedb200_llama_reserve_rows); eos_id < 0: no eos.  tokens_out [B, max_new_tokens] int64 (device); *n_generated_host
 * (may be NULL) receives the valid width.  With an eos id the call synchronises every 32 steps to stop early.
 * The first call allocates per row: the normalised context (2 * max_seq * hidden bytes), a logits row
 * (2 * vocab rounded up to 8), and the candidates' probabilities and rank maxima (see INTEGRATION.md C8).  Refused
 * with SEEDB200_ERR_INVALID before any device work: top_k outside [2, 8], a non-finite or non-positive
 * penalty_alpha, B * k > max_batch.                                                                              */
int seedb200_llama_contrastive_generate(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                        int max_new_tokens, const seedb200_contrastive_params* cp, int64_t eos_id,
                                        int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host,
                                        void* stream, const seedb200_logits_params* lp);
/* seedb200_llama_contrastive_generate with optional outputs (seedb200_gen_outputs; NULL: none, the launches of the
 * call without them).  R = B rows.  The candidates kernel copies each step's row; no launch is added. */
int seedb200_llama_contrastive_generate_ex(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                           int max_new_tokens, const seedb200_contrastive_params* cp, int64_t eos_id,
                                           int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host,
                                           void* stream, const seedb200_logits_params* lp,
                                           seedb200_gen_outputs* outputs);
/* The three kernels on their own, for tests.  candidates: logits [B, ld] fp16 (V valid, V >= 8) -> ids_out [B*k]
 * int64, probs_out [B*k] fp16.  rank: context [B, ctx_ld] fp16 holding ctx_rows normalised rows of `hidden` per
 * sequence, the first p (>= 1) valid; cand_hidden [B*k, hidden] (raw h_j), cand_probs [B*k] fp16 -> sel_out [B] int32
 * and scores_out [B*k] fp32 (the fp16 scores; both may be NULL); n(h_sel) is appended at context row p when
 * p < ctx_rows.  context_init: hidden_states [B*S, hidden] -> context rows [0, S) of each sequence.  hidden % 8 == 0,
 * 16-byte aligned operands.                                                                                      */
int seedb200_contrastive_candidates(const void* logits, int64_t ld, int B, int V, int top_k, int64_t* ids_out,
                                    void* probs_out, void* stream);
int seedb200_contrastive_rank(void* context, int64_t ctx_ld, int ctx_rows, int p, int hidden, const void* cand_hidden,
                              const void* cand_probs, int B, const seedb200_contrastive_params* cp, int32_t* sel_out,
                              float* scores_out, void* stream);
int seedb200_contrastive_context_init(const void* hidden_states, int B, int S, int hidden, void* context,
                                      int64_t ctx_ld, void* stream);
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

/* ---- unmerged LoRA adapters (PEFT lora.Linear, eval mode, fp16 module) -------------------------------------------
 * For a decoder linear with weight W [N,K], lora_A [r,K], lora_B [N,r] (all fp16) and s = lora_alpha / r:
 *   base = fp16(W x)                      the linear's kernel, unchanged
 *   t    = fp16(A x)                      fp32 accumulation over K, [r]
 *   u    = fp16(B t)                      fp32 accumulation over r
 *   c    = fp16(float(u) * float32(s))
 *   y    = fp16(base + c)
 * and y takes the linear's epilogue step in place of fp16(acc): o_proj / down_proj fp16(residual + y); gate / up
 * silu(y_gate) * y_up at the SiLU-gate epilogue's rounding points; q / k / v: y is what RoPE and the KV append read.
 * (Dropout is the identity, fan_in_fan_out = False, bias = "none".)  c is added before the residual, as PEFT does.
 * Merging adds fp16(fp16(B A) * s) to W (fp32 accumulation over r) and rounds to fp16.
 * t of the <= 4-row (decode) shrink sums K in a tree over 256 threads; the prefill shrink sums K in ascending order.
 * Rows n of a fused weight read t columns ((n / grp) % nsub) * r + [0, r): q|k|v grp = hidden, nsub 3; gate|up in
 * 128-row blocks grp = 128, nsub 2; o / down grp = N, nsub 1.  A sub-block whose bit in `mask` is clear has no
 * adapter there: y = base.  1 <= r <= 64.                                                                           */
typedef struct seedb200_lora_operand {
  const void* T;          /* [M, r * nsub] fp16: the shrink output t of every row                                  */
  int64_t ldt;
  const void* B;          /* [N, r] fp16 in the weight's fused row layout                                           */
  int32_t r, grp, nsub;
  uint32_t mask;
  float scale;            /* s = lora_alpha / r                                                                     */
  void* workspace;        /* [M, N] fp16 for the base product; may be NULL for mode 0 without residual (in place)   */
} seedb200_lora_operand;
typedef struct seedb200_gemm_lora_desc {
  seedb200_gemm_desc gemm;          /* mode 0 (optionally with residual) or 1; no bias, act, LN fold or row remap */
  seedb200_lora_operand lora;
} seedb200_gemm_lora_desc;
/* T [M, r_tot] (row stride ldt) = fp16(x . A^T), A [r_tot, K] fp16 dense, r_tot <= 192.  norm_w (M <= 4 only, x dense):
 * x is RMS-normalised while staged with seedb200_gemv's arithmetic, so T matches what the fused-norm GEMV multiplies. */
int seedb200_lora_shrink(const void* x, int64_t ldx, const void* norm_w, float eps, const void* A, int M, int K,
                         int r_tot, void* T, int64_t ldt, void* stream);
/* seedb200_gemm / seedb200_gemv with the LoRA branch.  GEMV (M <= 4): the expand runs in the GEMV's epilogue (no
 * workspace).  GEMM: the base product (unchanged kernel, mode 0 into the workspace), then an expand kernel (residual
 * add, or the SiLU gate with the GEMM epilogue's SiLU).                                                           */
int seedb200_gemm_lora(const seedb200_gemm_lora_desc* d, void* stream);
int seedb200_gemv_lora(const void* x, const void* W, int64_t ldw, void* out, const void* residual, const void* norm_w,
                       float eps, int M, int N, int K, int mode, const seedb200_lora_operand* lora, void* stream);
/* Loads a PEFT LoRA adapter into an fp16 handle: "model.layers.N.<self_attn|mlp>.<proj>.lora_A.weight" [r,K] and
 * ".lora_B.weight" [N,r], fp16.  Every layer must carry the same target set; one r and alpha for all (s = alpha / r).
 * Every tensor is validated before anything is allocated, then copied into handle-owned fused layouts (the caller
 * may free them).  A second load replaces the first.  Captured decode graphs are dropped.  int8 and 4-bit
 * handles refuse.                                                                                                    */
int seedb200_llama_lora_load(seedb200_llama* llm, const seedb200_tensor* tensors, int n, int r, float alpha);
/* Adds the loaded adapter into the fused weights (W = fp16(W + fp16(fp16(B A) * s))) and frees it; the model then
 * runs exactly the base kernels.  o_proj and down_proj are borrowed, so the caller's tensors change in place, as
 * PEFT's merge changes the base model's.  Fails when no adapter is loaded.                                        */
int seedb200_llama_lora_merge(seedb200_llama* llm);
/* Re-points borrowed fp16 tensors: "model.embed_tokens.weight" and "lm_head.weight" ([V', hidden]; a vocabulary
 * change needs both, with one V'), "model.norm.weight", "model.layers.N.input_layernorm.weight",
 * "model.layers.N.post_attention_layernorm.weight".  All are validated first.  A vocabulary change reallocates the
 * max_batch-sized buffers (the KV cache contents are dropped); captured graphs are always dropped.                  */
int seedb200_llama_replace_weights(seedb200_llama* llm, const seedb200_tensor* tensors, int n);

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
