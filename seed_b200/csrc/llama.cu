// llama.cu -- seedb200_llama: models/llama_xformer.py LlamaForCausalLM.forward (:661-743) /
// LlamaModel.forward (:496-627) / LlamaDecoderLayer.forward (:280-332) as a fixed launch sequence.
//
// What changes relative to the reference graph (SURVEY.md 2.4 rows L1-L10):
//   * q/k/v projections run as ONE GEMM over a fused [3h, h] weight, gate/up as ONE GEMM whose epilogue
//     applies SiLU(gate)*up (weights interleaved in 128-row blocks at create time);
//   * the dense additive mask (:50-92, :552-557) and the per-layer `attention_mask.sum() == 0` host sync
//     (:255) are gone: causality is a kernel flag;
//   * the KV cache is preallocated [B, H, max_seq, D] and appended in place by the RoPE kernel instead of
//     torch.cat per layer per step (:236-237);
//   * batch-1 decode (S == 1) switches to the HBM-bound GEMV / split-KV kernels.
// Weights named like the HF checkpoint (model.layers.N.self_attn.q_proj.weight ...); norms, embed_tokens and lm_head
// are borrowed.  The seven decoder linears of a layer (kLinear) are sub-blocks of four fused linears (fused()): q|k|v
// concatenated, o, gate|up interleaved in blocks of 128 rows, down.  Weights, their scales and LoRA B share that row
// order.  A handle holds its decoder linears in one WeightFormat -- fp16 (q|k|v and gate|up copied into handle-owned
// buffers, o and down borrowed), LLM.int8() CB + SCB, or bitsandbytes FP4 / NF4 codes + absmax -- and
// decoder_linear() is the one place that picks the kernels for it.
#include <string.h>

#include <map>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "common.cuh"
#include "ops.h"
#include "select.cuh"

namespace sb {
enum WeightFormat { W_F16, W_INT8, W_4BIT };
// one fused decoder linear [N, K]: fp16 w (s == nullptr), int8 CB [N, K] + SCB [N], or 4-bit packed codes [N, K/2] +
// absmax [N, K/64]
struct LinW { const void* w; const float* s; };
struct LlamaLayerW {
  const __half *in_ln, *post_ln;
  __half *k_cache, *v_cache;
  LinW lin[4];
};
// LoRA adapter of one layer, per fused linear g (0 q|k|v, 1 o, 2 gate|up, 3 down): A_cat [nsub r, K], B [N, r]
struct LoraLayer {
  const __half* A[4];
  const __half* B[4];
};
}  // namespace sb

struct seedb200_llama {
  seedb200_llama_config cfg;
  std::map<std::string, seedb200_tensor> w;
  std::vector<void*> owned;
  std::vector<void*> row_owned;   // buffers sized by max_batch (seedb200_llama_reserve_rows reallocates them)
  const __half *embed, *norm_w, *lm_head;
  std::vector<sb::LlamaLayerW> layers;
  const void *cos_t, *sin_t;
  int max_pos;
  __half *x, *nb, *qkv, *q, *att, *gu, *hn, *last;
  float* da_ws;
  int* da_tickets;
  int last_T;
  int device;
  // ---- device-resident generation loop (seedb200_llama_generate) ----
  int vpad;                       // logits row stride: vocab rounded up to a multiple of 8
  int* gstate;                    // [GS_SLOTS] the run's step counters
  int* gfinished;                 // [max_batch]
  int64_t* gtok;                  // [max_batch] token fed to the next decode forward
  int64_t* gout;                  // [max_batch, max_seq] each row's tokens: the prompt (kept when a history control
                                  // reads it), then the generated ones from column S
  __half* glogits;                // [max_batch, vpad]
  sb::GenParams* gparams;         // sampling parameters + eos/pad, read by the sampler at run time
  int* gstate_host;               // pinned mirror of gstate (early-stop polling)
  cudaStream_t gstream;           // private stream the decode step is captured on (the caller's may be the legacy
                                  // default stream, which cannot be captured); replays go to the caller's stream
  // captured decode units per (batch, beams, processing launch present, unit kind): beams 0 = the sampler loop;
  // contrastive units use beams = k; value = (graph, kernels inside one unit)
  std::map<std::tuple<int, int, int, int>, std::pair<cudaGraphExec_t, int>> graphs;
  sb::BeamState beam;             // beam-search state (rows = batch * beams <= max_batch)
  int used_graph;
  int gen_cache_len;
  sb::WeightFormat fmt;           // of the decoder linears
  // ---- int8 ----
  float threshold;
  std::vector<uint8_t> q_loaded;  // [layers][7]: the quantised (int8 or 4-bit) linear holds its weights
  __half* corr;                   // [max_batch * max_seq, 2 * ffn] outlier correction of the GEMM path
  int8_t* ca;                     // [max_batch * max_seq, max(hidden, ffn)] quantised activations (GEMM path)
  float* sca;                     // [max_batch * max_seq]
  int* olist;                     // [max(hidden, ffn)] outlier columns
  int* ocount;
  // ---- 4-bit ----
  int q4type;                     // SEEDB200_Q4_FP4 / SEEDB200_Q4_NF4
  __half* q4_scratch;             // [max fused linear] fp16 W' of the linear the GEMM path runs
  // ---- LoRA adapter (seedb200_llama_lora_load) ----
  int lora_r;                     // 0: no adapter
  float lora_s;                   // lora_alpha / r
  unsigned lora_mask[4];          // per fused linear: the sub-blocks (q, k, v / gate, up) that carry an adapter
  std::vector<sb::LoraLayer> lora;
  void* lora_mem;                 // every layer's A and B
  __half* lora_t;                 // [max_batch * max_seq, 3 * r] shrink output (row buffer)
  __half* lora_base;              // [max_batch * max_seq, max(2 ffn, hidden)] base product (row buffer)
  // ---- contrastive search: row buffers allocated by the first contrastive call ----
  __half* c_ctx;                  // [max_batch, max_seq, hidden] normalised context of each sequence
  __half* c_logits;               // [max_batch, vpad] each sequence's logits for the next step
  __half* c_probs;                // [max_batch] candidates' probabilities
  float* c_part;                  // [max_batch, CONTRAST_MAX_CTAS, CONTRAST_MAX_K] rank kernel's per-CTA maxima
  int* c_tickets;                 // [max_batch] rank kernel's arrival counters (zero between launches)
  sb::ContrastParams* c_params;   // k and the alpha scalars, read at run time (handle-owned)
};

namespace sb {

static int llama_find(const seedb200_llama* m, const std::string& name, const __half** out, int64_t n_expected) {
  auto it = m->w.find(name);
  if (it == m->w.end()) {
    set_error("llama_create: missing weight '%s'", name.c_str());
    return SEEDB200_ERR_INVALID;
  }
  const seedb200_tensor& t = it->second;
  int64_t n = 1;
  for (int i = 0; i < t.ndim; ++i) n *= t.shape[i];
  if (t.dtype != SEEDB200_F16 || n != n_expected || (reinterpret_cast<uintptr_t>(t.data) & 15) != 0) {
    set_error("llama_create: weight '%s' must be fp16, 16-byte aligned, %lld elements (got %lld)", name.c_str(),
              (long long)n_expected, (long long)n);
    return SEEDB200_ERR_INVALID;
  }
  *out = static_cast<const __half*>(t.data);
  return 0;
}

// an int8 linear: "<base>.weight" int8 [N,K] and "<base>.SCB" fp32 [N].  Both absent: *cb = *scb = NULL (the slot is
// filled later by seedb200_llama_int8_load_weight).
static int llama_find_i8(const seedb200_llama* m, const std::string& base, int64_t N, int64_t K, const int8_t** cb,
                         const float** scb) {
  const std::string wn = base + ".weight", sn = base + ".SCB";
  auto wi = m->w.find(wn), si = m->w.find(sn);
  *cb = nullptr;
  *scb = nullptr;
  if (wi == m->w.end() && si == m->w.end()) return 0;
  if (wi == m->w.end() || si == m->w.end()) {
    set_error("llama_create_int8: missing weight '%s'", (wi == m->w.end() ? wn : sn).c_str());
    return SEEDB200_ERR_INVALID;
  }
  const seedb200_tensor &w = wi->second, &s = si->second;
  int64_t nw = 1, ns = 1;
  for (int i = 0; i < w.ndim; ++i) nw *= w.shape[i];
  for (int i = 0; i < s.ndim; ++i) ns *= s.shape[i];
  if (w.dtype != SEEDB200_I8 || w.ndim != 2 || w.shape[0] != N || w.shape[1] != K || w.data == nullptr) {
    set_error("llama_create_int8: '%s' must be int8 [%lld, %lld] (dtype %d, %lld elements)", wn.c_str(),
              (long long)N, (long long)K, w.dtype, (long long)nw);
    return SEEDB200_ERR_INVALID;
  }
  if (s.dtype != SEEDB200_F32 || ns != N || s.data == nullptr) {
    set_error("llama_create_int8: '%s' must be fp32 [%lld] (dtype %d, %lld elements)", sn.c_str(), (long long)N,
              s.dtype, (long long)ns);
    return SEEDB200_ERR_INVALID;
  }
  *cb = static_cast<const int8_t*>(w.data);
  *scb = static_cast<const float*>(s.data);
  return 0;
}

// The decoder linears of a layer in HF order, each sub-block `sub` of fused linear g
struct DecoderLinear { const char* name; int g, sub; };
static const DecoderLinear kLinear[7] = {{"self_attn.q_proj", 0, 0}, {"self_attn.k_proj", 0, 1},
                                         {"self_attn.v_proj", 0, 2}, {"self_attn.o_proj", 1, 0},
                                         {"mlp.gate_proj", 2, 0},    {"mlp.up_proj", 2, 1},
                                         {"mlp.down_proj", 3, 0}};

// fused linear g of a layer: N x K, nsub sub-blocks of N / nsub rows interleaved in groups of grp rows
struct Fused { int N, K, grp, nsub; };
static Fused fused(const seedb200_llama* m, int g) {
  const int h = m->cfg.hidden, ffn = m->cfg.ffn;
  if (g == 0) return {3 * h, h, h, 3};
  if (g == 1) return {h, h, h, 1};
  if (g == 2) return {2 * ffn, h, 128, 2};
  return {h, ffn, h, 1};
}

// "model.layers.<l>.<linear i><suffix>" -> (l, i); false for any other name
static bool linear_of(const char* name, const char* suffix, int* layer, int* lin) {
  for (int k = 0; k < 7; ++k) {
    char tail[96];
    snprintf(tail, sizeof(tail), ".%s%s", kLinear[k].name, suffix);
    int l = -1, n = 0;
    if (sscanf(name, "model.layers.%d%n", &l, &n) == 1 && strcmp(name + n, tail) == 0) { *layer = l; *lin = k; return true; }
  }
  return false;
}

// copy the N / nsub rows (row_bytes each) of sub-block `sub` from src into their rows of fused linear F at dst
static int place_rows(void* dst, const void* src, size_t row_bytes, const Fused& F, int sub, cudaStream_t st) {
  const size_t grp = (size_t)F.grp * row_bytes;
  SB_CHECK_CUDA(cudaMemcpy2DAsync(static_cast<uint8_t*>(dst) + sub * grp, F.nsub * grp, src, grp, grp,
                                  (size_t)(F.N / F.nsub / F.grp), cudaMemcpyDeviceToDevice, st));
  return 0;
}

// bytes of one row of K weights (*w) and of its scales (*s) in the handle's format
static void row_bytes(const seedb200_llama* m, int64_t K, size_t* w, size_t* s) {
  if (m->fmt == W_INT8) { *w = K; *s = 4; }
  else if (m->fmt == W_4BIT) { *w = K / 2; *s = K / 64 * 4; }
  else { *w = 2 * K; *s = 0; }
}

// at least 256 bytes, recorded in `list` (m->owned, or m->row_owned for the buffers sized by max_batch)
template <typename T>
static int llama_alloc(std::vector<void*>& list, T** p, size_t elems) {
  void* q = nullptr;
  size_t bytes = elems * sizeof(T);
  SB_CHECK_CUDA(cudaMalloc(&q, bytes < 256 ? 256 : bytes));
  list.push_back(q);
  *p = static_cast<T*>(q);
  return 0;
}

// every buffer whose size follows max_batch: KV caches, activations, int8 workspaces, generation and beam state
static int llama_alloc_rows(seedb200_llama* m, cudaStream_t st) {
  const seedb200_llama_config& c = m->cfg;
  const int64_t h = c.hidden, ffn = c.ffn;
  const size_t cache_elems = (size_t)c.max_batch * c.heads * c.max_seq * c.head_dim;
  std::vector<void*>& rows = m->row_owned;
  for (LlamaLayerW& L : m->layers) {
    SB_PROPAGATE(llama_alloc(rows, &L.k_cache, cache_elems));
    SB_PROPAGATE(llama_alloc(rows, &L.v_cache, cache_elems));
  }
  const size_t T = (size_t)c.max_batch * c.max_seq;
  SB_PROPAGATE(llama_alloc(rows, &m->x, T * h));
  SB_PROPAGATE(llama_alloc(rows, &m->nb, T * h));
  SB_PROPAGATE(llama_alloc(rows, &m->qkv, T * 3 * h));
  SB_PROPAGATE(llama_alloc(rows, &m->q, T * h));
  SB_PROPAGATE(llama_alloc(rows, &m->att, T * h));
  SB_PROPAGATE(llama_alloc(rows, &m->gu, T * ffn));
  SB_PROPAGATE(llama_alloc(rows, &m->hn, T * h));
  SB_PROPAGATE(llama_alloc(rows, &m->last, (size_t)c.max_batch * h));
  m->ca = nullptr; m->sca = nullptr; m->corr = nullptr;
  if (m->fmt == W_INT8) {
    SB_PROPAGATE(llama_alloc(rows, &m->corr, T * (size_t)(2 * ffn > 3 * h ? 2 * ffn : 3 * h)));
    SB_PROPAGATE(llama_alloc(rows, &m->ca, T * (size_t)(ffn > h ? ffn : h)));
    SB_PROPAGATE(llama_alloc(rows, &m->sca, T));
  }
  m->lora_t = nullptr; m->lora_base = nullptr;
  if (m->lora_r > 0) {
    SB_PROPAGATE(llama_alloc(rows, &m->lora_t, T * 3 * (size_t)m->lora_r));
    SB_PROPAGATE(llama_alloc(rows, &m->lora_base, T * (size_t)(2 * ffn > h ? 2 * ffn : h)));
  }
  SB_PROPAGATE(llama_alloc(rows, &m->da_ws, (size_t)c.max_batch * c.heads * decode_attention_max_splits(c.max_seq) * (128 + 2)));
  SB_PROPAGATE(llama_alloc(rows, &m->da_tickets, (size_t)c.max_batch * c.heads));   // zero now, left zero by every launch
  SB_CHECK_CUDA(cudaMemsetAsync(m->da_tickets, 0, (size_t)c.max_batch * c.heads * sizeof(int), st));
  SB_PROPAGATE(llama_alloc(rows, &m->gfinished, (size_t)c.max_batch));
  SB_PROPAGATE(llama_alloc(rows, &m->gtok, (size_t)c.max_batch));
  SB_PROPAGATE(llama_alloc(rows, &m->gout, (size_t)c.max_batch * c.max_seq));
  SB_PROPAGATE(llama_alloc(rows, &m->glogits, (size_t)c.max_batch * m->vpad));
  BeamState& b = m->beam;
  const size_t R = (size_t)c.max_batch;
  b.tokens = reinterpret_cast<long long*>(m->gtok);
  b.state = m->gstate;
  SB_PROPAGATE(llama_alloc(rows, &b.beam_scores, R));
  SB_PROPAGATE(llama_alloc(rows, &b.row_stats, 5 * R));
  SB_PROPAGATE(llama_alloc(rows, &b.cand_score, 2 * R));
  SB_PROPAGATE(llama_alloc(rows, &b.cand_idx, 2 * R));
  SB_PROPAGATE(llama_alloc(rows, &b.slot, R * c.max_seq));
  SB_PROPAGATE(llama_alloc(rows, &b.slot_tmp, R * c.max_seq));
  SB_PROPAGATE(llama_alloc(rows, &b.hist_tok, R * c.max_seq));
  SB_PROPAGATE(llama_alloc(rows, &b.hist_par, R * c.max_seq));
  SB_PROPAGATE(llama_alloc(rows, &b.hyp_score, R));
  SB_PROPAGATE(llama_alloc(rows, &b.hyp_len, R));
  SB_PROPAGATE(llama_alloc(rows, &b.hyp_beam, R));
  SB_PROPAGATE(llama_alloc(rows, &b.hyp_step, R));
  SB_PROPAGATE(llama_alloc(rows, &b.hyp_n, R));
  SB_PROPAGATE(llama_alloc(rows, &b.worst, R));
  SB_PROPAGATE(llama_alloc(rows, &b.done, R));
  b.tok = nullptr;                 // allocated by the first beam run with a history control
  m->c_ctx = nullptr;              // allocated by the first contrastive run
  m->c_logits = nullptr; m->c_probs = nullptr; m->c_part = nullptr; m->c_tickets = nullptr;
  b.max_seq = c.max_seq;
  return 0;
}

static void llama_free_rows(seedb200_llama* m) {
  for (void* p : m->row_owned) cudaFree(p);
  m->row_owned.clear();
}

static int llama_build(seedb200_llama* m) {
  const seedb200_llama_config& c = m->cfg;
  const int64_t h = c.hidden, ffn = c.ffn, V = c.vocab;
  cudaStream_t st = 0;
  char nm[256];
  // every tensor is checked before anything is allocated
  SB_PROPAGATE(llama_find(m, "model.embed_tokens.weight", &m->embed, V * h));
  SB_PROPAGATE(llama_find(m, "model.norm.weight", &m->norm_w, h));
  SB_PROPAGATE(llama_find(m, "lm_head.weight", &m->lm_head, V * h));
  if (m->fmt == W_4BIT) {  // no pre-packed 4-bit names exist: every decoder linear comes through seedb200_llama_4bit_load_weight
    for (const auto& kv : m->w) {
      int l, i;
      SB_REQUIRE(!linear_of(kv.first.c_str(), ".weight", &l, &i), "llama_create_4bit: '%s' is a decoder linear: load "
                 "it with seedb200_llama_4bit_load_weight", kv.first.c_str());
    }
  }
  // [layer][linear] the checkpoint's fp16 weight or int8 CB, and the int8 SCB (null: quantised into its rows later)
  std::vector<const void*> src((size_t)c.layers * 7, nullptr);
  std::vector<const float*> src_s((size_t)c.layers * 7, nullptr);
  m->layers.assign(c.layers, LlamaLayerW{});
  for (int l = 0; l < c.layers; ++l) {
    LlamaLayerW& L = m->layers[l];
    auto key = [&](const char* s) { snprintf(nm, sizeof(nm), "model.layers.%d.%s", l, s); return std::string(nm); };
    SB_PROPAGATE(llama_find(m, key("input_layernorm.weight"), &L.in_ln, h));
    SB_PROPAGATE(llama_find(m, key("post_attention_layernorm.weight"), &L.post_ln, h));
    for (int i = 0; i < 7; ++i) {
      const Fused F = fused(m, kLinear[i].g);
      const int64_t N = F.N / F.nsub, K = F.K;
      const size_t j = (size_t)l * 7 + i;
      if (m->fmt == W_F16) {
        const __half* w;
        SB_PROPAGATE(llama_find(m, key(kLinear[i].name) + ".weight", &w, N * K));
        src[j] = w;
      } else if (m->fmt == W_INT8) {
        const int8_t* cb;
        SB_PROPAGATE(llama_find_i8(m, key(kLinear[i].name), N, K, &cb, &src_s[j]));
        src[j] = cb;
      }
    }
  }
  // then the fused linears: handle-owned buffers filled with the checkpoint's rows
  if (m->fmt != W_F16) m->q_loaded.assign((size_t)c.layers * 7, 0);
  for (int l = 0; l < c.layers; ++l)
    for (int g = 0; g < 4; ++g) {
      const Fused F = fused(m, g);
      const bool borrow = m->fmt == W_F16 && F.nsub == 1;   // fp16 o and down are used (and LoRA-merged) in place
      size_t wrow, srow;
      row_bytes(m, F.K, &wrow, &srow);
      uint8_t* w = nullptr;
      float* s = nullptr;
      if (!borrow) SB_PROPAGATE(llama_alloc(m->owned, &w, (size_t)F.N * wrow));
      if (srow > 0) SB_PROPAGATE(llama_alloc(m->owned, &s, (size_t)F.N * srow / 4));
      m->layers[l].lin[g] = {w, s};
      for (int i = 0; i < 7; ++i) {
        const size_t j = (size_t)l * 7 + i;
        if (kLinear[i].g != g || src[j] == nullptr) continue;
        if (borrow) m->layers[l].lin[g].w = src[j];
        else SB_PROPAGATE(place_rows(w, src[j], wrow, F, kLinear[i].sub, st));
        if (s) SB_PROPAGATE(place_rows(s, src_s[j], srow, F, kLinear[i].sub, st));
        if (m->fmt != W_F16) m->q_loaded[j] = 1;
      }
    }
  SB_PROPAGATE(get_rope_tables(c.head_dim, c.rope_base, c.max_seq, &m->cos_t, &m->sin_t, &m->max_pos, st));
  m->q4_scratch = nullptr;
  if (m->fmt == W_4BIT) {   // allocated here so that peak memory does not depend on the first prefill
    const size_t qkv = (size_t)3 * h * h, gu = (size_t)2 * ffn * h;
    SB_PROPAGATE(llama_alloc(m->owned, &m->q4_scratch, qkv > gu ? qkv : gu));
  }
  m->olist = nullptr; m->ocount = nullptr;
  if (m->fmt == W_INT8) {
    SB_PROPAGATE(llama_alloc(m->owned, &m->olist, (size_t)(ffn > h ? ffn : h)));
    SB_PROPAGATE(llama_alloc(m->owned, &m->ocount, 1));
  }
  m->vpad = (c.vocab + 7) / 8 * 8;
  SB_PROPAGATE(llama_alloc(m->owned, &m->gstate, GS_SLOTS));
  SB_PROPAGATE(llama_alloc(m->owned, &m->gparams, 1));
  SB_PROPAGATE(llama_alloc(m->owned, &m->beam.params, 1));
  SB_PROPAGATE(llama_alloc(m->owned, &m->beam.n_out, 1));
  SB_PROPAGATE(llama_alloc(m->owned, &m->c_params, 1));
  SB_PROPAGATE(llama_alloc_rows(m, st));
  SB_CHECK_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->gstate_host), GS_SLOTS * sizeof(int)));
  SB_CHECK_CUDA(cudaStreamCreateWithFlags(&m->gstream, cudaStreamNonBlocking));
  SB_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int get_option(const char* key);

static seedb200_gemm_desc gemm_desc(int ctas, int M, int N, int K, const void* A, const void* W, void* out, int64_t ldo,
                                    const void* residual, int mode) {
  seedb200_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.M = M; d.N = N; d.K = K; d.A = A; d.lda = K; d.W = W; d.ldw = K;
  d.out = out; d.ldo = ldo; d.residual = residual; d.ldr = ldo; d.mode = mode; d.ctas = ctas;
  return d;
}

static int lin(cudaStream_t st, int ctas, int M, int N, int K, const void* A, const void* W, void* out, int64_t ldo,
               const void* residual, int mode, const void* norm_w = nullptr, float eps = 0.0f) {
  // norm_w: only on the M <= 4 (decode) path, where the GEMV normalises its activations while staging them
  if (M <= 4) return gemv(A, W, K, out, residual, norm_w, eps, M, N, K, mode, st, ldo);
  return gemm(gemm_desc(ctas, M, N, K, A, W, out, ldo, residual, mode), st);
}

static seedb200_lora_operand lora_operand(const seedb200_llama* m, int l, int g, void* workspace) {
  const Fused G = fused(m, g);
  seedb200_lora_operand lo;
  memset(&lo, 0, sizeof(lo));
  lo.T = m->lora_t; lo.ldt = (int64_t)G.nsub * m->lora_r; lo.B = m->lora[l].B[g];
  lo.r = m->lora_r; lo.grp = G.grp; lo.nsub = G.nsub; lo.mask = m->lora_mask[g]; lo.scale = m->lora_s;
  lo.workspace = workspace;
  return lo;
}

// Fused decoder linear g of layer l on M rows of A, in the handle's weight format, plus the adapter's LoRA branch when
// one covers g.  Outputs are dense rows of N columns (N/2 in mode 1: SiLU(gate) * up).  norm_w: only for M <= 4, where
// the GEMV normalises its activations while staging them.
static int decoder_linear(seedb200_llama* m, cudaStream_t st, int l, int g, int M, const void* A, void* out,
                          const void* residual, int mode, const void* norm_w = nullptr, float eps = 0.0f) {
  const Fused F = fused(m, g);
  const LinW& W = m->layers[l].lin[g];
  const int64_t ldo = mode == 1 ? F.N / 2 : F.N;
  const int ctas = m->cfg.gemm_ctas;
  if (m->fmt == W_INT8) {   // more rows: activation quantisation + int8 wgmma GEMM
    if (M <= 4) return gemv_int8(A, norm_w, eps, m->threshold, W.w, W.s, out, residual, M, F.N, F.K, mode, st);
    SB_PROPAGATE(int8_quantize_act(A, F.K, M, F.K, m->threshold, m->ca, m->sca, m->olist, m->ocount, st));
    seedb200_gemm_int8_desc d;
    memset(&d, 0, sizeof(d));
    d.M = M; d.N = F.N; d.K = F.K;
    d.A = m->ca; d.SCA = m->sca; d.A16 = A; d.outliers = m->olist; d.n_outliers = m->ocount;
    d.W = W.w; d.SCB = W.s; d.out = out; d.residual = residual; d.mode = mode; d.workspace = m->corr;
    return gemm_int8(d, st);
  }
  if (m->fmt == W_4BIT) {   // more rows: MatMul4Bit's dequantise-then-linear, through the fp16 scratch
    if (M <= 4) return gemv_4bit(A, norm_w, eps, W.w, W.s, m->q4type, out, residual, M, F.N, F.K, mode, st);
    SB_PROPAGATE(dequantize_4bit(W.w, W.s, F.N, F.K, m->q4type, m->q4_scratch, F.K, st));
    return lin(st, ctas, M, F.N, F.K, A, m->q4_scratch, out, ldo, residual, mode);
  }
  if (m->lora_r == 0 || m->lora_mask[g] == 0)
    return lin(st, ctas, M, F.N, F.K, A, W.w, out, ldo, residual, mode, norm_w, eps);
  const seedb200_lora_operand lo =
      lora_operand(m, l, g, mode == 0 && residual == nullptr ? nullptr : static_cast<void*>(m->lora_base));
  SB_PROPAGATE(lora_shrink(A, F.K, norm_w, eps, m->lora[l].A[g], M, F.K, (int)lo.ldt, m->lora_t, lo.ldt, st));
  if (M <= 4) return gemv_lora(A, W.w, F.K, out, residual, norm_w, eps, M, F.N, F.K, mode, lo, st, ldo);
  return gemm_lora(gemm_desc(ctas, M, F.N, F.K, A, W.w, out, ldo, residual, mode), lo, st);
}

// decoder linear g on RMSNorm(m->x) with weight norm_w: folded into the GEMV for T <= 4 rows, otherwise normalised
// into m->nb first
static int normed_linear(seedb200_llama* m, cudaStream_t st, int l, int g, int T, const __half* norm_w, void* out,
                         int mode) {
  const int h = m->cfg.hidden;
  const float eps = m->cfg.rms_eps;
  if (T <= 4) return decoder_linear(m, st, l, g, T, m->x, out, nullptr, mode, norm_w, eps);
  SB_PROPAGATE(rmsnorm(m->x, h, norm_w, m->nb, h, T, h, eps, st));
  return decoder_linear(m, st, l, g, T, m->nb, out, nullptr, mode);
}

// dyn (device, optional): {cache length, ...} read by the RoPE/append and decode-attention kernels instead of the
// host value `past_len` -- what makes a captured decode step position independent (S must be 1).
static int llama_forward(seedb200_llama* m, const int64_t* input_ids, const void* inputs_embeds,
                         const int64_t* position_ids, int B, int S, int past_len, int logits_mode, void* logits,
                         int64_t logits_ld, cudaStream_t st, const int* dyn = nullptr, const int* slot = nullptr) {
  const seedb200_llama_config& c = m->cfg;
  const int h = c.hidden, H = c.heads, D = c.head_dim, V = c.vocab, ct = c.gemm_ctas;
  const int T = B * S;
  if (input_ids)
    SB_PROPAGATE(embedding(m->embed, h, input_ids, T, h, m->x, h, V, st));
  else
    SB_CHECK_CUDA(cudaMemcpyAsync(m->x, inputs_embeds, (size_t)T * h * 2, cudaMemcpyDeviceToDevice, st));
  const float scale = 1.0f / sqrtf((float)D);   // xformers default scale
  const int kv_len = past_len + S;
  PdlScope pdl(T <= 4 && get_option("decode_pdl") != 0);   // decode chain: programmatic dependent launches
  const bool fused_attn = S == 1 && get_option("decode_fused_attention") != 0 && decode_attention_rope_supported(D, c.max_seq);
  for (int l = 0; l < c.layers; ++l) {
    const LlamaLayerW& L = m->layers[l];
    SB_PROPAGATE(normed_linear(m, st, l, 0, T, L.in_ln, m->qkv, 0));
    // qkv rows are [q | k | v] per token, each [H, D]
    if (fused_attn) {
      // cached decode step: RoPE + append + attention in one launch (bit-identical to the pair below up to 512 keys)
      SB_PROPAGATE(decode_attention_rope(m->qkv, position_ids, B, H, D, past_len, c.max_seq, m->max_pos, m->cos_t,
                                         m->sin_t, L.k_cache, L.v_cache, m->att, scale, st, dyn, slot));
    } else {
    SB_PROPAGATE(rope_kv_append_tables(m->qkv, position_ids, B, S, H, D, past_len, c.max_seq, m->max_pos, m->cos_t,
                                       m->sin_t, m->q, L.k_cache, L.v_cache, st, dyn));
    if (S == 1) {
      SB_PROPAGATE(decode_attention(m->q, L.k_cache, L.v_cache, m->att, B, H, D, kv_len, c.max_seq, scale, m->da_ws, st, dyn,
                                    m->da_tickets, slot));
    } else {
      seedb200_attn_desc a;
      memset(&a, 0, sizeof(a));
      a.q = m->q; a.k = L.k_cache; a.v = L.v_cache; a.o = m->att;
      a.q_bs = (int64_t)S * h; a.q_hs = D; a.q_ts = h;
      a.k_bs = (int64_t)H * c.max_seq * D; a.k_hs = (int64_t)c.max_seq * D; a.k_ts = D;
      a.v_bs = a.k_bs; a.v_hs = a.k_hs; a.v_ts = a.k_ts;
      a.o_bs = (int64_t)S * h; a.o_hs = D; a.o_ts = h;
      a.batch = B; a.heads = H; a.nq = S; a.nk = kv_len; a.head_dim = D; a.causal = 1; a.scale = scale;
      SB_PROPAGATE(attention(a, st));
    }
    }
    SB_PROPAGATE(decoder_linear(m, st, l, 1, T, m->att, m->x, m->x, 0));
    SB_PROPAGATE(normed_linear(m, st, l, 2, T, L.post_ln, m->gu, 1));
    SB_PROPAGATE(decoder_linear(m, st, l, 3, T, m->gu, m->x, m->x, 0));
  }
  SB_PROPAGATE(rmsnorm(m->x, h, m->norm_w, m->hn, h, T, h, c.rms_eps, st));
  m->last_T = T;
  if (logits == nullptr) return 0;
  if (logits_mode == 0) {
    SB_PROPAGATE(lin(st, ct, T, V, h, m->hn, m->lm_head, logits, logits_ld, nullptr, 0));
  } else {
    const __half* src = m->hn;
    if (S > 1) {   // gather the last position of every sequence
      SB_CHECK_CUDA(cudaMemcpy2DAsync(m->last, (size_t)h * 2, m->hn + (size_t)(S - 1) * h, (size_t)S * h * 2,
                                      (size_t)h * 2, B, cudaMemcpyDeviceToDevice, st));
      src = m->last;
    }
    SB_PROPAGATE(lin(st, ct, B, V, h, src, m->lm_head, logits, logits_ld, nullptr, 0));
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// generation loop on the device (scripts/seed_llama_inference_8B.py:26-38 -> HF sample/greedy_search +
// llama_xformer.py:745-776): prefill, then max_new_tokens x (sampler -> cached decode forward).
// ---------------------------------------------------------------------------------------------------------------
__global__ void gen_reset_kernel(GenParams gp, GenParams* dst, int* state, int* finished, int past_len, int B) {
  if (threadIdx.x == 0) {
    *dst = gp;
    gen_state_reset(state, past_len);
  }
  if (threadIdx.x < B) finished[threadIdx.x] = 0;
}

// the lineage table of R = B * n sampling rows that share B prompts (num_return_sequences = n): row r reads prompt
// row r / n for positions < S and its own row from S on.  Sampling rows never change parent, so it is written once.
__global__ void sample_lineage_kernel(int* slot, int R, int n, int S, int max_seq) {
  const long long total = (long long)R * max_seq;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / max_seq), p = (int)(e - (long long)r * max_seq);
    slot[e] = p < S ? r / n : r;
  }
}

// the prologue of the sampler and contrastive loops: the parameters and the counters on the device, and the prompt as
// the rows' history in gout[:, :S] when a history control reads it (the loop appends from column S).  B prompts,
// n rows each: row r's history starts with prompt r / n.
static int gen_begin(seedb200_llama* m, const int64_t* prompt_ids, int B, int S, const GenParams& gp, cudaStream_t st,
                     int n = 1) {
  const int R = B * n;
  gen_reset_kernel<<<1, (R + 31) / 32 * 32, 0, st>>>(gp, m->gparams, m->gstate, m->gfinished, S, R);
  SB_LAUNCH_CHECK();
  if (logits_history_active(gp.proc))
    for (int j = 0; j < n; ++j)
      SB_CHECK_CUDA(cudaMemcpy2DAsync(m->gout + (size_t)j * m->cfg.max_seq, (size_t)n * m->cfg.max_seq * 8, prompt_ids,
                                      (size_t)S * 8, (size_t)S * 8, B, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// the prefill wrote prompt b's logits to glogits row b * n (rows n apart); copy it to rows b * n + 1 .. b * n + n - 1,
// so that the first step of every row (or beam group) reads its prompt's logits as if the prompt had been expanded
static int gen_spread_logits(seedb200_llama* m, int B, int n, cudaStream_t st) {
  const size_t row = (size_t)m->vpad * 2, pitch = (size_t)n * row;
  for (int j = 1; j < n; ++j)
    SB_CHECK_CUDA(cudaMemcpy2DAsync(m->glogits + (size_t)j * m->vpad, pitch, m->glogits, pitch, row, B,
                                    cudaMemcpyDeviceToDevice, st));
  return 0;
}

static int gen_state_read(seedb200_llama* m, cudaStream_t st) {
  SB_CHECK_CUDA(cudaMemcpyAsync(m->gstate_host, m->gstate, GS_SLOTS * sizeof(int), cudaMemcpyDeviceToHost, st));
  SB_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// the epilogue of the sampler and contrastive loops: n_valid steps ran; with an eos id, the steps HF keeps are
// GS_VALID.  Their tokens go to tokens_out [B, max_new] (optional).
static int gen_end(seedb200_llama* m, int B, int S, int max_new, int64_t eos, int n_valid, int64_t* tokens_out,
                   int* n_generated_host, cudaStream_t st) {
  if (eos >= 0) {
    SB_PROPAGATE(gen_state_read(m, st));
    n_valid = m->gstate_host[GS_VALID];
  }
  if (tokens_out != nullptr && n_valid > 0)
    SB_CHECK_CUDA(cudaMemcpy2DAsync(tokens_out, (size_t)max_new * 8, m->gout + S, (size_t)m->cfg.max_seq * 8,
                                    (size_t)n_valid * 8, B, cudaMemcpyDeviceToDevice, st));
  if (n_generated_host != nullptr) *n_generated_host = n_valid;
  return 0;
}

// the history processors of the step: on the sampler's rows (history = gout) or on every beam row (history = the
// token table; beam_ld 0 = the prefill's one row per sequence, which every beam reads)
static int gen_process(seedb200_llama* m, int B, int beams, int64_t beam_ld, cudaStream_t st) {
  if (beams == 0)
    return logits_process<int64_t>(m->glogits, m->vpad, 0, B, 1, m->cfg.vocab, nullptr, &m->gparams->proc, m->gstate,
                                   m->gout, m->cfg.max_seq, 1, 0, false, st);
  return logits_process<int>(m->glogits, beam_ld == 0 ? m->vpad : (int64_t)beams * m->vpad, beam_ld, B,
                             beam_ld == 0 ? 1 : beams, m->cfg.vocab, nullptr, &m->beam.params->proc, m->gstate,
                             m->beam.tok, m->cfg.max_seq, beams, 0, true, st);
}

// one step of contrastive search at k = beams: the history processors on each sequence's logits when `proc`, the
// candidates, the forward of B * k candidate rows through the lineage table, then rank + select (which also advances
// the device counters)
static int contrastive_unit(seedb200_llama* m, int B, int k, int proc, cudaStream_t st) {
  const seedb200_llama_config& c = m->cfg;
  if (proc)
    SB_PROPAGATE(logits_process<int64_t>(m->c_logits, m->vpad, 0, B, 1, c.vocab, nullptr, &m->gparams->proc,
                                         m->gstate, m->gout, c.max_seq, 1, 0, false, st));
  SB_PROPAGATE(contrastive_candidates(m->c_logits, m->vpad, B, c.vocab, nullptr, m->c_params, m->gstate, 0,
                                      m->beam.slot, c.max_seq, m->gtok, m->c_probs, st, m->gparams));
  SB_PROPAGATE(llama_forward(m, m->gtok, nullptr, nullptr, B * k, 1, 0, 1, m->glogits, m->vpad, st, m->gstate,
                             m->beam.slot));
  ContrastRank r;
  memset(&r, 0, sizeof(r));
  r.ctx = m->c_ctx; r.ctx_ld = (int64_t)c.max_seq * c.hidden; r.ctx_rows = c.max_seq; r.H = c.hidden;
  r.h = m->hn; r.probs = m->c_probs; r.p_dev = m->c_params; r.k = k; r.state = m->gstate;
  r.part = m->c_part; r.tickets = m->c_tickets; r.G = contrastive_rank_ctas(c.max_seq, B);
  r.cand_ids = reinterpret_cast<const long long*>(m->gtok); r.cand_logits = m->glogits; r.seq_logits = m->c_logits;
  r.vpad = m->vpad; r.slot = m->beam.slot; r.max_seq = c.max_seq; r.gp = m->gparams;
  r.out = reinterpret_cast<long long*>(m->gout); r.out_ld = c.max_seq; r.finished = m->gfinished; r.B = B;
  return contrastive_rank(r, st);
}

// what a decode unit runs, part of its graph key: the sampler or beam step, a contrastive step, the sampler step
// whose rows share their prompts through the lineage table, or the beam step that also warps beam sampling's scores
enum UnitKind { UNIT_PLAIN, UNIT_CONTRASTIVE, UNIT_SHARED, UNIT_BEAM_WARP };

// one unit of the loop: cached forward of the tokens in m->gtok, the history processors when `proc`, then the sampler
// (beams == 0) or the beam candidates and scorer (which also advance the device counters); or one contrastive step.
// Sampler rows of UNIT_SHARED read their prompt through the lineage table (num_return_sequences > 1).  Every launch
// argument is a handle-owned pointer or a constant: the unit can be captured once per (B, beams, proc, kind).
static int gen_unit(seedb200_llama* m, int B, int beams, int proc, int kind, cudaStream_t st) {
  PdlScope pdl(get_option("decode_pdl") != 0);
  if (kind == UNIT_CONTRASTIVE) return contrastive_unit(m, B, beams, proc, st);
  if (beams == 0) {
    SB_PROPAGATE(llama_forward(m, m->gtok, nullptr, nullptr, B, 1, 0, 1, m->glogits, m->vpad, st, m->gstate,
                               kind == UNIT_SHARED ? m->beam.slot : nullptr));
    if (proc) SB_PROPAGATE(gen_process(m, B, 0, 0, st));
    SB_PROPAGATE(sample(m->glogits, m->vpad, B, m->cfg.vocab, nullptr, m->gparams, 0, m->gstate, /*advance_cache=*/1,
                        m->gtok, m->gout, m->cfg.max_seq, m->gfinished, st));
    return 0;
  }
  const int rows = B * beams;
  SB_PROPAGATE(llama_forward(m, m->gtok, nullptr, nullptr, rows, 1, 0, 1, m->glogits, m->vpad, st, m->gstate,
                             m->beam.slot));
  if (proc) SB_PROPAGATE(gen_process(m, B, beams, m->vpad, st));
  SB_PROPAGATE(beam_select(m->glogits, (int64_t)beams * m->vpad, m->vpad, B, beams, m->cfg.vocab, m->beam.beam_scores,
                           nullptr, m->beam.params, 0, m->gstate, m->beam.row_stats, m->beam.cand_score,
                           m->beam.cand_idx, st, kind == UNIT_BEAM_WARP));
  SB_PROPAGATE(beam_score(m->beam, B, beams, m->cfg.vocab, /*advance_cache=*/1, st));
  return 0;
}

static int gen_capture(seedb200_llama* m, int B, int beams, int proc, int kind) {
  cudaGraph_t graph = nullptr;
  cudaStream_t st = m->gstream;
  SB_CHECK_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const int64_t before = seedb200_launch_count();
  const int s = gen_unit(m, B, beams, proc, kind, st);
  const int unit = (int)(seedb200_launch_count() - before);
  count_launch(-unit);                        // captured, not executed
  const cudaError_t e = cudaStreamEndCapture(st, &graph);
  if (s != 0) {
    if (graph) cudaGraphDestroy(graph);
    cudaGetLastError();
    return s;
  }
  if (e != cudaSuccess || graph == nullptr) {
    set_error("llama_generate: stream capture of the decode step failed: %s", cudaGetErrorString(e));
    cudaGetLastError();
    return SEEDB200_ERR_CUDA;
  }
  cudaGraphExec_t exec = nullptr;
  const cudaError_t ei = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ei != cudaSuccess) {
    set_error("llama_generate: cudaGraphInstantiate failed: %s", cudaGetErrorString(ei));
    cudaGetLastError();
    return SEEDB200_ERR_CUDA;
  }
  m->graphs[std::make_tuple(B, beams, proc, kind)] = std::make_pair(exec, unit);
  return 0;
}

// when a loop with an eos id stops early: a step ran with every sequence already finished, or every beam search is done
enum GenStop { STOP_NEVER, STOP_ALL_FINISHED, STOP_BEAMS_DONE };

// run `units` decode units (the first eagerly, the rest replayed from the (B, beams, proc, kind) graph when
// use_graph); unless STOP_NEVER, the counters are read every 32 units and the loop ends once `stop` holds.
// Returns units run.
static int gen_run_units(seedb200_llama* m, int B, int beams, int proc, int kind, int units, int use_graph,
                         GenStop stop, cudaStream_t st, int* done_out) {
  int done = 0;
  m->used_graph = 0;
  if (units > 0) {   // first unit eagerly (also resolves every lazily-set function attribute before a capture)
    SB_PROPAGATE(gen_unit(m, B, beams, proc, kind, st));
    done = 1;
  }
  const auto key = std::make_tuple(B, beams, proc, kind);
  if (units > done && use_graph) {
    if (m->graphs.find(key) == m->graphs.end()) {
      int s = gen_capture(m, B, beams, proc, kind);
      if (s != 0 && get_option("decode_pdl") != 0) {   // retry without programmatic launches inside the graph
        seedb200_set_option("decode_pdl", 0);
        s = gen_capture(m, B, beams, proc, kind);
        seedb200_set_option("decode_pdl", 1);
      }
      if (s != 0) return s;
    }
    m->used_graph = 1;
  }
  bool stopped = false;
  while (done < units && !stopped) {
    int chunk = units - done;
    if (stop != STOP_NEVER && chunk > 32) chunk = 32;
    for (int i = 0; i < chunk; ++i) {
      if (m->used_graph) {
        const auto& g = m->graphs[key];
        SB_CHECK_CUDA(cudaGraphLaunch(g.first, st));
        count_launch(g.second);
      } else {
        SB_PROPAGATE(gen_unit(m, B, beams, proc, kind, st));
      }
    }
    done += chunk;
    if (stop != STOP_NEVER && done < units) {
      SB_PROPAGATE(gen_state_read(m, st));
      const int* g = m->gstate_host;
      stopped = stop == STOP_ALL_FINISHED ? g[GS_VALID] < g[GS_STEP] : g[GS_ALL_DONE] != 0;
    }
  }
  *done_out = done;
  return 0;
}

// B prompts, n = num_return_sequences rows each (R = B * n, prompt-major): the prompts are prefilled once, row r reads
// prompt r / n's K/V through the lineage table and samples from Philox row r
static int llama_generate(seedb200_llama* m, const int64_t* prompt_ids, int B, int n, int S, int max_new,
                          const seedb200_sample_params* sp, int64_t eos, int64_t pad, int use_graph,
                          int64_t* tokens_out, int* n_generated_host, const seedb200_logits_params* lp,
                          seedb200_gen_outputs* outputs, cudaStream_t st) {
  const seedb200_llama_config& c = m->cfg;
  const int R = B * n;
  GenParams gp;
  gp.sp = *sp; gp.eos = eos; gp.pad = pad;
  gp.proc = logits_proc(lp, eos, S);
  gp.scores = outputs ? static_cast<__half*>(outputs->scores) : nullptr;
  gp.scores_pitch = outputs ? outputs->scores_pitch : 0;
  gp.scores_step = (long long)R * gp.scores_pitch;
  const int proc = logits_history_active(gp.proc) ? 1 : 0;
  SB_PROPAGATE(gen_begin(m, prompt_ids, B, S, gp, st, n));
  if (n > 1) {
    const long long blocks = ((long long)R * c.max_seq + 255) / 256;
    sample_lineage_kernel<<<blocks < 1024 ? (int)blocks : 1024, 256, 0, st>>>(m->beam.slot, R, n, S, c.max_seq);
    SB_LAUNCH_CHECK();
  }
  // prefill: cache rows [0, S), logits of the last position only (what the sampler needs)
  SB_PROPAGATE(llama_forward(m, prompt_ids, nullptr, nullptr, B, S, 0, 1, m->glogits, (int64_t)n * m->vpad, st));
  SB_PROPAGATE(gen_spread_logits(m, B, n, st));
  if (proc) SB_PROPAGATE(gen_process(m, R, 0, 0, st));
  // token 0 comes from the prefill logits: the step counter advances, the cache length does not
  SB_PROPAGATE(sample(m->glogits, m->vpad, R, c.vocab, nullptr, m->gparams, 0, m->gstate, /*advance_cache=*/0, m->gtok,
                      m->gout, c.max_seq, m->gfinished, st));
  int done = 0;
  SB_PROPAGATE(gen_run_units(m, R, 0, proc, n > 1 ? UNIT_SHARED : UNIT_PLAIN, max_new - 1, use_graph,
                             eos >= 0 ? STOP_ALL_FINISHED : STOP_NEVER, st, &done));
  int n_valid = 0;
  SB_PROPAGATE(gen_end(m, R, S, max_new, eos, done + 1, tokens_out, &n_valid, st));
  if (n_generated_host != nullptr) *n_generated_host = n_valid;
  if (outputs != nullptr) outputs->n_steps_out = n_valid;
  m->gen_cache_len = n > 1 ? 0 : S + done;   // tokens whose K/V are in the cache; with n > 1 the rows hold lineages
  return 0;
}

// beam search: prefill at B rows, candidates + scorer from the prefill logits (every beam reads its sequence's row),
// then max_new - 1 units of (forward of G * k rows through the lineage table -> candidates -> scorer), then finalize.
// G = B * n sequences (num_return_sequences = n, beam sampling only): sequence g searches prompt g / n on its own.
static int llama_beam_generate(seedb200_llama* m, const int64_t* prompt_ids, int B, int n, int S, int max_new,
                               const seedb200_beam_params* p, int64_t eos, int64_t pad, int use_graph,
                               int64_t* tokens_out, int* n_out_host, float* best_scores,
                               const seedb200_logits_params* lp, seedb200_gen_outputs* outputs, cudaStream_t st) {
  const seedb200_llama_config& c = m->cfg;
  const int k = p->num_beams, G = B * n;
  BeamParams bp = beam_params(*p, eos, pad, S, max_new, G, lp, n);
  if (outputs != nullptr) {
    bp.scores = static_cast<__half*>(outputs->scores);
    bp.scores_pitch = outputs->scores_pitch;
    bp.scores_step = (long long)G * k * outputs->scores_pitch;
    bp.beam_indices = reinterpret_cast<long long*>(outputs->beam_indices);
    bp.bi_ld = S + max_new;
  }
  const bool warp = outputs != nullptr && bp.do_sample;   // beam sampling's scores: one more launch per step
  if (bp.processed && m->beam.tok == nullptr)
    SB_PROPAGATE(llama_alloc(m->row_owned, &m->beam.tok, (size_t)c.max_batch * c.max_seq));
  SB_PROPAGATE(beam_init(m->beam, bp, prompt_ids, st));
  SB_PROPAGATE(llama_forward(m, prompt_ids, nullptr, nullptr, B, S, 0, 1, m->glogits, (int64_t)n * m->vpad, st));
  SB_PROPAGATE(gen_spread_logits(m, B, n, st));
  if (bp.processed) SB_PROPAGATE(gen_process(m, G, k, 0, st));
  SB_PROPAGATE(beam_select(m->glogits, m->vpad, 0, G, k, c.vocab, m->beam.beam_scores, nullptr, m->beam.params, 0,
                           m->gstate, m->beam.row_stats, m->beam.cand_score,
                           m->beam.cand_idx, st, warp));
  SB_PROPAGATE(beam_score(m->beam, G, k, c.vocab, /*advance_cache=*/0, st));
  int done = 0;
  SB_PROPAGATE(gen_run_units(m, G, k, bp.processed, warp ? UNIT_BEAM_WARP : UNIT_PLAIN, max_new - 1, use_graph,
                             eos >= 0 ? STOP_BEAMS_DONE : STOP_NEVER, st, &done));
  SB_PROPAGATE(beam_finalize(m->beam, G, tokens_out, max_new, best_scores, st));
  int n_out = 0;
  SB_CHECK_CUDA(cudaMemcpyAsync(&n_out, m->beam.n_out, sizeof(int), cudaMemcpyDeviceToHost, st));
  SB_CHECK_CUDA(cudaStreamSynchronize(st));
  if (n_out_host != nullptr) *n_out_host = n_out;
  if (outputs != nullptr) {   // transformers' process() calls: through the step every search became done, else all
    SB_PROPAGATE(gen_state_read(m, st));
    outputs->n_steps_out = m->gstate_host[GS_VALID] != 0 ? m->gstate_host[GS_VALID] : done + 1;
  }
  m->gen_cache_len = 0;            // the cache rows now hold beam lineages, not B plain sequences
  return 0;
}

// contrastive search: prefill at B rows (its logits and every prompt row's final hidden state), the normalised prompt
// into the context, then max_new units of (processors -> candidates -> forward of B * k rows -> rank + select)
static int llama_contrastive_generate(seedb200_llama* m, const int64_t* prompt_ids, int B, int S, int max_new,
                                      const seedb200_contrastive_params* cp, int64_t eos, int64_t pad, int use_graph,
                                      int64_t* tokens_out, int* n_generated_host, const seedb200_logits_params* lp,
                                      seedb200_gen_outputs* outputs, cudaStream_t st) {
  const seedb200_llama_config& c = m->cfg;
  const ContrastParams p = contrast_params(*cp);
  if (m->c_tickets == nullptr) {   // allocated last: a failed first call allocates again
    const size_t R = (size_t)c.max_batch;
    SB_PROPAGATE(llama_alloc(m->row_owned, &m->c_ctx, R * c.max_seq * c.hidden));
    SB_PROPAGATE(llama_alloc(m->row_owned, &m->c_logits, R * m->vpad));
    SB_PROPAGATE(llama_alloc(m->row_owned, &m->c_probs, R));
    SB_PROPAGATE(llama_alloc(m->row_owned, &m->c_part, R * CONTRAST_MAX_CTAS * CONTRAST_MAX_K));
    SB_PROPAGATE(llama_alloc(m->row_owned, &m->c_tickets, R));
    SB_CHECK_CUDA(cudaMemsetAsync(m->c_tickets, 0, R * sizeof(int), st));   // left zero by every launch
  }
  GenParams gp;
  memset(&gp, 0, sizeof(gp));
  gp.eos = eos; gp.pad = pad;
  gp.proc = logits_proc(lp, eos, S);
  gp.proc.lp.top_k = 0;                           // the candidate count, not a warper
  if (outputs != nullptr) {
    gp.scores = static_cast<__half*>(outputs->scores);
    gp.scores_pitch = outputs->scores_pitch;
    gp.scores_step = (long long)B * outputs->scores_pitch;
  }
  const int proc = logits_history_active(gp.proc) ? 1 : 0;
  SB_PROPAGATE(gen_begin(m, prompt_ids, B, S, gp, st));
  SB_PROPAGATE(llama_forward(m, prompt_ids, nullptr, nullptr, B, S, 0, 1, m->c_logits, m->vpad, st));
  SB_PROPAGATE(contrastive_context_init(m->hn, B, S, c.hidden, m->c_ctx, (int64_t)c.max_seq * c.hidden, m->beam.slot,
                                        p.k, c.max_seq, p, m->c_params, st));
  int done = 0;
  SB_PROPAGATE(gen_run_units(m, B, p.k, proc, UNIT_CONTRASTIVE, max_new, use_graph,
                             eos >= 0 ? STOP_ALL_FINISHED : STOP_NEVER, st, &done));
  int n_valid = 0;
  SB_PROPAGATE(gen_end(m, B, S, max_new, eos, done, tokens_out, &n_valid, st));
  if (n_generated_host != nullptr) *n_generated_host = n_valid;
  if (outputs != nullptr) outputs->n_steps_out = n_valid;
  m->gen_cache_len = 0;            // the cache rows now hold candidate lineages, not B plain sequences
  return 0;
}

static void llama_drop_graphs(seedb200_llama* m) {
  for (auto& g : m->graphs) cudaGraphExecDestroy(g.second.first);
  m->graphs.clear();
}

// every quantised (int8 or 4-bit) linear must hold its weights before the model runs
static int llama_linears_ready(const seedb200_llama* m) {
  for (size_t i = 0; i < m->q_loaded.size(); ++i)
    if (!m->q_loaded[i]) {
      if (m->fmt == W_4BIT)
        set_error("llama: 4-bit weight 'model.layers.%d.%s.weight' has not been loaded (seedb200_llama_4bit_load_weight)",
                  (int)(i / 7), kLinear[i % 7].name);
      else
        set_error("llama: int8 weight 'model.layers.%d.%s.weight' was neither given to create_int8 nor loaded",
                  (int)(i / 7), kLinear[i % 7].name);
      return SEEDB200_ERR_INVALID;
    }
  return 0;
}

// the checks the three generation entry points share, reported under `who`
static int gen_args_check(const char* who, const seedb200_llama* m, const int64_t* prompt_ids, const void* params,
                          int S, int max_new) {
  SB_REQUIRE(m && prompt_ids && params, "%s: null argument", who);
  SB_REQUIRE(S >= 1 && max_new >= 1 && S + max_new <= m->cfg.max_seq, "%s: prompt %d + %d new tokens exceeds max_seq %d",
             who, S, max_new, m->cfg.max_seq);
  return 0;
}

// seedb200_gen_outputs (NULL passes): a scores buffer of 16-byte aligned rows a multiple of 8 halves apart;
// beam_indices only for beam search (optional there).  The pitch is checked against the vocabulary once the handle
// has been.
static int gen_outputs_check(const char* who, const seedb200_gen_outputs* o, bool beams = false) {
  if (o == nullptr) return 0;
  SB_REQUIRE(o->scores != nullptr && (uintptr_t)o->scores % 16 == 0,
             "%s: outputs.scores must be a 16-byte aligned device pointer", who);
  SB_REQUIRE(o->scores_pitch > 0 && o->scores_pitch % 8 == 0,
             "%s: outputs.scores_pitch %lld must be a positive multiple of 8", who, (long long)o->scores_pitch);
  SB_REQUIRE(beams || o->beam_indices == nullptr, "%s: outputs.beam_indices is written by beam search only", who);
  return 0;
}

// seedb200_llama_{int8,4bit}_load_weight: quantise the fp16 decoder linear `name` ([N, K], rows ldw apart) into its
// rows of the handle's fused linear
static int load_quantised(seedb200_llama* m, const char* who, const char* name, const void* W, int64_t ldw,
                          cudaStream_t st) {
  int layer = -1, i = -1;
  SB_REQUIRE(linear_of(name, ".weight", &layer, &i) && layer >= 0 && layer < (int)m->layers.size(),
             "%s: '%s' is not a decoder linear of this model", who, name);
  const Fused F = fused(m, kLinear[i].g);
  const int N = F.N / F.nsub, K = F.K, grp = F.grp, gstride = F.grp * F.nsub, off = kLinear[i].sub * F.grp;
  if (ldw == 0) ldw = K;
  SB_REQUIRE(ldw >= K, "%s: ldw %lld below K %lld", who, (long long)ldw, (long long)K);
  void* w = const_cast<void*>(m->layers[layer].lin[kLinear[i].g].w);
  float* s = const_cast<float*>(m->layers[layer].lin[kLinear[i].g].s);
  DeviceGuard guard(m->device);
  if (m->fmt == W_INT8)
    SB_PROPAGATE(int8_quantize_weight_rows(W, ldw, N, K, w, s, grp, gstride, off, st));
  else
    SB_PROPAGATE(quantize_4bit_rows(W, ldw, N, K, m->q4type, w, s, grp, gstride, off, st));
  m->q_loaded[(size_t)layer * 7 + i] = 1;
  return 0;
}

}  // namespace sb

extern "C" {

// threshold: int8 only; q4type: 4-bit only (-1 otherwise)
static int llama_create(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights,
                        sb::WeightFormat fmt, float threshold, int q4type, seedb200_llama** out) {
  if (!cfg || !weights || !out) {
    sb::set_error("llama_create: null argument");
    return SEEDB200_ERR_INVALID;
  }
  SB_REQUIRE(cfg->head_dim == 128, "llama_create: head_dim must be 128 (got %d)", cfg->head_dim);
  SB_REQUIRE(cfg->hidden == cfg->heads * cfg->head_dim, "llama_create: hidden != heads * head_dim");
  SB_REQUIRE(cfg->ffn % 128 == 0, "llama_create: ffn %d must be a multiple of 128", cfg->ffn);
  SB_REQUIRE(cfg->hidden % 8 == 0 && cfg->layers >= 0 && cfg->vocab > 0, "llama_create: bad dims");
  SB_REQUIRE(cfg->max_batch >= 1 && cfg->max_seq >= 1, "llama_create: bad cache size");
  seedb200_llama* m = new seedb200_llama();
  m->cfg = *cfg;
  if (m->cfg.rope_base <= 0.0f) m->cfg.rope_base = 10000.0f;
  if (m->cfg.rms_eps <= 0.0f) m->cfg.rms_eps = 1e-6f;
  m->last_T = 0;
  m->device = sb::cur_device();
  m->gstate_host = nullptr;
  m->gstream = nullptr;
  m->used_graph = -1;
  m->gen_cache_len = 0;
  memset(&m->beam, 0, sizeof(m->beam));
  m->fmt = fmt;
  m->threshold = threshold;
  m->q4type = q4type;
  m->lora_r = 0;
  m->lora_s = 0.0f;
  memset(m->lora_mask, 0, sizeof(m->lora_mask));
  m->lora_mem = nullptr;
  for (int i = 0; i < n_weights; ++i) m->w[std::string(weights[i].name)] = weights[i];
  int s = sb::llama_build(m);
  if (s != 0) {
    seedb200_llama_destroy(m);
    return s;
  }
  m->w.clear();
  *out = m;
  return 0;
}

int seedb200_llama_create(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights,
                          seedb200_llama** out) {
  return llama_create(cfg, weights, n_weights, sb::W_F16, 0.0f, -1, out);
}

int seedb200_llama_create_int8(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights,
                               float threshold, seedb200_llama** out) {
  SB_REQUIRE(threshold > 0.0f, "llama_create_int8: threshold must be > 0 (got %g)", (double)threshold);
  SB_REQUIRE(cfg == nullptr || cfg->hidden % 16 == 0, "llama_create_int8: hidden must be a multiple of 16");
  return llama_create(cfg, weights, n_weights, sb::W_INT8, threshold, -1, out);
}

int seedb200_llama_create_4bit(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights,
                               int quant_type, seedb200_llama** out) {
  SB_REQUIRE(quant_type == SEEDB200_Q4_FP4 || quant_type == SEEDB200_Q4_NF4,
             "llama_create_4bit: quant_type %d is neither FP4 (0) nor NF4 (1)", quant_type);
  SB_REQUIRE(cfg == nullptr || (cfg->hidden % 64 == 0 && cfg->ffn % 64 == 0),
             "llama_create_4bit: hidden %d and ffn %d must be multiples of the 4-bit blocksize 64",
             cfg ? cfg->hidden : 0, cfg ? cfg->ffn : 0);
  return llama_create(cfg, weights, n_weights, sb::W_4BIT, 0.0f, quant_type, out);
}

int seedb200_llama_int8_load_weight(seedb200_llama* llm, const char* name, const void* W, int64_t ldw, void* stream) {
  SB_REQUIRE(llm && name && W, "llama_int8_load_weight: null argument");
  SB_REQUIRE(llm->fmt == sb::W_INT8, "llama_int8_load_weight: the handle was not made by seedb200_llama_create_int8");
  return sb::load_quantised(llm, "llama_int8_load_weight", name, W, ldw, static_cast<cudaStream_t>(stream));
}

int seedb200_llama_4bit_load_weight(seedb200_llama* llm, const char* name, const void* W, int64_t ldw, void* stream) {
  SB_REQUIRE(llm && name && W, "llama_4bit_load_weight: null argument");
  SB_REQUIRE(llm->fmt == sb::W_4BIT, "llama_4bit_load_weight: the handle was not made by seedb200_llama_create_4bit");
  return sb::load_quantised(llm, "llama_4bit_load_weight", name, W, ldw, static_cast<cudaStream_t>(stream));
}

void seedb200_llama_destroy(seedb200_llama* llm) {
  if (!llm) return;
  sb::llama_drop_graphs(llm);
  if (llm->gstate_host) cudaFreeHost(llm->gstate_host);
  if (llm->gstream) cudaStreamDestroy(llm->gstream);
  sb::llama_free_rows(llm);
  if (llm->lora_mem) cudaFree(llm->lora_mem);
  for (void* p : llm->owned) cudaFree(p);
  delete llm;
}

int seedb200_llama_forward_ld(seedb200_llama* llm, const int64_t* input_ids, const void* inputs_embeds,
                              const int64_t* position_ids, int B, int S, int past_len, int logits_mode,
                              void* logits_out, int64_t logits_ld, void* stream) {
  SB_REQUIRE(llm != nullptr, "llama_forward: null handle");
  SB_REQUIRE((input_ids != nullptr) != (inputs_embeds != nullptr),
             "llama_forward: specify exactly one of input_ids / inputs_embeds (llama_xformer.py:516-523)");
  SB_REQUIRE(B >= 1 && B <= llm->cfg.max_batch, "llama_forward: batch %d outside [1,%d]", B, llm->cfg.max_batch);
  SB_REQUIRE(S >= 1 && past_len >= 0 && past_len + S <= llm->cfg.max_seq,
             "llama_forward: past_len %d + S %d exceeds max_seq %d", past_len, S, llm->cfg.max_seq);
  SB_REQUIRE(logits_mode == 0 || logits_mode == 1, "llama_forward: logits_mode must be 0 or 1");
  SB_REQUIRE(logits_out == nullptr || logits_ld >= llm->cfg.vocab, "llama_forward: logits_ld %lld < vocab %d",
             (long long)logits_ld, llm->cfg.vocab);
  SB_PROPAGATE(sb::llama_linears_ready(llm));
  sb::DeviceGuard guard(llm->device);
  return sb::llama_forward(llm, input_ids, inputs_embeds, position_ids, B, S, past_len, logits_mode, logits_out,
                           logits_ld, static_cast<cudaStream_t>(stream));
}

int seedb200_llama_forward(seedb200_llama* llm, const int64_t* input_ids, const void* inputs_embeds,
                           const int64_t* position_ids, int B, int S, int past_len, int logits_mode, void* logits_out,
                           void* stream) {
  return seedb200_llama_forward_ld(llm, input_ids, inputs_embeds, position_ids, B, S, past_len, logits_mode, logits_out,
                                   llm ? llm->cfg.vocab : 0, stream);
}

int seedb200_llama_generate(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                            const seedb200_sample_params* sp, int64_t eos_id, int64_t pad_id, int use_graph,
                            int64_t* tokens_out, int* n_generated_host, void* stream) {
  return seedb200_llama_generate_n_processed(llm, prompt_ids, B, S, max_new_tokens, 1, sp, eos_id, pad_id, use_graph,
                                             tokens_out, n_generated_host, stream, nullptr);
}

int seedb200_llama_generate_processed(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                      int max_new_tokens, const seedb200_sample_params* sp, int64_t eos_id,
                                      int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host,
                                      void* stream, const seedb200_logits_params* lp) {
  return seedb200_llama_generate_n_processed(llm, prompt_ids, B, S, max_new_tokens, 1, sp, eos_id, pad_id, use_graph,
                                             tokens_out, n_generated_host, stream, lp);
}

int seedb200_llama_generate_n(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                              int num_return_sequences, const seedb200_sample_params* sp, int64_t eos_id,
                              int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host, void* stream) {
  return seedb200_llama_generate_n_processed(llm, prompt_ids, B, S, max_new_tokens, num_return_sequences, sp, eos_id,
                                             pad_id, use_graph, tokens_out, n_generated_host, stream, nullptr);
}

int seedb200_llama_generate_n_processed(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                        int max_new_tokens, int num_return_sequences,
                                        const seedb200_sample_params* sp, int64_t eos_id, int64_t pad_id,
                                        int use_graph, int64_t* tokens_out, int* n_generated_host, void* stream,
                                        const seedb200_logits_params* lp) {
  return seedb200_llama_generate_ex(llm, prompt_ids, B, S, max_new_tokens, num_return_sequences, sp, eos_id, pad_id,
                                    use_graph, tokens_out, n_generated_host, stream, lp, nullptr);
}

int seedb200_llama_generate_ex(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                               int num_return_sequences, const seedb200_sample_params* sp, int64_t eos_id,
                               int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host, void* stream,
                               const seedb200_logits_params* lp, seedb200_gen_outputs* outputs) {
  const int n = num_return_sequences;
  SB_REQUIRE(n >= 1, "llama_generate: num_return_sequences %d < 1", n);
  SB_PROPAGATE(sb::gen_outputs_check("llama_generate", outputs));
  SB_PROPAGATE(sb::logits_params_check("llama_generate", lp));
  SB_PROPAGATE(sb::gen_args_check("llama_generate", llm, prompt_ids, sp, S, max_new_tokens));
  SB_REQUIRE(B >= 1 && (int64_t)B * n <= llm->cfg.max_batch,
             "llama_generate: batch %d x %d sequences exceeds max_batch %d (seedb200_llama_reserve_rows)", B, n,
             llm->cfg.max_batch);
  SB_REQUIRE((int64_t)B * n <= 1024, "llama_generate: batch %d x %d sequences above 1024 rows", B, n);
  SB_REQUIRE(!sp->do_sample || (sp->temperature > 0.0f && sp->top_p > 0.0f), "llama_generate: temperature and top_p must be > 0");
  SB_REQUIRE(outputs == nullptr || outputs->scores_pitch >= llm->cfg.vocab,
             "llama_generate: outputs.scores_pitch %lld below the vocabulary %d", (long long)outputs->scores_pitch,
             llm->cfg.vocab);
  SB_PROPAGATE(sb::llama_linears_ready(llm));
  sb::DeviceGuard guard(llm->device);
  return sb::llama_generate(llm, prompt_ids, B, n, S, max_new_tokens, sp, eos_id, pad_id, use_graph, tokens_out,
                            n_generated_host, lp, outputs, static_cast<cudaStream_t>(stream));
}

int seedb200_llama_generate_used_graph(seedb200_llama* llm) { return llm ? llm->used_graph : -1; }

int seedb200_llama_beam_generate(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                                 const seedb200_beam_params* bp, int64_t eos_id, int64_t pad_id, int use_graph,
                                 int64_t* tokens_out, int* n_out_host, float* best_scores_out, void* stream) {
  return seedb200_llama_beam_generate_n_processed(llm, prompt_ids, B, S, max_new_tokens, 1, bp, eos_id, pad_id,
                                                  use_graph, tokens_out, n_out_host, best_scores_out, stream, nullptr);
}

int seedb200_llama_beam_generate_processed(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                           int max_new_tokens, const seedb200_beam_params* bp, int64_t eos_id,
                                           int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_out_host,
                                           float* best_scores_out, void* stream, const seedb200_logits_params* lp) {
  return seedb200_llama_beam_generate_n_processed(llm, prompt_ids, B, S, max_new_tokens, 1, bp, eos_id, pad_id,
                                                  use_graph, tokens_out, n_out_host, best_scores_out, stream, lp);
}

int seedb200_llama_beam_generate_n(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                                   int num_return_sequences, const seedb200_beam_params* bp, int64_t eos_id,
                                   int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_out_host,
                                   float* best_scores_out, void* stream) {
  return seedb200_llama_beam_generate_n_processed(llm, prompt_ids, B, S, max_new_tokens, num_return_sequences, bp,
                                                  eos_id, pad_id, use_graph, tokens_out, n_out_host, best_scores_out,
                                                  stream, nullptr);
}

int seedb200_llama_beam_generate_n_processed(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                             int max_new_tokens, int num_return_sequences,
                                             const seedb200_beam_params* bp, int64_t eos_id, int64_t pad_id,
                                             int use_graph, int64_t* tokens_out, int* n_out_host,
                                             float* best_scores_out, void* stream, const seedb200_logits_params* lp) {
  return seedb200_llama_beam_generate_ex(llm, prompt_ids, B, S, max_new_tokens, num_return_sequences, bp, eos_id,
                                         pad_id, use_graph, tokens_out, n_out_host, best_scores_out, stream, lp,
                                         nullptr);
}

int seedb200_llama_beam_generate_ex(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                                    int num_return_sequences, const seedb200_beam_params* bp, int64_t eos_id,
                                    int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_out_host,
                                    float* best_scores_out, void* stream, const seedb200_logits_params* lp,
                                    seedb200_gen_outputs* outputs) {
  const int n = num_return_sequences;
  SB_REQUIRE(n >= 1, "llama_beam_generate: num_return_sequences %d < 1", n);
  SB_PROPAGATE(sb::gen_outputs_check("llama_beam_generate", outputs, /*beams=*/true));
  SB_REQUIRE(n == 1 || bp == nullptr || bp->do_sample,
             "llama_beam_generate: num_return_sequences %d > 1 needs beam sampling (do_sample)", n);
  SB_PROPAGATE(sb::logits_params_check("llama_beam_generate", lp));
  SB_PROPAGATE(sb::gen_args_check("llama_beam_generate", llm, prompt_ids, bp, S, max_new_tokens));
  SB_REQUIRE(tokens_out != nullptr, "llama_beam_generate: null argument");
  SB_REQUIRE(bp->num_beams >= 1 && bp->num_beams <= sb::BEAM_MAX, "llama_beam_generate: num_beams %d outside [1,%d]",
             bp->num_beams, sb::BEAM_MAX);
  SB_REQUIRE(B >= 1 && (int64_t)B * n * bp->num_beams <= llm->cfg.max_batch,
             "llama_beam_generate: batch %d x %d sequences x %d beams exceeds max_batch %d (seedb200_llama_reserve_rows)",
             B, n, bp->num_beams, llm->cfg.max_batch);
  SB_REQUIRE((int64_t)B * n <= 1024, "llama_beam_generate: batch %d x %d sequences above 1024", B, n);
  SB_REQUIRE(!bp->do_sample || (bp->temperature > 0.0f && bp->top_p > 0.0f),
             "llama_beam_generate: temperature and top_p must be > 0 when sampling");
  SB_REQUIRE(bp->early_stopping >= 0 && bp->early_stopping <= 2, "llama_beam_generate: early_stopping %d not in {0,1,2}",
             bp->early_stopping);
  SB_REQUIRE(eos_id < llm->cfg.vocab, "llama_beam_generate: eos_id %lld outside the vocabulary", (long long)eos_id);
  SB_REQUIRE(outputs == nullptr || outputs->scores_pitch >= llm->cfg.vocab,
             "llama_beam_generate: outputs.scores_pitch %lld below the vocabulary %d", (long long)outputs->scores_pitch,
             llm->cfg.vocab);
  SB_PROPAGATE(sb::llama_linears_ready(llm));
  sb::DeviceGuard guard(llm->device);
  return sb::llama_beam_generate(llm, prompt_ids, B, n, S, max_new_tokens, bp, eos_id, pad_id, use_graph, tokens_out,
                                 n_out_host, best_scores_out, lp, outputs, static_cast<cudaStream_t>(stream));
}

int seedb200_llama_contrastive_generate(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                        int max_new_tokens, const seedb200_contrastive_params* cp, int64_t eos_id,
                                        int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host,
                                        void* stream, const seedb200_logits_params* lp) {
  return seedb200_llama_contrastive_generate_ex(llm, prompt_ids, B, S, max_new_tokens, cp, eos_id, pad_id, use_graph,
                                                tokens_out, n_generated_host, stream, lp, nullptr);
}

int seedb200_llama_contrastive_generate_ex(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S,
                                           int max_new_tokens, const seedb200_contrastive_params* cp, int64_t eos_id,
                                           int64_t pad_id, int use_graph, int64_t* tokens_out, int* n_generated_host,
                                           void* stream, const seedb200_logits_params* lp,
                                           seedb200_gen_outputs* outputs) {
  SB_PROPAGATE(sb::gen_outputs_check("llama_contrastive_generate", outputs));
  SB_PROPAGATE(sb::contrastive_params_check("llama_contrastive_generate", cp));
  SB_PROPAGATE(sb::logits_params_check("llama_contrastive_generate", lp));
  SB_PROPAGATE(sb::gen_args_check("llama_contrastive_generate", llm, prompt_ids, cp, S, max_new_tokens));
  SB_REQUIRE(B >= 1 && B <= 1024 && (int64_t)B * cp->top_k <= llm->cfg.max_batch,
             "llama_contrastive_generate: batch %d x top_k %d exceeds max_batch %d (seedb200_llama_reserve_rows)", B,
             cp->top_k, llm->cfg.max_batch);
  SB_REQUIRE(eos_id < llm->cfg.vocab, "llama_contrastive_generate: eos_id %lld outside the vocabulary",
             (long long)eos_id);
  SB_REQUIRE(llm->cfg.vocab >= sb::CONTRAST_MAX_K, "llama_contrastive_generate: vocabulary below %d",
             sb::CONTRAST_MAX_K);
  SB_REQUIRE(outputs == nullptr || outputs->scores_pitch >= llm->cfg.vocab,
             "llama_contrastive_generate: outputs.scores_pitch %lld below the vocabulary %d",
             (long long)outputs->scores_pitch, llm->cfg.vocab);
  SB_REQUIRE((size_t)cp->top_k * llm->cfg.hidden * 2 <= 200 * 1024,
             "llama_contrastive_generate: top_k %d x hidden %d exceed the rank kernel's shared memory", cp->top_k,
             llm->cfg.hidden);
  SB_PROPAGATE(sb::llama_linears_ready(llm));
  sb::DeviceGuard guard(llm->device);
  return sb::llama_contrastive_generate(llm, prompt_ids, B, S, max_new_tokens, cp, eos_id, pad_id, use_graph,
                                        tokens_out, n_generated_host, lp, outputs, static_cast<cudaStream_t>(stream));
}

int seedb200_llama_reserve_rows(seedb200_llama* llm, int rows) {
  SB_REQUIRE(llm != nullptr, "llama_reserve_rows: null handle");
  SB_REQUIRE(rows >= 1, "llama_reserve_rows: rows %d < 1", rows);
  if (rows <= llm->cfg.max_batch) return 0;
  sb::DeviceGuard guard(llm->device);
  SB_CHECK_CUDA(cudaDeviceSynchronize());
  sb::llama_drop_graphs(llm);
  sb::llama_free_rows(llm);
  const int old = llm->cfg.max_batch;
  llm->cfg.max_batch = rows;
  int s = sb::llama_alloc_rows(llm, 0);
  if (s != 0) {                      // keep the handle usable at its old size
    std::string err = seedb200_last_error();
    sb::llama_free_rows(llm);
    llm->cfg.max_batch = old;
    if (sb::llama_alloc_rows(llm, 0) != 0) llm->cfg.max_batch = 0;
    sb::set_error("llama_reserve_rows: %s", err.c_str());
    return s;
  }
  SB_CHECK_CUDA(cudaStreamSynchronize(0));
  llm->last_T = 0;
  llm->gen_cache_len = 0;
  return 0;
}

}  // extern "C"

namespace sb {

static void lora_free(seedb200_llama* m) {
  if (m->lora_mem) cudaFree(m->lora_mem);
  m->lora_mem = nullptr;
  m->lora.clear();
  m->lora_r = 0;
  memset(m->lora_mask, 0, sizeof(m->lora_mask));
  for (__half** p : {&m->lora_t, &m->lora_base}) {
    for (size_t i = 0; i < m->row_owned.size(); ++i)
      if (m->row_owned[i] == *p) { m->row_owned.erase(m->row_owned.begin() + i); break; }
    if (*p) cudaFree(*p);
    *p = nullptr;
  }
}

static int tensor_is(const seedb200_tensor& t, int64_t d0, int64_t d1) {
  return t.dtype == SEEDB200_F16 && t.ndim == 2 && t.shape[0] == d0 && t.shape[1] == d1 && t.data != nullptr &&
         (reinterpret_cast<uintptr_t>(t.data) & 15) == 0;
}

}  // namespace sb

extern "C" {

int seedb200_llama_lora_load(seedb200_llama* llm, const seedb200_tensor* tensors, int n, int r, float alpha) {
  SB_REQUIRE(llm && (tensors || n == 0), "llama_lora_load: null argument");
  SB_REQUIRE(llm->fmt != sb::W_INT8, "llama_lora_load: LoRA on an int8 (load_in_8bit) model is not supported");
  SB_REQUIRE(llm->fmt != sb::W_4BIT, "llama_lora_load: LoRA on a 4-bit (load_in_4bit) model is not supported");
  SB_REQUIRE(r >= 1 && r <= sb::LORA_MAX_R, "llama_lora_load: r %d outside [1,%d]", r, sb::LORA_MAX_R);
  SB_REQUIRE(alpha == alpha && alpha > -1e30f && alpha < 1e30f, "llama_lora_load: lora_alpha must be finite");
  const int nl = (int)llm->layers.size();
  std::vector<const seedb200_tensor*> found((size_t)nl * 7 * 2, nullptr);   // [layer][linear][A, B]
  for (int t = 0; t < n; ++t) {
    const seedb200_tensor& x = tensors[t];
    SB_REQUIRE(x.name != nullptr, "llama_lora_load: tensor %d has no name", t);
    int layer = -1, lin = -1, ab = 0;
    while (ab < 2 && !sb::linear_of(x.name, ab ? ".lora_B.weight" : ".lora_A.weight", &layer, &lin)) ++ab;
    SB_REQUIRE(ab < 2, "llama_lora_load: '%s' is not a lora_A / lora_B of a decoder linear", x.name);
    SB_REQUIRE(layer >= 0 && layer < nl, "llama_lora_load: '%s': the model has %d layers", x.name, nl);
    const sb::Fused G = sb::fused(llm, sb::kLinear[lin].g);
    const int64_t N = G.N / G.nsub, K = G.K;
    const bool ok = ab == 0 ? sb::tensor_is(x, r, K) : sb::tensor_is(x, N, r);
    SB_REQUIRE(ok, "llama_lora_load: '%s' must be fp16, 16-byte aligned, [%lld, %lld] (dtype %d, ndim %d)", x.name,
               (long long)(ab == 0 ? r : N), (long long)(ab == 0 ? K : r), x.dtype, x.ndim);
    const seedb200_tensor*& slot = found[((size_t)layer * 7 + lin) * 2 + ab];
    SB_REQUIRE(slot == nullptr, "llama_lora_load: '%s' given twice", x.name);
    slot = &x;
  }
  int targets = -1;   // bit i: linear i carries an adapter (the same in every layer)
  for (int l = 0; l < nl; ++l) {
    int here = 0;
    for (int i = 0; i < 7; ++i) {
      const bool a = found[((size_t)l * 7 + i) * 2] != nullptr, b = found[((size_t)l * 7 + i) * 2 + 1] != nullptr;
      SB_REQUIRE(a == b, "llama_lora_load: model.layers.%d.%s has lora_%c without lora_%c", l, sb::kLinear[i].name,
                 a ? 'A' : 'B', a ? 'B' : 'A');
      if (a) here |= 1 << i;
    }
    SB_REQUIRE(targets < 0 || here == targets, "llama_lora_load: layer %d has a different set of target modules", l);
    targets = here;
  }
  SB_REQUIRE(targets > 0, "llama_lora_load: no lora_A / lora_B tensors");
  sb::DeviceGuard guard(llm->device);
  SB_CHECK_CUDA(cudaDeviceSynchronize());
  sb::llama_drop_graphs(llm);
  sb::lora_free(llm);
  size_t per_layer = 0;
  for (int g = 0; g < 4; ++g) {
    const sb::Fused G = sb::fused(llm, g);
    per_layer += (size_t)G.nsub * r * G.K + (size_t)G.N * r;
  }
  SB_CHECK_CUDA(cudaMalloc(&llm->lora_mem, per_layer * nl * 2 + 256));
  cudaStream_t st = 0;
  SB_CHECK_CUDA(cudaMemsetAsync(llm->lora_mem, 0, per_layer * nl * 2, st));
  llm->lora.resize(nl);
  __half* p = static_cast<__half*>(llm->lora_mem);
  for (int l = 0; l < nl; ++l)
    for (int g = 0; g < 4; ++g) {
      const sb::Fused G = sb::fused(llm, g);
      llm->lora[l].A[g] = p; p += (size_t)G.nsub * r * G.K;
      llm->lora[l].B[g] = p; p += (size_t)G.N * r;
    }
  for (int l = 0; l < nl; ++l)
    for (int i = 0; i < 7; ++i) {
      if (!((targets >> i) & 1)) continue;
      const int g = sb::kLinear[i].g, sub = sb::kLinear[i].sub;
      const sb::Fused G = sb::fused(llm, g);
      const seedb200_tensor* A = found[((size_t)l * 7 + i) * 2];
      const seedb200_tensor* B = found[((size_t)l * 7 + i) * 2 + 1];
      __half* a_dst = const_cast<__half*>(llm->lora[l].A[g]) + (size_t)sub * r * G.K;
      SB_CHECK_CUDA(cudaMemcpyAsync(a_dst, A->data, (size_t)r * G.K * 2, cudaMemcpyDeviceToDevice, st));
      SB_PROPAGATE(sb::place_rows(const_cast<__half*>(llm->lora[l].B[g]), B->data, (size_t)r * 2, G, sub, st));
      llm->lora_mask[g] |= 1u << sub;
    }
  llm->lora_r = r;
  llm->lora_s = alpha / (float)r;
  const size_t T = (size_t)llm->cfg.max_batch * llm->cfg.max_seq;
  const size_t wide = (size_t)(2 * llm->cfg.ffn > llm->cfg.hidden ? 2 * llm->cfg.ffn : llm->cfg.hidden);
  int s = sb::llama_alloc(llm->row_owned, &llm->lora_t, T * 3 * (size_t)r);
  if (s == 0) s = sb::llama_alloc(llm->row_owned, &llm->lora_base, T * wide);
  if (s != 0) {
    sb::lora_free(llm);
    return s;
  }
  SB_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int seedb200_llama_lora_merge(seedb200_llama* llm) {
  SB_REQUIRE(llm != nullptr, "llama_lora_merge: null handle");
  SB_REQUIRE(llm->lora_r > 0, "llama_lora_merge: no adapter is loaded");
  sb::DeviceGuard guard(llm->device);
  cudaStream_t st = 0;
  SB_CHECK_CUDA(cudaDeviceSynchronize());
  for (int l = 0; l < (int)llm->layers.size(); ++l)
    for (int g = 0; g < 4; ++g) {
      if (llm->lora_mask[g] == 0) continue;
      const sb::Fused G = sb::fused(llm, g);
      const seedb200_lora_operand lo = sb::lora_operand(llm, l, g, nullptr);
      SB_PROPAGATE(sb::lora_merge(const_cast<void*>(llm->layers[l].lin[g].w), llm->lora[l].A[g], lo, G.N, G.K, st));
    }
  SB_CHECK_CUDA(cudaStreamSynchronize(st));
  sb::llama_drop_graphs(llm);
  sb::lora_free(llm);
  return 0;
}

int seedb200_llama_replace_weights(seedb200_llama* llm, const seedb200_tensor* tensors, int n) {
  SB_REQUIRE(llm && (tensors || n == 0), "llama_replace_weights: null argument");
  const int64_t h = llm->cfg.hidden;
  const int nl = (int)llm->layers.size();
  const seedb200_tensor *embed = nullptr, *head = nullptr, *norm = nullptr;
  std::vector<const seedb200_tensor*> ln((size_t)nl * 2, nullptr);
  for (int t = 0; t < n; ++t) {
    const seedb200_tensor& x = tensors[t];
    SB_REQUIRE(x.name != nullptr, "llama_replace_weights: tensor %d has no name", t);
    int l = -1, c = 0;
    const seedb200_tensor** slot = nullptr;
    if (strcmp(x.name, "model.embed_tokens.weight") == 0) slot = &embed;
    else if (strcmp(x.name, "lm_head.weight") == 0) slot = &head;
    else if (strcmp(x.name, "model.norm.weight") == 0) slot = &norm;
    else if (sscanf(x.name, "model.layers.%d%n", &l, &c) == 1 && l >= 0 && l < nl) {
      if (strcmp(x.name + c, ".input_layernorm.weight") == 0) slot = &ln[(size_t)l * 2];
      else if (strcmp(x.name + c, ".post_attention_layernorm.weight") == 0) slot = &ln[(size_t)l * 2 + 1];
    }
    SB_REQUIRE(slot != nullptr, "llama_replace_weights: '%s' is not embed_tokens, lm_head or a norm of this model",
               x.name);
    const bool vec = slot != &embed && slot != &head;
    const bool ok = vec ? (x.dtype == SEEDB200_F16 && x.ndim == 1 && x.shape[0] == h && x.data &&
                           (reinterpret_cast<uintptr_t>(x.data) & 15) == 0)
                        : (x.ndim == 2 && sb::tensor_is(x, x.shape[0], h) && x.shape[0] >= 1 && x.shape[0] < (1LL << 31));
    SB_REQUIRE(ok, "llama_replace_weights: '%s' must be fp16, 16-byte aligned, %s", x.name,
               vec ? "[hidden]" : "[vocab, hidden]");
    *slot = &x;
  }
  const int64_t V = llm->cfg.vocab;
  const int64_t ve = embed ? embed->shape[0] : V, vh = head ? head->shape[0] : V;
  SB_REQUIRE(ve == vh, "llama_replace_weights: embed_tokens has %lld rows and lm_head %lld: a vocabulary change "
             "needs both, with the same size", (long long)ve, (long long)vh);
  sb::DeviceGuard guard(llm->device);
  SB_CHECK_CUDA(cudaDeviceSynchronize());
  sb::llama_drop_graphs(llm);
  if (ve != V) {
    sb::llama_free_rows(llm);
    const int old = llm->cfg.vocab;
    llm->cfg.vocab = (int)ve;
    llm->vpad = (llm->cfg.vocab + 7) / 8 * 8;
    int s = sb::llama_alloc_rows(llm, 0);
    if (s != 0) {                      // keep the handle usable with its old tensors
      std::string err = seedb200_last_error();
      sb::llama_free_rows(llm);
      llm->cfg.vocab = old;
      llm->vpad = (old + 7) / 8 * 8;
      if (sb::llama_alloc_rows(llm, 0) != 0) llm->cfg.max_batch = 0;
      sb::set_error("llama_replace_weights: %s", err.c_str());
      return s;
    }
    SB_CHECK_CUDA(cudaStreamSynchronize(0));
    llm->last_T = 0;
    llm->gen_cache_len = 0;
  }
  if (embed) llm->embed = static_cast<const __half*>(embed->data);
  if (head) llm->lm_head = static_cast<const __half*>(head->data);
  if (norm) llm->norm_w = static_cast<const __half*>(norm->data);
  for (int l = 0; l < nl; ++l) {
    if (ln[(size_t)l * 2]) llm->layers[l].in_ln = static_cast<const __half*>(ln[(size_t)l * 2]->data);
    if (ln[(size_t)l * 2 + 1]) llm->layers[l].post_ln = static_cast<const __half*>(ln[(size_t)l * 2 + 1]->data);
  }
  return 0;
}

int seedb200_llama_kv_ptrs(seedb200_llama* llm, int layer, void** k, void** v) {
  SB_REQUIRE(llm && k && v && layer >= 0 && layer < (int)llm->layers.size(), "llama_kv_ptrs: bad arguments");
  *k = llm->layers[layer].k_cache;
  *v = llm->layers[layer].v_cache;
  return 0;
}

int seedb200_llama_kv_load(seedb200_llama* llm, int layer, const void* k, const void* v, int B, int past_len,
                           void* stream) {
  SB_REQUIRE(llm && k && v && layer >= 0 && layer < (int)llm->layers.size(), "llama_kv_load: bad arguments");
  SB_REQUIRE(B >= 1 && B <= llm->cfg.max_batch && past_len >= 0 && past_len <= llm->cfg.max_seq, "llama_kv_load: bad sizes");
  if (past_len == 0) return 0;
  sb::DeviceGuard guard(llm->device);
  const size_t D = llm->cfg.head_dim, H = llm->cfg.heads;
  const size_t w = (size_t)past_len * D * 2, dp = (size_t)llm->cfg.max_seq * D * 2;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // source [B,H,past,D] contiguous; destination rows of max_seq*D per (b,h); batch stride H*max_seq*D matches
  SB_CHECK_CUDA(cudaMemcpy2DAsync(llm->layers[layer].k_cache, dp, k, w, w, (size_t)B * H, cudaMemcpyDeviceToDevice, st));
  SB_CHECK_CUDA(cudaMemcpy2DAsync(llm->layers[layer].v_cache, dp, v, w, w, (size_t)B * H, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int64_t seedb200_llama_tap(seedb200_llama* llm, int what, void* dst, int64_t max_elems, void* stream) {
  if (!llm || !dst || llm->last_T <= 0 || what != 0) return -1;
  sb::DeviceGuard guard(llm->device);
  int64_t n = (int64_t)llm->last_T * llm->cfg.hidden;
  if (n > max_elems) n = max_elems;
  if (cudaMemcpyAsync(dst, llm->hn, (size_t)n * 2, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)) != cudaSuccess)
    return -1;
  return n;
}

}  // extern "C"
