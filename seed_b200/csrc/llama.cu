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
// Weights named like the HF checkpoint (model.layers.N.self_attn.q_proj.weight ...).  o_proj, down_proj,
// norms, embed_tokens and lm_head are borrowed; q/k/v and gate/up are copied into their fused layouts and
// the originals are not referenced after create.
// int8 mode (seedb200_llama_create_int8, LLM.int8()): the seven decoder linears of every layer arrive as int8 CB plus
// fp32 SCB and are copied into handle-owned fused layouts (q|k|v concatenated, gate|up interleaved in 128-row blocks,
// the scales the same way); lin8() sends them to the int8 GEMV (<= 4 rows) or quantises the activations and runs the
// int8 wgmma GEMM.
#include <string.h>

#include <map>
#include <string>
#include <utility>
#include <vector>

#include "common.cuh"
#include "ops.h"

namespace sb {
struct LlamaLayerW {
  const __half *in_ln, *post_ln, *qkv_w, *o_w, *gu_w, *down_w;
  __half *k_cache, *v_cache;
  // int8 mode: CB [N,K] and SCB [N] of the fused projections
  const int8_t *qkv8, *o8, *gu8, *down8;
  const float *qkv_s, *o_s, *gu_s, *down_s;
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
  int* gstate;                    // {cache length, step, arrive counter, valid steps, any-unfinished flag}
  int* gfinished;                 // [max_batch]
  int64_t* gtok;                  // [max_batch] token fed to the next decode forward
  int64_t* gout;                  // [max_batch, max_seq] generated tokens
  __half* glogits;                // [max_batch, vpad]
  sb::GenParams* gparams;         // sampling parameters + eos/pad, read by the sampler at run time
  int* gstate_host;               // pinned mirror of gstate (early-stop polling)
  cudaStream_t gstream;           // private stream the decode step is captured on (the caller's may be the legacy
                                  // default stream, which cannot be captured); replays go to the caller's stream
  // captured decode units per (batch, beams): beams 0 = the sampler loop; value = (graph, kernels inside one unit)
  std::map<std::pair<int, int>, std::pair<cudaGraphExec_t, int>> graphs;
  sb::BeamState beam;             // beam-search state (rows = batch * beams <= max_batch)
  int used_graph;
  int gen_cache_len;
  // ---- int8 mode ----
  int int8;
  float threshold;
  std::vector<uint8_t> i8_loaded; // [layers][7]: the int8 linear holds its weights
  __half* corr;                   // [max_batch * max_seq, 2 * ffn] outlier correction of the GEMM path
  int8_t* ca;                     // [max_batch * max_seq, max(hidden, ffn)] quantised activations (GEMM path)
  float* sca;                     // [max_batch * max_seq]
  int* olist;                     // [max(hidden, ffn)] outlier columns
  int* ocount;
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

static const char* const kI8Lin[7] = {"self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj",
                                     "mlp.gate_proj", "mlp.up_proj", "mlp.down_proj"};

// Where int8 linear i of layer L lives in the handle's fused buffers: CB rows r of [N,K] go to row
// (r / grp) * gstride + r % grp + off of the fused weight, SCB entries likewise (gate|up: blocks of 128 rows).
struct I8Slot { int8_t* cb; float* scb; int64_t N, K, grp, gstride, off; };
static I8Slot i8_slot(const seedb200_llama* m, int layer, int i) {
  const int64_t h = m->cfg.hidden, ffn = m->cfg.ffn;
  const sb::LlamaLayerW& L = m->layers[layer];
  I8Slot t;
  t.K = i == 6 ? ffn : h;
  t.N = i == 6 ? h : (i >= 4 ? ffn : h);
  t.grp = t.N; t.gstride = 0; t.off = 0;
  if (i < 3) { t.cb = const_cast<int8_t*>(L.qkv8); t.scb = const_cast<float*>(L.qkv_s); t.off = i * h; }
  else if (i == 3) { t.cb = const_cast<int8_t*>(L.o8); t.scb = const_cast<float*>(L.o_s); }
  else if (i < 6) { t.cb = const_cast<int8_t*>(L.gu8); t.scb = const_cast<float*>(L.gu_s); t.grp = 128; t.gstride = 256;
                    t.off = i == 5 ? 128 : 0; }
  else { t.cb = const_cast<int8_t*>(L.down8); t.scb = const_cast<float*>(L.down_s); }
  return t;
}

template <typename T>
static int llama_alloc(seedb200_llama* m, T** p, size_t elems) {
  void* q = nullptr;
  size_t bytes = elems * sizeof(T);
  SB_CHECK_CUDA(cudaMalloc(&q, bytes < 256 ? 256 : bytes));
  m->owned.push_back(q);
  *p = static_cast<T*>(q);
  return 0;
}

template <typename T>
static int llama_alloc_row(seedb200_llama* m, T** p, size_t elems) {
  void* q = nullptr;
  size_t bytes = elems * sizeof(T);
  SB_CHECK_CUDA(cudaMalloc(&q, bytes < 256 ? 256 : bytes));
  m->row_owned.push_back(q);
  *p = static_cast<T*>(q);
  return 0;
}

// every buffer whose size follows max_batch: KV caches, activations, int8 workspaces, generation and beam state
static int llama_alloc_rows(seedb200_llama* m, cudaStream_t st) {
  const seedb200_llama_config& c = m->cfg;
  const int64_t h = c.hidden, ffn = c.ffn;
  const size_t cache_elems = (size_t)c.max_batch * c.heads * c.max_seq * c.head_dim;
  for (LlamaLayerW& L : m->layers) {
    SB_PROPAGATE(llama_alloc_row(m, &L.k_cache, cache_elems));
    SB_PROPAGATE(llama_alloc_row(m, &L.v_cache, cache_elems));
  }
  const size_t T = (size_t)c.max_batch * c.max_seq;
  SB_PROPAGATE(llama_alloc_row(m, &m->x, T * h));
  SB_PROPAGATE(llama_alloc_row(m, &m->nb, T * h));
  SB_PROPAGATE(llama_alloc_row(m, &m->qkv, T * 3 * h));
  SB_PROPAGATE(llama_alloc_row(m, &m->q, T * h));
  SB_PROPAGATE(llama_alloc_row(m, &m->att, T * h));
  SB_PROPAGATE(llama_alloc_row(m, &m->gu, T * ffn));
  SB_PROPAGATE(llama_alloc_row(m, &m->hn, T * h));
  SB_PROPAGATE(llama_alloc_row(m, &m->last, (size_t)c.max_batch * h));
  m->ca = nullptr; m->sca = nullptr; m->corr = nullptr;
  if (m->int8) {
    SB_PROPAGATE(llama_alloc_row(m, &m->corr, T * (size_t)(2 * ffn > 3 * h ? 2 * ffn : 3 * h)));
    SB_PROPAGATE(llama_alloc_row(m, &m->ca, T * (size_t)(ffn > h ? ffn : h)));
    SB_PROPAGATE(llama_alloc_row(m, &m->sca, T));
  }
  SB_PROPAGATE(llama_alloc_row(m, &m->da_ws, (size_t)c.max_batch * c.heads * decode_attention_max_splits(c.max_seq) * (128 + 2)));
  SB_PROPAGATE(llama_alloc_row(m, &m->da_tickets, (size_t)c.max_batch * c.heads));   // zero now, left zero by every launch
  SB_CHECK_CUDA(cudaMemsetAsync(m->da_tickets, 0, (size_t)c.max_batch * c.heads * sizeof(int), st));
  SB_PROPAGATE(llama_alloc_row(m, &m->gfinished, (size_t)c.max_batch));
  SB_PROPAGATE(llama_alloc_row(m, &m->gtok, (size_t)c.max_batch));
  SB_PROPAGATE(llama_alloc_row(m, &m->gout, (size_t)c.max_batch * c.max_seq));
  SB_PROPAGATE(llama_alloc_row(m, &m->glogits, (size_t)c.max_batch * m->vpad));
  BeamState& b = m->beam;
  const size_t R = (size_t)c.max_batch;
  b.tokens = reinterpret_cast<long long*>(m->gtok);
  b.state = m->gstate;
  SB_PROPAGATE(llama_alloc_row(m, &b.beam_scores, R));
  SB_PROPAGATE(llama_alloc_row(m, &b.row_stats, 5 * R));
  SB_PROPAGATE(llama_alloc_row(m, &b.cand_score, 2 * R));
  SB_PROPAGATE(llama_alloc_row(m, &b.cand_idx, 2 * R));
  SB_PROPAGATE(llama_alloc_row(m, &b.slot, R * c.max_seq));
  SB_PROPAGATE(llama_alloc_row(m, &b.slot_tmp, R * c.max_seq));
  SB_PROPAGATE(llama_alloc_row(m, &b.hist_tok, R * c.max_seq));
  SB_PROPAGATE(llama_alloc_row(m, &b.hist_par, R * c.max_seq));
  SB_PROPAGATE(llama_alloc_row(m, &b.hyp_score, R));
  SB_PROPAGATE(llama_alloc_row(m, &b.hyp_len, R));
  SB_PROPAGATE(llama_alloc_row(m, &b.hyp_beam, R));
  SB_PROPAGATE(llama_alloc_row(m, &b.hyp_step, R));
  SB_PROPAGATE(llama_alloc_row(m, &b.hyp_n, R));
  SB_PROPAGATE(llama_alloc_row(m, &b.worst, R));
  SB_PROPAGATE(llama_alloc_row(m, &b.done, R));
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
  SB_PROPAGATE(llama_find(m, "model.embed_tokens.weight", &m->embed, V * h));
  SB_PROPAGATE(llama_find(m, "model.norm.weight", &m->norm_w, h));
  SB_PROPAGATE(llama_find(m, "lm_head.weight", &m->lm_head, V * h));
  if (m->int8) {    // every int8 tensor is checked before anything is allocated
    for (int l = 0; l < c.layers; ++l)
      for (int i = 0; i < 7; ++i) {
        const int64_t N = i == 6 ? h : (i >= 4 ? ffn : h), K = i == 6 ? ffn : h;
        const int8_t* cb;
        const float* scb;
        snprintf(nm, sizeof(nm), "model.layers.%d.%s", l, kI8Lin[i]);
        SB_PROPAGATE(llama_find_i8(m, nm, N, K, &cb, &scb));
      }
    m->i8_loaded.assign((size_t)c.layers * 7, 0);
  }
  m->layers.resize(c.layers);
  for (int l = 0; l < c.layers; ++l) {
    LlamaLayerW& L = m->layers[l];
    auto key = [&](const char* s) { snprintf(nm, sizeof(nm), "model.layers.%d.%s", l, s); return std::string(nm); };
    const __half *wq, *wk, *wv, *wg, *wu;
    SB_PROPAGATE(llama_find(m, key("input_layernorm.weight"), &L.in_ln, h));
    SB_PROPAGATE(llama_find(m, key("post_attention_layernorm.weight"), &L.post_ln, h));
    L.qkv_w = L.o_w = L.gu_w = L.down_w = nullptr;
    L.qkv8 = L.o8 = L.gu8 = L.down8 = nullptr;
    L.qkv_s = L.o_s = L.gu_s = L.down_s = nullptr;
    if (m->int8) {
      // handle-owned fused buffers: q|k|v, o, [ffn/128] blocks of [128 gate | 128 up], down; scales alike
      int8_t *q8, *o8, *g8, *d8;
      float *qs, *os, *gs, *ds;
      SB_PROPAGATE(llama_alloc(m, &q8, (size_t)3 * h * h));
      SB_PROPAGATE(llama_alloc(m, &qs, (size_t)3 * h));
      SB_PROPAGATE(llama_alloc(m, &o8, (size_t)h * h));
      SB_PROPAGATE(llama_alloc(m, &os, (size_t)h));
      SB_PROPAGATE(llama_alloc(m, &g8, (size_t)2 * ffn * h));
      SB_PROPAGATE(llama_alloc(m, &gs, (size_t)2 * ffn));
      SB_PROPAGATE(llama_alloc(m, &d8, (size_t)h * ffn));
      SB_PROPAGATE(llama_alloc(m, &ds, (size_t)h));
      L.qkv8 = q8; L.o8 = o8; L.gu8 = g8; L.down8 = d8;
      L.qkv_s = qs; L.o_s = os; L.gu_s = gs; L.down_s = ds;
      for (int i = 0; i < 7; ++i) {
        const I8Slot t = i8_slot(m, l, i);
        const int8_t* cb;
        const float* scb;
        SB_PROPAGATE(llama_find_i8(m, key(kI8Lin[i]), t.N, t.K, &cb, &scb));
        if (cb == nullptr) continue;     // quantised into its slot later
        const int64_t blocks = t.N / t.grp, dst_rows = t.grp == t.N ? t.N : t.gstride;
        SB_CHECK_CUDA(cudaMemcpy2DAsync(t.cb + t.off * t.K, (size_t)(dst_rows * t.K), cb, (size_t)(t.grp * t.K),
                                        (size_t)(t.grp * t.K), (size_t)blocks, cudaMemcpyDeviceToDevice, st));
        SB_CHECK_CUDA(cudaMemcpy2DAsync(t.scb + t.off, (size_t)(dst_rows * 4), scb, (size_t)(t.grp * 4),
                                        (size_t)(t.grp * 4), (size_t)blocks, cudaMemcpyDeviceToDevice, st));
        m->i8_loaded[(size_t)l * 7 + i] = 1;
      }
      continue;
    }
    SB_PROPAGATE(llama_find(m, key("self_attn.q_proj.weight"), &wq, h * h));
    SB_PROPAGATE(llama_find(m, key("self_attn.k_proj.weight"), &wk, h * h));
    SB_PROPAGATE(llama_find(m, key("self_attn.v_proj.weight"), &wv, h * h));
    SB_PROPAGATE(llama_find(m, key("self_attn.o_proj.weight"), &L.o_w, h * h));
    SB_PROPAGATE(llama_find(m, key("mlp.gate_proj.weight"), &wg, ffn * h));
    SB_PROPAGATE(llama_find(m, key("mlp.up_proj.weight"), &wu, ffn * h));
    SB_PROPAGATE(llama_find(m, key("mlp.down_proj.weight"), &L.down_w, h * ffn));
    __half *fq, *fg;
    SB_PROPAGATE(llama_alloc(m, &fq, (size_t)3 * h * h));
    SB_CHECK_CUDA(cudaMemcpyAsync(fq, wq, (size_t)h * h * 2, cudaMemcpyDeviceToDevice, st));
    SB_CHECK_CUDA(cudaMemcpyAsync(fq + (size_t)h * h, wk, (size_t)h * h * 2, cudaMemcpyDeviceToDevice, st));
    SB_CHECK_CUDA(cudaMemcpyAsync(fq + (size_t)2 * h * h, wv, (size_t)h * h * 2, cudaMemcpyDeviceToDevice, st));
    L.qkv_w = fq;
    // [ffn/128] blocks of [128 gate rows | 128 up rows]
    SB_PROPAGATE(llama_alloc(m, &fg, (size_t)2 * ffn * h));
    const size_t blk = (size_t)128 * h * 2;
    SB_CHECK_CUDA(cudaMemcpy2DAsync(fg, 2 * blk, wg, blk, blk, ffn / 128, cudaMemcpyDeviceToDevice, st));
    SB_CHECK_CUDA(cudaMemcpy2DAsync(reinterpret_cast<uint8_t*>(fg) + blk, 2 * blk, wu, blk, blk, ffn / 128,
                                    cudaMemcpyDeviceToDevice, st));
    L.gu_w = fg;
  }
  SB_PROPAGATE(get_rope_tables(c.head_dim, c.rope_base, c.max_seq, &m->cos_t, &m->sin_t, &m->max_pos, st));
  m->olist = nullptr; m->ocount = nullptr;
  if (m->int8) {
    SB_PROPAGATE(llama_alloc(m, &m->olist, (size_t)(ffn > h ? ffn : h)));
    SB_PROPAGATE(llama_alloc(m, &m->ocount, 1));
  }
  m->vpad = (c.vocab + 7) / 8 * 8;
  SB_PROPAGATE(llama_alloc(m, &m->gstate, 8));
  SB_PROPAGATE(llama_alloc(m, &m->gparams, 1));
  SB_PROPAGATE(llama_alloc(m, &m->beam.params, 1));
  SB_PROPAGATE(llama_alloc(m, &m->beam.n_out, 1));
  SB_PROPAGATE(llama_alloc_rows(m, st));
  SB_CHECK_CUDA(cudaMallocHost(reinterpret_cast<void**>(&m->gstate_host), 8 * sizeof(int)));
  SB_CHECK_CUDA(cudaStreamCreateWithFlags(&m->gstream, cudaStreamNonBlocking));
  SB_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int get_option(const char* key);

static int lin(cudaStream_t st, int ctas, int M, int N, int K, const void* A, const void* W, void* out, int64_t ldo,
               const void* residual, int mode, const void* norm_w = nullptr, float eps = 0.0f) {
  // norm_w: only on the M <= 4 (decode) path, where the GEMV normalises its activations while staging them
  if (M <= 4) return gemv(A, W, K, out, residual, norm_w, eps, M, N, K, mode, st, ldo);
  seedb200_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.M = M; d.N = N; d.K = K; d.A = A; d.lda = K; d.W = W; d.ldw = K;
  d.out = out; d.ldo = ldo; d.residual = residual; d.ldr = ldo; d.mode = mode; d.ctas = ctas;
  return gemm(d, st);
}

// int8 decoder linear: GEMV for M <= 4 (with the RMSNorm folded in when norm_w is given), otherwise activation
// quantisation + int8 wgmma GEMM.  Outputs are dense rows of N (N/2 in mode 1) columns.
static int lin8(seedb200_llama* m, cudaStream_t st, int M, int N, int K, const void* A, const int8_t* W,
                const float* scb, void* out, const void* residual, int mode, const void* norm_w = nullptr,
                float eps = 0.0f) {
  if (M <= 4) return gemv_int8(A, norm_w, eps, m->threshold, W, scb, out, residual, M, N, K, mode, st);
  SB_PROPAGATE(int8_quantize_act(A, K, M, K, m->threshold, m->ca, m->sca, m->olist, m->ocount, st));
  seedb200_gemm_int8_desc d;
  memset(&d, 0, sizeof(d));
  d.M = M; d.N = N; d.K = K;
  d.A = m->ca; d.SCA = m->sca; d.A16 = A; d.outliers = m->olist; d.n_outliers = m->ocount;
  d.W = W; d.SCB = scb; d.out = out; d.residual = residual; d.mode = mode; d.workspace = m->corr;
  return gemm_int8(d, st);
}

// dyn (device, optional): {cache length, ...} read by the RoPE/append and decode-attention kernels instead of the
// host value `past_len` -- what makes a captured decode step position independent (S must be 1).
static int llama_forward(seedb200_llama* m, const int64_t* input_ids, const void* inputs_embeds,
                         const int64_t* position_ids, int B, int S, int past_len, int logits_mode, void* logits,
                         int64_t logits_ld, cudaStream_t st, const int* dyn = nullptr, const int* slot = nullptr) {
  const seedb200_llama_config& c = m->cfg;
  const int h = c.hidden, H = c.heads, D = c.head_dim, ffn = c.ffn, V = c.vocab, ct = c.gemm_ctas;
  const int T = B * S;
  if (input_ids)
    SB_PROPAGATE(embedding(m->embed, h, input_ids, T, h, m->x, h, V, st));
  else
    SB_CHECK_CUDA(cudaMemcpyAsync(m->x, inputs_embeds, (size_t)T * h * 2, cudaMemcpyDeviceToDevice, st));
  const float scale = 1.0f / sqrtf((float)D);   // xformers default scale
  const int kv_len = past_len + S;
  const bool fuse_norm = T <= 4;     // decode: RMSNorm folded into the GEMV that consumes it
  PdlScope pdl(T <= 4 && get_option("decode_pdl") != 0);   // decode chain: programmatic dependent launches
  const bool fused_attn = S == 1 && get_option("decode_fused_attention") != 0 && decode_attention_rope_supported(D, c.max_seq);
  for (int l = 0; l < c.layers; ++l) {
    const LlamaLayerW& L = m->layers[l];
    if (m->int8) {
      if (fuse_norm) {
        SB_PROPAGATE(lin8(m, st, T, 3 * h, h, m->x, L.qkv8, L.qkv_s, m->qkv, nullptr, 0, L.in_ln, c.rms_eps));
      } else {
        SB_PROPAGATE(rmsnorm(m->x, h, L.in_ln, m->nb, h, T, h, c.rms_eps, st));
        SB_PROPAGATE(lin8(m, st, T, 3 * h, h, m->nb, L.qkv8, L.qkv_s, m->qkv, nullptr, 0));
      }
    } else if (fuse_norm) {
      SB_PROPAGATE(lin(st, ct, T, 3 * h, h, m->x, L.qkv_w, m->qkv, 3 * h, nullptr, 0, L.in_ln, c.rms_eps));
    } else {
      SB_PROPAGATE(rmsnorm(m->x, h, L.in_ln, m->nb, h, T, h, c.rms_eps, st));
      SB_PROPAGATE(lin(st, ct, T, 3 * h, h, m->nb, L.qkv_w, m->qkv, 3 * h, nullptr, 0));
    }
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
    if (m->int8) {
      SB_PROPAGATE(lin8(m, st, T, h, h, m->att, L.o8, L.o_s, m->x, m->x, 0));
      if (fuse_norm) {
        SB_PROPAGATE(lin8(m, st, T, 2 * ffn, h, m->x, L.gu8, L.gu_s, m->gu, nullptr, 1, L.post_ln, c.rms_eps));
      } else {
        SB_PROPAGATE(rmsnorm(m->x, h, L.post_ln, m->nb, h, T, h, c.rms_eps, st));
        SB_PROPAGATE(lin8(m, st, T, 2 * ffn, h, m->nb, L.gu8, L.gu_s, m->gu, nullptr, 1));
      }
      SB_PROPAGATE(lin8(m, st, T, h, ffn, m->gu, L.down8, L.down_s, m->x, m->x, 0));
      continue;
    }
    SB_PROPAGATE(lin(st, ct, T, h, h, m->att, L.o_w, m->x, h, m->x, 0));
    if (fuse_norm) {
      SB_PROPAGATE(lin(st, ct, T, 2 * ffn, h, m->x, L.gu_w, m->gu, ffn, nullptr, 1, L.post_ln, c.rms_eps));
    } else {
      SB_PROPAGATE(rmsnorm(m->x, h, L.post_ln, m->nb, h, T, h, c.rms_eps, st));
      SB_PROPAGATE(lin(st, ct, T, 2 * ffn, h, m->nb, L.gu_w, m->gu, ffn, nullptr, 1));
    }
    SB_PROPAGATE(lin(st, ct, T, h, ffn, m->gu, L.down_w, m->x, h, m->x, 0));
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
    state[0] = past_len; state[1] = 0; state[2] = 0; state[3] = 0; state[4] = 0;
  }
  if (threadIdx.x < B) finished[threadIdx.x] = 0;
}

// one unit of the loop: cached forward of the tokens in m->gtok, then the sampler (beams == 0) or the beam candidates
// and scorer (which also advance the device counters).  Every launch argument is a handle-owned pointer or a
// constant: the unit can be captured once per (B, beams).
static int gen_unit(seedb200_llama* m, int B, int beams, cudaStream_t st) {
  PdlScope pdl(get_option("decode_pdl") != 0);
  if (beams == 0) {
    SB_PROPAGATE(llama_forward(m, m->gtok, nullptr, nullptr, B, 1, 0, 1, m->glogits, m->vpad, st, m->gstate));
    SB_PROPAGATE(sample(m->glogits, m->vpad, B, m->cfg.vocab, nullptr, m->gparams, 0, m->gstate, /*advance_cache=*/1,
                        m->gtok, m->gout, m->cfg.max_seq, m->gfinished, st));
    return 0;
  }
  const int rows = B * beams;
  SB_PROPAGATE(llama_forward(m, m->gtok, nullptr, nullptr, rows, 1, 0, 1, m->glogits, m->vpad, st, m->gstate,
                             m->beam.slot));
  SB_PROPAGATE(beam_select(m->glogits, (int64_t)beams * m->vpad, m->vpad, B, beams, m->cfg.vocab, m->beam.beam_scores,
                           nullptr, m->beam.params, 0, m->gstate, m->beam.row_stats, m->beam.cand_score,
                           m->beam.cand_idx, st));
  SB_PROPAGATE(beam_score(m->beam, B, beams, m->cfg.vocab, /*advance_cache=*/1, st));
  return 0;
}

static int gen_capture(seedb200_llama* m, int B, int beams) {
  cudaGraph_t graph = nullptr;
  cudaStream_t st = m->gstream;
  SB_CHECK_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const int64_t before = seedb200_launch_count();
  const int s = gen_unit(m, B, beams, st);
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
  m->graphs[std::make_pair(B, beams)] = std::make_pair(exec, unit);
  return 0;
}

// run `units` decode units (the first eagerly, the rest replayed from the (B, beams) graph when use_graph); with
// `poll`, the device flag state[poll] is read every 32 units and the loop stops once it is set.  Returns units run.
static int gen_run_units(seedb200_llama* m, int B, int beams, int units, int use_graph, int poll, cudaStream_t st,
                         int* done_out) {
  int done = 0;
  m->used_graph = 0;
  if (units > 0) {   // first unit eagerly (also resolves every lazily-set function attribute before a capture)
    SB_PROPAGATE(gen_unit(m, B, beams, st));
    done = 1;
  }
  const auto key = std::make_pair(B, beams);
  if (units > done && use_graph) {
    if (m->graphs.find(key) == m->graphs.end()) {
      int s = gen_capture(m, B, beams);
      if (s != 0 && get_option("decode_pdl") != 0) {   // retry without programmatic launches inside the graph
        seedb200_set_option("decode_pdl", 0);
        s = gen_capture(m, B, beams);
        seedb200_set_option("decode_pdl", 1);
      }
      if (s != 0) return s;
    }
    m->used_graph = 1;
  }
  bool stop = false;
  while (done < units && !stop) {
    int chunk = units - done;
    if (poll >= 0 && chunk > 32) chunk = 32;
    for (int i = 0; i < chunk; ++i) {
      if (m->used_graph) {
        const auto& g = m->graphs[key];
        SB_CHECK_CUDA(cudaGraphLaunch(g.first, st));
        count_launch(g.second);
      } else {
        SB_PROPAGATE(gen_unit(m, B, beams, st));
      }
    }
    done += chunk;
    if (poll >= 0 && done < units) {
      SB_CHECK_CUDA(cudaMemcpyAsync(m->gstate_host, m->gstate, 8 * sizeof(int), cudaMemcpyDeviceToHost, st));
      SB_CHECK_CUDA(cudaStreamSynchronize(st));
      stop = poll == 3 ? m->gstate_host[3] < m->gstate_host[1] : m->gstate_host[poll] != 0;
    }
  }
  *done_out = done;
  return 0;
}

static int llama_generate(seedb200_llama* m, const int64_t* prompt_ids, int B, int S, int max_new,
                          const seedb200_sample_params* sp, int64_t eos, int64_t pad, int use_graph,
                          int64_t* tokens_out, int* n_generated_host, cudaStream_t st) {
  const seedb200_llama_config& c = m->cfg;
  GenParams gp;
  gp.sp = *sp; gp.eos = eos; gp.pad = pad;
  gen_reset_kernel<<<1, 32, 0, st>>>(gp, m->gparams, m->gstate, m->gfinished, S, B);
  SB_LAUNCH_CHECK();
  // prefill: cache rows [0, S), logits of the last position only (what the sampler needs)
  SB_PROPAGATE(llama_forward(m, prompt_ids, nullptr, nullptr, B, S, 0, 1, m->glogits, m->vpad, st));
  // token 0 comes from the prefill logits: the step counter advances, the cache length does not
  SB_PROPAGATE(sample(m->glogits, m->vpad, B, c.vocab, nullptr, m->gparams, 0, m->gstate, /*advance_cache=*/0, m->gtok,
                      m->gout, c.max_seq, m->gfinished, st));
  int done = 0;
  // early stop (only with an eos id): a step ran with every sequence already finished (state[3] < state[1])
  SB_PROPAGATE(gen_run_units(m, B, 0, max_new - 1, use_graph, eos >= 0 ? 3 : -1, st, &done));
  int n_valid = done + 1;
  if (eos >= 0) {
    SB_CHECK_CUDA(cudaMemcpyAsync(m->gstate_host, m->gstate, 8 * sizeof(int), cudaMemcpyDeviceToHost, st));
    SB_CHECK_CUDA(cudaStreamSynchronize(st));
    n_valid = m->gstate_host[3];
  }
  if (tokens_out != nullptr)
    SB_CHECK_CUDA(cudaMemcpy2DAsync(tokens_out, (size_t)max_new * 8, m->gout, (size_t)c.max_seq * 8, (size_t)n_valid * 8, B,
                                    cudaMemcpyDeviceToDevice, st));
  if (n_generated_host != nullptr) *n_generated_host = n_valid;
  m->gen_cache_len = S + done;     // tokens whose K/V are in the cache
  return 0;
}

// beam search: prefill at B rows, candidates + scorer from the prefill logits (every beam reads its sequence's row),
// then max_new - 1 units of (forward of B * k rows through the lineage table -> candidates -> scorer), then finalize
static int llama_beam_generate(seedb200_llama* m, const int64_t* prompt_ids, int B, int S, int max_new,
                               const seedb200_beam_params* p, int64_t eos, int64_t pad, int use_graph,
                               int64_t* tokens_out, int* n_out_host, float* best_scores, cudaStream_t st) {
  const seedb200_llama_config& c = m->cfg;
  const int k = p->num_beams;
  const BeamParams bp = beam_params(*p, eos, pad, S, max_new, B);
  SB_PROPAGATE(beam_init(m->beam, bp, st));
  SB_PROPAGATE(llama_forward(m, prompt_ids, nullptr, nullptr, B, S, 0, 1, m->glogits, m->vpad, st));
  SB_PROPAGATE(beam_select(m->glogits, m->vpad, 0, B, k, c.vocab, m->beam.beam_scores, nullptr, m->beam.params, 0,
                           m->gstate, m->beam.row_stats, m->beam.cand_score,
                           m->beam.cand_idx, st));
  SB_PROPAGATE(beam_score(m->beam, B, k, c.vocab, /*advance_cache=*/0, st));
  int done = 0;
  SB_PROPAGATE(gen_run_units(m, B, k, max_new - 1, use_graph, eos >= 0 ? 5 : -1, st, &done));
  SB_PROPAGATE(beam_finalize(m->beam, B, tokens_out, max_new, best_scores, st));
  int n_out = 0;
  SB_CHECK_CUDA(cudaMemcpyAsync(&n_out, m->beam.n_out, sizeof(int), cudaMemcpyDeviceToHost, st));
  SB_CHECK_CUDA(cudaStreamSynchronize(st));
  if (n_out_host != nullptr) *n_out_host = n_out;
  m->gen_cache_len = 0;            // the cache rows now hold beam lineages, not B plain sequences
  return 0;
}

static void llama_drop_graphs(seedb200_llama* m) {
  for (auto& g : m->graphs) cudaGraphExecDestroy(g.second.first);
  m->graphs.clear();
}

// every int8 linear must hold its weights before the model runs
static int llama_int8_ready(const seedb200_llama* m) {
  for (size_t i = 0; i < m->i8_loaded.size(); ++i)
    if (!m->i8_loaded[i]) {
      set_error("llama: int8 weight 'model.layers.%d.%s.weight' was neither given to create_int8 nor loaded",
                (int)(i / 7), kI8Lin[i % 7]);
      return SEEDB200_ERR_INVALID;
    }
  return 0;
}

}  // namespace sb

extern "C" {

static int llama_create(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights, int int8,
                        float threshold, seedb200_llama** out) {
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
  m->int8 = int8;
  m->threshold = threshold;
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
  return llama_create(cfg, weights, n_weights, 0, 0.0f, out);
}

int seedb200_llama_create_int8(const seedb200_llama_config* cfg, const seedb200_tensor* weights, int n_weights,
                               float threshold, seedb200_llama** out) {
  SB_REQUIRE(threshold > 0.0f, "llama_create_int8: threshold must be > 0 (got %g)", (double)threshold);
  SB_REQUIRE(cfg == nullptr || cfg->hidden % 16 == 0, "llama_create_int8: hidden must be a multiple of 16");
  return llama_create(cfg, weights, n_weights, 1, threshold, out);
}

int seedb200_llama_int8_load_weight(seedb200_llama* llm, const char* name, const void* W, int64_t ldw, void* stream) {
  SB_REQUIRE(llm && name && W, "llama_int8_load_weight: null argument");
  SB_REQUIRE(llm->int8, "llama_int8_load_weight: the handle was not made by seedb200_llama_create_int8");
  int layer = -1, i = -1;
  for (int k = 0; k < 7 && i < 0; ++k) {
    char tail[64];
    snprintf(tail, sizeof(tail), ".%s.weight", sb::kI8Lin[k]);
    int l = -1, n = 0;
    if (sscanf(name, "model.layers.%d%n", &l, &n) == 1 && strcmp(name + n, tail) == 0) { layer = l; i = k; }
  }
  SB_REQUIRE(i >= 0 && layer >= 0 && layer < (int)llm->layers.size(),
             "llama_int8_load_weight: '%s' is not a decoder linear of this model", name);
  const sb::I8Slot t = sb::i8_slot(llm, layer, i);
  if (ldw == 0) ldw = t.K;
  SB_REQUIRE(ldw >= t.K, "llama_int8_load_weight: ldw %lld below K %lld", (long long)ldw, (long long)t.K);
  sb::DeviceGuard guard(llm->device);
  SB_PROPAGATE(sb::int8_quantize_weight_rows(W, ldw, (int)t.N, (int)t.K, t.cb, t.scb, (int)t.grp, (int)t.gstride,
                                             (int)t.off, static_cast<cudaStream_t>(stream)));
  llm->i8_loaded[(size_t)layer * 7 + i] = 1;
  return 0;
}

void seedb200_llama_destroy(seedb200_llama* llm) {
  if (!llm) return;
  sb::llama_drop_graphs(llm);
  if (llm->gstate_host) cudaFreeHost(llm->gstate_host);
  if (llm->gstream) cudaStreamDestroy(llm->gstream);
  sb::llama_free_rows(llm);
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
  SB_PROPAGATE(sb::llama_int8_ready(llm));
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
  SB_REQUIRE(llm && prompt_ids && sp, "llama_generate: null argument");
  SB_REQUIRE(B >= 1 && B <= llm->cfg.max_batch && B <= 4, "llama_generate: batch %d outside [1,%d] (decode GEMV: <= 4 rows)",
             B, llm->cfg.max_batch < 4 ? llm->cfg.max_batch : 4);
  SB_REQUIRE(S >= 1 && max_new_tokens >= 1 && S + max_new_tokens <= llm->cfg.max_seq,
             "llama_generate: prompt %d + %d new tokens exceeds max_seq %d", S, max_new_tokens, llm->cfg.max_seq);
  SB_REQUIRE(!sp->do_sample || (sp->temperature > 0.0f && sp->top_p > 0.0f), "llama_generate: temperature and top_p must be > 0");
  SB_PROPAGATE(sb::llama_int8_ready(llm));
  sb::DeviceGuard guard(llm->device);
  return sb::llama_generate(llm, prompt_ids, B, S, max_new_tokens, sp, eos_id, pad_id, use_graph, tokens_out,
                            n_generated_host, static_cast<cudaStream_t>(stream));
}

int seedb200_llama_generate_used_graph(seedb200_llama* llm) { return llm ? llm->used_graph : -1; }

int seedb200_llama_beam_generate(seedb200_llama* llm, const int64_t* prompt_ids, int B, int S, int max_new_tokens,
                                 const seedb200_beam_params* bp, int64_t eos_id, int64_t pad_id, int use_graph,
                                 int64_t* tokens_out, int* n_out_host, float* best_scores_out, void* stream) {
  SB_REQUIRE(llm && prompt_ids && bp && tokens_out, "llama_beam_generate: null argument");
  SB_REQUIRE(bp->num_beams >= 1 && bp->num_beams <= sb::BEAM_MAX, "llama_beam_generate: num_beams %d outside [1,%d]",
             bp->num_beams, sb::BEAM_MAX);
  SB_REQUIRE(B >= 1 && (int64_t)B * bp->num_beams <= llm->cfg.max_batch,
             "llama_beam_generate: batch %d x %d beams exceeds max_batch %d (seedb200_llama_reserve_rows)", B,
             bp->num_beams, llm->cfg.max_batch);
  SB_REQUIRE(S >= 1 && max_new_tokens >= 1 && S + max_new_tokens <= llm->cfg.max_seq,
             "llama_beam_generate: prompt %d + %d new tokens exceeds max_seq %d", S, max_new_tokens, llm->cfg.max_seq);
  SB_REQUIRE(!bp->do_sample || (bp->temperature > 0.0f && bp->top_p > 0.0f),
             "llama_beam_generate: temperature and top_p must be > 0 when sampling");
  SB_REQUIRE(bp->early_stopping >= 0 && bp->early_stopping <= 2, "llama_beam_generate: early_stopping %d not in {0,1,2}",
             bp->early_stopping);
  SB_REQUIRE(eos_id < llm->cfg.vocab, "llama_beam_generate: eos_id %lld outside the vocabulary", (long long)eos_id);
  SB_PROPAGATE(sb::llama_int8_ready(llm));
  sb::DeviceGuard guard(llm->device);
  return sb::llama_beam_generate(llm, prompt_ids, B, S, max_new_tokens, bp, eos_id, pad_id, use_graph, tokens_out,
                                 n_out_host, best_scores_out, static_cast<cudaStream_t>(stream));
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
