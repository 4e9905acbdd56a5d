// encoder.cu -- seedb200_encoder: the SEED image tokenizer forward (Blip2QformerQuantizer,
// qformer_quantizer.py:143-338) as a fixed sequence of sm_90a kernel launches on the caller's stream.
//
//   encode      = get_codebook_indices (qformer_quantizer.py:288-307):
//                 EVA ViT-g/14 forward_features (eva_vit.py:369-385, 39 x Block :199-206)
//                 -> ln_vision (blip2.py:179-184) -> causal Q-Former (qformer_causual.py:769-931, 12 x BertLayer
//                 :359-444) -> encode_task_layer (:219-223) -> VectorQuantizer2 argmin (:94-98)
//   detokenize  = get_codebook_entry (qformer_quantizer.py:309-338): codebook gather -> decode_task_layer
//                 -> +pos_embed_image -> 4 x vit.Block (vit.py:147-150) -> image_down -> distill_image_proj
//
// The handle borrows the caller's fp16 weight tensors (reference state-dict names), repacks the few that
// change layout (fused QKV / fused cross-attention K|V of all layers / padded patch-embed / qkv bias), and
// owns one workspace sized for max_batch images, so encode() allocates nothing and is graph-capturable.
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "ops.h"

namespace sb {

constexpr int VIT_D = 1408, VIT_H = 16, VIT_HD = 88, VIT_FF = 6144, VIT_TOK = 257, VIT_PATCH = 256;
constexpr int PE_K = 588, PE_KPAD = 592;
constexpr int QF_D = 768, QF_H = 12, QF_HD = 64, QF_FF = 3072, QF_NQ = 32;
constexpr int CB_DIM = 32;
constexpr int DT_OUT = 1024;

struct VitBlockW {
  const __half *n1w, *n1b, *qkv_w, *qkv_b, *proj_w, *proj_b, *n2w, *n2b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
  // LayerNorm folded into the consuming GEMM (option "encoder_ln_fold"): W diag(gamma) in fp16, and the fp32
  // per-column vectors of seedb200_gemm_desc.ln_c / ln_b
  const __half *qkv_wf, *fc1_wf;
  const float *qkv_c, *qkv_bf, *fc1_c, *fc1_bf;
};
struct QfLayerW {
  const __half *qkv_w, *qkv_b, *ao_w, *ao_b, *aln_w, *aln_b;
  bool cross; int cross_idx;
  const __half *cq_w, *cq_b, *co_w, *co_b, *cln_w, *cln_b;
  const __half *fi_w, *fi_b, *fo_w, *fo_b, *fln_w, *fln_b;
};
struct DtBlockW {
  const __half *n1w, *n1b, *qkv_w, *qkv_b, *proj_w, *proj_b, *n2w, *n2b, *fc1_w, *fc1_b, *fc2_w, *fc2_b;
};

}  // namespace sb

struct seedb200_encoder {
  seedb200_encoder_config cfg;
  std::map<std::string, seedb200_tensor> w;
  std::vector<void*> owned;        // repacked weights + workspace (cudaFree on destroy)
  // ViT
  const __half *pe_w, *pe_b, *pos, *clspos, *lnv_w, *lnv_b;
  std::vector<sb::VitBlockW> vit;
  // Q-Former
  const __half* q0;                // LayerNorm(query_tokens) [32,768]
  std::vector<sb::QfLayerW> qf;
  int n_cross;
  const __half *ckv_w, *ckv_b;     // fused cross K|V of all cross layers [n_cross*1536, 1408]
  const __half *e0_w, *e0_b, *e2_w, *e2_b, *codebook, *d0_w, *d0_b, *d2_w, *d2_b;
  // de-tokenizer head
  const __half* pos_img;
  std::vector<sb::DtBlockW> dt;
  const __half *down0, *down2, *down4, *dist_w, *dist_b;
  // workspace
  __half *cols, *x, *ln, *att, *big;   // big = [qkv | mlp hidden] region, reused for the fused cross K|V
  __half *hq, *hq_t, *q_qkv, *q_ctx, *q_inter, *z, *quant, *dtmp;
  int64_t* ids_buf;
  float* row_stats;                // [T] (mean, rstd) pairs of the LayerNorm-folded GEMMs
  float* row_mom;                  // [T][VIT_D / 64] (sum, sum of squares) groups left by the proj / fc2 epilogues
  int ln_fold;
  int stats_fused;                 // option "encoder_stats_fused": statistics from the producing GEMM's epilogue
  __half* img_in;                  // staging for the host entry point
  int last_B;
  int device;                      // the device that was current at create (weights + workspace live there)
};

namespace sb {

static int find_w(const seedb200_encoder* e, const std::string& name, const __half** out, int64_t n_expected) {
  auto it = e->w.find(name);
  if (it == e->w.end()) {
    set_error("encoder_create: missing weight '%s'", name.c_str());
    return SEEDB200_ERR_INVALID;
  }
  const seedb200_tensor& t = it->second;
  if (t.dtype != SEEDB200_F16) {
    set_error("encoder_create: weight '%s' must be fp16", name.c_str());
    return SEEDB200_ERR_INVALID;
  }
  int64_t n = 1;
  for (int i = 0; i < t.ndim; ++i) n *= t.shape[i];
  if (n != n_expected) {
    set_error("encoder_create: weight '%s' has %lld elements, expected %lld", name.c_str(), (long long)n,
              (long long)n_expected);
    return SEEDB200_ERR_INVALID;
  }
  if ((reinterpret_cast<uintptr_t>(t.data) & 15) != 0) {
    set_error("encoder_create: weight '%s' is not 16-byte aligned", name.c_str());
    return SEEDB200_ERR_INVALID;
  }
  *out = static_cast<const __half*>(t.data);
  return 0;
}

#define SB_W(field, name, n) SB_PROPAGATE(find_w(e, (name), &(field), (n)))

static int dev_alloc(seedb200_encoder* e, void** p, size_t bytes) {
  SB_CHECK_CUDA(cudaMalloc(p, bytes < 256 ? 256 : bytes));
  e->owned.push_back(*p);
  return 0;
}
template <typename T>
static int dev_alloc_t(seedb200_encoder* e, T** p, size_t elems) {
  void* q = nullptr;
  SB_PROPAGATE(dev_alloc(e, &q, elems * sizeof(T)));
  *p = static_cast<T*>(q);
  return 0;
}

static int copy2d(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height,
                  cudaStream_t st) {
  SB_CHECK_CUDA(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, cudaMemcpyDeviceToDevice, st));
  return 0;
}

static int linear(cudaStream_t st, int ctas, int M, int N, int K, const void* A, int64_t lda, const void* W,
                  const void* bias, void* out, int64_t ldo, int act = 0, const void* residual = nullptr,
                  int64_t ldr = 0, void* row_moments = nullptr) {
  seedb200_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.M = M; d.N = N; d.K = K;
  d.A = A; d.lda = lda; d.W = W; d.ldw = K;
  d.out = out; d.ldo = ldo; d.bias = bias; d.residual = residual; d.ldr = ldr;
  d.act = act; d.ctas = ctas;
  d.row_moments = row_moments;
  return gemm(d, st);
}

// linear(LayerNorm(x), W, bias) with the LayerNorm folded into the GEMM (seedb200_gemm_desc.ln_stats)
static int linear_ln(cudaStream_t st, int ctas, int M, int N, int K, const void* x, const void* Wf, const void* stats,
                     const void* c, const void* bf, void* out, int64_t ldo, int act) {
  seedb200_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.M = M; d.N = N; d.K = K;
  d.A = x; d.lda = K; d.W = Wf; d.ldw = K;
  d.out = out; d.ldo = ldo; d.act = act; d.ctas = ctas;
  d.ln_stats = stats; d.ln_c = c; d.ln_b = bf;
  return gemm(d, st);
}

int get_option(const char* key);

static int build(seedb200_encoder* e) {
  const seedb200_encoder_config& c = e->cfg;
  cudaStream_t st = 0;
  char nm[256];
  // ---------------- ViT ----------------
  const __half *pe_w_raw, *cls;
  SB_W(pe_w_raw, "visual_encoder.patch_embed.proj.weight", (int64_t)VIT_D * PE_K);
  SB_W(e->pe_b, "visual_encoder.patch_embed.proj.bias", VIT_D);
  SB_W(cls, "visual_encoder.cls_token", VIT_D);
  SB_W(e->pos, "visual_encoder.pos_embed", (int64_t)VIT_TOK * VIT_D);
  SB_W(e->lnv_w, "ln_vision.weight", VIT_D);
  SB_W(e->lnv_b, "ln_vision.bias", VIT_D);
  {
    __half* pw;   // [1408, 592]: conv weight rows zero-padded so TMA rows are 16-byte multiples
    SB_PROPAGATE(dev_alloc_t(e, &pw, (size_t)VIT_D * PE_KPAD));
    SB_CHECK_CUDA(cudaMemsetAsync(pw, 0, (size_t)VIT_D * PE_KPAD * 2, st));
    SB_PROPAGATE(copy2d(pw, PE_KPAD * 2, pe_w_raw, PE_K * 2, PE_K * 2, VIT_D, st));
    e->pe_w = pw;
    __half* cp;   // cls_token + pos_embed[0] (eva_vit.py:372-375), fp16 add
    SB_PROPAGATE(dev_alloc_t(e, &cp, VIT_D));
    SB_PROPAGATE(add_rows(cls, e->pos, cp, 1, VIT_D, 1, st));
    e->clspos = cp;
  }
  e->vit.resize(c.vit_depth);
  for (int i = 0; i < c.vit_depth; ++i) {
    VitBlockW& b = e->vit[i];
    auto key = [&](const char* s) { snprintf(nm, sizeof(nm), "visual_encoder.blocks.%d.%s", i, s); return std::string(nm); };
    const __half *qb, *vb;
    SB_W(b.n1w, key("norm1.weight"), VIT_D); SB_W(b.n1b, key("norm1.bias"), VIT_D);
    SB_W(b.qkv_w, key("attn.qkv.weight"), (int64_t)3 * VIT_D * VIT_D);
    SB_W(qb, key("attn.q_bias"), VIT_D); SB_W(vb, key("attn.v_bias"), VIT_D);
    SB_W(b.proj_w, key("attn.proj.weight"), (int64_t)VIT_D * VIT_D); SB_W(b.proj_b, key("attn.proj.bias"), VIT_D);
    SB_W(b.n2w, key("norm2.weight"), VIT_D); SB_W(b.n2b, key("norm2.bias"), VIT_D);
    SB_W(b.fc1_w, key("mlp.fc1.weight"), (int64_t)VIT_FF * VIT_D); SB_W(b.fc1_b, key("mlp.fc1.bias"), VIT_FF);
    SB_W(b.fc2_w, key("mlp.fc2.weight"), (int64_t)VIT_D * VIT_FF); SB_W(b.fc2_b, key("mlp.fc2.bias"), VIT_D);
    __half* qkvb;   // (q_bias, 0, v_bias)  eva_vit.py:131-133
    SB_PROPAGATE(dev_alloc_t(e, &qkvb, 3 * VIT_D));
    SB_CHECK_CUDA(cudaMemsetAsync(qkvb, 0, 3 * VIT_D * 2, st));
    SB_CHECK_CUDA(cudaMemcpyAsync(qkvb, qb, VIT_D * 2, cudaMemcpyDeviceToDevice, st));
    SB_CHECK_CUDA(cudaMemcpyAsync(qkvb + 2 * VIT_D, vb, VIT_D * 2, cudaMemcpyDeviceToDevice, st));
    b.qkv_b = qkvb;
    b.qkv_wf = b.fc1_wf = nullptr;
    if (e->ln_fold) {
      // norm1 -> qkv and norm2 -> fc1 (eva_vit.py:201-202): the GEMM reads x itself, see seedb200_gemm_desc.ln_stats
      __half *wq, *wf;
      float *cq, *bq, *cf, *bf;
      SB_PROPAGATE(dev_alloc_t(e, &wq, (size_t)3 * VIT_D * VIT_D));
      SB_PROPAGATE(dev_alloc_t(e, &cq, 3 * VIT_D));
      SB_PROPAGATE(dev_alloc_t(e, &bq, 3 * VIT_D));
      SB_PROPAGATE(ln_fold_weights(b.qkv_w, VIT_D, b.n1w, b.n1b, b.qkv_b, 3 * VIT_D, VIT_D, wq, cq, bq, st));
      SB_PROPAGATE(dev_alloc_t(e, &wf, (size_t)VIT_FF * VIT_D));
      SB_PROPAGATE(dev_alloc_t(e, &cf, VIT_FF));
      SB_PROPAGATE(dev_alloc_t(e, &bf, VIT_FF));
      SB_PROPAGATE(ln_fold_weights(b.fc1_w, VIT_D, b.n2w, b.n2b, b.fc1_b, VIT_FF, VIT_D, wf, cf, bf, st));
      b.qkv_wf = wq; b.qkv_c = cq; b.qkv_bf = bq;
      b.fc1_wf = wf; b.fc1_c = cf; b.fc1_bf = bf;
    }
  }
  // ---------------- Q-Former ----------------
  const __half *qtok, *eln_w, *eln_b;
  SB_W(qtok, "query_tokens", (int64_t)QF_NQ * QF_D);
  SB_W(eln_w, "Qformer.bert.embeddings.LayerNorm.weight", QF_D);
  SB_W(eln_b, "Qformer.bert.embeddings.LayerNorm.bias", QF_D);
  {
    __half* q0;   // embeddings.LayerNorm(query_tokens) is input independent (qformer_causual.py:96)
    SB_PROPAGATE(dev_alloc_t(e, &q0, (size_t)QF_NQ * QF_D));
    SB_PROPAGATE(layernorm(qtok, QF_D, eln_w, eln_b, q0, QF_D, QF_NQ, QF_D, 1e-12f, st));
    e->q0 = q0;
  }
  e->qf.resize(c.qformer_layers);
  e->n_cross = 0;
  for (int l = 0; l < c.qformer_layers; ++l)
    if (l % 2 == 0) e->n_cross++;    // cross_attention_freq = 2 (blip2.py:52, qformer_causual.py:350)
  __half *ckv_w = nullptr, *ckv_b = nullptr;
  if (e->n_cross > 0) {
    SB_PROPAGATE(dev_alloc_t(e, &ckv_w, (size_t)e->n_cross * 2 * QF_D * VIT_D));
    SB_PROPAGATE(dev_alloc_t(e, &ckv_b, (size_t)e->n_cross * 2 * QF_D));
  }
  e->ckv_w = ckv_w; e->ckv_b = ckv_b;
  int ci = 0;
  for (int l = 0; l < c.qformer_layers; ++l) {
    QfLayerW& q = e->qf[l];
    auto key = [&](const char* s) { snprintf(nm, sizeof(nm), "Qformer.bert.encoder.layer.%d.%s", l, s); return std::string(nm); };
    const __half *wq, *bq, *wk, *bk, *wv, *bv;
    SB_W(wq, key("attention.self.query.weight"), (int64_t)QF_D * QF_D); SB_W(bq, key("attention.self.query.bias"), QF_D);
    SB_W(wk, key("attention.self.key.weight"), (int64_t)QF_D * QF_D);   SB_W(bk, key("attention.self.key.bias"), QF_D);
    SB_W(wv, key("attention.self.value.weight"), (int64_t)QF_D * QF_D); SB_W(bv, key("attention.self.value.bias"), QF_D);
    __half *fw, *fb;
    SB_PROPAGATE(dev_alloc_t(e, &fw, (size_t)3 * QF_D * QF_D));
    SB_PROPAGATE(dev_alloc_t(e, &fb, (size_t)3 * QF_D));
    const __half* ws[3] = {wq, wk, wv};
    const __half* bs[3] = {bq, bk, bv};
    for (int j = 0; j < 3; ++j) {
      SB_CHECK_CUDA(cudaMemcpyAsync(fw + (size_t)j * QF_D * QF_D, ws[j], (size_t)QF_D * QF_D * 2, cudaMemcpyDeviceToDevice, st));
      SB_CHECK_CUDA(cudaMemcpyAsync(fb + (size_t)j * QF_D, bs[j], QF_D * 2, cudaMemcpyDeviceToDevice, st));
    }
    q.qkv_w = fw; q.qkv_b = fb;
    SB_W(q.ao_w, key("attention.output.dense.weight"), (int64_t)QF_D * QF_D); SB_W(q.ao_b, key("attention.output.dense.bias"), QF_D);
    SB_W(q.aln_w, key("attention.output.LayerNorm.weight"), QF_D); SB_W(q.aln_b, key("attention.output.LayerNorm.bias"), QF_D);
    q.cross = (l % 2 == 0);
    q.cross_idx = -1;
    if (q.cross) {
      q.cross_idx = ci;
      const __half *ckw, *ckb, *cvw, *cvb;
      SB_W(q.cq_w, key("crossattention.self.query.weight"), (int64_t)QF_D * QF_D); SB_W(q.cq_b, key("crossattention.self.query.bias"), QF_D);
      SB_W(ckw, key("crossattention.self.key.weight"), (int64_t)QF_D * VIT_D);     SB_W(ckb, key("crossattention.self.key.bias"), QF_D);
      SB_W(cvw, key("crossattention.self.value.weight"), (int64_t)QF_D * VIT_D);   SB_W(cvb, key("crossattention.self.value.bias"), QF_D);
      SB_W(q.co_w, key("crossattention.output.dense.weight"), (int64_t)QF_D * QF_D); SB_W(q.co_b, key("crossattention.output.dense.bias"), QF_D);
      SB_W(q.cln_w, key("crossattention.output.LayerNorm.weight"), QF_D); SB_W(q.cln_b, key("crossattention.output.LayerNorm.bias"), QF_D);
      const size_t blk = (size_t)QF_D * VIT_D;
      SB_CHECK_CUDA(cudaMemcpyAsync(ckv_w + (size_t)(2 * ci) * blk, ckw, blk * 2, cudaMemcpyDeviceToDevice, st));
      SB_CHECK_CUDA(cudaMemcpyAsync(ckv_w + (size_t)(2 * ci + 1) * blk, cvw, blk * 2, cudaMemcpyDeviceToDevice, st));
      SB_CHECK_CUDA(cudaMemcpyAsync(ckv_b + (size_t)(2 * ci) * QF_D, ckb, QF_D * 2, cudaMemcpyDeviceToDevice, st));
      SB_CHECK_CUDA(cudaMemcpyAsync(ckv_b + (size_t)(2 * ci + 1) * QF_D, cvb, QF_D * 2, cudaMemcpyDeviceToDevice, st));
      ci++;
    }
    SB_W(q.fi_w, key("intermediate_query.dense.weight"), (int64_t)QF_FF * QF_D); SB_W(q.fi_b, key("intermediate_query.dense.bias"), QF_FF);
    SB_W(q.fo_w, key("output_query.dense.weight"), (int64_t)QF_D * QF_FF); SB_W(q.fo_b, key("output_query.dense.bias"), QF_D);
    SB_W(q.fln_w, key("output_query.LayerNorm.weight"), QF_D); SB_W(q.fln_b, key("output_query.LayerNorm.bias"), QF_D);
  }
  SB_W(e->e0_w, "encode_task_layer.0.weight", (int64_t)QF_D * QF_D); SB_W(e->e0_b, "encode_task_layer.0.bias", QF_D);
  SB_W(e->e2_w, "encode_task_layer.2.weight", (int64_t)CB_DIM * QF_D); SB_W(e->e2_b, "encode_task_layer.2.bias", CB_DIM);
  SB_W(e->codebook, "quantize.embedding.weight", (int64_t)c.n_codes * CB_DIM);
  SB_W(e->d0_w, "decode_task_layer.0.weight", (int64_t)CB_DIM * CB_DIM); SB_W(e->d0_b, "decode_task_layer.0.bias", CB_DIM);
  SB_W(e->d2_w, "decode_task_layer.2.weight", (int64_t)QF_D * CB_DIM); SB_W(e->d2_b, "decode_task_layer.2.bias", QF_D);
  // ---------------- de-tokenizer head ----------------
  e->dt.resize(c.detok_depth);
  if (c.detok_depth > 0) {
    SB_W(e->pos_img, "pos_embed_image", (int64_t)QF_NQ * QF_D);
    for (int i = 0; i < c.detok_depth; ++i) {
      DtBlockW& b = e->dt[i];
      auto key = [&](const char* s) { snprintf(nm, sizeof(nm), "blocks_image.%d.%s", i, s); return std::string(nm); };
      SB_W(b.n1w, key("norm1.weight"), QF_D); SB_W(b.n1b, key("norm1.bias"), QF_D);
      SB_W(b.qkv_w, key("attn.qkv.weight"), (int64_t)3 * QF_D * QF_D); SB_W(b.qkv_b, key("attn.qkv.bias"), 3 * QF_D);
      SB_W(b.proj_w, key("attn.proj.weight"), (int64_t)QF_D * QF_D); SB_W(b.proj_b, key("attn.proj.bias"), QF_D);
      SB_W(b.n2w, key("norm2.weight"), QF_D); SB_W(b.n2b, key("norm2.bias"), QF_D);
      SB_W(b.fc1_w, key("mlp.fc1.weight"), (int64_t)QF_FF * QF_D); SB_W(b.fc1_b, key("mlp.fc1.bias"), QF_FF);
      SB_W(b.fc2_w, key("mlp.fc2.weight"), (int64_t)QF_D * QF_FF); SB_W(b.fc2_b, key("mlp.fc2.bias"), QF_D);
    }
    SB_W(e->down0, "image_down.0.weight", (int64_t)256 * QF_D);
    SB_W(e->down2, "image_down.2.weight", (int64_t)128 * 256);
    SB_W(e->down4, "image_down.4.weight", (int64_t)32 * 128);
    SB_W(e->dist_w, "distill_image_proj.weight", (int64_t)DT_OUT * DT_OUT);
    SB_W(e->dist_b, "distill_image_proj.bias", DT_OUT);
  }
  // ---------------- workspace ----------------
  const size_t B = c.max_batch, T = B * VIT_TOK, Q = B * QF_NQ;
  size_t big_cols = (size_t)3 * VIT_D + VIT_FF;
  const size_t ckv_cols = (size_t)e->n_cross * 2 * QF_D;
  if (ckv_cols > big_cols) big_cols = ckv_cols;
  SB_PROPAGATE(dev_alloc_t(e, &e->cols, B * VIT_PATCH * PE_KPAD));
  SB_PROPAGATE(dev_alloc_t(e, &e->x, T * VIT_D));
  SB_PROPAGATE(dev_alloc_t(e, &e->ln, T * VIT_D));
  SB_PROPAGATE(dev_alloc_t(e, &e->att, T * VIT_D));
  SB_PROPAGATE(dev_alloc_t(e, &e->big, T * big_cols));
  SB_PROPAGATE(dev_alloc_t(e, &e->hq, Q * QF_D));
  SB_PROPAGATE(dev_alloc_t(e, &e->hq_t, Q * QF_D));
  SB_PROPAGATE(dev_alloc_t(e, &e->q_qkv, Q * 3 * QF_D));
  SB_PROPAGATE(dev_alloc_t(e, &e->q_ctx, Q * QF_D));
  SB_PROPAGATE(dev_alloc_t(e, &e->q_inter, Q * QF_FF));
  SB_PROPAGATE(dev_alloc_t(e, &e->z, Q * CB_DIM));
  SB_PROPAGATE(dev_alloc_t(e, &e->quant, Q * CB_DIM));
  SB_PROPAGATE(dev_alloc_t(e, &e->dtmp, Q * 256 + B * DT_OUT));
  SB_PROPAGATE(dev_alloc_t(e, &e->ids_buf, Q));
  SB_PROPAGATE(dev_alloc_t(e, &e->row_stats, 2 * T));
  SB_PROPAGATE(dev_alloc_t(e, &e->row_mom, (size_t)2 * T * (VIT_D / 64)));
  SB_PROPAGATE(dev_alloc_t(e, &e->img_in, B * 3 * 224 * 224));
  SB_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

static int attn_call(cudaStream_t st, const __half* q, int64_t q_bs, int64_t q_hs, int64_t q_ts, const __half* k,
                     const __half* v, int64_t kv_bs, int64_t kv_hs, int64_t kv_ts, __half* o, int64_t o_bs,
                     int64_t o_hs, int64_t o_ts, int batch, int heads, int nq, int nk, int hd, int causal,
                     float scale) {
  seedb200_attn_desc d;
  memset(&d, 0, sizeof(d));
  d.q = q; d.k = k; d.v = v; d.o = o;
  d.q_bs = q_bs; d.q_hs = q_hs; d.q_ts = q_ts;
  d.k_bs = kv_bs; d.k_hs = kv_hs; d.k_ts = kv_ts;
  d.v_bs = kv_bs; d.v_hs = kv_hs; d.v_ts = kv_ts;
  d.o_bs = o_bs; d.o_hs = o_hs; d.o_ts = o_ts;
  d.batch = batch; d.heads = heads; d.nq = nq; d.nk = nk; d.head_dim = hd; d.causal = causal; d.scale = scale;
  return attention(d, st);
}

// ViT-g forward_features + ln_vision for B images already in e->cols order (eva_vit.py:369-385)
static int run_vit(seedb200_encoder* e, const void* images, int B, cudaStream_t st) {
  const int ct = e->cfg.gemm_ctas;
  const int T = B * VIT_TOK;
  SB_PROPAGATE(patchify(images, B, e->cols, PE_KPAD, st));
  {
    // conv-as-GEMM + bias, rows scattered behind each image's cls row, + pos_embed[1 + patch]
    seedb200_gemm_desc d;
    memset(&d, 0, sizeof(d));
    d.M = B * VIT_PATCH; d.N = VIT_D; d.K = PE_KPAD;
    d.A = e->cols; d.lda = PE_KPAD; d.W = e->pe_w; d.ldw = PE_KPAD;
    d.out = e->x; d.ldo = VIT_D; d.bias = e->pe_b;
    d.residual = e->pos; d.ldr = VIT_D;
    d.row_group = VIT_PATCH; d.row_stride = VIT_TOK; d.row_offset = 1;
    d.res_mod = VIT_PATCH; d.res_offset = 1;
    d.ctas = ct;
    SB_PROPAGATE(gemm(d, st));
  }
  SB_PROPAGATE(broadcast_rows(e->clspos, 1, VIT_D, e->x, VIT_D, VIT_TOK, B, st));
  __half* qkv = e->big;
  __half* hid = e->big + (size_t)T * 3 * VIT_D;
  const float scale = 0.10660035817780521f;   // 88^-0.5 (eva_vit.py:93)
  for (size_t i = 0; i < e->vit.size(); ++i) {
    const VitBlockW& b = e->vit[i];
    // the statistics of norm1 / norm2: from the epilogue of the GEMM that wrote x (previous block's fc2, this block's
    // proj) when stats_fused, else (and for the first block) from a pass over x
    void* mom = (e->ln_fold && e->stats_fused) ? e->row_mom : nullptr;
    if (e->ln_fold) {
      if (mom != nullptr && i > 0) SB_PROPAGATE(row_stats_from_moments(mom, T, VIT_D, 1e-6f, e->row_stats, st));
      else SB_PROPAGATE(row_stats(e->x, VIT_D, T, VIT_D, 1e-6f, e->row_stats, st));
      SB_PROPAGATE(linear_ln(st, ct, T, 3 * VIT_D, VIT_D, e->x, b.qkv_wf, e->row_stats, b.qkv_c, b.qkv_bf, qkv, 3 * VIT_D, 0));
    } else {
      SB_PROPAGATE(layernorm(e->x, VIT_D, b.n1w, b.n1b, e->ln, VIT_D, T, VIT_D, 1e-6f, st));
      SB_PROPAGATE(linear(st, ct, T, 3 * VIT_D, VIT_D, e->ln, VIT_D, b.qkv_w, b.qkv_b, qkv, 3 * VIT_D));
    }
    SB_PROPAGATE(attn_call(st, qkv, (int64_t)VIT_TOK * 3 * VIT_D, VIT_HD, 3 * VIT_D, qkv + VIT_D, qkv + 2 * VIT_D,
                           (int64_t)VIT_TOK * 3 * VIT_D, VIT_HD, 3 * VIT_D, e->att, (int64_t)VIT_TOK * VIT_D, VIT_HD,
                           VIT_D, B, VIT_H, VIT_TOK, VIT_TOK, VIT_HD, 0, scale));
    SB_PROPAGATE(linear(st, ct, T, VIT_D, VIT_D, e->att, VIT_D, b.proj_w, b.proj_b, e->x, VIT_D, 0, e->x, VIT_D, mom));
    if (e->ln_fold) {
      if (mom != nullptr) SB_PROPAGATE(row_stats_from_moments(mom, T, VIT_D, 1e-6f, e->row_stats, st));
      else SB_PROPAGATE(row_stats(e->x, VIT_D, T, VIT_D, 1e-6f, e->row_stats, st));
      SB_PROPAGATE(linear_ln(st, ct, T, VIT_FF, VIT_D, e->x, b.fc1_wf, e->row_stats, b.fc1_c, b.fc1_bf, hid, VIT_FF,
                             SEEDB200_ACT_GELU));
    } else {
      SB_PROPAGATE(layernorm(e->x, VIT_D, b.n2w, b.n2b, e->ln, VIT_D, T, VIT_D, 1e-6f, st));
      SB_PROPAGATE(linear(st, ct, T, VIT_FF, VIT_D, e->ln, VIT_D, b.fc1_w, b.fc1_b, hid, VIT_FF, SEEDB200_ACT_GELU));
    }
    SB_PROPAGATE(linear(st, ct, T, VIT_D, VIT_FF, hid, VIT_FF, b.fc2_w, b.fc2_b, e->x, VIT_D, 0, e->x, VIT_D,
                        i + 1 < e->vit.size() ? mom : nullptr));
  }
  SB_PROPAGATE(layernorm(e->x, VIT_D, e->lnv_w, e->lnv_b, e->ln, VIT_D, T, VIT_D, 1e-5f, st));
  return 0;
}

// Causal Q-Former over the 32 queries (qformer_causual.py:359-444), e->ln holds image_embeds
static int run_qformer(seedb200_encoder* e, int B, cudaStream_t st) {
  const int ct = e->cfg.gemm_ctas;
  const int T = B * VIT_TOK, Q = B * QF_NQ;
  const int64_t ckv_ld = (int64_t)e->n_cross * 2 * QF_D;
  __half* ckv = e->big;
  if (e->n_cross > 0)   // K|V projections of every cross-attention layer in one GEMM (same input, SURVEY E12)
    SB_PROPAGATE(linear(st, ct, T, (int)ckv_ld, VIT_D, e->ln, VIT_D, e->ckv_w, e->ckv_b, ckv, ckv_ld));
  SB_PROPAGATE(broadcast_rows(e->q0, QF_NQ, QF_D, e->hq, QF_D, QF_NQ, B, st));
  const float scale = 0.125f;   // 1/sqrt(64) (qformer_causual.py:232)
  for (size_t l = 0; l < e->qf.size(); ++l) {
    const QfLayerW& w = e->qf[l];
    SB_PROPAGATE(linear(st, ct, Q, 3 * QF_D, QF_D, e->hq, QF_D, w.qkv_w, w.qkv_b, e->q_qkv, 3 * QF_D));
    SB_PROPAGATE(attn_call(st, e->q_qkv, (int64_t)QF_NQ * 3 * QF_D, QF_HD, 3 * QF_D, e->q_qkv + QF_D,
                           e->q_qkv + 2 * QF_D, (int64_t)QF_NQ * 3 * QF_D, QF_HD, 3 * QF_D, e->q_ctx,
                           (int64_t)QF_NQ * QF_D, QF_HD, QF_D, B, QF_H, QF_NQ, QF_NQ, QF_HD, 1, scale));
    SB_PROPAGATE(linear(st, ct, Q, QF_D, QF_D, e->q_ctx, QF_D, w.ao_w, w.ao_b, e->hq_t, QF_D, 0, e->hq, QF_D));
    SB_PROPAGATE(layernorm(e->hq_t, QF_D, w.aln_w, w.aln_b, e->hq, QF_D, Q, QF_D, 1e-12f, st));
    if (w.cross) {
      const __half* kk = ckv + (size_t)(2 * w.cross_idx) * QF_D;
      const __half* vv = ckv + (size_t)(2 * w.cross_idx + 1) * QF_D;
      SB_PROPAGATE(linear(st, ct, Q, QF_D, QF_D, e->hq, QF_D, w.cq_w, w.cq_b, e->q_qkv, QF_D));
      SB_PROPAGATE(attn_call(st, e->q_qkv, (int64_t)QF_NQ * QF_D, QF_HD, QF_D, kk, vv, (int64_t)VIT_TOK * ckv_ld,
                             QF_HD, ckv_ld, e->q_ctx, (int64_t)QF_NQ * QF_D, QF_HD, QF_D, B, QF_H, QF_NQ, VIT_TOK,
                             QF_HD, 0, scale));
      SB_PROPAGATE(linear(st, ct, Q, QF_D, QF_D, e->q_ctx, QF_D, w.co_w, w.co_b, e->hq_t, QF_D, 0, e->hq, QF_D));
      SB_PROPAGATE(layernorm(e->hq_t, QF_D, w.cln_w, w.cln_b, e->hq, QF_D, Q, QF_D, 1e-12f, st));
    }
    SB_PROPAGATE(linear(st, ct, Q, QF_FF, QF_D, e->hq, QF_D, w.fi_w, w.fi_b, e->q_inter, QF_FF, SEEDB200_ACT_GELU));
    SB_PROPAGATE(linear(st, ct, Q, QF_D, QF_FF, e->q_inter, QF_FF, w.fo_w, w.fo_b, e->hq_t, QF_D, 0, e->hq, QF_D));
    SB_PROPAGATE(layernorm(e->hq_t, QF_D, w.fln_w, w.fln_b, e->hq, QF_D, Q, QF_D, 1e-12f, st));
  }
  return 0;
}

static int encode_chunk(seedb200_encoder* e, const void* images, int B, int64_t* ids, void* z_out, void* qup_out,
                        cudaStream_t st) {
  const int ct = e->cfg.gemm_ctas;
  const int Q = B * QF_NQ;
  SB_PROPAGATE(run_vit(e, images, B, st));
  SB_PROPAGATE(run_qformer(e, B, st));
  // encode_task_layer: Linear(768,768) - Tanh - Linear(768,32)  (qformer_quantizer.py:219-223,301)
  SB_PROPAGATE(linear(st, ct, Q, QF_D, QF_D, e->hq, QF_D, e->e0_w, e->e0_b, e->hq_t, QF_D, SEEDB200_ACT_TANH));
  __half* z = z_out ? static_cast<__half*>(z_out) : e->z;
  SB_PROPAGATE(linear(st, ct, Q, CB_DIM, QF_D, e->hq_t, QF_D, e->e2_w, e->e2_b, z, CB_DIM));
  SB_PROPAGATE(vq_argmin(z, e->codebook, Q, e->cfg.n_codes, CB_DIM, e->cfg.vq_mode, ids, st));
  if (qup_out) {
    // quant = embedding(ids); decode_task_layer(quant)  (qformer_quantizer.py:99,305)
    SB_PROPAGATE(embedding(e->codebook, CB_DIM, ids, Q, CB_DIM, e->quant, CB_DIM, e->cfg.n_codes, st));
    SB_PROPAGATE(linear(st, ct, Q, CB_DIM, CB_DIM, e->quant, CB_DIM, e->d0_w, e->d0_b, e->z, CB_DIM, SEEDB200_ACT_TANH));
    SB_PROPAGATE(linear(st, ct, Q, QF_D, CB_DIM, e->z, CB_DIM, e->d2_w, e->d2_b, qup_out, QF_D));
  }
  e->last_B = B;
  return 0;
}

static int detok_chunk(seedb200_encoder* e, const int64_t* ids, int B, void* out, cudaStream_t st) {
  const int ct = e->cfg.gemm_ctas;
  const int Q = B * QF_NQ;
  SB_PROPAGATE(embedding(e->codebook, CB_DIM, ids, Q, CB_DIM, e->quant, CB_DIM, e->cfg.n_codes, st));
  SB_PROPAGATE(linear(st, ct, Q, CB_DIM, CB_DIM, e->quant, CB_DIM, e->d0_w, e->d0_b, e->z, CB_DIM, SEEDB200_ACT_TANH));
  {
    // decode_task_layer.2 + pos_embed_image (qformer_quantizer.py:314-317)
    seedb200_gemm_desc d;
    memset(&d, 0, sizeof(d));
    d.M = Q; d.N = QF_D; d.K = CB_DIM;
    d.A = e->z; d.lda = CB_DIM; d.W = e->d2_w; d.ldw = CB_DIM;
    d.out = e->hq; d.ldo = QF_D; d.bias = e->d2_b;
    d.residual = e->pos_img; d.ldr = QF_D; d.res_mod = QF_NQ; d.res_offset = 0;
    d.ctas = ct;
    SB_PROPAGATE(gemm(d, st));
  }
  const float scale = 0.125f;
  for (size_t i = 0; i < e->dt.size(); ++i) {
    const DtBlockW& b = e->dt[i];   // vit.Block: pre-LN attention + MLP (vit.py:147-150)
    SB_PROPAGATE(layernorm(e->hq, QF_D, b.n1w, b.n1b, e->hq_t, QF_D, Q, QF_D, 1e-6f, st));
    SB_PROPAGATE(linear(st, ct, Q, 3 * QF_D, QF_D, e->hq_t, QF_D, b.qkv_w, b.qkv_b, e->q_qkv, 3 * QF_D));
    SB_PROPAGATE(attn_call(st, e->q_qkv, (int64_t)QF_NQ * 3 * QF_D, QF_HD, 3 * QF_D, e->q_qkv + QF_D,
                           e->q_qkv + 2 * QF_D, (int64_t)QF_NQ * 3 * QF_D, QF_HD, 3 * QF_D, e->q_ctx,
                           (int64_t)QF_NQ * QF_D, QF_HD, QF_D, B, QF_H, QF_NQ, QF_NQ, QF_HD, 0, scale));
    SB_PROPAGATE(linear(st, ct, Q, QF_D, QF_D, e->q_ctx, QF_D, b.proj_w, b.proj_b, e->hq, QF_D, 0, e->hq, QF_D));
    SB_PROPAGATE(layernorm(e->hq, QF_D, b.n2w, b.n2b, e->hq_t, QF_D, Q, QF_D, 1e-6f, st));
    SB_PROPAGATE(linear(st, ct, Q, QF_FF, QF_D, e->hq_t, QF_D, b.fc1_w, b.fc1_b, e->q_inter, QF_FF, SEEDB200_ACT_GELU));
    SB_PROPAGATE(linear(st, ct, Q, QF_D, QF_FF, e->q_inter, QF_FF, b.fc2_w, b.fc2_b, e->hq, QF_D, 0, e->hq, QF_D));
  }
  // image_down: 768 -> 256 -> ReLU -> 128 -> ReLU -> 32 (no bias); reshape [B,1024]; distill_image_proj
  __half* t256 = e->dtmp;
  __half* t128 = e->q_ctx;
  __half* t32 = e->dtmp + (size_t)Q * 256;   // [Q,32] == [B,1024]
  SB_PROPAGATE(linear(st, ct, Q, 256, QF_D, e->hq, QF_D, e->down0, nullptr, t256, 256, SEEDB200_ACT_RELU));
  SB_PROPAGATE(linear(st, ct, Q, 128, 256, t256, 256, e->down2, nullptr, t128, 128, SEEDB200_ACT_RELU));
  SB_PROPAGATE(linear(st, ct, Q, 32, 128, t128, 128, e->down4, nullptr, t32, 32));
  SB_PROPAGATE(linear(st, ct, B, DT_OUT, DT_OUT, t32, DT_OUT, e->dist_w, e->dist_b, out, DT_OUT));
  return 0;
}

}  // namespace sb

extern "C" {

int seedb200_encoder_create(const seedb200_encoder_config* cfg, const seedb200_tensor* weights, int n_weights,
                            seedb200_encoder** out) {
  if (!cfg || !weights || !out) {
    sb::set_error("encoder_create: null argument");
    return SEEDB200_ERR_INVALID;
  }
  SB_REQUIRE(cfg->vit_depth >= 0 && cfg->qformer_layers >= 0 && cfg->detok_depth >= 0, "encoder_create: negative depth");
  SB_REQUIRE(cfg->max_batch >= 1, "encoder_create: max_batch must be >= 1");
  SB_REQUIRE(cfg->n_codes >= 1, "encoder_create: n_codes must be >= 1");
  seedb200_encoder* e = new seedb200_encoder();
  e->cfg = *cfg;
  e->last_B = 0;
  e->device = sb::cur_device();
  e->ln_fold = sb::get_option("encoder_ln_fold") != 0;
  e->stats_fused = sb::get_option("encoder_stats_fused") != 0;
  for (int i = 0; i < n_weights; ++i) e->w[std::string(weights[i].name)] = weights[i];
  int s = sb::build(e);
  if (s != 0) {
    seedb200_encoder_destroy(e);
    return s;
  }
  e->w.clear();
  *out = e;
  return 0;
}

void seedb200_encoder_destroy(seedb200_encoder* enc) {
  if (!enc) return;
  for (void* p : enc->owned) cudaFree(p);
  delete enc;
}

int seedb200_encoder_encode(seedb200_encoder* enc, const void* images, int B, int64_t* ids, void* z_out,
                            void* query_up_out, void* stream) {
  SB_REQUIRE(enc && images && ids, "encoder_encode: null argument");
  SB_REQUIRE(B >= 1, "encoder_encode: empty batch");
  sb::DeviceGuard guard(enc->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int mb = enc->cfg.max_batch;
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int nb = (B - b0) < mb ? (B - b0) : mb;
    const __half* img = static_cast<const __half*>(images) + (size_t)b0 * 3 * 224 * 224;
    void* z = z_out ? static_cast<__half*>(z_out) + (size_t)b0 * sb::QF_NQ * sb::CB_DIM : nullptr;
    void* qu = query_up_out ? static_cast<__half*>(query_up_out) + (size_t)b0 * sb::QF_NQ * sb::QF_D : nullptr;
    SB_PROPAGATE(sb::encode_chunk(enc, img, nb, ids + (size_t)b0 * sb::QF_NQ, z, qu, st));
  }
  return 0;
}

int seedb200_encoder_encode_host(seedb200_encoder* enc, const void* images_host, int B, int64_t* ids_host,
                                 void* stream) {
  SB_REQUIRE(enc && images_host && ids_host, "encoder_encode_host: null argument");
  SB_REQUIRE(B >= 1, "encoder_encode_host: empty batch");
  sb::DeviceGuard guard(enc->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int mb = enc->cfg.max_batch;
  const size_t img_elems = (size_t)3 * 224 * 224;
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int nb = (B - b0) < mb ? (B - b0) : mb;
    SB_CHECK_CUDA(cudaMemcpyAsync(enc->img_in, static_cast<const __half*>(images_host) + (size_t)b0 * img_elems,
                                  (size_t)nb * img_elems * 2, cudaMemcpyHostToDevice, st));
    SB_PROPAGATE(sb::encode_chunk(enc, enc->img_in, nb, enc->ids_buf, nullptr, nullptr, st));
    SB_CHECK_CUDA(cudaMemcpyAsync(ids_host + (size_t)b0 * sb::QF_NQ, enc->ids_buf, (size_t)nb * sb::QF_NQ * 8,
                                  cudaMemcpyDeviceToHost, st));
  }
  return 0;
}

int seedb200_encoder_encode_tokens(seedb200_encoder* enc, const void* images, int B, int64_t image_id_shift, int64_t boi,
                                   int64_t eoi, int64_t* tokens_out, int64_t out_stride, int64_t* ids_out, void* stream) {
  SB_REQUIRE(enc && images && tokens_out, "encoder_encode_tokens: null argument");
  SB_REQUIRE(B >= 1 && out_stride >= 34, "encoder_encode_tokens: bad sizes");
  sb::DeviceGuard guard(enc->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int mb = enc->cfg.max_batch;
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int nb = (B - b0) < mb ? (B - b0) : mb;
    const __half* img = static_cast<const __half*>(images) + (size_t)b0 * 3 * 224 * 224;
    int64_t* ids = ids_out ? ids_out + (size_t)b0 * sb::QF_NQ : enc->ids_buf;
    SB_PROPAGATE(sb::encode_chunk(enc, img, nb, ids, nullptr, nullptr, st));
    SB_PROPAGATE(sb::image_ids_to_tokens(ids, nb, image_id_shift, boi, eoi, tokens_out + (size_t)b0 * out_stride,
                                         out_stride, st));
  }
  return 0;
}

int seedb200_encoder_detokenize(seedb200_encoder* enc, const int64_t* ids, int B, void* embeds_out, void* stream) {
  SB_REQUIRE(enc && ids && embeds_out, "encoder_detokenize: null argument");
  SB_REQUIRE(enc->cfg.detok_depth > 0 || enc->down0 != nullptr, "encoder_detokenize: handle was created without the de-tokenizer head");
  SB_REQUIRE(B >= 1, "encoder_detokenize: empty batch");
  sb::DeviceGuard guard(enc->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int mb = enc->cfg.max_batch;
  for (int b0 = 0; b0 < B; b0 += mb) {
    const int nb = (B - b0) < mb ? (B - b0) : mb;
    SB_PROPAGATE(sb::detok_chunk(enc, ids + (size_t)b0 * sb::QF_NQ, nb,
                                 static_cast<__half*>(embeds_out) + (size_t)b0 * sb::DT_OUT, st));
  }
  return 0;
}

int64_t seedb200_encoder_tap(seedb200_encoder* enc, int what, void* dst, int64_t max_elems, void* stream) {
  if (!enc || !dst || enc->last_B <= 0) return -1;
  sb::DeviceGuard guard(enc->device);
  const __half* src = nullptr;
  int64_t n = 0;
  if (what == 0) { src = enc->x; n = (int64_t)enc->last_B * sb::VIT_TOK * sb::VIT_D; }
  else if (what == 1) { src = enc->hq; n = (int64_t)enc->last_B * sb::QF_NQ * sb::QF_D; }
  else if (what == 2) { src = enc->ln; n = (int64_t)enc->last_B * sb::VIT_TOK * sb::VIT_D; }
  else return -1;
  if (n > max_elems) n = max_elems;
  if (cudaMemcpyAsync(dst, src, (size_t)n * 2, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)) != cudaSuccess)
    return -1;
  return n;
}

}  // extern "C"
