"""Deterministic synthetic weights and inputs for the parity tests and bench.py (data generation only: no
model arithmetic lives here, and nothing in the kernels or the Python mirror imports it).

There is no network, so real checkpoints (seed_quantizer.pt, eva_vit_g.pth, SEED-LLaMA) are unavailable.
Weights are drawn per tensor from a generator seeded by a hash of (seed, tensor name), so any subset can be
regenerated independently and identically on any machine with the same torch.  Every value is rounded to
fp16 so that the fp32 CPU oracle and the fp16 GPU path consume bit-identical parameters.

Deviation from the reference initialisers (documented in the bench output):
  * the codebook is drawn N(0, CODEBOOK_STD) instead of U(+-1/8192) (qformer_quantizer.py:39): with the default
    init every distance rounds to |z|^2 in fp16 and argmin is 0 for all tokens, which makes id parity vacuous
    (SURVEY.md section 7 "degenerate synthetic codebook");
  * biases and LayerNorm affine parameters are non-trivial (the reference inits them to 0 / 1) so that the
    bias / affine code paths are exercised.
Names and shapes are the reference's own (qformer_quantizer.py:161-286 constructed through oracle/ref_shim.py;
HF LLaMA names for llama_xformer.py).
"""
from __future__ import annotations

import hashlib
import math
from typing import Dict

import torch

CODEBOOK_STD = 0.28  # ~ std of encode_task_layer outputs under these weights (measured, see make_golden.py)


def _gen(seed: int, name: str) -> torch.Generator:
    h = hashlib.sha256(f"{seed}:{name}".encode()).digest()
    return torch.Generator(device="cpu").manual_seed(int.from_bytes(h[:7], "little"))


def _normal(seed, name, shape, std, mean=0.0):
    t = torch.randn(*shape, generator=_gen(seed, name)) * std + mean
    return t.to(torch.float16).to(torch.float32)


def encoder_state_dict(vit_depth: int = 39, qformer_layers: int = 12, detok_depth: int = 4, n_codes: int = 8192,
                       seed: int = 1234) -> Dict[str, torch.Tensor]:
    """fp32 tensors holding fp16-representable values, keyed by the reference state-dict names."""
    sd: Dict[str, torch.Tensor] = {}
    D, FF = 1408, 6144

    def lin(prefix, out_f, in_f, std=0.02, bias=True, scale=1.0):
        sd[prefix + ".weight"] = _normal(seed, prefix + ".weight", (out_f, in_f), std * scale)
        if bias:
            sd[prefix + ".bias"] = _normal(seed, prefix + ".bias", (out_f,), 0.02)

    def ln(prefix, n):
        sd[prefix + ".weight"] = _normal(seed, prefix + ".weight", (n,), 0.05, 1.0)
        sd[prefix + ".bias"] = _normal(seed, prefix + ".bias", (n,), 0.02)

    sd["visual_encoder.cls_token"] = _normal(seed, "visual_encoder.cls_token", (1, 1, D), 0.02)
    sd["visual_encoder.pos_embed"] = _normal(seed, "visual_encoder.pos_embed", (1, 257, D), 0.02)
    sd["visual_encoder.patch_embed.proj.weight"] = _normal(seed, "visual_encoder.patch_embed.proj.weight",
                                                            (D, 3, 14, 14), 0.02)
    sd["visual_encoder.patch_embed.proj.bias"] = _normal(seed, "visual_encoder.patch_embed.proj.bias", (D,), 0.02)
    for i in range(vit_depth):
        p = f"visual_encoder.blocks.{i}."
        rescale = 1.0 / math.sqrt(2.0 * (i + 1))       # fix_init_weight (eva_vit.py:343-349)
        ln(p + "norm1", D)
        sd[p + "attn.qkv.weight"] = _normal(seed, p + "attn.qkv.weight", (3 * D, D), 0.02)
        sd[p + "attn.q_bias"] = _normal(seed, p + "attn.q_bias", (D,), 0.02)
        sd[p + "attn.v_bias"] = _normal(seed, p + "attn.v_bias", (D,), 0.02)
        lin(p + "attn.proj", D, D, scale=rescale)
        ln(p + "norm2", D)
        lin(p + "mlp.fc1", FF, D)
        lin(p + "mlp.fc2", D, FF, scale=rescale)
    ln("ln_vision", D)

    H, QFF = 768, 3072
    sd["query_tokens"] = _normal(seed, "query_tokens", (1, 32, H), 0.02)
    ln("Qformer.bert.embeddings.LayerNorm", H)
    for l in range(qformer_layers):
        p = f"Qformer.bert.encoder.layer.{l}."
        for n in ("query", "key", "value"):
            lin(p + "attention.self." + n, H, H)
        # small residual branches (std 0.005) keep the 32 post-LN query states from collapsing onto one
        # direction over 12 random layers, so the synthetic ids differ per query token
        lin(p + "attention.output.dense", H, H, std=0.005)
        ln(p + "attention.output.LayerNorm", H)
        if l % 2 == 0:
            lin(p + "crossattention.self.query", H, H)
            lin(p + "crossattention.self.key", H, D)
            # 1.5x the default std: makes the query outputs (hence the ids) depend visibly on the image
            lin(p + "crossattention.self.value", H, D, std=0.03)
            lin(p + "crossattention.output.dense", H, H, std=0.03)
            ln(p + "crossattention.output.LayerNorm", H)
        lin(p + "intermediate_query.dense", QFF, H)
        lin(p + "output_query.dense", H, QFF, std=0.005)
        ln(p + "output_query.LayerNorm", H)
    lin("encode_task_layer.0", H, H)
    lin("encode_task_layer.2", 32, H)
    sd["quantize.embedding.weight"] = _normal(seed, "quantize.embedding.weight", (n_codes, 32), CODEBOOK_STD)
    lin("decode_task_layer.0", 32, 32, std=0.2)
    lin("decode_task_layer.2", H, 32, std=0.2)
    if detok_depth > 0:
        sd["pos_embed_image"] = _normal(seed, "pos_embed_image", (1, 32, H), 0.02)
        for i in range(detok_depth):
            p = f"blocks_image.{i}."
            ln(p + "norm1", H)
            lin(p + "attn.qkv", 3 * H, H)
            lin(p + "attn.proj", H, H)
            ln(p + "norm2", H)
            lin(p + "mlp.fc1", QFF, H)
            lin(p + "mlp.fc2", H, QFF)
        lin("image_down.0", 256, H, bias=False, std=0.05)
        lin("image_down.2", 128, 256, bias=False, std=0.08)
        lin("image_down.4", 32, 128, bias=False, std=0.1)
        lin("distill_image_proj", 1024, 1024, std=0.03)
    return sd


def images(batch: int, seed: int = 1234) -> torch.Tensor:
    """[B,3,224,224] fp32 holding fp16-representable values with CLIP-normalised statistics (SURVEY 8d)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(batch, 3, 224, 224, generator=g).to(torch.float16).to(torch.float32)


def llama_state_dict(hidden: int, layers: int, ffn: int, vocab: int, seed: int = 1234) -> Dict[str, torch.Tensor]:
    sd: Dict[str, torch.Tensor] = {}
    sd["model.embed_tokens.weight"] = _normal(seed, "model.embed_tokens.weight", (vocab, hidden), 0.02)
    for l in range(layers):
        p = f"model.layers.{l}."
        for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
            sd[p + f"self_attn.{n}.weight"] = _normal(seed, p + f"self_attn.{n}.weight", (hidden, hidden), 0.02)
        sd[p + "mlp.gate_proj.weight"] = _normal(seed, p + "mlp.gate_proj.weight", (ffn, hidden), 0.02)
        sd[p + "mlp.up_proj.weight"] = _normal(seed, p + "mlp.up_proj.weight", (ffn, hidden), 0.02)
        sd[p + "mlp.down_proj.weight"] = _normal(seed, p + "mlp.down_proj.weight", (hidden, ffn), 0.02)
        sd[p + "input_layernorm.weight"] = _normal(seed, p + "input_layernorm.weight", (hidden,), 0.05, 1.0)
        sd[p + "post_attention_layernorm.weight"] = _normal(seed, p + "post_attention_layernorm.weight", (hidden,),
                                                            0.05, 1.0)
    sd["model.norm.weight"] = _normal(seed, "model.norm.weight", (hidden,), 0.05, 1.0)
    sd["lm_head.weight"] = _normal(seed, "lm_head.weight", (vocab, hidden), 0.02)
    return sd


def prompt_ids(batch: int, seq: int, n_image_spans: int = 1, text_vocab: int = 32000, n_codes: int = 8192,
               seed: int = 1234) -> torch.Tensor:
    """Interleaved text + <img> 32 image ids </img> sequences (scripts/seed_llama_inference_8B.py:16-23,60,100):
    text ids uniform in [0, text_vocab), image token id = text_vocab + code, BOI/EOI = the two ids after."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    ids = torch.randint(0, text_vocab, (batch, seq), generator=g)
    boi, eoi = text_vocab + n_codes, text_vocab + n_codes + 1
    span = 34
    for b in range(batch):
        for s in range(n_image_spans):
            start = 1 + s * (span + 3)
            if start + span > seq:
                break
            ids[b, start] = boi
            ids[b, start + 1:start + 33] = text_vocab + torch.randint(0, n_codes, (32,), generator=g)
            ids[b, start + 33] = eoi
    return ids
