"""TEST INFRASTRUCTURE ONLY -- per-op restatements (plain torch, fp32 math) of the reference expressions each
CUDA kernel replaces.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this.

Every function takes fp16 (or int) tensors, computes in fp32 on whatever device they live on, and rounds to
fp16 at the points where the reference's fp16 GPU mode rounds (SURVEY.md section 8a precision table), so the
kernels can be compared with a tolerance of a few fp16 ulps.  `dtype=torch.float64` computes the same expression
with the same fp16 rounding points in double precision (tests/test_kernel_edges_gpu.py bounds the kernels against it).
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F


def r16(x: torch.Tensor) -> torch.Tensor:
    """round an fp32 / fp64 tensor to fp16 and back (the rounding torch applies when it stores an fp16 result)."""
    return x.to(torch.float16).to(x.dtype)


def linear_ref(a, w, bias=None, act: int = 0, residual=None, dtype=torch.float32):
    """torch.nn.functional.linear + activation + residual with fp16 rounding after each torch op
    (eva_vit.py:133-135,157,60-65; qformer_causual.py:251-255,320-337)."""
    y = a.to(dtype) @ w.to(dtype).t()
    if bias is not None:
        y = y + bias.to(dtype)
    y = r16(y)
    if act == 1:
        y = r16(F.gelu(y))            # exact erf GELU (nn.GELU / ACT2FN['gelu'])
    elif act == 2:
        y = r16(torch.tanh(y))
    elif act == 3:
        y = r16(torch.relu(y))
    if residual is not None:
        y = r16(y + residual.to(dtype))
    return y.to(torch.float16)


def silu_gate_ref(a, w_gate, w_up, dtype=torch.float32):
    """LlamaMLP: act_fn(gate_proj(x)) * up_proj(x)  (llama_xformer.py:186), fp16 tensors at every step."""
    g = r16(a.to(dtype) @ w_gate.to(dtype).t())
    u = r16(a.to(dtype) @ w_up.to(dtype).t())
    s = r16(F.silu(g))
    return r16(s * u).to(torch.float16)


def interleave_gate_up(w_gate, w_up):
    """[ffn,h] x2 -> [2*ffn,h] in blocks of [128 gate rows | 128 up rows] (the layout seedb200 mode 1 expects)."""
    ffn, h = w_gate.shape
    assert ffn % 128 == 0
    g = w_gate.reshape(ffn // 128, 128, h)
    u = w_up.reshape(ffn // 128, 128, h)
    return torch.cat([g, u], dim=1).reshape(2 * ffn, h).contiguous()


def layernorm_ref(x, w, b, eps: float, dtype=torch.float32):
    """nn.LayerNorm evaluated in fp32, result cast to fp16 (blip2.py:179-184; autocast fp32 LN in eva_vit.py:201)."""
    return F.layer_norm(x.to(dtype), (x.shape[-1],), w.to(dtype), b.to(dtype), eps).to(torch.float16)


def rmsnorm_ref(x, w, eps: float, dtype=torch.float32):
    """LlamaRMSNorm.forward (llama_xformer.py:105-113): the normalised row is rounded to fp16 before the fp16
    multiply by the weight (a product of two fp16 values is exact in fp32, so that multiply rounds once)."""
    xf = x.to(dtype)
    var = xf.pow(2).mean(-1, keepdim=True)
    h = (xf * torch.rsqrt(var + eps)).to(torch.float16)
    return (w.to(dtype) * h.to(dtype)).to(torch.float16)


def attention_ref(q, k, v, scale: float, causal: bool = False, dtype=torch.float32):
    """softmax(scale * q k^T [+ causal mask]) v in fp32; q [B,H,Nq,D], k/v [B,H,Nk,D] -> [B,Nq,H,D] fp16
    (eva_vit.py:139-156; qformer_causual.py:189-236; llama_xformer.py:240-256)."""
    qf, kf, vf = q.to(dtype), k.to(dtype), v.to(dtype)
    s = (qf @ kf.transpose(-1, -2)) * scale
    if causal:
        nq, nk = q.shape[2], k.shape[2]
        i = torch.arange(nq, device=q.device)[:, None]
        j = torch.arange(nk, device=q.device)[None, :]
        s = s.masked_fill(j > i + (nk - nq), float("-inf"))
    p = torch.softmax(s, dim=-1)
    o = p @ vf
    return o.permute(0, 2, 1, 3).contiguous().to(torch.float16)


def vq_torch_ref(z, codebook):
    """The reference expression itself (qformer_quantizer.py:94-98) on whatever dtype it is given."""
    d = torch.sum(z ** 2, dim=1, keepdim=True) + torch.sum(codebook ** 2, dim=1) - 2 * torch.einsum(
        "bd,dn->bn", z, codebook.t())
    return torch.argmin(d, dim=1), d


def patchify_ref(images, kpad: int = 592):
    """Unfold for Conv2d(3, 1408, 14, stride 14) (eva_vit.py:222,229): [B,3,224,224] -> [B*256, kpad]."""
    B = images.shape[0]
    cols = F.unfold(images.float(), kernel_size=14, stride=14)      # [B, 588, 256], column = c*196+dy*14+dx
    cols = cols.transpose(1, 2).reshape(B * 256, 588)
    out = torch.zeros((B * 256, kpad), dtype=torch.float32, device=images.device)
    out[:, :588] = cols
    return out.to(torch.float16)


def rope_tables(max_pos: int, dim: int, base: float = 10000.0, device="cpu"):
    """LlamaRotaryEmbedding cos/sin caches (llama_xformer.py:118-135), cast to fp16 like :147-150."""
    inv_freq = 1.0 / (base ** (torch.arange(0, dim, 2, device=device).float() / dim))
    t = torch.arange(max_pos, device=device, dtype=inv_freq.dtype)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().to(torch.float16), emb.sin().to(torch.float16)


def rope_ref(x, positions, base: float = 10000.0):
    """apply_rotary_pos_emb on fp16 tensors (llama_xformer.py:138-161): x [B,H,S,D], positions [B,S]."""
    D = x.shape[-1]
    cos, sin = rope_tables(int(positions.max().item()) + 1, D, base, x.device)
    cos = cos[positions].unsqueeze(1)
    sin = sin[positions].unsqueeze(1)
    x1, x2 = x[..., : D // 2], x[..., D // 2:]
    rot = torch.cat((-x2, x1), dim=-1)
    return (x * cos) + (rot * sin)          # fp16 ops: each product and the sum are rounded to fp16
