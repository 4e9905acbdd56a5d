"""TEST INFRASTRUCTURE ONLY -- restatement of LLM.int8() (transformers `load_in_8bit=True`: bitsandbytes
Linear8bitLt with has_fp16_weights=False and llm_int8_threshold=6.0) as plain torch, the oracle of the int8 kernels.

Formulas (fp32 unless stated; rint = round half to even):
  weights       SCB[n] = max_k |W[n,k]|;  CB[n,k] = rint(W[n,k] * (127 / SCB[n])) as int8, 0 where SCB[n] == 0
  activations   (m,k) is an outlier when !(|A[m,k]| < threshold) -- NaN and +-inf are outliers; O = the columns
                holding an outlier in any row, ascending;  SCA[m] = max |A[m,k]| over the row's non-outlier elements;
                CA[m,k] = rint(A[m,k] * (127 / SCA[m])), 0 for k in O and where SCA[m] == 0
  output        acc = sum_k CA CB (exact integers);  base = fp16(((float)acc * 6.200012e-05) * SCA[m] * SCB[n]);
                O empty: y = base;  else subB[n,j] = fp16(CB[n,j] * SCB[n] / 127),
                corr = fp16(sum over j in O, ascending, of A[m,j] * subB[n,j] accumulated in fp32), y = fp16(base + corr)
  after         residual: fp16(r + y);  SiLU-gate (W rows in blocks of [128 gate | 128 up]): fp16(fp16(silu(g)) * u)
The 6.200012e-05 is bitsandbytes' MM_DEQUANT_CONST (1/127^2).  bitsandbytes itself is not used or installed; where
this restates its arithmetic from memory, the formulas above are the contract the kernels are held to.

The GPU's SiLU uses the ex2/rcp approximations of the fp16 GEMM epilogue, so silu_gate() here is exact sigmoid and
the tests compare mode 1 within one fp16 rounding of silu(g) (modes 0 and residual are compared bit for bit).
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional

import torch
import torch.nn.functional as F

from oracle import restatement as R

DEQUANT = 6.200012e-05


def quantize_weight(w: torch.Tensor):
    """fp16 [N,K] -> (CB int8 [N,K], SCB fp32 [N])"""
    wf = w.float()
    scb = wf.abs().amax(dim=1)
    inv = torch.tensor(127.0, dtype=torch.float32) / scb
    q = torch.round(wf * inv[:, None])
    q = torch.where((scb == 0)[:, None], torch.zeros_like(q), q)
    return q.to(torch.int8), scb


def quantize_act(a: torch.Tensor, threshold: float = 6.0):
    """fp16 [M,K] -> (CA int8 [M,K], SCA fp32 [M], O int64 [|O|] ascending)"""
    af = a.float()
    outl = ~(af.abs() < threshold)
    cols = outl.any(dim=0)
    sca = af.abs().masked_fill(outl, 0.0).amax(dim=1)
    inv = torch.tensor(127.0, dtype=torch.float32) / sca
    q = torch.round(af * inv[:, None])
    zero = cols[None, :] | (sca == 0)[:, None]
    q = torch.where(zero, torch.zeros_like(q), q)
    return q.to(torch.int8), sca, torch.nonzero(cols).flatten()


def linear8_parts(a: torch.Tensor, cb: torch.Tensor, scb: torch.Tensor, threshold: float = 6.0) -> torch.Tensor:
    """y = the fp16 LLM.int8() output of nn.Linear(a) before any residual / gate (see the module docstring)"""
    ca, sca, O = quantize_act(a, threshold)
    acc = (ca.double() @ cb.double().t()).to(torch.int64)        # exact: |acc| < 2^31
    base = ((acc.float() * DEQUANT) * sca[:, None]) * scb[None, :]
    base = base.half()
    if O.numel() == 0:
        return base
    sub = ((cb[:, O].float() * scb[:, None]) / 127.0).half().float()    # [N, |O|]
    af = a.float()
    corr = torch.zeros(base.shape, dtype=torch.float32)
    for i, j in enumerate(O.tolist()):                  # ascending, one fp32 rounding per term
        corr = corr + af[:, j:j + 1] * sub[:, i][None, :]
    return (base.float() + corr.half().float()).half()


def silu_gate(y: torch.Tensor) -> torch.Tensor:
    """[M, N] fp16 with columns in blocks of [128 gate | 128 up] -> fp16(fp16(silu(gate)) * up) [M, N/2]"""
    M, N = y.shape
    blk = y.float().view(M, N // 256, 2, 128)
    g, u = blk[:, :, 0], blk[:, :, 1]
    s = (g * torch.sigmoid(g)).half().float()
    return (s * u).half().reshape(M, N // 2)


def linear8(a: torch.Tensor, cb: torch.Tensor, scb: torch.Tensor, threshold: float = 6.0,
            residual: Optional[torch.Tensor] = None, mode: int = 0) -> torch.Tensor:
    y = linear8_parts(a.cpu(), cb.cpu(), scb.cpu(), threshold)
    if mode == 1:
        return silu_gate(y)
    if residual is not None:
        y = (residual.cpu().float() + y.float()).half()
    return y


def interleave_gate_up(g: torch.Tensor, u: torch.Tensor) -> torch.Tensor:
    """rows of gate and up in the fused [128 gate | 128 up] block layout (dim 0)"""
    n = g.shape[0] // 128
    return torch.stack([g.reshape(n, 128, *g.shape[1:]), u.reshape(n, 128, *u.shape[1:])], 1).reshape(2 * g.shape[0],
                                                                                                    *g.shape[1:])


def _rms16(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """LlamaRMSNorm in fp16 mode: fp32 normalise, round to fp16, multiply by the fp16 weight, round"""
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return ((xf * rstd).half().float() * w.float()).half()


def llama_forward8(sd, input_ids: torch.Tensor, heads: int, layers: int, eps: float = 1e-6,
                   threshold: float = 6.0, outlier_counts: Optional[List[int]] = None):
    """LLaMA forward (oracle/restatement.py llama_forward's structure) with fp16 activations between the ops and every
    decoder linear as linear8 -- the int8 model's oracle.  Returns fp16 logits [B,S,V]; outlier_counts (if given)
    receives |O| of each layer's q/k/v input."""
    B, S = input_ids.shape
    x = F.embedding(input_ids, sd["model.embed_tokens.weight"]).half()
    h = x.shape[-1]
    D = h // heads
    pos = torch.arange(S).unsqueeze(0).expand(B, S)
    q8 = {}
    for k, v in sd.items():
        if k.endswith(".weight") and ".layers." in k and k.split(".")[-2] in (
                "q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj"):
            q8[k] = quantize_weight(v.half())

    def lin(t, name, residual=None):
        cb, scb = q8[name]
        return linear8(t.reshape(-1, t.shape[-1]), cb, scb, threshold,
                       None if residual is None else residual.reshape(-1, residual.shape[-1])).view(*t.shape[:-1], -1)

    for l in range(layers):
        p = f"model.layers.{l}."
        n = _rms16(x, sd[p + "input_layernorm.weight"].half(), eps)
        if outlier_counts is not None:
            outlier_counts.append(int(quantize_act(n.reshape(-1, h), threshold)[2].numel()))
        q = lin(n, p + "self_attn.q_proj.weight").view(B, S, heads, D).transpose(1, 2).float()
        k = lin(n, p + "self_attn.k_proj.weight").view(B, S, heads, D).transpose(1, 2).float()
        v = lin(n, p + "self_attn.v_proj.weight").view(B, S, heads, D).transpose(1, 2).float()
        q, k = R._rope(q, k, pos)
        q, k = q.half().float(), k.half().float()
        scores = (q @ k.transpose(-1, -2)) / math.sqrt(D)
        i = torch.arange(S)[:, None]
        j = torch.arange(S)[None, :]
        scores = scores.masked_fill(j > i, float("-inf"))
        a = (torch.softmax(scores, dim=-1) @ v).transpose(1, 2).reshape(B, S, h).half()
        x = lin(a, p + "self_attn.o_proj.weight", residual=x)
        n = _rms16(x, sd[p + "post_attention_layernorm.weight"].half(), eps)
        g = lin(n, p + "mlp.gate_proj.weight")
        u = lin(n, p + "mlp.up_proj.weight")
        m = ((g.float() * torch.sigmoid(g.float())).half().float() * u.float()).half()
        x = lin(m, p + "mlp.down_proj.weight", residual=x)
    hidden = _rms16(x, sd["model.norm.weight"].half(), eps)
    return (hidden.float() @ sd["lm_head.weight"].half().float().t()).half()
