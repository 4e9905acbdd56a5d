"""Torch restatement of the LoRA arithmetic in include/seedb200.h (PEFT lora.Linear.forward, fp16 module, eval mode):

    base = fp16(W x)                      the linear's kernel
    t    = fp16(A x)                      fp32 accumulation
    u    = fp16(B t)                      fp32 accumulation over r
    c    = fp16(float(u) * float32(s))
    y    = fp16(base + c)

then the layer's epilogue step on y (residual add, or the SiLU gate).  Merge: W' = fp16(W + fp16(fp16(B A) * s)).
Sums are taken in float64 and rounded once.  A kernel that sums in fp32 differs by up to one fp16 ulp plus the fp32
summation error (sum_bound), which exceeds an ulp where the terms cancel; that difference then passes through the
later rounding points.
"""
import torch


def fp16(x):
    return x.to(torch.float16)


def shrink(x, a):
    """t = fp16(x . a^T) from fp16 x [M, K] and a [r, K]"""
    return fp16(x.double() @ a.double().T)


def expand(base, t, b, s):
    """y = fp16(base + fp16(fp16(b . t) * s)) from the kernel's own base [M, N] and t [M, r]"""
    u = fp16(t.double() @ b.double().T)
    c = fp16(u.float() * torch.tensor(s, dtype=torch.float32))
    return fp16(base.float() + c.float())


def linear(x, w, a, b, s):
    """the whole LoRA linear from fp16 operands"""
    return expand(fp16(x.double() @ w.double().T), shrink(x, a), b, s)


def silu_gate(g, u):
    """silu(fp16 gate) rounded to fp16, times fp16 up, rounded (llama_xformer.py:186)"""
    g = g.float()
    return fp16(fp16(g * torch.sigmoid(g)).float() * u.float())


def merge(w, a, b, s):
    d = fp16(fp16(b.double() @ a.double()).float() * torch.tensor(s, dtype=torch.float32))
    return fp16(w.float() + d.float())


def sum_bound(abs_sum, n):
    """error bound of an n-term fp32 sum, sum of |terms| = abs_sum (fp16 products are exact in fp32): n * 2^-24 * abs_sum.
    Where the terms cancel, this exceeds an ulp of the fp16 result."""
    return n * 2.0 ** -24 * abs_sum


def shrink_bound(x, a):
    """|kernel t - shrink(x, a)| <= this: one rounding plus the fp32 summation error"""
    ref = shrink(x, a)
    return ulp(ref) + sum_bound(x.double().abs() @ a.double().abs().T, x.shape[1])


def ulp(x):
    """fp16 spacing at |x| (normal range; subnormal spacing below)"""
    x = x.double().abs().clamp(min=2.0 ** -14)
    return 2.0 ** (torch.floor(torch.log2(x)) - 10)
