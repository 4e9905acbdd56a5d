"""Shared helpers of the kernel edge tests (test_kernel_edges_gpu.py, test_decode_edges_gpu.py): fp16 ulps, the
elementwise bound check, the derived GEMM / SiLU-gate / norm bounds against float64 references that keep the
reference's fp16 rounding points (oracle/ops_ref.py with dtype=torch.float64), and sentinel-guarded buffers."""
import torch
import torch.nn.functional as F

from oracle import ops_ref as R

DEV = "cuda"
F64 = torch.float64
U24 = 2.0 ** -24          # unit roundoff of fp32
SENTINEL = 0x7E5A         # an fp16 NaN with a payload no kernel produces: guard words must keep exactly these bits
NAN = float("nan")


def rand16(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.float16).to(DEV)


def ulp16(x):
    """spacing of the fp16 numbers at |x| (2^-24 in the subnormal range, 32 at the top of the finite range)"""
    x = x.to(F64).abs()
    return torch.pow(2.0, torch.floor(torch.log2(x.clamp(2.0 ** -14, 65504.0))) - 10)


def violations(out, ref, tol):
    """(number of elements of `out` outside ref +- tol, description of the first).  Where the reference is not finite
    the output must be the same infinity, or NaN."""
    o, r = out.to(F64), ref.to(F64)
    fin = torch.isfinite(r)
    same = (o == r) | (torch.isnan(o) & torch.isnan(r))
    bad = torch.where(fin, ~((o - r).abs() <= tol), ~same)
    n = int(bad.sum())
    if n == 0:
        return 0, ""
    i = tuple(int(v) for v in bad.nonzero()[0])
    tol_i = tol[i].item() if torch.is_tensor(tol) and tol.dim() > 0 else float(tol)
    return n, f"{n}/{bad.numel()} outside the bound; first at {i}: out {o[i].item()!r} ref {r[i].item()!r} tol {tol_i:.3e}"


def check16(out, ref, tol, what=""):
    n, msg = violations(out, ref, tol)
    assert n == 0, f"{what}: {msg}"


def gemm_tol(a, w, mags, roundings=1, lip=1.0, extra=0.0, bias=None):
    """Elementwise bound on |out - ref64| of a GEMM and its epilogue chain, ref64 = the float64 reference with the
    same fp16 rounding points (`mags` = the reference and every fp16 intermediate on the way):

        tol = lip * (ulp16(m) + (K + 1) 2^-23 (|a| @ |w|^T + |bias|)) + (roundings - 1) ulp16(m) + extra
        m   = max(|t| for t in mags)

    * the fp32 accumulator differs from the exact dot product by at most K 2^-23 sum_k |a_k w_k|: K fp32 additions,
      each off by at most 2 units of roundoff (truncating hardware included), one more for the bias add.  Unlike a
      count of ulps of |ref|, this stays valid when the sum cancels;
    * both sides then round to fp16 at the same points, at most half an ulp each: one ulp of the largest magnitude
      per rounding point;
    * an activation between two rounding points scales the error before it by its Lipschitz constant `lip`;
    * `extra` is the kernel's own error in evaluating the activation (act_extra)."""
    ab = a.to(F64).abs() @ w.to(F64).abs().t()
    if bias is not None:
        ab = ab + bias.to(F64).abs()
    acc = (a.shape[1] + 1) * 2.0 ** -23 * ab
    m = torch.zeros_like(acc)
    for t in mags:
        m = torch.maximum(m, t.to(F64).abs())
    u = ulp16(m)
    return lip * (u + acc) + (roundings - 1) * u + extra


def act_extra(act, pre):
    """the epilogue's error in evaluating the activation at the fp16 pre-activation `pre`:
    GELU = 0.5 (x + |x| erf(|x|/sqrt2)) with erf from Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7), 1 - p e rounded
    to fp32 next to 1 (<= 3e-8) and approximate reciprocal / exp2 on p e <= 1 (<= 3.2e-7): at most
    0.5 |x| (1.5e-7 + 3e-8 + 3.2e-7) <= 2.5e-7 |x|.  Negligible against an fp16 ulp for x > -3, up to ~10 ulps
    near x = -5, where GELU(x) ~ -1e-6 (test_activation_epilogue_over_every_fp16_input measures it).
    tanhf: 2 fp32 ulps of |tanh| <= 1.  ReLU and identity: exact."""
    if act == 1:
        return 2.5e-7 * pre.to(F64).abs()
    if act == 2:
        return 2.4e-7
    return 0.0


def in_buffer(t, pad_cols, pad_rows, fill=NAN, dtype=torch.float16):
    """-> (buffer, view): t [r, c] copied into the top-left of an [r + pad_rows, c + pad_cols] buffer of `fill`"""
    r, c = t.shape
    buf = torch.full((r + pad_rows, c + pad_cols), fill, dtype=dtype, device=DEV)
    buf[:r, :c] = t
    return buf, buf[:r, :c]


def bit_diff(a, b):
    """"" when the fp16 tensors hold identical bits (any NaN matching any NaN: payloads are not part of any contract),
    else the number of differing elements and the first of them"""
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    bad = (na != nb) | (~na & ~nb & (a.view(torch.int16) != b.view(torch.int16)))
    if not bad.any():
        return ""
    i = tuple(int(v) for v in bad.nonzero()[0])
    return f"{int(bad.sum())}/{bad.numel()} differ; first at {i}: {a[i].item()!r} vs {b[i].item()!r}"


def sentinel_buffer(rows, cols):
    return torch.full((rows, cols), SENTINEL, dtype=torch.int16, device=DEV).view(torch.float16)


def assert_guards(buf, written, what=""):
    """every word of `buf` outside the boolean mask `written` still holds the sentinel bits"""
    bits = buf.view(torch.int16)
    bad = (bits != SENTINEL) & ~written
    assert not bad.any(), f"{what}: {int(bad.sum())} guard words overwritten, first at {tuple(bad.nonzero()[0].tolist())}"


def region(buf, rows, cols):
    m = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
    m[:rows, :cols] = True
    return m


def up8(n):
    return (n + 7) // 8 * 8


def silu_gate_tol(a, wg, wu, ref, silu_rel=None, a_err=None):
    """bound of the SiLU-gate epilogue (derived in test_gemm_silu_gate_padded_out).  silu_rel(g): the kernel's
    relative error in silu (default 1.5e-6, the GEMM epilogue's); a_err: an elementwise bound on the error of the
    kernel's fp16 operand `a` (a folded RMSNorm), which adds a_err @ |w|^T to the gate and up accumulators."""
    g = R.linear_ref(a, wg, dtype=F64).to(F64)
    u = R.linear_ref(a, wu, dtype=F64).to(F64)
    s = R.r16(F.silu(g))
    eg = gemm_tol(a, wg, (g,)) - ulp16(g)
    eu = gemm_tol(a, wu, (u,)) - ulp16(u)
    if a_err is not None:
        eg = eg + a_err @ wg.to(F64).abs().t()
        eu = eu + a_err @ wu.to(F64).abs().t()
    xs = (1.5e-6 if silu_rel is None else silu_rel(g)) * s.abs()
    return (u.abs() * (1.1 * (ulp16(g) + eg) + ulp16(s) + xs) + (s.abs() + ulp16(s)) * (ulp16(u) + eu)
            + ulp16(ref))


# Statistics bound: a thread adds 8 VPT <= 64 values, then 5 shuffle levels and <= 8 warp partials: <= 77 fp32
# additions, so |error of a sum| <= 77 2^-24 sum|terms| < 4.6e-6 sum|terms|.  The mean is then off by < 4.6e-6 mean|x|,
# the two-pass variance by < 4.6e-6 var (+ (mean error)^2), rstd by < 2.3e-6 + rsqrtf's 2^-22: both below
# ST = 2^-16 (1.5e-5) relative to mean|x| and rstd.
ST = 2.0 ** -16                # relative error of the row statistics (mean, rstd)


def norm_bounds(kind, x, w, b, eps):
    """(ref, tol).  LayerNorm y = fp16((x - mean) rstd w + b):
         tol = ulp16(max(|y|, |ref|)) + ST rstd |w| (|x - mean| + mean|x|) + 4 2^-24 (|x - mean| rstd |w| + |b|)
       (statistics error, then 4 fp32 operations).  RMSNorm h = fp16(x rstd), y = fp16(h w):
         tol = |w| (ulp16(h) + ST |x| rstd) + ulp16(max(|y|, |ref|))"""
    xd = x.to(F64)
    if kind == "ln":
        ref = R.layernorm_ref(x, w, b, eps, dtype=F64)
        mean = xd.mean(-1, keepdim=True)
        rstd = torch.rsqrt(xd.var(-1, unbiased=False, keepdim=True) + eps)
        core = (xd - mean).abs() * rstd * w.to(F64).abs()
        tol = (ulp16(ref.to(F64).abs() + core * ST * 4) + ST * rstd * w.to(F64).abs() * ((xd - mean).abs() + xd.abs().mean(-1, keepdim=True))
               + 4 * U24 * (core + b.to(F64).abs()))
    else:
        ref = R.rmsnorm_ref(x, w, eps, dtype=F64)
        rstd = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
        h = xd * rstd
        tol = w.to(F64).abs() * (ulp16(h) + ST * h.abs()) + ulp16(ref.to(F64).abs() + ST * 4 * (h * w.to(F64)).abs())
    return ref, tol
