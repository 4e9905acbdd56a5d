"""Edge cases of the GEMM, attention and row kernels against float64 references that keep the reference's fp16
rounding points (oracle/ops_ref.py with dtype=torch.float64): operands that are views into larger NaN-filled buffers,
outputs inside sentinel buffers, K below one k-block, every tile width and epilogue, exact NaN-dependency probes, the
ends of the fp16 range, every attention dispatch variant and every row-kernel instantiation at both ends of its width
range.

Every bound is derived where it is built.  Each kind of bound has a negative control: the same check must reject a
reference computed with the last 8 reduction columns dropped, or with one row shifted, so a bound too loose to see
such an error fails its own test."""
import ctypes as C
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import ops_ref as R

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from edge_ref import (DEV, F64, NAN, SENTINEL, ST, U24, act_extra, assert_guards, check16, gemm_tol,  # noqa: E402
                      in_buffer, norm_bounds, rand16, region, sentinel_buffer, silu_gate_tol, ulp16, up8,
                      violations)

pytestmark = pytest.mark.gpu
BNS = (32, 64, 128, 176, 192, 256)
LIP = {0: 1.0, 1: 1.13, 2: 1.0, 3: 1.0}   # Lipschitz constants of identity, GELU (max slope 1.129), tanh, ReLU


def linear_bound(a, w, bias=None, act=0, residual=None):
    """(ref64, tol) of out = fp16(fp16(act(fp16(a w^T + bias))) + residual)"""
    pre = R.linear_ref(a, w, bias, dtype=F64)
    post = R.linear_ref(a, w, bias, act, dtype=F64)
    ref = R.linear_ref(a, w, bias, act, residual, dtype=F64)
    mags = (ref, pre, post) + ((residual,) if residual is not None else ())
    n = 1 + (act != 0) + (residual is not None)
    return ref, gemm_tol(a, w, mags, n, LIP[act], act_extra(act, pre), bias)


# ----------------------------------------------------------------------------------------------
# GEMM: operand views with guard bands, a pairwise cover of tile width x K x M x N tail
# ----------------------------------------------------------------------------------------------
KS = (8, 16, 24, 32, 40, 56, 72, 592)
MS = (1, 63, 64, 65, 129, 257)
VIEW_CASES = [(bn, K, MS[(ib + ik) % 6], (ik + ib // 3) % 2, (ib + ik) % 4)
              for ib, bn in enumerate(BNS) for ik, K in enumerate(KS)]


def view_case_n(bn, K, tail):
    n = bn * (1 + KS.index(K) % 2)
    return n - 13 if tail else n          # odd N: the last column of the last tile is a single-half store


@pytest.mark.parametrize("bn,K,M,tail,act", VIEW_CASES)
def test_gemm_views_and_guard_bands(lib, bn, K, M, tail, act):
    """A, W and the residual are views whose padding columns and trailing rows hold NaN (any read of them reaches the
    output); out is a view into a sentinel buffer with ldo > N (any write outside [M, N] shows)"""
    N = view_case_n(bn, K, tail)
    seed = bn * 1000 + K
    _, a = in_buffer(rand16(M, K, seed=seed), 8 * (1 + K % 3), 5)
    _, w = in_buffer(rand16(N, K, scale=K ** -0.5, seed=seed + 1), 8 * (1 + bn % 3), 7)
    _, res = in_buffer(rand16(M, N, seed=seed + 2), up8(N) - N + 16, 3)
    bias = rand16(N, scale=0.5, seed=seed + 3) if (bn // 16 + K // 8) % 2 else None
    obuf = sentinel_buffer(M + 2, up8(N) + 8)
    out = obuf[:M, :N]
    lib.gemm(a, w, bias=bias, act=act, residual=res, out=out, bn=bn)
    torch.cuda.synchronize()
    ref, tol = linear_bound(a, w, bias, act, res)
    check16(out, ref, tol, f"gemm view bn={bn} K={K} M={M} N={N} act={act}")
    assert_guards(obuf, region(obuf, M, N), "gemm out")


@pytest.mark.parametrize("mode", [0, 1])
def test_gemm_zero_leading_dimensions_mean_packed_rows(lib, mode):
    """a descriptor with lda = ldw = ldo = ldr = 0 (zero-initialised) runs on packed rows: bit-identical to the same
    call with explicit leading dimensions"""
    M, N, K = 70, 512, 40
    a = rand16(M, K, seed=31)
    w = rand16(N, K, scale=K ** -0.5, seed=32)
    res = rand16(M, N, seed=33) if mode == 0 else None
    n_out = N // 2 if mode == 1 else N
    want = lib.gemm(a, w, residual=res, mode=mode)
    out = torch.full((M, n_out), NAN, dtype=torch.float16, device=DEV)
    d = lib.GemmDesc()
    d.M, d.N, d.K, d.mode = M, N, K, mode
    d.A, d.W, d.out = a.data_ptr(), w.data_ptr(), out.data_ptr()
    d.residual = None if res is None else res.data_ptr()
    lib.check(lib.load().seedb200_gemm(C.byref(d), lib.stream_ptr()), "seedb200_gemm")
    torch.cuda.synchronize()
    assert torch.equal(out, want)


def test_gemm_bound_rejects_a_wrong_reference(lib):
    """negative control of gemm_tol: the K = 8 GEMM's reference without its last 8 columns (all of K), the K = 592
    one's without its last 8, and a reference shifted by one row, all fail the check"""
    for K in (8, 592):
        a = rand16(65, K, seed=5)
        w = rand16(96, K, scale=K ** -0.5, seed=6)
        bias = rand16(96, scale=0.5, seed=7)
        out = lib.gemm(a, w, bias=bias, act=1, bn=64)
        ref, tol = linear_bound(a, w, bias, 1)
        check16(out, ref, tol, "control baseline")
        short, _ = linear_bound(a[:, :K - 8], w[:, :K - 8], bias, 1)
        assert violations(out, short, tol)[0] > 0, K
        assert violations(out, torch.roll(ref, 1, 0), tol)[0] > 0, K


# ----------------------------------------------------------------------------------------------
# GEMM epilogue matrix at a tail shape, for each tile width
# ----------------------------------------------------------------------------------------------
EPILOGUES = ("bias_act", "residual", "inplace", "ln_fold", "row_moments", "row_remap")


@pytest.mark.parametrize("variant", EPILOGUES)
@pytest.mark.parametrize("bn", BNS)
def test_gemm_epilogue_matrix(lib, bn, variant):
    M, K = 129, 200                                        # M tail, 3 full k-blocks + an 8-column tail
    N = bn + 64 if variant == "row_moments" else bn + 40   # the last tile reaches past N
    if variant == "row_moments" and bn % 64:
        pytest.skip("row moments need 64-column groups inside every tile (refused for this width)")
    seed = bn + 17 * EPILOGUES.index(variant)
    a = rand16(M, K, seed=seed)
    w = rand16(N, K, scale=K ** -0.5, seed=seed + 1)
    bias = rand16(N, scale=0.5, seed=seed + 2)
    what = f"bn={bn} {variant}"
    if variant == "bias_act":
        for act in range(4):
            ref, tol = linear_bound(a, w, bias, act)
            check16(lib.gemm(a, w, bias=bias, act=act, bn=bn), ref, tol, f"{what} act={act}")
    elif variant == "residual":
        _, res = in_buffer(rand16(M, N, seed=seed + 3), 24, 2)
        ref, tol = linear_bound(a, w, bias, 2, res)
        check16(lib.gemm(a, w, bias=bias, act=2, residual=res, bn=bn), ref, tol, what)
    elif variant == "inplace":
        obuf = sentinel_buffer(M + 1, N + 16)
        x = obuf[:M, :N]
        x.copy_(rand16(M, N, seed=seed + 3))
        ref, tol = linear_bound(a, w, bias, 0, x.clone())
        lib.gemm(a, w, bias=bias, residual=x, out=x, bn=bn)
        torch.cuda.synchronize()
        check16(x, ref, tol, what)
        assert_guards(obuf, region(obuf, M, N), what)
    elif variant == "ln_fold":
        _check_ln_fold(lib, a, w, bias, bn, seed)
    elif variant == "row_moments":
        res = rand16(M, N, seed=seed + 3)
        mbuf = torch.full((M + 1, N // 64, 2), NAN, dtype=torch.float32, device=DEV)
        out = lib.gemm(a, w, bias=bias, residual=res, bn=bn, row_moments=mbuf[:M])
        torch.cuda.synchronize()
        ref, tol = linear_bound(a, w, bias, 0, res)
        check16(out, ref, tol, what)
        # per 64-column group each thread adds 16 values, then 2 shuffle levels: <= 18 fp32 additions
        g = out.to(F64).view(M, N // 64, 64)
        for i, (want, mag) in enumerate(((g.sum(-1), g.abs().sum(-1)), ((g * g).sum(-1), (g * g).sum(-1)))):
            got = mbuf[:M, :, i].to(F64)
            assert ((got - want).abs() <= 18 * U24 * mag + 1e-30).all(), (what, i, (got - want).abs().max().item())
        assert torch.isnan(mbuf[M]).all(), "row moments written behind the last row"
    elif variant == "row_remap":
        # out row (m // 64) * 67 + m % 64 + 2, residual row m % 50 + 3 (the patch-embedding remap, other numbers)
        rg, rs, ro, rm, rof = 64, 67, 2, 50, 3
        res_full = rand16(rm + rof + 2, N, seed=seed + 3)
        rows = torch.arange(M, device=DEV)
        orow = (rows // rg) * rs + rows % rg + ro
        obuf = sentinel_buffer(int(orow.max()) + 3, N + 8)
        lib.gemm(a, w, bias=bias, act=3, residual=res_full, out=obuf[:, :N], bn=bn, row_group=rg, row_stride=rs,
                 row_offset=ro, res_mod=rm, res_offset=rof)
        torch.cuda.synchronize()
        ref, tol = linear_bound(a, w, bias, 3, res_full[rows % rm + rof])
        check16(obuf[orow, :N], ref, tol, what)
        written = torch.zeros(obuf.shape, dtype=torch.bool, device=DEV)
        written[orow, :N] = True
        assert_guards(obuf, written, what)


def _check_ln_fold(lib, a_unused, w, bias, bn, seed):
    """linear(LayerNorm(x)) through the folded epilogue against the rounding-point reference (LN(x) rounded to fp16,
    then the GEMM).  On top of gemm_tol for (fp16 LN(x), W):
    * the two sides round different operands (LN(x) there, W gamma here): at most 2^-11 (|xhat| @ |W gamma|^T) each;
    * the kernel accumulates the un-normalised rows, W' x, and cancels mean * c afterwards:
      (K + 2) 2^-23 rstd (|x| @ |W'|^T + |mean| sum|W'|) of fp32 error;
    * fp32 (mean, rstd) from row_stats: relative error below 2^-16 each (see test_row_kernels_at_every_instantiation),
      2^-16 rstd (|x - mean| @ |W'|^T + |mean| sum|W'|) in all."""
    M, K = a_unused.shape
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, K, generator=g) * 1.5 + 0.5 * torch.randn(M, 1, generator=g)).half().to(DEV)
    gamma = (1.0 + 0.2 * torch.randn(K, generator=g)).half().to(DEV)
    beta = (0.1 * torch.randn(K, generator=g)).half().to(DEV)
    wf, c, bf = lib.ln_fold_weights(w, gamma, beta, bias)
    for act in (0, 1):
        out = lib.gemm(x, wf, act=act, bn=bn, ln=(lib.row_stats(x, 1e-6), c, bf))
        xh = R.layernorm_ref(x, gamma, beta, 1e-6, dtype=F64)
        ref, tol = linear_bound(xh, w, bias, act)
        xd = x.to(F64)
        mean = xd.mean(-1, keepdim=True)
        rstd = torch.rsqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-6)
        wfa = wf.to(F64).abs()
        xhat = ((xd - mean) * rstd).abs()
        fold = (2.0 ** -10 * (xhat @ (w.to(F64) * gamma.to(F64)).abs().t())
                + (K + 2) * 2.0 ** -23 * rstd * (xd.abs() @ wfa.t() + mean.abs() * wfa.sum(-1))
                + 2.0 ** -16 * rstd * ((xd - mean).abs() @ wfa.t() + mean.abs() * wfa.sum(-1)))
        check16(out, ref, tol + LIP[act] * fold, f"bn={bn} ln_fold act={act}")


@pytest.mark.parametrize("M", [1, 65, 300])
def test_gemm_silu_gate_padded_out(lib, M):
    """mode 1 into a view with ldo > N/2 inside a sentinel buffer.  Bound: g = fp16(gate), s = fp16(silu(g)),
    out = fp16(s u); with eg, eu the accumulator bounds of gate / up and L(silu) <= 1.1:
    |out - ref| <= |u| (1.1 (ulp(g) + eg) + ulp(s) + xs) + (|s| + ulp(s)) (ulp(u) + eu) + ulp(out), xs the kernel's own
    error in silu (see test_activation_epilogue_over_every_fp16_input)."""
    ffn, K = 512, 136
    a = rand16(M, K, seed=M)
    wg = rand16(ffn, K, scale=K ** -0.5 * 3, seed=M + 1)
    wu = rand16(ffn, K, scale=K ** -0.5, seed=M + 2)
    obuf = sentinel_buffer(M + 1, ffn + 24)
    out = obuf[:M, :ffn]
    lib.gemm(a, R.interleave_gate_up(wg, wu), mode=1, out=out)
    torch.cuda.synchronize()
    ref = R.silu_gate_ref(a, wg, wu, dtype=F64)
    check16(out, ref, silu_gate_tol(a, wg, wu, ref), f"silu gate M={M}")
    assert_guards(obuf, region(obuf, M, ffn), "silu gate")


# ----------------------------------------------------------------------------------------------
# dependency probes: one NaN in an operand must reach exactly its output row / column
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bn", BNS)
def test_gemm_nan_probes_reach_exactly_their_row_and_column(lib, bn):
    """a swizzle or tile-boundary addressing error moves an operand element to another row / column / k: a single NaN
    then shows up elsewhere, or nowhere"""
    M, N, K = 200, 2 * bn + 24, 136
    a0 = rand16(M, K, seed=bn)
    w0 = rand16(N, K, scale=K ** -0.5, seed=bn + 1)
    for i in (0, 63, 64, 127, M - 1):
        for k in (0, 63, 64, K - 1):
            a = a0.clone()
            a[i, k] = NAN
            bad = ~torch.isfinite(lib.gemm(a, w0, bn=bn).float())
            rows = bad.any(1).nonzero().flatten().tolist()
            assert rows == [i] and bool(bad[i].all()), (bn, "A", i, k, rows)
    for j in sorted({0, 63, 64, bn - 1, bn, N - 1}):
        for k in (0, 64, K - 1):
            w = w0.clone()
            w[j, k] = NAN
            bad = ~torch.isfinite(lib.gemm(a0, w, bn=bn).float())
            cols = bad.any(0).nonzero().flatten().tolist()
            assert cols == [j] and bool(bad[:, j].all()), (bn, "W", j, k, cols)


def test_gemm_silu_gate_nan_probes(lib):
    """mode 1: W row r is gate (r % 256 < 128) or up of output column (r // 256) * 128 + r % 128"""
    M, ffn, K = 130, 512, 72
    a = rand16(M, K, seed=3)
    wgu = R.interleave_gate_up(rand16(ffn, K, scale=0.1, seed=4), rand16(ffn, K, scale=0.1, seed=5))
    for r in (0, 127, 128, 255, 256, 383, 2 * ffn - 1):
        w = wgu.clone()
        w[r, K - 1] = NAN
        bad = ~torch.isfinite(lib.gemm(a, w, mode=1).float())
        cols = bad.any(0).nonzero().flatten().tolist()
        assert cols == [(r // 256) * 128 + r % 128] and bool(bad[:, cols[0]].all()), (r, cols)
    for i in (0, 64, M - 1):
        x = a.clone()
        x[i, 0] = NAN
        bad = ~torch.isfinite(lib.gemm(x, wgu, mode=1).float())
        assert bad.any(1).nonzero().flatten().tolist() == [i]


@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_gemm_nan_propagation_matches_torch(lib, act):
    """NaN operands, a NaN bias entry and a NaN residual entry leave NaN exactly where torch's ops do
    (torch.relu(nan) is nan, so ReLU must not use fmaxf)"""
    M, N, K = 70, 96, 40
    a = rand16(M, K, seed=act)
    w = rand16(N, K, scale=K ** -0.5, seed=act + 1)
    bias = rand16(N, scale=0.5, seed=act + 2)
    res = rand16(M, N, seed=act + 3)
    a[3, 5] = NAN
    w[40, 39] = NAN
    bias[7] = NAN
    res[66, 90] = NAN
    out = lib.gemm(a, w, bias=bias, act=act, residual=res, bn=64)
    ref = R.linear_ref(a, w, bias, act, res, dtype=F64)
    assert torch.equal(torch.isnan(out), torch.isnan(ref)), (act, int((torch.isnan(out) ^ torch.isnan(ref)).sum()))
    fin = ~torch.isnan(ref)
    _, tol = linear_bound(a.nan_to_num(), w.nan_to_num(), bias.nan_to_num(), act, res.nan_to_num())
    check16(out[fin], ref[fin], tol[fin], f"finite part act={act}")


def test_gemm_silu_gate_nan_propagation_matches_torch(lib):
    M, ffn, K = 40, 256, 64
    a = rand16(M, K, seed=9)
    wg, wu = rand16(ffn, K, scale=0.2, seed=10), rand16(ffn, K, scale=0.2, seed=11)
    a[5, 3] = NAN
    wg[17, 0] = NAN
    wu[200, 63] = NAN
    out = lib.gemm(a, R.interleave_gate_up(wg, wu), mode=1)
    ref = R.silu_gate_ref(a, wg, wu, dtype=F64)
    assert torch.equal(torch.isnan(out), torch.isnan(ref))


# ----------------------------------------------------------------------------------------------
# fp16 range: overflow to inf, and the activation epilogue over every fp16 input in [-12, 12]
# ----------------------------------------------------------------------------------------------
def test_gemm_overflow_stores_inf_like_the_reference(lib):
    """accumulators past the fp16 range: 65519 rounds to 65504, 65520 and beyond to inf (the reference stores the
    fp32 result of F.linear as fp16); inf then goes through the activation and the residual add"""
    targets = [(65504, 0), (65504, 15), (65504, 16), (65504, 4496), (65504, 34496), (-65504, -16), (-65504, -34496),
               (1, 0)]
    M, N, K = len(targets), 40, 16
    a = torch.zeros(M, K, dtype=torch.float16, device=DEV)
    for m, (hi, lo) in enumerate(targets):
        a[m, 0], a[m, 1] = hi, lo
    w = torch.zeros(N, K, dtype=torch.float16, device=DEV)
    w[:, 0] = w[:, 1] = 1
    w[1::2, :2] = -1                                       # odd columns see the negated sums
    res = rand16(M, N, seed=12)
    res[:, 4] = float("-inf")                              # inf + -inf = NaN where the sum overflowed upwards
    for act in (0, 2, 3):
        for r in (None, res):
            out = lib.gemm(a, w, act=act, residual=r, bn=32)
            ref, tol = linear_bound(a, w, None, act, r)
            assert act == 2 or not torch.isfinite(ref[2]).all()     # the case under test is there (tanh(inf) = 1)
            check16(out, ref, tol, f"overflow act={act} residual={r is not None}")


def _all_fp16_in(lo, hi):
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    v = v[torch.isfinite(v) & (v >= lo) & (v <= hi)]
    return torch.unique(v.float()).half().to(DEV)         # +0 and -0 once


def test_activation_epilogue_over_every_fp16_input(lib):
    """out = act(x) for every fp16 x in [-12, 12] (subnormals included): A[m, 0] = x, W[:, 0] = 1, so the accumulator
    is x exactly and only the epilogue is measured.  Bound: |out - fp16(act64(x))| <= ulp16(|ref| + e) + e, e the
    kernel's own activation error (act_extra; SiLU: 1.5e-6 |silu(x)|, from ex2/rcp approximations and the fp32 rounding
    of x log2(e) with |x| <= 12).  Prints the measured GELU error below x = -3, where GELU loses relative accuracy."""
    x = _all_fp16_in(-12.0, 12.0)
    M = x.numel()
    a = torch.zeros(M, 8, dtype=torch.float16, device=DEV)
    a[:, 0] = x
    w = torch.zeros(8, 8, dtype=torch.float16, device=DEV)
    w[:, 0] = 1
    xd = x.to(F64)
    exact = {1: F.gelu(xd), 2: torch.tanh(xd), 3: torch.relu(xd)}
    for act in (1, 2, 3):
        out = lib.gemm(a, w, act=act)
        torch.cuda.synchronize()
        assert (out == out[:, :1]).all()
        ref = exact[act].half()
        e = act_extra(act, x)
        check16(out[:, 0], ref, ulp16(ref.to(F64).abs() + e) + e, f"act={act} sweep")
        if act == 1:
            for lo, hi in ((-12.0, -6.0), (-6.0, -4.5), (-4.5, -3.0), (-3.0, 12.0)):
                sel = (xd >= lo) & (xd < hi)
                err = (out[:, 0].to(F64) - exact[1])[sel].abs()
                flips = (out[:, 0] != ref)[sel]
                print(f"MEASURED gelu x in [{lo}, {hi}): max |out - gelu(x)| {err.max().item():.3e} = "
                      f"{(err / ulp16(exact[1][sel])).max().item():.2f} fp16 ulps of the result; "
                      f"{int(flips.sum())}/{int(sel.sum())} results differ from fp16(gelu(x)), by at most "
                      f"{((out[:, 0].to(F64) - ref.to(F64)).abs() / ulp16(ref))[sel].max().item():.0f} ulp")
    # SiLU through mode 1: gate row = x, up row = 1
    a2 = a.clone()
    a2[:, 1] = 1
    wgu = torch.zeros(256, 8, dtype=torch.float16, device=DEV)
    wgu[:128, 0] = 1
    wgu[128:, 1] = 1
    out = lib.gemm(a2, wgu, mode=1)
    torch.cuda.synchronize()
    silu = F.silu(xd)
    e = 1.5e-6 * silu.abs()
    check16(out[:, 0], silu.half(), ulp16(silu.abs() + e) + e, "silu sweep")
    assert (out == out[:, :1]).all()


# ----------------------------------------------------------------------------------------------
# attention: every dispatch variant, strided views with NaN gaps, output into a sentinel buffer
# ----------------------------------------------------------------------------------------------
ATTN_EDGE = [
    # B, H, nq, nk, D, causal        kernel variant <DPAD, warps>
    (2, 3, 32, 63, 64, False),       # <64,2>
    (1, 2, 32, 32, 64, True),
    (1, 2, 1, 1, 64, True),
    (2, 2, 33, 65, 64, True),        # <64,4>
    (1, 3, 100, 64, 64, False),      # nq > nk
    (1, 2, 40, 1, 64, False),
    (1, 2, 64, 65, 88, False),       # <96,4>, nq <= 64
    (1, 2, 64, 64, 88, True),
    (2, 2, 65, 63, 88, False),       # <96,9>, 65 <= nq <= 288
    (1, 2, 65, 65, 88, True),
    (1, 2, 288, 300, 88, True),
    (1, 2, 288, 257, 88, False),
    (1, 2, 289, 289, 88, True),      # <96,4>, nq > 288
    (1, 2, 300, 64, 88, False),
    (1, 2, 289, 1, 88, False),
    (1, 2, 64, 64, 128, True),       # <128,4>
    (2, 2, 64, 1, 128, False),
    (1, 1, 1, 63, 128, True),
    (1, 2, 65, 65, 128, True),       # <128,8>
    (1, 2, 65, 63, 128, False),
    (1, 2, 200, 65, 128, False),
    (1, 3, 130, 300, 128, True),
]


def gapped_heads(B, H, n, D, seed):
    """[B, H, n, D] view of a [B, n + 8, H + 1, D + 8] NaN buffer: NaN after every head's D values, a NaN head after
    every token's H heads, and 8 NaN tokens after the last"""
    buf = torch.full((B, n + 8, H + 1, D + 8), NAN, dtype=torch.float16, device=DEV)
    buf[:, :n, :H, :D] = rand16(B, n, H, D, seed=seed)
    return buf[:, :n, :H, :D].permute(0, 2, 1, 3)


def attention_bound(q, k, v, scale, causal, drop_dims=0):
    """float64 softmax(scale q k^T [+ bottom-right causal mask]) v -> (o64 [B, nq, H, D], tol), per output element

        tol = (2^-10 + 2 ds) (P @ |v| + |o|) + nk 2^-23 (P @ |v|) + nk 2^-25 max|v| + ulp16(o)

    * the kernel rounds the unnormalised probabilities exp(s_j - max) <= 1 to fp16 (relative error d_j <= 2^-11) and
      divides by the sum of the rounded values, so o - o_exact = sum_j p_j (d_j - mean d)(v_j - o_exact) / (1 + mean d),
      at most 2^-10 (P @ |v| + |o|); a probability below 2^-14 is an fp16 subnormal, absolute error <= 2^-25;
    * ds = D 2^-23 scale max(|q| @ |k|^T) + 2^-23 max|scale s| bounds the fp32 error of a scaled score; it scales
      every p_j by a factor within exp(+-ds): another 2 ds (P @ |v| + |o|);
    * fp32 accumulation of P V: nk 2^-23 (P @ |v|); the fp16 store: half an ulp of o (one ulp allowed).
    `drop_dims` leaves the last head dims out of the scores (negative control)."""
    D = q.shape[-1]
    qd, kd, vd = q.to(F64), k.to(F64), v.to(F64)
    Dk = D - drop_dims
    s = (qd[..., :Dk] @ kd[..., :Dk].transpose(-1, -2)) * scale
    nq, nk = q.shape[2], k.shape[2]
    if causal:
        i = torch.arange(nq, device=DEV)[:, None]
        j = torch.arange(nk, device=DEV)[None, :]
        s = s.masked_fill(j > i + (nk - nq), float("-inf"))
    p = torch.softmax(s, -1)
    o = p @ vd
    pv = p @ vd.abs()
    ds = D * 2.0 ** -23 * scale * (qd.abs() @ kd.abs().transpose(-1, -2)).max() + 2.0 ** -23 * s[torch.isfinite(s)].abs().max()
    tol = (2.0 ** -10 + 2 * ds) * (pv + o.abs()) + nk * 2.0 ** -23 * pv + nk * 2.0 ** -25 * vd.abs().max() + ulp16(o)
    return o.permute(0, 2, 1, 3), tol.permute(0, 2, 1, 3)


def run_attention(lib, q, k, v, scale, causal):
    """seedb200_attention through a hand-built descriptor; O goes to a [B, nq, H, D + 8] sentinel buffer (o_ts > H D)"""
    B, H, nq, D = q.shape
    nk = k.shape[2]
    obuf = torch.full((B, nq, H, D + 8), SENTINEL, dtype=torch.int16, device=DEV).view(torch.float16)
    d = lib.AttnDesc()
    d.q, d.k, d.v, d.o = q.data_ptr(), k.data_ptr(), v.data_ptr(), obuf.data_ptr()
    d.q_bs, d.q_hs, d.q_ts = q.stride(0), q.stride(1), q.stride(2)
    d.k_bs, d.k_hs, d.k_ts = k.stride(0), k.stride(1), k.stride(2)
    d.v_bs, d.v_hs, d.v_ts = v.stride(0), v.stride(1), v.stride(2)
    d.o_bs, d.o_hs, d.o_ts = obuf.stride(0), obuf.stride(2), obuf.stride(1)
    d.batch, d.heads, d.nq, d.nk, d.head_dim, d.causal, d.scale = B, H, nq, nk, D, int(causal), scale
    lib.check(lib.load().seedb200_attention(C.byref(d), lib.stream_ptr()), "seedb200_attention")
    torch.cuda.synchronize()
    return obuf


def row_violations(o, o64, tol):
    """query rows (b, q, h) whose error norm exceeds the norm of the elementwise bound, i.e. whose relative error
    |o - o64| / |o64| exceeds |tol| / |o64|; -> (count, worst relative error, its bound)"""
    err = (o.to(F64) - o64).norm(dim=-1)
    err = torch.where(torch.isfinite(o.to(F64)).all(-1), err, torch.full_like(err, float("inf")))
    bound = tol.norm(dim=-1)
    nrm = o64.norm(dim=-1).clamp_min(1e-300)
    worst = torch.argmax(err / nrm)
    return int((err > bound).sum()), (err / nrm).flatten()[worst].item(), (bound / nrm).flatten()[worst].item()


@pytest.mark.parametrize("B,H,nq,nk,D,causal", ATTN_EDGE)
def test_attention_variants_on_strided_views(lib, B, H, nq, nk, D, causal):
    q = gapped_heads(B, H, nq, D, 1)
    k = gapped_heads(B, H, nk, D, 2)
    v = gapped_heads(B, H, nk, D, 3)
    scale = D ** -0.5
    obuf = run_attention(lib, q, k, v, scale, causal)
    written = torch.zeros(obuf.shape, dtype=torch.bool, device=DEV)
    written[..., :D] = True
    assert_guards(obuf, written, "attention output")
    o = obuf[..., :D]
    o64, tol = attention_bound(q, k, v, scale, causal)
    n, worst, bound = row_violations(o, o64, tol)
    assert n == 0, f"{n} query rows outside the bound; worst relative error {worst:.3e} (bound {bound:.3e})"


def test_attention_bound_rejects_a_wrong_reference(lib):
    B, H, nq, nk, D = 1, 2, 65, 130, 88
    q, k, v = (gapped_heads(B, H, n, D, s) for n, s in ((nq, 4), (nk, 5), (nk, 6)))
    o = run_attention(lib, q, k, v, D ** -0.5, True)[..., :D]
    o64, tol = attention_bound(q, k, v, D ** -0.5, True)
    assert row_violations(o, o64, tol)[0] == 0
    short, _ = attention_bound(q, k, v, D ** -0.5, True, drop_dims=8)
    assert row_violations(o, short, tol)[0] > 0
    assert row_violations(o, torch.roll(o64, 1, 1), tol)[0] > 0


# ----------------------------------------------------------------------------------------------
# row kernels: LayerNorm, RMSNorm, row_stats at both ends of every instantiation's width range, strided
# ----------------------------------------------------------------------------------------------
NORM_COLS = (8, 256, 264, 512, 520, 768, 776, 1408, 1536, 1544, 4096, 4104, 5120, 6144, 6152, 16384)
NORM_ROWS = (1, 7, 9, 300)
def _norm_inputs(rows, cols, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(rows, cols, generator=g) * 2.0 + 0.5).half().to(DEV)
    w = (1.0 + 0.1 * torch.randn(cols, generator=g)).half().to(DEV)
    b = (0.1 * torch.randn(cols, generator=g)).half().to(DEV)
    return x, w, b


def _norm_call(lib, kind, x, w, b, y, eps):
    L = lib.load()
    rows, cols = x.shape
    if kind == "ln":
        st = L.seedb200_layernorm(x.data_ptr(), x.stride(0), w.data_ptr(), b.data_ptr(), y.data_ptr(), y.stride(0), rows,
                                  cols, eps, lib.stream_ptr())
    else:
        st = L.seedb200_rmsnorm(x.data_ptr(), x.stride(0), w.data_ptr(), y.data_ptr(), y.stride(0), rows, cols, eps,
                                lib.stream_ptr())
    lib.check(st, kind)
    torch.cuda.synchronize()


@pytest.mark.parametrize("cols", NORM_COLS)
def test_row_kernels_at_every_instantiation(lib, cols):
    """LayerNorm, RMSNorm and row_stats at both ends of every (threads per row, vectors per thread) width range, on a
    strided view with NaN padding and trailing NaN rows, into a sentinel buffer with guard columns"""
    for i, rows in enumerate(NORM_ROWS):
        x0, w, b = _norm_inputs(rows, cols, seed=cols + rows)
        _, x = in_buffer(x0, 8 * (1 + i), 2)
        for kind in ("ln", "rms"):
            ybuf = sentinel_buffer(rows + 1, cols + 16)
            y = ybuf[:rows, :cols]
            _norm_call(lib, kind, x, w, b, y, 1e-6)
            ref, tol = norm_bounds(kind, x, w, b, 1e-6)
            check16(y, ref, tol, f"{kind} rows={rows} cols={cols}")
            assert_guards(ybuf, region(ybuf, rows, cols), f"{kind} rows={rows} cols={cols}")
        st = lib.row_stats(x, 1e-6).to(F64)
        xd = x.to(F64)
        mean = xd.mean(-1)
        rstd = torch.rsqrt(xd.var(-1, unbiased=False) + 1e-6)
        assert ((st[:, 0] - mean).abs() <= ST * xd.abs().mean(-1)).all(), (rows, cols, (st[:, 0] - mean).abs().max())
        assert ((st[:, 1] / rstd - 1).abs() <= ST).all(), (rows, cols, (st[:, 1] / rstd - 1).abs().max())


def test_row_bounds_reject_a_wrong_reference(lib):
    rows, cols = 9, 776
    x, w, b = _norm_inputs(rows, cols, seed=1)
    for kind in ("ln", "rms"):
        y = torch.empty_like(x)
        _norm_call(lib, kind, x, w, b, y, 1e-6)
        ref, tol = norm_bounds(kind, x, w, b, 1e-6)
        assert violations(y, ref, tol)[0] == 0
        short, _ = norm_bounds(kind, x[:, :-8], w[:-8], b[:-8], 1e-6)
        assert violations(y[:, :-8], short, tol[:, :-8])[0] > 0, kind
        assert violations(y, torch.roll(ref, 1, 0), tol)[0] > 0, kind


@pytest.mark.parametrize("cols", [1408, 4096])
def test_row_stats_from_moments_against_float64(lib, cols):
    """rows x = mean + std z with |mean| / std up to 100; moments = the exact per-64-column (sum, sum of squares)
    rounded to fp32.  The kernel adds the G = cols / 64 groups in fp32 and finishes in fp64, so
        |d mean| <= G 2^-24 mean|x|
        |d rstd| / rstd <= 0.5 G 2^-24 (mean(x^2) + 2 |mean| mean|x|) / var + 2^-21
    which grows with (mean / std)^2: about 2e-2 at |mean| / std = 100 for G = 22.  Prints the measured errors."""
    G, rows = cols // 64, 64
    g = torch.Generator().manual_seed(cols)
    ratios = torch.tensor([0.0, 1.0, 3.0, 10.0, 30.0, 100.0, -100.0, -10.0]).repeat_interleave(rows // 8)
    std = 0.05 + torch.rand(rows, generator=g)
    x = (ratios[:, None] * std[:, None] + std[:, None] * torch.randn(rows, cols, generator=g)).half().to(DEV)
    xd = x.to(F64)
    grp = xd.view(rows, G, 64)
    mom = torch.stack((grp.sum(-1), (grp * grp).sum(-1)), -1).float().contiguous()
    st = lib.row_stats_from_moments(mom, cols, 0.0).to(F64)
    mean = xd.mean(-1)
    var = xd.var(-1, unbiased=False)
    rstd = torch.rsqrt(var)
    d_mean = (st[:, 0] - mean).abs()
    d_rstd = (st[:, 1] / rstd - 1).abs()
    assert (d_mean <= G * U24 * xd.abs().mean(-1)).all(), d_mean.max().item()
    bound = 0.5 * G * U24 * ((xd * xd).mean(-1) + 2 * mean.abs() * xd.abs().mean(-1)) / var + 2.0 ** -21
    assert (d_rstd <= bound).all(), (d_rstd / bound).max().item()
    r = (mean.abs() / var.sqrt()).cpu()
    for lo, hi in ((0, 0.5), (0.5, 2), (2, 5), (5, 20), (20, 50), (50, 200)):
        sel = ((r >= lo) & (r < hi)).to(DEV)
        if sel.any():
            print(f"MEASURED row_stats_from_moments cols={cols} |mean|/std in [{lo}, {hi}): max rel rstd err "
                  f"{d_rstd[sel].max().item():.3e} (bound {bound[sel].max().item():.3e}), max |d mean| / mean|x| "
                  f"{(d_mean / xd.abs().mean(-1))[sel].max().item():.3e}")
