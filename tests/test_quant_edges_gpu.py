"""Edge cases of the quantised-weight kernels against the restatements in tests/int8_ref.py and tests/quant4_ref.py,
bit for bit (NaN matching NaN): the LLM.int8() quantisers, the int8 wgmma GEMM (seedb200_gemm_int8) and the int8 GEMV
(seedb200_gemv_int8); the bitsandbytes 4-bit quantiser, dequantiser and GEMV (seedb200_quantize_4bit,
seedb200_dequantize_4bit, seedb200_gemv_4bit).

The int8 GEMM is persistent: a CTA runs tile after tile through one TMA / mbarrier ring, and the ring's stage and
phase carry over from tile to tile.  The multi-round cases give every tile width (and the SiLU-gate mode) more tiles
than the device has SMs, with k-loops of 1, STAGES - 1, STAGES + 1 and 2 STAGES + 1 stages so that each tile starts at
another point of the ring.  The other cases walk K, M and N across the 128-deep stage, the 128-row tile, the tile
widths and the 64 x 64 tiles / 32-column chunks of the outlier correction; they run on padded operands through
hand-built descriptors (fp16 padding NaN, int8 padding 0x7F: a stray read changes the result) into sentinel buffers,
with the residual in place where the model uses it so.  The SiLU-gate output is compared within one fp16 rounding of
silu(gate) (int8_ref.silu_gate_tol, the bound of test_int8_gpu.py's test_silu_gate).  Each comparison has a negative
control: it must reject a wrong restatement."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import int8_ref as Q8  # noqa: E402
import quant4_ref as Q4  # noqa: E402
from edge_ref import DEV, NAN, assert_guards, bit_diff, in_buffer, region, sentinel_buffer  # noqa: E402

pytestmark = pytest.mark.gpu
ERR_INVALID = 1                  # SEEDB200_ERR_INVALID
PAD8 = 0x7F                      # int8 padding: 127 times a weight or activation byte if it is ever read
EPS = 1e-6
STAGES = {256: 4, 128: 6, 64: 8}   # GemmCfg<bn>::STAGES of the int8 GEMM (200 KiB of 128-deep stages, at most 8)
QTS = [(Q4.FP4, "fp4"), (Q4.NF4, "nf4")]
MAX_SMEM = 220 * 1024            # the int8 GEMV's shared-memory budget for its staged rows
MAX_SMEM_Q4 = 200 * 1024         # the fp16 / 4-bit GEMV's


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def H(lib):
    return lib.load()


def same(out, ref, what):
    msg = bit_diff(out, ref)
    assert msg == "", f"{what}: {msg}"


# ----------------------------------------------------------------------------------------------
# operands
# ----------------------------------------------------------------------------------------------
def act(M, K, n_out, seed, cols=None):
    """fp16 activations in [-5.5, 5.5] with outliers (|a| in [8, 57]) in n_out random columns, or in `cols`"""
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * 1.5).clamp(-5.5, 5.5)
    if cols is None:
        cols = torch.randperm(K, generator=g)[:n_out].tolist()
    for i, c in enumerate(cols):
        a[(i * 7919 + c) % M, c] = (8.0 + (i % 50)) * (-1 if i % 2 else 1)
    return a.half()


def weight(N, K, seed):
    """CB, SCB of random fp16 weights whose row N // 3 is zero (SCB 0)"""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * torch.rand(N, 1, generator=g) * 0.05
    w[N // 3] = 0.0
    return Q8.quantize_weight(w.half())


def residual(M, n, seed):
    return (torch.randn(M, n, generator=torch.Generator().manual_seed(seed)) * 4).half()


# ----------------------------------------------------------------------------------------------
# C ABI calls with explicit leading dimensions
# ----------------------------------------------------------------------------------------------
def quantize_act(lib, a, threshold=6.0):
    """seedb200_int8_quantize_act on the fp16 view `a` (lda = its row stride) -> (CA, SCA, outliers, n) on the device"""
    M, K = a.shape
    ca = torch.empty((M, K), dtype=torch.int8, device=DEV)
    sca = torch.empty(M, dtype=torch.float32, device=DEV)
    ol = torch.empty(K, dtype=torch.int32, device=DEV)
    n = torch.empty(1, dtype=torch.int32, device=DEV)
    lib.check(H(lib).seedb200_int8_quantize_act(a.data_ptr(), a.stride(0), M, K, threshold, ca.data_ptr(),
                                                sca.data_ptr(), ol.data_ptr(), n.data_ptr(), lib.stream_ptr()),
              "seedb200_int8_quantize_act")
    return ca, sca, ol, n


def gemm8(lib, a, cb, scb, r=None, mode=0, bn=0, strided=False, inplace=False):
    """seedb200_gemm_int8 through a hand-built descriptor -> (out view, out buffer, written mask).  The activations
    are quantised by seedb200_int8_quantize_act from the A16 the GEMM reads.  Always: out inside a sentinel buffer
    with two guard rows, the correction workspace NaN.  strided: A16 and the residual are views into NaN-padded
    buffers, CA (lda = K + 48) and CB (ldw = K + 16) views into 0x7F-padded ones, and ldo = n_out + 9 (odd: every
    other row starts off a 4-byte boundary).  inplace: the residual is the output itself (ldr = ldo)."""
    M, K = a.shape
    N = cb.shape[0]
    n_out = N // 2 if mode == 1 else N
    a16 = in_buffer(a.to(DEV), 24, 1)[1] if strided else a.to(DEV).contiguous()
    ca, sca, ol, n = quantize_act(lib, a16)
    w = cb.to(DEV)
    if strided:
        ca = in_buffer(ca, 48, 2, fill=PAD8, dtype=torch.int8)[1]
        w = in_buffer(w, 16, 3, fill=PAD8, dtype=torch.int8)[1]
    buf = sentinel_buffer(M + 2, n_out + (9 if strided else 0))
    out = buf[:M, :n_out]
    res = None
    if inplace:
        out.copy_(r.to(DEV))
        res = out
    elif r is not None:
        res = in_buffer(r.to(DEV), 8, 1)[1] if strided else r.to(DEV).contiguous()
    ws = torch.full((M, N), NAN, dtype=torch.float16, device=DEV)
    scb = scb.to(DEV)
    d = lib.GemmInt8Desc()
    d.M, d.N, d.K = M, N, K
    d.A, d.lda, d.SCA = ca.data_ptr(), ca.stride(0), sca.data_ptr()
    d.A16, d.lda16 = a16.data_ptr(), a16.stride(0)
    d.outliers, d.n_outliers = ol.data_ptr(), n.data_ptr()
    d.W, d.ldw, d.SCB = w.data_ptr(), w.stride(0), scb.data_ptr()
    d.out, d.ldo = out.data_ptr(), out.stride(0)
    d.residual, d.ldr = (None, 0) if res is None else (res.data_ptr(), res.stride(0))
    d.mode, d.bn, d.workspace = mode, bn, ws.data_ptr()
    lib.check(H(lib).seedb200_gemm_int8(C.byref(d), lib.stream_ptr()), "seedb200_gemm_int8")
    torch.cuda.synchronize()
    return out, buf, region(buf, M, n_out)


def gemv8(lib, x, cb, scb, r=None, nw=None, mode=0, inplace=False, guard=40):
    """seedb200_gemv_int8 into a packed [M, n_out] block `guard` halves inside a sentinel buffer -> (out, buf, mask)"""
    M, K = x.shape
    N = cb.shape[0]
    n_out = N // 2 if mode == 1 else N
    buf = sentinel_buffer(1, M * n_out + 2 * guard)[0]
    out = buf[guard:guard + M * n_out].view(M, n_out)
    res = None
    if inplace:
        out.copy_(r.to(DEV))
        res = out
    elif r is not None:
        res = r.to(DEV).contiguous()
    x, cb, scb = x.to(DEV).contiguous(), cb.to(DEV).contiguous(), scb.to(DEV)
    lib.check(H(lib).seedb200_gemv_int8(x.data_ptr(), None if nw is None else nw.data_ptr(), EPS, 6.0,
                                        cb.data_ptr(), scb.data_ptr(), out.data_ptr(),
                                        None if res is None else res.data_ptr(), M, N, K, mode, lib.stream_ptr()),
              "seedb200_gemv_int8")
    torch.cuda.synchronize()
    mask = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
    mask[guard:guard + M * n_out] = True
    return out, buf, mask


def check_silu(out, y, what):
    """mode 1 against int8_ref.silu_gate of the bit-exact gate / up values y, within silu_gate_tol"""
    ref = Q8.silu_gate(y)
    tol = Q8.silu_gate_tol(y, ref)
    o, rf = out.cpu().float(), ref.float()
    assert torch.equal(torch.isnan(o), torch.isnan(rf)) and torch.equal(torch.isinf(o), torch.isinf(rf)), what
    fin = torch.isfinite(rf)
    bad = ~((o - rf).abs() <= tol) & fin
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        blk = y.float().view(y.shape[0], -1, 2, 128)
        g, u = blk[i[0], i[1] // 128, 0, i[1] % 128].item(), blk[i[0], i[1] // 128, 1, i[1] % 128].item()
        raise AssertionError(f"{what}: {int(bad.sum())} outside the SiLU-gate bound; first at {i}: gate {g!r} up "
                             f"{u!r} out {o[i].item()!r} ref {rf[i].item()!r} tol {tol[i].item():.3e}")


def check_linear8(out, a, cb, scb, r=None, mode=0, what=""):
    if mode == 1:
        check_silu(out, Q8.linear8_parts(a.cpu(), cb.cpu(), scb.cpu()), what)
    else:
        same(out, Q8.linear8(a, cb, scb, residual=r), what)


# ----------------------------------------------------------------------------------------------
# int8 GEMM: persistent multi-round runs
# ----------------------------------------------------------------------------------------------
def schedule(lib, M, N, bn, units):
    """(tiles, CTAs, the most tiles any CTA runs) of the int8 GEMM's schedule (make_schedule: 128-row tiles, round
    robin over min(units, tiles) CTAs), walked through seedb200_gemm_schedule_tile"""
    mt, nt = (M + 127) // 128, (N + bn - 1) // bn
    tiles = mt * nt
    ctas = max(1, min(units, tiles))
    rounds = 0
    for u in range(ctas):
        k = 0
        while H(lib).seedb200_gemm_schedule_tile(0, k, u, ctas, mt, nt, 0) < tiles:
            k += 1
        rounds = max(rounds, k)
    return tiles, ctas, rounds


# (bn, mode, M, N, K, |O|, operands: 0 packed / 1 strided (with a residual in mode 0) / 2 residual in place, tile
# class).  Tile classes at 132 SMs: "below" (< 132 tiles), "at" (132), "above" (133..160) and "multi" (2-3 x 132);
# K gives num_kb = ceil(K / 128) of 1, STAGES - 1, STAGES + 1 or 2 STAGES + 1 (bn 256: 4 stages, bn 128: 6, bn 64: 8).
MULTI_ROUND = [
    (256, 0, 1243, 3272, 112, 3, 0, "below"), (256, 0, 1408, 2900, 272, 5, 1, "at"),
    (256, 0, 833, 4757, 528, 7, 2, "above"), (256, 0, 1000, 4500, 384, 4, 1, "above"),
    (256, 0, 1900, 5500, 1040, 4, 2, "multi"), (256, 0, 1900, 5500, 16, 2, 1, "multi"),
    (128, 0, 2000, 1000, 64, 3, 2, "below"), (128, 0, 500, 4200, 592, 6, 0, "at"),
    (128, 0, 1000, 2100, 784, 5, 1, "above"), (128, 0, 1500, 2900, 640, 4, 2, "multi"),
    (128, 0, 1300, 3400, 1552, 3, 1, "multi"), (128, 0, 1300, 3400, 128, 33, 2, "multi"),
    (64, 0, 1100, 870, 128, 4, 1, "below"), (64, 0, 700, 1379, 880, 3, 2, "at"),
    (64, 0, 768, 1440, 1056, 6, 0, "above"), (64, 0, 1250, 1700, 896, 5, 1, "multi"),
    (64, 0, 1250, 2150, 2064, 5, 2, "multi"), (64, 0, 1250, 2149, 144, 9, 0, "multi"),
    (256, 1, 600, 8192, 128, 2, 1, "above"), (256, 1, 1100, 4096, 528, 5, 0, "above"),
    (256, 1, 2000, 5632, 272, 7, 1, "multi"), (256, 1, 1500, 6144, 1040, 3, 0, "multi"),
]


@pytest.mark.parametrize("bn,mode,M,N,K,n_out,res,cls", MULTI_ROUND)
def test_gemm8_multi_round(lib, bn, mode, M, N, K, n_out, res, cls):
    tiles, ctas, rounds = schedule(lib, M, N, bn, sms())
    num_kb = (K + 127) // 128
    print(f"int8 GEMM bn={bn} mode={mode} M={M} N={N} K={K}: {tiles} tiles on {ctas} CTAs, up to {rounds} rounds "
          f"per CTA at {sms()} SMs; {num_kb} k-blocks through {STAGES[bn]} stages")
    if cls in ("above", "multi"):
        assert rounds >= 2, (tiles, ctas)
    a = act(M, K, n_out, seed=M + N + K)
    cb, scb = weight(N, K, seed=N * 3 + K)
    r = residual(M, N, seed=M) if res and mode == 0 else None
    out, buf, mask = gemm8(lib, a, cb, scb, r, mode=mode, bn=bn, strided=res == 1, inplace=res == 2)
    assert_guards(buf, mask, "int8 GEMM out")
    check_linear8(out, a, cb, scb, r, mode, f"bn={bn} M={M} N={N} K={K}")


# ----------------------------------------------------------------------------------------------
# int8 GEMM: K, M and N tails on padded operands
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [16, 32, 48, 112, 128, 144, 240])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_gemm8_k_tails(lib, K, bn):
    """K below one 128-deep stage, at it and one 16-wide step past it: TMA's zero fill must stand in for the int8
    columns past K (the padding bytes are 0x7F)"""
    M, N = 200, 136
    a = act(M, K, 3 + K % 5, seed=K + bn)
    cb, scb = weight(N, K, seed=K)
    r = residual(M, N, seed=K)
    out, buf, mask = gemm8(lib, a, cb, scb, r, bn=bn, strided=True)
    assert_guards(buf, mask, "int8 GEMM out")
    same(out, Q8.linear8(a, cb, scb, residual=r), f"K={K} bn={bn}")


@pytest.mark.parametrize("M", [5, 63, 64, 65, 127, 128, 129, 257])
def test_gemm8_m_tails(lib, M):
    """M around the 128-row tile and the 64-row correction tile, with outliers, the residual in place"""
    N, K = 264, 144
    bn = (64, 128, 256)[M % 3]
    a = act(M, K, 5, seed=M)
    cb, scb = weight(N, K, seed=M + 1)
    r = residual(M, N, seed=M + 2)
    out, buf, mask = gemm8(lib, a, cb, scb, r, bn=bn, strided=True, inplace=M % 2 == 1)
    assert_guards(buf, mask, "int8 GEMM out")
    same(out, Q8.linear8(a, cb, scb, residual=r), f"M={M} bn={bn}")


@pytest.mark.parametrize("N", [8, 63, 64, 65, 127, 129, 255, 257])
@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("res", [False, True])
def test_gemm8_n_tails(lib, N, bn, res):
    """N around every tile width and the 64-column correction tile (odd N: the epilogue's single-half store)"""
    M, K = 70, 144
    a = act(M, K, 4, seed=N + bn)
    cb, scb = weight(N, K, seed=N)
    r = residual(M, N, seed=N + 1) if res else None
    out, buf, mask = gemm8(lib, a, cb, scb, r, bn=bn, strided=True)
    assert_guards(buf, mask, "int8 GEMM out")
    same(out, Q8.linear8(a, cb, scb, residual=r), f"N={N} bn={bn} res={res}")


def test_quantisers_on_strided_views(lib):
    """seedb200_int8_quantize_act / _weight read rows lda / ldw apart from NaN-padded buffers: a NaN read past K
    would flag an outlier column or poison a scale"""
    for M, K, n_out, pad in [(3, 16, 1, 8), (129, 144, 33, 40), (64, 4096, 7, 24)]:
        a = act(M, K, n_out, seed=M + K)
        ca, sca, ol, n = quantize_act(lib, in_buffer(a.to(DEV), pad, 2)[1])
        rca, rsca, rO = Q8.quantize_act(a)
        assert int(n.item()) == rO.numel() and torch.equal(ol[:rO.numel()].cpu().long(), rO), (M, K)
        assert torch.equal(sca.cpu(), rsca) and torch.equal(ca.cpu(), rca), (M, K)
    for N, K, pad in [(5, 16, 3), (300, 144, 40), (129, 4096, 8)]:
        g = torch.Generator().manual_seed(N)
        w = (torch.randn(N, K, generator=g) * 0.05).half()
        w[N // 2] = 0.0
        w[0, K - 1] = 60000.0
        wv = in_buffer(w.to(DEV), pad, 1)[1]
        cb = torch.empty((N, K), dtype=torch.int8, device=DEV)
        scb = torch.empty(N, dtype=torch.float32, device=DEV)
        lib.check(H(lib).seedb200_int8_quantize_weight(wv.data_ptr(), wv.stride(0), N, K, cb.data_ptr(),
                                                       scb.data_ptr(), lib.stream_ptr()), "quantize_weight")
        rcb, rscb = Q8.quantize_weight(w)
        assert torch.equal(cb.cpu(), rcb) and torch.equal(scb.cpu(), rscb), (N, K)


# ----------------------------------------------------------------------------------------------
# int8: outlier extremes
# ----------------------------------------------------------------------------------------------
def outlier_case(kind, M, K):
    """fp16 activations [M, K] for the outlier extremes; -> (a, rows whose output must be NaN)"""
    g = torch.Generator().manual_seed(K + M)
    a = ((torch.randn(M, K, generator=g) * 1.5).clamp(-5.5, 5.5)).half()
    nan_rows = []
    if kind.startswith("count"):
        a = act(M, K, int(kind[5:]), seed=K)
    elif kind == "all":              # every column an outlier (CA all zero); rows 0 and 1 nothing else (SCA 0)
        a[0] = 7.0
        a[1] = -9.0
    elif kind == "last":             # the only outlier in column K - 1
        a[M // 2, K - 1] = 11.0
    elif kind == "threshold":        # |a| = 6.0 is an outlier, the largest fp16 below it is not
        a[0, 3], a[M - 1, K - 2] = 6.0, -6.0
        a[1, 5], a[2, 7] = 5.99609375, -5.99609375
    elif kind == "nonfinite":        # +inf, -inf, NaN: each its own row
        a[1, 2], a[M - 2, K - 1] = float("inf"), -float("inf")
        a[M // 2, 9] = float("nan")
        nan_rows = [M // 2]
    return a, nan_rows


OUTLIER_KINDS = ["count31", "count32", "count33", "count64", "count65", "all", "last", "threshold", "nonfinite"]


@pytest.mark.parametrize("kind", OUTLIER_KINDS)
def test_gemm8_outlier_extremes(lib, kind):
    """counts around the correction's 32-column chunk, every column, the last column, the threshold itself and
    non-finite values, on M and N tails of its 64 x 64 tiles; the GEMV on the first rows gives the GEMM's bits"""
    M, N, K = 130, 200, 400 if kind.startswith("count") else 144
    a, nan_rows = outlier_case(kind, M, K)
    cb, scb = weight(N, K, seed=K + 7)
    O = Q8.quantize_act(a)[2]
    expect = int(kind[5:]) if kind.startswith("count") else {"all": K, "last": 1, "threshold": 2, "nonfinite": 3}[kind]
    assert O.numel() == expect, (kind, O.numel())
    if kind == "last":
        assert O.tolist() == [K - 1]
    if kind == "threshold":
        assert O.tolist() == [3, K - 2]
    ref = Q8.linear8(a, cb, scb)
    for bn in (64, 128, 256):
        for strided in (False, True):
            out, buf, mask = gemm8(lib, a, cb, scb, bn=bn, strided=strided)
            assert_guards(buf, mask, "int8 GEMM out")
            same(out, ref, f"{kind} bn={bn} strided={strided}")
    if kind == "nonfinite":           # the NaN fills its own row and reaches no other; rows without inf stay finite
        o = out.cpu().float()
        assert torch.isnan(o[M // 2]).all()
        assert torch.isfinite(o[[m for m in range(M) if m not in (1, M // 2, M - 2)]]).all()
    # M <= 4: the GEMV on the same rows (its own quantisation of those rows) gives the GEMM's bits
    rows = a[nan_rows[0] - 1:nan_rows[0] + 2] if nan_rows else a[:3]
    v, vb, vm = gemv8(lib, rows, cb, scb)
    assert_guards(vb, vm, "int8 GEMV out")
    same(v, gemm8(lib, rows, cb, scb)[0], f"{kind}: GEMV vs GEMM")
    same(v, Q8.linear8(rows, cb, scb), f"{kind}: GEMV")


def test_int8_comparison_rejects_a_wrong_restatement(lib):
    """negative controls of the bit-exact int8 comparison: the restatement without the last 16 columns of K,
    without one outlier column's correction term, or shifted by one row, must not match"""
    for bn, M, N, K, n_out in [(128, 300, 264, 144, 5), (256, 1100, 4096, 528, 7), (64, 65, 63, 32, 2)]:
        a = act(M, K, n_out, seed=bn + K)
        cb, scb = weight(N, K, seed=N)
        out = gemm8(lib, a, cb, scb, bn=bn, strided=True)[0]
        ref = Q8.linear8(a, cb, scb)
        same(out, ref, "control baseline")
        short = Q8.linear8(a[:, :K - 16], cb[:, :K - 16], scb)
        assert bit_diff(out, short) != "", (bn, M, N, K)
        for i in (0, n_out - 1):
            assert bit_diff(out, Q8.linear8_parts(a, cb, scb, skip_outlier=i)) != "", (bn, M, N, K, i)
        assert bit_diff(out, torch.roll(ref, 1, 0)) != "", (bn, M, N, K)
    # ... and the GEMV's comparison
    a = act(3, 528, 4, seed=5)
    cb, scb = weight(77, 528, seed=6)
    v = gemv8(lib, a, cb, scb)[0]
    same(v, Q8.linear8(a, cb, scb), "control baseline")
    assert bit_diff(v, Q8.linear8(a[:, :512], cb[:, :512], scb)) != ""
    assert bit_diff(v, Q8.linear8_parts(a, cb, scb, skip_outlier=0)) != ""
    assert bit_diff(v, torch.roll(Q8.linear8(a, cb, scb), 1, 0)) != ""


def test_silu_gate_bound_rejects_a_wrong_restatement(lib):
    """negative control of check_silu (mode 1): gate / up values without the last 16 columns of K, without one
    outlier column's correction term, or shifted by one row, fall outside the bound"""
    M, N, K = 300, 1024, 272
    a = act(M, K, 5, seed=9)
    cb, scb = weight(N, K, seed=10)
    out = gemm8(lib, a, cb, scb, mode=1, strided=True)[0]
    check_silu(out, Q8.linear8_parts(a, cb, scb), "control baseline")
    for wrong in (Q8.linear8_parts(a[:, :K - 16], cb[:, :K - 16], scb), Q8.linear8_parts(a, cb, scb, skip_outlier=2),
                  torch.roll(Q8.linear8_parts(a, cb, scb), 1, 0)):
        with pytest.raises(AssertionError, match="outside the SiLU-gate bound"):
            check_silu(out, wrong, "wrong restatement")


# ----------------------------------------------------------------------------------------------
# int8 GEMV
# ----------------------------------------------------------------------------------------------
def big_n(mode):
    """more row pairs than 8 warps x 8 resident CTAs x SMs can take at once: every CTA iterates (odd in mode 0)"""
    n = 16 * sms() * 8
    return n + 37 if mode == 0 else (n // 256 + 1) * 256


def staged_rows(lib, x, nw):
    """the rows the GEMVs stage: x, or with norm_w its RMSNorm as seedb200_gemv computes it (through an identity
    weight, exact), which the int8 GEMV reproduces operation for operation"""
    if nw is None:
        return x
    K = x.shape[1]
    return lib.gemv(x.to(DEV), torch.eye(K, dtype=torch.float16, device=DEV), norm_w=nw, eps=EPS).cpu()


# (M, mode, norm, residual: 0 none / 1 separate / 2 in place, K, N).  K: 16 (one 16-byte vector), 32, 528 (just past
# one vector per lane), 2032 / 2064 (one 16-step below / above the 4-vector unroll of 32 lanes).  N: odd, < 16, big.
GEMV8_CASES = [
    (1, 0, 0, 0, 16, 7), (1, 0, 1, 2, 2032, "big"), (1, 0, 0, 1, 528, 15), (1, 1, 0, 0, 2064, 256),
    (1, 1, 1, 0, 32, "big"),
    (2, 0, 0, 2, 32, 1), (2, 0, 1, 1, 16, 129), (2, 0, 0, 0, 2064, "big"), (2, 1, 0, 0, 528, "big"),
    (2, 1, 1, 0, 2032, 512),
    (3, 0, 0, 1, 2032, 9), (3, 0, 1, 0, 528, 3), (3, 0, 0, 2, 16, "big"), (3, 1, 0, 0, 16, 256),
    (3, 1, 1, 0, 2064, 768),
    (4, 0, 0, 0, 528, 2), (4, 0, 1, 2, 2064, 63), (4, 0, 0, 1, 32, "big"), (4, 1, 0, 0, 2032, "big"),
    (4, 1, 1, 0, 16, 256),
]


@pytest.mark.parametrize("M,mode,norm,res,K,N", GEMV8_CASES)
def test_gemv8_edges(lib, M, mode, norm, res, K, N):
    N = big_n(mode) if N == "big" else N
    seed = M * 1000 + K + N
    x = act(M, K, 2 if K >= 32 else 1, seed=seed)
    nw = (torch.rand(K, generator=torch.Generator().manual_seed(seed)) + 0.5).half().to(DEV) if norm else None
    if norm:
        nw[K // 3] = 40.0                                  # a channel that crosses the threshold after the norm
    cb, scb = weight(N, K, seed=seed + 1)
    r = residual(M, N, seed=seed + 2) if res else None
    out, buf, mask = gemv8(lib, x, cb, scb, r, nw, mode, inplace=res == 2)
    assert_guards(buf, mask, "int8 GEMV out")
    n = staged_rows(lib, x, nw)
    check_linear8(out, n, cb, scb, r, mode, f"GEMV M={M} mode={mode} norm={norm} K={K} N={N}")
    # the GEMM on the same (staged) rows gives the same bits
    same(out, gemm8(lib, n, cb, scb, r, mode=mode)[0], f"GEMV vs GEMM M={M} mode={mode} K={K} N={N}")


def gemv8_kmax(M):
    """the largest K the int8 GEMV accepts for M rows: fp16 rows M K 2 + int8 rows M K + flags K + list K 2 bytes"""
    return MAX_SMEM // (3 * M + 3) // 16 * 16


@pytest.mark.parametrize("M", [1, 2, 3, 4])
def test_gemv8_shared_memory_limit(lib, M):
    """the largest K that fits runs and matches; 16 more are refused with SEEDB200_ERR_INVALID and a message, before
    any launch (the stream stays usable)"""
    K, N = gemv8_kmax(M), 33
    x = act(M, K, 3, seed=M)
    cb, scb = weight(N, K, seed=M)
    out, buf, mask = gemv8(lib, x, cb, scb)
    assert_guards(buf, mask, "int8 GEMV out")
    same(out, Q8.linear8(x, cb, scb), f"M={M} K={K}")
    K2 = K + 16
    x2 = torch.zeros(M, K2, dtype=torch.float16, device=DEV)
    w2 = torch.zeros(N, K2, dtype=torch.int8, device=DEV)
    o2 = torch.zeros(M, N, dtype=torch.float16, device=DEV)
    s2 = torch.ones(N, dtype=torch.float32, device=DEV)
    st = H(lib).seedb200_gemv_int8(x2.data_ptr(), None, EPS, 6.0, w2.data_ptr(), s2.data_ptr(), o2.data_ptr(), None,
                                   M, N, K2, 0, lib.stream_ptr())
    msg = H(lib).seedb200_last_error().decode()
    assert st == ERR_INVALID and "shared memory" in msg, (st, msg)
    torch.cuda.synchronize()
    assert not o2.any()


# ----------------------------------------------------------------------------------------------
# 4-bit
# ----------------------------------------------------------------------------------------------
SUB = 2.0 ** -24                 # the smallest fp16 subnormal


def extreme_blocks():
    """fp16 [16, 128]: block 0 of each row is one kind of extreme block, block 1 random"""
    g = torch.Generator().manual_seed(11)
    w = torch.randn(16, 128, generator=g) * 0.1
    b = w[:, :64]
    b[0, 5] = NAN                                     # NaN among normal values
    b[1, 7] = float("inf")                            # +inf
    b[2, 63] = -float("inf")                          # -inf
    b[3] = NAN                                        # only NaN
    b[4, 0], b[4, 9] = 65504.0, -65504.0              # the fp16 extremes
    b[5] = torch.randint(-1023, 1024, (64,), generator=g).float() * SUB   # only subnormals
    b[6] = 0.0
    b[6, 17] = -0.375                                 # a single nonzero
    b[7] = 0.0
    b[7, 0] = 3 * SUB                                 # a single nonzero subnormal
    b[8] = 0.0                                        # all zero
    b[9] = 0.0
    b[9, 4] = -0.0                                    # all zero with a -0
    b[10, ::2] = -0.0                                 # -0 among normal values
    b[11, 3] = NAN
    b[11, 4] = 65504.0                                # NaN next to the largest value
    b[12] = 0.0
    b[12, 40] = NAN                                   # zeros and one NaN: absmax 0
    b[13, 8] = -65504.0
    b[13, 9] = -float("inf")                          # -inf beats -65504
    return w.half()


def quantize4(lib, w, qt, pad):
    """seedb200_quantize_4bit on a view with ldw = K + pad into a NaN-padded buffer"""
    N, K = w.shape
    wv = in_buffer(w.to(DEV), pad, 2)[1]
    packed = torch.empty((N, K // 2), dtype=torch.uint8, device=DEV)
    am = torch.empty((N, K // 64), dtype=torch.float32, device=DEV)
    lib.check(H(lib).seedb200_quantize_4bit(wv.data_ptr(), wv.stride(0), N, K, qt, packed.data_ptr(),
                                            am.data_ptr(), lib.stream_ptr()), "seedb200_quantize_4bit")
    return packed, am


def dequantize4(lib, packed, am, qt, pad):
    """seedb200_dequantize_4bit into a sentinel buffer with ldo = K + pad and two guard rows -> (W', buf, mask)"""
    N, K = packed.shape[0], packed.shape[1] * 2
    buf = sentinel_buffer(N + 2, K + pad)
    out = buf[:N, :K]
    lib.check(H(lib).seedb200_dequantize_4bit(packed.data_ptr(), am.data_ptr(), N, K, qt, out.data_ptr(),
                                              out.stride(0), lib.stream_ptr()), "seedb200_dequantize_4bit")
    torch.cuda.synchronize()
    return out, buf, region(buf, N, K)


@pytest.mark.parametrize("qt,name", QTS)
def test_quant4_extreme_blocks(lib, qt, name):
    """NaN, +-inf, 65504, subnormal-only, single-nonzero, all-zero and -0 blocks, quantised from a NaN-padded view
    (ldw > K) and dequantised into a sentinel buffer (ldo > K): bit for bit against quant4_ref, and the header's
    non-finite rules checked directly"""
    w = extreme_blocks()
    for pad in (8, 56):
        packed, am = quantize4(lib, w, qt, pad)
        rp, ram = Q4.quantize(w, qt)
        assert torch.equal(am.cpu(), ram), (name, pad)
        assert torch.equal(packed.cpu(), rp), (name, pad, (packed.cpu() != rp).nonzero()[:4].tolist())
        out, buf, mask = dequantize4(lib, packed, am, qt, pad)
        assert_guards(buf, mask, "dequantize_4bit out")
        same(out, Q4.dequantize(rp, ram, qt), f"{name} dequantise")
    # include/seedb200.h's rules, stated here independently of the restatement
    am, codes = am.cpu(), Q4.unpack(packed.cpu())[:, :64]
    wf = w[:, :64].float()
    assert am[0, 0] == wf[0].nan_to_num(0.0).abs().max()           # fmaxf: NaN dropped
    assert am[1, 0] == float("inf") and am[2, 0] == float("inf") and am[13, 0] == float("inf")
    assert am[3, 0] == 0 and am[8, 0] == 0 and am[9, 0] == 0 and am[12, 0] == 0
    assert am[4, 0] == 65504.0 and am[11, 0] == 65504.0
    assert am[5, 0] == wf[5].abs().max() and am[7, 0] == 3 * SUB
    assert (codes[0, 5] == 0) and (codes[3] == 0).all() and (codes[11, 3] == 0) and (codes[12] == 0).all()  # NaN
    assert (codes[8] == 0).all() and (codes[9] == 0).all()          # all-zero block: v NaN, code 0
    assert codes[1, 7] == 0 and codes[2, 63] == 0                    # inf * (1 / inf) = NaN
    top = 3 if qt == Q4.FP4 else 15                                  # the code of +1 (|v| rounds to 1 either side)
    assert codes[6, 17] == (top | 8 if qt == Q4.FP4 else 0) and codes[7, 0] == top and codes[4, 0] == top
    zero = 0 if qt == Q4.FP4 else 7                                  # the code of +-0 (FP4 -0: no sign bit)
    assert (codes[6, torch.arange(64) != 17] == zero).all() and (codes[10, ::2] == zero).all()


def gemv4(lib, x, packed, am, qt, r=None, nw=None, mode=0, inplace=False, guard=40):
    """seedb200_gemv_4bit into a packed [M, n_out] block inside a sentinel buffer -> (out, buf, mask)"""
    M, K = x.shape
    N = packed.shape[0]
    n_out = N // 2 if mode == 1 else N
    buf = sentinel_buffer(1, M * n_out + 2 * guard)[0]
    out = buf[guard:guard + M * n_out].view(M, n_out)
    res = None
    if inplace:
        out.copy_(r)
        res = out
    elif r is not None:
        res = r
    lib.check(H(lib).seedb200_gemv_4bit(x.data_ptr(), None if nw is None else nw.data_ptr(), EPS, packed.data_ptr(),
                                        am.data_ptr(), qt, out.data_ptr(), None if res is None else res.data_ptr(),
                                        M, N, K, mode, lib.stream_ptr()), "seedb200_gemv_4bit")
    torch.cuda.synchronize()
    mask = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
    mask[guard:guard + M * n_out] = True
    return out, buf, mask


# (M, mode, norm, residual: 0 / 1 / 2 in place, K, N)
GEMV4_CASES = [
    (1, 0, 0, 2, 64, 7), (2, 0, 1, 1, 64, "big"), (3, 0, 0, 0, 192, 1), (4, 0, 0, 2, 64, 255),
    (1, 1, 0, 0, 64, "big"), (4, 1, 1, 0, 128, 256), (2, 0, 0, 2, 1088, "big"), (3, 0, 1, 2, 4160, 13),
]


@pytest.mark.parametrize("qt,name", QTS)
@pytest.mark.parametrize("M,mode,norm,res,K,N", GEMV4_CASES)
def test_gemv4_edges(lib, qt, name, M, mode, norm, res, K, N):
    """K = 64 (one block), odd N, more row pairs than the grid holds, the residual in place: bit-identical to
    seedb200_gemv on the dequantised weight"""
    N = big_n(mode) if N == "big" else N
    g = torch.Generator().manual_seed(M + K + N)
    x = torch.randn(M, K, generator=g).half().to(DEV)
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    w[N // 2, :64] = 0.0
    packed, am = quantize4(lib, w, qt, 8)
    wd = lib.dequantize_4bit(packed, am, name)
    r = (torch.randn(M, N, generator=g) * 4).half().to(DEV) if res else None
    nw = (torch.rand(K, generator=g) + 0.5).half().to(DEV) if norm else None
    out, buf, mask = gemv4(lib, x, packed, am, qt, r, nw, mode, inplace=res == 2)
    assert_guards(buf, mask, "gemv_4bit out")
    same(out, lib.gemv(x, wd, residual=r, norm_w=nw, eps=EPS, mode=mode), f"{name} M={M} K={K} N={N}")


@pytest.mark.parametrize("qt,name", QTS)
def test_gemv4_on_extreme_blocks(lib, qt, name):
    """non-finite and extreme W' (NaN, inf, 65504-scaled, subnormal) flow through the 4-bit GEMV as through the fp16
    GEMV on the dequantised weight"""
    w = extreme_blocks()
    packed, am = quantize4(lib, w, qt, 8)
    wd = lib.dequantize_4bit(packed, am, name)
    x = torch.randn(3, 128, generator=torch.Generator().manual_seed(2)).half().to(DEV) * 1e-3
    out, buf, mask = gemv4(lib, x, packed, am, qt)
    assert_guards(buf, mask, "gemv_4bit out")
    same(out, lib.gemv(x, wd), name)


def gemv4_kmax(M):
    return MAX_SMEM_Q4 // (2 * M) // 64 * 64


@pytest.mark.parametrize("M", [1, 2, 3, 4])
def test_gemv4_shared_memory_limit(lib, M):
    """the largest K that fits runs and equals the fp16 GEMV; 64 more are refused with SEEDB200_ERR_INVALID"""
    K, N = gemv4_kmax(M), 9
    g = torch.Generator().manual_seed(M)
    x = torch.randn(M, K, generator=g).half().to(DEV)
    packed, am = quantize4(lib, (torch.randn(N, K, generator=g) * 0.05).half(), Q4.NF4, 0)
    out, buf, mask = gemv4(lib, x, packed, am, Q4.NF4)
    assert_guards(buf, mask, "gemv_4bit out")
    same(out, lib.gemv(x, lib.dequantize_4bit(packed, am, "nf4")), f"M={M} K={K}")
    K2 = K + 64
    x2 = torch.zeros(M, K2, dtype=torch.float16, device=DEV)
    p2 = torch.zeros(N, K2 // 2, dtype=torch.uint8, device=DEV)
    a2 = torch.ones(N, K2 // 64, dtype=torch.float32, device=DEV)
    o2 = torch.zeros(M, N, dtype=torch.float16, device=DEV)
    st = H(lib).seedb200_gemv_4bit(x2.data_ptr(), None, EPS, p2.data_ptr(), a2.data_ptr(), Q4.NF4, o2.data_ptr(),
                                   None, M, N, K2, 0, lib.stream_ptr())
    msg = H(lib).seedb200_last_error().decode()
    assert st == ERR_INVALID and "shared memory" in msg, (st, msg)
    torch.cuda.synchronize()
    assert not o2.any()


@pytest.mark.parametrize("qt,name", QTS)
def test_quant4_comparison_rejects_the_other_quant_type(lib, qt, name):
    """negative control: codes, W' and the GEMV output must not match a restatement built with the other type"""
    other = Q4.NF4 if qt == Q4.FP4 else Q4.FP4
    w = extreme_blocks()
    packed, am = quantize4(lib, w, qt, 8)
    out = dequantize4(lib, packed, am, qt, 8)[0]
    rp, ram = Q4.quantize(w, qt)
    assert torch.equal(packed.cpu(), rp)
    same(out, Q4.dequantize(rp, ram, qt), "control baseline")
    op, oam = Q4.quantize(w, other)
    assert not torch.equal(packed.cpu(), op)
    assert bit_diff(out, Q4.dequantize(op, oam, other)) != ""
    assert bit_diff(out, Q4.dequantize(rp, ram, other)) != ""     # the right codes read with the other table
    x = torch.randn(2, 128, generator=torch.Generator().manual_seed(4)).half().to(DEV)
    v = gemv4(lib, x, packed, am, qt)[0]
    wrong = Q4.dequantize(op, oam, other).to(DEV)
    assert bit_diff(v, lib.gemv(x, wrong)) != ""
