"""Edge cases of the decode-step kernels against float64 references: the GEMV (seedb200_gemv) over M = 1..4, both
epilogues, the folded RMSNorm, K and N tails, strided weights and every tuning switch; the split-KV decode attention
across the 8192-key split-size change; the fused RoPE + append + attention kernel; the RoPE table and rotation; the
model's split-KV decode path; and the sampler's guards.

Every bound is derived where it is built.  Each kind of bound has a negative control: the same check must reject a
reference computed with the last 8 reduction columns dropped, or with one row, head or position shifted, so a bound
too loose to see such an error fails its own test.  Measured errors are printed as MEASURED lines."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F
from transformers.models.llama.configuration_llama import LlamaConfig

from oracle import ops_ref as R
from oracle import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from edge_ref import (DEV, F64, NAN, SENTINEL, assert_guards, check16, gemm_tol, in_buffer,  # noqa: E402
                      norm_bounds, rand16, silu_gate_tol, ulp16, violations)

pytestmark = pytest.mark.gpu
LOG2E = 1.4426950408889634
LN2 = math.log(2.0)
U = 2.0 ** -24            # unit roundoff of fp32
EPS = 1e-6


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------------
# GEMV
# ----------------------------------------------------------------------------------------------
def gemv_silu_rel(g):
    """relative error of the GEMV's silu(g) = g / (1 + __expf(-g)) in fp32: __expf is ex2.approx of the fp32 product
    -g log2(e), so the exponential is off by 2^-22 (ex2.approx) plus |g| log2(e) 2^-24 (rounding of its argument);
    1 + e and the IEEE division round once each (2 2^-24).  A relative error d of e moves silu by at most d
    e / (1 + e) <= d relative.  In all: 2^-20 + 2^-24 log2(e) |g| (2^-20 covers 2^-22 + 2^-23 with room)."""
    return 2.0 ** -20 + U * LOG2E * g.abs()


def gemv_call(lib, x, w, residual=None, norm_w=None, mode=0, guard=24):
    """seedb200_gemv into an [M, n_out] block `guard` halves inside a sentinel buffer -> (out view, buffer, mask)"""
    M, K = x.shape
    N = w.shape[0]
    n_out = N // 2 if mode == 1 else N
    buf = torch.full((M * n_out + 2 * guard,), SENTINEL, dtype=torch.int16, device=DEV).view(torch.float16)
    out = buf[guard:guard + M * n_out].view(M, n_out)
    lib.check(lib.load().seedb200_gemv(x.data_ptr(), w.data_ptr(), w.stride(0), out.data_ptr(),
                                       None if residual is None else residual.data_ptr(),
                                       None if norm_w is None else norm_w.data_ptr(), EPS, M, N, K, mode,
                                       lib.stream_ptr()), "seedb200_gemv")
    torch.cuda.synchronize()
    mask = torch.zeros(buf.shape, dtype=torch.bool, device=DEV)
    mask[guard:guard + M * n_out] = True
    return out, buf, mask


def gemv_bound(x, w, residual=None, norm_w=None, mode=0, drop=0):
    """(ref64, tol) of the GEMV.  mode 0: gemm_tol (its K 2^-23 accumulator term holds for any summation order, the
    lane / warp-shuffle tree and the ksplit fold included).  norm_w: the operand is the fp16 RMSNorm of x; the
    kernel's staged value is within e = norm_bounds("rms") of the reference's (the GEMV's sum of squares runs through
    <= 100 values per thread + 5 shuffle levels + 8 warp partials, well inside norm_bounds' 2^-16), which adds
    e @ |W|^T before the output rounding.  mode 1: silu_gate_tol with gemv_silu_rel and the same operand error.
    `drop` leaves the last reduction columns out of the reference (negative control)."""
    K = x.shape[1] - drop
    xin, e = x, None
    if norm_w is not None:
        xin, e = norm_bounds("rms", x, norm_w, None, EPS)
        e = e[:, :K]
    xin, wk = xin[:, :K], w[:, :K]
    if mode == 1:
        wg, wu = deinterleave(wk)
        ref = R.silu_gate_ref(xin, wg, wu, dtype=F64)
        return ref, silu_gate_tol(xin, wg, wu, ref, gemv_silu_rel, e)
    ref = R.linear_ref(xin, wk, residual=residual, dtype=F64)
    mags = (ref, R.linear_ref(xin, wk, dtype=F64)) + ((residual,) if residual is not None else ())
    tol = gemm_tol(xin, wk, mags, 1 + (residual is not None))
    if e is not None:
        tol = tol + e @ wk.to(F64).abs().t()
    return ref, tol


def deinterleave(wgu):
    n2, K = wgu.shape
    b = wgu.reshape(n2 // 256, 2, 128, K)
    return b[:, 0].reshape(n2 // 2, K), b[:, 1].reshape(n2 // 2, K)


def big_n(mode):
    """N > 16 x SMs x 8: more row pairs than 8 per CTA x 8 resident CTAs per SM can take, so whatever the occupancy
    every CTA runs >= 2 iterations (odd in mode 0: the last pair is a single row)"""
    n = 16 * sms() * 8
    return n + 37 if mode == 0 else (n // 256 + 1) * 256


# M, mode, norm, residual, K, N ("big" = big_n).  K: 8 (one vector), < 256 (fewer than 32 vectors, idle lanes), not a
# multiple of 1024 (a partial U = 4 pass), M K 2 just above 48 KiB (cudaFuncSetAttribute), 25600 at M = 4 (200 KiB)
GEMV_CASES = [
    (1, 0, 0, 0, 8, 1), (1, 0, 0, 1, 248, 17), (1, 0, 1, 0, 24584, 15), (1, 0, 1, 1, 1032, "big"),
    (1, 1, 0, 0, 16, 256), (1, 1, 1, 0, 3080, "big"),
    (2, 0, 0, 0, 12296, 2), (2, 0, 0, 1, 120, 15), (2, 0, 1, 0, 256, "big"), (2, 0, 1, 1, 40, 1),
    (2, 1, 0, 0, 12296, 512), (2, 1, 1, 0, 8, 256),
    (3, 0, 0, 0, 8200, 17), (3, 0, 0, 1, 2056, 1), (3, 0, 1, 0, 64, 2), (3, 0, 1, 1, 200, "big"),
    (3, 1, 0, 0, 1024, "big"), (3, 1, 1, 0, 8200, 256),
    (4, 0, 0, 0, 25600, 15), (4, 0, 0, 1, 6152, 2), (4, 0, 1, 0, 72, "big"), (4, 0, 1, 1, 25600, 17),
    (4, 1, 0, 0, 6152, 768), (4, 1, 1, 0, 25600, 256),
]


def gemv_operands(M, mode, norm, res, K, N, seed):
    """x [M, K]; W a view with ldw = K + 8..24 into a NaN buffer with 3 NaN trailing rows; residual; norm weight"""
    N = big_n(mode) if N == "big" else N
    g = torch.Generator().manual_seed(seed)
    x = ((torch.randn(M, K, generator=g) * 1.5).half() if norm else torch.randn(M, K, generator=g).half()).to(DEV)
    _, w = in_buffer(rand16(N, K, scale=K ** -0.5 * (3 if mode else 1), seed=seed + 1), 8 * (1 + seed % 3), 3)
    r = rand16(M, N, seed=seed + 2) if res else None
    nw = (1.0 + 0.1 * torch.randn(K, generator=g)).half().to(DEV) if norm else None
    return x, w, r, nw


@pytest.mark.parametrize("M,mode,norm,res,K,N", GEMV_CASES)
def test_gemv_against_float64(lib, M, mode, norm, res, K, N):
    x, w, r, nw = gemv_operands(M, mode, norm, res, K, N, seed=M * 1000 + K + mode)
    out, buf, mask = gemv_call(lib, x, w, r, nw, mode)
    assert_guards(buf, mask, "gemv out")
    ref, tol = gemv_bound(x, w, r, nw, mode)
    check16(out, ref, tol, f"gemv M={M} mode={mode} norm={norm} res={res} K={K} N={w.shape[0]}")
    err = (out.to(F64) - ref.to(F64)).abs()
    print(f"MEASURED gemv M={M} mode={mode} norm={norm} res={res} K={K} N={w.shape[0]}: max |out - ref64| "
          f"{(err / ulp16(ref)).max().item():.2f} fp16 ulps, max err / bound {(err / tol).max().item():.3f}")


def test_gemv_bound_rejects_a_wrong_reference(lib):
    """negative control of gemv_bound: references without the last 8 reduction columns, or shifted by one output
    column, fail the same check, in both modes and with the folded norm"""
    for M, mode, norm, res, K, N in ((2, 0, 0, 1, 120, 15), (3, 0, 1, 0, 2056, 17), (2, 1, 1, 0, 264, 256),
                                     (1, 0, 0, 0, 8, 3)):
        x, w, r, nw = gemv_operands(M, mode, norm, res, K, N, seed=7 + K)
        out, _, _ = gemv_call(lib, x, w, r, nw, mode)
        ref, tol = gemv_bound(x, w, r, nw, mode)
        check16(out, ref, tol, "control baseline")
        short, _ = gemv_bound(x, w, r, nw, mode, drop=8)
        assert violations(out, short, tol)[0] > 0, (M, mode, norm, K)
        assert violations(out, torch.roll(ref, 1, 1), tol)[0] > 0, (M, mode, norm, K)


def test_gemv_silu_over_every_fp16_input(lib):
    """silu(g) * 1 for every finite fp16 g: x = e0, gate row j = value j, up rows = 1, so the accumulators are g and
    1 exactly and only the epilogue is measured.  Bound: |out - fp16(silu64(g))| <= ulp16(|ref| + e) + e with
    e = gemv_silu_rel(g) |silu(g)|."""
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    v = torch.unique(v[torch.isfinite(v)].float()).half()
    n = (v.numel() + 127) // 128 * 128
    gate = torch.zeros(n, dtype=torch.float16)
    gate[:v.numel()] = v
    K = 8
    wg = torch.zeros(n, K, dtype=torch.float16)
    wg[:, 0] = gate
    wu = torch.zeros(n, K, dtype=torch.float16)
    wu[:, 0] = 1
    x = torch.zeros(1, K, dtype=torch.float16, device=DEV)
    x[0, 0] = 1
    out, buf, mask = gemv_call(lib, x, R.interleave_gate_up(wg, wu).to(DEV), mode=1)
    assert_guards(buf, mask, "silu sweep")
    g = gate.to(DEV).to(F64)
    silu = F.silu(g)
    e = gemv_silu_rel(g) * silu.abs()
    ref = silu.half()
    check16(out[0], ref, ulp16(silu.abs() + e) + e, "gemv silu sweep")
    nz = silu.abs() > 2.0 ** -14                      # normal fp16 results: relative error is meaningful
    rel = ((out[0].to(F64) - silu).abs() / silu.abs().clamp_min(1e-300))[nz]
    flips = (out[0] != ref)[:v.numel()]
    print(f"MEASURED gemv silu over {v.numel()} fp16 inputs: max relative error {rel.max().item():.3e} where "
          f"|silu| >= 2^-14 (fp16 rounding included); {int(flips.sum())} results differ from fp16(silu(g)), by at most "
          f"{((out[0].to(F64) - ref.to(F64)).abs() / ulp16(ref)).max().item():.0f} ulp")


def test_gemv_nan_probes_reach_exactly_their_row_and_column(lib):
    """x[m, k] reaches row m only; W[r, k] reaches column r only (mode 1: (r // 256) 128 + r % 128), for r at the
    row-pair, CTA-pass (8 pairs) and N-tail boundaries and k at the 16-byte vector and 32-lane (256 halves) edges"""
    M, K = 3, 1032
    for mode in (0, 1):
        N = big_n(mode)
        x, w, _, _ = gemv_operands(M, mode, 0, 0, K, N, seed=41 + mode)
        for m in range(M):
            for k in (0, 7, 8, 255, 256, K - 1):
                xx = x.clone()
                xx[m, k] = NAN
                bad = ~torch.isfinite(gemv_call(lib, xx, w, mode=mode)[0].float())
                assert bad.any(1).nonzero().flatten().tolist() == [m] and bool(bad[m].all()), (mode, m, k)
        rows = sorted({0, 1, 15, 16, 17, 255, 256, N // 2, N // 2 + 1, N - 2, N - 1})
        for r in rows:
            for k in (0, 8, 255, 256, 1023, K - 1):
                old = w[r, k].item()
                w[r, k] = NAN
                bad = ~torch.isfinite(gemv_call(lib, x, w, mode=mode)[0].float())
                w[r, k] = old
                want = (r // 256) * 128 + r % 128 if mode == 1 else r
                cols = bad.any(0).nonzero().flatten().tolist()
                assert cols == [want] and bool(bad[:, want].all()), (mode, r, k, cols)


def _with_option(lib, key, value, fn):
    lib.set_option(key, value)
    try:
        return fn()
    finally:
        lib.set_option(key, {"gemv_no_allocate": 1, "gemv_prefetch_mb": 0, "gemv_ksplit": 0,
                             "decode_fused_attention": 1, "decode_pdl": 1}[key])


@pytest.mark.parametrize("case", [GEMV_CASES[i] for i in (3, 5, 10, 15, 16, 20, 23)])
def test_gemv_switches(lib, case):
    """gemv_no_allocate 0 and gemv_prefetch_mb 24 change loads only: bit-identical to the default.  gemv_ksplit 2 / 4
    re-associate the K sum (each slice folded in slice order, double-buffered across iterations): within the bound,
    including N that needs >= 2 iterations per CTA."""
    M, mode, norm, res, K, N = case
    x, w, r, nw = gemv_operands(M, mode, norm, res, K, N, seed=M * 1000 + K + mode)
    base = gemv_call(lib, x, w, r, nw, mode)[0].clone()
    ref, tol = gemv_bound(x, w, r, nw, mode)
    check16(base, ref, tol, "default")
    for key, val in (("gemv_no_allocate", 0), ("gemv_prefetch_mb", 24)):
        out = _with_option(lib, key, val, lambda: gemv_call(lib, x, w, r, nw, mode))
        assert_guards(out[1], out[2], f"{key}={val}")
        assert torch.equal(out[0], base), (key, val)
    for ks in (2, 4):
        out = _with_option(lib, "gemv_ksplit", ks, lambda: gemv_call(lib, x, w, r, nw, mode))
        assert_guards(out[1], out[2], f"ksplit={ks}")
        check16(out[0], ref, tol, f"ksplit={ks} {case}")


# ----------------------------------------------------------------------------------------------
# split-KV decode attention
# ----------------------------------------------------------------------------------------------
def da_split(kv_len):
    """misc.cu da_split: (splits, keys per split)"""
    n = min(64, -(-kv_len // 128))
    chunk = -(-(-(-kv_len // n)) // 128) * 128
    return -(-kv_len // chunk), chunk


def decode_bound(q, k, v, scale, blocks, merged, drop_dims=0):
    """float64 softmax(scale q k^T) v of one query per (b, h): q [B, H, D], k / v [B, H, n, D] the attended keys ->
    (o64 [B, H, D], tol).  The kernel keeps scores and probabilities in fp32 (no fp16 P: attention_bound's 2^-10
    term does not apply):
    * a score in log2 units, t = fp32(fp32(q.k) * fp32(scale log2 e)), is off by at most
      Et = (D + 3) 2^-23 scale log2(e) max_j |q|.|k_j| (D fma roundings, the rounded scale and the product);
    * p_j = exp2f(t_j - m): both t_j and m carry Et, the subtraction rounds (2^-24 |t_j - m| <= 2^-23 T, T = max|t|)
      and exp2f is within 2 fp32 ulps: a relative error of LN2 (2 Et + 2^-23 T) + 2^-22;
    * each rescale exp2f(m_old - m_new) of the online softmax (`blocks` per split) and of the merge (1) is exact
      except for its own rounding, 2^-22 + LN2 2^-23 T, because m_old's error cancels against the p_j it rescales;
    * fp32 sums: 16 P.V fmas per key group, the 8-group fold, 2 operations per block, `merged` splits and the final
      scaling: depth = 16 + 8 + 2 blocks + merged + 4 additions, each 2^-24 relative;
    * weights off by a relative eta move o = sum w_j v_j / sum w_j by at most 2 eta (P @ |v| + |o|); p_j below the
      fp32 subnormal range contribute n 2^-126 max|v|; the fp16 store adds one ulp of o.
    `drop_dims` leaves the last head dims out of the scores (negative control)."""
    D = q.shape[-1]
    qd, kd, vd = q.to(F64), k.to(F64), v.to(F64)
    Dk = D - drop_dims
    s = torch.einsum("bhd,bhnd->bhn", qd[..., :Dk], kd[..., :Dk]) * scale
    p = torch.softmax(s, -1)
    o = torch.einsum("bhn,bhnd->bhd", p, vd)
    pv = torch.einsum("bhn,bhnd->bhd", p, vd.abs())
    qk = torch.einsum("bhd,bhnd->bhn", qd.abs(), kd.abs()).amax(-1, keepdim=True)
    T = (s.abs().amax(-1, keepdim=True) * LOG2E)
    Et = (D + 3) * 2.0 ** -23 * scale * LOG2E * qk
    eta = LN2 * (2 * Et + 2.0 ** -23 * T) + 2.0 ** -22 + (blocks + 1) * (2.0 ** -22 + LN2 * 2.0 ** -23 * T)
    depth = 16 + 8 + 2 * blocks + merged + 4
    n = k.shape[2]
    tol = 2 * (eta + depth * U) * (pv + o.abs()) + n * 2.0 ** -126 * vd.abs().amax((-1, -2))[..., None] + ulp16(o)
    return o, tol


def split_shape(kv_len):
    ns, chunk = da_split(kv_len)
    return chunk // 128, ns


def nan_caches(B, H, max_seq, kv_len, seed, scale=1.0):
    """[B, H, max_seq, 128] caches with random rows below kv_len and NaN from kv_len on"""
    k = rand16(B, H, max_seq, 128, scale=scale, seed=seed)
    v = rand16(B, H, max_seq, 128, seed=seed + 1)
    k[:, :, kv_len:] = NAN
    v[:, :, kv_len:] = NAN
    return k, v


KV_LENS = [1, 2, 127, 128, 129, 4225, 8191, 8192, 8193, 8320, 16384, 16385]


@pytest.mark.parametrize("kv_len", KV_LENS)
def test_decode_attention_against_float64(lib, kv_len):
    """B = 2, H = 3, at every max_seq in {kv_len, 8300, 12000, 16385} that holds the cache: the workspace is sized
    for max_seq while the split count follows kv_len (64 splits of 128 keys at 8192, 33 of 256 at 8193).  Rows from
    kv_len on hold NaN: any read of them would show."""
    B, H, D = 2, 3, 128
    scale = D ** -0.5
    q = rand16(B, H, D, seed=kv_len)
    blocks, ns = split_shape(kv_len)
    for max_seq in sorted({kv_len, 8300, 12000, 16385}):
        if max_seq < kv_len:
            continue
        k, v = nan_caches(B, H, max_seq, kv_len, seed=kv_len + 1)
        out = lib.decode_attention(q, k, v, kv_len, scale)
        torch.cuda.synchronize()
        o64, tol = decode_bound(q, k[:, :, :kv_len], v[:, :, :kv_len], scale, blocks, ns)
        check16(out.view(B, H, D), o64, tol, f"decode attention kv={kv_len} max_seq={max_seq}")
        err = (out.view(B, H, D).to(F64) - o64).abs()
        print(f"MEASURED decode attention kv={kv_len} max_seq={max_seq} ({ns} splits of {blocks} blocks): max err "
              f"{(err / ulp16(o64)).max().item():.2f} fp16 ulps of o, max err / bound {(err / tol).max().item():.3f}")


def test_decode_attention_bound_rejects_a_wrong_reference(lib):
    for kv_len in (129, 8193):
        B, H, D = 1, 4, 128
        q = rand16(B, H, D, seed=3)
        k, v = nan_caches(B, H, kv_len, kv_len, seed=4)
        blocks, ns = split_shape(kv_len)
        out = lib.decode_attention(q, k, v, kv_len, D ** -0.5).view(B, H, D)
        o64, tol = decode_bound(q, k, v, D ** -0.5, blocks, ns)
        check16(out, o64, tol, "control baseline")
        short, _ = decode_bound(q, k, v, D ** -0.5, blocks, ns, drop_dims=8)
        assert violations(out, short, tol)[0] > 0, kv_len
        assert violations(out, torch.roll(o64, 1, 1), tol)[0] > 0, kv_len
        shifted, _ = decode_bound(q, k, torch.roll(v, 1, 2), D ** -0.5, blocks, ns)     # V[j] paired with K[j - 1]
        assert violations(out, shifted, tol)[0] > 0, kv_len


@pytest.mark.parametrize("kv_len", [8193, 12000, 16385])
@pytest.mark.parametrize("shape", ["up", "down", "spike"])
def test_decode_attention_online_softmax_across_blocks(lib, kv_len, shape):
    """above 8192 keys a split walks several 128-key blocks, rescaling its running (m, l, o) at each: scores ramping
    up (the max moves in every block), ramping down (the first block holds it) and one spike in the last block"""
    B, H, D = 1, 2, 128
    scale = D ** -0.5
    q = rand16(B, H, D, scale=0.25, seed=kv_len)
    q[..., 0] = 8.0
    k, v = nan_caches(B, H, kv_len, kv_len, seed=kv_len + 2, scale=0.25)
    ramp = torch.linspace(-10.0, 10.0, kv_len, device=DEV)
    if shape == "up":
        k[..., 0] = ramp.half()
    elif shape == "down":
        k[..., 0] = ramp.flip(0).half()
    else:
        k[..., 0] = 0
        k[:, :, kv_len - 3, 0] = 12.0
    blocks, ns = split_shape(kv_len)
    out = lib.decode_attention(q, k, v, kv_len, scale).view(B, H, D)
    o64, tol = decode_bound(q, k, v, scale, blocks, ns)
    check16(out, o64, tol, f"online softmax {shape} kv={kv_len}")


def dominant_keys(q, scale):
    """a key whose score beats N(0, 1) keys by > 40 nats: sign(q) * 8 in every dim (score 8 scale sum|q| ~ 72)"""
    return (torch.sign(q.float()) * 8).half()


@pytest.mark.parametrize("kv_len,max_seq", [(129, 129), (4225, 8300), (8193, 16385), (16385, 16385)])
def test_decode_attention_dominant_key_is_copied_exactly(lib, kv_len, max_seq):
    """one key per head wins by > 40 nats (every other weight < e^-40 relative): the output is V[j] bit for bit, for j
    at 0, 127, 128, the split boundaries and kv_len - 1.  A dominant key at row kv_len (outside the cache) must not
    show: its head matches the float64 reference of the first kv_len keys."""
    ns, chunk = da_split(kv_len)
    js = sorted({j for j in (0, 127, 128, chunk - 1, chunk, (ns - 1) * chunk - 1, (ns - 1) * chunk, kv_len - 1)
                 if 0 <= j < kv_len})
    B, H, D = 1, len(js) + (1 if kv_len < max_seq else 0), 128
    scale = D ** -0.5
    q = rand16(B, H, D, seed=kv_len + 5)
    k, v = nan_caches(B, H, max_seq, kv_len, seed=kv_len + 6)
    dom = dominant_keys(q, scale)
    for h, j in enumerate(js):
        k[0, h, j] = dom[0, h]
    if kv_len < max_seq:
        k[0, H - 1, kv_len] = dom[0, H - 1]
        v[0, H - 1, kv_len] = 100.0
    out = lib.decode_attention(q, k, v, kv_len, scale).view(B, H, D)
    for h, j in enumerate(js):
        assert torch.equal(out[0, h], v[0, h, j]), (kv_len, j)
    if kv_len < max_seq:
        blocks, _ = split_shape(kv_len)
        o64, tol = decode_bound(q[:, -1:], k[:, -1:, :kv_len], v[:, -1:, :kv_len], scale, blocks, ns)
        check16(out[:, -1:], o64, tol, "dominant key behind the cache")


def test_decode_attention_nan_propagation_matches_torch(lib):
    """a NaN key entry in (b, h) makes all of (b, h) NaN (softmax over a NaN score), a NaN V[j, d] only dim d of its
    head, and NaN rows behind kv_len or in other heads stay out"""
    B, H, D, kv_len, max_seq = 2, 3, 128, 8193, 8300
    scale = D ** -0.5
    q = rand16(B, H, D, seed=71)
    k, v = nan_caches(B, H, max_seq, kv_len, seed=72)
    k[0, 1, 4096, 17] = NAN
    v[1, 2, 8192, 5] = NAN
    v[1, 0, 0, 127] = NAN
    out = lib.decode_attention(q, k, v, kv_len, scale).view(B, H, D)
    s = torch.einsum("bhd,bhnd->bhn", q.to(F64), k[:, :, :kv_len].to(F64)) * scale
    ref = torch.einsum("bhn,bhnd->bhd", torch.softmax(s, -1), v[:, :, :kv_len].to(F64))
    assert torch.equal(torch.isnan(out), torch.isnan(ref)), int((torch.isnan(out) ^ torch.isnan(ref)).sum())
    assert bool(torch.isnan(out[0, 1]).all()) and int(torch.isnan(out).sum()) == D + 2


@pytest.mark.parametrize("kv_len", [8193, 16385])
def test_lineage_attention_long_caches_bit_identical_to_gathered(lib, kv_len):
    g = torch.Generator().manual_seed(kv_len)
    rows, used, H, D, max_seq = 4, 3, 2, 128, 16385
    k = torch.randn((rows, H, max_seq, D), generator=g).half()
    v = torch.randn((rows, H, max_seq, D), generator=g).half()
    k[used:] = NAN
    v[used:] = NAN
    slot = torch.randint(0, used, (used, max_seq), generator=g, dtype=torch.int32)
    slot[:, :kv_len // 3] = 0
    q = torch.randn((used, H, D), generator=g).half().cuda()
    k, v, slot = k.cuda(), v.cuda(), slot.cuda()
    pos = torch.arange(max_seq, device=DEV)
    gk = k[slot.long(), :, pos[None, :], :].permute(0, 2, 1, 3).contiguous()
    gv = v[slot.long(), :, pos[None, :], :].permute(0, 2, 1, 3).contiguous()
    ref = lib.decode_attention(q, gk, gv, kv_len, 0.0883883)
    got = lib.decode_attention_lineage(q, k, v, slot, kv_len, 0.0883883)
    torch.cuda.synchronize()
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, ref)


# ----------------------------------------------------------------------------------------------
# RoPE: the device table and the rotation
# ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev_table(lib):
    """the device's fp16 cos / sin table [8192, 64], read through rope_kv_append: q = ones in the low half and zeros
    in the high half gives q_out = (fp16(1 c) + fp16(-0 s), fp16(0 c) + fp16(1 s)) = (c, s) exactly.  max_seq = 5000
    builds (or reuses) a table of >= 8192 rows; positions go up to 8191."""
    H, D, S = 1, 128, 4096
    qkv = torch.zeros(S, 3 * H * D, dtype=torch.float16, device=DEV)
    qkv[:, :64] = 1
    kc = torch.zeros((1, H, 5000, D), dtype=torch.float16, device=DEV)
    cos, sin = [], []
    for p0 in (0, 4096):
        pos = (p0 + torch.arange(S, device=DEV))[None]
        qo = lib.rope_kv_append(qkv, pos, 1, S, H, D, 0, kc, kc.clone())
        torch.cuda.synchronize()
        cos.append(qo[:, :64])
        sin.append(qo[:, 64:])
    return torch.cat(cos), torch.cat(sin)


def rope_table_tol(ref, pos, inv_freq):
    """|device - CPU table| per entry: both evaluate fp16(cos(fp32(pos * inv_freq))).  inv_freq = 1 / base^(2i/D) is
    within 2^-20 relative between powf and torch.pow (a few fp32 ulps), the product rounds (2^-24 each side), and
    cosf / sinf are within 2 fp32 ulps (<= 2^-22 absolute for |value| <= 1): the fp32 values differ by at most
    f (2^-20 + 2^-23) + 2^-21, f = pos inv_freq; each side then rounds to fp16: one fp16 ulp."""
    f = pos.to(F64)[:, None] * inv_freq.to(F64)[None, :]
    return ulp16(ref.to(F64).abs()) + f * (2.0 ** -20 + 2.0 ** -23) + 2.0 ** -21


def test_rope_table_against_cpu_construction(lib, dev_table):
    """the device table against ops_ref.rope_tables built on the CPU (the reference's construction) under
    rope_table_tol; a table shifted by one position fails the same check.  Prints, per frequency column, how many
    fp16 entries differ from the CPU's (a one-ulp change of one fp32 inv_freq alone flips thousands of a high-frequency
    column's 8192 entries, each by one ulp)."""
    cos_d, sin_d = dev_table
    n = cos_d.shape[0]
    cos_c, sin_c = R.rope_tables(n, 128)
    cos_c, sin_c = cos_c[:, :64].to(DEV), sin_c[:, :64].to(DEV)
    inv_freq = 1.0 / (10000.0 ** (torch.arange(0, 128, 2).float() / 128))
    pos = torch.arange(n, device=DEV)
    for name, d, c in (("cos", cos_d, cos_c), ("sin", sin_d, sin_c)):
        tol = rope_table_tol(c, pos, inv_freq.to(DEV))
        check16(d, c, tol, f"rope {name} table")
        assert violations(d, torch.roll(c, 1, 0), tol)[0] > 0, name
        flips = (d != c).sum(0).tolist()
        worst = ((d.to(F64) - c.to(F64)).abs() / ulp16(c)).max(0).values
        print(f"MEASURED rope {name} table, {n} positions: entries differing from the CPU table per column "
              f"{flips}; max difference {worst.max().item():.0f} fp16 ulps (column {int(worst.argmax())})")


def rope_apply(x, pos, cos, sin):
    """rope_ref's fp16 arithmetic on a given table: x [..., 128] fp16, pos [...] -> x cos + rotate_half(x) sin with
    every product and the sum rounded to fp16"""
    c, s = cos[pos], sin[pos]
    lo, hi = x[..., :64], x[..., 64:]
    return torch.cat((lo * c + (-hi) * s, hi * c + lo * s), -1)


def test_rope_rotation_bit_identical_on_the_device_table(lib, dev_table):
    """given the device's own table, rope_kv_append's q and appended K equal rope_ref's fp16 arithmetic bit for bit
    (positions up to 8191, through the positions argument); V is copied"""
    cos, sin = dev_table
    B, S, H, D, max_seq = 2, 300, 3, 128, 700
    qkv = rand16(B * S, 3 * H * D, scale=2.0, seed=81)
    g = torch.Generator().manual_seed(82)
    pos = torch.randint(0, 8192, (B, S), generator=g).to(DEV)
    pos[0, :4] = torch.tensor([0, 4095, 4096, 8191])
    kc = torch.full((B, H, max_seq, D), NAN, dtype=torch.float16, device=DEV)
    vc = kc.clone()
    past = 100
    q_out = lib.rope_kv_append(qkv, pos, B, S, H, D, past, kc, vc)
    torch.cuda.synchronize()
    x = qkv.view(B, S, 3, H, D)
    pp = pos[:, :, None].expand(B, S, H)
    assert torch.equal(q_out.view(B, S, H, D), rope_apply(x[:, :, 0], pp, cos, sin))
    assert torch.equal(kc[:, :, past:past + S], rope_apply(x[:, :, 1], pp, cos, sin).permute(0, 2, 1, 3))
    assert torch.equal(vc[:, :, past:past + S], x[:, :, 2].permute(0, 2, 1, 3))
    assert torch.isnan(kc[:, :, :past].float()).all() and torch.isnan(kc[:, :, past + S:].float()).all()
    shifted = rope_apply(x[:, :, 0], (pp + 1).clamp(max=8191), cos, sin)
    assert not torch.equal(q_out.view(B, S, H, D), shifted)


# ----------------------------------------------------------------------------------------------
# fused RoPE + append + attention
# ----------------------------------------------------------------------------------------------
FUSED_PAST = [0, 1, 127, 128, 129, 511, 512, 513, 1023, 2047]


@pytest.mark.parametrize("max_seq", [1, 128, 129, 512, 513, 2048])
def test_decode_attention_rope_against_float64(lib, dev_table, max_seq):
    """1..4 thread groups (ng = min(4, ceil(max_seq / 128))), groups walking several blocks from 513 keys on.  Cache
    rows behind past_len hold NaN and stay bit-unchanged; row past_len is the RoPE reference of the new K (bit for
    bit) and V; the output is within decode_bound of float64 attention of the rotated q over past_len + 1 keys
    (blocks per group = ceil(kv / (128 ng)), ng groups merged)."""
    cos, sin = dev_table
    B, H, D = 2, 2, 128
    scale = D ** -0.5
    ng = min(4, -(-max_seq // 128))
    for past in FUSED_PAST:
        if past >= max_seq:
            continue
        qkv = rand16(B, 3 * H * D, seed=past + 91)
        k, v = nan_caches(B, H, max_seq, past, seed=past + 92)
        k0, v0 = k.clone(), v.clone()
        out = lib.decode_attention_rope(qkv, None, H, past, k, v, scale).view(B, H, D)
        torch.cuda.synchronize()
        x = qkv.view(B, 3, H, D)
        pp = torch.full((B, H), past, dtype=torch.long, device=DEV)
        q_rot, k_rot = rope_apply(x[:, 0], pp, cos, sin), rope_apply(x[:, 1], pp, cos, sin)
        assert torch.equal(k[:, :, past], k_rot) and torch.equal(v[:, :, past], x[:, 2]), past
        keep = torch.ones(max_seq, dtype=torch.bool, device=DEV)
        keep[past] = False
        assert torch.equal(k.view(torch.int16)[:, :, keep], k0.view(torch.int16)[:, :, keep]), past
        assert torch.equal(v.view(torch.int16)[:, :, keep], v0.view(torch.int16)[:, :, keep]), past
        kv = past + 1
        o64, tol = decode_bound(q_rot, k[:, :, :kv], v[:, :, :kv], scale, -(-kv // (128 * ng)), ng)
        check16(out, o64, tol, f"fused decode attention past={past} max_seq={max_seq}")
        if past in (1, 513):
            short, _ = decode_bound(q_rot, k[:, :, :kv], v[:, :, :kv], scale, -(-kv // (128 * ng)), ng, drop_dims=8)
            assert violations(out, short, tol)[0] > 0, past
            assert violations(out, torch.roll(o64, 1, 1), tol)[0] > 0, past


@pytest.mark.parametrize("past,max_seq", [(0, 1), (128, 129), (511, 2048), (1023, 2048), (2047, 2048)])
def test_decode_attention_rope_dominant_fresh_key(lib, past, max_seq):
    """q = k in qkv: after the same rotation the new key scores |k|^2 scale (~180), far above any cached key, so the
    output is the new V bit for bit -- the fresh key / value taken from shared memory reach the group that owns
    row past_len"""
    B, H, D = 1, 2, 128
    qkv = rand16(B, 3 * H * D, seed=past + 3)
    x = qkv.view(B, 3, H, D)
    x[:, 1] = (torch.sign(x[:, 1].float()) * 4).half()
    x[:, 0] = x[:, 1]
    k, v = nan_caches(B, H, max_seq, past, seed=past + 4)
    out = lib.decode_attention_rope(qkv, None, H, past, k, v, D ** -0.5).view(B, H, D)
    torch.cuda.synchronize()
    assert torch.equal(out, x[:, 2]), past


# ----------------------------------------------------------------------------------------------
# the model's split-KV decode path
# ----------------------------------------------------------------------------------------------
HID, LAYERS, HEADS, FFN, VOCAB = 512, 2, 4, 1408, 1056


def make_llama(max_seq, max_batch=4, seed=9):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=VOCAB, hidden_size=HID, intermediate_size=FFN, num_hidden_layers=LAYERS,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=16385)
    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=seed)
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=max_batch, max_seq=max_seq)


def prompt(B, S, seed=10):
    return synth.prompt_ids(B, S, n_image_spans=1, text_vocab=VOCAB - 66, n_codes=64, seed=seed).cuda()


def step_logits(model, ids, steps):
    """prefill, then `steps` eager decode forwards of the greedy token: the logits of every step"""
    out = model(input_ids=ids, use_cache=True, last_logits_only=True)
    logits = [out.logits[:, -1].clone()]
    past = out.past_key_values
    for _ in range(steps):
        tok = logits[-1].argmax(-1, keepdim=True)
        out = model(input_ids=tok, past_key_values=past, use_cache=True, last_logits_only=True)
        past = out.past_key_values
        logits.append(out.logits[:, -1].clone())
    return torch.stack(logits)


def test_model_split_kv_path_equals_fused_path(lib):
    """max_seq 2048 runs the fused decode attention, 2049 rope_kv_append + the split-KV kernel with the handle's
    self-resetting tickets (and, in graphs, the device-side cache length).  While the cache holds <= 512 keys the two
    are bit-identical: eager logits, greedy generate eager and graph, beam search eager and graph; the same holds for
    decode_fused_attention = 0 at max_seq 2048 and for decode_pdl 0 against 1."""
    fused, split = make_llama(2048), make_llama(2049)
    ids = prompt(2, 40)
    a = step_logits(fused, ids, 60)
    b = step_logits(split, ids, 60)
    assert torch.isfinite(a.float()).all() and torch.equal(a, b)
    kw = dict(max_new_tokens=100, do_sample=False, eos_token_id=-1)
    for use_graph in (True, False):
        ref = fused.generate(input_ids=ids, use_graph=use_graph, **kw)
        assert torch.equal(split.generate(input_ids=ids, use_graph=use_graph, **kw), ref), use_graph
        assert split._llm.used_graph == int(use_graph)
        bkw = dict(max_new_tokens=30, num_beams=2, eos_token_id=-1, use_graph=use_graph)
        assert torch.equal(split.generate(input_ids=ids, **bkw), fused.generate(input_ids=ids, **bkw)), use_graph
    ref = fused.generate(input_ids=ids, **kw)
    for key, val in (("decode_fused_attention", 0), ("decode_pdl", 0)):
        got = _with_option(lib, key, val, lambda: fused.generate(input_ids=ids, **kw))
        assert torch.equal(got, ref), key
        got = _with_option(lib, key, val, lambda: step_logits(fused, ids, 8))
        assert torch.equal(got, a[:9]), key


def test_model_long_cache_graph_equals_eager_across_split_change(lib):
    """max_seq = 8300 (33 splits at max_seq, up to 64 at shorter caches): decoding across 4224 / 4225, 8192 and
    8193 cached keys, the graph-replayed steps (device-side cache length, grid sized for every length) give the same
    tokens as eager steps, and the eager logits of one step equal a model with max_seq = 16385 bit for bit (the same
    split rule applies at the same cache length)."""
    model = make_llama(8300, max_batch=1)
    other = make_llama(16385, max_batch=1)
    for S in (4220, 8188):
        ids = prompt(1, S, seed=S)
        kw = dict(max_new_tokens=10, do_sample=False, eos_token_id=-1)
        g = model.generate(input_ids=ids, use_graph=True, **kw)
        assert model._llm.used_graph == 1
        e = model.generate(input_ids=ids, use_graph=False, **kw)
        assert torch.equal(g, e), S
        la, lb = step_logits(model, ids, 8), step_logits(other, ids, 8)
        assert torch.isfinite(la.float()).all() and torch.equal(la, lb), S


# ----------------------------------------------------------------------------------------------
# sampler guards
# ----------------------------------------------------------------------------------------------
def test_sampler_ignores_nan_row_padding(lib):
    """logits rows with ld > V whose padding holds NaN: greedy and sampled tokens equal those of the unpadded rows"""
    B, V = 3, 40194
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(B, V, generator=g) * 3).half().to(DEV)
    buf = torch.full((B, V + 14), NAN, dtype=torch.float16, device=DEV)
    buf[:, :V] = x
    for samp in (dict(), dict(do_sample=True, temperature=0.8, top_p=0.9, seed=3, offset=1)):
        got = lib.sample(buf[:, :V], **samp)
        assert torch.equal(got, lib.sample(x.contiguous(), **samp)), samp
        assert (got < V).all()
    assert lib.sample(buf[:, :V]).tolist() == x.float().argmax(-1).tolist()


@pytest.mark.parametrize("V", [1, 1023, 1024, 1025, 40194])
def test_sampler_argmax_at_chunk_edges(lib, V):
    """each of the 1024 threads scans ceil(V / 1024) tokens: the maximum at the last token of a chunk, the first of
    the next, V - 1, and a tie across a chunk edge (the lower id wins, as torch.argmax)"""
    per = -(-V // 1024)
    spots = sorted({j for j in (0, per - 1, per, 2 * per - 1, V - 1) if 0 <= j < V})
    g = torch.Generator().manual_seed(V)
    rows = (torch.randn(len(spots) + 1, V, generator=g)).half()
    for i, j in enumerate(spots):
        rows[i, j] = 20.0
    if V > per:
        rows[-1, per - 1] = rows[-1, per] = 20.0
    got = lib.sample(rows.to(DEV)).cpu()
    assert got.tolist() == rows.float().argmax(-1).tolist()
    tiny = lib.sample(rows.to(DEV), do_sample=True, temperature=1.0, top_p=1e-6, seed=1).cpu()
    assert tiny[:len(spots)].tolist() == got[:len(spots)].tolist()
    if V > per:
        assert int(tiny[-1]) in (per - 1, per)


def test_sampler_tiny_top_p_keeps_only_the_argmax_and_its_ties(lib):
    """top_p -> 0 keeps the most probable token and every token tied with it: 64 seeds draw only from the tie set,
    and from more than one member of it"""
    V = 5000
    x = (torch.randn(1, V, generator=torch.Generator().manual_seed(2)) * 2).half()
    ties = [17, 2048, 4999]
    x[0, ties] = 15.0
    rows = x.expand(64, V).contiguous().to(DEV)
    got = set(lib.sample(rows, do_sample=True, temperature=1.0, top_p=1e-7, seed=77).tolist())
    assert got <= set(ties) and len(got) > 1, got
