"""GPU parity tests of every per-op C-ABI entry point against the oracle restatements (oracle/ops_ref.py,
oracle/vq_oracle.c).  Integer outputs are bit-exact; fp16 outputs are compared with the tolerance written
next to each test (a few fp16 ulps: the accumulation order inside a tensor-core tile is not the oracle's)."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from oracle import ops_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def max_ulp_err(a, b):
    """max |a-b| in units of the fp16 spacing at |b| (floor at 2^-14)."""
    a, b = a.float(), b.float()
    ulp = torch.pow(2.0, torch.floor(torch.log2(b.abs().clamp_min(2.0 ** -14))) - 10)
    return ((a - b).abs() / ulp).max().item()


def assert_close16(out, ref, mags=(), ulps=2.0, atol=3e-5, what=""):
    """|out-ref| <= ulps * 2^-10 * max(|ref|, |m| for m in mags) + atol, elementwise.  `mags` lists the
    intermediates that were rounded to fp16 on the way (a 1-ulp flip of an intermediate survives a
    cancelling add), `atol` covers the fp32 accumulation-order noise on near-zero outputs."""
    o, r = out.float(), ref.float()
    mag = r.abs()
    for m in mags:
        mag = torch.maximum(mag, m.float().abs())
    tol = ulps * mag * 2.0 ** -10 + atol
    diff = (o - r).abs()
    bad = diff > tol
    assert not bad.any(), (f"{what}: {int(bad.sum())}/{bad.numel()} elements outside tolerance; max diff "
                           f"{diff.max().item():.3e}, rel fro {rel_err(out, ref):.3e}, worst idx "
                           f"{int(torch.argmax(diff - tol))}")


def rand16(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.float16).to(DEV)


# ----------------------------------------------------------------------------------------------
# GEMM (wgmma): every tile width, tails in M/N/K, persistent multi-tile schedules; ctas = 2 is accepted and runs
# the same single-CTA tiles
# ----------------------------------------------------------------------------------------------
GEMM_SHAPES = [
    # M, N, K, bn, ctas
    (128, 256, 64, 256, 1),       # one tile, one k-block
    (128, 256, 256, 256, 1),      # k loop within one pipeline round
    (300, 256, 1408, 256, 1),     # M tail, pipeline wraps (22 k-blocks)
    (512, 512, 592, 256, 1),      # K tail (592 = 9*64 + 16)
    (257, 1408, 1408, 176, 1),    # BN=176 (proj / fc2)
    (257, 4224, 1408, 192, 1),    # BN=192 (ViT qkv)
    (1000, 768, 768, 128, 1),
    (96, 96, 768, 64, 1),         # N tail inside a 64-wide tile (scalar store path)
    (64, 32, 768, 32, 1),         # z projection
    (4096, 1024, 256, 32, 1),     # 1024 tiles over 132 CTAs: >= 7 tiles per persistent CTA
    (2048, 40194, 512, 256, 1),   # lm_head-like: odd ldo -> unaligned rows, N tail
    (512, 512, 1408, 256, 2),
    (300, 256, 592, 256, 2),
    (1028, 4224, 1408, 192, 2),
    (1028, 1408, 1408, 176, 2),
    (1000, 768, 768, 128, 2),
    (4096, 1024, 256, 64, 2),
    (1028, 1408, 1408, 256, 2),   # ragged N: 5 full tiles + a half-empty last column
    (513, 1408, 6144, 256, 2),    # same with a long reduction (fc2)
    (300, 40194, 512, 256, 2),    # last column holds 2 columns (lm_head)
    (300, 1000, 768, 256, 1),     # last column 232 of 256 wide
    (200, 272, 256, 256, 1),      # last column 16 of 256 wide
]


@pytest.mark.parametrize("M,N,K,bn,ctas", GEMM_SHAPES)
def test_gemm_plain(lib, M, N, K, bn, ctas):
    a = rand16(M, K, seed=1)
    w = rand16(N, K, scale=K ** -0.5, seed=2)
    out = lib.gemm(a, w, bn=bn, ctas=ctas)
    torch.cuda.synchronize()
    ref = R.linear_ref(a, w)
    # tolerance: 2 fp16 ulps of the output (fp32 accumulation order differs from the oracle's)
    assert rel_err(out, ref) < 1e-3, rel_err(out, ref)
    assert_close16(out, ref, what="gemm")


# a 256-token prompt on the 13B shapes: the plan picks 128-wide tiles when 256-wide ones leave most SMs idle; the M = 2048 shapes keep the 256-wide tiling.  K kept short so the fp32 oracle stays cheap
PLANNED_SHAPES = [(256, 5120, 320), (256, 15360, 128), (200, 5120, 192), (2048, 4096, 320), (2048, 5120, 192)]


@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("M,N,K", PLANNED_SHAPES)
def test_gemm_planned_tilings(lib, M, N, K, residual):
    a = rand16(M, K, seed=21)
    w = rand16(N, K, scale=K ** -0.5, seed=22)
    res = rand16(M, N, seed=23) if residual else None
    out = lib.gemm(a, w, residual=res, ctas=2)
    torch.cuda.synchronize()
    ref = R.linear_ref(a, w, None, 0, res)
    assert_close16(out, ref, mags=(R.linear_ref(a, w),) + ((res,) if residual else ()), ulps=3.0, what="planned gemm")
    # ... and the fixed heuristics (option off) give bit-identical results: the tiling never changes the k order
    lib.set_option("gemm_sched", 0)
    try:
        out0 = lib.gemm(a, w, residual=res, ctas=2)
        torch.cuda.synchronize()
    finally:
        lib.set_option("gemm_sched", 1)
    assert torch.equal(out, out0)


@pytest.mark.parametrize("bn", [192, 256, 128])
def test_gemm_balanced_tail_order_with_explicit_width(lib, bn):
    M, N, K = 2048, 4096, 256
    a = rand16(M, K, seed=24)
    w = rand16(N, K, scale=K ** -0.5, seed=25)
    bias = rand16(N, scale=0.5, seed=26)
    ref = lib.gemm(a, w, bias=bias, bn=256, ctas=2)
    lib.set_option("gemm_sched", 2)
    try:
        out = lib.gemm(a, w, bias=bias, bn=bn, ctas=2)
        torch.cuda.synchronize()
    finally:
        lib.set_option("gemm_sched", 1)
    assert torch.equal(out, ref)
    assert_close16(out, R.linear_ref(a, w, bias), what="balanced tail")


@pytest.mark.parametrize("act", [0, 1, 2, 3])
@pytest.mark.parametrize("ctas", [1, 2])
def test_gemm_bias_act_residual(lib, act, ctas):
    M, N, K = 515, 768, 320
    a = rand16(M, K, seed=3)
    w = rand16(N, K, scale=K ** -0.5, seed=4)
    bias = rand16(N, scale=0.5, seed=5)
    res = rand16(M, N, seed=6)
    out = lib.gemm(a, w, bias=bias, act=act, residual=res, ctas=ctas)
    torch.cuda.synchronize()
    ref = R.linear_ref(a, w, bias, act, res)
    pre = R.linear_ref(a, w, bias)            # fp16-rounded pre-activation
    post = R.linear_ref(a, w, bias, act)      # fp16-rounded activation output (before the residual add)
    # a 1-ulp flip of an fp16-rounded intermediate survives into the result: 4 ulps of the largest magnitude
    assert_close16(out, ref, mags=(pre, post, res), ulps=4.0, what=f"gemm act={act}")


def test_gemm_inplace_residual(lib):
    M, N, K = 514, 1408, 1408
    a = rand16(M, K, seed=7)
    w = rand16(N, K, scale=K ** -0.5, seed=8)
    bias = rand16(N, scale=0.1, seed=9)
    x = rand16(M, N, seed=10)
    ref = R.linear_ref(a, w, bias, 0, x)
    out = lib.gemm(a, w, bias=bias, residual=x, out=x)
    torch.cuda.synchronize()
    assert out.data_ptr() == x.data_ptr()
    assert_close16(out, ref, mags=(R.linear_ref(a, w, bias),), ulps=3.0, what="inplace residual")


def test_gemm_row_remap_patch_embed(lib):
    """patch rows land behind each image's cls row and pick up pos_embed[1 + patch] (eva_vit.py:373-377)."""
    B = 3
    a = rand16(B * 256, 592, seed=11)
    a[:, 588:] = 0
    w = rand16(1408, 592, scale=588 ** -0.5, seed=12)
    bias = rand16(1408, scale=0.1, seed=13)
    pos = rand16(257, 1408, scale=0.1, seed=14)
    x = torch.zeros((B * 257, 1408), dtype=torch.float16, device=DEV)
    lib.gemm(a, w, bias=bias, residual=pos, out=x, row_group=256, row_stride=257, row_offset=1, res_mod=256,
             res_offset=1)
    torch.cuda.synchronize()
    y = R.linear_ref(a, w, bias).float().reshape(B, 256, 1408)
    ref = R.r16(y + pos[1:].float()[None])
    got = x.reshape(B, 257, 1408)
    assert (got[:, 0] == 0).all()                      # cls rows untouched
    assert_close16(got[:, 1:], ref, mags=(y,), ulps=3.0, what="patch embed")


@pytest.mark.parametrize("ctas", [1, 2])
@pytest.mark.parametrize("M,ffn,h", [(300, 1408, 512), (2048, 11008, 256)])
def test_gemm_silu_gate(lib, M, ffn, h, ctas):
    a = rand16(M, h, seed=15)
    wg = rand16(ffn, h, scale=h ** -0.5, seed=16)
    wu = rand16(ffn, h, scale=h ** -0.5, seed=17)
    wgu = R.interleave_gate_up(wg, wu)
    out = lib.gemm(a, wgu, mode=1, ctas=ctas)
    torch.cuda.synchronize()
    ref = R.silu_gate_ref(a, wg, wu)
    assert out.shape == (M, ffn)
    g = R.linear_ref(a, wg); u = R.linear_ref(a, wu)
    # out = silu(g)*u: a 1-ulp flip of g or u moves the product by |u| or |g| ulps -> bound by |g*u| + |u| + |g|
    assert_close16(out, ref, mags=(g.float() * u.float(), 0.5 * u.float(), 0.5 * g.float()), ulps=4.0, what="silu gate")


def test_gemm_rejects_bad_args(lib):
    a = rand16(64, 100, seed=1)          # K not a multiple of 8
    w = rand16(32, 100, seed=2)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        lib.gemm(a, w)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        lib.gemm(a.cpu(), w.cpu())


# ----------------------------------------------------------------------------------------------
# norms
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols,eps", [(257, 1408, 1e-6), (1028, 1408, 1e-5), (64, 768, 1e-12), (1, 768, 1e-6),
                                           (33, 256, 1e-6), (7, 4096, 1e-5)])
def test_layernorm(lib, rows, cols, eps):
    x = rand16(rows, cols, scale=2.0, seed=20) + 0.5
    w = (1.0 + 0.1 * torch.randn(cols)).to(torch.float16).to(DEV)
    b = (0.1 * torch.randn(cols)).to(torch.float16).to(DEV)
    y = lib.layernorm(x, w, b, eps)
    torch.cuda.synchronize()
    ref = R.layernorm_ref(x, w, b, eps)
    # fp32 statistics on both sides: 1 fp16 ulp (+ floor near zero)
    assert_close16(y, ref, ulps=1.5, atol=1e-4, what="layernorm")


@pytest.mark.parametrize("rows,cols", [(2048, 4096), (5, 5120), (1, 4096), (300, 512)])
def test_rmsnorm(lib, rows, cols):
    x = rand16(rows, cols, scale=1.5, seed=21)
    w = (1.0 + 0.1 * torch.randn(cols)).to(torch.float16).to(DEV)
    y = lib.rmsnorm(x, w, 1e-6)
    torch.cuda.synchronize()
    ref = R.rmsnorm_ref(x, w, 1e-6)
    assert_close16(y, ref, ulps=2.5, atol=1e-4, what="rmsnorm")


# ----------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------
ATTN_CASES = [
    # B, H, Nq, Nk, D, causal
    (2, 16, 257, 257, 88, False),     # ViT-g
    (3, 12, 32, 32, 64, True),        # Q-Former self (causal)
    (3, 12, 32, 257, 64, False),      # Q-Former cross
    (2, 12, 32, 32, 64, False),       # de-tokenizer blocks
    (1, 4, 300, 300, 128, True),      # LLaMA prefill
    (2, 2, 2048, 2048, 128, True),
    (1, 2, 5, 133, 128, True),        # chunked prefill with past: bottom-right aligned causal
    (2, 8, 100, 200, 128, True),      # 100 new tokens after a 100-token past (8-warp tile, nk != nq)
    (1, 2, 130, 300, 128, True),
    (1, 3, 512, 640, 128, True),      # two 128-row query tiles after a 128-token past
    (2, 5, 257, 257, 128, True),      # ragged second pair (one row)
    (1, 2, 128, 128, 128, True),      # single tile, second tile of the pair absent
    (1, 40, 1024, 1024, 128, True),   # 160 (head, query tile) items and more
    (1, 3, 1, 77, 128, False),        # single query through the prefill kernel
    (1, 2, 100, 100, 64, False),
]


@pytest.mark.parametrize("B,H,Nq,Nk,D,causal", ATTN_CASES)
def test_attention(lib, B, H, Nq, Nk, D, causal):
    q = rand16(B, H, Nq, D, seed=30)
    k = rand16(B, H, Nk, D, seed=31)
    v = rand16(B, H, Nk, D, seed=32)
    scale = D ** -0.5
    o = lib.attention(q, k, v, scale, causal)
    torch.cuda.synchronize()
    ref = R.attention_ref(q, k, v, scale, causal)
    # probabilities are rounded to fp16 before P.V (as the reference does): relative Frobenius 2e-3
    assert rel_err(o, ref) < 2e-3, rel_err(o, ref)
    assert (o.float() - ref.float()).abs().max().item() < 1e-2
    # ... and every query row on its own, so that one wrong row (a ragged last tile) is not averaged away: 2^-11
    # relative for the fp16 probabilities and 2 x 2^-12 for the two fp16 outputs, typically; 4e-3 leaves room for the
    # worst of up to 80k rows
    row_err = (o.float() - ref.float()).norm(dim=-1) / ref.float().norm(dim=-1).clamp_min(1e-6)
    assert row_err.max().item() < 4e-3, (row_err.max().item(), tuple(int(i) for i in (row_err == row_err.max()).nonzero()[0]))


@pytest.mark.parametrize("B", [1, 2, 3, 5, 8, 13, 40, 64, 100])
def test_vit_attention_packed_qkv_batches(lib, B):
    """the 257x257x88 ViT shape read from the packed [B*257, 3*16*88] qkv GEMM output; B=40..100 give 640..1600
    (image, head) items, several waves of CTAs"""
    H, N, D = 16, 257, 88
    qkv = rand16(B * N, 3 * H * D, seed=34)
    v4 = qkv.view(B, N, 3, H, D)
    q, k, v = (v4[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    ref = R.attention_ref(q, k, v, D ** -0.5, False)
    o = lib.attention(q, k, v, D ** -0.5, False)
    torch.cuda.synchronize()
    assert rel_err(o, ref) < 2e-3, rel_err(o, ref)
    assert (o.float() - ref.float()).abs().max().item() < 1e-2
    # the 257th query row sits alone in the last query tile: check it on its own
    assert rel_err(o[:, 256], ref[:, 256]) < 2e-3


def test_vit_attention_large_scores(lib):
    """scores up to ~+-60 (peaked softmax, fp16 P underflow in the tail) at head_dim 88 against the fp32 reference"""
    B, H, N, D = 3, 16, 257, 88
    q = rand16(B, H, N, D, scale=3.0, seed=71)
    k = rand16(B, H, N, D, scale=3.0, seed=72)
    v = rand16(B, H, N, D, seed=73)
    ref = R.attention_ref(q, k, v, D ** -0.5, False)
    o = lib.attention(q, k, v, D ** -0.5, False)
    torch.cuda.synchronize()
    assert rel_err(o, ref) < 3e-3, rel_err(o, ref)


@pytest.mark.parametrize("B,S,past,max_seq", [(2, 700, 333, 1200), (1, 2048, 0, 2048), (3, 130, 7, 200),
                                              (1, 128, 0, 128), (1, 129, 64, 256), (2, 256, 1, 300),
                                              (1, 1000, 1048, 2048), (4, 64, 500, 600), (1, 513, 2, 1024)])
def test_causal_attention_prefill_cache_layout(lib, B, S, past, max_seq):
    """LLaMA prefill layout: q sliced from a fused projection buffer, K/V from a [B,H,max_seq,D] cache holding a past;
    the cache rows behind the sequence are NaN, so any read of them that reaches the MMAs shows in the output"""
    H, D = 4, 128
    qbuf = rand16(B * S, H * D, seed=35)
    kc = rand16(B, H, max_seq, D, seed=36)
    vc = rand16(B, H, max_seq, D, seed=37)
    q = qbuf.view(B, S, H, D).permute(0, 2, 1, 3)
    k, v = kc[:, :, :past + S], vc[:, :, :past + S]
    kc[:, :, past + S:] = float("nan")          # rows past the sequence must never reach the MMAs
    vc[:, :, past + S:] = float("nan")
    o = lib.attention(q, k, v, D ** -0.5, True)
    torch.cuda.synchronize()
    ref = R.attention_ref(q, k, v, D ** -0.5, True)
    assert torch.isfinite(o.float()).all()
    assert rel_err(o, ref) < 2e-3, rel_err(o, ref)
    assert (o.float() - ref.float()).abs().max().item() < 1e-2


def test_causal_attention_large_scores_rescale(lib):
    """scores that grow along the sequence force the lazy O-rescaling branch (row max jumps by > 2^8 between tiles)"""
    B, H, S, D = 1, 2, 512, 128
    q = rand16(B, H, S, D, seed=38)
    k = rand16(B, H, S, D, seed=39)
    v = rand16(B, H, S, D, seed=40)
    ramp = torch.linspace(0.2, 6.0, S, device=DEV, dtype=torch.float32)[None, None, :, None]
    k = (k.float() * ramp).to(torch.float16)
    q = (q.float() * 2.0).to(torch.float16)
    o = lib.attention(q, k, v, D ** -0.5, True)
    torch.cuda.synchronize()
    ref = R.attention_ref(q, k, v, D ** -0.5, True)
    assert torch.isfinite(o.float()).all()
    assert rel_err(o, ref) < 3e-3, rel_err(o, ref)


def test_attention_strided_qkv_layout(lib):
    """the ViT layout: q/k/v are column slices of one [B*257, 4224] GEMM output."""
    B, H, N, D = 2, 16, 257, 88
    qkv = rand16(B * N, 3 * H * D, seed=33)
    v4 = qkv.view(B, N, 3, H, D)
    q, k, v = (v4[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    o = lib.attention(q, k, v, D ** -0.5, False)
    torch.cuda.synchronize()
    ref = R.attention_ref(q, k, v, D ** -0.5, False)
    assert rel_err(o, ref) < 2e-3


# ----------------------------------------------------------------------------------------------
# VQ argmin: bit-exact against the C oracle, both arithmetic modes
# ----------------------------------------------------------------------------------------------
def _oracle_vq(z, cb, mode):
    from seed_b200.build import ORACLE_LIB, build_oracle

    if not os.path.exists(ORACLE_LIB):
        build_oracle()
    o = C.CDLL(ORACLE_LIB)
    zn = z.cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
    cn = cb.cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
    ids = np.zeros(zn.shape[0], dtype=np.int64)
    margin = np.zeros(zn.shape[0], dtype=np.float32)
    rc = o.vq_oracle_argmin(zn.ctypes.data_as(C.c_void_p), cn.ctypes.data_as(C.c_void_p), zn.shape[0], cn.shape[0],
                            zn.shape[1], mode, ids.ctypes.data_as(C.c_void_p), margin.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return ids, margin


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n,n_codes,scale", [(64, 8192, 0.26), (1000, 8192, 0.26), (33, 1000, 1.0), (256, 8192, 1.0 / 8192)])
def test_vq_bit_exact_vs_c_oracle(lib, mode, n, n_codes, scale):
    z = rand16(n, 32, scale=0.26, seed=40)
    cb = rand16(n_codes, 32, scale=scale, seed=41)
    if scale < 1e-3:   # the reference's default init U(+-1/8192): every distance collapses, ties everywhere
        cb = ((torch.rand(n_codes, 32) * 2 - 1) / 8192).to(torch.float16).to(DEV)
    ids = lib.vq_argmin(z, cb, mode)
    torch.cuda.synchronize()
    ref, _ = _oracle_vq(z, cb, mode)
    assert ids.dtype == torch.int64
    assert np.array_equal(ids.cpu().numpy(), ref)


def test_vq_duplicate_codes_pick_lowest_index(lib):
    z = rand16(128, 32, scale=0.3, seed=42)
    cb = rand16(512, 32, scale=0.3, seed=43)
    cb = torch.cat([cb, cb, cb], dim=0).contiguous()      # every code three times
    for mode in (0, 1):
        ids = lib.vq_argmin(z, cb, mode)
        assert (ids < 512).all()


# ----------------------------------------------------------------------------------------------
# patchify, embedding, RoPE + KV append
# ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1])
def test_vq_code_split_path_equals_the_single_cta_walk(lib, mode):
    """few rows (a single image = 32 rows): the codebook is split over CTAs and the winners meet through a 64-bit
    atomicMin on the (d, id) key; the same rows inside a full batch take the one-CTA walk -- identical ids, ties and
    degenerate rows included"""
    cb = rand16(8192, 32, scale=0.26, seed=83)
    cb[4000] = cb[17]                               # duplicates in different splits: the lower index must win
    cb[8191] = cb[300]
    z = rand16(8192, 32, scale=0.3, seed=84)
    z[3] = cb[17]
    z[5] = cb[300]
    z[7] = float("inf")                             # every distance inf / NaN: id 0 on both paths
    full = lib.vq_argmin(z, cb, mode=mode)          # 256 row blocks: no split
    for n in (32, 33, 64, 700):
        part = lib.vq_argmin(z[:n].contiguous(), cb, mode=mode)
        torch.cuda.synchronize()
        assert torch.equal(part, full[:n]), n
    assert full[3].item() == 17 and full[5].item() == 300 and full[7].item() == 0


def test_patchify_exact(lib):
    img = rand16(3, 3, 224, 224, seed=50)
    cols = lib.patchify(img, 592)
    torch.cuda.synchronize()
    assert torch.equal(cols, R.patchify_ref(img, 592))


def test_embedding_exact(lib):
    table = rand16(1000, 4096, seed=51)
    ids = torch.randint(0, 1000, (3, 77), device=DEV)
    out = lib.embedding(table, ids)
    torch.cuda.synchronize()
    assert torch.equal(out, table[ids.reshape(-1)])


@pytest.mark.parametrize("B,S,H,past", [(1, 64, 4, 0), (2, 17, 3, 5), (1, 1, 8, 300)])
def test_rope_kv_append(lib, B, S, H, past):
    D, max_seq = 128, 512
    qkv = rand16(B * S, 3 * H * D, seed=52)
    pos = (past + torch.arange(S, device=DEV))[None].expand(B, S).contiguous()
    kc = torch.zeros((B, H, max_seq, D), dtype=torch.float16, device=DEV)
    vc = torch.zeros_like(kc)
    q_out = lib.rope_kv_append(qkv, pos, B, S, H, D, past, kc, vc)
    torch.cuda.synchronize()
    v5 = qkv.view(B, S, 3, H, D)
    q, k, v = (v5[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    q_ref = R.rope_ref(q, pos).permute(0, 2, 1, 3).reshape(B * S, H * D)
    k_ref = R.rope_ref(k, pos)
    # cos/sin come from the device's cosf/sinf instead of torch's: allow 2 fp16 ulps
    assert (q_out.float() - q_ref.float()).abs().max().item() < 2e-2
    assert rel_err(q_out, q_ref) < 1e-3, rel_err(q_out, q_ref)
    assert rel_err(kc[:, :, past:past + S], k_ref) < 1e-3
    assert torch.equal(vc[:, :, past:past + S], v)
    assert (kc[:, :, past + S:] == 0).all() and (kc[:, :, :past] == 0).all()
    # positions=None means past_len + arange(S) (llama_xformer.py:530-539)
    kc2 = torch.zeros_like(kc); vc2 = torch.zeros_like(vc)
    q2 = lib.rope_kv_append(qkv, None, B, S, H, D, past, kc2, vc2)
    assert torch.equal(q2, q_out) and torch.equal(kc2, kc)


# ----------------------------------------------------------------------------------------------
# decode-step kernels at the LLaMA-13B / 7B bench shapes (seedb200_gemv, seedb200_decode_attention)
# ----------------------------------------------------------------------------------------------
GEMV_SHAPES = [
    # M, N, K, what
    (1, 15360, 5120, "13B fused qkv"),
    (1, 5120, 5120, "13B o_proj"),
    (1, 5120, 13824, "13B down_proj"),
    (1, 40194, 5120, "13B lm_head (odd N: last row pair is a single row)"),
    (1, 12288, 4096, "7B fused qkv"),
    (1, 4096, 11008, "7B down_proj"),
    (4, 5120, 13824, "4 activation rows"),
    (3, 1000, 264, "tails: N not a multiple of the CTA's 8 row pairs, K < one warp pass"),
]


@pytest.mark.parametrize("M,N,K,what", GEMV_SHAPES)
@pytest.mark.parametrize("variant", ["plain", "residual", "rmsnorm"])
def test_gemv_decode_shapes(lib, M, N, K, what, variant):
    """y = x W^T (+ residual) with the fp16 rounding points of nn.Linear on fp16 tensors (llama_xformer.py:223-225,
    258,718); `rmsnorm`: LlamaRMSNorm fused into the activation staging (llama_xformer.py:105-113)."""
    x = rand16(M, K, seed=11)
    w = rand16(N, K, scale=K ** -0.5, seed=12)
    res = rand16(M, N, seed=13) if variant == "residual" else None
    nw = (1.0 + 0.1 * torch.randn(K, generator=torch.Generator().manual_seed(14))).half().to(DEV) if variant == "rmsnorm" else None
    out = lib.gemv(x, w, residual=res, norm_w=nw, eps=1e-6)
    xin = R.rmsnorm_ref(x, nw, 1e-6) if nw is not None else x
    ref = R.linear_ref(xin, w, residual=res)
    mags = [R.linear_ref(xin, w)] if res is not None else []
    assert_close16(out, ref, mags=mags, ulps=2.0, what=f"gemv {what} {variant}")


@pytest.mark.parametrize("M,ffn,K", [(1, 13824, 5120), (1, 11008, 4096), (2, 256, 512)])
def test_gemv_silu_gate(lib, M, ffn, K):
    """LlamaMLP.forward (llama_xformer.py:186): silu(gate_proj(x)) * up_proj(x) over the interleaved [128 gate | 128 up]
    weight, RMSNorm fused (the decode form of post_attention_layernorm + MLP input)."""
    x = rand16(M, K, seed=21)
    wg = rand16(ffn, K, scale=K ** -0.5, seed=22)
    wu = rand16(ffn, K, scale=K ** -0.5, seed=23)
    nw = (1.0 + 0.1 * torch.randn(K, generator=torch.Generator().manual_seed(24))).half().to(DEV)
    out = lib.gemv(x, R.interleave_gate_up(wg, wu), norm_w=nw, eps=1e-6, mode=1)
    xin = R.rmsnorm_ref(x, nw, 1e-6)
    ref = R.silu_gate_ref(xin, wg, wu)
    g = R.linear_ref(xin, wg).float()
    u = R.linear_ref(xin, wu).float()
    # a 1-ulp flip of fp16(gate) or fp16(up) moves the product by ~ulp(g)*|u| or ulp(u)*|s|
    assert_close16(out, ref, mags=[g.abs() * u.abs(), u], ulps=3.0, what="gemv silu-gate")


@pytest.mark.parametrize("B,H,kv_len,max_seq", [(1, 40, 257, 392), (1, 40, 300, 392), (1, 32, 1024, 1024),
                                                (2, 8, 1, 64), (1, 4, 128, 128), (1, 4, 129, 8300), (1, 2, 8200, 8300)])
def test_decode_attention_cache_lengths(lib, B, H, kv_len, max_seq):
    """one query token against the first kv_len rows of a [B,H,max_seq,128] cache, no mask
    (llama_xformer.py:240-256 with attn_bias=None); fp32 softmax, fp16 output."""
    D = 128
    q = rand16(B, H, D, seed=31)
    kc = rand16(B, H, max_seq, D, seed=32)
    vc = rand16(B, H, max_seq, D, seed=33)
    scale = D ** -0.5
    out = lib.decode_attention(q, kc, vc, kv_len, scale)
    ref = R.attention_ref(q[:, :, None, :], kc[:, :, :kv_len], vc[:, :, :kv_len], scale)     # [B,1,H,D]
    assert_close16(out.view(B, H, D), ref.view(B, H, D), ulps=2.0, atol=2e-4, what=f"decode attention kv={kv_len}")


@pytest.mark.parametrize("B,H,past,max_seq,use_pos", [(1, 40, 256, 392, False), (1, 40, 299, 392, True), (2, 8, 0, 64, False),
                                                      (1, 4, 127, 128, False), (1, 4, 128, 512, True), (3, 5, 511, 512, False),
                                                      (1, 8, 1500, 2048, False), (2, 4, 600, 1100, True)])
def test_decode_attention_rope_fused_matches_the_two_kernel_form(lib, B, H, past, max_seq, use_pos):
    """RoPE + KV append + attention in one launch (the cached decode step) vs rope_kv_append -> decode_attention on the
    same inputs: caches identical, output bit-identical while one 128-key block per thread group covers the cache
    (<= 512 keys), within 2 fp16 ulps beyond; both against the fp32 oracle (llama_xformer.py:152-161,234-256)."""
    D = 128
    qkv = rand16(B, 3 * H * D, seed=61)
    kc = rand16(B, H, max_seq, D, seed=62)
    vc = rand16(B, H, max_seq, D, seed=63)
    kc[:, :, past:] = 0
    vc[:, :, past:] = 0
    kc2, vc2 = kc.clone(), vc.clone()
    pos = torch.full((B, 1), past, dtype=torch.int64, device=DEV)
    if use_pos:
        pos = pos - torch.arange(B, device=DEV)[:, None].clamp(max=past)       # left-padded rows: position < cache row
    scale = D ** -0.5
    q_rot = lib.rope_kv_append(qkv, pos, B, 1, H, D, past, kc, vc)
    ref2 = lib.decode_attention(q_rot.view(B, H, D), kc, vc, past + 1, scale)
    out = lib.decode_attention_rope(qkv, pos if use_pos else None, H, past, kc2, vc2, scale)
    torch.cuda.synchronize()
    assert torch.equal(kc, kc2) and torch.equal(vc, vc2)
    if past + 1 <= 512:
        assert torch.equal(out, ref2)
    assert_close16(out, ref2, ulps=2.0, atol=2e-4, what="fused vs two-kernel decode attention")
    v5 = qkv.view(B, 1, 3, H, D)
    q = R.rope_ref(v5[:, :, 0].permute(0, 2, 1, 3), pos)
    ref = R.attention_ref(q, kc[:, :, :past + 1], vc[:, :, :past + 1], scale)
    assert_close16(out.view(B, H, D), ref.view(B, H, D), ulps=3.0, atol=4e-4, what="fused decode attention")


def test_decode_attention_rope_rejects_long_caches(lib):
    qkv = rand16(1, 3 * 2 * 128, seed=64)
    kc = torch.zeros((1, 2, 2049, 128), dtype=torch.float16, device=DEV)
    with pytest.raises(RuntimeError, match="max_seq"):
        lib.decode_attention_rope(qkv, None, 2, 5, kc, kc.clone(), 0.1)


# ----------------------------------------------------------------------------------------------
# token side of the generation loop: sampler and id -> token arithmetic
# ----------------------------------------------------------------------------------------------
def test_sampler_greedy_is_torch_argmax(lib):
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(4, 40194, generator=g) * 2).half()
    logits[1, 777] = logits[1].max() + 1
    logits[1, 30000] = logits[1, 777]                 # tie: the lowest index wins (torch.argmax)
    logits[2, :] = 0.0                                # all equal -> 0
    logits[3, 40193] = 100.0                          # last column
    pad = torch.zeros(4, 40200, dtype=torch.float16)  # padded row stride, as the generate loop uses
    pad[:, :40194] = logits
    got = lib.sample(pad.to(DEV)[:, :40194])
    assert got.dtype == torch.int64
    assert got.cpu().tolist() == [int(logits[0].float().argmax()), 777, 0, 40193]


@pytest.mark.parametrize("V,T,P", [(40194, 1.0, 0.5), (40194, 0.7, 0.9), (1000, 1.3, 0.05), (50, 1.0, 1.0), (5120, 1.0, 0.97)])
def test_sampler_matches_oracle_draw_by_draw(lib, V, T, P):
    """temperature / top-p / inverse-CDF draw vs oracle/sampler_oracle.py (HF TemperatureLogitsWarper +
    TopPLogitsWarper semantics, pinned to transformers on the CPU side); same Philox uniforms.  A draw whose uniform
    lands within 1e-5 of a CDF edge, or a nucleus whose boundary token is within 2e-6 of the threshold, may differ
    by fp32 summation order and is excluded (counted)."""
    from oracle import sampler_oracle as S

    g = torch.Generator().manual_seed(V + int(P * 1000))
    B = 64
    logits = (torch.randn(B, V, generator=g) * 3.0).half()
    seed, offset, step = 0x1234ABCD5678, 1000, 7
    got = lib.sample(logits.to(DEV), do_sample=True, temperature=T, top_p=P, seed=seed, offset=offset, step=step).cpu()
    checked, bad = 0, []
    for b in range(B):
        tok, dmargin, nmargin = S.sample_ref(logits[b].float().numpy(), True, T, P, seed, offset, step, b)
        if dmargin < 1e-5 or nmargin < 2e-6:
            continue
        checked += 1
        if int(got[b]) != tok:
            bad.append((b, int(got[b]), tok, dmargin, nmargin))
    assert not bad, bad[:8]
    assert checked >= B // 2, checked


def test_sampler_distribution_and_nucleus(lib):
    """4096 sequences with identical logits draw independently (Philox counter = row): sampled tokens stay inside
    HF's nucleus and their frequencies match the warped distribution."""
    from oracle import sampler_oracle as S

    V, T, P, B = 40, 0.9, 0.8, 4096
    base = (torch.randn(V, generator=torch.Generator().manual_seed(9)) * 2.0).half()
    logits = base[None].expand(B, V).contiguous()
    got = lib.sample(logits.to(DEV), do_sample=True, temperature=T, top_p=P, seed=42, offset=0, step=0).cpu()
    q, keep, _ = S.warp(base.float().numpy(), T, P)
    assert keep[got.numpy()].all()
    freq = np.bincount(got.numpy(), minlength=V) / B
    assert np.abs(freq - q).max() < 4.0 * np.sqrt(q.max() * (1 - q.max()) / B) + 1e-3, np.abs(freq - q).max()
    # another step -> another draw; same (seed, offset, step) -> the same draw
    again = lib.sample(logits.to(DEV), do_sample=True, temperature=T, top_p=P, seed=42, offset=0, step=0).cpu()
    other = lib.sample(logits.to(DEV), do_sample=True, temperature=T, top_p=P, seed=42, offset=0, step=1).cpu()
    assert torch.equal(again, got) and not torch.equal(other, got)


def test_image_ids_to_tokens_kernel(lib):
    """scripts/seed_llama_inference_8B.py:16-23,60,98-100: '<img>' + '<img_%05d>' x 32 + '</img>' as id arithmetic."""
    ids = torch.randint(0, 8192, (5, 32), generator=torch.Generator().manual_seed(1))
    toks = lib.image_ids_to_tokens(ids.to(DEV), 32000, 40192, 40193).cpu()
    assert tuple(toks.shape) == (5, 34)
    assert (toks[:, 0] == 40192).all() and (toks[:, 33] == 40193).all() and torch.equal(toks[:, 1:33], ids + 32000)
    # spans written straight into a prompt buffer (row stride 40)
    buf = torch.full((5, 40), -1, dtype=torch.int64, device=DEV)
    lib.image_ids_to_tokens(ids.to(DEV), 32000, 40192, 40193, out=buf)
    assert torch.equal(buf[:, :34].cpu(), toks) and (buf[:, 34:] == -1).all()


# ----------------------------------------------------------------------------------------------
# LayerNorm folded into the consuming GEMM (seedb200_gemm_desc.ln_stats): norm1 -> qkv, norm2 -> fc1
# ----------------------------------------------------------------------------------------------
def test_row_stats_match_torch_layernorm_statistics(lib):
    x = rand16(1000, 1408, scale=2.0, seed=81) + 0.5
    st = lib.row_stats(x, 1e-6)
    xf = x.float()
    mean = xf.mean(-1)
    rstd = torch.rsqrt(xf.var(-1, unbiased=False) + 1e-6)
    assert torch.allclose(st[:, 0], mean, rtol=0, atol=2e-6 * xf.abs().max().item())
    assert torch.allclose(st[:, 1], rstd, rtol=2e-6, atol=0)


@pytest.mark.parametrize("M,N,K,act,ctas", [(1028, 4224, 1408, 0, 2), (1028, 6144, 1408, 1, 2), (300, 512, 768, 0, 1),
                                            (2056, 1408, 1408, 1, 2)])
def test_gemm_layernorm_folded(lib, M, N, K, act, ctas):
    """linear(LayerNorm(x), W, bias) [+ GELU] without materialising LayerNorm(x): W' = fp16(W gamma) as the operand,
    rstd * (acc - mean * c) + b' in the epilogue (eva_vit.py:201-202 with :133-135 / :60-65).  The reference rounds
    LN(x) to fp16 before the GEMM; here W gamma is rounded instead -- the two differ by a few fp16 ulps of the
    output (both are one rounding of one operand), and both sit equally close to the fp32 value."""
    g = torch.Generator().manual_seed(82)
    x = (torch.randn(M, K, generator=g) * 1.5 + 0.3 * torch.randn(M, 1, generator=g)).half().to(DEV)
    x[:, 7] += 20.0                                            # an outlier channel, as real ViT activations have
    w = rand16(N, K, scale=K ** -0.5, seed=83)
    gamma = (1.0 + 0.2 * torch.randn(K, generator=g)).half().to(DEV)
    beta = (0.1 * torch.randn(K, generator=g)).half().to(DEV)
    bias = rand16(N, scale=0.1, seed=84)
    wf, c, bf = lib.ln_fold_weights(w, gamma, beta, bias)
    # the folded vectors are what they claim to be
    assert torch.equal(wf, (w.float() * gamma.float()).half())
    assert torch.allclose(c, wf.float().sum(-1), rtol=1e-5, atol=1e-4)
    assert torch.allclose(bf, w.float() @ beta.float() + bias.float(), rtol=1e-5, atol=1e-4)
    out = lib.gemm(x, wf, act=act, ctas=ctas, ln=(lib.row_stats(x, 1e-6), c, bf))
    ref16 = R.linear_ref(R.layernorm_ref(x, gamma, beta, 1e-6), w, bias, act)          # the reference's rounding points
    ref32 = torch.nn.functional.layer_norm(x.float(), (K,), gamma.float(), beta.float(), 1e-6) @ w.float().t() + bias.float()
    if act == 1:
        ref32 = torch.nn.functional.gelu(ref32)
    e_ours, e_ref = rel_err(out, ref32), rel_err(ref16, ref32)
    assert e_ours <= 1.5 * e_ref + 1e-4, (e_ours, e_ref)      # as close to exact arithmetic as the reference's own rounding
    assert rel_err(out, ref16) < 1.5e-3
    assert_close16(out, ref16, ulps=6.0, atol=2e-3, what="LN-folded GEMM vs rounding-point reference")


@pytest.mark.parametrize("M,N,K,ctas", [(2056, 1408, 1408, 2), (2056, 1408, 6144, 2), (300, 1408, 1408, 1), (257, 512, 768, 1)])
def test_gemm_row_moments_give_the_layernorm_statistics_of_the_output(lib, M, N, K, ctas):
    """x += linear(a) with the (sum, sum of squares) of every 64-column group of the NEW x left by the epilogue
    (seedb200_gemm_desc.row_moments): row_stats_from_moments == row_stats of the stored rows, so the next
    LayerNorm-folded GEMM does not have to re-read x (eva_vit.py:201-202)."""
    _check_row_moments(lib, M, N, K, ctas, 0)


# the last column of tiles reaches past N (320 = 256 + 64 with the planned 256-wide tiles, 1408 = 5.5 x 256): the groups
# beyond N belong to no row and must not be written -- not into the next row's slots, not behind the buffer
@pytest.mark.parametrize("M,N,K,bn", [(257, 320, 256, 0), (300, 1408, 1408, 256), (129, 1408, 512, 256)])
def test_gemm_row_moments_when_the_last_tile_reaches_past_n(lib, M, N, K, bn):
    _check_row_moments(lib, M, N, K, 1, bn)


def _check_row_moments(lib, M, N, K, ctas, bn):
    a = rand16(M, K, seed=85)
    w = rand16(N, K, scale=K ** -0.5, seed=86)
    bias = rand16(N, scale=0.1, seed=87)
    x = rand16(M, N, scale=2.0, seed=88) + 0.25
    x[:, 7] += 20.0
    plain = lib.gemm(a, w, bias, residual=x, ctas=ctas, bn=bn)
    mom_buf = torch.full((M + 1, N // 64, 2), float("nan"), dtype=torch.float32, device=DEV)
    mom = mom_buf[:M]                                          # one guard row behind the buffer the GEMM gets
    out = lib.gemm(a, w, bias, residual=x, out=x, ctas=ctas, bn=bn, row_moments=mom)   # in place, like proj / fc2
    torch.cuda.synchronize()
    assert torch.equal(out, plain)                             # the moments do not change the result
    assert not torch.isnan(mom).any()                          # every group slot was written
    assert torch.isnan(mom_buf[M]).all()                       # and nothing behind the last row
    of = out.float()
    assert torch.allclose(mom[:, :, 0].sum(-1), of.sum(-1), rtol=1e-5, atol=1e-2)
    assert torch.allclose(mom[:, :, 1].sum(-1), (of * of).sum(-1), rtol=1e-5, atol=1e-2)
    st = lib.row_stats_from_moments(mom, N, 1e-6)
    st2 = lib.row_stats(out, 1e-6)
    assert torch.allclose(st[:, 0], st2[:, 0], rtol=0, atol=4e-6 * of.abs().max().item())
    assert torch.allclose(st[:, 1], st2[:, 1], rtol=2e-5, atol=0)
    # same call twice: bit-identical moments (fixed slots, fixed order -- no atomics)
    x2 = rand16(M, N, scale=2.0, seed=88) + 0.25
    x2[:, 7] += 20.0
    mom2 = torch.empty_like(mom)
    lib.gemm(a, w, bias, residual=x2, out=x2, ctas=ctas, bn=bn, row_moments=mom2)
    torch.cuda.synchronize()
    assert torch.equal(mom, mom2)


def test_gemm_row_moments_refused_where_the_epilogue_cannot_provide_them(lib):
    a = rand16(64, 256, seed=89)
    w = rand16(96, 256, seed=90)
    mom = torch.empty((64, 1, 2), dtype=torch.float32, device=DEV)
    with pytest.raises(RuntimeError):
        lib.gemm(a, w, row_moments=mom)                        # N = 96 is not a multiple of 64
