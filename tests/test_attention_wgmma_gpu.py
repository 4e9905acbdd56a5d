"""Edges of the wgmma ViT attention kernel (non-causal, head_dim 88, nk <= 272 keys; attention.cu vit_attn_kernel):
key counts around its n256 + n16 chunks and one past the dispatch maximum (the mma.sync kernel), query counts around
its 64-row tiles, (image, head) item counts around the SM count (uneven items per persistent CTA), NaN-gapped views,
the packed-qkv layout at the bench shape and peaked scores, each against the float64 bound of test_kernel_edges_gpu."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import ops_ref as R  # noqa: E402
from edge_ref import DEV, assert_guards, rand16  # noqa: E402
from test_kernel_edges_gpu import attention_bound, gapped_heads, row_violations, run_attention  # noqa: E402

pytestmark = pytest.mark.gpu

D = 88
NK_MAX = 272          # the kernel's dispatch maximum (one n256 and one n16 wgmma chunk)


def check_gapped(lib, B, H, nq, nk, scale=D ** -0.5, qscale=1.0):
    q = gapped_heads(B, H, nq, D, 11)
    k = gapped_heads(B, H, nk, D, 12)
    v = gapped_heads(B, H, nk, D, 13)
    if qscale != 1.0:
        q, k = q * qscale, k * qscale
    obuf = run_attention(lib, q, k, v, scale, False)
    written = torch.zeros(obuf.shape, dtype=torch.bool, device=DEV)
    written[..., :D] = True
    assert_guards(obuf, written, "attention output")
    o64, tol = attention_bound(q, k, v, scale, False)
    n, worst, bound = row_violations(obuf[..., :D], o64, tol)
    assert n == 0, f"{n} query rows outside the bound; worst relative error {worst:.3e} (bound {bound:.3e})"


@pytest.mark.parametrize("nk", [1, 63, 64, 255, 256, 257, 258, NK_MAX, NK_MAX + 1])
def test_key_counts(lib, nk):
    check_gapped(lib, 2, 3, 257, nk)


@pytest.mark.parametrize("nq", [1, 64, 65, 256, 257, 300, 700])
def test_query_counts(lib, nq):
    check_gapped(lib, 2, 3, nq, 257)


@pytest.mark.parametrize("B,H", [(1, 5), (8, 16), (33, 4), (11, 25)])   # 5, 128, 132 (an H100's SMs), 275 items
def test_item_counts_around_the_sm_count(lib, B, H):
    check_gapped(lib, B, H, 257, 257)


def test_peaked_scores(lib):
    """queries and keys of scale 3 (scores up to ~60 after the 88^-0.5 scale): fp16 P underflows in the row tails"""
    check_gapped(lib, 2, 4, 257, 257, qscale=3.0)


def test_packed_qkv_bench_shape_row_by_row(lib):
    """the ViT layout at the bench batch: q / k / v are column slices of one [256 * 257, 3 * 16 * 88] buffer"""
    B, H, N = 256, 16, 257
    qkv = rand16(B * N, 3 * H * D, seed=81)
    v5 = qkv.view(B, N, 3, H, D)
    q, k, v = (v5[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    o = lib.attention(q, k, v, D ** -0.5, False)
    torch.cuda.synchronize()
    for b0 in range(0, B, 32):                   # the reference in slices of 32 images
        ref = R.attention_ref(q[b0:b0 + 32], k[b0:b0 + 32], v[b0:b0 + 32], D ** -0.5, False).float()
        got = o[b0:b0 + 32].float()
        assert torch.isfinite(got).all()
        row_err = (got - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-6)
        worst = row_err.max().item()
        assert worst < 4e-3, (b0, worst, tuple(int(i) for i in (row_err == row_err.max()).nonzero()[0]))


@pytest.mark.parametrize("nk", [1, 64, 200, 257, NK_MAX])
def test_same_bits_as_the_mma_sync_kernel(lib, nk):
    """K and V broadcast over the heads (head stride 0) take the mma.sync kernel, the same values materialised take
    the wgmma kernel: both follow one softmax arithmetic, so the outputs are bit-identical"""
    B, H, nq = 2, 4, 257
    q = gapped_heads(B, H, nq, D, 21)
    k1, v1 = rand16(B, 1, nk, D, seed=22), rand16(B, 1, nk, D, seed=23)
    k_b, v_b = k1.expand(B, H, nk, D), v1.expand(B, H, nk, D)
    o_mma = lib.attention(q, k_b, v_b, D ** -0.5, False)
    o_wgmma = lib.attention(q, k_b.contiguous(), v_b.contiguous(), D ** -0.5, False)
    torch.cuda.synchronize()
    assert torch.equal(o_mma.view(torch.int16), o_wgmma.view(torch.int16)), \
        int((o_mma.view(torch.int16) != o_wgmma.view(torch.int16)).sum())
