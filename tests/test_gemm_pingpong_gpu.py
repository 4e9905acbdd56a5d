"""The ping-pong GEMM (one 128 x 128 tile per consumer warpgroup) against the cooperative one: bit-identical outputs
over the mode-0 epilogue matrix, M / N / K tails, operand views with NaN padding, outputs in sentinel buffers, and
schedules that give a CTA one, two, three or many tiles (an odd count leaves one warpgroup a round short).  A few
cases are also bounded against the float64 reference."""
import os
import sys

import pytest
import torch

from oracle import ops_ref as R

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from edge_ref import (F64, act_extra, assert_guards, check16, gemm_tol, in_buffer, rand16, region,  # noqa: E402
                      sentinel_buffer, up8)

pytestmark = pytest.mark.gpu
EPILOGUES = ["none", "bias", "bias_gelu", "bias_tanh", "bias_relu", "ln", "ln_gelu", "residual_moments", "remap"]
MS = (1, 127, 128, 129, 257, 1028)


def _operands(M, N, K, seed):
    """A and W as views whose padding columns and trailing rows are NaN: any read past [M, K] / [N, K] shows"""
    _, a = in_buffer(rand16(M, K, scale=0.5, seed=seed), 8, 3)
    _, w = in_buffer(rand16(N, K, scale=K ** -0.5, seed=seed + 1), 16, 5)
    return a, w


def _run_both(lib, M, N, K, epi, seed):
    """-> (cooperative output buffer, ping-pong output buffer, rows written, moments pair or None)"""
    a, w = _operands(M, N, K, seed)
    bias = rand16(N, scale=0.5, seed=seed + 2)
    act = {"bias_gelu": 1, "bias_tanh": 2, "bias_relu": 3, "ln_gelu": 1}.get(epi, 0)
    kw = {"act": act}
    if epi.startswith("bias"):
        kw["bias"] = bias
    if epi.startswith("ln"):
        kw["ln"] = (lib.row_stats(a.contiguous(), 1e-6),
                    rand16(N, scale=0.1, seed=seed + 3).float(), rand16(N, scale=0.1, seed=seed + 4).float())
    rows = M
    if epi == "remap":
        # patch-embed layout: groups of 4 rows land behind one cls row, the residual is a 4-row table (pos_embed)
        kw.update(bias=bias, row_group=4, row_stride=5, row_offset=1, res_mod=4, res_offset=1)
        kw["residual"] = rand16(5, N, seed=seed + 5)
        rows = (M + 3) // 4 * 5 + 1
    outs, moms = [], []
    for sched in (lib.GEMM_COOPERATIVE, lib.GEMM_PINGPONG):
        obuf = sentinel_buffer(rows + 2, up8(N) + 8)
        out = obuf[:rows, :N]
        extra = {}
        if epi == "residual_moments":
            # x += proj(h) in place, with the 64-column moments of the stored rows
            out.copy_(rand16(M, N, seed=seed + 6))
            extra = {"residual": out, "row_moments": torch.full((M, N // 64, 2), float("nan"), device=a.device)}
            moms.append(extra["row_moments"])
        lib.gemm(a, w, out=out, wg_schedule=sched, **kw, **extra)
        outs.append(obuf)
    torch.cuda.synchronize()
    return outs[0], outs[1], rows, (moms if moms else None)


def _assert_same(coop, pp, rows, N, moms, what):
    assert torch.equal(coop.view(torch.int16), pp.view(torch.int16)), f"{what}: ping-pong differs from cooperative"
    assert_guards(pp, region(pp, rows, N), what)
    if moms is not None:
        assert torch.equal(moms[0], moms[1]), f"{what}: row moments differ"


@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("epi", EPILOGUES)
def test_pingpong_matches_cooperative_over_the_epilogues(lib, epi, M):
    # N: a tail of 64 columns past two full 128-wide tiles (row moments need N % 64 == 0) or of 13 (odd N, a
    # single-half store at the end of the row); K: one full k-block and a 24-column tail
    N = 320 if epi == "residual_moments" else 384 - 13 * (M % 2)
    K = 88
    coop, pp, rows, moms = _run_both(lib, M, N, K, epi, seed=M * 31 + EPILOGUES.index(epi))
    if epi == "remap":
        # rows between the groups of 4 (the cls rows) are not written: compare them as sentinels on both sides
        written = torch.zeros(pp.shape, dtype=torch.bool, device=pp.device)
        for m in range(M):
            written[(m // 4) * 5 + m % 4 + 1, :N] = True
        assert torch.equal(coop.view(torch.int16), pp.view(torch.int16)), f"remap M={M}: differs"
        assert_guards(pp, written, f"remap M={M}")
        return
    _assert_same(coop, pp, rows, N, moms, f"{epi} M={M} N={N}")


@pytest.mark.parametrize("epi", EPILOGUES)
def test_pingpong_matches_cooperative_with_both_warpgroups_busy(lib, epi):
    """every epilogue with several tiles per CTA, so that warpgroup 2 runs it too (its half of the column vectors,
    its named barrier, its double buffer across rounds) and the order barrier alternates the k-loops: 100 x 3 (or
    x 11) tiles, at least two per CTA on a 132-SM H100"""
    M = 12800 - 37
    N = 1408 if epi == "residual_moments" else 384 - 13
    coop, pp, rows, moms = _run_both(lib, M, N, 200, epi, seed=700 + EPILOGUES.index(epi))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert (M + 127) // 128 * ((N + 127) // 128) >= 2 * sms
    if epi == "remap":
        written = torch.zeros(pp.shape, dtype=torch.bool, device=pp.device)
        m = torch.arange(M, device=pp.device)
        written[(m // 4) * 5 + m % 4 + 1, :N] = True
        assert torch.equal(coop.view(torch.int16), pp.view(torch.int16)), f"remap M={M}: differs"
        assert_guards(pp, written, f"remap M={M}")
        return
    _assert_same(coop, pp, rows, N, moms, f"{epi} M={M} N={N}")


@pytest.mark.parametrize("N,K", [(128, 64), (256, 8), (1408, 1408), (200, 136), (129, 64)])
def test_pingpong_matches_cooperative_at_tile_and_k_tails(lib, N, K):
    M = 257
    coop, pp, rows, moms = _run_both(lib, M, N, K, "bias_gelu", seed=N + K)
    _assert_same(coop, pp, rows, N, moms, f"N={N} K={K}")


@pytest.mark.parametrize("per_cta", ["1", "2", "3", "2+1", "many"])
def test_pingpong_tiles_per_cta(lib, per_cta):
    """128-row tiles of one 128-wide column: tiles = sms hands out one per CTA, 2 sms two (both warpgroups busy),
    3 sms three (warpgroup 2 has one round fewer), sms + 5 gives some CTAs two and the rest one"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = {"1": sms, "2": 2 * sms, "3": 3 * sms, "2+1": sms + 5, "many": 0}[per_cta]
    if per_cta == "many":
        M, N, K = 8224, 1408, 1408          # 65 x 11 tiles: about 5.4 per CTA
    else:
        M, N, K = tiles * 128 - 37, 128, 64
    coop, pp, rows, moms = _run_both(lib, M, N, K, "residual_moments", seed=tiles + 7)
    _assert_same(coop, pp, rows, N, moms, f"per_cta={per_cta} M={M}")


@pytest.mark.parametrize("act", [0, 1])
def test_pingpong_against_float64_reference(lib, act):
    """bias, activation and residual: out = fp16(fp16(act(fp16(a w^T + bias))) + residual) within the derived bound"""
    M, N, K = 1028, 328, 200
    a, w = _operands(M, N, K, seed=90 + act)
    bias = rand16(N, scale=0.5, seed=92)
    res = rand16(M, N, seed=93)
    out = lib.gemm(a, w, bias=bias, act=act, residual=res, wg_schedule=lib.GEMM_PINGPONG)
    torch.cuda.synchronize()
    pre = R.linear_ref(a, w, bias, dtype=F64)
    post = R.linear_ref(a, w, bias, act, dtype=F64)
    ref = R.linear_ref(a, w, bias, act, res, dtype=F64)
    tol = gemm_tol(a, w, (ref, pre, post, res), 2 + (act != 0), 1.13 if act else 1.0, act_extra(act, pre), bias)
    check16(out, ref, tol, f"ping-pong act={act}")


def test_pingpong_refuses_other_tile_widths_and_mode_1(lib):
    a, w = rand16(256, 64), rand16(512, 64)
    with pytest.raises(RuntimeError, match="ping-pong"):
        lib.gemm(a, w, bn=256, wg_schedule=lib.GEMM_PINGPONG)
    with pytest.raises(RuntimeError, match="ping-pong"):
        lib.gemm(a, w, mode=1, wg_schedule=lib.GEMM_PINGPONG)
