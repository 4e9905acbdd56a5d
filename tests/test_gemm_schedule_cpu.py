"""The GEMM planner's consumer schedule (seedb200_gemm_plan_schedule, host-only) at the encode and LLaMA-7B shapes:
ping-pong for a residual epilogue over K <= 6144 (ViT proj / fc2, Q-Former output projections, LLaMA o_proj) and for
the LayerNorm fold (ViT qkv / fc1); cooperative for LLaMA down_proj (K = 11008), bias-only, activation-only,
row-remapped and plain GEMMs; and the tile width each schedule runs."""
import ctypes as C

import pytest

SMS = 132
ENC = 256 * 257          # rows of the 256-image encode
LN, RES, ACT = "ln", "residual", "act"


def _desc(L, M, N, K, *parts, bn=0, mode=0, wg_schedule=0):
    d = L.GemmDesc()
    d.M, d.N, d.K, d.mode, d.bn, d.wg_schedule = M, N, K, mode, bn, wg_schedule
    if LN in parts:
        d.ln_stats = d.ln_c = d.ln_b = 1       # pointers are only tested against NULL
    if RES in parts:
        d.residual = d.row_moments = 1
    if ACT in parts:
        d.act = L.ACT_GELU
    if "bias" in parts:
        d.bias = 1
    return d


def _schedule(L, d, sms=SMS):
    s = C.c_int32(-1)
    assert L.load().seedb200_gemm_plan_schedule(C.byref(d), sms, C.byref(s)) == 0, L.load().seedb200_last_error()
    out9 = (C.c_int32 * 9)()
    assert L.load().seedb200_gemm_plan(C.byref(d), sms, out9) == 0
    return s.value, out9[0]


@pytest.fixture(scope="module")
def L():
    from seed_b200 import lib
    return lib


@pytest.mark.parametrize("name,M,N,K,parts,pingpong,bn", [
    ("qkv", ENC, 4224, 1408, (LN,), True, 128),
    ("proj", ENC, 1408, 1408, ("bias", RES), True, 128),
    ("fc1", ENC, 6144, 1408, (LN, ACT), True, 128),
    ("fc2", ENC, 1408, 6144, ("bias", RES), True, 128),
    ("cross_kv", ENC, 9216, 1408, ("bias",), False, 256),
    ("plain", ENC, 6144, 1408, (), False, 256),
    ("qformer_out", 8192, 768, 768, ("bias", RES), True, 128),
    ("qformer_fc1", 8192, 3072, 768, ("bias", ACT), False, 256),
    ("qformer_fc2", 8192, 768, 3072, ("bias", RES), True, 128),
    ("llama_o_proj", 2048, 4096, 4096, (RES,), True, 128),
    ("llama_down_proj", 2048, 4096, 11008, (RES,), False, 256),
    ("llama_o_proj_4k", 4096, 4096, 4096, (RES,), True, 128),
    ("llama_down_proj_4k", 4096, 4096, 11008, (RES,), False, 256),
    ("llama_qkv", 2048, 12288, 4096, (), False, 256),
    ("short_prompt_o_proj", 256, 4096, 4096, (RES,), False, 256),
])
def test_planner_schedule_at_encode_and_llama_shapes(L, name, M, N, K, parts, pingpong, bn):
    sched, plan_bn = _schedule(L, _desc(L, M, N, K, *parts))
    assert (sched == L.GEMM_PINGPONG, plan_bn) == (pingpong, bn), name


def test_planner_needs_two_tiles_per_sm(L):
    """ping-pong alternates tiles: with fewer than two 128 x 128 tiles per SM the cooperative kernel runs"""
    M, N = 128 * 33, 128 * 8                 # 264 tiles = 2 x 132
    assert _schedule(L, _desc(L, M, N, 64, RES))[0] == L.GEMM_PINGPONG
    assert _schedule(L, _desc(L, M - 128, N, 64, RES))[0] == L.GEMM_COOPERATIVE
    assert _schedule(L, _desc(L, M - 128, N, 64, RES), sms=60)[0] == L.GEMM_PINGPONG


def test_planner_residual_k_limit_and_row_remap(L):
    assert _schedule(L, _desc(L, ENC, 1408, 6144, RES))[0] == L.GEMM_PINGPONG
    assert _schedule(L, _desc(L, ENC, 1408, 6152, RES))[0] == L.GEMM_COOPERATIVE
    d = _desc(L, 256 * 256, 1408, 592, "bias", RES)          # the patch embed: rows remapped behind the cls rows
    d.row_moments = None
    d.row_group, d.row_stride, d.row_offset, d.res_mod, d.res_offset = 256, 257, 1, 256, 1
    assert _schedule(L, d)[0] == L.GEMM_COOPERATIVE


def test_schedule_hint_forces_either_kernel(L):
    fc1 = _desc(L, ENC, 6144, 1408, LN, ACT, wg_schedule=L.GEMM_COOPERATIVE)
    assert _schedule(L, fc1) == (L.GEMM_COOPERATIVE, 256)
    plain = _desc(L, ENC, 6144, 1408, wg_schedule=L.GEMM_PINGPONG)
    assert _schedule(L, plain) == (L.GEMM_PINGPONG, 128)
    # an explicit tile width keeps the cooperative kernel unless ping-pong is forced
    assert _schedule(L, _desc(L, ENC, 6144, 1408, LN, ACT, bn=256))[0] == L.GEMM_COOPERATIVE


@pytest.mark.parametrize("fields", [dict(wg_schedule=3), dict(wg_schedule=-1),
                                    dict(wg_schedule=2, bn=256), dict(wg_schedule=2, mode=1)])
def test_schedule_hint_out_of_range_is_refused(L, fields):
    d = _desc(L, 512, 512, 64, **fields)
    s = C.c_int32(-1)
    assert L.load().seedb200_gemm_plan_schedule(C.byref(d), SMS, C.byref(s)) != 0
