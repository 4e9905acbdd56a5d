"""CPU-only checks (-m "not gpu"): the C-ABI library builds/loads, exports every symbol include/seedb200.h
declares, reports errors without a GPU, and the product path refuses to run without CUDA (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def L():
    from seed_b200 import build, lib

    if not os.path.exists(lib.LIB_PATH):
        build.build_cuda()
    lib.load()
    return lib


def test_header_symbols_are_all_exported(L):
    hdr = open(os.path.join(REPO, "include", "seedb200.h")).read()
    declared = set(re.findall(r"\b(seedb200_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"seedb200_status", "seedb200_dtype"}
    assert declared == set(L.EXPORTS), declared ^ set(L.EXPORTS)
    handle = L.load()
    for sym in sorted(declared):
        assert hasattr(handle, sym), f"libseedb200.so does not export {sym}"
    assert handle.seedb200_version() == 200


def test_errors_are_reported_not_thrown(L):
    handle = L.load()
    assert handle.seedb200_gemm(None, None) != 0
    assert b"null descriptor" in handle.seedb200_last_error()
    d = L.GemmDesc()
    d.M, d.N, d.K = 16, 16, 12     # K not a multiple of 8
    d.A = d.W = d.out = 16
    assert handle.seedb200_gemm(C.byref(d), None) == 1
    assert b"multiple of 8" in handle.seedb200_last_error()
    # inconsistent GEMM descriptors are refused by the planner, before any device work
    out9 = (C.c_int32 * 9)()

    def plan_error(**fields):
        g = L.GemmDesc()
        g.M, g.N, g.K, g.lda, g.ldw, g.ldo = 64, 512, 64, 64, 64, 512
        for k, v in fields.items():
            setattr(g, k, v)
        if handle.seedb200_gemm_plan(C.byref(g), 132, out9) == 0:
            return None
        return handle.seedb200_last_error()

    assert plan_error() is None and plan_error(mode=1, ldo=256) is None
    assert plan_error(lda=0, ldw=0, ldo=0) is None                             # 0 = packed rows
    assert plan_error(mode=1, ldo=0) is None
    assert b"residual" in plan_error(mode=1, ldo=256, residual=16, ldr=256)      # SiLU-gate has no residual (as the GEMV)
    assert b"lda=56" in plan_error(lda=56)
    assert b"ldw=8" in plan_error(ldw=8)
    assert b"ldo=504" in plan_error(ldo=504)
    assert b"ldo=248" in plan_error(mode=1, ldo=248)                           # mode 1 writes N / 2 columns
    assert plan_error(residual=16) is None                                     # ldr = 0: packed, N
    assert b"ldo=-8" in plan_error(ldo=-8)
    assert b"ldr=511" in plan_error(residual=16, ldr=511)
    assert plan_error(residual=16, ldr=520, ldo=520, lda=72, ldw=128) is None
    a = L.AttnDesc()
    a.q = a.k = a.v = a.o = 16
    a.batch = a.heads = a.nq = a.nk = 1
    a.head_dim = 80
    assert handle.seedb200_attention(C.byref(a), None) == 1
    assert b"head_dim" in handle.seedb200_last_error()
    assert handle.seedb200_vq_argmin(16, 16, 4, 8192, 48, 0, 16, None) == 1
    assert b"dim=48" in handle.seedb200_last_error()
    cfg = L.EncoderConfig(1, 1, 0, 8192, 0, 0, 0)
    h = C.c_void_p()
    arr = (L.Tensor * 1)()
    arr[0].name = b"x"
    assert handle.seedb200_encoder_create(C.byref(cfg), arr, 1, C.byref(h)) == 1
    assert b"max_batch" in handle.seedb200_last_error()


def test_product_path_refuses_cpu():
    from seed_b200 import lib
    from seed_b200.qformer_quantizer import Blip2QformerQuantizer

    with pytest.raises(RuntimeError, match="CUDA"):
        lib.gemm(torch.zeros(8, 8, dtype=torch.float16), torch.zeros(8, 8, dtype=torch.float16))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU path"):
            Blip2QformerQuantizer({}, device="cuda")
    with pytest.raises(RuntimeError, match="no CPU path"):
        Blip2QformerQuantizer({}, device="cpu")
    with pytest.raises(ValueError, match="fp16"):
        Blip2QformerQuantizer({}, device="cuda", vit_precision="fp32")


def test_missing_library_fails_loudly(tmp_path):
    code = ("import seed_b200.lib as L, sys\n"
            f"L.LIB_PATH = r'{tmp_path}/nope.so'\n"
            "try:\n    L.load()\nexcept RuntimeError as e:\n    print('RAISED', 'no CPU or PyTorch fallback' in str(e))\n")
    out = subprocess.run([sys.executable, "-c", code], cwd=REPO, capture_output=True, text=True)
    assert "RAISED True" in out.stdout, out.stdout + out.stderr


def test_no_oracle_imports_in_product_code():
    """only tests/, __graft_entry__.smoke() and bench.py may touch oracle/ (tier rule 3)."""
    bad = []
    for root in ("seed_b200", "models", "tools", "include"):
        for dp, _, files in os.walk(os.path.join(REPO, root)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h")):
                    txt = open(os.path.join(dp, f)).read()
                    if (re.search(r"^\s*(from|import)\s+oracle\b", txt, re.M) or re.search(r"#include\s+[\"<].*oracle", txt)
                            or re.search(r"(CDLL|dlopen)\(.*oracle", txt)):
                        bad.append(os.path.join(dp, f))
    assert not bad, bad


def test_image_ids_to_tokens_and_transform_contract():
    from models.seed_llama_tokenizer import SeedImageTokenMixin
    from models.transforms import get_transform

    ids = torch.arange(64).reshape(2, 32)
    toks = SeedImageTokenMixin.image_ids_to_tokens(ids)
    assert toks.tolist()[0][:3] == [40192, 32000, 32001] and toks[1, 33] == 40193
    t = get_transform("clip", keep_ratio=False, image_size=224)
    from PIL import Image

    x = t(Image.new("RGB", (300, 200), (128, 64, 32)))
    assert tuple(x.shape) == (3, 224, 224)
    with pytest.raises(NotImplementedError):
        get_transform("other")


def _plan(L, M, N, K, ctas=2, mode=0, bn=0, sms=132):
    d = L.GemmDesc()
    d.M, d.N, d.K, d.ctas, d.mode, d.bn = M, N, K, ctas, mode, bn
    out = (C.c_int32 * 9)()
    assert L.load().seedb200_gemm_plan(C.byref(d), sms, out) == 0, L.load().seedb200_last_error()
    keys = ("bn", "ctas", "sched", "ksub", "m_tiles", "n_tiles", "units", "tile_shift", "tail_w")
    return dict(zip(keys, list(out)))


def _unit_loads(L, p, sched=None):
    """Walk the persistent schedule of every unit; returns (tiles seen, columns per unit)."""
    h = L.load()
    sched = p["sched"] if sched is None else sched
    total = p["m_tiles"] * p["n_tiles"]
    w_last = p["tail_w"] if p["tail_w"] > 0 else p["bn"]
    seen, loads = [], []
    for u in range(p["units"]):
        cols = 0
        for rnd in range(total + 2):
            t = h.seedb200_gemm_schedule_tile(sched, rnd, u, p["units"], p["m_tiles"], p["n_tiles"], p["tile_shift"])
            if t >= total:
                # a finished unit stays finished
                assert h.seedb200_gemm_schedule_tile(sched, rnd + 1, u, p["units"], p["m_tiles"], p["n_tiles"],
                                                     p["tile_shift"]) >= total
                break
            seen.append(t)
            cols += w_last if t % p["n_tiles"] == p["n_tiles"] - 1 else p["bn"]
        loads.append(cols)
    return seen, loads


@pytest.mark.parametrize("shape", [(2048, 4096, 4096), (2048, 12288, 4096), (2048, 4096, 11008), (2048, 40200, 4096),
                                   (256, 5120, 5120), (256, 15360, 5120), (256, 5120, 13824), (65792, 1408, 1408),
                                   (65792, 4224, 1408), (8192, 3072, 768), (300, 1040, 64), (129, 2050, 64)])
def test_gemm_tile_schedules_hand_out_every_tile_exactly_once(L, shape):
    M, N, K = shape
    for sms in (148, 132, 7):
        p = _plan(L, M, N, K, sms=sms)
        total = p["m_tiles"] * p["n_tiles"]
        for sched in ((0, 1) if p["n_tiles"] >= 2 else (0,)):
            q = dict(p)
            if sched != p["sched"]:
                q["tile_shift"] = 0
            seen, _ = _unit_loads(L, q, sched)
            assert sorted(seen) == list(range(total)), (shape, sms, sched, p)


def test_gemm_plan_for_single_tile_rows_and_tuned_shapes(L):
    """A 256-token prompt (two rows of 128-row tiles): N = 5120 runs on 128-wide tiles (80 busy SMs instead of 40),
    N = 15360 keeps 256; the M = 2048 prefill shapes and the ViT shapes take the widest tile that divides N (no
    half-empty last column), all on single CTAs (ctas = 2 is accepted and runs the same tiles)."""
    assert _plan(L, 256, 5120, 5120)["bn"] == 128
    assert _plan(L, 256, 5120, 13824)["bn"] == 128
    assert _plan(L, 256, 15360, 5120)["bn"] == 256
    for M, N, K, bn in ((2048, 4096, 4096, 256), (2048, 12288, 4096, 256), (2048, 4096, 11008, 256),
                        (65792, 1408, 1408, 176), (65792, 4224, 1408, 192), (65792, 6144, 1408, 256),
                        (65792, 1408, 6144, 176)):
        p = _plan(L, M, N, K)
        assert (p["bn"], p["ctas"], p["sched"]) == (bn, 1, 0), p
