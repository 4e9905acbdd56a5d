"""Per-shape timing of the wgmma GEMM at the encode shapes (B = 256 images: M = 65792 ViT rows, 8192 Q-Former rows)
and at the residual GEMMs of LLaMA-7B prefills.

For every GEMM shape with its model's epilogue (LayerNorm fold from row_stats, GELU / tanh, bias, in-place residual,
row moments, row remap) it times at the same M x N x K:
  coop      the cooperative kernel (both consumer warpgroups on one tile);
  pingpong  the ping-pong kernel (one 128 x 128 tile per consumer warpgroup);
  plain     seed_b200.lib.gemm with no bias, LayerNorm, activation or residual (cooperative tiles);
  cublas    torch.nn.functional.linear in fp16, the vendor library's rate on the same card.
"schedule" is the kernel seedb200_gemm picks for the shape.  On a power-capped card one window is noisy, so each
entry is timed in --repeats CUDA-event windows of >= --seconds, the four entries taking turns window by window; the
result gives the median, min and max TFLOP/s per entry and, per window pair, the ping-pong / cooperative ratio of the
adjacent coop and pingpong windows (median, min, max).  One JSON document, with the GPU name, its power limit and the
median SM clock sampled while the entries ran.

    python tools/gemm_shapes.py [--rows 65792] [--seconds 0.25] [--repeats 7] [--only qkv,fc1]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from seed_b200 import lib as L  # noqa: E402

D, FF = 1408, 6144
QD, QFF, QROWS = 768, 3072, 256 * 32
# name: (N, K, epilogue, rows or None for --rows)
SHAPES = {
    "patch_embed": (D, 592, "remap", 256 * 256),
    "qkv": (3 * D, D, "ln", None),
    "proj": (D, D, "residual", None),
    "fc1": (FF, D, "ln_gelu", None),
    "fc2": (D, FF, "residual", None),
    "cross_kv": (9216, D, "bias", None),
    "qformer_out": (QD, QD, "bias_residual", QROWS),
    "qformer_fc1": (QFF, QD, "bias_gelu", QROWS),
    "qformer_fc2": (QD, QFF, "bias_residual", QROWS),
    "qformer_tanh": (QD, QD, "bias_tanh", QROWS),
    "llama_o_proj": (4096, 4096, "residual_only", 2048),
    "llama_down_proj": (4096, 11008, "residual_only", 2048),
    "llama_o_proj_4k": (4096, 4096, "residual_only", 4096),
    "llama_down_proj_4k": (4096, 11008, "residual_only", 4096),
}


def time_launches(fn, seconds: float) -> float:
    """ms per call of fn: warm-up, a short probe to size the window, then one event-timed window of >= seconds."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        fn()
    e1.record()
    e1.synchronize()
    probe = e0.elapsed_time(e1) / 5
    n = max(10, int(seconds * 1000.0 / max(probe, 1e-3)) + 1)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


REMAP = (256, 257, 1, 256, 1)    # patch tokens behind each image's cls row, + pos_embed[1 + patch]


def planned(M: int, N: int, K: int, kind: str) -> tuple[int, str]:
    """(the cooperative kernel's tile width, the schedule gemm() picks) for the model's epilogue"""
    d = L.GemmDesc()
    d.M, d.N, d.K = M, N, K
    if kind in ("residual", "residual_only", "bias_residual", "remap"):
        d.residual = 1             # pointers are only tested against null by the planner
    if kind == "residual":
        d.row_moments = 1
    if kind.startswith("ln"):
        d.ln_stats = d.ln_c = d.ln_b = 1
    d.act = {"ln_gelu": L.ACT_GELU, "bias_gelu": L.ACT_GELU, "bias_tanh": L.ACT_TANH}.get(kind, L.ACT_NONE)
    if kind in ("bias", "residual", "bias_residual", "bias_gelu", "bias_tanh", "remap"):
        d.bias = 1
    if kind == "remap":
        d.row_group, d.row_stride, d.row_offset, d.res_mod, d.res_offset = REMAP
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sched = C.c_int32()
    L.check(L.load().seedb200_gemm_plan_schedule(C.byref(d), sms, C.byref(sched)), "seedb200_gemm_plan_schedule")
    d.wg_schedule = L.GEMM_COOPERATIVE
    out = (C.c_int32 * 9)()
    L.check(L.load().seedb200_gemm_plan(C.byref(d), sms, out), "seedb200_gemm_plan")
    return int(out[0]), "pingpong" if sched.value == L.GEMM_PINGPONG else "coop"


def make_case(name: str, M: int, dev):
    N, K, kind, _ = SHAPES[name]
    bn, schedule = planned(M, N, K, kind)
    g = torch.Generator(device=dev).manual_seed(1234)
    a = (torch.randn(M, K, generator=g, device=dev) * 0.5).half()
    w = (torch.randn(N, K, generator=g, device=dev) * K ** -0.5).half()
    bias = (torch.randn(N, generator=g, device=dev) * 0.1).half()
    out = torch.empty(M, N, dtype=torch.float16, device=dev)
    plain = lambda: L.gemm(a, w, out=out, bn=bn)  # noqa: E731   same tiles as the full epilogue
    if kind in ("ln", "ln_gelu"):
        stats = L.row_stats(a, 1e-6)
        c = (torch.randn(N, generator=g, device=dev) * 0.1)
        b = (torch.randn(N, generator=g, device=dev) * 0.1)
        act = L.ACT_GELU if kind == "ln_gelu" else L.ACT_NONE
        full = lambda s=0: L.gemm(a, w, act=act, out=out, ln=(stats, c, b), wg_schedule=s)  # noqa: E731
    elif kind == "residual":
        # x += proj(h) in place, with the moments the next LayerNorm takes its statistics from
        x = (torch.randn(M, N, generator=g, device=dev) * 0.5).half()
        mom = torch.empty(M, N // 64, 2, dtype=torch.float32, device=dev)
        full = lambda s=0: L.gemm(a, w, bias=bias, residual=x, out=x, row_moments=mom, wg_schedule=s)  # noqa: E731
    elif kind in ("residual_only", "bias_residual"):
        x = (torch.randn(M, N, generator=g, device=dev) * 0.5).half()
        bb = bias if kind == "bias_residual" else None
        full = lambda s=0: L.gemm(a, w, bias=bb, residual=x, out=x, wg_schedule=s)  # noqa: E731
    elif kind == "remap":
        pos = (torch.randn(257, N, generator=g, device=dev) * 0.5).half()
        xo = torch.empty(M // 256 * 257, N, dtype=torch.float16, device=dev)
        rg, rs, ro, rm, rf = REMAP
        full = lambda s=0: L.gemm(a, w, bias=bias, residual=pos, out=xo, row_group=rg, row_stride=rs,  # noqa: E731
                                  row_offset=ro, res_mod=rm, res_offset=rf, wg_schedule=s)
    else:
        act = {"bias_gelu": L.ACT_GELU, "bias_tanh": L.ACT_TANH}.get(kind, L.ACT_NONE)
        full = lambda s=0: L.gemm(a, w, bias=bias, act=act, out=out, wg_schedule=s)  # noqa: E731
    cublas = lambda: torch.nn.functional.linear(a, w)  # noqa: E731
    fns = {"coop": lambda: full(L.GEMM_COOPERATIVE), "pingpong": lambda: full(L.GEMM_PINGPONG),
           "plain": plain, "cublas": cublas}
    return N, K, kind, bn, schedule, fns


def spread(v: list, nd: int = 1) -> dict:
    v = sorted(v)
    return {"median": round(v[len(v) // 2], nd), "min": round(v[0], nd), "max": round(v[-1], nd)}


def gpu_info(index: int) -> dict:
    try:
        q = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, plim, smax = [s.strip() for s in q.strip().split(",")]
        return {"name": name, "power_limit_w": float(plim), "sm_max_mhz": float(smax)}
    except Exception:
        return {"name": torch.cuda.get_device_name(index), "power_limit_w": None, "sm_max_mhz": None}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=256 * 257, help="M (default: the 256-image encode, 257 tokens each)")
    ap.add_argument("--seconds", type=float, default=0.25, help="one timed window")
    ap.add_argument("--repeats", type=int, default=7, help="windows per entry, the entries taking turns")
    ap.add_argument("--only", default="", help="comma-separated subset of " + ",".join(SHAPES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_shapes.py: needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    names = [s for s in args.only.split(",") if s] or list(SHAPES)
    res = {"gpu": gpu_info(0), "rows": args.rows, "shapes": {}}
    with ClockSampler(0) as cs:
        for name in names:
            rows = SHAPES[name][3] or args.rows
            N, K, kind, bn, schedule, fns = make_case(name, rows, dev)
            flop = 2.0 * rows * N * K
            entry = {"M": rows, "N": N, "K": K, "bn": bn, "epilogue": kind, "schedule": schedule}
            tf = {k: [] for k in fns}
            for _ in range(args.repeats):
                for k, fn in fns.items():
                    tf[k].append(flop / time_launches(fn, args.seconds) / 1e9)
            for k, v in tf.items():
                entry[k] = spread(v)
            entry["pingpong_over_coop"] = spread([p / c for p, c in zip(tf["pingpong"], tf["coop"])], 3)
            res["shapes"][name] = entry
            del fns
            torch.cuda.empty_cache()
    res["clocks"] = cs.summary()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
