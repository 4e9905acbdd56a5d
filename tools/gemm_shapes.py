"""Per-shape timing of the wgmma GEMM at the ViT-g encode shapes (B = 256 images, M = 65792 rows).

For every GEMM of a ViT block and for the Q-Former cross-attention K|V projection it times three things at the same
M x N x K:
  full    seed_b200.lib.gemm with the epilogue the encode runs (LayerNorm fold from row_stats, GELU, bias + in-place
          residual + row moments);
  plain   seed_b200.lib.gemm with no bias, LayerNorm, activation or residual;
  cublas  torch.nn.functional.linear in fp16, the vendor library's rate on the same card.
"full - plain" is what the epilogue costs, "plain vs cublas" what the mainloop leaves.  Each entry is timed with CUDA
events over enough back-to-back launches to fill --seconds after a warm-up, and the result is one JSON document with
TFLOP/s per entry, the GPU name, its power limit and the median SM clock sampled while the entries ran.

    python tools/gemm_shapes.py [--rows 65792] [--seconds 1.0] [--only qkv,fc1]
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
# name: (N, K, epilogue of the encode)
SHAPES = {
    "qkv": (3 * D, D, "ln"),
    "proj": (D, D, "residual"),
    "fc1": (FF, D, "ln_gelu"),
    "fc2": (D, FF, "residual"),
    "cross_kv": (9216, D, "bias"),
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


def planned_bn(M: int, N: int, K: int, kind: str) -> int:
    """The tile width gemm() picks for the encode's epilogue (row moments need 64-column multiples)."""
    d = L.GemmDesc()
    d.M, d.N, d.K = M, N, K
    if kind == "residual":
        d.row_moments = 1          # only tested against null by the planner
    out = (C.c_int32 * 9)()
    L.check(L.load().seedb200_gemm_plan(C.byref(d), torch.cuda.get_device_properties(0).multi_processor_count, out),
            "seedb200_gemm_plan")
    return int(out[0])


def make_case(name: str, M: int, dev):
    N, K, kind = SHAPES[name]
    bn = planned_bn(M, N, K, kind)
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
        full = lambda: L.gemm(a, w, act=act, out=out, ln=(stats, c, b))  # noqa: E731
    elif kind == "residual":
        # x += proj(h) in place, with the moments the next LayerNorm takes its statistics from
        x = (torch.randn(M, N, generator=g, device=dev) * 0.5).half()
        mom = torch.empty(M, N // 64, 2, dtype=torch.float32, device=dev)
        full = lambda: L.gemm(a, w, bias=bias, residual=x, out=x, row_moments=mom)  # noqa: E731
    else:
        full = lambda: L.gemm(a, w, bias=bias, out=out)  # noqa: E731
    cublas = lambda: torch.nn.functional.linear(a, w)  # noqa: E731
    return N, K, kind, bn, {"full": full, "plain": plain, "cublas": cublas}


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
    ap.add_argument("--seconds", type=float, default=1.0, help="timed window per entry")
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
            N, K, kind, bn, fns = make_case(name, args.rows, dev)
            flop = 2.0 * args.rows * N * K
            entry = {"N": N, "K": K, "bn": bn, "epilogue": kind}
            for k, fn in fns.items():
                ms = time_launches(fn, args.seconds)
                entry[k] = {"ms": round(ms, 4), "tflops": round(flop / ms / 1e9, 1)}
            entry["epilogue_ms"] = round(entry["full"]["ms"] - entry["plain"]["ms"], 4)
            res["shapes"][name] = entry
            del fns
            torch.cuda.empty_cache()
    res["clocks"] = cs.summary()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
