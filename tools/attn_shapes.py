"""Timing of seedb200_attention at the encode shapes: the ViT-g self attention (257 x 257 x 88, 16 heads, q / k / v
read from the packed [B * 257, 3 * 16 * 88] qkv buffer, the wgmma kernel) and, as a regression guard, the Q-Former
cross and causal self attention (32 queries, 12 heads x 64, the mma.sync kernel).

Each shape is timed in --repeats CUDA-event windows of >= --seconds, the shapes taking turns window by window.  Per
shape: median / min / max ms per call, the algorithmic TFLOP/s (4 B H nq nk d) and the achieved GB/s against the
algorithmic traffic (q, k, v read once, o written once: 741 MB per ViT layer at B = 256).  One JSON document, with the
GPU name, its power limit and the median SM clock sampled while the shapes ran.

    python tools/attn_shapes.py [--batch 256] [--seconds 0.25] [--repeats 7]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from bench import ClockSampler  # noqa: E402
from gemm_shapes import gpu_info, spread, time_launches  # noqa: E402
from seed_b200 import lib as L  # noqa: E402


def shapes(B: int) -> dict:
    """name -> (fn, flops, bytes)"""
    g = torch.Generator(device="cpu").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, generator=g).to(torch.float16).cuda()  # noqa: E731
    out = {}
    H, N, D = 16, 257, 88
    qkv = rnd(B * N, 3 * H * D).view(B, N, 3, H, D)
    q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    out["vit"] = (lambda: L.attention(q, k, v, D ** -0.5, False), 4.0 * B * H * N * N * D, 4 * B * H * N * D * 2)
    QH, QD, NQ = 12, 64, 32
    qq = rnd(B, QH, NQ, QD)
    ck, cv = rnd(B, QH, N, QD), rnd(B, QH, N, QD)
    out["qformer_cross"] = (lambda: L.attention(qq, ck, cv, QD ** -0.5, False), 4.0 * B * QH * NQ * N * QD,
                            (2 * B * QH * NQ + 2 * B * QH * N) * QD * 2)
    sk, sv = rnd(B, QH, NQ, QD), rnd(B, QH, NQ, QD)
    out["qformer_self_causal"] = (lambda: L.attention(qq, sk, sv, QD ** -0.5, True), 2.0 * B * QH * NQ * NQ * QD,
                                  4 * B * QH * NQ * QD * 2)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=0.25)
    ap.add_argument("--repeats", type=int, default=7)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_shapes: no CUDA device")
    L.load()
    sh = shapes(a.batch)
    ms = {n: [] for n in sh}
    with ClockSampler(torch.cuda.current_device()) as clk:
        for _ in range(a.repeats):
            for n, (fn, _, _) in sh.items():
                ms[n].append(time_launches(fn, a.seconds))
    res = {}
    for n, (_, flops, nbytes) in sh.items():
        med = spread(ms[n], 4)["median"]
        res[n] = {"ms": spread(ms[n], 4), "tflops": round(flops / med / 1e9, 1), "gb_s": round(nbytes / med / 1e6, 1),
                  "mb_per_call": round(nbytes / 1e6, 1)}
    print(json.dumps({"gpu": gpu_info(torch.cuda.current_device()), "clocks": clk.summary(), "batch": a.batch,
                      "shapes": res}, indent=1))


if __name__ == "__main__":
    main()
