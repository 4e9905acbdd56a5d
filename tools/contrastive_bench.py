"""Contrastive search on the device against greedy decoding, on one GPU.

    python tools/contrastive_bench.py [--reps 2] [--json OUT] [--shapes 7b,13b] [--sweep 256,1024,1792] [--profile]

Random-init 7B / 13B fp16 weights made on the device (SEED vocabulary, 40194), B = 1, 128 new tokens, eos disabled.
ms/token excludes the prefill: (time(129 new tokens) - time(1 new token)) / 128, greedy and contrastive alternating in
one process.
  * greedy          seedb200_llama_generate (one row per decode step)
  * contrastive     seedb200_llama_contrastive_generate, k = 4, alpha = 0.6 (four candidate rows per step)
  * ratio           contrastive / greedy
The default run covers 7B and 13B at a 256-token prompt, then the 13B context sweep (prompts of --sweep tokens) that
shows how the rank kernel's cost grows with the context.  --profile instead traces 32 contrastive steps at 13B with the
longest sweep prompt and reports the rank kernel's device time per launch and its context bytes (p * hidden * 2 per
launch, read once) over that time against the H100 SXM's 3.35 TB/s.  The card name and power limit are read in the
same call.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from int8_bench import SHAPES, build, timed  # noqa: E402
from seed_b200 import synth  # noqa: E402

V_SEED, NEW, K, ALPHA = 40194, 128, 4, 0.6
HBM_BYTES_PER_S = 3.35e12


def pair(L, ids, reps):
    """(greedy, contrastive) ms per generated token, alternating"""
    greedy = lambda n: L.generate(ids, n, eos_token_id=-1)                               # noqa: E731
    contr = lambda n: L.contrastive_generate(ids, n, K, ALPHA, eos_token_id=-1)          # noqa: E731
    g, c = [], []
    for _ in range(reps):
        g.append((timed(lambda: greedy(NEW + 1)) - timed(lambda: greedy(1))) / NEW)
        c.append((timed(lambda: contr(NEW + 1)) - timed(lambda: contr(1))) / NEW)
    return min(g), min(c)


def profile_rank(L, ids, steps=32):
    from torch.profiler import ProfilerActivity, profile

    L.contrastive_generate(ids, steps, K, ALPHA, eos_token_id=-1)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        L.contrastive_generate(ids, steps, K, ALPHA, eos_token_id=-1)
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "contrastive_rank_kernel" in e.name]   # us
    P = ids.shape[1]
    ctx_bytes = sum((P + t) * L.hidden * 2 for t in range(steps)) / steps
    us = sum(times) / max(len(times), 1)
    return {"launches": len(times), "rank_us_per_launch": us, "context_MB_per_launch": ctx_bytes / 1e6,
            "context_TB_per_s": ctx_bytes / (us * 1e-6) / 1e12 if us > 0 else None,
            "share_of_3.35TB_per_s": ctx_bytes / (us * 1e-6) / HBM_BYTES_PER_S if us > 0 else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--json", default=None)
    ap.add_argument("--shapes", default="7b,13b")
    ap.add_argument("--sweep", default="256,1024,1792")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contrastive_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card, "rows": []}
    sweep = [int(p) for p in args.sweep.split(",")]
    runs = [] if args.profile else [(s, 256) for s in args.shapes.split(",") if s != "13b" or 256 not in sweep]
    runs += [("13b", p) for p in (sweep[-1:] if args.profile else sweep)]
    built = {}
    for shape_name, P in runs:
        h, nl, nh, ffn, _ = SHAPES[shape_name]
        if shape_name not in built:
            built.clear()
            torch.cuda.empty_cache()
            built[shape_name] = build((h, nl, nh, ffn, V_SEED), "fp16", max(sweep) + NEW + 8, max_batch=K)
        L = built[shape_name]._llm
        ids = synth.prompt_ids(1, P, 4, seed=99).cuda()
        row = {"model": shape_name, "prompt": P}
        if args.profile:
            row.update(profile_rank(L, ids))
        else:
            g, c = pair(L, ids, args.reps)
            row.update({"greedy_ms_per_token": g, "contrastive_ms_per_token": c, "ratio": c / g})
        print(json.dumps(row), flush=True)
        res["rows"].append(row)
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
