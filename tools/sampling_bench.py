"""Cost of the generation controls (top_k, repetition_penalty, no_repeat_ngram_size) in LLaMA decoding, on one GPU.

    python tools/sampling_bench.py [--reps 3] [--json OUT] [--shapes 7b,13b]

Random-init 7B / 13B fp16 weights made on the device (SEED vocabulary, 40194); the config-#5 prompt (4 image spans
plus text, 256 tokens), batch 1, 128 new tokens, eos disabled.  ms/token excludes the prefill:
(time(129 new tokens) - time(1 new token)) / 128, as tools/beam_bench.py.
  * sample   seedb200_llama_generate, do_sample with temperature 1.0 and top_p 0.5 (the reference's call site)
  * greedy   the same without sampling
  * beam4    seedb200_llama_beam_generate, num_beams = 4, beam search
each with the controls off and with top_k=50, repetition_penalty=1.1, no_repeat_ngram_size=3; the two variants
alternate within every repetition.  The card name and power limit are read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from int8_bench import SHAPES, build, timed  # noqa: E402
from seed_b200 import synth  # noqa: E402

V_SEED = 40194
ON = {"top_k": 50, "repetition_penalty": 1.1, "no_repeat_ngram_size": 3}
MODES = {"greedy": dict(num_beams=0, do_sample=False),
         "sample": dict(num_beams=0, do_sample=True, temperature=1.0, top_p=0.5),
         "beam4": dict(num_beams=4, do_sample=False)}


def per_token(fn, new, reps=1):
    return (timed(lambda: fn(new + 1), reps) - timed(lambda: fn(1), reps)) / new


def runner(L, ids, mode, ctl):
    kw = dict(MODES[mode])
    k = kw.pop("num_beams")
    if k:
        return lambda n: L.beam_generate(ids, n, k, eos_token_id=-1, **kw, **ctl)
    return lambda n: L.generate(ids, n, eos_token_id=-1, **kw, **ctl)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--shapes", default="7b,13b")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampling_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card, "rows": []}
    P, NEW = 256, 128
    ids = synth.prompt_ids(1, P, 4, seed=99).cuda()
    for shape_name in args.shapes.split(","):
        h, nl, nh, ffn, _ = SHAPES[shape_name]
        m = build((h, nl, nh, ffn, V_SEED), "fp16", P + NEW + 8, max_batch=4)
        L = m._llm
        for mode in MODES:
            t = {"off": [], "on": []}
            for _ in range(args.reps):
                for name, ctl in (("off", {}), ("on", ON)):
                    t[name].append(per_token(runner(L, ids, mode, ctl), NEW))
            off, on = statistics.median(t["off"]), statistics.median(t["on"])
            row = {"model": shape_name, "mode": mode, "off_ms_per_token": off, "on_ms_per_token": on,
                   "added_ms": on - off, "added_pct": 100.0 * (on - off) / off,
                   "off_all": t["off"], "on_all": t["on"]}
            print(json.dumps(row), flush=True)
            res["rows"].append(row)
        del m, L
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
