"""Generation scores on and off (generate(output_scores=True, return_dict_in_generate=True)), on one GPU.

    python tools/scores_bench.py [--reps 3] [--json OUT] [--shapes 7b,13b]
                                 [--modes greedy,sample,contrastive,beam,beam_sample]

Random-init 7B / 13B fp16 weights made on the device (SEED vocabulary, 40194), one prompt of 256 tokens (the
llama_decode workload's prompt length), 128 new tokens, eos disabled.  Modes: greedy, sampling with the Flask
defaults (temperature 0.7, top_p 0.5), contrastive search (top_k 4, penalty_alpha 0.6), beam search (4 beams) and beam
sampling (4 beams, temperature 0.7, top_p 0.5).  For each mode the device loop runs with a scores buffer (and, for
beams, beam_indices) through the `_ex` entry points, and without them, alternating in one process.  Reported, each the median of --reps runs:
  * step_ms    per decode step: (time(129 new tokens) - time(1 new token)) / 128
The scores buffer (max_new_tokens x rows x V fp16) is allocated once per mode, outside the timed window, as the
caching allocator serves it after the first call.  The card name, its power limit and the median SM clock sampled
during the timed runs are read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from int8_bench import SHAPES, build  # noqa: E402
from return_sequences_bench import ClockSampler, ms, smi  # noqa: E402
from seed_b200 import lib as Lib  # noqa: E402
from seed_b200 import synth  # noqa: E402

V_SEED, NEW, PROMPT = 40194, 128, 256
MODES = {"greedy": dict(do_sample=False, eos_token_id=-1),
         "sample": dict(do_sample=True, temperature=0.7, top_p=0.5, eos_token_id=-1),
         "contrastive": dict(top_k=4, penalty_alpha=0.6, eos_token_id=-1),
         "beam": dict(num_beams=4, eos_token_id=-1),
         "beam_sample": dict(num_beams=4, do_sample=True, temperature=0.7, top_p=0.5, eos_token_id=-1)}
ROWS = 4   # contrastive candidates and beams per prompt


def measure(L, ids, mode, reps, clocks):
    """{"off"/"on": step_ms}, medians of reps, the variants alternating; clocks samples the timed runs"""
    kw = MODES[mode]
    beams = mode.startswith("beam")
    buf = Lib.scores_buffer(NEW + 1, ROWS if beams else 1, V_SEED, ids.device)
    if beams:
        bi = {m: torch.empty((1, ids.shape[1] + m), dtype=torch.int64, device=ids.device) for m in (1, NEW + 1)}
        kw = dict(kw)
        nb = kw.pop("num_beams")
        runs = {"off": lambda m: L.beam_generate(ids, m, nb, **kw),
                "on": lambda m: L.beam_generate(ids, m, nb, scores=buf[:m], beam_indices=bi[m], **kw)}
    else:
        gen = L.contrastive_generate if mode == "contrastive" else L.generate
        runs = {"off": lambda m: gen(ids, m, **kw),
                "on": lambda m: gen(ids, m, scores=buf[:m], **kw)}
    for run in runs.values():                        # warm-up: modules, graph capture
        run(NEW + 1)
    step = {k: [] for k in runs}
    clocks.timing.set()
    for _ in range(reps):
        for name, run in runs.items():
            t1 = ms(lambda: run(1))
            tn = ms(lambda: run(NEW + 1))
            step[name].append((tn - t1) / NEW)
    clocks.timing.clear()
    return {k: statistics.median(v) for k, v in step.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--shapes", default="7b,13b")
    ap.add_argument("--modes", default=",".join(MODES))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scores_bench needs a CUDA device")
    res = {"card": smi("name"), "power_limit_W": smi("power.limit"), "rows": []}
    print(json.dumps(res), flush=True)
    with ClockSampler() as clocks:
        for shape_name in args.shapes.split(","):
            h, nl, nh, ffn, _ = SHAPES[shape_name]
            torch.cuda.empty_cache()
            model = build((h, nl, nh, ffn, V_SEED), "fp16", PROMPT + NEW + 8, max_batch=ROWS)
            ids = synth.prompt_ids(1, PROMPT, 4, seed=99).cuda()
            for mode in args.modes.split(","):
                r = measure(model._llm, ids, mode, args.reps, clocks)
                row = {"model": shape_name, "mode": mode, "off_step_ms": r["off"], "on_step_ms": r["on"],
                       "extra_step_ms": r["on"] - r["off"]}
                print(json.dumps(row), flush=True)
                res["rows"].append(row)
            del model
    res["median_sm_clock_MHz"] = statistics.median(clocks.samples) if clocks.samples else None
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
