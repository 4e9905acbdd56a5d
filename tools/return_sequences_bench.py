"""Sampling with num_return_sequences = n on the device against the expanded call, on one GPU.

    python tools/return_sequences_bench.py [--reps 3] [--json OUT] [--shapes 7b,13b] [--prompts 256,1792] [--n 1,2,4,8]

Random-init 7B / 13B fp16 weights made on the device (SEED vocabulary, 40194), one prompt, the Flask defaults
(temperature 0.7, top_p 0.5), 128 new tokens, eos disabled.  For each n two variants run, alternating in one process:
  * shared     seedb200_llama_generate_n(prompt, n): the prompt prefilled once, n rows through the lineage table
  * expanded   seedb200_llama_generate on prompt.repeat_interleave(n, 0) (what generate(device_loop=True) runs on a
               hand-expanded batch): n prefills, n copies of the prompt's K/V, plain decode attention
Reported per variant, each the median of --reps runs:
  * first_ms   prefill + first token: one call with max_new_tokens = 1
  * step_ms    per decode step: (time(129 new tokens) - time(1 new token)) / 128
The card name, its power limit and the median SM clock sampled during the timed runs are read in the same call.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from int8_bench import SHAPES, build  # noqa: E402
from seed_b200 import synth  # noqa: E402

V_SEED, NEW = 40194, 128
SAMP = dict(do_sample=True, temperature=0.7, top_p=0.5, eos_token_id=-1)


def smi(query):
    return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader,nounits", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()


class ClockSampler:
    """SM clock (MHz) read every 0.25 s while `timing` is set: only during the timed runs, so that model builds and
    warm-ups do not mix idle clocks into the median"""

    def __init__(self):
        self.samples, self._stop, self.timing = [], threading.Event(), threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.wait(0.25):
            if not self.timing.is_set():
                continue
            try:
                self.samples.append(int(smi("clocks.sm")))
            except ValueError:
                pass

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()


def ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def measure(L, ids, n, reps, clocks):
    """{variant: (first_ms, step_ms)}, medians of reps, the variants alternating; clocks samples the timed runs"""
    runs = {"shared": lambda m: L.generate(ids, m, num_return_sequences=n, **SAMP),
            "expanded": lambda m: L.generate(ids.repeat_interleave(n, 0), m, **SAMP)}
    for run in runs.values():                        # warm-up: modules, graph capture of both units
        run(NEW + 1)
    first = {k: [] for k in runs}
    step = {k: [] for k in runs}
    clocks.timing.set()
    for _ in range(reps):
        for name, run in runs.items():
            t1 = ms(lambda: run(1))
            tn = ms(lambda: run(NEW + 1))
            first[name].append(t1)
            step[name].append((tn - t1) / NEW)
    clocks.timing.clear()
    return {k: (statistics.median(first[k]), statistics.median(step[k])) for k in runs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--shapes", default="7b,13b")
    ap.add_argument("--prompts", default="256,1792")
    ap.add_argument("--n", default="1,2,4,8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("return_sequences_bench needs a CUDA device")
    prompts = [int(p) for p in args.prompts.split(",")]
    ns = [int(n) for n in args.n.split(",")]
    res = {"card": smi("name"), "power_limit_W": smi("power.limit"), "rows": []}
    print(json.dumps(res), flush=True)
    with ClockSampler() as clocks:
        for shape_name in args.shapes.split(","):
            h, nl, nh, ffn, _ = SHAPES[shape_name]
            torch.cuda.empty_cache()
            model = build((h, nl, nh, ffn, V_SEED), "fp16", max(prompts) + NEW + 8, max_batch=max(ns))
            for P in prompts:
                ids = synth.prompt_ids(1, P, 4, seed=99).cuda()
                for n in ns:
                    r = measure(model._llm, ids, n, args.reps, clocks)
                    row = {"model": shape_name, "prompt": P, "n": n,
                           "shared_first_ms": r["shared"][0], "expanded_first_ms": r["expanded"][0],
                           "shared_step_ms": r["shared"][1], "expanded_step_ms": r["expanded"][1]}
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
