"""Beam search on the device against sampling at the same row count and against the reference's strategy, on one GPU.

    python tools/beam_bench.py [--reps 2] [--json OUT] [--shapes 7b,13b] [--dtypes fp16,int8]

Random-init 7B / 13B weights made on the device (SEED vocabulary, 40194), fp16 and LLM.int8(); the config-#5 prompt
(4 image spans plus text, 256 tokens), 128 new tokens, eos disabled.  ms/token excludes the prefill:
(time(129 new tokens) - time(1 new token)) / 128.
  * beam k      seedb200_llama_beam_generate, num_beams = k (2, 4, 5): B * k rows per decode step
  * beam-sample k  the same with do_sample=True, temperature 0.7, top_p 0.5 (the Flask backend's defaults)
  * select k    the candidate kernel alone (seedb200_beam_select) on [k, V] logits with those sampling settings, us
  * sample k    seedb200_llama_generate at batch k with sampling (k <= 4): the same rows per step, no beam bookkeeping
  * hf-loop k   the reference's strategy: forward() per step from Python with past_key_values reordered by
                index_select (models/llama_xformer.py:779-782 _reorder_cache), k = 4, 32 steps timed; the drop-in
                forward() then copies the reordered past back into its cache, so this counts two cache copies per
                step where HF makes one, and no log_softmax / top-k on the host
The card name, power limit and the median SM clock during the timed runs are read in the same call.
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

from int8_bench import SHAPES, build, timed  # noqa: E402
from seed_b200 import synth  # noqa: E402

V_SEED = 40194


class Clock:
    """median SM clock (MHz) sampled by nvidia-smi while the block runs"""

    def __init__(self):
        self.samples, self._stop = [], threading.Event()

    def _run(self):
        while not self._stop.is_set():
            out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                                 capture_output=True, text=True).stdout.strip()
            if out.isdigit():
                self.samples.append(int(out))
            self._stop.wait(0.2)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    def median(self):
        return statistics.median(self.samples) if self.samples else None


def per_token(fn, new, reps):
    return (timed(lambda: fn(new + 1), reps) - timed(lambda: fn(1), reps)) / new


def select_only(lg, bs, k):
    from seed_b200 import lib
    lib.beam_select(lg, bs, 1, k, do_sample=True, temperature=0.7, top_p=0.5)


def hf_loop_ms(m, ids, k, steps=32):
    rows = ids.repeat_interleave(k, 0)
    out = m(input_ids=rows, use_cache=True, last_logits_only=True)
    past = out.past_key_values
    g = torch.Generator(device="cuda").manual_seed(0)
    tok = out.logits[:, -1].float().argmax(-1, keepdim=True)

    def step():
        nonlocal past, tok
        beam_idx = torch.randint(0, k, (k,), device="cuda", generator=g)
        past = tuple((a.index_select(0, beam_idx), b.index_select(0, beam_idx)) for a, b in past)
        o = m(input_ids=tok, past_key_values=past, use_cache=True, last_logits_only=True)
        past, tok = o.past_key_values, o.logits[:, -1].float().argmax(-1, keepdim=True)

    step()
    return timed(lambda: [step() for _ in range(steps)], 1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--json", default=None)
    ap.add_argument("--shapes", default="7b,13b")
    ap.add_argument("--dtypes", default="fp16,int8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("beam_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card, "rows": []}
    P, NEW = 256, 128
    ids = synth.prompt_ids(1, P, 4, seed=99).cuda()
    for shape_name in args.shapes.split(","):
        h, nl, nh, ffn, _ = SHAPES[shape_name]
        shape = (h, nl, nh, ffn, V_SEED)
        for dt in args.dtypes.split(","):
            m = build(shape, dt == "int8", P + NEW + 8, max_batch=5)
            L = m._llm
            row = {"model": shape_name, "dtype": dt}
            with Clock() as clk:
                for k in (2, 4, 5):
                    row[f"beam{k}_ms_per_token"] = per_token(
                        lambda n: L.beam_generate(ids, n, k, eos_token_id=-1), NEW, args.reps)
                    row[f"beam{k}_sample_ms_per_token"] = per_token(
                        lambda n: L.beam_generate(ids, n, k, do_sample=True, temperature=0.7, top_p=0.5,
                                                  eos_token_id=-1), NEW, args.reps)
                for k in (2, 4):
                    pk = ids.repeat_interleave(k, 0).contiguous()
                    row[f"sample{k}_ms_per_token"] = per_token(
                        lambda n: L.generate(pk, n, do_sample=True, top_p=0.9, eos_token_id=-1), NEW, args.reps)
                row["hf_loop4_ms_per_token"] = hf_loop_ms(m, ids, 4)
            row["sm_clock_median_MHz"] = clk.median()
            if dt == args.dtypes.split(",")[0]:
                for k in (2, 4, 5):
                    lg = (torch.randn((k, V_SEED), device="cuda") * 3).half()
                    bs = torch.zeros(k, device="cuda")
                    row[f"select{k}_sample_us"] = 1e3 * timed(
                        lambda: select_only(lg, bs, k), 50)
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
