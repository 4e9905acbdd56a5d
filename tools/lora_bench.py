"""Base vs unmerged LoRA (r = 16, all seven decoder linears) LLaMA on one GPU, random-init weights made on the device.

    python tools/lora_bench.py [--reps 2] [--shapes 7b,13b] [--json OUT]

For each shape, a base model and a LoRA model (same base weights plus an adapter) are built in one process and timed
alternately (base, lora, base, lora, ...); then the LoRA model is merged (merge_and_unload) and timed against the base
again.  Figures, all from CUDA events:
  * prefill tokens/s: B = 1, S = 2048, logits of the last position only;
  * decode ms/token: prompt P = 256, 128 new tokens through seedb200_llama_generate (greedy, graph-replayed steps),
    (time(129 new tokens) - time(1 new token)) / 128;
  * beam ms/token: the same with num_beams = 4 and 5 (seedb200_llama_beam_generate), 7B only: two 13B models with
    5 cache rows of 2048 positions do not fit one 80 GB card next to each other.
The card name, power limit and the median SM clock sampled between timed blocks are read in the same run.

    python tools/lora_bench.py --profile OUT.json [--shapes 7b]

instead runs one prefill (S = 2048) and one 32-token decode of the base and the LoRA model under torch.profiler (CUDA
activity only, in a run of its own, decode launches without programmatic dependent launch so that kernel spans do not
overlap) and reports the device time per kernel name, summed, for each: where the LoRA model's extra time goes.
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

from transformers.models.llama.configuration_llama import LlamaConfig  # noqa: E402

from seed_b200.llama import LlamaForCausalLM  # noqa: E402

SHAPES = {"7b": (4096, 32, 32, 11008, 32000), "13b": (5120, 40, 40, 13824, 32000)}
LINS = (("self_attn.q_proj", 0, 0), ("self_attn.k_proj", 0, 0), ("self_attn.v_proj", 0, 0), ("self_attn.o_proj", 0, 0),
        ("mlp.gate_proj", 1, 0), ("mlp.up_proj", 1, 0), ("mlp.down_proj", 0, 1))
P, NEW, S = 256, 128, 2048
CLOCKS = []


def state_dict(h, nl, ffn, V, g):
    def rnd(*shape, scale=0.02):
        return torch.randn(*shape, device="cuda", dtype=torch.float16, generator=g) * scale

    sd = {"model.embed_tokens.weight": rnd(V, h), "model.norm.weight": torch.ones(h, device="cuda", dtype=torch.float16),
          "lm_head.weight": rnd(V, h)}
    for l in range(nl):
        p = f"model.layers.{l}."
        sd[p + "input_layernorm.weight"] = torch.ones(h, device="cuda", dtype=torch.float16)
        sd[p + "post_attention_layernorm.weight"] = torch.ones(h, device="cuda", dtype=torch.float16)
        for nm, n_ffn, k_ffn in LINS:
            sd[p + nm + ".weight"] = rnd(ffn if n_ffn else h, ffn if k_ffn else h)
    return sd


def adapter(h, nl, ffn, r, g):
    ad = {}
    for l in range(nl):
        for nm, n_ffn, k_ffn in LINS:
            p = f"model.layers.{l}.{nm}."
            ad[p + "lora_A.weight"] = torch.randn(r, ffn if k_ffn else h, device="cuda", dtype=torch.float16,
                                                  generator=g) * 0.01
            ad[p + "lora_B.weight"] = torch.randn(ffn if n_ffn else h, r, device="cuda", dtype=torch.float16,
                                                  generator=g) * 0.01
    return ad


def sample_clock():
    out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    if out.isdigit():
        CLOCKS.append(int(out))


def timed(fn, reps=1):
    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    sample_clock()
    return s.elapsed_time(e) / reps


def measure(m, prompt, ids, beams):
    llm = m._llm
    out = {"prefill_tokens_per_s": S / (timed(lambda: llm.forward(input_ids=ids, last_only=True), 2) * 1e-3)}
    gen = lambda n: llm.generate(prompt, n, use_graph=True, eos_token_id=-1)   # noqa: E731
    out["decode_ms_per_token"] = (timed(lambda: gen(NEW + 1), 2) - timed(lambda: gen(1), 2)) / NEW
    for k in beams:
        bg = lambda n: llm.beam_generate(prompt, n, k, eos_token_id=-1)   # noqa: E731
        out[f"beam{k}_ms_per_token"] = (timed(lambda: bg(NEW + 1)) - timed(lambda: bg(1))) / NEW
    return out


def kernel_times(fn):
    """device milliseconds per kernel name over one call of fn (torch.profiler, CUDA activity)"""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and getattr(e, "self_device_time_total", 0) > 0:
            name = e.key.split("<")[0].split("(")[0]
            out[name] = out.get(name, 0.0) + e.self_device_time_total / 1e3
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def profile_run(args, card):
    from seed_b200 import lib as L

    # with programmatic dependent launches a kernel's recorded span includes its wait for the predecessor, so spans
    # overlap and per-kernel sums mislead: the profile runs the decode chain with plain launches
    L.set_option("decode_pdl", 0)
    res = {"card": card, "r": args.r, "decode_pdl": 0}
    for name in args.shapes.split(","):
        h, nl, nh, ffn, V = SHAPES[name]
        cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=ffn, num_hidden_layers=nl,
                          num_attention_heads=nh, num_key_value_heads=nh, rms_norm_eps=1e-6,
                          max_position_embeddings=S)
        g = torch.Generator(device="cuda").manual_seed(0)
        m = LlamaForCausalLM(cfg, state_dict(h, nl, ffn, V, g), device="cuda", max_batch=1, max_seq=S)
        prompt = torch.randint(0, V, (1, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
        ids = torch.randint(0, V, (1, S), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        for tag in ("base", "lora"):
            if tag == "lora":
                m._llm.lora_load(adapter(h, nl, ffn, args.r, g), args.r, 2.0 * args.r)
            res[f"{name}_{tag}_prefill_ms"] = kernel_times(lambda: m._llm.forward(input_ids=ids, last_only=True))
            res[f"{name}_{tag}_decode32_ms"] = kernel_times(
                lambda: m._llm.generate(prompt, 32, use_graph=False, eos_token_id=-1))
        del m
        torch.cuda.empty_cache()
    with open(args.profile, "w") as f:
        json.dump(res, f, indent=1)
    for k, v in res.items():
        if isinstance(v, dict):
            print(k, f"total {sum(v.values()):.2f} ms:", ", ".join(f"{n} {t:.2f}" for n, t in list(v.items())[:8]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--shapes", default="7b,13b")
    ap.add_argument("--r", type=int, default=16)
    ap.add_argument("--json", default=None)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    if args.profile:
        return profile_run(args, card)
    res = {"card": card, "r": args.r}
    for name in args.shapes.split(","):
        h, nl, nh, ffn, V = SHAPES[name]
        cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=ffn, num_hidden_layers=nl,
                          num_attention_heads=nh, num_key_value_heads=nh, rms_norm_eps=1e-6,
                          max_position_embeddings=S)
        g = torch.Generator(device="cuda").manual_seed(0)
        sd = state_dict(h, nl, ffn, V, g)
        # the handles copy q|k|v and gate|up into fused layouts and borrow the rest; merging changes o_proj / down_proj
        # in place, so only those are cloned for the LoRA model.  Beams need 5 cache rows of S: 7B only.
        rows = 5 if name == "7b" else 1
        models = {k: LlamaForCausalLM(cfg, sd if k == "base" else
                                      {k2: v.clone() if ("o_proj" in k2 or "down_proj" in k2) else v for k2, v in sd.items()},
                                      device="cuda", max_batch=rows, max_seq=S) for k in ("base", "lora")}
        del sd
        models["lora"]._llm.lora_load(adapter(h, nl, ffn, args.r, g), args.r, 2.0 * args.r)
        torch.cuda.empty_cache()
        beams = (4, 5) if rows >= 5 else ()
        prompt = torch.randint(0, V, (1, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
        ids = torch.randint(0, V, (1, S), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
        runs = {"base": [], "lora": []}
        for _ in range(args.reps):
            for k, m in models.items():
                runs[k].append(measure(m, prompt, ids, beams))
        models["lora"]._llm.lora_merge()
        runs["base_again"], runs["merged"] = [], []
        for _ in range(args.reps):
            runs["base_again"].append(measure(models["base"], prompt, ids, beams))
            runs["merged"].append(measure(models["lora"], prompt, ids, beams))
        for k, lst in runs.items():
            for metric in lst[0]:
                vals = [x[metric] for x in lst]
                res[f"{name}_{k}_{metric}"] = statistics.median(vals)
        print(json.dumps({k: v for k, v in res.items() if k.startswith(name)}), flush=True)
        del models, m
        torch.cuda.empty_cache()
    res["median_sm_clock_mhz"] = statistics.median(CLOCKS) if CLOCKS else None
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
