"""fp16 vs LLM.int8() vs 4-bit (NF4) LLaMA on one GPU: 13B decode and 7B prefill, random-init weights made on the device.

    python tools/int8_bench.py [--reps 3] [--json OUT]

The three handles of a shape are built in one process and timed alternately (fp16, int8, nf4, fp16, ...):
  * 13B decode: prompt P = 256, 128 new tokens through seedb200_llama_generate (greedy, graph-replayed steps);
    ms/token = (time(129 new tokens) - time(1 new token)) / 128, i.e. without the prefill.  Achieved GB/s counts the
    weight bytes one decode step must read (quantised decoder linears + their scales + fp16 lm_head row reads).
  * 13B beam search, B = 1, k = 5: ms per decode step = (time(33 new tokens) - time(1 new token)) / 32.  Five rows
    take the GEMM path: the 4-bit model dequantises every decoder linear in every step.
  * 7B prefill: B = 1, S = 2048, logits of the last position only; tokens/s.
  * device memory: get_memory_footprint() (weights) of each model.
The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from transformers.models.llama.configuration_llama import LlamaConfig  # noqa: E402

from seed_b200.llama import LlamaForCausalLM  # noqa: E402

SHAPES = {"7b": (4096, 32, 32, 11008, 32000), "13b": (5120, 40, 40, 13824, 32000)}


def random_state_dict(h, nl, ffn, V, seed=0):
    """yields the tensors one at a time, on the device, so that the int8 build never holds the fp16 model"""
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rnd(*shape, scale=0.02):
        return torch.randn(*shape, device="cuda", dtype=torch.float16, generator=g) * scale

    class SD(dict):
        def items(self):
            yield "model.embed_tokens.weight", rnd(V, h)
            yield "model.norm.weight", torch.ones(h, device="cuda", dtype=torch.float16)
            yield "lm_head.weight", rnd(V, h)
            for l in range(nl):
                p = f"model.layers.{l}."
                yield p + "input_layernorm.weight", torch.ones(h, device="cuda", dtype=torch.float16)
                yield p + "post_attention_layernorm.weight", torch.ones(h, device="cuda", dtype=torch.float16)
                for nm, shp in (("self_attn.q_proj", (h, h)), ("self_attn.k_proj", (h, h)), ("self_attn.v_proj", (h, h)),
                                ("self_attn.o_proj", (h, h)), ("mlp.gate_proj", (ffn, h)), ("mlp.up_proj", (ffn, h)),
                                ("mlp.down_proj", (h, ffn))):
                    yield p + nm + ".weight", rnd(*shp)

    return SD()


KINDS = ("fp16", "int8", "nf4")


def build(shape, kind, max_seq, max_batch=1):
    h, nl, nh, ffn, V = shape
    cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=ffn, num_hidden_layers=nl, num_attention_heads=nh,
                      num_key_value_heads=nh, rms_norm_eps=1e-6, max_position_embeddings=max(max_seq, 2048))
    q = {"int8": {"load_in_8bit": True}, "nf4": {"load_in_4bit": True, "bnb_4bit_quant_type": "nf4"}}.get(kind, {})
    return LlamaForCausalLM(cfg, random_state_dict(h, nl, ffn, V), device="cuda", max_batch=max_batch,
                            max_seq=max_seq, **q)


def timed(fn, reps=1):
    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps


def decode_ms_per_token(m, prompt, new):
    gen = lambda n: m._llm.generate(prompt, n, use_graph=True, eos_token_id=-1)   # noqa: E731
    return (timed(lambda: gen(new + 1), 2) - timed(lambda: gen(1), 2)) / new


def beam_ms_per_step(m, prompt, new, k):
    gen = lambda n: m._llm.beam_generate(prompt, n, k, eos_token_id=-1)   # noqa: E731
    return (timed(lambda: gen(new + 1), 2) - timed(lambda: gen(1), 2)) / new


def step_bytes(shape, kind):
    h, nl, nh, ffn, V = shape
    lin = nl * (4 * h * h + 3 * h * ffn)
    rows = nl * (3 * h + h + 2 * ffn + h)
    q = {"fp16": 2 * lin, "int8": lin + 4 * rows, "nf4": lin // 2 + 4 * (lin // 64)}[kind]
    return q + 2 * V * h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("int8_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card}
    P, NEW = 256, 128
    shape = SHAPES["13b"]
    BEAMS, BNEW = 5, 32
    models = {k: build(shape, k, P + NEW + 8, max_batch=BEAMS) for k in KINDS}
    for k, m in models.items():
        res[f"13b_{k}_weight_GB"] = m.get_memory_footprint() / 1e9
    prompt = torch.randint(0, shape[4], (1, P), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    dec = {k: [] for k in KINDS}
    beam = {k: [] for k in KINDS}
    for _ in range(args.reps):
        for k, m in models.items():
            dec[k].append(decode_ms_per_token(m, prompt, NEW))
            beam[k].append(beam_ms_per_step(m, prompt, BNEW, BEAMS))
    for k in dec:
        ms = min(dec[k])
        res[f"13b_decode_{k}_ms_per_token"] = dec[k]
        res[f"13b_decode_{k}_GBps"] = step_bytes(shape, k) / (ms * 1e-3) / 1e9
        res[f"13b_beam{BEAMS}_{k}_ms_per_step"] = beam[k]
    del models, m
    torch.cuda.empty_cache()
    shape = SHAPES["7b"]
    S = 2048
    models = {k: build(shape, k, S) for k in KINDS}
    for k, m in models.items():
        res[f"7b_{k}_weight_GB"] = m.get_memory_footprint() / 1e9
    ids = torch.randint(0, shape[4], (1, S), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    pre = {k: [] for k in KINDS}
    for _ in range(args.reps):
        for k, m in models.items():
            pre[k].append(S / (timed(lambda: m._llm.forward(input_ids=ids, last_only=True), 3) * 1e-3))
    for k in pre:
        res[f"7b_prefill_{k}_tokens_per_s"] = pre[k]
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
