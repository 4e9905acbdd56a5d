"""One small launch of every LoRA kernel through the C ABI, for compute-sanitizer:

    compute-sanitizer --tool memcheck  --error-exitcode 1 python tests/sanitize_lora_driver.py
    compute-sanitizer --tool racecheck --error-exitcode 1 python tests/sanitize_lora_driver.py

Covers the decode shrink (every M, with and without the folded RMSNorm), the prefill shrink (GEMM), the GEMV with the
expand in its epilogue (every M, both modes, with and without residual), the GEMM + expand kernel (every r bucket,
both modes), and load / forward / decode / merge of a LoRA model.  Each result is also checked against
tests/lora_ref.py, so a clean run is known to have computed the right thing.  `--only name` runs one family.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import lora_ref as R  # noqa: E402
from seed_b200 import lib as L

DEV = "cuda"


def rnd(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half().to(DEV)


def shrink():
    K = 512
    a = rnd(48, K, seed=1, scale=0.05)
    w = (1.0 + rnd(K, seed=2, scale=0.1).float()).half()
    for M in (1, 2, 3, 4, 37):
        x = rnd(M, K, seed=M)
        t = L.lora_shrink(x, a)
        assert torch.all((t.cpu().double() - R.shrink(x.cpu(), a.cpu()).double()).abs()
                         <= R.shrink_bound(x.cpu(), a.cpu())), M
        if M <= 4:
            L.lora_shrink(x, a, norm_w=w)


def expand():
    K, N = 256, 512
    x1, x8 = rnd(3, K, seed=3), rnd(40, K, seed=4)
    w = rnd(N, K, seed=5, scale=0.05)
    res1, res8 = rnd(3, N, seed=6), rnd(40, N, seed=7)
    for r in (5, 16, 30, 64):
        a = rnd(2 * r, K, seed=8 + r, scale=0.05)
        b = rnd(N, r, seed=9 + r, scale=0.3)
        for x, res, fn in ((x1, res1, L.gemv_lora), (x8, res8, L.gemm_lora)):
            t = L.lora_shrink(x, a)
            lo = L.lora_operand(t, b, r, 128, 2, 2.0)
            y = fn(x, w, lo)
            base = (L.gemv if fn is L.gemv_lora else L.gemm)(x, w)
            assert torch.equal(fn(x, w, lo, residual=res), (y.float() + res.float()).half()), r
            assert bool(torch.isfinite(y.float()).all()) and bool((y != base).any()), r
            fn(x, w, lo, mode=1)


def models():
    from transformers.models.llama.configuration_llama import LlamaConfig

    from oracle import synth
    from seed_b200.llama import LlamaForCausalLM

    H, NL, FFN, V = 256, 2, 512, 1000
    cfg = LlamaConfig(vocab_size=V, hidden_size=H, intermediate_size=FFN, num_hidden_layers=NL, num_attention_heads=2,
                      num_key_value_heads=2, rms_norm_eps=1e-6, max_position_embeddings=2048)
    m = LlamaForCausalLM(cfg, synth.llama_state_dict(H, NL, FFN, V, seed=1), device=DEV, max_batch=2, max_seq=64)
    ad = {}
    for l in range(NL):
        for nm, n, k in (("self_attn.q_proj", H, H), ("self_attn.k_proj", H, H), ("self_attn.v_proj", H, H),
                         ("self_attn.o_proj", H, H), ("mlp.gate_proj", FFN, H), ("mlp.up_proj", FFN, H),
                         ("mlp.down_proj", H, FFN)):
            ad[f"model.layers.{l}.{nm}.lora_A.weight"] = rnd(8, k, seed=len(ad), scale=k ** -0.5)
            ad[f"model.layers.{l}.{nm}.lora_B.weight"] = rnd(n, 8, seed=len(ad) + 1, scale=0.3)
    ids = torch.randint(3, V, (2, 12), generator=torch.Generator().manual_seed(2)).to(DEV)
    base = m(ids).logits.clone()
    m._llm.lora_load(ad, 8, 16.0)
    lora = m(ids).logits.clone()
    assert not torch.equal(lora, base)
    m.generate(ids[:1], max_new_tokens=4, eos_token_id=-1)                 # decode through the fused GEMV
    m._llm.lora_merge()
    merged = m(ids).logits
    assert ((merged.float() - lora.float()).norm() / lora.float().norm()).item() <= 1e-2


FAMILIES = {"shrink": shrink, "expand": expand, "models": models}

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", nargs="*", default=None)
    a = ap.parse_args()
    for name, fn in FAMILIES.items():
        if a.only and name not in a.only:
            continue
        fn()
        torch.cuda.synchronize()
        print(f"{name}: ok ({L.launch_count()} launches so far)", flush=True)
