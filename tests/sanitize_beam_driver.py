"""One small launch of every beam-search kernel through the C ABI, for compute-sanitizer:

    compute-sanitizer --tool memcheck  --error-exitcode 1 python tests/sanitize_beam_driver.py
    compute-sanitizer --tool racecheck --error-exitcode 1 python tests/sanitize_beam_driver.py

Covers the candidate kernel (greedy and sampling, first step and decode step, every NC instantiation), the lineage
forms of the split-KV and fused decode attention, and beam_generate end to end (init, scorer with its cross-CTA
arrival counter and slot gather, finalize) eagerly and from a captured graph, on a fused (max_seq <= 2048) and a
split-KV (max_seq > 2048) model.  Each result is also checked, so a clean run is known to have computed the right
thing.  `--only name` runs one family.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import beam_ref as BR  # noqa: E402
from seed_b200 import lib as L

DEV = "cuda"


def select():
    g = torch.Generator().manual_seed(0)
    B, V = 2, 1000
    for k in (1, 2, 5, 8):                                # NC = 4, 4, 16, 16 (and 8 through k = 3 below)
        logits = (torch.randn((B * k, V), generator=g) * 3).half()
        bs = torch.zeros(B * k)
        bs.view(B, k)[:, 1:] = -1e9
        for first in (True, False):
            lg = logits[::k].contiguous() if first else logits
            rows = lg.repeat_interleave(k, 0) if first else lg
            s = (BR.log_probs(rows) + bs[:, None]).view(B, k * V)
            sc, ix = L.beam_select(lg.to(DEV), bs.to(DEV), B, k, first_step=first)
            rsc, _, _, _ = BR.select(s, k)
            assert torch.allclose(sc.cpu(), rsc, atol=4e-3, rtol=0), (k, first)
            L.beam_select(lg.to(DEV), bs.to(DEV), B, k, first_step=first, step=1, do_sample=True, temperature=0.7,
                          top_p=0.5, seed=3)
    logits = torch.randn((3, V), generator=g).half().to(DEV)
    L.beam_select(logits, torch.zeros(3, device=DEV), 1, 3, do_sample=True, top_p=0.9)


def attention():
    g = torch.Generator().manual_seed(1)
    H, D = 2, 128
    for max_seq, past in ((2500, 300), (256, 130)):
        k = torch.randn((5, H, max_seq, D), generator=g).half().to(DEV)
        v = torch.randn((5, H, max_seq, D), generator=g).half().to(DEV)
        slot = torch.randint(0, 4, (4, max_seq), generator=g, dtype=torch.int32)
        slot[:, past] = torch.arange(4, dtype=torch.int32)
        slot = slot.to(DEV)
        pos = torch.arange(max_seq, device=DEV)
        gk = k[slot.long(), :, pos[None, :], :].permute(0, 2, 1, 3).contiguous()
        gv = v[slot.long(), :, pos[None, :], :].permute(0, 2, 1, 3).contiguous()
        q = torch.randn((4, H, D), generator=g).half().to(DEV)
        assert torch.equal(L.decode_attention_lineage(q, k, v, slot, past + 1, D ** -0.5),
                           L.decode_attention(q, gk, gv, past + 1, D ** -0.5))
        if max_seq <= 2048:
            qkv = torch.randn((4, 3 * H * D), generator=g).half().to(DEV)
            assert torch.equal(L.decode_attention_rope_lineage(qkv, slot, H, past, k, v, D ** -0.5),
                               L.decode_attention_rope(qkv, None, H, past, gk, gv, D ** -0.5))


def models():
    from transformers.models.llama.configuration_llama import LlamaConfig

    from models.llama_xformer import LlamaForCausalLM
    from seed_b200 import synth

    h, nl, nh, ffn, V = 512, 2, 4, 1408, 1056
    cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=ffn, num_hidden_layers=nl, num_attention_heads=nh,
                      num_key_value_heads=nh, rms_norm_eps=1e-6, max_position_embeddings=4096)
    p = synth.prompt_ids(2, 40, 1, text_vocab=V - 66, n_codes=64).to(DEV)
    for max_seq in (96, 2100):                            # fused decode attention, then split-KV
        llm = LlamaForCausalLM(cfg, synth.llama_state_dict(h, nl, ffn, V), device=DEV, max_batch=1, max_seq=max_seq)
        free = llm.generate(input_ids=p, max_new_tokens=8, num_beams=3, eos_token_id=-1, use_graph=False)
        eos = int(free[0, 42])
        for use_graph in (False, True):
            a = llm.generate(input_ids=p, max_new_tokens=8, num_beams=3, eos_token_id=eos, pad_token_id=V - 1,
                             use_graph=use_graph)
            b = llm.generate(input_ids=p, max_new_tokens=8, num_beams=3, do_sample=True, top_p=0.5, temperature=0.7,
                             seed=1, eos_token_id=eos, pad_token_id=V - 1, use_graph=use_graph)
            assert a.shape[0] == 2 and b.shape[0] == 2
        del llm


FAMILIES = {"select": select, "attention": attention, "models": models}

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
