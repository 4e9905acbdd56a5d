"""One small launch of every kernel the generation controls touch, through the C ABI, for compute-sanitizer:

    compute-sanitizer --tool memcheck  --error-exitcode 1 python tests/sanitize_processors_driver.py
    compute-sanitizer --tool racecheck --error-exitcode 1 python tests/sanitize_processors_driver.py

Covers logits_process_kernel on int64 histories (seedb200_sample_processed, the device loop) and on the int32 beam
token table with the fp16 log_softmax pass, its shared bitmap and in-place writes; the top-k histogram select inside
sample_kernel (T == 1 and T != 1, top_k < V) and inside beam_row_stats_kernel; and the token-table gather of
beam_score_kernel, eagerly and from a captured graph.  Vocabularies: 40194 and an odd 1001.  Each result is also
checked, so a clean run is known to have computed the right thing.  `--only name` runs one family.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import processors_ref as PR  # noqa: E402
from seed_b200 import lib as L

DEV = "cuda"
ALL = {"top_k": 7, "repetition_penalty": 1.3, "no_repeat_ngram_size": 2, "min_length": 30, "min_new_tokens": 4}


def sample():
    g = torch.Generator().manual_seed(0)
    B, S, eos = 3, 9, 5
    for V in (40194, 1001):
        logits = (torch.randn((B, V), generator=g) * 3).half()
        hist = torch.randint(0, V, (B, 21), generator=g)
        hist[:, 19:] = hist[:, 3:5]                        # a repeated bigram: the n-gram ban fires
        lg, hd = logits.to(DEV), hist.to(DEV)
        for T in (1.0, 0.7):
            for do_sample in (False, True):
                got = L.sample(lg, do_sample=do_sample, temperature=T, top_p=0.9, seed=2, step=1, history=hd,
                               prompt_len=S, eos_token_id=eos, **ALL).cpu()
                for b in range(B):
                    tok, dm, nm = PR.sample_row(logits[b], hist[b].tolist(), S, eos, ALL, do_sample, T, 0.9, 2, 0,
                                                1, b)
                    assert dm < 1e-5 or nm < 2e-6 or int(got[b]) == tok, (V, T, do_sample, b)


def models():
    from transformers.models.llama.configuration_llama import LlamaConfig

    from models.llama_xformer import LlamaForCausalLM
    from seed_b200 import synth

    h, nl, nh, ffn, V = 512, 2, 4, 1408, 1056
    cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=ffn, num_hidden_layers=nl, num_attention_heads=nh,
                      num_key_value_heads=nh, rms_norm_eps=1e-6, max_position_embeddings=2048)
    p = synth.prompt_ids(2, 40, 1, text_vocab=V - 66, n_codes=64).to(DEV)
    llm = LlamaForCausalLM(cfg, synth.llama_state_dict(h, nl, ffn, V), device=DEV, max_batch=6, max_seq=96)
    for use_graph in (False, True):
        llm._draws = 0
        a = llm.generate(input_ids=p, max_new_tokens=8, do_sample=True, temperature=0.8, top_p=0.9, seed=1,
                         eos_token_id=3, use_graph=use_graph, **ALL)
        llm._draws = 0
        b = llm.generate(input_ids=p, max_new_tokens=8, num_beams=3, do_sample=True, temperature=0.8, top_p=0.9,
                         seed=1, eos_token_id=3, pad_token_id=V - 1, use_graph=use_graph, **ALL)
        assert a.shape[0] == 2 and b.shape[0] == 2
        if use_graph:
            assert torch.equal(a, a_eager) and torch.equal(b, b_eager)
        a_eager, b_eager = a, b


FAMILIES = {"sample": sample, "models": models}

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
