"""Launches each contrastive-search kernel once through the C ABI, eagerly and from a captured CUDA graph, and checks
every result against tests/contrastive_ref.py.  Meant to run under compute-sanitizer (memcheck, racecheck):

    compute-sanitizer --tool memcheck python tests/sanitize_contrastive_driver.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import contrastive_ref as CR  # noqa: E402
from seed_b200 import lib as L  # noqa: E402
from transformers.models.llama.configuration_llama import LlamaConfig  # noqa: E402


def kernels(capture: bool):
    g = torch.Generator().manual_seed(1)
    B, k, V, H, S, rows = 2, 4, 1001, 512, 9, 16
    logits = (torch.randn((B, V), generator=g) * 3).half().cuda()
    hs = torch.randn((B, S, H), generator=g).half().cuda()
    cand = torch.randn((B, k, H), generator=g).half().cuda()
    ctx = torch.zeros((B, rows, H), dtype=torch.float16, device="cuda")
    run = lambda: (L.contrastive_context_init(hs, ctx), L.contrastive_candidates(logits, k))   # noqa: E731
    if capture:
        run()
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            _, (ids, probs) = run()
        gr.replay()
    else:
        _, (ids, probs) = run()
    sel, sc = L.contrastive_rank(ctx, S, cand, probs, 0.6)
    torch.cuda.synchronize()
    for b in range(B):
        assert (ctx[b, :S].float() - CR.normalise(hs[b].cpu()).cuda().float()).abs().max() <= 1e-3
        rv, ri = CR.topk(CR.softmax16(logits[b].cpu()), k)
        assert ids[b].cpu().tolist() == ri.tolist(), (ids[b], ri)
        rsel, rsc, rhn = CR.rank(ctx[b, :S].cpu(), cand[b].cpu(), probs[b].cpu(), 0.6)
        assert (sc[b].cpu() - rsc.float()).abs().max() <= 2e-3
        assert CR.gap(rsc) <= 2e-3 or int(sel[b]) == rsel


def loop(use_graph: bool):
    from seed_b200 import synth
    from seed_b200.llama import LlamaForCausalLM

    h, nl, nh, ffn, V = 256, 1, 2, 512, 512
    cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=ffn, num_hidden_layers=nl, num_attention_heads=nh,
                      num_key_value_heads=nh, rms_norm_eps=1e-6, max_position_embeddings=2048)
    m = LlamaForCausalLM(cfg, synth.llama_state_dict(h, nl, ffn, V, seed=2), device="cuda", max_batch=8, max_seq=48)
    ids = torch.randint(3, V, (2, 12), generator=torch.Generator().manual_seed(3)).cuda()
    out = m.generate(input_ids=ids, max_new_tokens=20, penalty_alpha=0.6, top_k=4, eos_token_id=-1,
                     use_graph=use_graph, repetition_penalty=1.2)
    torch.cuda.synchronize()
    assert out.shape == (2, 32) and bool((out >= 0).all() and (out < V).all())
    return out


if __name__ == "__main__":
    kernels(False)
    kernels(True)
    assert torch.equal(loop(False), loop(True))
    print("sanitize_contrastive_driver: ok")
