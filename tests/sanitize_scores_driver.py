"""One small run of every kernel that the generation scores changed, through the C ABI, for compute-sanitizer:

    compute-sanitizer --tool memcheck  --error-exitcode 1 python tests/sanitize_scores_driver.py
    compute-sanitizer --tool racecheck --error-exitcode 1 python tests/sanitize_scores_driver.py

Covers every kernel that writes scores or beam indices, on a vocabulary that is not a multiple of 8 so that the last
row ends inside its pitch, eagerly and from a captured graph, with and without the history controls, with an eos id:
  - sample_kernel (greedy and warped rows) through seedb200_llama_generate_ex, num_return_sequences 1 and 3, and
    through seedb200_sample_scores (the per-token route, compared at num_return_sequences 1);
  - contrastive_candidates_kernel through seedb200_llama_contrastive_generate_ex;
  - beam_row_stats_kernel, beam_scores_warp_kernel, beam_score_kernel (the done step) and beam_finalize_kernel
    (beam_indices) through seedb200_llama_beam_generate_ex, beam search and beam sampling.
Each result is checked against another route (eager against graph for the loops), so a clean run is known to have
computed the same thing both ways.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

from oracle import synth

HID, LAYERS, HEADS, FFN, VOCAB = 256, 1, 2, 512, 523


def model():
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=VOCAB, hidden_size=HID, intermediate_size=FFN, num_hidden_layers=LAYERS,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=4096)
    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=3)
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=6, max_seq=64)


def main():
    torch.cuda.set_device(0)
    m = model()
    ids = synth.prompt_ids(2, 9, n_image_spans=0, text_vocab=VOCAB - 8, n_codes=4, seed=1).cuda()
    for mode in (dict(do_sample=False), dict(do_sample=True, temperature=0.9, top_p=0.8)):
        for ctl in ({}, dict(top_k=20, repetition_penalty=1.2, min_new_tokens=2)):
            for n in ((1, 3) if mode["do_sample"] else (1,)):
                outs = []
                # the per-token route prefills the expanded batch when n > 1, which may round some prefill logits
                # differently; there the eager and graph-replayed device loops are compared with each other
                routes = [dict(device_loop=True, use_graph=False), dict(device_loop=True, use_graph=True)]
                for route in routes + ([dict(device_loop=False)] if n == 1 else []):
                    m._draws = 0
                    outs.append(m.generate(input_ids=ids, seed=7, max_new_tokens=8, eos_token_id=5,
                                           num_return_sequences=n, return_dict_in_generate=True, output_scores=True,
                                           **mode, **ctl, **route))
                torch.cuda.synchronize()
                for o in outs[1:]:
                    assert torch.equal(o.sequences, outs[0].sequences), (mode, ctl, n)
                    assert len(o.scores) == len(outs[0].scores) == o.sequences.shape[1] - 9
                    for a, b in zip(o.scores, outs[0].scores):
                        assert torch.equal(a, b), (mode, ctl, n)
    for mode in (dict(penalty_alpha=0.6, top_k=3), dict(num_beams=2), dict(num_beams=3, do_sample=True, top_p=0.8)):
        for ctl in ({}, dict(repetition_penalty=1.2, min_new_tokens=2)):
            outs = []
            for graph in (False, True):
                m._draws = 0
                outs.append(m.generate(input_ids=ids, seed=7, max_new_tokens=8, eos_token_id=5, use_graph=graph,
                                       return_dict_in_generate=True, output_scores=True, **mode, **ctl))
            torch.cuda.synchronize()
            a, b = outs
            assert torch.equal(a.sequences, b.sequences) and len(a.scores) == len(b.scores) > 0, (mode, ctl)
            for x, y in zip(a.scores, b.scores):
                assert torch.equal(x, y), (mode, ctl)
            if "num_beams" in mode:
                assert torch.equal(a.beam_indices, b.beam_indices) and torch.equal(a.sequences_scores,
                                                                                   b.sequences_scores), (mode, ctl)
    print("sanitize_scores_driver: all checks passed")


if __name__ == "__main__":
    main()
