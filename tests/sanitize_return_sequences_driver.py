"""One small run of every kernel that num_return_sequences changed, through the C ABI, for compute-sanitizer:

    compute-sanitizer --tool memcheck  --error-exitcode 1 python tests/sanitize_return_sequences_driver.py
    compute-sanitizer --tool racecheck --error-exitcode 1 python tests/sanitize_return_sequences_driver.py

Covers the lineage init of sampling rows (sample_lineage_kernel) and of beam-sample searches (beam_init_kernel with
several searches per prompt), and the first-step sampler and beam candidates reading prompt rows shared by n rows,
through seedb200_llama_generate_n{,_processed} and seedb200_llama_beam_generate_n{,_processed}, eagerly and from a
captured graph, on a fused (max_seq <= 2048) and a split-KV (max_seq > 2048) model.  Each result is checked against
the same call on the expanded prompt, so a clean run is known to have computed the right thing.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

from oracle import synth

HID, LAYERS, HEADS, FFN, VOCAB = 256, 1, 2, 512, 520


def model(max_seq):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=VOCAB, hidden_size=HID, intermediate_size=FFN, num_hidden_layers=LAYERS,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=4096)
    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=3)
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=12, max_seq=max_seq)


def main():
    torch.cuda.set_device(0)
    samp = dict(do_sample=True, temperature=0.9, top_p=0.8)
    for max_seq in (64, 2304):
        m = model(max_seq)
        ids = synth.prompt_ids(2, 9, n_image_spans=0, text_vocab=VOCAB - 8, n_codes=4, seed=1).cuda()
        for ctl in ({}, dict(repetition_penalty=1.2, min_new_tokens=2)):
            for graph in (False, True):
                for n, beams in ((3, 1), (2, 2), (3, 2)):
                    kw = dict(max_new_tokens=8, eos_token_id=5, use_graph=graph, num_beams=beams, **samp, **ctl)
                    m._draws = 0
                    got = m.generate(input_ids=ids, seed=7, num_return_sequences=n, **kw)
                    m._draws = 0
                    exp = m.generate(input_ids=ids.repeat_interleave(n, 0), seed=7, device_loop=True, **kw)
                    torch.cuda.synchronize()
                    assert torch.equal(got, exp), (max_seq, ctl, graph, n, beams)
        print(f"max_seq {max_seq}: ok")
    print("sanitize_return_sequences_driver: all checks passed")


if __name__ == "__main__":
    main()
