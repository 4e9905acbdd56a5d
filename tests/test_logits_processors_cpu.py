"""The generation-control restatement (tests/processors_ref.py) against the installed transformers' processor classes
and generate(), and the C ABI surface of seedb200_logits_params, without a GPU."""
import ctypes as C
import os
import re
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import processors_ref as PR  # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fp16_row(V, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(V, generator=g) * 4).half()


@pytest.mark.parametrize("penalty", [2.0, 0.5, 1.3])
def test_repetition_penalty_matches_transformers(penalty):
    from transformers import RepetitionPenaltyLogitsProcessor

    V = 50
    row = fp16_row(V, 1)
    hist = [3, 7, 7, 12, 3, 49, 0, 7]                       # repeated ids are penalised once
    ref = RepetitionPenaltyLogitsProcessor(penalty)(torch.tensor([hist]), row[None].float().clone())[0]
    got = PR.process(row, hist, 4, -1, {"repetition_penalty": penalty}).float()
    touched = torch.zeros(V, dtype=torch.bool)
    touched[hist] = True
    assert torch.equal(got[~touched], row.float()[~touched])
    # fp16 rounding of the fp32 result; a CPU division and the CUDA reciprocal may differ by one fp16 ulp
    assert torch.allclose(got[touched], ref[touched].half().float(), rtol=1e-3, atol=0)
    if penalty in (2.0, 0.5):                               # exact reciprocals: bit-identical
        assert torch.equal(got, ref.half().float())


@pytest.mark.parametrize("n", [1, 2, 3, 4, 9])
def test_no_repeat_ngram_matches_transformers(n):
    from transformers import NoRepeatNGramLogitsProcessor

    V = 20
    row = fp16_row(V, n)
    # prompt [5, 6, 5, 6, 7], generated [5, 6]: the 3-gram (5, 6) -> {5, 7} spans the prompt boundary
    hist = [5, 6, 5, 6, 7, 5, 6]
    ref = NoRepeatNGramLogitsProcessor(n)(torch.tensor([hist]), row[None].float().clone())[0]
    got = PR.process(row, hist, 5, -1, {"no_repeat_ngram_size": n}).float()
    assert torch.equal(got, ref)
    if n == 3:
        assert got[7] == float("-inf") and got[5] == float("-inf") and torch.isfinite(got[6])
    if n == 9:                                              # L + 1 < n: nothing banned
        assert torch.equal(got, row.float())


def test_length_rules_match_transformers():
    from transformers import MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor

    V, eos, S = 16, 4, 3
    row = fp16_row(V, 9)
    for L in range(S, S + 6):
        hist = list(range(L))
        for m in (0, 2, 5, 7):
            ref = MinLengthLogitsProcessor(m, eos)(torch.tensor([hist]), row[None].float().clone())[0]
            assert torch.equal(PR.process(row, hist, S, eos, {"min_length": m}).float(), ref), (L, m)
            ref = MinNewTokensLengthLogitsProcessor(S, m, eos)(torch.tensor([hist]), row[None].float().clone())[0]
            assert torch.equal(PR.process(row, hist, S, eos, {"min_new_tokens": m}).float(), ref), (L, m)
    assert torch.equal(PR.process(row, [1, 2], 2, -1, {"min_length": 9, "min_new_tokens": 9}), row)   # no eos


@pytest.mark.parametrize("k,min_keep", [(1, 1), (3, 1), (4, 1), (1, 2), (7, 2), (40, 1)])
def test_top_k_matches_transformers_with_ties(k, min_keep):
    from transformers import TopKLogitsWarper

    V = 12
    row = torch.tensor([1.0, 5.0, 3.0, 5.0, 3.0, 3.0, -2.0, 0.5, 3.0, float("-inf"), 4.0, 3.0]).half()
    keep = PR.top_k_keep(row, k, min_keep)
    ref = TopKLogitsWarper(k, min_tokens_to_keep=min_keep)(None, row[None].float().clone())[0]
    fin = torch.isfinite(row.float())                       # HF's -inf filter value hides a -inf input either way
    assert torch.equal(keep[fin], torch.isfinite(ref)[fin]), (keep, ref)
    if k >= V:
        assert bool(keep[torch.isfinite(row.float())].all())


def test_sample_row_top_k_then_top_p_keeps_the_argmax():
    V = 64
    row = fp16_row(V, 3)
    for seed in range(20):
        tok, _, _ = PR.sample_row(row, [], 0, -1, {"top_k": 1}, True, 0.7, 0.9, seed=seed)
        assert tok == int(torch.argmax(row.float()))
        tok, _, _ = PR.sample_row(row, [], 0, -1, {"top_k": 5}, True, 1.0, 1.0, seed=seed)
        assert tok in torch.topk(row.float(), 5).indices.tolist()


def _tiny_model(seed):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(seed)
    cfg = LlamaConfig(vocab_size=97, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                      num_attention_heads=4, num_key_value_heads=4, max_position_embeddings=128)
    model = LlamaForCausalLM(cfg).eval()
    model.generation_config.eos_token_id = None
    model.generation_config.pad_token_id = 0
    return model


CTLS = [{"repetition_penalty": 1.5}, {"no_repeat_ngram_size": 2}, {"repetition_penalty": 0.7, "no_repeat_ngram_size": 3}]


@pytest.mark.parametrize("ctl", CTLS)
def test_restated_greedy_matches_transformers_generate(ctl):
    model = _tiny_model(3)
    ids = torch.randint(3, 97, (2, 6), generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        hf = model.generate(ids, do_sample=False, max_new_tokens=10, eos_token_id=None, pad_token_id=0, **ctl)
        ref = PR.generate(lambda seq: model(seq).logits[:, -1].float(), ids, 10, ctl)[0]
    assert torch.equal(ref, hf), (ref.tolist(), hf.tolist())


@pytest.mark.parametrize("ctl", CTLS)
@pytest.mark.parametrize("k", [2, 4])
def test_restated_beam_search_matches_transformers_generate(ctl, k):
    model = _tiny_model(5 + k)
    ids = torch.randint(3, 97, (2, 6), generator=torch.Generator().manual_seed(k))
    with torch.no_grad():
        hf = model.generate(ids, num_beams=k, do_sample=False, max_new_tokens=8, eos_token_id=None, pad_token_id=0,
                            length_penalty=1.0, early_stopping=False, **ctl)
        ref = PR.beam_generate(lambda seq, bi: model(seq).logits[:, -1].float(), ids, 8, k, ctl)[0]
    assert torch.equal(ref, hf), (ref.tolist(), hf.tolist())


def test_generate_keywords_are_validated_as_transformers_does():
    from seed_b200.llama import LlamaForCausalLM as M

    ok = dict(M._GEN_DEFAULTS)
    assert M._controls(ok) == PR.NEUTRAL
    for name, bad in (("top_k", -1), ("repetition_penalty", 0.0), ("repetition_penalty", float("nan")),
                      ("repetition_penalty", float("inf")), ("no_repeat_ngram_size", -2), ("min_length", -1),
                      ("min_new_tokens", -3)):
        with pytest.raises(ValueError):
            M._controls(dict(ok, **{name: bad}))


def test_ctypes_struct_matches_header():
    from seed_b200 import lib as L

    hdr = open(os.path.join(REPO, "include", "seedb200.h")).read()
    body = re.search(r"typedef struct seedb200_logits_params \{(.*?)\} seedb200_logits_params;", hdr, re.S).group(1)
    fields = re.findall(r"\b(int32_t|float)\s+(\w+);", body)
    ctype = {"int32_t": C.c_int32, "float": C.c_float}
    assert [(n, ctype[t]) for t, n in fields] == list(L.LogitsParams._fields_)
    assert C.sizeof(L.LogitsParams) == 20
    assert L.logits_params() is None
    assert L.logits_params(top_k=50).top_k == 50


@pytest.fixture(scope="module")
def clib():
    from seed_b200 import lib as L

    if not os.path.exists(L.LIB_PATH):
        pytest.skip("libseedb200.so not built")
    try:
        return L.load()
    except OSError as e:            # the CUDA runtime may be absent
        pytest.skip(f"library does not load here: {e}")


BAD = [dict(top_k=-1), dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0),
       dict(repetition_penalty=float("inf")), dict(repetition_penalty=float("nan")), dict(no_repeat_ngram_size=-1),
       dict(min_length=-1), dict(min_new_tokens=-1)]


@pytest.mark.parametrize("bad", BAD)
def test_entry_points_refuse_bad_parameters(clib, bad):
    from seed_b200 import lib as L

    lp = L.LogitsParams(0, 1.0, 0, 0, 0)
    for k, v in bad.items():
        setattr(lp, k, v)
    sp = L.SampleParams(1, 1.0, 1.0, 0, 0)
    fake = C.c_void_p(16)                     # never dereferenced: the parameters are refused first
    assert clib.seedb200_sample_processed(fake, 8, 1, 8, C.byref(sp), 0, fake, None, C.byref(lp), fake, 8, 1, 0,
                                          -1) == 1
    assert b"seedb200_sample_processed" in clib.seedb200_last_error()
    assert clib.seedb200_llama_generate_processed(None, None, 1, 1, 1, C.byref(sp), -1, 0, 0, None, None, None,
                                                  C.byref(lp)) == 1
    assert b"llama_generate" in clib.seedb200_last_error() and b"null" not in clib.seedb200_last_error()
    bp = L.beam_params(2)
    assert clib.seedb200_llama_beam_generate_processed(None, None, 1, 1, 1, C.byref(bp), -1, 0, 0, None, None, None,
                                                       None, C.byref(lp)) == 1
    assert b"llama_beam_generate" in clib.seedb200_last_error() and b"null" not in clib.seedb200_last_error()
