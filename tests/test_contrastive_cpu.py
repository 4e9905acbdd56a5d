"""The contrastive-search restatement (tests/contrastive_ref.py) pinned on hand-worked cases, the C ABI surface of
seedb200_contrastive_params and the refusals of generate(penalty_alpha=...), without a GPU."""
import ctypes as C
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import contrastive_ref as CR  # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float("nan")


def h(*v):
    return torch.tensor(v, dtype=torch.float16)


def test_normalise_rounds_the_norm_to_fp16_first():
    # ||(30, 16, 15)|| = 37.16180... -> fp16 37.15625; 30 / 37.15625 = 0.80740... -> fp16 0.8076171875.  Dividing by
    # the unrounded norm would give 0.80712890625.
    got = CR.normalise(h(30, 16, 15))
    assert got.tolist() == [0.8076171875, 0.4306640625, 0.40380859375]
    assert float(torch.tensor(30.0 ** 2 + 16 ** 2 + 15 ** 2).sqrt().half()) == 37.15625
    assert (h(30, 16, 15).float() / h(30, 16, 15).float().norm()).half().tolist()[0] == 0.80712890625
    assert CR.normalise(h(3, 4)).tolist() == [0.60009765625, 0.7998046875]


def test_cosine_is_one_fp16_rounding_of_the_dot():
    c = CR.normalise(h(3, 4))[None]                       # (0.60009765625, 0.7998046875)
    n = CR.normalise(h(4, 3))[None]                       # (0.7998046875, 0.60009765625)
    # 2 * 0.60009765625 * 0.7998046875 = 0.95992279..., one rounding to fp16: 0.9599609375
    cos = CR.cosines(c, n)
    assert cos.dtype == torch.float16 and cos.shape == (1, 1)
    assert float(cos) == 0.9599609375
    assert CR.cosines(c, c).item() == 1.0                 # 0.60009765625^2 + 0.7998046875^2 = 1.00000...


def test_penalty_is_the_max_over_the_context_and_nan_propagates():
    cos = torch.tensor([[0.25, -0.5], [0.75, -0.25], [0.5, -1.0]]).half()
    assert CR.nan_max(cos).tolist() == [0.75, -0.25]
    cos[1, 1] = NAN
    pen = CR.nan_max(cos)
    assert pen[0] == 0.75 and math.isnan(float(pen[1]))


def test_score_rounding_points():
    # alpha 0.6: fp16(fp32(0.4) * 0.5) = 0.199951171875, fp16(fp32(0.6) * 0.75) = 0.449951171875, and their fp16
    # difference is -0.25
    sc = CR.scores(h(0.5), h(0.75), 0.6)
    t1 = float(torch.tensor(np.float32(0.4) * np.float32(0.5)).half())
    t2 = float(torch.tensor(np.float32(0.6) * np.float32(0.75)).half())
    assert t1 == 0.199951171875 and t2 == 0.449951171875
    assert float(sc) == float(torch.tensor(t1 - t2).half()) == -0.25


def test_one_minus_alpha_is_rounded_from_double():
    # alpha 0.65: fp32(1 - 0.65) = 0.35 (0.3499999940...) but 1 - fp32(0.65) = 0.35000002; on the subnormal
    # probability 2^-19 * 15 the two scalars give different fp16 products, and the contract takes the first.
    alpha, q = 0.65, 1.7881393432617188e-06
    assert CR.c_prob(alpha) == np.float32(0.35) != np.float32(1.0 - np.float64(np.float32(alpha)))
    from_double = float(torch.tensor(np.float32(0.35) * np.float32(q)).half())
    from_fp32 = float(torch.tensor(np.float32(1.0 - np.float64(np.float32(alpha))) * np.float32(q)).half())
    assert from_double != from_fp32
    got = CR.scores(h(q), h(0.0), alpha)
    assert float(got) == from_double


def test_topk_ties_go_to_the_lower_id():
    probs = h(0.1, 0.3, 0.1, 0.3, 0.2, 0.0)
    v, ids = CR.topk(probs, 4)
    assert ids.tolist() == [1, 3, 4, 0] and v.tolist() == [float(h(0.3)), float(h(0.3)), float(h(0.2)), float(h(0.1))]


def test_topk_compares_fp16_probabilities_not_logits():
    # two different logits whose probabilities may round to one fp16 value: then the lower id comes first
    logits = torch.tensor([0.0, 5.0, 5.00390625, -30.0]).half()
    p = CR.softmax16(logits)
    assert logits[2] > logits[1]
    if p[1] == p[2]:
        assert CR.topk(p, 2)[1].tolist() == [1, 2]
    else:
        assert CR.topk(p, 2)[1].tolist() == [2, 1]


def test_softmax_is_one_rounding_of_the_reciprocal_product():
    logits = torch.tensor([1.0, 2.0, 3.0, -1.0]).half()
    x = logits.float()
    e = torch.exp(x - 3.0)
    assert torch.equal(CR.softmax16(logits), (e * (torch.tensor(1.0) / e.sum())).half())


def test_select_ties_and_nan():
    assert CR.select(h(0.5, 0.75, 0.75, 0.25)) == 1
    assert CR.select(h(0.5, NAN, 0.75, NAN)) == 1          # the first NaN wins
    assert CR.select(h(NAN, 0.75)) == 0
    assert CR.select(h(-0.25, -0.25)) == 0


def test_rank_end_to_end_on_a_two_dimensional_case():
    ctx = CR.normalise(torch.tensor([[1.0, 0.0], [0.0, 1.0]]).half())
    hs = torch.tensor([[1.0, 0.1], [1.0, 1.0]]).half()    # j=0 nearly repeats c_0; j=1 sits between both
    q = h(0.5, 0.375)
    sel, sc, hn = CR.rank(ctx, hs, q, 0.5)
    pen = CR.nan_max(CR.cosines(ctx, CR.normalise(hs)))
    assert sc.tolist() == CR.scores(q, pen, 0.5).tolist()
    assert sel == 1 and sc[1] > sc[0]


MODES = [({}, "greedy"), (dict(penalty_alpha=0.6), "greedy"), (dict(penalty_alpha=0.6, top_k=4), "contrastive"),
         (dict(penalty_alpha=0.6, top_k=1), "greedy"), (dict(penalty_alpha=0.0, top_k=4), "greedy"),
         (dict(penalty_alpha=-0.5, top_k=4), "greedy"), (dict(penalty_alpha=0.6, top_k=4, do_sample=True), "sample"),
         (dict(penalty_alpha=0.6, top_k=4, num_beams=2), "beam"),
         (dict(penalty_alpha=0.6, top_k=4, num_beams=2, do_sample=True), "beam_sample"),
         (dict(top_k=4), "greedy"), (dict(top_k=4, do_sample=True), "sample")]


@pytest.mark.parametrize("kw,expected", MODES)
def test_mode_selection_table(kw, expected):
    assert CR.mode(**kw) == expected


class _Forward:
    """candidates whose logits always favour token 3 and whose h are orthogonal to the context: eos is 3"""

    def __init__(self, V, H):
        self.V, self.H = V, H

    def __call__(self, t, ids):
        B, k = ids.shape
        lg = torch.zeros((B, k, self.V)).half()
        lg[..., 3] = 8.0
        hh = torch.zeros((B, k, self.H)).half()
        hh[..., 1] = 1.0
        return lg, hh

    def on_select(self, t, sels):
        pass


def test_pad_after_eos_and_stop_when_all_finished():
    V, H = 8, 4

    def prefill(prompt):
        B, S = prompt.shape
        lg = torch.zeros((B, V)).half()
        lg[0, 3] = 8.0                                       # sequence 0 emits eos at once
        lg[1, 5] = 8.0
        hs = torch.zeros((B, S, H)).half()
        hs[..., 0] = 1.0
        return lg, hs

    prompt = torch.tensor([[1, 2], [2, 1]])
    toks, gaps, _ = CR.generate(prefill, _Forward(V, H), prompt, 6, 2, 0.5, dict(CR.PR.NEUTRAL), eos=3, pad=0)
    assert toks.tolist() == [[3, 0], [5, 3]]                 # pad after eos, and the loop stops once both finished


def test_ctypes_struct_matches_header():
    from seed_b200 import lib as L

    hdr = open(os.path.join(REPO, "include", "seedb200.h")).read()
    body = re.search(r"typedef struct seedb200_contrastive_params \{(.*?)\} seedb200_contrastive_params;", hdr,
                     re.S).group(1)
    fields = re.findall(r"\b(int32_t|double)\s+(\w+);", body)
    ctype = {"int32_t": C.c_int32, "double": C.c_double}
    assert [(n, ctype[t]) for t, n in fields] == list(L.ContrastiveParams._fields_)
    assert C.sizeof(L.ContrastiveParams) == 16
    for name in ("seedb200_llama_contrastive_generate", "seedb200_contrastive_candidates", "seedb200_contrastive_rank",
                 "seedb200_contrastive_context_init"):
        assert name in L.EXPORTS and re.search(r"\b%s\(" % name, hdr)


@pytest.fixture(scope="module")
def clib():
    from seed_b200 import lib as L

    if not os.path.exists(L.LIB_PATH):
        pytest.skip("libseedb200.so not built")
    try:
        return L.load()
    except OSError as e:            # the CUDA runtime may be absent
        pytest.skip(f"library does not load here: {e}")


@pytest.mark.parametrize("top_k,alpha", [(1, 0.6), (9, 0.6), (0, 0.6), (4, 0.0), (4, -0.5), (4, NAN),
                                         (4, float("inf"))])
def test_entry_points_refuse_bad_parameters(clib, top_k, alpha):
    from seed_b200 import lib as L

    cp = L.ContrastiveParams(top_k, alpha)
    fake = C.c_void_p(16)                     # never dereferenced: the parameters are refused first
    assert clib.seedb200_llama_contrastive_generate(fake, fake, 1, 1, 1, C.byref(cp), -1, 0, 0, fake, None, None,
                                                    None) == 1
    err = clib.seedb200_last_error()
    assert b"llama_contrastive_generate" in err and (b"top_k" in err or b"penalty_alpha" in err)
    assert clib.seedb200_contrastive_rank(fake, 64, 4, 1, 16, fake, fake, 1, C.byref(cp), fake, fake, None) == 1
    assert b"seedb200_contrastive_rank" in clib.seedb200_last_error()
    if not 2 <= top_k <= 8:
        assert clib.seedb200_contrastive_candidates(fake, 64, 1, 64, top_k, fake, fake, None) == 1
        assert b"top_k" in clib.seedb200_last_error()


def _stub_model():
    """a LlamaForCausalLM with no handle: generate() must refuse before it touches one"""
    import torch.nn as nn
    from transformers.models.llama.configuration_llama import LlamaConfig

    from seed_b200.llama import LlamaForCausalLM

    m = LlamaForCausalLM.__new__(LlamaForCausalLM)
    nn.Module.__init__(m)
    m.config = LlamaConfig(vocab_size=32, hidden_size=16, intermediate_size=32, num_hidden_layers=1,
                           num_attention_heads=2, eos_token_id=2)
    m._device, m.max_seq, m.max_batch, m._draws = torch.device("cpu"), 64, 1, 0
    m._llm = None
    return m


@pytest.mark.parametrize("kw,exc,words", [
    (dict(penalty_alpha=0.6), ValueError, "top_k"),
    (dict(penalty_alpha=0.6, top_k=9), ValueError, "top_k"),
    (dict(penalty_alpha=float("inf"), top_k=4), ValueError, "penalty_alpha"),
    (dict(penalty_alpha=0.6, top_k=4, attention_mask=torch.tensor([[0, 1, 1]])), NotImplementedError, "attention_mask"),
    (dict(penalty_alpha=0.6, top_k=4, eos_token_id=[2, 3]), NotImplementedError, "eos_token_id"),
    (dict(penalty_alpha=0.6, top_k=4, num_return_sequences=2), NotImplementedError, "num_return_sequences"),
])
def test_generate_refuses_before_device_work(kw, exc, words):
    m = _stub_model()
    with pytest.raises(exc, match=words):
        m.generate(torch.tensor([[1, 5, 7]]), max_new_tokens=4, **kw)


def test_generation_config_penalty_alpha_is_read_and_overridden():
    from transformers import GenerationConfig

    m = _stub_model()
    cfg = GenerationConfig(penalty_alpha=0.6, top_k=12)
    with pytest.raises(ValueError, match="top_k"):            # the config's top_k (12) selects contrastive search
        m.generate(torch.tensor([[1, 5, 7]]), max_new_tokens=4, generation_config=cfg)
    with pytest.raises(ValueError, match="top_k"):            # a keyword overrides the config's penalty_alpha too
        m.generate(torch.tensor([[1, 5, 7]]), max_new_tokens=4, penalty_alpha=0.6, top_k=9)
