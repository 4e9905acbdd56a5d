"""generate(output_scores, return_dict_in_generate) and compute_transition_scores without a GPU: the restatement of
greedy and sampling `scores` (tests/scores_ref.py) against the installed transformers on a tiny random model and on
hand-worked rows, compute_transition_scores against the installed implementation, the keyword table on a stub model,
and the C ABI surface of seedb200_llama_generate_ex / seedb200_sample_scores."""
import ctypes as C
import os
import re
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import scores_ref as SR  # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEG = float("-inf")


# ---- the restatement on hand-worked rows -------------------------------------------------------------------------
def test_greedy_row_is_the_processed_logits():
    x = torch.tensor([1.0, 3.0, -2.0, 0.5, 2.0], dtype=torch.float16)
    got, _ = SR.score_row(x, [4, 1, 1], 2, 2, dict(repetition_penalty=2.0, min_new_tokens=2), do_sample=False)
    # tokens 4 and 1 are in the history: 2.0 / 2 and 3.0 / 2; eos 2 is banned (one new token < 2)
    assert got.tolist() == [1.0, 1.5, NEG, 0.5, 1.0]


def test_sample_row_tempers_the_kept_tokens_and_masks_the_rest():
    x = torch.tensor([2.0, 1.0, 0.0, -1.0, 3.0], dtype=torch.float16)
    got, _ = SR.score_row(x, [], 0, -1, dict(top_k=3), do_sample=True, temperature=0.5)
    assert got.tolist() == [4.0, 2.0, NEG, NEG, 6.0]
    got, _ = SR.score_row(x, [], 0, -1, {}, do_sample=True, temperature=1.0, top_p=0.5)
    # p ~ [.24, .09, .03, .01, .64]: the 0.64 token alone reaches 0.5
    assert got.tolist() == [NEG, NEG, NEG, NEG, 3.0]
    got, _ = SR.score_row(x, [], 0, -1, {}, do_sample=True, temperature=1.0, top_p=0.8)
    assert got.tolist() == [2.0, NEG, NEG, NEG, 3.0]


def test_sample_row_keeps_ties_with_the_least_kept_token():
    x = torch.tensor([1.0, 1.0, 1.0, 0.0], dtype=torch.float16)
    got, _ = SR.score_row(x, [], 0, -1, dict(top_k=1), do_sample=True)
    assert got.tolist() == [1.0, 1.0, 1.0, NEG]


# ---- against the installed transformers ----------------------------------------------------------------------------
def _tiny_hf(vocab=97):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(0)
    cfg = LlamaConfig(vocab_size=vocab, hidden_size=32, intermediate_size=64, num_hidden_layers=2,
                      num_attention_heads=4, num_key_value_heads=4, max_position_embeddings=128,
                      pad_token_id=0, bos_token_id=1, eos_token_id=2)
    m = LlamaForCausalLM(cfg).eval()
    with torch.no_grad():
        m.lm_head.weight.mul_(20.0)                 # logits spread over several units, so TopP has a boundary
    return m


def _step_logits(m):
    def f(ids):
        with torch.no_grad():
            return m(input_ids=ids).logits[:, -1]
    return f


CASES = [  # (do_sample, keywords)
    (False, {}),
    (False, dict(repetition_penalty=1.5, no_repeat_ngram_size=2)),
    (True, dict(temperature=1.0, top_p=1.0, top_k=0)),
    (True, dict(temperature=0.5, top_p=0.7, top_k=0)),
    (True, dict(temperature=1.0, top_p=0.9, top_k=10, repetition_penalty=1.3)),
    (True, dict(temperature=2.0, top_p=1.0, top_k=5)),
]


@pytest.mark.parametrize("do_sample,kw", CASES)
def test_restatement_equals_installed_generate(do_sample, kw):
    """transformers' scores of greedy_search / sample (5.5 keeps 4.30.2's) against the restatement on the logits of
    the same model; T is a power of two so that x / T and x * (1 / T) agree"""
    m = _tiny_hf()
    ids = torch.tensor([[1, 5, 9, 13, 5, 9], [1, 40, 41, 42, 43, 44]])
    torch.manual_seed(3)
    out = m.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=8, do_sample=do_sample,
                     output_scores=True, return_dict_in_generate=True, eos_token_id=None, pad_token_id=0, **kw)
    ctl = {k: v for k, v in kw.items() if k in ("top_k", "repetition_penalty", "no_repeat_ngram_size")}
    ref, margin = SR.teacher_forced(_step_logits(m), out.sequences, ids.shape[1], ctl, do_sample,
                                    kw.get("temperature", 1.0), kw.get("top_p", 1.0))
    assert len(out.scores) == len(ref) == out.sequences.shape[1] - ids.shape[1]
    if margin <= 1e-5:
        pytest.skip(f"a TopP boundary within {margin:.1e}: not comparable")
    for t, (a, b) in enumerate(zip(out.scores, ref)):
        assert torch.equal(torch.isinf(a), torch.isinf(b)), t
        fin = torch.isfinite(b)
        assert torch.allclose(a[fin], b[fin], rtol=1e-5, atol=1e-5), t


def test_scores_stop_with_the_last_row():
    """with an eos id, transformers stops once every row has finished: len(scores) is the generated width"""
    m = _tiny_hf()
    ids = torch.tensor([[1, 5, 9, 13]])
    free = m.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=10, do_sample=False,
                      eos_token_id=None, pad_token_id=0)
    eos = int(free[0, 6])
    out = m.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=10, do_sample=False, eos_token_id=eos,
                     pad_token_id=0, output_scores=True, return_dict_in_generate=True)
    assert out.sequences.shape[1] - 4 == len(out.scores) <= 3


# ---- compute_transition_scores --------------------------------------------------------------------------------------
def test_compute_transition_scores_equals_installed():
    from transformers.generation.utils import GenerationMixin

    m = _stub_model(vocab=6)
    g = torch.Generator().manual_seed(1)
    scores = tuple(torch.randn(4, 6, generator=g).half() for _ in range(3))
    seq = torch.randint(0, 6, (2, 5), generator=g)
    bi = torch.tensor([[0, 2, 3], [1, 1, -1]])                 # the second hypothesis is one step shorter
    for kw in (dict(), dict(normalize_logits=True)):
        for beams in (None, bi):
            sc = scores if beams is not None else tuple(s[:2] for s in scores)
            got = m.compute_transition_scores(seq, sc, beam_indices=beams, **kw)
            exp = GenerationMixin.compute_transition_scores(m, seq, sc, beam_indices=beams, **kw)
            assert torch.equal(got, exp)
    got = m.compute_transition_scores(seq, scores, beam_indices=bi)
    # hand-gathered: step t of hypothesis h reads scores[t][bi[h, t], seq[h, 2 + t]]; -1 is scored 0
    assert got[0].tolist() == [float(scores[t][bi[0, t], seq[0, 2 + t]]) for t in range(3)]
    assert got[1, 2] == 0 and got[1, 0] == scores[0][1, seq[1, 2]]


def test_peft_forwards_compute_transition_scores():
    from seed_b200.peft import PeftModel

    pm = PeftModel(_stub_model(vocab=6), {})
    scores = (torch.zeros(1, 6).half(),)
    seq = torch.tensor([[1, 2, 3]])
    assert torch.equal(pm.compute_transition_scores(seq, scores), torch.zeros(1, 1, dtype=torch.float16))


# ---- keyword table on a stub model --------------------------------------------------------------------------------
class Handle:
    """stands in for the device handle: generated tokens are zeros, scores rows are filled with the step index"""

    vocab = 6

    def __init__(self):
        self.calls = []

    @staticmethod
    def _fill(scores, new):
        if scores is not None:
            for t in range(new):
                scores[t] = t

    def generate(self, ids, new, **kw):
        self.calls.append(("sample", kw.get("scores") is not None))
        self._fill(kw.get("scores"), new)
        return torch.zeros((ids.shape[0] * kw["num_return_sequences"], new), dtype=torch.int64)

    def beam_generate(self, ids, new, k, **kw):
        """with scores: the searches ended one step before the last process() call, as when every search is done
        after an eos candidate at the last step"""
        G = ids.shape[0] * kw["num_return_sequences"]
        self.calls.append(("beam", kw.get("scores") is not None))
        if kw.get("scores") is None:
            return torch.zeros((G, new), dtype=torch.int64), torch.ones(G)
        self._fill(kw["scores"], new)
        kw["beam_indices"].fill_(-1)
        kw["beam_indices"][:, :new] = 0
        return torch.zeros((G, new - 1), dtype=torch.int64), torch.ones(G), new

    def contrastive_generate(self, ids, new, k, alpha, **kw):
        self.calls.append(("contrastive", kw.get("scores") is not None))
        self._fill(kw.get("scores"), new)
        return torch.zeros((ids.shape[0], new), dtype=torch.int64)

    def reserve_rows(self, rows):
        pass


def _stub_model(vocab=32):
    import torch.nn as nn
    from transformers.models.llama.configuration_llama import LlamaConfig

    from seed_b200.llama import LlamaForCausalLM

    m = LlamaForCausalLM.__new__(LlamaForCausalLM)
    nn.Module.__init__(m)
    m.config = LlamaConfig(vocab_size=vocab, hidden_size=16, intermediate_size=32, num_hidden_layers=1,
                           num_attention_heads=2, eos_token_id=-1)
    m._device, m.max_seq, m.max_batch, m._draws = torch.device("cpu"), 64, 8, 0
    m._llm = Handle()
    m._llm.vocab = vocab
    return m


def _gen(m, **kw):
    return m.generate(torch.tensor([[4, 5, 6]]), max_new_tokens=3, **kw)


@pytest.mark.parametrize("kw,kind,scored", [
    (dict(), torch.Tensor, False),
    (dict(return_dict_in_generate=False, output_scores=True), torch.Tensor, False),
    (dict(output_scores=True), torch.Tensor, False),
    (dict(return_dict_in_generate=True), "GenerateDecoderOnlyOutput", False),
    (dict(return_dict_in_generate=True, output_scores=True), "GenerateDecoderOnlyOutput", True),
    (dict(return_dict_in_generate=True, output_scores=True, do_sample=True, num_return_sequences=2),
     "GenerateDecoderOnlyOutput", True),
    (dict(return_dict_in_generate=True, num_beams=2), "GenerateBeamDecoderOnlyOutput", False),
    (dict(return_dict_in_generate=True, output_scores=True, num_beams=2), "GenerateBeamDecoderOnlyOutput", True),
    (dict(return_dict_in_generate=True, output_scores=True, num_beams=2, do_sample=True, num_return_sequences=2),
     "GenerateBeamDecoderOnlyOutput", True),
    (dict(num_beams=2, output_scores=True), torch.Tensor, False),
    (dict(return_dict_in_generate=True, penalty_alpha=0.5, top_k=2), "GenerateDecoderOnlyOutput", False),
    (dict(return_dict_in_generate=True, output_scores=True, penalty_alpha=0.5, top_k=2), "GenerateDecoderOnlyOutput",
     True),
    (dict(num_beams=2), torch.Tensor, False),
    (dict(penalty_alpha=0.5, top_k=2, output_scores=True), torch.Tensor, False),
])
def test_keyword_table(kw, kind, scored):
    m = _stub_model(vocab=6)
    out = _gen(m, **kw)
    if kind is torch.Tensor:
        assert isinstance(out, torch.Tensor)
        assert all(not s for _, s in m._llm.calls)              # nothing extra computed
        return
    assert type(out).__name__ == kind
    beams = kind == "GenerateBeamDecoderOnlyOutput"
    assert isinstance(out.sequences, torch.Tensor) and out.sequences.shape[1] == (5 if beams and scored else 6)
    assert out.attentions is None and out.hidden_states is None and out.past_key_values is None
    if beams and not scored:
        assert out.sequences_scores is None and out.beam_indices is None
    if not scored:
        assert out.scores is None and all(not s for _, s in m._llm.calls)
        return
    rows = out.sequences.shape[0] * (kw.get("num_beams", 1))
    if beams:         # len(scores) is the device's process() count, here one more than the generated width
        assert out.sequences_scores.shape == (out.sequences.shape[0],)
        assert out.beam_indices.shape == out.sequences.shape and out.beam_indices[:, 3:].eq(-1).all()
    assert len(out.scores) == 3
    for t, s in enumerate(out.scores):
        assert s.shape == (rows, 6) and s.dtype == torch.float16 and bool((s == t).all())


def test_generation_config_fields_and_keyword_override():
    from transformers import GenerationConfig

    m = _stub_model(vocab=6)
    cfg = GenerationConfig(output_scores=True, return_dict_in_generate=True)
    out = _gen(m, generation_config=cfg)
    assert len(out.scores) == 3
    assert _gen(m, generation_config=cfg, output_scores=False).scores is None
    assert isinstance(_gen(m, generation_config=cfg, return_dict_in_generate=False), torch.Tensor)


@pytest.mark.parametrize("name", ["output_attentions", "output_hidden_states"])
def test_attentions_and_hidden_states_are_refused_with_return_dict(name):
    m = _stub_model(vocab=6)
    with pytest.raises(NotImplementedError, match=name):
        _gen(m, return_dict_in_generate=True, **{name: True})
    assert m._llm.calls == []
    assert isinstance(_gen(m, **{name: True}), torch.Tensor)          # ignored without return_dict_in_generate




# ---- C ABI --------------------------------------------------------------------------------------------------------
def test_header_declares_the_new_entry_points():
    from seed_b200 import lib as L

    h = open(os.path.join(REPO, "include", "seedb200.h")).read()
    for name in ("seedb200_llama_generate_ex", "seedb200_sample_scores", "seedb200_llama_contrastive_generate_ex",
                 "seedb200_llama_beam_generate_ex"):
        assert re.search(r"\bint " + name + r"\(", h) and name in L.EXPORTS
    body = re.search(r"typedef struct seedb200_gen_outputs \{(.*?)\} seedb200_gen_outputs;", h, re.S).group(1)
    fields = re.findall(r"(\w+);", body)
    assert fields == [f for f, _ in L.GenOutputs._fields_]


@pytest.fixture(scope="module")
def clib():
    from seed_b200 import lib as L

    if not os.path.exists(L.LIB_PATH):
        pytest.skip("libseedb200.so not built")
    try:
        return L.load()
    except OSError as e:            # the CUDA runtime may be absent
        pytest.skip(f"library does not load here: {e}")


@pytest.mark.parametrize("scores,pitch,beam,words", [(None, 1056, None, b"16-byte"), (24, 1056, None, b"16-byte"),
                                                     (32, 1052, None, b"multiple of 8"), (32, 0, None, b"multiple"),
                                                     (32, 1056, 64, b"beam_indices")])
def test_generate_ex_refuses_bad_outputs_before_device_work(clib, scores, pitch, beam, words):
    from seed_b200 import lib as L

    fake = C.c_void_p(16)                     # never dereferenced: the outputs are refused first
    sp = L.SampleParams(1, 1.0, 1.0, 0, 0)
    o = L.GenOutputs(scores, pitch, beam, 0)
    assert clib.seedb200_llama_generate_ex(fake, fake, 1, 4, 2, 1, C.byref(sp), -1, 0, 0, fake, None, None, None,
                                           C.byref(o)) == 1
    assert words in clib.seedb200_last_error()
    cp = L.ContrastiveParams(4, 0.6)
    assert clib.seedb200_llama_contrastive_generate_ex(fake, fake, 1, 4, 2, C.byref(cp), -1, 0, 0, fake, None, None,
                                                       None, C.byref(o)) == 1
    assert words in clib.seedb200_last_error()
    if beam is None:              # the beam entry point takes beam_indices; the scores checks are the same
        bp = L.beam_params(2, do_sample=False)
        assert clib.seedb200_llama_beam_generate_ex(fake, fake, 1, 4, 2, 1, C.byref(bp), -1, 0, 0, fake, None, None,
                                                    None, None, C.byref(o)) == 1
        assert words in clib.seedb200_last_error()


@pytest.mark.parametrize("off,ld,words", [(0, 1000, b"pitch"), (0, 4004, b"pitch"), (2, 4008, b"aligned")])
def test_sample_scores_refuses_bad_pitch_and_base(clib, off, ld, words):
    from seed_b200 import lib as L

    sp = L.SampleParams(0, 1.0, 1.0, 0, 0)
    base = 4096 + off                         # never dereferenced: the arguments are refused first
    assert clib.seedb200_sample_scores(base, 4000, 2, 4000, C.byref(sp), 0, base, None, None, None, 0, 0, 0, -1,
                                       base, ld) == 1
    assert words in clib.seedb200_last_error()


# ---- beams: the restatement on hand-worked logit streams ----------------------------------------------------------
def _const_logits(row):
    """every beam row sees the same logits at every step"""
    row = torch.tensor(row, dtype=torch.float16)

    def step(ids, beam_idx):
        return row.expand(ids.shape[0], -1).clone()
    return step


def test_beam_eos_hypothesis_has_its_extra_index_and_scores_outlast_the_width():
    # eos (4) is the most probable token at every step: step 0 closes hypothesis [prompt] from row 0, step 1 closes a
    # second one and, with early_stopping=True and k = 2, every search is done.  The best is the first (score
    # lp(eos) / 1 against (lp(1) + lp(eos)) / 2), so sequences = prompt + eos: one generated column, two scores
    # entries, and beam_indices [row 0, -1].
    step = _const_logits([0.0, 2.0, 1.0, 0.0, 4.0])
    seq, scores, seq_scores, bi, _, _ = SR.beam_generate(step, torch.tensor([[1]]), 5, 2, {}, early_stopping=True,
                                                         eos=4, pad=0)
    assert seq.tolist() == [[1, 4]]
    assert len(scores) == 2 > seq.shape[1] - 1
    assert bi.tolist() == [[0, -1]]
    assert torch.equal(scores[0][0], scores[0][1])                          # step 0: the k rows are identical
    lp = torch.log_softmax(torch.tensor([0.0, 2.0, 1.0, 0.0, 4.0]), -1).half()
    assert torch.equal(scores[0][0], lp) and float(seq_scores[0]) == float(lp[4])


def test_beam_indices_follow_the_parent_rows():
    # no eos: two beams run to max_new_tokens; token t of the best hypothesis came from the row its parent held
    step = _const_logits([0.0, 3.0, 2.5, 0.0, 0.0])
    seq, scores, seq_scores, bi, _, _ = SR.beam_generate(step, torch.tensor([[1, 2]]), 3, 2, {})
    assert len(scores) == 3 and seq.shape[1] == 5
    assert bi[0, :3].tolist()[0] == 0 and bi[0, 3:].tolist() == [-1, -1]
    assert all(0 <= int(x) < 2 for x in bi[0, :3])
    from transformers.generation.utils import GenerationMixin

    m = _stub_model(vocab=5)
    ts = GenerationMixin.compute_transition_scores(m, seq, tuple(s.float() for s in scores), beam_indices=bi)
    # HF's identity: the transition scores sum to the hypothesis' score times its length ** length_penalty
    assert abs(float(ts.sum()) / 5 - float(seq_scores[0])) < 1e-5


def test_beam_sampling_scores_are_warped_without_the_beam_score():
    # at step 1 both beams hold identical rows but different beam scores: the scores rows must still be equal, and
    # equal to the warp of the processed row alone
    row = [0.0, 3.0, 2.5, 1.0, -1.0, 0.5]
    step = _const_logits(row)
    _, scores, _, _, _, _ = SR.beam_generate(step, torch.tensor([[1]]), 2, 2, {"top_k": 3}, do_sample=True,
                                             temperature=0.5, top_p=0.9, seed=1)
    lp = torch.log_softmax(torch.tensor(row), -1).half()
    want, _ = SR.beam_warp_row(lp, 0.5, 3, 0.9)
    for t in range(2):
        assert torch.equal(scores[t][0], want) and torch.equal(scores[t][1], want)
    assert int(torch.isfinite(want).sum()) >= 2                             # min_tokens_to_keep = 2


@pytest.mark.parametrize("T,top_k,top_p", [(1.0, 0, 1.0), (0.5, 0, 0.6), (2.0, 5, 1.0), (1.0, 1, 0.01),
                                           (0.5, 20, 0.8)])
def test_beam_warp_equals_installed_warpers(T, top_k, top_p):
    """beam_sample's warpers are Temperature, TopK and TopP with min_tokens_to_keep = 2 (4.30.2 _get_logits_warper
    for num_beams > 1); the installed classes are the same algorithm.  fp32 rows without ties, T a power of two."""
    from transformers import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper

    g = torch.Generator().manual_seed(int(T * 10 + top_k + top_p * 100))
    for _ in range(5):
        lp = torch.log_softmax(torch.randn(64, generator=g) * 3, -1)
        got, margin = SR.beam_warp_row(lp, T, top_k, top_p)
        x = lp[None].clone()
        if T != 1.0:
            x = TemperatureLogitsWarper(T)(None, x)
        if top_k > 0:
            x = TopKLogitsWarper(top_k, min_tokens_to_keep=2)(None, x)
        if top_p < 1.0:
            x = TopPLogitsWarper(top_p, min_tokens_to_keep=2)(None, x)
        if margin <= 1e-6:
            continue
        assert torch.equal(torch.isinf(got), torch.isinf(x[0]))
        fin = torch.isfinite(got)
        assert torch.allclose(got[fin], x[0][fin])
