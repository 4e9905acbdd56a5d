"""generate(num_return_sequences=n) without a GPU: which mode each call runs and what it refuses, the row order against
the installed transformers, the beam-sample rule (tests/return_sequences_ref.py) on a hand-worked logit stream, and
the C ABI surface of seedb200_llama_generate_n / seedb200_llama_beam_generate_n."""
import ctypes as C
import os
import re
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_ref as BR  # noqa: E402
import return_sequences_ref as RS  # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("seedb200_llama_generate_n", "seedb200_llama_generate_n_processed", "seedb200_llama_beam_generate_n",
       "seedb200_llama_beam_generate_n_processed")


class Loop(Exception):
    """raised by the stub's forward(): the call took the per-token Python loop"""


class Handle:
    """stands in for the device handle and records which entry point a generate() call reached"""

    def __init__(self):
        self.calls = []

    def generate(self, ids, new, **kw):
        self.calls.append(("sample", ids.shape[0], kw["num_return_sequences"]))
        return torch.zeros((ids.shape[0] * kw["num_return_sequences"], new), dtype=torch.int64)

    def beam_generate(self, ids, new, k, **kw):
        self.calls.append(("beam", ids.shape[0], kw["num_return_sequences"]))
        G = ids.shape[0] * kw["num_return_sequences"]
        return torch.zeros((G, new), dtype=torch.int64), torch.zeros(G)

    def contrastive_generate(self, ids, new, k, alpha, **kw):
        self.calls.append(("contrastive", ids.shape[0], 1))
        return torch.zeros((ids.shape[0], new), dtype=torch.int64)

    def reserve_rows(self, rows):
        self.calls.append(("reserve", rows))


def _stub_model():
    """a LlamaForCausalLM whose handle only records calls (max_batch 1)"""
    import torch.nn as nn
    from transformers.models.llama.configuration_llama import LlamaConfig

    from seed_b200.llama import LlamaForCausalLM

    m = LlamaForCausalLM.__new__(LlamaForCausalLM)
    nn.Module.__init__(m)
    m.config = LlamaConfig(vocab_size=32, hidden_size=16, intermediate_size=32, num_hidden_layers=1,
                           num_attention_heads=2, eos_token_id=2)
    m._device, m.max_seq, m.max_batch, m._draws = torch.device("cpu"), 64, 1, 0
    m._llm = Handle()

    def forward(input_ids=None, **_):
        raise Loop(tuple(input_ids.shape))
    m.forward = forward
    return m


def _ids(B):
    return torch.arange(3 * B).view(B, 3) + 4


PAD_MASK = torch.tensor([[0, 1, 1]])
MODES = [  # (B, keywords, what runs: entry point, prompts, n, rows reserved) or (exception, words)
    (1, dict(do_sample=True), ("sample", 1, 1, None)),
    (1, dict(do_sample=True, num_return_sequences=1), ("sample", 1, 1, None)),
    (1, dict(do_sample=True, num_return_sequences=3), ("sample", 1, 3, 3)),
    (2, dict(do_sample=True, num_return_sequences=4), ("sample", 2, 4, 8)),
    (2, dict(do_sample=True, num_return_sequences=4, top_k=5, repetition_penalty=1.2), ("sample", 2, 4, 8)),
    (1, dict(do_sample=True, penalty_alpha=0.6, top_k=4, num_return_sequences=2), ("sample", 1, 2, 2)),
    (1, dict(num_beams=4, do_sample=True, num_return_sequences=2), ("beam", 1, 2, 8)),
    (2, dict(num_beams=2, do_sample=True, num_return_sequences=3), ("beam", 2, 3, 12)),
    (1, dict(num_beams=4, do_sample=True, penalty_alpha=0.6, top_k=4, num_return_sequences=3), ("beam", 1, 3, 12)),
    (1, dict(num_beams=4), ("beam", 1, 1, 4)),
    (1, dict(penalty_alpha=0.6, top_k=4), ("contrastive", 1, 1, 4)),
    (1, dict(), ("sample", 1, 1, None)),
    (6, dict(do_sample=True, device_loop=True), ("sample", 6, 1, 6)),
    (1, dict(num_return_sequences=2), (NotImplementedError, "num_return_sequences")),
    (1, dict(num_beams=4, num_return_sequences=2), (NotImplementedError, "num_return_sequences")),
    (1, dict(penalty_alpha=0.6, top_k=4, num_return_sequences=2), (NotImplementedError, "num_return_sequences")),
    (1, dict(penalty_alpha=0.6, num_return_sequences=2), (NotImplementedError, "num_return_sequences")),
    (1, dict(do_sample=True, num_return_sequences=0), (ValueError, "num_return_sequences")),
    (1, dict(num_beams=4, do_sample=True, num_return_sequences=-1), (ValueError, "num_return_sequences")),
    (1, dict(do_sample=True, num_return_sequences=2, device_loop=True, attention_mask=PAD_MASK),
     (ValueError, "device_loop")),
    (1, dict(num_beams=2, do_sample=True, num_return_sequences=2, attention_mask=PAD_MASK),
     (NotImplementedError, "attention_mask")),
    (1, dict(num_beams=9, do_sample=True, num_return_sequences=2), (ValueError, "num_beams")),
]


@pytest.mark.parametrize("B,kw,want", MODES)
def test_mode_table(B, kw, want):
    m = _stub_model()
    if isinstance(want[0], type):
        with pytest.raises(want[0], match=want[1]):
            m.generate(_ids(B), max_new_tokens=4, **kw)
        assert [c for c in m._llm.calls if c[0] != "reserve"] == []       # refused before any device work
        return
    what, prompts, n, reserved = want
    out = m.generate(_ids(B), max_new_tokens=4, **kw)
    runs = [c for c in m._llm.calls if c[0] != "reserve"]
    assert runs == [(what, prompts, n)]
    assert [c[1] for c in m._llm.calls if c[0] == "reserve"] == ([reserved] if reserved else [])
    assert out.shape == (B * n, 3 + 4)
    assert torch.equal(out[:, :3], RS.expand(_ids(B), n))


@pytest.mark.parametrize("B,kw", [
    (1, dict(attention_mask=torch.tensor([[0, 1, 1]]))),
    (2, dict(attention_mask=torch.tensor([[0, 1, 1], [1, 1, 1]]))),
    (1, dict(eos_token_id=[2, 3])),
    (2, dict(device_loop=False)),
])
def test_padded_or_several_eos_expand_then_take_the_python_loop(B, kw):
    m = _stub_model()
    with pytest.raises(Loop) as e:
        m.generate(_ids(B), max_new_tokens=4, do_sample=True, num_return_sequences=3, **kw)
    assert e.value.args[0] == (3 * B, 3)                    # the expanded batch, prefilled as HF does
    assert m._llm.calls == [("reserve", 3 * B)]


def test_default_route_of_unpadded_n1_batches_is_unchanged():
    m = _stub_model()
    with pytest.raises(Loop):
        m.generate(_ids(5), max_new_tokens=4, do_sample=True)
    assert m._llm.calls == []


def test_generation_config_num_return_sequences_is_read_and_overridden():
    from transformers import GenerationConfig

    cfg = GenerationConfig(do_sample=True, num_return_sequences=3)
    m = _stub_model()
    assert m.generate(_ids(2), max_new_tokens=4, generation_config=cfg).shape == (6, 7)
    assert m._llm.calls[-1] == ("sample", 2, 3)
    assert m.generate(_ids(2), max_new_tokens=4, generation_config=cfg, num_return_sequences=2).shape == (4, 7)
    assert m._llm.calls[-1] == ("sample", 2, 2)
    cfg = GenerationConfig(num_beams=4, do_sample=True, num_return_sequences=3)
    assert m.generate(_ids(1), max_new_tokens=4, generation_config=cfg).shape == (3, 7)
    assert m._llm.calls[-1] == ("beam", 1, 3)
    with pytest.raises(NotImplementedError, match="num_return_sequences"):
        m.generate(_ids(1), max_new_tokens=4, generation_config=cfg, do_sample=False)


@pytest.mark.parametrize("B,n", [(1, 3), (2, 2), (3, 4)])
def test_row_order_matches_installed_transformers(B, n):
    """top_k=1 makes sampling deterministic: row b * n + j must be prompt b's greedy continuation"""
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(5 * B + n)
    cfg = LlamaConfig(vocab_size=97, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                      num_attention_heads=4, num_key_value_heads=4, max_position_embeddings=128)
    model = LlamaForCausalLM(cfg).eval()
    ids = torch.randint(3, 97, (B, 5))
    kw = dict(max_new_tokens=6, eos_token_id=None, pad_token_id=0)
    with torch.no_grad():
        hf = model.generate(ids, do_sample=True, top_k=1, num_return_sequences=n, **kw)
        ref = model.generate(RS.expand(ids, n), do_sample=False, **kw)
        per_prompt = model.generate(ids, do_sample=False, **kw)
    assert torch.equal(hf, ref)
    assert [RS.prompt_of(r, n) for r in range(B * n)] == [r // n for r in range(B * n)]
    for r in range(B * n):
        assert torch.equal(hf[r], per_prompt[RS.prompt_of(r, n)])
    if B > 1:
        assert not torch.equal(per_prompt[0], per_prompt[1])       # the prompts are told apart


def _uniform(V, k):
    """step_logits with one logit for every token of every row (and a record of the rows it was called with)"""
    seen = []

    def step(ids, beam_idx):
        seen.append(ids.clone())
        return torch.zeros((ids.shape[0], V))
    return step, seen


def test_beam_sample_group_reads_philox_sequence_g():
    # k = 2, V = 8, uniform logits, one new token.  Beams 1..k-1 start at -1e9, so the 2k draws are the four beam-0
    # tokens with the largest Gumbel keys; with equal w the keys order as the uniforms u.  Equal w sorts the draws by
    # token, so the two running beams are the two smallest of those four ids, with equal scores, and finalize keeps
    # the later-added one (the last of a stable ascending sort): the second-smallest id among the top four u of
    # Philox sequence g.
    V, k, n, seed = 8, 2, 3, 1234
    step, _ = _uniform(V, k)
    out, scores, _, _, _ = RS.beam_sample_generate(step, torch.tensor([[5, 6, 7]]), 1, k, n, seed=seed, offset=0)
    want = []
    for g in range(n):
        u = BR.open_uniform(seed, 0, g, k * V)[:V]
        top4 = sorted(torch.argsort(u, descending=True)[:4].tolist())
        want.append(top4[1])
    assert out[:, 3].tolist() == want
    assert len(set(want)) > 1                                      # the searches are independent draws
    assert out.shape == (n, 4) and scores.shape == (n,)


def test_beam_sample_group_reads_prompt_g_over_n():
    # logits that put all the mass on (first prompt token + 1) % V: search g continues prompt g // n
    V, k, n = 16, 2, 3

    def step(ids, beam_idx):
        logits = torch.full((ids.shape[0], V), -30.0)
        logits[torch.arange(ids.shape[0]), (ids[:, 0] + 1) % V] = 30.0
        return logits
    prompt = torch.tensor([[3, 9, 9], [7, 9, 9]])
    out = RS.beam_sample_generate(step, prompt, 2, k, n, seed=1, offset=0)[0]
    assert out.shape == (2 * n, 5)
    for g in range(2 * n):
        first = int(prompt[RS.prompt_of(g, n), 0])
        assert out[g, :3].tolist() == prompt[g // n].tolist()
        assert out[g, 3:].tolist() == [(first + 1) % V] * 2


def test_return_sequences_entry_points_are_declared():
    from seed_b200 import lib as L

    hdr = open(os.path.join(REPO, "include", "seedb200.h")).read()
    for name in NEW:
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


def test_return_sequences_exports_and_argument_errors(clib):
    from seed_b200 import lib as L

    for name in NEW:
        assert hasattr(clib, name)
    fake = C.c_void_p(16)                     # never dereferenced: the arguments are refused first
    sp = L.SampleParams(1, 1.0, 1.0, 0, 0)
    for n in (0, -3):
        assert clib.seedb200_llama_generate_n(fake, fake, 1, 1, 1, n, C.byref(sp), -1, 0, 0, fake, None, None) == 1
        assert b"num_return_sequences" in clib.seedb200_last_error()
        assert clib.seedb200_llama_generate_n_processed(fake, fake, 1, 1, 1, n, C.byref(sp), -1, 0, 0, fake, None,
                                                        None, None) == 1
        assert b"num_return_sequences" in clib.seedb200_last_error()
    bp = L.beam_params(2, do_sample=False)
    assert clib.seedb200_llama_beam_generate_n(fake, fake, 1, 1, 1, 2, C.byref(bp), -1, 0, 0, fake, None, None,
                                               None) == 1
    err = clib.seedb200_last_error()
    assert b"num_return_sequences" in err and b"do_sample" in err
    assert clib.seedb200_llama_beam_generate_n_processed(fake, fake, 1, 1, 1, 0, C.byref(L.beam_params(2, True)), -1,
                                                         0, 0, fake, None, None, None, None) == 1
    assert b"num_return_sequences" in clib.seedb200_last_error()
    assert clib.seedb200_llama_generate_n(None, None, 1, 1, 1, 2, C.byref(sp), -1, 0, 0, None, None, None) == 1
    assert b"null" in clib.seedb200_last_error()
    assert clib.seedb200_llama_beam_generate_n(None, None, 1, 1, 1, 2, C.byref(L.beam_params(2, True)), -1, 0, 0,
                                               None, None, None, None) == 1
    assert b"null" in clib.seedb200_last_error()
