"""The beam-search restatement (tests/beam_ref.py) against the installed transformers and on hand-worked logit streams
that pin each transformers 4.30.2 rule, and the beam C ABI surface, without a GPU."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_ref as BR  # noqa: E402

NEG = -30.0


def stream(rows):
    """step_logits replaying fixed fp32 rows: rows[t] is [B*k, V] for step t"""
    it = iter(rows)

    def step(ids, beam_idx):
        return torch.tensor(next(it), dtype=torch.float32)
    return step


def lp_rows(*probs):
    """rows whose log_softmax is log(p) exactly enough for hand-worked scores"""
    return [[float(torch.tensor(p).log()) if p > 0 else NEG for p in row] for row in probs]


@pytest.mark.parametrize("k", [2, 4, 5])
@pytest.mark.parametrize("B", [1, 2])
def test_restatement_matches_transformers_beam_search(k, B):
    from transformers import LlamaConfig, LlamaForCausalLM

    torch.manual_seed(7 * k + B)
    cfg = LlamaConfig(vocab_size=97, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                      num_attention_heads=4, num_key_value_heads=4, max_position_embeddings=128)
    model = LlamaForCausalLM(cfg).eval()
    model.generation_config.eos_token_id = None
    model.generation_config.pad_token_id = 0
    ids = torch.randint(3, 97, (B, 6))
    new = 8
    with torch.no_grad():
        hf = model.generate(ids, num_beams=k, do_sample=False, max_new_tokens=new, eos_token_id=None, pad_token_id=0,
                            length_penalty=1.0, early_stopping=False)

        def step(seq, beam_idx):
            return model(seq).logits[:, -1].float()
        ref = BR.beam_generate(step, ids, new, k)[0]
    assert torch.equal(ref, hf), (ref.tolist(), hf.tolist())


def test_init_keeps_only_beam_0_on_the_first_step():
    # identical first rows: with beams 1..k-1 at -1e9 every first candidate comes from beam 0
    rows = [lp_rows([0.5, 0.3, 0.2, 0.0], [0.5, 0.3, 0.2, 0.0]), lp_rows([0.25] * 4, [0.25] * 4)]
    s = (BR.log_probs(torch.tensor(rows[0])) + torch.tensor([0.0, -1e9])[:, None]).view(1, 8)
    sc, ix, _, _ = BR.select(s, 2)
    assert ix[0].tolist() == [0, 1, 2, 3]
    assert sc[0, 3] < -20


def test_eos_at_rank_below_k_is_a_hypothesis_at_rank_k_is_skipped():
    # k=2, V=4, eos=3, S=3, 2 new tokens; beams 1..k-1 start at -1e9, so step 0 ranks beam 0's row only.
    S, eos, prompt = 3, 3, torch.tensor([[5, 6, 7]])
    step1 = lp_rows([0.7, 0.2, 0.05, 0.05], [0.7, 0.2, 0.05, 0.05])
    # eos at rank k-1 = 1: it is a hypothesis "prompt" with score log(.3) / 3 = -0.401; the beams are tokens 0 and 1
    # (log .45 and log .2).  At the end the running beams [.., 0, 0] score log(.45 * .7) / 5 = -0.231 and
    # [.., 1, 0] log(.2 * .7) / 5 = -0.393: the eos hypothesis (-0.401) is the worst of three and is dropped
    # (k = 2 hypotheses), so the output is [5, 6, 7, 0, 0] -- while the hypothesis list did change:
    at_k_minus_1 = [lp_rows([0.45, 0.2, 0.05, 0.3], [0.45, 0.2, 0.05, 0.3]), step1]
    out, best, _, _, st = BR.beam_generate(stream(at_k_minus_1), prompt, 2, 2, eos=eos, pad=9)
    assert st["hyps_added"] == 1
    assert out.tolist() == [[5, 6, 7, 0, 0]]
    # a stronger eos candidate at rank k-1, length_penalty 0 (raw sums):
    strong = [lp_rows([0.5, 0.01, 0.09, 0.4], [0.5, 0.01, 0.09, 0.4]), step1]
    out, best, _, _, st = BR.beam_generate(stream(strong), prompt, 2, 2, eos=eos, pad=9, length_penalty=0.0)
    # eos (log .4 = -0.916) at rank 1 < k: hypothesis [5, 6, 7]; beams 0 (log .5) and 2 (log .09); finalize adds
    # [.., 0, 0] (log .35 = -1.05) and [.., 2, 0]: the eos hypothesis wins; width min(3 + 1, 5): prompt, eos
    assert st["hyps_added"] == 1
    assert out.tolist() == [[5, 6, 7, 3]]
    assert abs(float(best[0]) - float(torch.tensor(0.4).log())) < 1e-6
    # the same eos probability at rank k = 2 (two tokens above it): skipped, never a hypothesis; the output is a
    # running beam of the full length
    at_k = [lp_rows([0.46, 0.45, 0.01, 0.08], [0.46, 0.45, 0.01, 0.08]), step1]
    out, best, _, _, st = BR.beam_generate(stream(at_k), prompt, 2, 2, eos=eos, pad=9, length_penalty=0.0)
    assert st["hyps_added"] == 0
    assert out.tolist() == [[5, 6, 7, 0, 0]]
    # rank k with a strong eos: two tokens above it, eos (log .3) would beat every running beam if it were added
    at_k_strong = [lp_rows([0.36, 0.34, 0.0, 0.3], [0.36, 0.34, 0.0, 0.3]), step1]
    out, best, _, _, st = BR.beam_generate(stream(at_k_strong), prompt, 2, 2, eos=eos, pad=9, length_penalty=0.0)
    assert st["hyps_added"] == 0
    assert out.tolist() == [[5, 6, 7, 0, 0]]      # log(.36 * .7) = -1.38 < log(.3) = -1.20: only the skip explains it


def test_length_normalisation_includes_the_prompt():
    for lp in (0.0, 1.0, 2.0):
        h = BR.Hyps(1, lp, False, 20)
        h.add([1] * 7, -2.0)
        assert h.beams[0][0] == -2.0 / 7 ** lp


def test_hypothesis_replacement_and_ties():
    h = BR.Hyps(2, 0.0, False, 20)
    h.add([1], -1.0)
    h.add([2], -3.0)
    assert h.worst == -3.0
    h.add([3], -3.0)                      # not > worst: rejected
    assert [b[1] for b in h.beams] == [[1], [2]]
    h.add([4], -2.0)                      # replaces the lowest; worst = the second lowest
    assert [b[1] for b in h.beams] == [[1], [4]] and h.worst == -2.0
    h.add([5], -1.0)                      # -2 dropped; tie at -1 between [1] and [5]: worst = -1.0
    assert [b[1] for b in h.beams] == [[1], [5]] and h.worst == -1.0
    h.add([6], -0.5)                      # the tied lowest: the earliest added ([1]) goes
    assert [b[1] for b in h.beams] == [[5], [6]]


def test_early_stopping_modes():
    for es, expect in ((True, True), (False, False), ("never", False)):
        h = BR.Hyps(2, 1.0, es, 40)
        h.add([1] * 10, -5.0)
        h.add([1] * 10, -6.0)
        # worst -0.6; best running -4.0: False -> -4/10 = -0.4 > -0.6 not done; "never" -> -4/40 = -0.1 not done
        assert h.is_done(-4.0, 10) is expect
    h = BR.Hyps(2, 1.0, False, 40)
    h.add([1] * 10, -5.0)
    assert not h.is_done(-100.0, 10)      # fewer than k hypotheses
    h.add([1] * 10, -6.0)
    assert h.is_done(-7.0, 10)            # -0.6 >= -0.7
    h = BR.Hyps(2, 1.0, "never", 40)
    h.add([1] * 10, -5.0)
    h.add([1] * 10, -6.0)
    assert not h.is_done(-7.0, 10)        # -7/40 = -0.175 > -0.6
    assert h.is_done(-30.0, 10)
    h = BR.Hyps(2, 0.0, "never", 40)      # lp <= 0: the cur_len form
    h.add([1] * 10, -5.0)
    h.add([1] * 10, -6.0)
    assert h.is_done(-7.0, 10)


def test_finalize_eos_and_pad_layout():
    # k=2, V=4, eos=3, pad=9, S=2, 3 new tokens.  Sequence 0, step 0: eos at rank 0 -> hypothesis [5, 6] with score
    # log(.7) / 2 = -0.178, which beats its running beams (log(.1 * .9 * .9) / 5 = -0.503) at finalize.  Sequence 1
    # never finishes: its best is a running beam of the full length 5.  Width = min(2 + 1, 5) for sequence 0 alone
    # (3), min(5 + 1, 5) with sequence 1: eos after the short hypothesis, then pad.
    hi, flat = [0.1, 0.1, 0.1, 0.7], [0.9, 0.04, 0.03, 0.03]
    one = BR.beam_generate(stream([lp_rows(hi, hi), lp_rows(flat, flat), lp_rows(flat, flat)]),
                           torch.tensor([[5, 6]]), 3, 2, eos=3, pad=9)[0]
    assert one.tolist() == [[5, 6, 3]]
    two = BR.beam_generate(stream([lp_rows(hi, hi, flat, flat)] + [lp_rows(flat, flat, flat, flat)] * 2),
                           torch.tensor([[5, 6], [7, 8]]), 3, 2, eos=3, pad=9)[0]
    assert two.tolist() == [[5, 6, 3, 9, 9], [7, 8, 0, 0, 0]]


def test_beam_sample_scores_accumulate_temperature_scaled_sums():
    k, V, T = 2, 3, 0.5
    logits = torch.tensor(lp_rows([0.5, 0.3, 0.2], [0.5, 0.3, 0.2]))
    bs = torch.tensor([0.0, -1e9])
    s = (BR.log_probs(logits) + bs[:, None]).view(1, k * V)
    sc, ix, _, _ = BR.select(s, k, do_sample=True, temperature=T, top_p=1.0, seed=1)
    for r in range(2 * k):
        assert float(sc[0, r]) == float(s[0, int(ix[0, r])] / T)
    assert all(float(sc[0, r]) >= float(sc[0, r + 1]) for r in range(2 * k - 1))


def test_open_uniform_is_strictly_inside_the_unit_interval():
    u = BR.open_uniform(3, 5, 1, 100000)
    assert float(u.min()) > 0.0 and float(u.max()) < 1.0
    assert bool((torch.log(-torch.log(u))).isfinite().all())


@pytest.fixture(scope="module")
def clib():
    from seed_b200 import lib as L

    if not os.path.exists(L.LIB_PATH):
        pytest.skip("libseedb200.so not built")
    try:
        return L.load()
    except OSError as e:            # the CUDA runtime may be absent
        pytest.skip(f"library does not load here: {e}")


def test_beam_exports_and_argument_errors(clib):
    from seed_b200 import lib as L

    for name in ("seedb200_beam_select", "seedb200_llama_beam_generate", "seedb200_llama_reserve_rows",
                 "seedb200_decode_attention_lineage"):
        assert name in L.EXPORTS and hasattr(clib, name)
    bp = L.beam_params(9)
    sc = C.c_void_p(16)
    st = clib.seedb200_beam_select(C.c_void_p(16), 8, 8, 1, 8, C.c_void_p(16), C.byref(bp), 0, sc, sc, None)
    assert st != 0 and b"k" in clib.seedb200_last_error()
    assert clib.seedb200_llama_beam_generate(None, None, 1, 1, 1, C.byref(bp), -1, 0, 0, None, None, None, None) != 0
    assert b"null" in clib.seedb200_last_error()
    assert clib.seedb200_llama_reserve_rows(None, 4) != 0
    assert clib.seedb200_decode_attention_lineage(None, None, None, None, None, 1, 1, 128, 1, 1, 1.0, None, None) != 0
    with pytest.raises(ValueError):
        L.beam_params(2, early_stopping="sometimes")
