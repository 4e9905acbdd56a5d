"""generate(num_return_sequences=n) on the device (seedb200_llama_generate_n / seedb200_llama_beam_generate_n).

Every comparison is bit-exact on tokens:
  - against a composed oracle: the B prompts prefilled with forward(), each prompt's K/V copied into its n rows through
    seedb200_llama_kv_load, then forward() + L.sample per token over the B * n rows with the same seed and offset;
  - against the expanded call: the same generate() on input_ids.repeat_interleave(n, 0) with n = 1;
  - for beam sampling, against tests/return_sequences_ref.py driven as in test_beam_gpu (tokens where the
    restatement's Gumbel-key and nucleus margins allow a comparison; scores within one fp16 rounding).
"""
import os
import sys

import pytest
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

from oracle import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import return_sequences_ref as RS  # noqa: E402

pytestmark = pytest.mark.gpu
KEY_EPS = 1e-5
SCORE_TOL = 4e-3
HID, LAYERS, HEADS, FFN, VOCAB = 512, 2, 4, 1408, 1056
C7 = dict(top_k=40, repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=3)
SAMP = dict(do_sample=True, temperature=0.9, top_p=0.8)


def make(max_batch=24, max_seq=160, seed=9, **kw):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=VOCAB, hidden_size=HID, intermediate_size=FFN, num_hidden_layers=LAYERS,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=2048)
    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=seed)
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=max_batch, max_seq=max_seq, **kw)


def prompt(B, S=24, seed=10):
    return synth.prompt_ids(B, S, n_image_spans=1, text_vocab=VOCAB - 66, n_codes=64, seed=seed).cuda()


@pytest.fixture(scope="module")
def model():
    return make()


def gen(m, ids, **kw):
    m._draws = 0
    return m.generate(input_ids=ids, seed=kw.pop("seed", 5), **kw)


def composed(m, ids, n, new, seed=5, eos=-1, pad=0, ctl=None, samp=SAMP):
    """the oracle of the module docstring; returns [B * n, S + steps] like generate()"""
    from seed_b200 import lib as L

    ctl = ctl or {}
    B, S = ids.shape
    new = min(new, m.max_seq - S)
    out = m(input_ids=ids, use_cache=True, last_logits_only=True)
    past = [(k.repeat_interleave(n, 0).contiguous(), v.repeat_interleave(n, 0).contiguous())
            for k, v in out.past_key_values]
    logits = out.logits[:, -1].repeat_interleave(n, 0).contiguous()
    seq = RS.expand(ids, n)
    unfinished = torch.ones(B * n, dtype=torch.bool, device="cuda")
    for step in range(new):
        nxt = L.sample(logits, seed=seed, offset=0, step=step, history=seq, prompt_len=S, eos_token_id=eos,
                       **samp, **ctl)
        nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad))
        seq = torch.cat([seq, nxt[:, None]], dim=1)
        if eos >= 0:
            unfinished &= nxt != eos
            if not bool(unfinished.any()):
                break
        if step == new - 1:
            break
        o = m(input_ids=seq[:, -1:], past_key_values=past, use_cache=True, last_logits_only=True)
        past, logits = o.past_key_values, o.logits[:, -1].contiguous()
    return seq


@pytest.mark.parametrize("controls", [False, True])
@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("B", [1, 2])
def test_sampling_equals_composed_oracle(model, B, n, controls):
    ids, ctl = prompt(B), (C7 if controls else {})
    got = gen(model, ids, max_new_tokens=20, num_return_sequences=n, eos_token_id=-1, **SAMP, **ctl)
    ref = composed(model, ids, n, 20, ctl=ctl)
    assert got.shape == (B * n, 24 + 20)
    assert torch.equal(got, ref), (got[:, 24:].tolist(), ref[:, 24:].tolist())
    assert len({tuple(r) for r in got[:, 24:].tolist()}) > 1          # the rows sample on their own


@pytest.mark.parametrize("controls", [False, True])
def test_sampling_eos_fires_early_in_some_rows(model, controls):
    ids, n, ctl = prompt(2), 4, (C7 if controls else {})
    free = gen(model, ids, max_new_tokens=24, num_return_sequences=n, eos_token_id=-1, **SAMP, **ctl)[:, 24:]
    eos = int(free[1, 4])                                           # a token row 1 emits: it finishes early
    got = gen(model, ids, max_new_tokens=24, num_return_sequences=n, eos_token_id=eos, pad_token_id=VOCAB - 1,
              **SAMP, **ctl)
    ref = composed(model, ids, n, 24, eos=eos, pad=VOCAB - 1, ctl=ctl)
    assert torch.equal(got, ref), (got[:, 24:].tolist(), ref[:, 24:].tolist())
    tail = got[:, 24:]
    ended = [(r == eos).any().item() for r in tail]
    assert any(ended) and bool((tail == VOCAB - 1).any())


def test_sampling_truncates_at_max_seq(model):
    ids, n = prompt(2, S=150), 3
    got = gen(model, ids, max_new_tokens=30, num_return_sequences=n, eos_token_id=-1, **SAMP)
    assert got.shape == (6, model.max_seq)
    assert torch.equal(got, composed(model, ids, n, 30))


@pytest.mark.parametrize("B,n", [(1, 2), (1, 8), (2, 3), (2, 4), (3, 5)])
def test_sampling_equals_expanded_call(model, B, n):
    ids = prompt(B)
    got = gen(model, ids, max_new_tokens=20, num_return_sequences=n, eos_token_id=-1, **SAMP)
    exp = gen(model, RS.expand(ids, n), max_new_tokens=20, eos_token_id=-1, device_loop=True, **SAMP)
    assert torch.equal(got, exp), (got[:, 24:].tolist(), exp[:, 24:].tolist())


def test_prompt_is_written_once(model):
    """the rows past the B prompt rows hold a sentinel at positions [0, S) during the call, so tokens that match the
    oracle show that every row reads its prompt through the lineage table, not from its own cache row"""
    B, n, S = 2, 4, 24
    H, D = HEADS, HID // HEADS
    ids = prompt(B)
    sentinel = torch.full((B * n, H, S, D), 7.0, dtype=torch.float16, device="cuda")
    for l in range(LAYERS):
        model._llm.kv_load(l, sentinel, sentinel)
    got = gen(model, ids, max_new_tokens=8, num_return_sequences=n, eos_token_id=-1, **SAMP)
    torch.cuda.synchronize()
    for l, (k, v) in enumerate(model._kv_tuple(B * n, S)):
        assert bool((k[B:] == 7.0).all()) and bool((v[B:] == 7.0).all()), l      # rows B .. B*n-1 never prefilled
        assert not bool((k[:B] == 7.0).all())                                   # the B prompt rows were
    assert torch.equal(got, composed(model, ids, n, 8))


def test_graph_equals_eager_seeds_differ_and_n1_is_the_plain_call(model):
    ids = prompt(2)
    kw = dict(max_new_tokens=20, eos_token_id=-1, **SAMP)
    a = gen(model, ids, num_return_sequences=3, use_graph=True, **kw)
    assert model._llm.used_graph == 1
    b = gen(model, ids, num_return_sequences=3, use_graph=False, **kw)
    assert model._llm.used_graph == 0
    c = gen(model, ids, num_return_sequences=3, seed=6, **kw)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert torch.equal(gen(model, ids, num_return_sequences=1, **kw), gen(model, ids, **kw))
    assert torch.equal(gen(model, ids, num_return_sequences=1, **kw, **C7), gen(model, ids, **kw, **C7))


def test_generation_config_is_honoured(model):
    from transformers import GenerationConfig

    ids = prompt(1)
    cfg = GenerationConfig(do_sample=True, temperature=0.9, top_p=0.8, num_return_sequences=3, max_new_tokens=12)
    a = gen(model, ids, generation_config=cfg, eos_token_id=-1)
    assert torch.equal(a, gen(model, ids, num_return_sequences=3, max_new_tokens=12, eos_token_id=-1, **SAMP))
    b = gen(model, ids, generation_config=cfg, eos_token_id=-1, num_return_sequences=2)
    assert b.shape[0] == 2 and torch.equal(b, a[:2])           # rows of prompt 0 draw from Philox rows 0, 1


def test_rows_grow_and_forward_still_matches():
    m = make(max_batch=1)
    ids = prompt(1)
    before = m(input_ids=ids).logits
    got = gen(m, ids, max_new_tokens=12, num_return_sequences=6, eos_token_id=-1, **SAMP)
    assert m.max_batch == 6 and got.shape == (6, 36)
    assert torch.equal(m(input_ids=ids).logits, before)
    assert torch.equal(got, gen(make(max_batch=6), ids, max_new_tokens=12, num_return_sequences=6, eos_token_id=-1,
                                **SAMP))


@pytest.mark.parametrize("padded", [True, False])
def test_python_loop_route_equals_hand_expanded_batch(model, padded):
    ids, n = prompt(2), 3
    if padded:
        mask = torch.ones_like(ids)
        mask[1, :3] = 0
        kw, ekw = dict(attention_mask=mask), dict(attention_mask=RS.expand(mask, n))
    else:
        kw = ekw = dict(eos_token_id=[3, 4])
    got = gen(model, ids, max_new_tokens=12, num_return_sequences=n, **SAMP, **kw)
    ref = gen(model, RS.expand(ids, n), max_new_tokens=12, **SAMP, **ekw)
    assert got.shape[0] == 6 and torch.equal(got, ref)


@pytest.mark.parametrize("fmt", ["int8", "nf4"])
def test_quantised_weights_equal_expanded_call(fmt):
    kw = dict(load_in_8bit=True) if fmt == "int8" else dict(load_in_4bit=True, bnb_4bit_quant_type="nf4")
    m = make(max_batch=8, **kw)
    ids = prompt(2)
    got = gen(m, ids, max_new_tokens=16, num_return_sequences=4, eos_token_id=-1, **SAMP)
    exp = gen(m, RS.expand(ids, 4), max_new_tokens=16, eos_token_id=-1, device_loop=True, **SAMP)
    assert torch.equal(got, exp)
    beams = gen(m, ids[:1], max_new_tokens=12, num_beams=2, num_return_sequences=3, eos_token_id=-1, **SAMP)
    assert torch.equal(beams, gen(m, RS.expand(ids[:1], 3), max_new_tokens=12, num_beams=2, eos_token_id=-1, **SAMP))


def test_lora_equals_expanded_call(tmp_path):
    import test_lora_gpu as TL
    from seed_b200.peft import PeftModel

    lm, _ = TL.build(max_batch=8)
    pm = PeftModel.from_pretrained(lm, TL.write(str(tmp_path / "a"), TL.adapter(16), 16, 32))
    ids = torch.randint(3, TL.V, (2, 12), generator=torch.Generator().manual_seed(2)).cuda()
    lm._draws = 0
    got = pm.generate(ids, max_new_tokens=16, num_return_sequences=4, eos_token_id=-1, seed=3, **SAMP)
    lm._draws = 0
    exp = pm.generate(RS.expand(ids, 4), max_new_tokens=16, eos_token_id=-1, seed=3, device_loop=True, **SAMP)
    assert torch.equal(got, exp)


# ---------------------------------------------------------------------------------------------------------------
# beam sampling
# ---------------------------------------------------------------------------------------------------------------
def _driver(m, ids, k, n):
    """the reference's strategy over B * n searches: the B prompts prefilled once, then expanded k * n times, and
    forward() per step with past_key_values reordered by index_select"""
    state = {}

    def step(seq, beam_idx):
        if beam_idx is None:
            out = m(input_ids=ids, use_cache=True, last_logits_only=True)
            state["past"] = [(a.repeat_interleave(k * n, 0), b.repeat_interleave(k * n, 0))
                             for a, b in out.past_key_values]
            return out.logits[:, -1].repeat_interleave(k * n, 0)
        bi = beam_idx.cuda()
        past = [(a.index_select(0, bi), b.index_select(0, bi)) for a, b in state["past"]]
        out = m(input_ids=seq[:, -1:].cuda(), past_key_values=past, use_cache=True, last_logits_only=True)
        state["past"] = [(a.clone(), b.clone()) for a, b in out.past_key_values]
        return out.logits[:, -1]

    return step


BEAM_CASES = [  # (k, n, B, length_penalty, early_stopping, controls)
    (2, 2, 1, 1.0, False, False),
    (2, 3, 2, 2.0, True, False),
    (4, 2, 1, 0.0, "never", False),
    (4, 3, 1, 1.0, True, False),
    (2, 3, 1, 1.0, "never", True),
    (4, 2, 2, 1.0, False, True),
]


@pytest.mark.parametrize("k,n,B,lp,es,controls", BEAM_CASES)
def test_beam_sampling_equals_expanded_call_and_restatement(model, k, n, B, lp, es, controls):
    ids, new = prompt(B), 16
    ctl = dict(repetition_penalty=1.3, no_repeat_ngram_size=2) if controls else {}
    kw = dict(num_beams=k, temperature=0.8, top_p=0.7, length_penalty=lp, early_stopping=es, do_sample=True, **ctl)
    free = gen(model, ids, max_new_tokens=new, num_return_sequences=n, eos_token_id=-1, **kw)[:, 24:]
    eos = int(free[0, 3])
    got = gen(model, ids, max_new_tokens=new, num_return_sequences=n, eos_token_id=eos, pad_token_id=VOCAB - 1, **kw)
    exp = gen(model, RS.expand(ids, n), max_new_tokens=new, eos_token_id=eos, pad_token_id=VOCAB - 1, **kw)
    assert got.shape[0] == B * n
    assert torch.equal(got, exp), (got[:, 24:].tolist(), exp[:, 24:].tolist())
    # the [B * n] scores, through the handle: the same as the expanded call's, bit for bit
    from seed_b200 import lib as L

    lkw = dict(num_beams=k, do_sample=True, temperature=0.8, top_p=0.7, length_penalty=lp, early_stopping=es,
               seed=5, eos_token_id=eos, pad_token_id=VOCAB - 1, **ctl)
    t1, s1 = model._llm.beam_generate(ids, new, num_return_sequences=n, **lkw)
    t2, s2 = model._llm.beam_generate(RS.expand(ids, n), new, **lkw)
    assert s1.shape == (B * n,) and torch.equal(s1, s2) and torch.equal(t1, t2)
    if controls:
        return                                   # the restatement states the scorer without the logits processors
    rkw = {x: y for x, y in kw.items() if x not in ("num_beams", "do_sample")}
    ref, rs, kmin, nmin, stats = RS.beam_sample_generate(_driver(model, ids, k, n), ids, new, k, n, eos=eos,
                                                         pad=VOCAB - 1, seed=5, offset=0, **rkw)
    print(f"eos {eos}: smallest key margin {kmin:.2e}, nucleus margin {nmin:.2e}, {stats}")
    if kmin <= KEY_EPS or nmin <= 1e-6:
        pytest.skip(f"a draw sits within {KEY_EPS} of a tie (margin {kmin:.2e} / {nmin:.2e}): not comparable")
    assert torch.equal(got.cpu(), ref), (got.cpu().tolist(), ref.tolist())
    assert torch.allclose(s1.cpu(), rs, atol=SCORE_TOL, rtol=0), (s1.tolist(), rs.tolist())


def test_beam_sampling_graph_equals_eager_and_n1(model):
    ids = prompt(2)
    kw = dict(max_new_tokens=16, num_beams=2, do_sample=True, temperature=1.0, top_p=0.9, eos_token_id=-1)
    a = gen(model, ids, num_return_sequences=3, use_graph=True, **kw)
    b = gen(model, ids, num_return_sequences=3, use_graph=False, **kw)
    assert torch.equal(a, b)
    assert torch.equal(gen(model, ids, num_return_sequences=1, **kw), gen(model, ids, **kw))
