"""generate(output_scores=True, return_dict_in_generate=True) in greedy decoding, sampling and contrastive search, on
the device.

The device loop (seedb200_llama_generate_ex: the sampler writes each step's row, graph-replayed) is compared bit for
bit against the per-token Python loop (forward() + seedb200_sample_scores per token) on the same seed: tokens and every
`scores` entry.  With num_return_sequences = n > 1 the per-token loop prefills the expanded batch, whose prefill GEMM
may round some logits differently from the device loop's prefill of the B prompts, so there the scores are compared
against the composed oracle of tests/test_return_sequences_gpu.py (the B prompts prefilled once, their K/V copied into
n rows each), and the tokens against the per-token loop.  The per-op sampler is also compared against tests/scores_ref.py on its own logits, which pins which
tokens are -inf.  Contrastive search's rows are compared against the processed logits of the composed oracle of
tests/test_contrastive_gpu.py.  The calls without scores are checked to issue the launches and return the tokens they
did before.
"""
import os
import sys

import pytest
import torch
from transformers.generation import GenerateBeamDecoderOnlyOutput, GenerateDecoderOnlyOutput
from transformers.utils import ModelOutput
from transformers.models.llama.configuration_llama import LlamaConfig

from oracle import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import scores_ref as SR  # noqa: E402

pytestmark = pytest.mark.gpu
HID, LAYERS, HEADS, FFN, VOCAB = 512, 2, 4, 1408, 1056
S0 = 24
C7 = dict(top_k=40, repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=3)
MODES = {"greedy": dict(do_sample=False), "sample": dict(do_sample=True, temperature=0.9, top_p=0.8),
         "sample_t1": dict(do_sample=True, temperature=1.0, top_p=0.5)}
CONTRASTIVE = dict(penalty_alpha=0.6, top_k=4)
BEAM = dict(num_beams=4)
BEAM_SAMPLE = dict(num_beams=2, do_sample=True, temperature=0.8, top_p=0.7, top_k=20)
OTHER = {"contrastive": CONTRASTIVE, "beam": BEAM, "beam_sample": BEAM_SAMPLE}


def make(max_batch=24, max_seq=160, seed=9, **kw):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=VOCAB, hidden_size=HID, intermediate_size=FFN, num_hidden_layers=LAYERS,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=2048)
    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=seed)
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=max_batch, max_seq=max_seq, **kw)


def prompt(B, S=S0, seed=10):
    return synth.prompt_ids(B, S, n_image_spans=1, text_vocab=VOCAB - 66, n_codes=64, seed=seed).cuda()


@pytest.fixture(scope="module")
def model():
    return make()


def gen(m, ids, **kw):
    m._draws = 0
    return m.generate(input_ids=ids, seed=kw.pop("seed", 5), **kw)


def scored(m, ids, **kw):
    return gen(m, ids, return_dict_in_generate=True, output_scores=True, **kw)


def assert_same(a, b, S, V=VOCAB):
    assert torch.equal(a.sequences, b.sequences), (a.sequences[:, S:].tolist(), b.sequences[:, S:].tolist())
    assert len(a.scores) == len(b.scores) == a.sequences.shape[1] - S
    for t, (x, y) in enumerate(zip(a.scores, b.scores)):
        assert x.dtype == torch.float16 and x.shape == (a.sequences.shape[0], V)
        assert torch.equal(x, y), f"step {t}"


def composed(m, ids, n, new, eos, pad, **kw):
    """the composed oracle of tests/test_return_sequences_gpu.py with scores: prefill the B prompts once, copy their
    K/V into n rows each, then forward() + L.sample(scores_out=...) per token over the B * n rows"""
    from seed_b200 import lib as L

    B, S = ids.shape
    out = m(input_ids=ids, use_cache=True, last_logits_only=True)
    past = [(k.repeat_interleave(n, 0).contiguous(), v.repeat_interleave(n, 0).contiguous())
            for k, v in out.past_key_values]
    logits = out.logits[:, -1].repeat_interleave(n, 0).contiguous()
    seq, scores = ids.repeat_interleave(n, 0), []
    unfinished = torch.ones(B * n, dtype=torch.bool, device="cuda")
    for step in range(new):
        buf = L.scores_buffer(1, B * n, VOCAB, "cuda")[0]
        nxt = L.sample(logits, seed=5, offset=0, step=step, history=seq, prompt_len=S, eos_token_id=eos,
                       scores_out=buf, **kw)
        scores.append(buf[:, :VOCAB])
        nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad))
        seq = torch.cat([seq, nxt[:, None]], dim=1)
        unfinished &= nxt != eos
        if not bool(unfinished.any()) or step == new - 1:
            break
        o = m(input_ids=seq[:, -1:], past_key_values=past, use_cache=True, last_logits_only=True)
        past, logits = o.past_key_values, o.logits[:, -1].contiguous()
    return GenerateDecoderOnlyOutput(sequences=seq, scores=tuple(scores))


def assert_tokens_scored(out, S, eos=None, greedy=False):
    """each emitted token of an unfinished row has a finite score; greedy tokens are the argmax of their row"""
    seq = out.sequences
    alive = torch.ones(seq.shape[0], dtype=torch.bool, device=seq.device)
    for t, sc in enumerate(out.scores):
        tok = seq[:, S + t]
        v = sc.gather(1, tok[:, None])[:, 0]
        assert bool(torch.isfinite(v[alive]).all()), f"step {t}"
        if greedy:
            assert torch.equal(tok[alive], sc.float().argmax(1)[alive]), f"step {t}"
        if eos is not None:
            alive &= tok != eos


LOOP_CASES = [(mode, B, n) for mode in MODES for B in (1, 3) for n in (1, 3)
              if n == 1 or mode != "greedy"]            # num_return_sequences > 1 needs sampling


@pytest.mark.parametrize("controls", [False, True])
@pytest.mark.parametrize("mode,B,n", LOOP_CASES)
def test_device_loop_equals_token_loop(model, mode, B, n, controls):
    ids, kw = prompt(B), dict(MODES[mode], **(C7 if controls else {}))
    free = gen(model, ids, max_new_tokens=20, num_return_sequences=n, eos_token_id=-1, device_loop=True, **kw)
    eos = int(free[-1, S0 + 3])                          # a token the last row emits: it finishes early
    common = dict(max_new_tokens=20, num_return_sequences=n, eos_token_id=eos, pad_token_id=VOCAB - 1, **kw)
    dev = scored(model, ids, device_loop=True, **common)
    loop = scored(model, ids, device_loop=False, **common)
    assert isinstance(dev, GenerateDecoderOnlyOutput) and isinstance(loop, GenerateDecoderOnlyOutput)
    assert dev.sequences.shape[0] == B * n
    if n == 1:
        assert_same(dev, loop, S0)
    else:
        assert torch.equal(dev.sequences, loop.sequences) and len(loop.scores) == len(dev.scores)
        assert_same(dev, composed(model, ids, n, 20, eos, VOCAB - 1, **kw), S0)
    assert_tokens_scored(dev, S0, eos=eos, greedy=mode == "greedy")
    if not controls:            # (min_new_tokens bans eos for 3 steps, so the run may leave the free run's path)
        assert bool((dev.sequences[-1, S0:] == eos).any())


@pytest.mark.parametrize("mode", list(MODES) + list(OTHER))
def test_tokens_and_launches_unchanged_without_scores(model, mode):
    from seed_b200 import lib as L

    ids, kw = prompt(2), dict(MODES.get(mode) or OTHER[mode], max_new_tokens=16, eos_token_id=-1)
    results = []
    for extra in ({}, dict(return_dict_in_generate=False), dict(return_dict_in_generate=True),
                  dict(return_dict_in_generate=True, output_scores=False), dict(output_scores=True)):
        gen(model, ids, **kw)                                            # graphs captured before counting
        before = L.launch_count()
        out = gen(model, ids, **kw, **extra)
        torch.cuda.synchronize()
        results.append((extra, out, L.launch_count() - before))
    base = results[0][1]
    assert isinstance(base, torch.Tensor)
    for extra, out, launches in results:
        if extra.get("return_dict_in_generate"):
            assert isinstance(out, ModelOutput) and out.scores is None
            out = out.sequences
        else:
            assert isinstance(out, torch.Tensor)       # output_scores alone: the bare tensor
        assert torch.equal(out, base), extra
        assert launches == results[0][2], (extra, launches, results[0][2])


def test_graph_replay_equals_eager(model):
    ids = prompt(3)
    for mode in ("greedy", "sample", "contrastive", "beam", "beam_sample"):
        kw = dict(MODES.get(mode) or OTHER[mode], max_new_tokens=20, eos_token_id=-1, device_loop=True)
        a = scored(model, ids, use_graph=True, **kw)
        b = scored(model, ids, use_graph=False, **kw)
        assert len(a.scores) == len(b.scores)
        for x, y in zip(a.scores, b.scores):
            assert torch.equal(x, y), mode
        assert torch.equal(a.sequences, b.sequences), mode
        if mode.startswith("beam"):
            assert torch.equal(a.sequences_scores, b.sequences_scores)
            assert torch.equal(a.beam_indices, b.beam_indices)


def test_consecutive_calls_write_their_own_buffers(model):
    """the decode graph of (B=1, sampling) is captured by the first call and replayed by the third: its scores must
    land in the third call's buffer, and the first call's must stay as they were"""
    kw = dict(MODES["sample"], max_new_tokens=18, eos_token_id=-1, device_loop=True)
    a = scored(model, prompt(1), **kw)
    a_saved = [s.clone() for s in a.scores]
    b = scored(model, prompt(3, seed=11), **kw)
    b_saved = [s.clone() for s in b.scores]
    c = scored(model, prompt(1), **kw)
    assert_same(a, c, S0)
    for x, y in zip(a.scores, a_saved):
        assert torch.equal(x, y)
    for x, y in zip(b.scores, b_saved):
        assert torch.equal(x, y)
    loop = scored(model, prompt(3, seed=11), **dict(kw, device_loop=False))
    assert_same(b, loop, S0)


def test_truncation_at_max_seq(model):
    ids = prompt(2, S=150)
    kw = dict(MODES["sample"], max_new_tokens=30, eos_token_id=-1)
    dev = scored(model, ids, device_loop=True, **kw)
    assert dev.sequences.shape == (2, model.max_seq) and len(dev.scores) == model.max_seq - 150
    assert_same(dev, scored(model, ids, device_loop=False, **kw), 150)


def test_generation_config_fields(model):
    from transformers import GenerationConfig

    ids = prompt(1)
    cfg = GenerationConfig(max_new_tokens=8, do_sample=True, top_p=0.8, output_scores=True,
                           return_dict_in_generate=True, eos_token_id=-1)
    out = gen(model, ids, generation_config=cfg)
    assert isinstance(out, GenerateDecoderOnlyOutput) and len(out.scores) == 8
    assert isinstance(gen(model, ids, generation_config=cfg, return_dict_in_generate=False), torch.Tensor)
    assert gen(model, ids, generation_config=cfg, output_scores=False).scores is None


@pytest.mark.parametrize("T,top_p,top_k", [(1.0, 1.0, 0), (0.7, 1.0, 0), (1.0, 0.6, 0), (0.8, 0.9, 30),
                                           (1.3, 0.5, 5)])
def test_per_op_scores_equal_restatement(T, top_p, top_k):
    """seedb200_sample_scores on random rows: finite exactly on the restatement's kept set, with its tempered values"""
    from seed_b200 import lib as L

    g = torch.Generator().manual_seed(int(T * 100 + top_p * 10 + top_k))
    B, V = 6, 4000
    logits = (torch.randn(B, V, generator=g) * 3).half()
    logits[0, :7] = logits[0, 7]                                          # ties
    logits[1, 100:200] = float("-inf")
    buf = L.scores_buffer(1, B, V, "cuda")[0]
    tok = L.sample(logits.cuda(), do_sample=True, temperature=T, top_p=top_p, top_k=top_k, seed=3, scores_out=buf)
    got = buf[:, :V].cpu()
    for b in range(B):
        ref, margin = SR.score_row(logits[b], [], 0, -1, dict(top_k=top_k), True, T, top_p)
        if margin <= 1e-5:
            continue
        assert torch.equal(torch.isinf(got[b]), torch.isinf(ref)), b
        fin = torch.isfinite(ref)
        assert torch.equal(got[b][fin], ref[fin]), b
        assert torch.isfinite(got[b, int(tok[b])])
    greedy = L.scores_buffer(1, B, V, "cuda")[0]
    L.sample(logits.cuda(), do_sample=False, scores_out=greedy)
    assert torch.equal(greedy[:, :V].cpu(), logits)


@pytest.mark.parametrize("fmt", ["int8", "nf4"])
def test_quantised_weights(fmt):
    kw = dict(load_in_8bit=True) if fmt == "int8" else dict(load_in_4bit=True, bnb_4bit_quant_type="nf4")
    m = make(max_batch=6, max_seq=96, **kw)
    ids = prompt(2)
    common = dict(MODES["sample"], max_new_tokens=12, num_return_sequences=2, eos_token_id=-1, **C7)
    assert_same(scored(m, ids, device_loop=True, **common), scored(m, ids, device_loop=False, **common), S0)


def test_lora(tmp_path):
    import test_lora_gpu as TL
    from seed_b200.peft import PeftModel

    lm, _ = TL.build(max_batch=8)
    pm = PeftModel.from_pretrained(lm, TL.write(str(tmp_path / "a"), TL.adapter(16), 16, 32))
    ids = torch.randint(3, TL.V, (2, 12), generator=torch.Generator().manual_seed(2)).cuda()
    outs = []
    for loop in (True, False):
        lm._draws = 0
        outs.append(pm.generate(ids, max_new_tokens=10, eos_token_id=-1, seed=3, device_loop=loop,
                                return_dict_in_generate=True, output_scores=True, **MODES["sample"]))
    assert_same(outs[0], outs[1], 12, V=TL.V)
    ts = pm.compute_transition_scores(outs[0].sequences, outs[0].scores, normalize_logits=True)
    assert ts.shape == (2, 10) and bool(torch.isfinite(ts).all()) and bool((ts <= 0).all())


@pytest.mark.parametrize("seed,alpha,eos,controls", [(10, 0.6, None, False), (3, 0.5, 7, True)])
def test_contrastive_scores_equal_composed_oracle(seed, alpha, eos, controls):
    """the rows the composed oracle hands to its softmax are the processed logits contrastive_search stores; step 0
    (the prefill's logits) is compared bit for bit, later steps (candidate rows through the lineage table on one side,
    through kv_load on the other) within fp16 rounding, up to the first step whose selection is within the oracle's
    tolerance"""
    import contrastive_ref as CR
    import processors_ref as PR
    from test_contrastive_gpu import ON, _first_uncertain, _Oracle
    from test_contrastive_gpu import make as make_peaked      # its sharper head keeps the selections off near-ties

    m = make_peaked()
    ids, n, k = prompt(2, seed=seed), 20, 4
    ctl = ON if controls else {}
    dev = scored(m, ids, max_new_tokens=n, penalty_alpha=alpha, top_k=k, eos_token_id=-1 if eos is None else eos,
                 **ctl)
    steps = len(dev.scores)
    assert steps == dev.sequences.shape[1] - ids.shape[1]
    rows = []

    def probs(row):
        rows.append(row.clone())
        return torch.softmax(row.cuda(), dim=-1).cpu()

    o = _Oracle(m, k)
    _, gaps, edges = CR.generate(o.prefill, o, ids.cpu(), n, k, alpha, dict(PR.NEUTRAL, **ctl), eos=eos,
                                 pad=0 if eos is None else eos, probs_fn=probs)
    stop = min(_first_uncertain(gaps, edges) + 1, steps)     # step t's row follows the selections of steps < t
    assert stop >= min(4, steps), stop
    for t in range(stop):
        for b in range(2):
            got, ref = dev.scores[t][b].cpu(), rows[t * 2 + b]
            if t == 0:
                assert torch.equal(got, ref), b
            assert torch.equal(torch.isinf(got), torch.isinf(ref)), (t, b)
            fin = torch.isfinite(ref)
            assert torch.allclose(got[fin].float(), ref[fin].float(), rtol=2e-3, atol=2e-3), (t, b)
    # each token of an unfinished row is one of its step's k candidates: among the k largest processed logits
    for t in range(steps if eos is None else 0):
        tok = dev.sequences[:, ids.shape[1] + t]
        kth = dev.scores[t].float().topk(k, dim=1).values[:, -1]
        assert bool((dev.scores[t].float().gather(1, tok[:, None])[:, 0] >= kth).all()), t


# ---------------------------------------------------------------------------------------------------------------
# beam search and beam sampling
# ---------------------------------------------------------------------------------------------------------------
BEAM_CASES = [  # (k, n, do_sample, length_penalty, early_stopping)
    (2, 1, False, 1.0, False), (4, 1, False, 2.0, True), (4, 1, False, 0.0, "never"), (2, 1, False, 1.0, "never"),
    (2, 1, True, 1.0, False), (4, 1, True, 1.0, True), (2, 2, True, 1.0, "never"), (4, 2, True, 2.0, False),
]


def _transition_identity(m, out, S, lp, eos):
    """HF's documented identity for beam search: transition scores summed over a hypothesis, divided by its length **
    length_penalty, give sequences_scores; the length is the prompt plus the tokens before a closing eos"""
    ts = m.compute_transition_scores(out.sequences, tuple(s.float() for s in out.scores),
                                     beam_indices=out.beam_indices)
    n = (out.beam_indices >= 0).sum(1)
    last = out.sequences.gather(1, (S + n - 1)[:, None])[:, 0]
    length = (S + n - (last == eos).long()).double()
    rec = ts.double().sum(1) / length ** lp
    assert torch.allclose(rec.float(), out.sequences_scores, rtol=1e-5, atol=1e-4), (rec, out.sequences_scores)


@pytest.mark.parametrize("k,n,do_sample,lp,es", BEAM_CASES)
def test_beam_scores_equal_restatement(model, k, n, do_sample, lp, es):
    """against tests/scores_ref.beam_generate driven by the composed oracle of tests/test_return_sequences_gpu.py
    (forward() per step with the past reordered by index_select): tokens, len(scores), beam_indices exactly; the score
    rows and sequences_scores within fp16 rounding of the logits the two sides compute"""
    from test_return_sequences_gpu import KEY_EPS, _driver

    ids, new = prompt(1), 16
    kw = dict(num_beams=k, do_sample=do_sample, length_penalty=lp, early_stopping=es, num_return_sequences=n)
    if do_sample:
        kw.update(temperature=0.8, top_p=0.7, top_k=30)
    free = gen(model, ids, max_new_tokens=new, eos_token_id=-1, **kw)
    eos = int(free[0, S0 + 3])
    out = scored(model, ids, max_new_tokens=new, eos_token_id=eos, pad_token_id=VOCAB - 1, **kw)
    assert isinstance(out, GenerateBeamDecoderOnlyOutput)
    plain = gen(model, ids, max_new_tokens=new, eos_token_id=eos, pad_token_id=VOCAB - 1, **kw)
    assert torch.equal(out.sequences, plain)                               # scores change no token
    G = n
    assert out.sequences_scores.shape == (G,) and out.beam_indices.shape == out.sequences.shape
    assert all(s.shape == (G * k, VOCAB) and s.dtype == torch.float16 for s in out.scores)
    assert len(out.scores) >= out.sequences.shape[1] - S0
    for g in range(G):                                                     # step 0: a search's k rows are identical
        for j in range(1, k):
            assert torch.equal(out.scores[0][g * k], out.scores[0][g * k + j])
    if not do_sample:
        _transition_identity(model, out, S0, lp, eos)
    rkw = {x: y for x, y in kw.items() if x not in ("num_beams", "do_sample", "num_return_sequences", "top_k",
                                                      "length_penalty", "early_stopping")}
    ref, rscores, rss, rbi, kmin, nmin = SR.beam_generate(
        _driver(model, ids, k, n), ids.repeat_interleave(n, 0), new, k, {"top_k": kw.get("top_k", 0)},
        do_sample=do_sample, length_penalty=lp, early_stopping=es, eos=eos, pad=VOCAB - 1, seed=5, offset=0, **rkw)
    if kmin <= KEY_EPS or nmin <= 1e-5:
        pytest.skip(f"a draw or TopP boundary within its margin ({kmin:.2e} / {nmin:.2e}): not comparable")
    assert torch.equal(out.sequences.cpu(), ref), (out.sequences[:, S0:].tolist(), ref[:, S0:].tolist())
    assert len(out.scores) == len(rscores)
    assert torch.equal(out.beam_indices.cpu(), rbi), (out.beam_indices.tolist(), rbi.tolist())
    assert torch.allclose(out.sequences_scores.cpu(), rss, atol=4e-3, rtol=0)
    for t, (a, b) in enumerate(zip(out.scores, rscores)):
        a = a.cpu()
        assert torch.equal(torch.isinf(a), torch.isinf(b)), t
        fin = torch.isfinite(b)
        assert torch.allclose(a[fin].float(), b[fin].float(), atol=2e-2, rtol=1e-3), t


def test_beam_sampling_warp_keeps_the_nucleus_at_t1(model):
    """at T = 1 the warped row is log-probabilities on the kept set: its mass reaches top_p, the mass without its least
    token does not (threshold form, min_tokens_to_keep = 2)"""
    ids, top_p = prompt(2), 0.6
    out = scored(model, ids, max_new_tokens=12, num_beams=2, do_sample=True, temperature=1.0, top_p=top_p,
                 eos_token_id=-1)
    for s in out.scores:
        p = s.float().exp()
        kept = torch.isfinite(s)
        assert bool((kept.sum(1) >= 2).all())
        mass = p.sum(1)
        least = torch.where(kept, p, torch.full_like(p, 2.0)).min(1).values
        ok = (mass >= top_p - 1e-2) & ((mass - least < top_p + 1e-2) | (kept.sum(1) == 2))
        assert bool(ok.all()), (mass, least)


def test_beam_consecutive_calls_write_their_own_buffers(model):
    kw = dict(num_beams=2, max_new_tokens=14, eos_token_id=-1)
    a = scored(model, prompt(1), **kw)
    saved = [s.clone() for s in a.scores]
    scored(model, prompt(2, seed=11), **kw)
    c = scored(model, prompt(1), **kw)
    assert torch.equal(a.sequences, c.sequences) and torch.equal(a.beam_indices, c.beam_indices)
    for x, y, z in zip(a.scores, c.scores, saved):
        assert torch.equal(x, y) and torch.equal(x, z)


def test_beam_truncation_at_max_seq(model):
    ids = prompt(1, S=150)
    out = scored(model, ids, max_new_tokens=30, num_beams=2, eos_token_id=-1)
    assert out.sequences.shape == (1, model.max_seq) and len(out.scores) == model.max_seq - 150
    _transition_identity(model, out, 150, 1.0, -1)
