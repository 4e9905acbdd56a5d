"""Contrastive search on the device (seedb200_llama_contrastive_generate) against tests/contrastive_ref.py.

Stated tolerances.  The candidates' probabilities agree with the restatement within one fp16 step (the fp32 sum of
the softmax runs in another order than torch's), and their ids agree wherever neighbouring probabilities are further
apart than that.  Cosines agree within one fp16 step (fp32 sums of unit vectors in another order, then one fp16
rounding), so scores agree within SCORE_TOL and the selection agrees wherever the restatement's top-2
score gap exceeds SCORE_TOL.  The appended context row n(h_sel) and the context init agree within one fp16 step, and
bit for bit on nearly every element (the norm's fp32 sum order is free).  The composed oracle runs the candidates
through the handle's own forward on a past copied k times, as HF does; the device must give its tokens at every step
up to the first whose top-2 score gap is at most SCORE_TOL or whose k-th and (k+1)-th probabilities are within one
fp16 step (that step is reported).
"""
import os
import sys

import pytest
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

from oracle import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import contrastive_ref as CR  # noqa: E402
import processors_ref as PR  # noqa: E402

pytestmark = pytest.mark.gpu
SCORE_TOL = 2e-3
HID, LAYERS, HEADS, FFN, VOCAB = 512, 2, 4, 1408, 1056
ON = {"repetition_penalty": 1.1, "no_repeat_ngram_size": 3, "min_new_tokens": 3}


def make(max_batch=16, max_seq=160, seed=9, **q):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=VOCAB, hidden_size=HID, intermediate_size=FFN, num_hidden_layers=LAYERS,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=2048)
    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=seed)
    # a peaked next-token distribution: the random head alone gives near-uniform probabilities over 1056 tokens, where
    # most contrastive choices are near-ties
    sd["lm_head.weight"] = (sd["lm_head.weight"].float() * 8).half()
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=max_batch, max_seq=max_seq, **q)


def prompt(B, S=24, seed=10):
    return synth.prompt_ids(B, S, n_image_spans=1, text_vocab=VOCAB - 66, n_codes=64, seed=seed).cuda()


def ulp16(x: torch.Tensor) -> torch.Tensor:
    a = x.float().abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


# ---------------------------------------------------------------------------------------------------------------
# the three kernels on crafted inputs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [40194, 1001])
@pytest.mark.parametrize("k", [2, 4, 8])
def test_candidates_match_restatement(lib, k, V):
    g = torch.Generator().manual_seed(31 * k + V)
    B = 3
    logits = (torch.randn((B, V), generator=g) * 3).half()
    logits[1, 100:110] = 20.0                             # ten tied maxima: ids ascending
    logits[2, V - 3:] = float("-inf")
    ids, probs = lib.contrastive_candidates(logits.cuda(), k)
    torch.cuda.synchronize()
    ids, probs = ids.cpu(), probs.cpu()
    assert ids[1].tolist() == list(range(100, 100 + k))
    for b in range(B):
        rp = CR.softmax16(logits[b])
        rv, ri = CR.topk(rp, k + 1)
        assert (probs[b].float() - rv[:k].float()).abs().le(ulp16(rv[:k])).all(), (b, probs[b], rv)
        for j in range(k):
            near = [abs(float(rv[j]) - float(rv[q])) <= float(ulp16(rv[j])) for q in (j - 1, j + 1) if 0 <= q <= k]
            if not any(near):
                assert int(ids[b, j]) == int(ri[j]), (b, j, ids[b].tolist(), ri.tolist())
            assert float(probs[b, j]) == float(rp[ids[b, j]]) or abs(float(probs[b, j]) - float(rp[ids[b, j]])) <= \
                float(ulp16(rp[ids[b, j]]))


def test_softmax_epilogue_is_torchs_reciprocal_product():
    """torch's CUDA softmax of an fp16 row is fp16(exp(x - max) * (1 / sum)): that form agrees with it on (nearly)
    every element, better than the division form, and the kernel's probabilities are torch's"""
    from seed_b200 import lib as L

    g = torch.Generator().manual_seed(5)
    x = (torch.randn((4, 40194), generator=g) * 3).half()
    t = torch.softmax(x.cuda(), dim=-1).cpu()
    xf = x.float()
    e = torch.exp(xf - xf.max(dim=-1, keepdim=True).values)
    s = e.sum(dim=-1, keepdim=True)
    div = (e / s).half()
    mul = (e * (1.0 / s)).half()
    agree_div = (div == t).float().mean().item()
    agree_mul = (mul == t).float().mean().item()
    print(f"torch softmax fp16: division form agrees on {agree_div:.6f}, reciprocal form on {agree_mul:.6f}")
    assert agree_mul >= 0.9999 and agree_mul > agree_div
    ids, probs = L.contrastive_candidates(x.cuda(), 8)
    tp = torch.gather(t, 1, ids.cpu())
    assert ((probs.cpu().float() - tp.float()).abs() <= ulp16(tp)).all()
    assert (probs.cpu() == tp).float().mean().item() >= 0.95


def _ctx(B, rows, p, H, g):
    raw = torch.randn((B, rows, H), generator=g).half()
    ctx = CR.normalise(raw)
    ctx[:, p:] = float("nan")                             # rows past p are never read
    return ctx


@pytest.mark.parametrize("H", [4096, 5120])
@pytest.mark.parametrize("k", [2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("p", [1, 15, 16, 17, 300, 2047, 2048])
def test_rank_matches_restatement(lib, p, k, H):
    rows = 2048
    g = torch.Generator().manual_seed(p * 131 + k * 7 + H)
    B = 2
    ctx = _ctx(B, rows, p, H, g)
    hs = torch.randn((B, k, H), generator=g).half()
    i = int(torch.randint(0, p, (1,), generator=g))
    hs[0, k - 1] = ctx[0, i] * 3                           # a near-repeat of one context row: pen ~ 1
    q = CR.topk(CR.softmax16((torch.randn(VOCAB, generator=g) * 2).half()), k)[0]
    q = torch.stack([q, q])
    alpha = 0.6
    dctx = ctx.cuda()
    sel, sc = lib.contrastive_rank(dctx, p, hs.cuda(), q.cuda(), alpha)
    torch.cuda.synchronize()
    for b in range(B):
        rsel, rsc, rhn = CR.rank(ctx[b, :p], hs[b], q[b], alpha)
        assert (sc[b].cpu() - rsc.float()).abs().max() <= SCORE_TOL, (b, sc[b], rsc)
        if CR.gap(rsc) > SCORE_TOL:
            assert int(sel[b]) == rsel, (b, sel[b], rsc)
        if p < rows:
            got = dctx[b, p].cpu()
            want = rhn[int(sel[b])]
            assert ((got.float() - want.float()).abs() <= ulp16(want)).all()
            assert (got == want).float().mean() >= 0.99
        assert torch.equal(dctx[b, :p].cpu(), ctx[b, :p])  # the context itself is only read


def test_rank_ties_nan_and_alpha_rounding(lib):
    H, rows, k = 512, 8, 4
    g = torch.Generator().manual_seed(2)
    ctx = _ctx(3, rows, 4, H, g)
    hs = torch.randn((3, k, H), generator=g).half()
    hs[0, 2] = hs[0, 1]                                    # sequence 0: candidates 1 and 2 identical, same q
    q = torch.tensor([[0.25, 0.5, 0.5, 0.125]] * 3).half()
    ctx[1, 2, 7] = float("nan")                            # sequence 1: a NaN in the context -> every score NaN
    sel, sc = lib.contrastive_rank(ctx.cuda(), 4, hs.cuda(), q.cuda(), 0.6)
    torch.cuda.synchronize()
    assert sc[0, 1] == sc[0, 2] and int(sel[0]) != 2
    assert torch.isnan(sc[1]).all() and int(sel[1]) == 0
    # alpha 0.65 on a subnormal probability, where fp32(1 - alpha) and 1 - fp32(alpha) give different products
    q2 = torch.full((1, k), 1.7881393432617188e-06).half()
    far = torch.zeros((1, 4, H)).half()
    far[..., 0] = 1.0
    hz = torch.zeros((1, k, H)).half()
    hz[..., 1] = 1.0                                       # orthogonal: pen = 0, the score is the probability term
    _, sc2 = lib.contrastive_rank(far.cuda().contiguous(), 3, hz.cuda(), q2.cuda(), 0.65)
    torch.cuda.synchronize()
    assert torch.equal(sc2.cpu().half(), CR.scores(q2[0], torch.zeros(k).half(), 0.65)[None])


@pytest.mark.parametrize("H", [512, 4096, 5120])
def test_context_init_matches_restatement(lib, H):
    g = torch.Generator().manual_seed(H)
    B, S, rows = 2, 37, 64
    hs = (torch.randn((B, S, H), generator=g) * 4).half()
    ctx = torch.full((B, rows, H), float("nan")).half().cuda()
    lib.contrastive_context_init(hs.cuda(), ctx)
    torch.cuda.synchronize()
    want = CR.normalise(hs)
    got = ctx[:, :S].cpu()
    assert ((got.float() - want.float()).abs() <= ulp16(want)).all()
    assert (got == want).float().mean() >= 0.99
    assert torch.isnan(ctx[:, S:].float()).all()


# ---------------------------------------------------------------------------------------------------------------
# composed oracle: HF's loop with the candidate forward on a past copied k times
# ---------------------------------------------------------------------------------------------------------------
class _Oracle:
    """prefill / candidates_forward of contrastive_ref.generate on the handle: kv_load of each sequence's selected past
    repeated k times, the handle's own forward of the B*k candidate rows, tap_hidden for h"""

    def __init__(self, model, k):
        self.m, self.llm, self.k = model, model._llm, k

    def prefill(self, ids):
        B, S = ids.shape
        lg = self.llm.forward(input_ids=ids.cuda(), past_len=0, last_only=True)[:, 0]
        hs = self.llm.tap_hidden(B * S).view(B, S, -1)
        self.past = [(k[:, :, :S].clone(), v[:, :, :S].clone()) for k, v in self.m._kv_tuple(B, S)]
        self.B = B
        return lg.cpu(), hs.cpu()

    def __call__(self, t, ids):
        B, k = self.B, self.k
        p = self.past[0][0].shape[2]
        for l, (pk, pv) in enumerate(self.past):
            self.llm.kv_load(l, pk.repeat_interleave(k, 0), pv.repeat_interleave(k, 0))
        lg = self.llm.forward(input_ids=ids.view(B * k, 1).cuda(), past_len=p, last_only=True)[:, 0]
        hs = self.llm.tap_hidden(B * k)
        self.p = p
        return lg.view(B, k, -1).cpu(), hs.view(B, k, -1).cpu()

    def on_select(self, t, sels):
        rows = torch.tensor([b * self.k + s for b, s in enumerate(sels)], device="cuda")
        kv = self.m._kv_tuple(self.B * self.k, self.p + 1)
        self.past = [(torch.cat([pk, k[rows, :, self.p:self.p + 1]], 2), torch.cat([pv, v[rows, :, self.p:self.p + 1]], 2))
                     for (pk, pv), (k, v) in zip(self.past, kv)]


def _oracle(model, ids, n, k, alpha, ctl, eos=None, pad=0):
    o = _Oracle(model, k)
    probs = lambda row: torch.softmax(row.cuda(), dim=-1).cpu()      # HF's own fp16 softmax on CUDA
    return CR.generate(o.prefill, o, ids.cpu(), n, k, alpha, ctl, eos=eos, pad=pad, probs_fn=probs)


def _first_uncertain(gaps, edges):
    for t, (gp, ed) in enumerate(zip(gaps, edges)):
        for g_, (pk, pk1) in zip(gp, ed):
            if g_ <= SCORE_TOL or abs(pk - pk1) <= float(ulp16(torch.tensor(pk))):
                return t
    return len(gaps)


def _compare(dev, ref, gaps, edges, tag, least=4):
    stop = _first_uncertain(gaps, edges)
    print(f"{tag}: compared {stop} of {ref.shape[1]} steps" + ("" if stop == len(gaps) else
                                                                  f"; step {stop} is within the tolerance"))
    assert stop >= min(least, ref.shape[1]), f"{tag}: too few steps above the tolerance ({stop})"
    assert torch.equal(dev[:, :stop].cpu(), ref[:, :stop]), (tag, dev.tolist(), ref.tolist())
    return stop


@pytest.mark.parametrize("B,k", [(1, 2), (1, 4), (1, 8), (2, 4)])
def test_matches_composed_oracle(B, k):
    model = make()
    ids = prompt(B)
    n, alpha = 24, 0.6
    dev = model.generate(input_ids=ids, max_new_tokens=n, penalty_alpha=alpha, top_k=k, eos_token_id=-1)
    ref, gaps, edges = _oracle(model, ids, n, k, alpha, dict(PR.NEUTRAL))
    _compare(dev[:, ids.shape[1]:], ref, gaps, edges, f"B={B} k={k}")


def test_matches_composed_oracle_with_processors():
    model = make()
    ids = prompt(2, seed=3)
    n, k, alpha, eos = 20, 4, 0.5, 7
    dev = model.generate(input_ids=ids, max_new_tokens=n, penalty_alpha=alpha, top_k=k, eos_token_id=eos, **ON)
    ref, gaps, edges = _oracle(model, ids, n, k, alpha, dict(PR.NEUTRAL, **ON), eos=eos, pad=eos)
    new = dev[:, ids.shape[1]:]
    assert new.shape[1] == ref.shape[1] or _first_uncertain(gaps, edges) < ref.shape[1]
    _compare(new, ref[:, :new.shape[1]], gaps, edges, "processors")


@pytest.mark.parametrize("fmt", ["lora", "int8", "nf4"])
def test_weight_formats_match_composed_oracle(fmt):
    q = {"int8": dict(load_in_8bit=True), "nf4": dict(load_in_4bit=True, bnb_4bit_quant_type="nf4")}.get(fmt, {})
    model = make(**q)
    if fmt == "lora":
        g = torch.Generator().manual_seed(4)
        t = {}
        for l in range(LAYERS):
            for proj in ("q_proj", "v_proj"):
                t[f"model.layers.{l}.self_attn.{proj}.lora_A.weight"] = (torch.randn(8, HID, generator=g) * 0.05).half().cuda()
                t[f"model.layers.{l}.self_attn.{proj}.lora_B.weight"] = (torch.randn(HID, 8, generator=g) * 0.05).half().cuda()
        model._llm.lora_load(t, 8, 16)
    compared = 0
    for seed in (6, 7, 8):                                 # three prompts, at least 8 steps above the tolerance in all
        ids = prompt(1, seed=seed)
        dev = model.generate(input_ids=ids, max_new_tokens=16, penalty_alpha=0.6, top_k=4, eos_token_id=-1)
        ref, gaps, edges = _oracle(model, ids, 16, 4, 0.6, dict(PR.NEUTRAL))
        compared += _compare(dev[:, ids.shape[1]:], ref, gaps, edges, f"{fmt} prompt {seed}", least=0)
    assert compared >= 8, compared


# ---------------------------------------------------------------------------------------------------------------
# loop behaviour
# ---------------------------------------------------------------------------------------------------------------
def test_graph_replay_matches_eager_with_constant_launches(lib):
    model = make()
    ids = prompt(2, seed=8)
    kw = dict(penalty_alpha=0.6, top_k=4, eos_token_id=-1)
    counts, outs = [], []
    for n in (10, 20):
        for use_graph in (True, False):
            lib.reset_launch_count()
            outs.append(model.generate(input_ids=ids, max_new_tokens=n, use_graph=use_graph, **kw))
            torch.cuda.synchronize()
            counts.append(lib.launch_count())
            assert model._llm.used_graph == int(use_graph)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[2], outs[3])
    assert torch.equal(outs[0], outs[2][:, :outs[0].shape[1]])
    # the same launches per unit eagerly and replayed, and a constant number per unit
    assert counts[0] == counts[1] and counts[2] == counts[3]
    assert (counts[2] - counts[0]) % 10 == 0


def test_eos_pad_and_early_stop():
    model = make()
    ids = prompt(2, seed=8)
    base = model.generate(input_ids=ids, max_new_tokens=30, penalty_alpha=0.6, top_k=4, eos_token_id=-1)
    new = base[:, ids.shape[1]:].cpu()
    eos = int(new[0, 3])                                   # sequence 0 emits it at step 3 at the latest
    out = model.generate(input_ids=ids, max_new_tokens=30, penalty_alpha=0.6, top_k=4, eos_token_id=eos,
                         pad_token_id=1).cpu()[:, ids.shape[1]:]
    for b in range(2):
        hit = [t for t in range(new.shape[1]) if int(new[b, t]) == eos]
        if hit:                                            # identical up to eos, pad afterwards
            e = hit[0]
            assert torch.equal(out[b, :e + 1], new[b, :e + 1]) and (out[b, e + 1:] == 1).all()
        else:
            assert torch.equal(out[b], new[b, :out.shape[1]])
    done = [any(int(x) == eos for x in new[b]) for b in range(2)]
    if all(done):                                          # stopped at the step where the last sequence finished
        last = max(min(t for t in range(new.shape[1]) if int(new[b, t]) == eos) for b in range(2))
        assert out.shape[1] == last + 1
    else:
        assert out.shape[1] == 30


def test_max_seq_truncates():
    model = make(max_seq=40)
    ids = prompt(1)                                        # 24 tokens: 16 fit
    out = model.generate(input_ids=ids, max_new_tokens=64, penalty_alpha=0.6, top_k=4, eos_token_id=-1)
    assert tuple(out.shape) == (1, 40)
    ref = model.generate(input_ids=ids, max_new_tokens=16, penalty_alpha=0.6, top_k=4, eos_token_id=-1)
    assert torch.equal(out, ref)


def test_reserve_rows_growth():
    small = make(max_batch=1)
    big = make(max_batch=16)
    ids = prompt(2, seed=12)
    kw = dict(max_new_tokens=12, penalty_alpha=0.6, top_k=4, eos_token_id=-1)
    a = small.generate(input_ids=ids, **kw)
    assert small.max_batch == 8
    assert torch.equal(a, big.generate(input_ids=ids, **kw))
    assert torch.equal(small.generate(input_ids=ids[:1], **kw), big.generate(input_ids=ids[:1], **kw))


@pytest.mark.parametrize("kw", [dict(do_sample=True, top_p=0.9, seed=3), dict(num_beams=2), dict(), dict(top_k=1)])
def test_penalty_alpha_ignored_outside_contrastive_mode(lib, kw):
    model = make()
    ids = prompt(1, seed=13)
    outs, counts = [], []
    for extra in ({}, {"penalty_alpha": 0.6}, {"penalty_alpha": None}):
        if extra.get("penalty_alpha") and "top_k" not in kw and not kw.get("do_sample") and kw.get("num_beams", 1) == 1:
            continue                                        # greedy without top_k: refused (covered on the CPU)
        lib.reset_launch_count()
        model._draws = 0                                    # the same Philox offset for every sampled run
        outs.append(model.generate(input_ids=ids, max_new_tokens=10, eos_token_id=-1, **kw, **extra))
        torch.cuda.synchronize()
        counts.append(lib.launch_count())
    assert all(torch.equal(o, outs[0]) for o in outs) and len(set(counts)) == 1
