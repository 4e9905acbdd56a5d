"""Generation controls on the device (seedb200_logits_params: top_k, repetition_penalty, no_repeat_ngram_size,
min_length, min_new_tokens) against tests/processors_ref.py, and the neutral settings against the entry points
without them.

Greedy decisions must match exactly.  Sampled draws are compared where the restatement's draw and nucleus margins
exceed those of the existing sampler tests (the kernel sums in fp32 in another order); beam candidates where the
Gumbel-key margin exceeds KEY_EPS, as tests/test_beam_gpu.py does.
"""
import ctypes as C
import os
import sys

import pytest
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

from oracle import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import processors_ref as PR  # noqa: E402

pytestmark = pytest.mark.gpu
KEY_EPS = 1e-5
HID, LAYERS, HEADS, FFN, VOCAB = 512, 2, 4, 1408, 1056
ON = {"top_k": 50, "repetition_penalty": 1.1, "no_repeat_ngram_size": 3}


def make(max_batch=8, max_seq=160, seed=9, **q):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=VOCAB, hidden_size=HID, intermediate_size=FFN, num_hidden_layers=LAYERS,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=2048)
    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=seed)
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=max_batch, max_seq=max_seq, **q)


def prompt(B, S=24, seed=10):
    return synth.prompt_ids(B, S, n_image_spans=1, text_vocab=VOCAB - 66, n_codes=64, seed=seed).cuda()


def _sample_driver(model, ids):
    """the HF-shaped strategy: prefill, then forward() of the last token with the cache"""
    state = {}

    def step(seq):
        if "past" not in state:
            out = model(input_ids=seq.cuda(), use_cache=True, last_logits_only=True)
        else:
            out = model(input_ids=seq[:, -1:].cuda(), past_key_values=state["past"], use_cache=True,
                        last_logits_only=True)
        state["past"] = out.past_key_values
        return out.logits[:, -1]
    return step


def _beam_driver(model, ids, k):
    state = {}

    def step(seq, beam_idx):
        if beam_idx is None:
            out = model(input_ids=ids, use_cache=True, last_logits_only=True)
            state["past"] = [(a.repeat_interleave(k, 0), b.repeat_interleave(k, 0)) for a, b in out.past_key_values]
            return out.logits[:, -1].repeat_interleave(k, 0)
        bi = beam_idx.cuda()
        past = [(a.index_select(0, bi), b.index_select(0, bi)) for a, b in state["past"]]
        out = model(input_ids=seq[:, -1:].cuda(), past_key_values=past, use_cache=True, last_logits_only=True)
        state["past"] = [(a.clone(), b.clone()) for a, b in out.past_key_values]
        return out.logits[:, -1]
    return step


# ---------------------------------------------------------------------------------------------------------------
# fp16 arithmetic the contract rests on
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [1.1, 1.2, 1.3, 0.7, 3.0, 0.5])
def test_cuda_scalar_division_is_the_fp32_reciprocal_product(p):
    """torch's CUDA `fp16 tensor / Python float` -- what RepetitionPenalty and TemperatureLogitsWarper run -- equals
    fp16(x * fp32(1 / p)), the rule the header states and the kernels follow; `* p` is fp16(x * fp32(p))"""
    x = torch.arange(0, 1 << 16, dtype=torch.int32).to(torch.int16).view(torch.float16)
    x = x[torch.isfinite(x.float())]
    got = (x.cuda() / p).cpu()
    assert torch.equal(got.view(torch.int16), PR.scalar_div(x, p).view(torch.int16))
    assert torch.equal((x.cuda() * p).cpu().view(torch.int16), (x.float() * PR.f32(p)).half().view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------
# seedb200_sample_processed on crafted rows
# ---------------------------------------------------------------------------------------------------------------
def _rows(B, V, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((B, V), generator=g) * 3).half()


@pytest.mark.parametrize("V", [1056, 40194])
def test_sample_processed_matches_restatement(lib, V):
    B, S, eos = 4, 12, 7
    logits = _rows(B, V, V)
    g = torch.Generator().manual_seed(V + 1)
    hist = torch.randint(0, V, (B, 20), generator=g)
    am = logits.float().argmax(-1)
    # row 0: its argmax is in the history and positive (the penalty moves it down)
    hist[0, 3] = am[0]
    logits[0, am[0]] = 8.0
    # row 1: its argmax is banned by the 3-gram that ends the history
    hist[1, 5:8] = torch.tensor([11, 12, int(am[1])])
    hist[1, 18:20] = torch.tensor([11, 12])
    logits[1, am[1]] = 9.0
    # row 2: eos is the argmax and masked while fewer than min_new_tokens were generated
    logits[2, eos] = 10.0
    # row 3: a plateau of ties around the top-k boundary
    logits[3, 100:140] = 5.0
    hist_d, lg_d = hist.cuda(), logits.cuda()
    cases = [dict(repetition_penalty=3.0), dict(no_repeat_ngram_size=3), dict(min_new_tokens=9),
             dict(min_length=21, repetition_penalty=0.8), dict(top_k=7), dict(top_k=50, repetition_penalty=1.1,
                                                                              no_repeat_ngram_size=2)]
    for ctl in cases:
        for samp in (dict(do_sample=False), dict(do_sample=True, temperature=0.7, top_p=0.9),
                     dict(do_sample=True, temperature=1.0, top_p=0.5), dict(do_sample=True, temperature=1.3)):
            for seed in range(3):
                got = lib.sample(lg_d, seed=seed, offset=1, step=2, history=hist_d, prompt_len=S, eos_token_id=eos,
                                 **samp, **ctl).cpu()
                for b in range(B):
                    tok, dm, nm = PR.sample_row(logits[b], hist[b].tolist(), S, eos, ctl, samp["do_sample"],
                                                samp.get("temperature", 1.0), samp.get("top_p", 1.0), seed, 1, 2, b)
                    if dm < 1e-5 or nm < 2e-6:
                        continue
                    assert int(got[b]) == tok, (ctl, samp, seed, b, int(got[b]), tok)
    assert torch.equal(lg_d.cpu(), logits)                 # sample() leaves the caller's logits alone
    # the crafted rows did what they were built for (greedy)
    g0 = lib.sample(lg_d, history=hist_d, prompt_len=S, eos_token_id=eos, repetition_penalty=3.0).cpu()
    g1 = lib.sample(lg_d, history=hist_d, prompt_len=S, eos_token_id=eos, no_repeat_ngram_size=3).cpu()
    g2 = lib.sample(lg_d, history=hist_d, prompt_len=S, eos_token_id=eos, min_new_tokens=9).cpu()
    assert int(g0[0]) != int(am[0]) and int(g1[1]) != int(am[1]) and int(g2[2]) != eos


@pytest.mark.parametrize("V", [1001, 40194])
def test_top_k_select_is_exact_at_the_boundary(lib, V):
    """deterministic pins of the histogram select inside sample_kernel.  top_k=1 samples the argmax for every seed
    and temperature (unless tempering ties it).  With k-1 values above a tied plateau of 20 and the rest of the row
    just below it, top_k = k keeps exactly the plateau and the values above, where every other token would be drawn
    almost surely; k-1 keeps none of the plateau, k+19 the same as k, k+20 adds the top of the rest."""
    g = torch.Generator().manual_seed(V)
    logits = (torch.randn((4, V), generator=g) * 3).half()
    am = logits.float().argmax(-1)
    for T in (1.0, 0.7, 1.9):
        for seed in range(16):
            got = lib.sample(logits.cuda(), do_sample=True, temperature=T, top_k=1, seed=seed).cpu()
            for b in range(4):
                key = logits[b] if T == 1.0 else PR.scalar_div(logits[b], T)
                kept = PR.top_k_keep(key, 1, 1)
                assert bool(kept[got[b]]), (T, seed, b)
                if int(kept.sum()) == 1:
                    assert int(got[b]) == int(am[b]), (T, seed, b)
    k = 6
    idx = torch.randperm(V, generator=g)
    above, plateau = idx[:k - 1], idx[k - 1:k + 19]
    row = (4.9 - torch.rand(V, generator=g) * 0.5).half()
    row[above], row[plateau] = 6.0, 5.0
    row_d = row[None].cuda()
    in_set = lambda t, ids: bool((ids == t).any())       # noqa: E731
    compared = total = 0
    for kk in (k - 1, k, k + 19, k + 20):
        for T in (1.0, 0.7, 300.0):
            for seed in range(32):
                got = int(lib.sample(row_d, do_sample=True, temperature=T, top_k=kk, seed=seed)[0])
                if kk < k:
                    assert in_set(got, above), (kk, T, seed, got)
                elif kk < k + 20:
                    assert in_set(got, above) or in_set(got, plateau), (kk, T, seed, got)
                tok, dm, nm = PR.sample_row(row, [], 0, -1, {"top_k": kk}, True, T, 1.0, seed)
                total += 1
                if dm < 1e-5:
                    continue
                compared += 1
                assert got == tok, (kk, T, seed, got, tok)
    assert compared >= 0.9 * total, (compared, total)


def _raw_c(lib_mod, name, *args):
    lib_mod.check(getattr(lib_mod.load(), name)(*args), name)


def test_neutral_params_are_bit_identical_with_the_same_launch_count(lib):
    """seedb200_*_processed with every control neutral = the entry points without them, launch for launch"""
    neutral = lib.LogitsParams(0, 1.0, 0, 0, 0)
    V, B = 40194, 3
    lg = _rows(B, V, 5).cuda()
    for sp in (lib.SampleParams(0, 1.0, 1.0, 0, 0), lib.SampleParams(1, 0.8, 0.6, 7, 3)):
        a = torch.empty(B, dtype=torch.int64, device="cuda")
        b = torch.empty(B, dtype=torch.int64, device="cuda")
        lib.reset_launch_count()
        _raw_c(lib, "seedb200_sample", lg.data_ptr(), V, B, V, C.byref(sp), 4, a.data_ptr(), None)
        n0 = lib.launch_count()
        lib.reset_launch_count()
        _raw_c(lib, "seedb200_sample_processed", lg.data_ptr(), V, B, V, C.byref(sp), 4, b.data_ptr(), None,
               C.byref(neutral), None, 0, 0, 0, 2)
        assert lib.launch_count() == n0 and torch.equal(a, b)
    model = make()
    L = model._llm
    ids = prompt(2)
    for fn, params, extra in (
            ("seedb200_llama_generate", lib.SampleParams(1, 0.9, 0.7, 3, 0), ()),
            ("seedb200_llama_beam_generate", lib.beam_params(3, True, 0.8, 0.7, seed=3), (None,))):
        outs, counts = [], []
        for processed in (False, True):
            out = torch.empty((2, 20), dtype=torch.int64, device="cuda")
            n = C.c_int(0)
            lib.reset_launch_count()
            args = [L._h, ids.data_ptr(), 2, ids.shape[1], 20, C.byref(params), 5, 0, 1, out.data_ptr(), C.byref(n),
                    *extra, None]
            if processed:
                _raw_c(lib, fn + "_processed", *args, C.byref(neutral))
            else:
                _raw_c(lib, fn, *args)
            torch.cuda.synchronize()
            counts.append(lib.launch_count())
            outs.append(out[:, :n.value].clone())
        assert counts[0] == counts[1], (fn, counts)
        assert torch.equal(outs[0], outs[1]), fn


# ---------------------------------------------------------------------------------------------------------------
# the generation loops
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("samp", [dict(do_sample=False), dict(do_sample=True, temperature=0.9, top_p=0.8, seed=31)])
def test_device_loop_hf_loop_eager_and_graph_agree(samp):
    model = make()
    ids = prompt(2)
    ctl = dict(ON, min_new_tokens=4)
    outs = []
    for kw in (dict(use_graph=True), dict(use_graph=False), dict(device_loop=False)):
        model._draws = 0
        outs.append(model.generate(input_ids=ids, max_new_tokens=24, eos_token_id=5, pad_token_id=0, **samp, **ctl,
                                   **kw))
        if "use_graph" in kw:
            assert model._llm.used_graph == int(kw["use_graph"])
    assert torch.equal(outs[0], outs[1]), "graph replay differs from eager launches"
    assert torch.equal(outs[0], outs[2]), "device loop differs from the per-token Python loop"
    model._draws = 0
    off = model.generate(input_ids=ids, max_new_tokens=24, eos_token_id=5, pad_token_id=0, **samp)
    assert not torch.equal(off, outs[0])                   # the controls changed the output


@pytest.mark.parametrize("samp", [dict(do_sample=False), dict(do_sample=True, temperature=0.8, top_p=0.9, seed=5)])
@pytest.mark.parametrize("ctl", [dict(repetition_penalty=1.8), dict(no_repeat_ngram_size=2, top_k=20),
                                 dict(ON, min_length=30)])
def test_generate_matches_restatement(samp, ctl):
    model = make()
    ids = prompt(2)
    new, eos = 20, 3
    model._draws = 0
    got = model.generate(input_ids=ids, max_new_tokens=new, eos_token_id=eos, pad_token_id=0, **samp, **ctl)
    p = dict(samp)
    p.pop("seed", None)
    ref, dmin, nmin = PR.generate(_sample_driver(model, ids), ids, new, ctl, eos=eos, pad=0, seed=samp.get("seed", 0),
                                  **p)
    if dmin < 1e-5 or nmin < 2e-6:
        pytest.skip(f"a draw sits within {dmin:.1e} / {nmin:.1e} of a boundary: not comparable")
    assert torch.equal(got.cpu(), ref), (got.cpu().tolist(), ref.tolist())


BEAM_CASES = [  # (k, do_sample, ctl)
    (4, False, dict(repetition_penalty=1.5)),
    (3, False, dict(no_repeat_ngram_size=2, min_new_tokens=6)),
    (4, True, dict(ON)),
    (2, True, dict(top_k=5, repetition_penalty=0.9)),
]


@pytest.mark.parametrize("k,do_sample,ctl", BEAM_CASES)
def test_beam_generate_matches_restatement(k, do_sample, ctl):
    model = make()
    ids = prompt(2)
    new, eos = 16, 3
    kw = dict(do_sample=do_sample, temperature=0.8 if do_sample else 1.0, top_p=0.8 if do_sample else 1.0)
    model._draws = 0
    got = model.generate(input_ids=ids, max_new_tokens=new, num_beams=k, eos_token_id=eos, pad_token_id=VOCAB - 1,
                         seed=11, **kw, **ctl)
    ref, kmin, nmin = PR.beam_generate(_beam_driver(model, ids, k), ids, new, k, ctl, eos=eos, pad=VOCAB - 1,
                                       seed=11, **kw)
    if do_sample and (kmin <= KEY_EPS or nmin <= 1e-6):
        pytest.skip(f"a draw sits within {KEY_EPS} of a tie (margin {kmin:.2e} / {nmin:.2e}): not comparable")
    assert torch.equal(got.cpu(), ref), (got.cpu().tolist(), ref.tolist())
    model._draws = 0
    eager = model.generate(input_ids=ids, max_new_tokens=new, num_beams=k, eos_token_id=eos, pad_token_id=VOCAB - 1,
                           seed=11, use_graph=False, **kw, **ctl)
    assert torch.equal(got, eager)


def test_beam_rows_use_their_own_history():
    """no_repeat_ngram_size=1 bans every token of a row's own sequence: once the beams diverge their bans differ, and
    a restatement that gives every beam row its sequence's first beam's history produces another output"""
    model = make()
    ids = prompt(1)
    k, new, ctl = 4, 14, dict(no_repeat_ngram_size=1)
    got = model.generate(input_ids=ids, max_new_tokens=new, num_beams=k, eos_token_id=-1, **ctl)
    step = _beam_driver(model, ids, k)
    ref = PR.beam_generate(step, ids, new, k, ctl)[0]
    assert torch.equal(got.cpu(), ref)
    shared = PR.beam_generate(_beam_driver(model, ids, k), ids, new, k, ctl, shared_history=True)[0]
    assert not torch.equal(shared, ref), "the case does not tell per-row histories from shared ones"


def test_changed_parameters_take_effect_on_the_captured_graph():
    model = make()
    ids = prompt(2)
    for beams in (1, 3):
        outs = []
        for pen in (3.0, 0.05, 3.0):                       # 0.05 strongly favours tokens already in the row
            model._draws = 0
            g = model.generate(input_ids=ids, max_new_tokens=20, num_beams=beams, eos_token_id=-1,
                               repetition_penalty=pen, top_k=10)
            assert model._llm.used_graph == 1
            model._draws = 0
            e = model.generate(input_ids=ids, max_new_tokens=20, num_beams=beams, eos_token_id=-1,
                               repetition_penalty=pen, top_k=10, use_graph=False)
            assert torch.equal(g, e), (beams, pen)
            outs.append(g)
        assert not torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


# ---------------------------------------------------------------------------------------------------------------
# weight formats
# ---------------------------------------------------------------------------------------------------------------
def _lora(model, r=8, seed=4):
    g = torch.Generator().manual_seed(seed)
    t = {}
    for l in range(LAYERS):
        for proj in ("q_proj", "v_proj"):
            t[f"model.layers.{l}.self_attn.{proj}.lora_A.weight"] = (torch.randn(r, HID, generator=g) * 0.05).half().cuda()
            t[f"model.layers.{l}.self_attn.{proj}.lora_B.weight"] = (torch.randn(HID, r, generator=g) * 0.05).half().cuda()
    model._llm.lora_load(t, r, 2 * r)
    return model


@pytest.mark.parametrize("fmt", ["int8", "nf4", "lora"])
def test_weight_formats_run_the_controls(fmt):
    q = {"int8": dict(load_in_8bit=True), "nf4": dict(load_in_4bit=True, bnb_4bit_quant_type="nf4")}.get(fmt, {})
    model = make(**q)
    if fmt == "lora":
        _lora(model)
    ids = prompt(1)
    ctl = dict(ON, min_new_tokens=3)
    a = model.generate(input_ids=ids, max_new_tokens=16, eos_token_id=-1, **ctl)
    b = model.generate(input_ids=ids, max_new_tokens=16, eos_token_id=-1, device_loop=False, **ctl)
    assert torch.equal(a, b)
    ref = PR.generate(_sample_driver(model, ids), ids, 16, ctl)[0]
    assert torch.equal(a.cpu(), ref)
    c = model.generate(input_ids=ids, max_new_tokens=8, num_beams=2, eos_token_id=-1, **ctl)
    assert tuple(c.shape) == (1, ids.shape[1] + 8)


# ---------------------------------------------------------------------------------------------------------------
# memory
# ---------------------------------------------------------------------------------------------------------------
def test_memory_neutral_allocates_nothing_and_the_token_table_is_as_documented():
    """a one-layer 128-wide model with max_batch * max_seq = 2^19, so that the 4 * ms bytes per row of the token
    table (2 MiB) are one whole page of the driver's allocator and show in the free memory"""
    from models.llama_xformer import LlamaForCausalLM

    h, V, ms = 128, 64, 65536
    cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=h, num_hidden_layers=1, num_attention_heads=1,
                      num_key_value_heads=1, rms_norm_eps=1e-6, max_position_embeddings=ms)
    model = LlamaForCausalLM(cfg, synth.llama_state_dict(h, 1, h, V, seed=3), device="cuda", max_batch=8, max_seq=ms)
    ids = torch.randint(3, V, (2, 8), generator=torch.Generator().manual_seed(1)).cuda()
    kw = dict(max_new_tokens=12, eos_token_id=-1)
    model.generate(input_ids=ids, **kw)                    # warm: torch's allocator holds the output blocks
    model.generate(input_ids=ids, num_beams=4, **kw)
    model.generate(input_ids=ids, **kw, **ON)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    model.generate(input_ids=ids, **kw)
    model.generate(input_ids=ids, num_beams=4, **kw)
    model.generate(input_ids=ids, **kw, **ON)              # the sampler path keeps its history in existing rows
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0
    model.generate(input_ids=ids, num_beams=4, **kw, **ON)  # first beam call with a history control: the token table
    torch.cuda.synchronize()
    grown = free0 - torch.cuda.mem_get_info()[0]
    expect = 4 * model.max_batch * model.max_seq          # INTEGRATION.md C4: 4 * ms per row
    print(f"token table: {grown} bytes, documented {expect}")
    assert grown == expect
    model.generate(input_ids=ids, num_beams=4, **kw, **ON)
    torch.cuda.synchronize()
    assert free0 - torch.cuda.mem_get_info()[0] == grown
