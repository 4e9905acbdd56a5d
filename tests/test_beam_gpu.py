"""Beam search / beam sampling on the device (seedb200_llama_beam_generate) against tests/beam_ref.py, and the
lineage-indexed decode attention against the same kernel on a gathered cache.

Stated tolerances: the lineage attention is bit-identical.  Candidate scores agree within one fp16 rounding of the
log-probability (the kernel's fp32 log-sum-exp sums in another order than torch's, which can move an fp16 rounding);
indices agree wherever neighbouring scores are further apart than that, and, when sampling, wherever the
restatement's Gumbel-key margin exceeds KEY_EPS (log of a uniform can differ by 1 ulp between libraries).
"""
import importlib
import os
import sys

import pytest
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

from oracle import synth

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_ref as BR  # noqa: E402

pytestmark = pytest.mark.gpu
KEY_EPS = 1e-5
SCORE_TOL = 4e-3
HID, LAYERS, HEADS, FFN, VOCAB = 512, 2, 4, 1408, 1056


def make(max_batch=10, max_seq=160, int8=False, seed=9):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=VOCAB, hidden_size=HID, intermediate_size=FFN, num_hidden_layers=LAYERS,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=2048)
    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=seed)
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=max_batch, max_seq=max_seq, load_in_8bit=int8)


def prompt(B, S=24, seed=10):
    return synth.prompt_ids(B, S, n_image_spans=1, text_vocab=VOCAB - 66, n_codes=64, seed=seed).cuda()


# ---------------------------------------------------------------------------------------------------------------
# lineage-indexed decode attention
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv_len", [1, 127, 128, 129, 511, 512, 513, 2048, 3001])
def test_lineage_attention_bit_identical_to_gathered_cache(lib, kv_len):
    g = torch.Generator().manual_seed(kv_len)
    rows, used, H, D, max_seq = 8, 6, 4, 128, 4096
    k = torch.randn((rows, H, max_seq, D), generator=g).half()
    v = torch.randn((rows, H, max_seq, D), generator=g).half()
    k[used:] = float("nan")                                 # rows no table entry references
    v[used:] = float("nan")
    S = max(1, kv_len // 3)                                 # prompt part: shared by every beam of a sequence
    slot = torch.randint(0, used, (used, max_seq), generator=g, dtype=torch.int32)
    slot[:, :S] = (torch.arange(used, dtype=torch.int32) // 3)[:, None]
    slot[:, kv_len - 1] = torch.arange(used, dtype=torch.int32)
    q = torch.randn((used, H, D), generator=g).half().cuda()
    k, v, slot = k.cuda(), v.cuda(), slot.cuda()
    pos = torch.arange(max_seq, device="cuda")
    gk = k[slot.long(), :, pos[None, :], :].permute(0, 2, 1, 3).contiguous()    # [used, H, max_seq, D]
    gv = v[slot.long(), :, pos[None, :], :].permute(0, 2, 1, 3).contiguous()
    ref = lib.decode_attention(q, gk, gv, kv_len, 0.0883883)
    got = lib.decode_attention_lineage(q, k, v, slot, kv_len, 0.0883883)
    torch.cuda.synchronize()
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, ref)


@pytest.mark.parametrize("past_len", [0, 126, 127, 128, 510, 511, 512, 1500, 2047])
def test_fused_lineage_attention_bit_identical_to_gathered_cache(lib, past_len):
    """the fused RoPE + append + attention kernel every model with max_seq <= 2048 runs in its beam decode steps"""
    g = torch.Generator().manual_seed(past_len + 7)
    rows, used, H, D, max_seq = 8, 6, 4, 128, 2048
    k = torch.randn((rows, H, max_seq, D), generator=g).half()
    v = torch.randn((rows, H, max_seq, D), generator=g).half()
    k[used:] = float("nan")
    v[used:] = float("nan")
    S = max(1, past_len // 2)
    slot = torch.randint(0, used, (used, max_seq), generator=g, dtype=torch.int32)
    slot[:, :S] = (torch.arange(used, dtype=torch.int32) // 3)[:, None]
    slot[:, past_len] = torch.arange(used, dtype=torch.int32)     # the new token is appended at its own row
    qkv = torch.randn((used, 3 * H * D), generator=g).half().cuda()
    k, v, slot = k.cuda(), v.cuda(), slot.cuda()
    pos = torch.arange(max_seq, device="cuda")
    gk = k[slot.long(), :, pos[None, :], :].permute(0, 2, 1, 3).contiguous()
    gv = v[slot.long(), :, pos[None, :], :].permute(0, 2, 1, 3).contiguous()
    ref = lib.decode_attention_rope(qkv, None, H, past_len, gk, gv, 0.0883883)
    got = lib.decode_attention_rope_lineage(qkv, slot, H, past_len, k, v, 0.0883883)
    torch.cuda.synchronize()
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, ref)
    assert torch.equal(k[:used, :, past_len], gk[:, :, past_len]) and torch.equal(v[:used, :, past_len], gv[:, :, past_len])
    assert torch.isnan(k[used:].float()).all()                     # unreferenced rows neither read nor written


# ---------------------------------------------------------------------------------------------------------------
# candidates
# ---------------------------------------------------------------------------------------------------------------
def _check_candidates(sc, ix, rsc, rix, kmargin, tag):
    assert torch.allclose(sc.cpu(), rsc, atol=SCORE_TOL, rtol=0), (tag, (sc.cpu() - rsc).abs().max())
    for i in range(sc.shape[0]):
        if kmargin[i] <= KEY_EPS:
            print(f"{tag} seq {i}: key margin {kmargin[i]:.2e} <= {KEY_EPS}, not compared")
            continue
        s = rsc[i]
        for r in range(sc.shape[1]):
            near = [abs(float(s[r] - s[q])) <= SCORE_TOL for q in (r - 1, r + 1) if 0 <= q < sc.shape[1]]
            if not any(near):
                assert int(ix[i, r]) == int(rix[i, r]), (tag, i, r, ix[i].tolist(), rix[i].tolist())


@pytest.mark.parametrize("V", [1056, 40194])
@pytest.mark.parametrize("k", [1, 2, 4, 5, 8])
def test_beam_select_matches_restatement(lib, k, V):
    g = torch.Generator().manual_seed(100 * k + V % 97)
    B = 2
    logits = (torch.randn((B * k, V), generator=g) * 3).half()
    scores = (torch.randn((B * k,), generator=g) * 5).float()
    for first in (True, False):
        lg = logits[::k].contiguous() if first else logits
        bs = scores.clone()
        if first:
            bs.view(B, k)[:, 1:] = -1e9
            bs.view(B, k)[:, 0] = 0
        rows = lg.repeat_interleave(k, 0) if first else lg
        s = (BR.log_probs(rows) + bs[:, None]).view(B, k * V)
        for samp in (dict(do_sample=False), dict(do_sample=True, temperature=0.7, top_p=0.5, seed=5, offset=3),
                     dict(do_sample=True, temperature=1.0, top_p=1.0, seed=6, offset=0)):
            sc, ix = lib.beam_select(lg.cuda(), bs.cuda(), B, k, first_step=first, step=2, **samp)
            torch.cuda.synchronize()
            p = dict(samp)
            rsc, rix, km, nm = BR.select(s, k, p.pop("do_sample"), step=2, **p)
            print(f"k={k} V={V} first={first} {samp}: key margins {['%.2e' % m for m in km]}, nucleus {nm:.2e}")
            if nm <= 1e-6:
                continue
            _check_candidates(sc, ix, rsc, rix, km, f"k={k} V={V} first={first} {samp}")


# ---------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------
def _driver(model, ids, k):
    """the reference's strategy: forward() per step with past_key_values reordered by index_select"""
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


CASES = [  # (int8, k, B, do_sample, length_penalty, early_stopping)
    (False, 2, 1, False, 1.0, False),
    (False, 4, 2, False, 0.0, True),
    (False, 5, 2, False, 2.0, "never"),
    (False, 4, 1, True, 1.0, "never"),
    (False, 2, 2, True, 2.0, False),
    (False, 5, 1, True, 0.0, True),
    (True, 4, 2, False, 1.0, False),
    (True, 5, 1, True, 2.0, "never"),
]


@pytest.mark.parametrize("int8,k,B,do_sample,lp,es", CASES)
def test_beam_generate_matches_restatement(int8, k, B, do_sample, lp, es):
    model = make(int8=int8)
    ids = prompt(B)
    S, new = ids.shape[1], 20
    kw = dict(do_sample=do_sample, temperature=0.8 if do_sample else 1.0, top_p=0.7 if do_sample else 1.0,
              length_penalty=lp, early_stopping=es)
    model._draws = 0
    free = model.generate(input_ids=ids, max_new_tokens=new, num_beams=k, eos_token_id=-1, seed=11, **kw)[:, S:]
    eos = int(free[0, 3])                                   # a token this model emits: hypotheses will finish
    model._draws = 0
    got = model.generate(input_ids=ids, max_new_tokens=new, num_beams=k, eos_token_id=eos, pad_token_id=VOCAB - 1,
                         seed=11, **kw)
    ref, _, kmin, nmin, stats = BR.beam_generate(_driver(model, ids, k), ids, new, k, eos=eos, pad=VOCAB - 1, seed=11,
                                                 offset=0, **kw)
    print(f"eos {eos}: output {tuple(got.shape)}, smallest key margin {kmin:.2e}, nucleus margin {nmin:.2e}, {stats}")
    if do_sample and (kmin <= KEY_EPS or nmin <= 1e-6):
        pytest.skip(f"a draw sits within {KEY_EPS} of a tie (margin {kmin:.2e} / {nmin:.2e}): not comparable")
    assert torch.equal(got.cpu(), ref), (got.cpu().tolist(), ref.tolist())
    # the scorer's hypothesis path ran (the device output equals the restatement's, which went through it)
    assert stats["hyps_added"] > 0, stats
    tail = got[:, S:]
    finished = got.shape[1] < S + new or bool(((tail == eos) | (tail == VOCAB - 1)).any())
    _FINISHED.setdefault(es, []).append(finished)


_FINISHED = {}


def test_every_early_stopping_mode_finished_a_sequence():
    """each early_stopping mode had a case above that stopped early or ended with an eos / pad tail, so is_done and
    finalize's eos layout ran under all three"""
    if set(_FINISHED) != {False, True, "never"}:
        pytest.skip("needs the end-to-end cases of this module to have run first")
    assert all(any(v) for v in _FINISHED.values()), _FINISHED


def test_beam_graph_equals_eager_and_seeds():
    model = make()
    ids = prompt(2)
    kw = dict(max_new_tokens=24, num_beams=4, do_sample=True, temperature=1.0, top_p=0.9, eos_token_id=-1)
    model._draws = 0
    a = model.generate(input_ids=ids, seed=3, use_graph=True, **kw)
    assert model._llm.used_graph == 1
    model._draws = 0
    b = model.generate(input_ids=ids, seed=3, use_graph=False, **kw)
    assert model._llm.used_graph == 0
    model._draws = 0
    c = model.generate(input_ids=ids, seed=4, use_graph=True, **kw)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)
    g1 = model.generate(input_ids=ids, max_new_tokens=24, num_beams=4, eos_token_id=-1, use_graph=True)
    g2 = model.generate(input_ids=ids, max_new_tokens=24, num_beams=4, eos_token_id=-1, use_graph=False)
    assert torch.equal(g1, g2)


def _row_bytes(m):
    """device bytes seedb200_llama_reserve_rows adds per row (INTEGRATION.md C4)"""
    c, L = m.config, m._llm
    h, ffn, H, D, ms, vpad = c.hidden_size, c.intermediate_size, L.heads, L.head_dim, m.max_seq, L.vpad
    splits = min(64, (ms + 127) // 128)
    n = c.num_hidden_layers * 2 * H * ms * D * 2 + ms * (8 * h + ffn) * 2 + h * 2 + H * splits * 130 * 4 + H * 4
    n += 4 + 8 + ms * 8 + vpad * 2 + ms * 20 + 76
    if m.is_loaded_in_8bit:
        n += ms * (max(2 * ffn, 3 * h) * 2 + max(ffn, h) + 4)
    return n


def test_max_batch_1_model_runs_beams_and_forward_stays_correct():
    model = make(max_batch=1, max_seq=2048)
    ids = prompt(1)
    before = model(input_ids=ids).logits.clone()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    out = model.generate(input_ids=ids, max_new_tokens=16, num_beams=4, eos_token_id=-1)
    torch.cuda.synchronize()
    grown = free0 - torch.cuda.mem_get_info()[0]
    expect = 3 * _row_bytes(model)
    print(f"reserve_rows 1 -> 4: {grown} bytes, formula {expect}")
    assert model.max_batch == 4 and tuple(out.shape) == (1, ids.shape[1] + 16)
    assert abs(grown - expect) <= 0.03 * expect + (4 << 20)
    after = model(input_ids=ids).logits
    assert torch.equal(after, before)


def test_generation_config_is_honoured():
    from transformers import GenerationConfig

    model = make(max_batch=8)
    ids = prompt(2)
    gc = GenerationConfig(temperature=0.0, num_beams=4)
    a = model.generate(input_ids=ids, generation_config=gc, max_new_tokens=12)
    b = model.generate(input_ids=ids, num_beams=4, do_sample=False, eos_token_id=-1, max_new_tokens=12)
    assert torch.equal(a, b)
    with pytest.raises(NotImplementedError):
        model.generate(input_ids=ids, num_beams=2, attention_mask=torch.tensor([[0] + [1] * 23] * 2).cuda())
    with pytest.raises(NotImplementedError):
        model.generate(input_ids=ids, num_beams=2, eos_token_id=[3, 4])
    with pytest.raises(NotImplementedError):
        model.generate(input_ids=ids, num_beams=2, num_return_sequences=2)
    with pytest.raises(ValueError):
        model.generate(input_ids=ids, num_beams=9)


def test_flask_generation_dict_through_target_path(tmp_path):
    """gradio_demo/seed_llama_flask.py:164-172: num_beams from the request with do_sample, temperature and top_p,
    on the 8-bit model the default launcher loads, built through the `_target_` path from a checkpoint on disk"""
    import json

    from safetensors.torch import save_file

    sd = synth.llama_state_dict(HID, LAYERS, FFN, VOCAB, seed=21)
    save_file({k: v.half().contiguous() for k, v in sd.items()}, str(tmp_path / "model.safetensors"))
    with open(tmp_path / "config.json", "w") as f:
        json.dump({"vocab_size": VOCAB, "hidden_size": HID, "intermediate_size": FFN, "num_hidden_layers": LAYERS,
                   "num_attention_heads": HEADS, "rms_norm_eps": 1e-6, "max_position_embeddings": 256}, f)
    cfg = {"_target_": "models.model_tools.get_pretrained_llama_causal_model",
           "pretrained_model_name_or_path": str(tmp_path), "torch_dtype": "fp16", "low_cpu_mem_usage": True}
    mod, fn = cfg.pop("_target_").rsplit(".", 1)
    model = getattr(importlib.import_module(mod), fn)(**cfg, load_in_8bit=True, device_map="cuda:0")
    generation_config = {"temperature": 0.7, "num_beams": 4, "max_new_tokens": 16, "top_p": 0.5, "do_sample": True}
    ids = prompt(1)
    out = model.generate(input_ids=ids, **generation_config)
    assert model.max_batch == 4
    assert out.shape[0] == 1 and ids.shape[1] < out.shape[1] <= ids.shape[1] + 16
    assert torch.equal(out[:, :ids.shape[1]], ids)
