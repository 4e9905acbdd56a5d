"""LoRA kernels and the LoRA LLaMA against the restatement in tests/lora_ref.py.

Shrink: within one fp16 ulp plus the fp32 summation error of the float64 product rounded once (the two only differ by
more than an ulp where the terms cancel; each test prints how often).  Expand (GEMV epilogue and GEMM + expand kernel):
fed with the kernels' own base and t, bit for bit against the chain with u summed in fp32 in ascending j (exact
emulation), over r in {1, 8, 13, 64}, partial adapters, inf / NaN rows and guard-word outputs.  Merge: bit for bit
against the same emulation.  Model: a synthetic adapter with B != 0 that moves the logits by more than 5 % matches the
composed restatement and, in beam search, tests/beam_ref.py; a zero adapter gives the base model's outputs.
"""
import json
import os
import sys

import pytest
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_ref  # noqa: E402
import lora_ref as R  # noqa: E402
from oracle import synth  # noqa: E402

pytestmark = pytest.mark.gpu
LINS = (("self_attn", "q_proj"), ("self_attn", "k_proj"), ("self_attn", "v_proj"), ("self_attn", "o_proj"),
        ("mlp", "gate_proj"), ("mlp", "up_proj"), ("mlp", "down_proj"))


def randh(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half()


def within(got, ref, bound):
    """|got - ref| <= bound elementwise (same non-finite pattern); -> number of outputs that are not exact"""
    got, ref, bound = got.cpu().double(), ref.cpu().double(), bound.cpu().double()
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isfinite(got), fin)
    d = (got - ref).abs()
    bad = fin & (d > bound + 1e-30)
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{int(bad.sum())} outputs beyond the bound, first at {list(i)}: got {got[i].item()!r} "
                             f"ref {ref[i].item()!r} bound {bound[i].item()!r}")
    return int((d[fin] > 0).sum())


def within_ulp(got, ref, n=1):
    return within(got, ref, n * R.ulp(ref.cpu().double()))


@pytest.mark.parametrize("M", [1, 2, 3, 4, 5, 257, 2048])
@pytest.mark.parametrize("K", [512, 1408])
@pytest.mark.parametrize("r", [1, 8, 16, 64])
def test_shrink(lib, M, K, r):
    rtot = 3 * r                      # q|k|v: 192 columns at r = 64, the widest operand a model builds
    x = randh(M, K, seed=M + K)
    a = randh(rtot, K, seed=r, scale=0.05)
    if M > 2:
        x[1, 7] = float("inf")
        x[2, 9] = float("nan")
    t = lib.lora_shrink(x.cuda(), a.cuda())
    ref = R.shrink(x, a)
    ok = [i for i in range(M) if i not in (1, 2) or M <= 2]
    n = within(t[ok], ref[ok], R.shrink_bound(x[ok], a))
    n1 = int(((t[ok].cpu().double() - ref[ok].double()).abs() > R.ulp(ref[ok])).sum())
    print(f"shrink M={M} K={K} r={r}: {n} of {len(ok) * rtot} not exact, {n1} beyond one ulp (cancellation)")
    if M > 2:   # a non-finite input stays in its own row
        assert not torch.isfinite(t[1].float()).all() and torch.isnan(t[2].float()).all()


@pytest.mark.parametrize("M", [1, 4])
def test_shrink_fused_norm_matches_gemv_staging(lib, M):
    K = 1024
    x = randh(M, K, seed=3).cuda()
    w = (1.0 + randh(K, seed=4, scale=0.2).float()).half().cuda()
    a = randh(16, K, seed=5, scale=0.05).cuda()
    eye = torch.eye(K, dtype=torch.float16, device="cuda")
    staged = lib.gemv(x, eye, norm_w=w)          # the GEMV's normalised activations, exactly
    assert torch.equal(lib.lora_shrink(x, a, norm_w=w), lib.lora_shrink(staged, a))


SENT = 0x7E5A          # a NaN payload no kernel writes


def guarded(M, n):
    """an [M, n] fp16 output inside a buffer whose guard words must keep their bits"""
    G = 64
    buf = torch.full((G + M * n + G,), SENT, dtype=torch.int16, device="cuda")
    return buf, buf[G:G + M * n].view(torch.float16).view(M, n), G


def same_bits(a, b):
    """identical fp16 values, NaN matching NaN (payloads are not part of the contract); +0 == -0 is not accepted"""
    a, b = a.cpu(), b.cpu()
    nan = torch.isnan(a.float())
    return torch.equal(nan, torch.isnan(b.float())) and torch.equal(a.view(torch.int16)[~nan], b.view(torch.int16)[~nan])


def same_values(a, b):
    """equal values with +0 == -0 and NaN matching NaN"""
    a, b = a.cpu().float(), b.cpu().float()
    return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def expand_exact(base, t, b, r, grp, nsub, mask, s):
    """the kernels' expand, bit for bit: u summed in fp32 in ascending j (fp16 x fp16 products are exact in fp32, so
    each fp32 add equals the kernels' fmaf), then the restated roundings; a cleared mask bit passes base through"""
    M, N = base.shape
    rows = torch.arange(N)
    sub = (rows // grp) % nsub
    tcols = sub[:, None] * r + torch.arange(r)[None, :]
    tt = t.cpu().float()[:, tcols]                       # [M, N, r]
    bb = b.cpu().float()
    acc = torch.zeros(M, N)
    for j in range(r):
        acc = acc + bb[None, :, j] * tt[:, :, j]
    u = R.fp16(acc)
    c = R.fp16(u.float() * torch.tensor(s, dtype=torch.float32))
    y = R.fp16(base.cpu().float() + c.float())
    on = ((mask >> sub) & 1).bool()
    return torch.where(on[None, :], y, base.cpu())


SHAPES = [(384, 128, 3, 0b111), (384, 128, 3, 0b101), (512, 128, 2, 0b11), (512, 128, 2, 0b01), (320, 320, 1, 1),
          (200, 200, 1, 1)]


@pytest.mark.parametrize("M", [1, 3, 8, 200])
@pytest.mark.parametrize("N,grp,nsub,mask", SHAPES)
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
@pytest.mark.parametrize("r", [1, 8, 13, 64])
def test_expand(lib, M, N, grp, nsub, mask, bn, r):
    """GEMV (M <= 4, expand in its epilogue) and GEMM + expand kernel: y bit for bit against expand_exact fed the
    kernels' own base and t, the residual step exactly fp16(residual + y), a zero B exactly the base kernel, an inf /
    NaN row confined to its row, and guard words around every output."""
    if M <= 4 and bn != 0:
        pytest.skip("the GEMV has no tile width")
    K, s = 256, 2.0
    x = randh(M, K, seed=M + r).cuda()
    if M >= 3:
        x[1, 5] = float("inf")
        x[2, 6] = float("nan")
    w = randh(N, K, seed=N, scale=0.05).cuda()
    a = randh(nsub * r, K, seed=7 + r, scale=0.05).cuda()
    b = randh(N, r, seed=8 + r, scale=0.3).cuda()
    res = randh(M, N, seed=9).cuda()
    t = lib.lora_shrink(x, a)
    lo = lib.lora_operand(t, b, r, grp, nsub, s, mask)
    bz = torch.zeros_like(b)          # the operand holds raw pointers: keep the tensor alive
    zero = lib.lora_operand(t, bz, r, grp, nsub, s, mask)
    gemv = M <= 4

    def run(op, mode=0, residual=None):
        n_out = N // 2 if mode == 1 else N
        buf, out, G = guarded(M, n_out)
        if gemv:
            lib.gemv_lora(x, w, op, residual=residual, mode=mode, out=out)
        else:
            lib.gemm_lora(x, w, op, residual=residual, mode=mode, bn=bn if mode == 0 else 0, out=out)
        bb = buf.cpu()
        assert torch.all(bb[:G] == SENT) and torch.all(bb[G + M * n_out:] == SENT)
        return out.clone()

    def base(mode=0, residual=None):
        if gemv:
            return lib.gemv(x, w, residual=residual, mode=mode)
        return lib.gemm(x, w, residual=residual, mode=mode, bn=bn if mode == 0 else 0)

    b0 = base()
    y = run(lo)
    ref = expand_exact(b0, t, b, r, grp, nsub, mask, s)
    assert same_bits(y, ref)
    if M >= 3:   # rows without a non-finite input are unaffected by rows 1 and 2
        keep = [m for m in range(M) if m not in (1, 2)]
        assert torch.isfinite(y[keep].float()).all()
    assert same_bits(run(lo, residual=res), (y.float() + res.float()).half())
    assert same_bits(run(zero), expand_exact(b0, t, bz, r, grp, nsub, mask, s))
    # a zero B is the base kernel on rows with finite inputs (an inf in t gives 0 * inf = NaN, as PEFT's matmul does)
    fr = [m for m in range(M) if M < 3 or m not in (1, 2)]
    assert same_values(run(zero)[fr], b0[fr]) and same_values(run(zero, residual=res)[fr], base(residual=res)[fr])
    if N % 256 == 0 and nsub == 2:
        assert same_values(run(zero, mode=1)[fr], base(mode=1)[fr])
        g = y.view(M, N // 256, 2, 128)
        fin = [m for m in range(M) if M < 3 or m not in (1, 2)]
        got1 = run(lo, mode=1)[fin]
        within_ulp(got1, R.silu_gate(g[fin, :, 0].reshape(len(fin), -1).cpu(), g[fin, :, 1].reshape(len(fin), -1).cpu()), 2)


# ---- model -------------------------------------------------------------------------------------------------------
H, NL, HEADS, FFN, V = 256, 2, 2, 512, 1000


def build(max_batch=6, vocab=V, seed=11, sd=None):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=vocab, hidden_size=H, intermediate_size=FFN, num_hidden_layers=NL,
                      num_attention_heads=HEADS, num_key_value_heads=HEADS, rms_norm_eps=1e-6,
                      max_position_embeddings=2048, eos_token_id=2)
    sd = synth.llama_state_dict(H, NL, FFN, vocab, seed=seed) if sd is None else sd
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=max_batch, max_seq=256), sd


def adapter(r=16, zero_b=False, scale=0.4, seed=21, targets=tuple(p for _, p in LINS)):
    sd = {}
    for l in range(NL):
        for par, proj in LINS:
            if proj not in targets:
                continue
            n_out = FFN if proj in ("gate_proj", "up_proj") else H
            k_in = FFN if proj == "down_proj" else H
            pre = f"base_model.model.model.layers.{l}.{par}.{proj}"
            sd[pre + ".lora_A.weight"] = randh(r, k_in, seed=seed + l * 10 + len(sd), scale=k_in ** -0.5).float()
            sd[pre + ".lora_B.weight"] = (torch.zeros(n_out, r) if zero_b
                                          else randh(n_out, r, seed=seed + 100 + len(sd), scale=scale).float())
    return sd


def write(path, sd, r=16, alpha=32, save=(), fmt="safetensors", targets=tuple(p for _, p in LINS)):
    os.makedirs(path, exist_ok=True)
    cfg = {"peft_type": "LORA", "r": r, "lora_alpha": alpha, "bias": "none", "target_modules": list(targets),
           "modules_to_save": list(save) or None, "task_type": "CAUSAL_LM"}
    with open(os.path.join(path, "adapter_config.json"), "w") as f:
        json.dump(cfg, f)
    sd = {k: v.contiguous().clone() for k, v in sd.items()}
    if fmt == "bin":
        torch.save(sd, os.path.join(path, "adapter_model.bin"))
    else:
        from safetensors.torch import save_file

        save_file(sd, os.path.join(path, "adapter_model.safetensors"))
    return path


def merged_sd(sd, ad, s):
    out = dict(sd)
    for l in range(NL):
        for par, proj in LINS:
            k = f"model.layers.{l}.{par}.{proj}"
            a = ad[f"base_model.model.{k}.lora_A.weight"].half()
            b = ad[f"base_model.model.{k}.lora_B.weight"].half()
            out[k + ".weight"] = R.merge(sd[k + ".weight"].half(), a, b, s)
    return out


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


def test_zero_adapter_is_the_base_model(tmp_path):
    from seed_b200.peft import PeftModel

    base, _ = build()
    lm, _ = build()
    pm = PeftModel.from_pretrained(lm, write(str(tmp_path / "z"), adapter(zero_b=True)))
    ids = torch.randint(3, V, (3, 37), generator=torch.Generator().manual_seed(1)).cuda()
    assert torch.equal(pm(ids).logits, base(ids).logits)                       # prefill (GEMM)
    o1, o2 = pm(ids[:1, :20]), base(ids[:1, :20])
    d1 = pm(ids[:1, 20:21], past_key_values=o1.past_key_values).logits         # cached decode (GEMV)
    d2 = base(ids[:1, 20:21], past_key_values=o2.past_key_values).logits
    assert torch.equal(d1, d2)
    p = ids[:2, :12]
    assert torch.equal(pm.generate(p, max_new_tokens=16, eos_token_id=-1), base.generate(p, max_new_tokens=16, eos_token_id=-1))
    assert torch.equal(pm.generate(p, max_new_tokens=10, num_beams=3, eos_token_id=-1),
                       base.generate(p, max_new_tokens=10, num_beams=3, eos_token_id=-1))


def test_model_against_merged_restatement_and_merge(tmp_path):
    from seed_b200.peft import PeftModel

    r, alpha = 16, 32
    ad = adapter(r)
    base, sd = build()
    lm, _ = build()
    pm = PeftModel.from_pretrained(lm, write(str(tmp_path / "a"), ad, r, alpha))
    ids = torch.randint(3, V, (2, 40), generator=torch.Generator().manual_seed(2)).cuda()
    got, b0 = pm(ids).logits, base(ids).logits
    moved = rel(got, b0)
    print(f"adapter moves the logits by {moved:.3f} relative")
    assert moved >= 0.05
    ref_model, _ = build(sd=merged_sd(sd, ad, alpha / r))
    err = rel(got, ref_model(ids).logits)
    print(f"LoRA vs merged-weight model {err:.3e}")
    assert err <= 1e-2
    # chunked prefill + cached decode, and a batch of 6 through the GEMM path
    o = pm(ids[:, :24])
    o = pm(ids[:, 24:39], past_key_values=o.past_key_values)
    last = pm(ids[:, 39:40], past_key_values=o.past_key_values).logits
    assert rel(last, got[:, 39:40]) <= 1e-2
    ids6 = torch.randint(3, V, (6, 20), generator=torch.Generator().manual_seed(3)).cuda()
    o = pm(ids6[:, :19])
    step6 = pm(ids6[:, 19:20], past_key_values=o.past_key_values).logits
    assert rel(step6, pm(ids6).logits[:, 19:20]) <= 1e-2
    # generation: graph, eager and the Python loop agree
    p = ids[:1, :10]
    g1 = pm.generate(p, max_new_tokens=24, eos_token_id=-1)
    g2 = pm.generate(p, max_new_tokens=24, eos_token_id=-1, use_graph=False)
    g3 = pm.generate(p, max_new_tokens=24, eos_token_id=-1, device_loop=False)
    assert torch.equal(g1, g2) and torch.equal(g1, g3)
    # composed restatement: restated LoRA linears between the GPU's own embedding, norms, RoPE, attention and lm_head
    comp = composed(sd, ad, ids, alpha / r)
    err_c = rel(got, comp)
    print(f"LoRA vs composed restatement {err_c:.3e}; chunked {rel(last, comp[:, 39:40]):.3e}")
    assert err_c <= 1e-2 and rel(last, comp[:, 39:40]) <= 1e-2
    comp6 = composed(sd, ad, ids6, alpha / r)
    assert rel(pm(ids6).logits, comp6) <= 1e-2 and rel(step6, comp6[:, 19:20]) <= 1e-2
    # merge: every merged weight equals the kernel's arithmetic emulated exactly (o_proj / down_proj are borrowed and
    # read back; q|k|v and gate|up are checked through the model), and the merged model's logits equal a base model
    # built from the emulated weights, bit for bit
    merged = pm.merge_and_unload()
    ref_m = dict(sd)
    for l in range(NL):
        for par, proj in LINS:
            k = f"model.layers.{l}.{par}.{proj}"
            ref_m[k + ".weight"] = merge_exact(sd[k + ".weight"].half(), ad[f"base_model.model.{k}.lora_A.weight"].half(),
                                               ad[f"base_model.model.{k}.lora_B.weight"].half(), alpha / r)
    for k, v in lm._llm._weights.items():
        if "o_proj" in k or "down_proj" in k:
            assert same_bits(v, ref_m[k]), k
    exact, _ = build(sd=ref_m)
    assert torch.equal(merged(ids).logits, exact(ids).logits)
    assert rel(merged(ids).logits, got) <= 1e-2


def merge_exact(w, a, b, s):
    """the merge kernel bit for bit: fp32 sum over r in ascending j, then fp16(fp16(.) * s) added to W and rounded"""
    acc = torch.zeros(w.shape)
    for j in range(a.shape[0]):
        acc = acc + b.float()[:, j, None] * a.float()[None, j, :]
    d = R.fp16(R.fp16(acc).float() * torch.tensor(s, dtype=torch.float32))
    return R.fp16(w.float() + d.float())


def composed(sd, ad, ids, s, eps=1e-6):
    """The LoRA forward with the restated linears (lora_ref.linear / silu_gate, on the CPU in float64 + fp16 roundings)
    between the GPU's own embedding, RMSNorm, RoPE + KV append, causal attention and lm_head kernels."""
    from seed_b200 import lib as L

    B, S = ids.shape
    h, D, dev = H, H // HEADS, "cuda"

    def half(k):
        return sd[k].half().to(dev)

    def lin(t, k, residual=None):
        rows = t.reshape(-1, t.shape[-1]).cpu()
        y = R.linear(rows, sd[k + ".weight"].half(), ad[f"base_model.model.{k}.lora_A.weight"].half(),
                     ad[f"base_model.model.{k}.lora_B.weight"].half(), s)
        if residual is not None:
            y = R.fp16(y.float() + residual.reshape(-1, y.shape[-1]).cpu().float())
        return y.view(B, S, -1).to(dev)

    x = L.embedding(half("model.embed_tokens.weight"), ids.to(dev).reshape(-1)).view(B, S, h)
    for l in range(NL):
        p = f"model.layers.{l}."
        kc = torch.zeros(B, HEADS, S, D, dtype=torch.float16, device=dev)
        vc = torch.zeros_like(kc)
        n = L.rmsnorm(x.reshape(-1, h), half(p + "input_layernorm.weight"), eps).view(B, S, h)
        qkv = torch.cat([lin(n, p + f"self_attn.{w}") for w in ("q_proj", "k_proj", "v_proj")], -1)
        q = L.rope_kv_append(qkv.reshape(-1, 3 * h).contiguous(), None, B, S, HEADS, D, 0, kc, vc)
        att = L.attention(q.view(B, S, HEADS, D).transpose(1, 2), kc, vc, D ** -0.5, causal=True).view(B, S, h)
        x = lin(att, p + "self_attn.o_proj", residual=x)
        n = L.rmsnorm(x.reshape(-1, h), half(p + "post_attention_layernorm.weight"), eps).view(B, S, h)
        g, u = lin(n, p + "mlp.gate_proj"), lin(n, p + "mlp.up_proj")
        x = lin(R.silu_gate(g.cpu(), u.cpu()).to(dev), p + "mlp.down_proj", residual=x)
    hn = L.rmsnorm(x.reshape(-1, h), half("model.norm.weight"), eps)
    return L.gemm(hn, half("lm_head.weight")).view(B, S, -1)


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


@pytest.mark.parametrize("k,do_sample", [(4, False), (5, False), (4, True), (5, True)])
def test_beams_match_restatement(tmp_path, k, do_sample):
    """beam search / beam sampling of the LoRA model (k = 5 sends the decode step through the GEMM shrink and expand
    inside the captured graph) against tests/beam_ref.py driven by the same model's forward()"""
    from seed_b200.peft import PeftModel

    lm, _ = build(max_batch=10)
    pm = PeftModel.from_pretrained(lm, write(str(tmp_path / "b"), adapter()))
    ids = torch.randint(3, V, (2, 16), generator=torch.Generator().manual_seed(5)).cuda()
    kw = dict(do_sample=do_sample, temperature=0.8 if do_sample else 1.0, top_p=0.7 if do_sample else 1.0,
              length_penalty=1.0, early_stopping=False)
    lm._draws = 0
    free = pm.generate(input_ids=ids, max_new_tokens=12, num_beams=k, eos_token_id=-1, seed=11, **kw)[:, ids.shape[1]:]
    eos = int(free[0, 3])                                   # a token this model emits: hypotheses will finish
    lm._draws = 0
    got = pm.generate(input_ids=ids, max_new_tokens=12, num_beams=k, eos_token_id=eos, pad_token_id=V - 1, seed=11, **kw)
    ref, _, kmin, nmin, _ = beam_ref.beam_generate(_driver(pm, ids, k), ids, 12, k, eos=eos, pad=V - 1, seed=11,
                                                   offset=0, **kw)
    if do_sample and (kmin <= 1e-5 or nmin <= 1e-6):
        pytest.skip(f"a draw sits within 1e-5 of a tie (margin {kmin:.2e} / {nmin:.2e}): not comparable")
    assert torch.equal(got.cpu(), ref), (got.cpu().tolist(), ref.tolist())


def test_resize_and_modules_to_save_eval_body(tmp_path):
    from models.peft_model import get_peft_model_with_resize_embedding

    class Tok:
        def __len__(self):
            return 1234

    save = {"base_model.model.model.embed_tokens.weight": randh(1234, H, seed=5, scale=0.02).float(),
            "base_model.model.lm_head.weight": randh(1234, H, seed=6, scale=0.02).float(),
            "base_model.model.model.norm.weight": torch.ones(H) * 1.5}
    for l in range(NL):
        save[f"base_model.model.model.layers.{l}.input_layernorm.weight"] = torch.ones(H) * 0.9
        save[f"base_model.model.model.layers.{l}.post_attention_layernorm.weight"] = torch.ones(H) * 1.1
    for fmt in ("safetensors", "bin"):
        ad = dict(adapter(), **save)
        path = write(str(tmp_path / fmt), ad, save=("embed_tokens", "lm_head", "input_layernorm",
                                                     "post_attention_layernorm", "norm"), fmt=fmt)
        lm, _ = build()
        model = get_peft_model_with_resize_embedding(lm, model_id=path, tokenizer=Tok()).eval().half().to("cuda")
        assert model.config.vocab_size == 1234
        ids = torch.randint(3, 1234, (1, 16), generator=torch.Generator().manual_seed(4)).cuda()
        assert model(ids).logits.shape == (1, 16, 1234)
        out = model.generate(ids, max_new_tokens=8, num_beams=4, eos_token_id=-1)
        assert out.shape == (1, 24) and int(out.max()) < 1234
        assert model.get_memory_footprint() > lm._weight_bytes


def test_int8_model_refuses_lora():
    from seed_b200 import lib as L

    lm, _ = build()
    lm8 = type(lm)(lm.config, synth.llama_state_dict(H, NL, FFN, V, seed=1), device="cuda", load_in_8bit=True)
    ad = {k.replace("base_model.model.", ""): v.half().cuda() for k, v in adapter().items()}
    with pytest.raises(RuntimeError, match="int8"):
        lm8._llm.lora_load(ad, 16, 32.0)
    with pytest.raises(RuntimeError, match="lora_B"):
        lm._llm.lora_load({k: v for k, v in ad.items() if "layers.1.mlp.up_proj.lora_B" not in k}, 16, 32.0)
    del L
