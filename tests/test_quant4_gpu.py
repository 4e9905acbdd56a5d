"""bitsandbytes 4-bit kernels and the 4-bit LLaMA (load_in_4bit=True) against tests/quant4_ref.py and the fp16 path.

The quantiser and dequantiser are compared bit for bit with the restatement.  The 4-bit GEMV is compared bit for bit
with the fp16 GEMV run on the dequantised weight, and the 4-bit model with an fp16 model holding the dequantised
weights: prefill (dequantise + the fp16 GEMM) and decode (the 4-bit GEMV) are both exact there.
"""
import os
import sys

import pytest
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import quant4_ref as Q  # noqa: E402
from oracle import synth  # noqa: E402

pytestmark = pytest.mark.gpu
SENT = 0x7E5A          # a NaN payload no kernel writes
QTS = [(Q.FP4, "fp4"), (Q.NF4, "nf4")]


def weight(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * torch.rand(N, 1, generator=g) * 0.05
    w[N // 3, :64] = 0.0                                # an all-zero block
    w[N // 2, 0] = -0.0
    if K >= 128:                                        # values exactly on the fp16-exact FP4 pivot, absmax 1
        w[1, 64:128] = 0.0
        w[1, 64], w[1, 65], w[1, 66] = 1.0, 0.0859375, -0.0859375
    return w.half()


def guarded(M, n):
    G = 64
    buf = torch.full((G + M * n + G,), SENT, dtype=torch.int16, device="cuda")
    return buf, buf[G:G + M * n].view(torch.float16).view(M, n), G


def check_guards(buf, G, M, n):
    b = buf.cpu()
    assert torch.all(b[:G] == SENT) and torch.all(b[G + M * n:] == SENT)


def same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.view(torch.int16)[~na], b.view(torch.int16)[~nb])


@pytest.mark.parametrize("qt,name", QTS)
def test_quantise_dequantise_bit_exact(lib, qt, name):
    L = lib
    for N, K in [(3, 64), (300, 4096), (13824, 5120), (5120, 13824)]:
        w = weight(N, K, seed=N + K)
        p, am = L.quantize_4bit(w.cuda(), name)
        rp, ram = Q.quantize(w, qt)
        assert torch.equal(am.cpu(), ram) and torch.equal(p.cpu(), rp), (N, K)
        d = L.dequantize_4bit(p, am, name)
        assert same_bits(d, Q.dequantize(rp, ram, qt)), (N, K)
    # a strided source and a strided destination
    w = weight(64, 512, seed=9).cuda()
    big = torch.zeros(64, 640, dtype=torch.float16, device="cuda")
    big[:, :512] = w
    p, am = L.quantize_4bit(big[:, :512], name)
    p2, am2 = L.quantize_4bit(w, name)
    assert torch.equal(p, p2) and torch.equal(am, am2)
    out = torch.full((64, 520), float("nan"), dtype=torch.float16, device="cuda")
    L.dequantize_4bit(p, am, name, out=out[:, :512])
    assert same_bits(out[:, :512], L.dequantize_4bit(p, am, name)) and torch.isnan(out[:, 512:].float()).all()


CASES = [  # (M, N, K)
    (1, 256, 64), (2, 200, 4096), (3, 513, 4096), (4, 136, 5120), (1, 5120, 13824), (2, 257, 11008), (4, 384, 128),
    (3, 1024, 13824), (1, 13824, 5120),
]


@pytest.mark.parametrize("qt,name", QTS)
@pytest.mark.parametrize("M,N,K", CASES)
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("norm", [False, True])
def test_gemv_4bit_equals_gemv_on_dequantised(lib, qt, name, M, N, K, residual, norm):
    L = lib
    g = torch.Generator().manual_seed(M * 7 + N + K)
    x = (torch.randn(M, K, generator=g)).half().cuda()
    p, am = L.quantize_4bit(weight(N, K, seed=K + N).cuda(), name)
    wd = L.dequantize_4bit(p, am, name)
    r = (torch.randn(M, N, generator=g) * 4).half().cuda() if residual else None
    nw = (torch.rand(K, generator=g) + 0.5).half().cuda() if norm else None
    ref = L.gemv(x, wd, residual=r, norm_w=nw)
    buf, out, G = guarded(M, N)
    L.gemv_4bit(x, p, am, name, residual=r, norm_w=nw, out=out)
    torch.cuda.synchronize()
    check_guards(buf, G, M, N)
    assert same_bits(out, ref), (out.float() - ref.float()).abs().max()
    if not norm and not residual and K <= 4096:       # and within fp16 rounding of the restated linear
        y = Q.linear4(x.cpu(), p.cpu(), am.cpu(), qt).float()
        assert torch.all((out.cpu().float() - y).abs() <= 2.0 ** -9 * y.abs() + 1e-3)


@pytest.mark.parametrize("qt,name", QTS)
@pytest.mark.parametrize("M,N,K", [(1, 512, 4096), (2, 256, 64), (3, 768, 5120), (4, 27648, 5120)])
@pytest.mark.parametrize("norm", [False, True])
def test_gemv_4bit_silu_gate(lib, qt, name, M, N, K, norm):
    L = lib
    g = torch.Generator().manual_seed(N + M)
    x = torch.randn(M, K, generator=g).half().cuda()
    p, am = L.quantize_4bit(weight(N, K, seed=N).cuda(), name)
    nw = (torch.rand(K, generator=g) + 0.5).half().cuda() if norm else None
    ref = L.gemv(x, L.dequantize_4bit(p, am, name), norm_w=nw, mode=1)
    buf, out, G = guarded(M, N // 2)
    L.gemv_4bit(x, p, am, name, norm_w=nw, mode=1, out=out)
    torch.cuda.synchronize()
    check_guards(buf, G, M, N // 2)
    assert same_bits(out, ref)


# ---------------------------------------------------------------------------------------------------------------
# model level
# ---------------------------------------------------------------------------------------------------------------
LINS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


def dequantised(lib, sd, name):
    """the state dict with every decoder linear replaced by W' (quantised and dequantised on the GPU)"""
    out = {}
    for k, v in sd.items():
        if k.endswith(".weight") and ".layers." in k and k.split(".")[-2] in LINS:
            p, am = lib.quantize_4bit(v.half().cuda(), name)
            v = lib.dequantize_4bit(p, am, name).cpu()
        out[k] = v
    return out


def build(lib, name, hidden=512, layers=2, heads=4, ffn=1408, vocab=1056, max_batch=6, max_seq=256):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=vocab, hidden_size=hidden, intermediate_size=ffn, num_hidden_layers=layers,
                      num_attention_heads=heads, num_key_value_heads=heads, rms_norm_eps=1e-6,
                      max_position_embeddings=2048)
    sd = synth.llama_state_dict(hidden, layers, ffn, vocab, seed=1234)
    kw = dict(device="cuda", max_batch=max_batch, max_seq=max_seq)
    m4 = LlamaForCausalLM(cfg, sd, load_in_4bit=True, bnb_4bit_quant_type=name, **kw)
    m16 = LlamaForCausalLM(cfg, dequantised(lib, sd, name), **kw)
    return m4, m16, sd, cfg, kw


@pytest.mark.parametrize("qt,name", QTS)
def test_model_bit_identical_to_fp16_on_dequantised_weights(lib, qt, name):
    from models.llama_xformer import LlamaForCausalLM

    m4, m16, sd, cfg, kw = build(lib, name)
    assert m4.is_loaded_in_4bit and not m4.is_loaded_in_8bit
    ids = torch.randint(0, 1056, (2, 40), generator=torch.Generator().manual_seed(7)).cuda()
    a4 = m4(input_ids=ids, use_cache=True).logits
    a16 = m16(input_ids=ids, use_cache=True).logits
    assert same_bits(a4, a16)
    orig = LlamaForCausalLM(cfg, sd, **kw)
    print(f"{name}: 4-bit logits vs the fp16 model on the original weights: relative error "
          f"{rel(a4, orig(input_ids=ids).logits):.3e}")
    del orig
    # chunked: 24 / 15 / 1 positions (the last is a 2-row decode step through the 4-bit GEMV)
    outs = []
    for m in (m4, m16):
        a = m(input_ids=ids[:, :24], use_cache=True)
        b = m(input_ids=ids[:, 24:39], past_key_values=a.past_key_values, use_cache=True)
        c = m(input_ids=ids[:, 39:], past_key_values=b.past_key_values, use_cache=True)
        outs.append(torch.cat([a.logits, b.logits, c.logits], 1))
    assert same_bits(outs[0], outs[1])
    # batch 6: the cached decode step takes the dequantise + GEMM path
    ids6 = torch.randint(0, 1056, (6, 20), generator=torch.Generator().manual_seed(4)).cuda()
    res = []
    for m in (m4, m16):
        a = m(input_ids=ids6[:, :19], use_cache=True)
        b = m(input_ids=ids6[:, 19:], past_key_values=a.past_key_values, use_cache=True)
        res.append((a.logits, b.logits))
    assert same_bits(res[0][0], res[1][0]) and same_bits(res[0][1], res[1][1])
    # ... and captured in a CUDA graph, it replays bit for bit
    eager = res[0][1].clone()
    m4(input_ids=ids6[:, :19], use_cache=True)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        cap = m4._llm.forward(input_ids=ids6[:, 19:], past_len=19)
    gr.replay()
    torch.cuda.synchronize()
    assert same_bits(cap, eager)


@pytest.mark.parametrize("qt,name", QTS)
def test_generate_and_beam_search(lib, qt, name):
    m4, m16, _, _, _ = build(lib, name, max_batch=2)
    ids = torch.randint(0, 1056, (2, 17), generator=torch.Generator().manual_seed(3)).cuda()
    ref = m16.generate(ids, max_new_tokens=12, device_loop=True, eos_token_id=-1)
    host = m4.generate(ids, max_new_tokens=12, device_loop=False, eos_token_id=-1)
    g = m4.generate(ids, max_new_tokens=12, device_loop=True, use_graph=True, eos_token_id=-1)
    assert m4._llm.used_graph == 1
    e = m4.generate(ids, max_new_tokens=12, device_loop=True, use_graph=False, eos_token_id=-1)
    assert torch.equal(host, ref) and torch.equal(g, ref) and torch.equal(e, ref)
    for k in (4, 5):           # 4 rows: the 4-bit GEMV; 5 rows: dequantise + GEMM in every captured step
        b4 = m4.generate(ids[:1], max_new_tokens=10, num_beams=k, eos_token_id=-1)
        b16 = m16.generate(ids[:1], max_new_tokens=10, num_beams=k, eos_token_id=-1)
        assert torch.equal(b4, b16), k


def test_load_weight_and_lora_refusals(lib):
    m4, _, _, _, _ = build(lib, "nf4", layers=1, max_batch=1)
    with pytest.raises(RuntimeError, match="is not a decoder linear"):
        m4._llm.load_4bit_weight("model.layers.0.self_attn.rotary.weight", torch.zeros(512, 512).half().cuda())
    with pytest.raises(RuntimeError, match="is not a decoder linear"):
        m4._llm.load_4bit_weight("model.layers.3.mlp.up_proj.weight", torch.zeros(1408, 512).half().cuda())
    with pytest.raises(RuntimeError, match="expected shape"):
        m4._llm.load_4bit_weight("model.layers.0.mlp.up_proj.weight", torch.zeros(512, 512).half().cuda())
    with pytest.raises(RuntimeError, match="4-bit"):
        m4._llm.lora_load({"model.layers.0.self_attn.q_proj.lora_A.weight": torch.zeros(8, 512).half().cuda(),
                           "model.layers.0.self_attn.q_proj.lora_B.weight": torch.zeros(512, 8).half().cuda()}, 8, 16)
    # a handle whose linears are not all loaded refuses to run, naming the first missing one
    from seed_b200 import lib as L

    w = {k: v for k, v in m4._llm._weights.items()}
    h = L.Llama(w, hidden=512, layers=1, heads=4, ffn=1408, vocab=1056, max_seq=64, quant4="fp4")
    with pytest.raises(RuntimeError, match="model.layers.0.self_attn.q_proj.weight' has not been loaded"):
        h.forward(input_ids=torch.zeros(1, 4, dtype=torch.int64, device="cuda"))
    h.close()


def test_memory_7b_shape():
    """7B-shaped model, random-init on the device: the 4-bit footprint is <= 0.32x the fp16 model's (4.17 / 13.5 GB
    from the byte counts) and the construction peak stays below 0.4x the fp16 weight bytes"""
    from seed_b200.llama import LlamaForCausalLM

    h, ffn, V, nl = 4096, 11008, 32000, 32
    cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=ffn, num_hidden_layers=nl,
                      num_attention_heads=32, num_key_value_heads=32, rms_norm_eps=1e-6, max_position_embeddings=64)

    def sd_on_device():
        sd = {"model.embed_tokens.weight": torch.randn(V, h, device="cuda", dtype=torch.float16) * 0.02,
              "model.norm.weight": torch.ones(h, device="cuda", dtype=torch.float16),
              "lm_head.weight": torch.randn(V, h, device="cuda", dtype=torch.float16) * 0.02}
        for l in range(nl):
            p = f"model.layers.{l}."
            sd[p + "input_layernorm.weight"] = torch.ones(h, device="cuda", dtype=torch.float16)
            sd[p + "post_attention_layernorm.weight"] = torch.ones(h, device="cuda", dtype=torch.float16)
        return sd

    class Lazy(dict):
        """the linears are made one at a time while the model consumes them; free memory is sampled at each step"""
        lowest = None

        def items(self):
            def gen():
                yield from dict.items(self)
                for l in range(nl):
                    p = f"model.layers.{l}."
                    for nm, shp in (("self_attn.q_proj", (h, h)), ("self_attn.k_proj", (h, h)),
                                    ("self_attn.v_proj", (h, h)), ("self_attn.o_proj", (h, h)),
                                    ("mlp.gate_proj", (ffn, h)), ("mlp.up_proj", (ffn, h)),
                                    ("mlp.down_proj", (h, ffn))):
                        yield p + nm + ".weight", torch.randn(*shp, device="cuda", dtype=torch.float16) * 0.02
            for k, v in gen():
                torch.cuda.synchronize()
                f = torch.cuda.mem_get_info()[0]
                Lazy.lowest = f if Lazy.lowest is None else min(Lazy.lowest, f)
                yield k, v

    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    m4 = LlamaForCausalLM(cfg, Lazy(sd_on_device()), device="cuda", max_seq=64, load_in_4bit=True,
                          bnb_4bit_quant_type="nf4")
    torch.cuda.synchronize()
    peak4 = free0 - Lazy.lowest
    assert m4.is_loaded_in_4bit
    fp4 = m4.get_memory_footprint()
    del m4
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    m16 = LlamaForCausalLM(cfg, dict(Lazy(sd_on_device()).items()), device="cuda", max_seq=64)
    fp16 = m16.get_memory_footprint()
    del m16
    print(f"footprint nf4 {fp4 / 2**30:.2f} GiB fp16 {fp16 / 2**30:.2f} GiB ({fp4 / fp16:.3f}x); peak device bytes "
          f"during 4-bit construction {peak4 / 2**30:.2f} GiB ({peak4 / fp16:.3f}x the fp16 weights)")
    assert fp4 <= 0.32 * fp16
    assert peak4 < 0.4 * fp16, (peak4, fp16)
