"""LLM.int8() kernels and the int8 LLaMA against the restatement in tests/int8_ref.py.

Quantisers, the int8 GEMM and the int8 GEMV are compared bit for bit (integer accumulation, elementwise
dequantisation, the outlier correction summed in ascending column order).  The SiLU-gate output is compared bit
for bit between the GEMM and the GEMV, and against the oracle within one fp16 rounding of silu(gate): the kernels
use the ex2/rcp approximations of the fp16 GEMM's SiLU epilogue.
"""
import os
import sys

import pytest
import torch
from transformers.models.llama.configuration_llama import LlamaConfig

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import int8_ref as Q  # noqa: E402
from oracle import synth  # noqa: E402

pytestmark = pytest.mark.gpu
SENT = 0x7E5A          # a NaN payload no kernel writes


def act(M, K, n_out, seed, nan_row=None):
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * 1.5).clamp(-5.5, 5.5)
    cols = torch.randperm(K, generator=g)[:n_out].tolist()
    for i, c in enumerate(cols):
        a[(i * 7919) % M, c] = (8.0 + (i % 50)) * (-1 if i % 2 else 1)
    if M > 2:
        a[M // 2] = 0.0                                # a zero row
    if n_out >= 7 and nan_row is None:
        a[0, cols[1]] = float("inf")
        a[M - 1, cols[2]] = -float("inf")
    if nan_row is not None:
        a[nan_row, cols[0] if cols else 0] = float("nan")
    return a.half()


def weight(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g) * torch.rand(N, 1, generator=g) * 0.05
    w[N // 3] = 0.0                                     # SCB == 0 row
    return w.half()


def guarded(M, n):
    """an [M, n] fp16 output inside a buffer whose guard words must keep their bits"""
    G = 64
    buf = torch.full((G + M * n + G,), SENT, dtype=torch.int16, device="cuda")
    return buf, buf[G:G + M * n].view(torch.float16).view(M, n), G


def check_guards(buf, G, M, n):
    b = buf.cpu()
    assert torch.all(b[:G] == SENT) and torch.all(b[G + M * n:] == SENT)


def same_bits(a, b):
    """identical fp16 bits, any NaN matching any NaN (payloads are not part of the contract)"""
    a, b = a.cpu(), b.cpu()
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a.view(torch.int16)[~na], b.view(torch.int16)[~nb])


def test_quantisers_bit_exact(lib):
    L = lib
    for (M, K, n_out) in [(1, 128, 0), (5, 4096, 7), (257, 11008, 300), (64, 4096, 1)]:
        a = act(M, K, n_out, seed=M + K)
        ca, sca, ol, n = L.int8_quantize_act(a.cuda())
        rca, rsca, rO = Q.quantize_act(a)
        assert int(n.item()) == rO.numel()
        assert torch.equal(ol[:rO.numel()].cpu().long(), rO)
        assert torch.equal(sca.cpu(), rsca) and torch.equal(ca.cpu(), rca)
    w = weight(300, 4096, 5)
    w[7, 9] = 60000.0
    cb, scb = L.int8_quantize_weight(w.cuda())
    rcb, rscb = Q.quantize_weight(w)
    assert torch.equal(cb.cpu(), rcb) and torch.equal(scb.cpu(), rscb)


CASES = [  # (M, N, K, |O|, bn)
    (1, 256, 128, 0, 0), (2, 200, 4096, 1, 0), (3, 384, 128, 7, 0), (4, 136, 4096, 300, 0),
    (5, 256, 4096, 7, 256), (64, 200, 128, 1, 128), (257, 136, 4096, 0, 64), (2048, 256, 11008, 300, 0),
    (257, 264, 11008, 7, 128), (64, 512, 4096, 300, 256), (1, 264, 11008, 1, 0), (4, 256, 11008, 0, 0),
]


@pytest.mark.parametrize("M,N,K,n_out,bn", CASES)
@pytest.mark.parametrize("residual", [False, True])
def test_linear_bit_exact(lib, M, N, K, n_out, bn, residual):
    L = lib
    nan = M > 1 and n_out > 0
    a = act(M, K, n_out, seed=M * 31 + K + n_out, nan_row=M - 1 if nan else None)
    cb, scb = Q.quantize_weight(weight(N, K, seed=N + K))
    r = (torch.randn(M, N, generator=torch.Generator().manual_seed(2)) * 4).half() if residual else None
    ref = Q.linear8(a, cb, scb, residual=r)
    buf, out, G = guarded(M, N)
    args = dict(residual=None if r is None else r.cuda(), out=out)
    if M <= 4:
        L.gemv_int8(a.cuda(), cb.cuda(), scb.cuda(), **args)
    else:
        L.gemm_int8(a.cuda(), cb.cuda(), scb.cuda(), bn=bn, **args)
    torch.cuda.synchronize()
    check_guards(buf, G, M, N)
    assert same_bits(out, ref), (out.cpu().float() - ref.float()).abs().nan_to_num(1e9).max()
    if nan:   # the NaN reaches exactly its own row
        o = out.cpu().float()
        assert torch.isnan(o[M - 1]).all() and not torch.isnan(o[:M - 1]).any()
    if M <= 4 and bn == 0:   # the GEMM on the same rows gives the same bits
        out2 = L.gemm_int8(a.cuda(), cb.cuda(), scb.cuda(), residual=args["residual"])
        assert same_bits(out2, out)


@pytest.mark.parametrize("M,K,n_out", [(1, 4096, 0), (3, 128, 7), (4, 11008, 300), (5, 4096, 1), (257, 128, 7)])
def test_silu_gate(lib, M, K, n_out):
    L = lib
    N = 512
    a = act(M, K, n_out, seed=K + M)
    cb, scb = Q.quantize_weight(weight(N, K, seed=K))
    y = Q.linear8_parts(a, cb, scb)                       # fp16 gate / up values, bit-exact contract
    ref = Q.silu_gate(y)
    out = L.gemm_int8(a.cuda(), cb.cuda(), scb.cuda(), mode=1)
    if M <= 4:
        buf, o2, G = guarded(M, N // 2)
        L.gemv_int8(a.cuda(), cb.cuda(), scb.cuda(), mode=1, out=o2)
        torch.cuda.synchronize()
        check_guards(buf, G, M, N // 2)
        assert same_bits(o2, out)
    out = out.cpu().float()
    tol = Q.silu_gate_tol(y, ref)
    rf = ref.float()
    assert torch.equal(torch.isnan(out), torch.isnan(rf)) and torch.equal(torch.isinf(out), torch.isinf(rf))
    fin = torch.isfinite(rf)
    assert torch.all((out - rf).abs()[fin] <= tol[fin])


def test_gemv_rmsnorm_staging_matches_gemv(lib):
    """norm_w: the int8 GEMV normalises exactly as the fp16 GEMV stages its rows"""
    L = lib
    M, K, N = 2, 4096, 256
    x = act(M, K, 0, seed=3).cuda()
    w = (torch.rand(K) + 0.5).half().cuda()
    w[11] = 40.0                                        # this channel crosses the threshold after the norm
    cb, scb = Q.quantize_weight(weight(N, K, seed=4))
    y = L.gemv_int8(x, cb.cuda(), scb.cuda(), norm_w=w, eps=1e-6)
    ident = torch.eye(K, dtype=torch.float16, device="cuda")
    n = L.gemv(x, ident, norm_w=w, eps=1e-6)            # the fp16 GEMV's staged rows, via an identity weight
    assert same_bits(y, Q.linear8(n.cpu(), cb, scb))


# ---------------------------------------------------------------------------------------------------------------
# model level
# ---------------------------------------------------------------------------------------------------------------
def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


def build(hidden, layers, heads, ffn, vocab, max_batch=2, max_seq=256, int8=True, seed=1234, hot=True):
    from models.llama_xformer import LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=vocab, hidden_size=hidden, intermediate_size=ffn, num_hidden_layers=layers,
                      num_attention_heads=heads, num_key_value_heads=heads, rms_norm_eps=1e-6,
                      max_position_embeddings=2048)
    sd = synth.llama_state_dict(hidden, layers, ffn, vocab, seed=seed)
    if hot:   # one input_layernorm channel scaled so that it crosses the outlier threshold
        sd["model.layers.0.input_layernorm.weight"] = sd["model.layers.0.input_layernorm.weight"].clone()
        sd["model.layers.0.input_layernorm.weight"][5] *= 40.0
    return LlamaForCausalLM(cfg, sd, device="cuda", max_batch=max_batch, max_seq=max_seq, load_in_8bit=int8), sd


LINS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def composed(L, sd, ids, heads, layers, chunks, eps=1e-6):
    """The int8 forward with the oracle's linears (int8_ref.linear8, computed on the CPU) between the GPU's own
    embedding, RMSNorm, RoPE + KV append, attention and lm_head kernels.  `chunks` = the sequence positions of each
    forward call: activation quantisation is per call, so each call's rows are quantised together, as the model does.
    The SiLU-gate of the MLP uses the int8 GEMM in mode 1, whose linear part matches the oracle bit for bit
    (test_silu_gate).  Attention runs once over the whole sequence."""
    B, S = ids.shape
    h = sd["model.embed_tokens.weight"].shape[1]
    D = h // heads
    dev = "cuda"
    q8 = {}
    for k, v in sd.items():
        if k.endswith(".weight") and ".layers." in k and k.split(".")[-2] in LINS:
            q8[k] = Q.quantize_weight(v.half())

    def lin(t, name, residual=None):      # t [B, S, K] on the GPU: one oracle call per chunk of positions
        cb, scb = q8[name]
        out = []
        for s0, s1 in chunks:
            rows = t[:, s0:s1].reshape(-1, t.shape[-1]).cpu()
            r = None if residual is None else residual[:, s0:s1].reshape(-1, residual.shape[-1]).cpu()
            out.append(Q.linear8(rows, cb, scb, residual=r).view(B, s1 - s0, -1))
        return torch.cat(out, 1).to(dev)

    def silu_gate(t, p):
        g, u = (q8[p + "mlp.gate_proj.weight"], q8[p + "mlp.up_proj.weight"])
        cb = Q.interleave_gate_up(g[0], u[0]).to(dev)
        scb = Q.interleave_gate_up(g[1], u[1]).to(dev)
        out = [L.gemm_int8(t[:, s0:s1].reshape(-1, t.shape[-1]).contiguous(), cb, scb, mode=1).view(B, s1 - s0, -1)
               if B * (s1 - s0) > 4 else
               L.gemv_int8(t[:, s0:s1].reshape(-1, t.shape[-1]).contiguous(), cb, scb, mode=1).view(B, s1 - s0, -1)
               for s0, s1 in chunks]
        return torch.cat(out, 1)

    def half(k):
        return sd[k].half().to(dev)

    x = L.embedding(half("model.embed_tokens.weight"), ids.to(dev).reshape(-1)).view(B, S, h)
    kc = torch.zeros(B, heads, S, D, dtype=torch.float16, device=dev)
    vc = torch.zeros_like(kc)
    for l in range(layers):
        p = f"model.layers.{l}."
        n = L.rmsnorm(x.reshape(-1, h), half(p + "input_layernorm.weight"), eps).view(B, S, h)
        qkv = torch.cat([lin(n, p + f"self_attn.{w}.weight") for w in ("q_proj", "k_proj", "v_proj")], -1)
        q = L.rope_kv_append(qkv.reshape(-1, 3 * h).contiguous(), None, B, S, heads, D, 0, kc, vc)
        a = L.attention(q.view(B, S, heads, D).transpose(1, 2), kc, vc, D ** -0.5, causal=True).view(B, S, h)
        x = lin(a, p + "self_attn.o_proj.weight", residual=x)
        n = L.rmsnorm(x.reshape(-1, h), half(p + "post_attention_layernorm.weight"), eps).view(B, S, h)
        x = lin(silu_gate(n, p), p + "mlp.down_proj.weight", residual=x)
    hn = L.rmsnorm(x.reshape(-1, h), half("model.norm.weight"), eps)
    return L.gemm(hn, half("lm_head.weight")).view(B, S, -1)


@pytest.mark.parametrize("shape", [(512, 2, 4, 1408, 1056), (1024, 3, 8, 2816, 1056)])
def test_model_against_int8_oracle(lib, shape):
    """The handle against the oracle's linears fed the GPU's own attention and norm outputs (relative Frobenius
    error <= 1e-2, the fp16 path's bound), whole and in chunks; the plain restated int8 forward is reported."""
    hidden, layers, heads, ffn, vocab = shape
    m8, sd = build(*shape)
    m16, _ = build(*shape, int8=False)
    ids = torch.randint(0, vocab, (2, 40), generator=torch.Generator().manual_seed(7))
    counts = []
    ref = Q.llama_forward8(sd, ids, heads, layers, outlier_counts=counts)
    assert counts[0] > 0, counts                       # the hot channel makes outliers in layer 0
    out = m8(input_ids=ids.cuda(), use_cache=True)
    tf = composed(lib, sd, ids, heads, layers, [(0, 40)])
    err = rel(out.logits, tf)
    l16 = m16(input_ids=ids.cuda()).logits
    print(f"int8 vs composed oracle {err:.3e} (max abs {(out.logits.float() - tf.float()).abs().max().item():.3e}); "
          f"vs restated int8 forward {rel(out.logits, ref):.3e}; vs fp16 model {rel(out.logits, l16):.3e}; "
          f"restated int8 vs fp16 model {rel(ref, l16):.3e}; |O| of the q/k/v input per layer {counts}")
    assert err <= 1e-2, err
    # chunked prefill and a cached decode step (three calls: 24, 15 and 1 positions) against the same chunking
    a = m8(input_ids=ids[:, :24].cuda(), use_cache=True)
    b = m8(input_ids=ids[:, 24:39].cuda(), past_key_values=a.past_key_values, use_cache=True)
    c = m8(input_ids=ids[:, 39:].cuda(), past_key_values=b.past_key_values, use_cache=True)
    tfc = composed(lib, sd, ids, heads, layers, [(0, 24), (24, 39), (39, 40)])
    got = torch.cat([a.logits, b.logits, c.logits], 1)
    print(f"chunked vs composed oracle {rel(got, tfc):.3e}")
    assert rel(got, tfc) <= 1e-2


def test_generate_device_loop_and_batch6(lib):
    m8, sd = build(512, 2, 4, 1408, 1056, max_batch=6)
    ids = torch.randint(0, 1056, (2, 17), generator=torch.Generator().manual_seed(3)).cuda()
    host = m8.generate(ids, max_new_tokens=12, device_loop=False, eos_token_id=-1)
    g = m8.generate(ids, max_new_tokens=12, device_loop=True, use_graph=True, eos_token_id=-1)
    assert m8._llm.used_graph == 1
    e = m8.generate(ids, max_new_tokens=12, device_loop=True, use_graph=False, eos_token_id=-1)
    assert torch.equal(host, g) and torch.equal(host, e)
    # B = 6: the cached decode step has 6 rows and goes through activation quantisation + the int8 wgmma GEMM
    ids6 = torch.randint(0, 1056, (6, 20), generator=torch.Generator().manual_seed(4))
    a = m8(input_ids=ids6[:, :19].cuda(), use_cache=True)
    b = m8(input_ids=ids6[:, 19:].cuda(), past_key_values=a.past_key_values, use_cache=True)
    tf = composed(lib, sd, ids6, 4, 2, [(0, 19), (19, 20)])
    got = torch.cat([a.logits, b.logits], 1)
    print(f"B=6 chunked vs composed oracle {rel(got, tf):.3e}")
    assert rel(got, tf) <= 1e-2
    # ... and it can be captured in a CUDA graph (quantiser memset + kernels, correction, GEMM) and replayed
    eager = b.logits.clone()
    gr = torch.cuda.CUDAGraph()
    step = ids6[:, 19:].cuda()
    with torch.cuda.graph(gr):
        cap = m8._llm.forward(input_ids=step, past_len=19)
    gr.replay()
    torch.cuda.synchronize()
    assert same_bits(cap, eager)


def test_load_weight_refuses_a_wrong_shape(lib):
    """the handle quantises the [N, K] rows the linear's name implies: a tensor of another shape is refused"""
    m8, _ = build(512, 1, 4, 1408, 1056, max_batch=1, hot=False)
    with pytest.raises(RuntimeError, match=r"expected shape \[1408, 512\]"):
        m8._llm.int8_load_weight("model.layers.0.mlp.up_proj.weight", torch.zeros(1407, 512).half().cuda())


def test_memory_7b_shape():
    """7B-shaped model, random-init on the device: int8 needs <= 0.56x the fp16 model's weight bytes"""
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

    def lazy_linears(sd):
        """the linears are made one at a time while the model consumes them (random init on the device)"""
        class SD(dict):
            def items(self):
                yield from dict.items(self)
                for l in range(nl):
                    p = f"model.layers.{l}."
                    for nm, shp in (("self_attn.q_proj", (h, h)), ("self_attn.k_proj", (h, h)),
                                    ("self_attn.v_proj", (h, h)), ("self_attn.o_proj", (h, h)),
                                    ("mlp.gate_proj", (ffn, h)), ("mlp.up_proj", (ffn, h)),
                                    ("mlp.down_proj", (h, ffn))):
                        yield p + nm + ".weight", torch.randn(*shp, device="cuda", dtype=torch.float16) * 0.02
        return SD(sd)

    lowest = [None]

    def sampled(sd):
        """the device's free memory after every tensor is made, i.e. at each construction step's peak"""
        class SD(dict):
            def items(self):
                for k, v in sd.items():
                    torch.cuda.synchronize()
                    f = torch.cuda.mem_get_info()[0]
                    lowest[0] = f if lowest[0] is None else min(lowest[0], f)
                    yield k, v
        return SD(sd)

    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    m8 = LlamaForCausalLM(cfg, sampled(lazy_linears(sd_on_device())), device="cuda", max_seq=64, load_in_8bit=True)
    torch.cuda.synchronize()
    peak8 = free0 - lowest[0]
    torch.cuda.empty_cache()
    dev8 = free0 - torch.cuda.mem_get_info()[0]
    fp8 = m8.get_memory_footprint()
    del m8
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free1 = torch.cuda.mem_get_info()[0]
    m16 = LlamaForCausalLM(cfg, dict(lazy_linears(sd_on_device()).items()), device="cuda", max_seq=64)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    dev16 = free1 - torch.cuda.mem_get_info()[0]
    fp16 = m16.get_memory_footprint()
    del m16
    print(f"footprint int8 {fp8 / 2**30:.2f} GiB fp16 {fp16 / 2**30:.2f} GiB; device bytes int8 {dev8 / 2**30:.2f} "
          f"fp16 {dev16 / 2**30:.2f} GiB; peak device bytes during int8 construction {peak8 / 2**30:.2f} GiB")
    # device bytes (cudaMemGetInfo: the handle's own allocations included; KV cache and workspaces are small here)
    assert fp8 <= 0.56 * fp16
    assert dev8 <= 0.56 * dev16, (dev8, dev16)
    assert peak8 < fp16, (peak8, fp16)
