"""One small launch of every kernel family through the C ABI, for compute-sanitizer (SURVEY.md section 5):

    compute-sanitizer --tool memcheck  --error-exitcode 1 python tests/sanitize_driver.py
    compute-sanitizer --tool racecheck --error-exitcode 1 python tests/sanitize_driver.py
    compute-sanitizer --tool synccheck --error-exitcode 1 python tests/sanitize_driver.py
    compute-sanitizer --tool initcheck --error-exitcode 1 python tests/sanitize_driver.py

Shapes are the smallest that still walk every code path (pipeline wrap-around, ragged tail tile, K below one k-block,
strided operand views, every head_dim variant of the attention kernel, split-KV decode attention, top-p sampler); each
result is also compared with the per-op oracle so a sanitizer-clean run is known to have computed the right thing.
`--only name` runs one family.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from oracle import ops_ref as R
from seed_b200 import lib as L

DEV = "cuda"


def r16(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half().to(DEV)


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def gemm():
    for (M, N, K, bn, ctas) in [(300, 256, 1408, 256, 1), (512, 512, 1408, 256, 2), (520, 1408, 768, 256, 2),
                                (200, 272, 256, 256, 1), (96, 96, 768, 64, 1)]:
        a, w, b = r16(M, K, seed=1), r16(N, K, scale=K ** -0.5, seed=2), r16(N, seed=3)
        res = r16(M, N, seed=4)
        out = L.gemm(a, w, bias=b, act=L.ACT_GELU, residual=res, bn=bn, ctas=ctas)
        assert rel(out, R.linear_ref(a, w, b, 1, res)) < 2e-3, (M, N, K)
    # K below one k-block (the encoder's K = 32 linears), on views into wider buffers with trailing rows: lda, ldw, ldr
    # and ldo all above the logical widths
    for (M, N, K, bn) in [(65, 40, 8, 64), (129, 200, 24, 176), (64, 768, 32, 256), (1, 33, 32, 32)]:
        a = r16(M + 3, K + 16, seed=5)[:M, :K]
        w = r16(N + 5, K + 8, scale=K ** -0.5, seed=6)[:N, :K]
        res = r16(M + 1, N + 24, seed=7)[:M, :N]
        obuf = torch.zeros((M + 2, N + 40), dtype=torch.float16, device=DEV)
        out = L.gemm(a, w, act=L.ACT_RELU, residual=res, out=obuf[:M, :N], bn=bn)
        assert rel(out, R.linear_ref(a, w, None, 3, res)) < 2e-3, (M, N, K)
        assert (obuf[M:] == 0).all() and (obuf[:, N:] == 0).all()
    # staged epilogue with TMA residual boxes, in place, leaving the row moments (the encoder's proj / fc2 calls)
    a, w, b = r16(520, 768, seed=1), r16(1408, 768, scale=768 ** -0.5, seed=2), r16(1408, seed=3)
    x = r16(520, 1408, seed=4)
    want = R.linear_ref(a, w, b, 0, x)
    mom = torch.empty((520, 1408 // 64, 2), dtype=torch.float32, device=DEV)
    out = L.gemm(a, w, bias=b, residual=x, out=x, ctas=2, row_moments=mom)
    assert rel(out, want) < 2e-3
    st = L.row_stats_from_moments(mom, 1408, 1e-6)
    assert torch.allclose(st, L.row_stats(out, 1e-6), rtol=1e-4, atol=1e-4)
    a = r16(300, 512, seed=5)
    wg, wu = r16(1408, 512, scale=0.04, seed=6), r16(1408, 512, scale=0.04, seed=7)
    out = L.gemm(a, R.interleave_gate_up(wg, wu), mode=1, ctas=2)
    assert rel(out, R.silu_gate_ref(a, wg, wu)) < 3e-3


def attention():
    for (B, H, Nq, Nk, D, causal) in [(2, 16, 257, 257, 88, False),      # ViT shape
                                      (1, 4, 300, 300, 128, True),        # causal, ragged tiles
                                      (1, 4, 128, 428, 128, True),        # ... with a past
                                      (2, 12, 32, 32, 64, True),          # mma.sync kernel: Q-Former self
                                      (2, 12, 32, 257, 64, False),        # Q-Former cross
                                      (2, 3, 40, 100, 88, True),          # head_dim 88, short query tile <96,4>
                                      (1, 2, 300, 64, 88, False)]:        # head_dim 88, nq > 288, nq > nk
        q, k, v = r16(B, H, Nq, D, seed=11), r16(B, H, Nk, D, seed=12), r16(B, H, Nk, D, seed=13)
        out = L.attention(q, k, v, D ** -0.5, causal)
        assert rel(out, R.attention_ref(q, k, v, D ** -0.5, causal)) < 3e-3, (B, H, Nq, Nk, D, causal)
    # the ViT shape on the packed projection buffer: Q / K / V by TMA, O by TMA store (what the encoder launches)
    B, H, N, D = 2, 16, 257, 88
    qkv = r16(B * N, 3 * H * D, seed=14)
    q, k, v = (qkv.view(B, N, 3, H, D)[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    out = L.attention(q, k, v, D ** -0.5, False)
    assert rel(out, R.attention_ref(q, k, v, D ** -0.5, False)) < 3e-3


def rowwise():
    x, w, b = r16(300, 1408, seed=21), r16(1408, seed=22), r16(1408, seed=23)
    assert rel(L.layernorm(x, w, b, 1e-6), R.layernorm_ref(x, w, b, 1e-6)) < 1e-3
    x, w = r16(5, 5120, seed=24), r16(5120, seed=25)
    assert rel(L.rmsnorm(x, w, 1e-6), R.rmsnorm_ref(x, w, 1e-6)) < 1e-3
    img = r16(2, 3, 224, 224, seed=26)
    assert torch.equal(L.patchify(img), R.patchify_ref(img))
    table, ids = r16(100, 64, seed=27), torch.randint(0, 100, (7,), device=DEV)
    assert torch.equal(L.embedding(table, ids), table[ids])
    B, S, H, D, past, ms = 2, 17, 3, 128, 5, 64
    qkv = r16(B * S, 3 * H * D, seed=28)
    kc, vc = torch.zeros(B, H, ms, D, dtype=torch.float16, device=DEV), torch.zeros(B, H, ms, D, dtype=torch.float16, device=DEV)
    L.rope_kv_append(qkv, None, B, S, H, D, past, kc, vc)


def vq():
    z, cb = r16(100, 32, scale=0.26, seed=31), r16(8192, 32, scale=0.28, seed=32)
    ids = L.vq_argmin(z, cb, L.VQ_FP32)
    ref, _ = R.vq_torch_ref(z.float(), cb.float())
    assert (ids == ref).float().mean().item() > 0.97
    L.vq_argmin(z, cb, L.VQ_FP16)


def decode():
    x, w = r16(1, 5120, seed=41), r16(1000, 5120, scale=5120 ** -0.5, seed=42)
    nw = r16(5120, seed=43)
    assert rel(L.gemv(x, w, norm_w=nw), R.linear_ref(R.rmsnorm_ref(x, nw, 1e-6), w)) < 2e-3
    wg, wu = r16(256, 512, scale=0.04, seed=44), r16(256, 512, scale=0.04, seed=45)
    x2 = r16(2, 512, seed=46)
    assert rel(L.gemv(x2, R.interleave_gate_up(wg, wu), mode=1), R.silu_gate_ref(x2, wg, wu)) < 3e-3
    B, H, D, kv, ms = 1, 8, 128, 300, 392
    q, kc, vc = r16(B, H, D, seed=47), r16(B, H, ms, D, seed=48), r16(B, H, ms, D, seed=49)
    out = L.decode_attention(q, kc, vc, kv, D ** -0.5)
    ref = R.attention_ref(q[:, :, None], kc[:, :, :kv], vc[:, :, :kv], D ** -0.5)
    assert rel(out.view(B, H, D), ref.view(B, H, D)) < 3e-3
    # fused RoPE + append + attention (three thread groups; the new key / value come from shared memory)
    qkv = r16(B, 3 * H * D, seed=51)
    kc2, vc2 = kc.clone(), vc.clone()
    q_rot = L.rope_kv_append(qkv, None, B, 1, H, D, kv, kc, vc)
    two = L.decode_attention(q_rot.view(B, H, D), kc, vc, kv + 1, D ** -0.5)
    one = L.decode_attention_rope(qkv, None, H, kv, kc2, vc2, D ** -0.5)
    assert torch.equal(one, two) and torch.equal(kc, kc2) and torch.equal(vc, vc2)
    logits = r16(4, 5000, scale=3.0, seed=50)
    L.sample(logits)
    L.sample(logits, do_sample=True, temperature=0.9, top_p=0.5, seed=1, offset=2, step=3)
    ids = torch.randint(0, 8192, (3, 32), device=DEV)
    L.image_ids_to_tokens(ids, 32000, 40192, 40193)


def models():
    """depth-1 encoder + 2-layer LLaMA through the handle-level entries, incl. the graph-replayed generate loop"""
    from transformers.models.llama.configuration_llama import LlamaConfig

    from models.llama_xformer import LlamaForCausalLM
    from models.seed_qformer.qformer_quantizer import Blip2QformerQuantizer
    from seed_b200 import synth

    enc = Blip2QformerQuantizer(synth.encoder_state_dict(1, 1, 1), device=DEV, max_batch=2)
    ids = enc.encode_ids(synth.images(2).to(DEV))
    enc.get_codebook_entry(ids)
    enc.encode_tokens(synth.images(2).to(DEV), 32000, 40192, 40193)
    h, nl, nh, ffn, V = 512, 2, 4, 1408, 1056
    cfg = LlamaConfig(vocab_size=V, hidden_size=h, intermediate_size=ffn, num_hidden_layers=nl, num_attention_heads=nh,
                      num_key_value_heads=nh, rms_norm_eps=1e-6)
    llm = LlamaForCausalLM(cfg, synth.llama_state_dict(h, nl, ffn, V), device=DEV, max_batch=1, max_seq=96)
    p = synth.prompt_ids(1, 40, 1, text_vocab=V - 66, n_codes=64).to(DEV)
    llm(input_ids=p)
    llm.generate(input_ids=p, max_new_tokens=6, do_sample=True, top_p=0.5, seed=3, eos_token_id=-1)
    llm.generate(input_ids=p, max_new_tokens=6, do_sample=False, eos_token_id=-1, use_graph=False)


def preprocess():
    u8 = torch.randint(0, 256, (2, 97, 131, 3), dtype=torch.uint8, device=DEV)
    L.Preprocess(97, 131, 224, "bicubic", max_batch=2)(u8)
    L.Preprocess(97, 131, 224, "bilinear", max_batch=2, resize=(224, 302), crop=(0, 39))(u8)


FAMILIES = {"gemm": gemm, "attention": attention, "rowwise": rowwise, "vq": vq, "decode": decode, "models": models,
            "preprocess": preprocess}

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", nargs="*", default=None)
    a = ap.parse_args()
    for name, fn in FAMILIES.items():
        if a.only and name not in a.only:
            continue
        fn()
        torch.cuda.synchronize()
        print(f"{name}: ok ({L.launch_count()} launches so far)", flush=True)
