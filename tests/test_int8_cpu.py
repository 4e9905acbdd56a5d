"""LLM.int8() oracle properties (tests/int8_ref.py) and the int8 C ABI surface, without a GPU."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import int8_ref as Q  # noqa: E402


def _act(M, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(M, K, generator=g) * 1.5).clamp(-5.5, 5.5).half()


def test_weight_roundtrip_error_is_at_most_half_a_step():
    g = torch.Generator().manual_seed(1)
    w = (torch.randn(96, 320, generator=g) * torch.rand(96, 1, generator=g) * 3).half()
    w[5] = 0
    cb, scb = Q.quantize_weight(w)
    assert cb.dtype == torch.int8 and scb.dtype == torch.float32
    assert int(cb.abs().max()) <= 127 and torch.all(cb[5] == 0) and scb[5] == 0
    err = (cb.double() * scb.double()[:, None] / 127 - w.double()).abs()
    assert torch.all(err <= scb.double()[:, None] / 254 * (1 + 1e-6))


def test_outlier_set_is_exactly_the_threshold_columns():
    a = _act(9, 256)
    hot = {3: 6.0, 17: -7.5, 100: float("nan"), 200: float("inf"), 201: -float("inf")}
    for r, (c, v) in enumerate(hot.items()):
        a[r, c] = v
    a[4, 50] = 5.99                                  # just below the threshold: not an outlier
    ca, sca, O = Q.quantize_act(a, 6.0)
    assert O.tolist() == sorted(hot)
    assert torch.all(ca[:, O] == 0)
    assert torch.isfinite(sca).all()
    nonout = a.float().abs().masked_fill(~(a.float().abs() < 6.0), 0).amax(1)
    assert torch.equal(sca, nonout)


def test_zero_and_all_outlier_rows_give_zero_without_nan():
    a = _act(4, 128)
    a[1] = 0
    a[2] = 9.0                                       # every column an outlier
    ca, sca, O = Q.quantize_act(a, 6.0)
    assert O.numel() == 128 and torch.all(ca == 0)
    cb, scb = Q.quantize_weight(_act(64, 128, seed=3))
    y = Q.linear8(a, cb, scb)
    assert torch.isfinite(y.float()).all()
    a = _act(4, 128)
    a[1] = 0
    y = Q.linear8(a, cb, scb)
    assert torch.all(y[1] == 0)


@pytest.mark.parametrize("n_out", [0, 1, 7])
def test_linear8_against_float64_of_the_same_integers(n_out):
    M, K, N = 6, 384, 80
    a = _act(M, K, seed=n_out)
    cols = torch.randperm(K, generator=torch.Generator().manual_seed(9))[:n_out]
    for i, c in enumerate(cols.tolist()):
        a[i % M, c] = 8.0 + i
    cb, scb = Q.quantize_weight(_act(N, K, seed=11))
    ca, sca, O = Q.quantize_act(a)
    assert O.numel() == n_out
    ref = (ca.double() @ cb.double().t()) * sca.double()[:, None] * scb.double()[None, :] / (127.0 * 127.0)
    if n_out:
        sub = (cb[:, O].double() * scb.double()[:, None] / 127.0)
        ref = ref + a[:, O].double() @ sub.t()
    y = Q.linear8(a, cb, scb).double()
    # three fp16 roundings (base, corr, sum) and fp16 rounding of subB
    tol = 3 * 2.0 ** -11 * (ref.abs() + (a[:, O].double().abs() @ sub.abs().t() if n_out else 0)) + 1e-6
    assert torch.all((y - ref).abs() <= tol)


def _lib():
    from seed_b200 import lib as L

    if not os.path.exists(L.LIB_PATH):
        pytest.skip("libseedb200.so not built")
    return L


def test_int8_symbols_resolve():
    L = _lib()
    h = L.load()
    for sym in ("seedb200_int8_quantize_weight", "seedb200_int8_quantize_act", "seedb200_gemm_int8",
                "seedb200_gemv_int8", "seedb200_llama_create_int8"):
        assert sym in L.EXPORTS and hasattr(h, sym)


def _cfg(L):
    return L.LlamaConfig(256, 1, 2, 128, 256, 64, 1, 32, 1e-6, 10000.0, 0)


def _create(L, tensors, threshold=6.0):
    arr = (L.Tensor * len(tensors))()
    keep = []
    for i, (name, dtype, shape) in enumerate(tensors):
        b = name.encode()
        keep.append(b)
        arr[i].name = b
        arr[i].data = 4096 * (i + 1)        # never dereferenced: validation fails first
        arr[i].dtype = dtype
        arr[i].ndim = len(shape)
        for j in range(4):
            arr[i].shape[j] = shape[j] if j < len(shape) else 1
    h = C.c_void_p()
    cfg = _cfg(L)
    st = L.load().seedb200_llama_create_int8(C.byref(cfg), arr, len(tensors), threshold, C.byref(h))
    return st, L.load().seedb200_last_error().decode()


def _tensors(L, h=256, ffn=256, V=64):
    t = [("model.embed_tokens.weight", L.DTYPE_F16, (V, h)), ("model.norm.weight", L.DTYPE_F16, (h,)),
         ("lm_head.weight", L.DTYPE_F16, (V, h)),
         ("model.layers.0.input_layernorm.weight", L.DTYPE_F16, (h,)),
         ("model.layers.0.post_attention_layernorm.weight", L.DTYPE_F16, (h,))]
    for nm, n, k in (("self_attn.q_proj", h, h), ("self_attn.k_proj", h, h), ("self_attn.v_proj", h, h),
                     ("self_attn.o_proj", h, h), ("mlp.gate_proj", ffn, h), ("mlp.up_proj", ffn, h),
                     ("mlp.down_proj", h, ffn)):
        t.append((f"model.layers.0.{nm}.weight", L.DTYPE_I8, (n, k)))
        t.append((f"model.layers.0.{nm}.SCB", L.DTYPE_F32, (n,)))
    return t


def test_create_int8_reports_bad_names_dtypes_and_shapes():
    L = _lib()
    # every tensor is validated before the handle allocates anything, so no GPU is needed
    st, msg = _create(L, [x for x in _tensors(L) if x[0] != "model.layers.0.mlp.up_proj.SCB"])
    assert st != 0 and "missing weight 'model.layers.0.mlp.up_proj.SCB'" in msg, msg
    t = [(n, L.DTYPE_F16 if n.endswith("q_proj.weight") else d, s) for n, d, s in _tensors(L)]
    st, msg = _create(L, t)
    assert st != 0 and "q_proj.weight' must be int8" in msg, msg
    t = [(n, d, (s[0], s[1] + 16) if n.endswith("down_proj.weight") else s) for n, d, s in _tensors(L)]
    st, msg = _create(L, t)
    assert st != 0 and "down_proj.weight' must be int8 [256, 256]" in msg, msg
    t = [(n, L.DTYPE_F16 if n.endswith("o_proj.SCB") else d, s) for n, d, s in _tensors(L)]
    st, msg = _create(L, t)
    assert st != 0 and "o_proj.SCB' must be fp32" in msg, msg
    st, msg = _create(L, _tensors(L), threshold=0.0)
    assert st != 0 and "threshold" in msg, msg
