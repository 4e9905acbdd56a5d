"""bitsandbytes 4-bit restatement (tests/quant4_ref.py), the load_in_4bit option parsing and the 4-bit C ABI surface,
without a GPU."""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import quant4_ref as Q  # noqa: E402


def test_thresholds_are_fp32_midpoints():
    v = Q.NF4_VALUES
    for i in range(15):
        mid = torch.tensor(float(v[i]) + float(v[i + 1]), dtype=torch.float32) * 0.5
        assert Q.NF4_THRESHOLDS[i] == mid
        assert v[i] < Q.NF4_THRESHOLDS[i] < v[i + 1]
    assert float(Q.NF4_THRESHOLDS[7]) == pytest.approx(0.03979014977812767)   # bitsandbytes' first NF4 pivot
    fp4 = Q.FP4_VALUES[:8][Q.FP4_BUCKET_CODE].tolist()                         # magnitudes in bucket order
    assert fp4 == sorted(fp4)
    for i in range(7):
        assert float(Q.FP4_PIVOTS[i]) == pytest.approx((fp4[i] + fp4[i + 1]) / 2, rel=1e-5)


@pytest.mark.parametrize("qt", [Q.FP4, Q.NF4])
def test_value_on_a_threshold_takes_the_lower_code(qt):
    thr = Q.NF4_THRESHOLDS if qt == Q.NF4 else Q.FP4_PIVOTS
    c = Q.codes(thr.clone(), qt)
    up = Q.codes(torch.nextafter(thr, torch.full_like(thr, 2.0)), qt)
    if qt == Q.NF4:
        assert c.tolist() == list(range(15)) and up.tolist() == list(range(1, 16))
    else:
        assert c.tolist() == Q.FP4_BUCKET_CODE[:7].tolist() and up.tolist() == Q.FP4_BUCKET_CODE[1:].tolist()
    # ... and the same through quantize(): a block with absmax 1 holding the fp16-exact FP4 pivot 0.0859375
    w = torch.zeros(1, 64, dtype=torch.float16)
    w[0, 0], w[0, 1], w[0, 2] = 1.0, 0.0859375, -0.0859375
    p, _ = Q.quantize(w, Q.FP4)
    assert Q.unpack(p)[0, :3].tolist() == [0b011, 0b001, 0b1001]


@pytest.mark.parametrize("qt", [Q.FP4, Q.NF4])
def test_roundtrip_error_within_half_the_local_gap(qt):
    g = torch.Generator().manual_seed(5)
    w = (torch.randn(48, 512, generator=g) * torch.rand(48, 1, generator=g) * 0.1).half()
    p, am = Q.quantize(w, qt)
    wd = Q.dequantize(p, am, qt).float()
    vals = torch.sort(Q.values(qt).unique()).values
    gaps = vals[1:] - vals[:-1]
    n = w.float().reshape(48, -1, 64) / am[..., None]
    idx = torch.searchsorted(vals, n.clamp(-1, 1)).clamp(1, len(vals) - 1)
    local = gaps[idx - 1].reshape(48, -1)
    err = (wd - w.float()).abs()
    bound = 0.5 * local * am.repeat_interleave(64, 1) + 2.0 ** -11 * wd.abs() + 2.0 ** -24
    assert torch.all(err <= bound * (1 + 1e-6))


def test_zero_block_and_signed_zero():
    w = torch.zeros(2, 128, dtype=torch.float16)
    w[1, 64] = 0.5
    w[1, 65] = -0.0
    for qt in (Q.FP4, Q.NF4):
        p, am = Q.quantize(w, qt)
        assert am.tolist() == [[0.0, 0.0], [0.0, 0.5]]
        assert torch.all(Q.dequantize(p, am, qt).float() == 0.0 + (w.float()))   # exact for 0 and +-1 * absmax
        c = Q.unpack(p)
        zero = 0 if qt == Q.FP4 else 7
        assert torch.all(c[0] == 0)                                 # 0 * inf = NaN -> code 0
        assert c[1, 65] == zero and c[1, 66] == zero                # -0 and +0 in a non-zero block
    nan = torch.tensor([float("nan")])
    assert Q.codes(nan, Q.FP4).item() == 0 and Q.codes(nan, Q.NF4).item() == 0


def test_nibble_order():
    w = torch.zeros(1, 64, dtype=torch.float16)
    w[0, 0], w[0, 1] = 1.0, -1.0                                     # FP4: 1.0 = 0b011, -1.0 = 0b1011
    p, _ = Q.quantize(w, Q.FP4)
    assert p[0, 0].item() == 0x3B
    p, _ = Q.quantize(w, Q.NF4)                                      # NF4: 1.0 = 15, -1.0 = 0
    assert p[0, 0].item() == 0xF0


def test_linear4_is_the_linear_of_the_dequantised_weight():
    g = torch.Generator().manual_seed(2)
    w = (torch.randn(40, 256, generator=g) * 0.05).half()
    x = torch.randn(3, 256, generator=g).half()
    p, am = Q.quantize(w, Q.NF4)
    wd = Q.dequantize(p, am, Q.NF4)
    ref = (x.double() @ wd.double().t())
    y = Q.linear4(x, p, am, Q.NF4).double()
    assert torch.all((y - ref).abs() <= 2.0 ** -11 * ref.abs() + 1e-5)


# ---- option parsing ---------------------------------------------------------------------------------------------
def test_quant_options():
    from seed_b200.llama import quant_options

    assert quant_options() == {"load_in_8bit": False, "llm_int8_threshold": 6.0, "load_in_4bit": False,
                               "bnb_4bit_quant_type": "fp4"}
    o = quant_options(load_in_4bit=True, bnb_4bit_quant_type="nf4", bnb_4bit_compute_dtype=torch.float16)
    assert o["load_in_4bit"] and o["bnb_4bit_quant_type"] == "nf4"
    assert quant_options(load_in_4bit=True, bnb_4bit_compute_dtype="float32")["load_in_4bit"]
    cfg = SimpleNamespace(load_in_4bit=True, load_in_8bit=False, bnb_4bit_quant_type="nf4",
                          bnb_4bit_compute_dtype=torch.float32, bnb_4bit_use_double_quant=False, llm_int8_threshold=6.0)
    assert quant_options(cfg)["bnb_4bit_quant_type"] == "nf4"
    assert quant_options({"load_in_4bit": True})["load_in_4bit"]
    assert quant_options({"load_in_8bit": True, "llm_int8_threshold": 5.0})["llm_int8_threshold"] == 5.0
    with pytest.raises(ValueError, match="load_in_8bit and load_in_4bit"):
        quant_options(load_in_8bit=True, load_in_4bit=True)
    with pytest.raises(ValueError, match="load_in_8bit and load_in_4bit"):
        quant_options({"load_in_8bit": True, "load_in_4bit": True})
    with pytest.raises(NotImplementedError, match="bnb_4bit_use_double_quant"):
        quant_options(load_in_4bit=True, bnb_4bit_use_double_quant=True)
    with pytest.raises(NotImplementedError, match="bnb_4bit_use_double_quant"):
        quant_options(SimpleNamespace(load_in_4bit=True, bnb_4bit_use_double_quant=True))
    for bad in (torch.bfloat16, "bfloat16", torch.float64):
        with pytest.raises(NotImplementedError, match="bnb_4bit_compute_dtype"):
            quant_options(load_in_4bit=True, bnb_4bit_compute_dtype=bad)
    with pytest.raises(ValueError, match="bnb_4bit_quant_type"):
        quant_options(load_in_4bit=True, bnb_4bit_quant_type="int4")
    with pytest.raises(ValueError, match="not both"):
        quant_options({"load_in_4bit": True}, load_in_4bit=True)


def test_from_pretrained_refuses_before_reading_weights(tmp_path):
    """the refusals come before the checkpoint is read (the directory here holds none) and before any allocation"""
    from seed_b200.llama import LlamaForCausalLM, get_pretrained_llama_causal_model

    d = str(tmp_path)
    with pytest.raises(NotImplementedError, match="bnb_4bit_use_double_quant"):
        LlamaForCausalLM.from_pretrained(d, load_in_4bit=True, bnb_4bit_use_double_quant=True)
    with pytest.raises(NotImplementedError, match="bnb_4bit_compute_dtype"):
        get_pretrained_llama_causal_model(d, load_in_4bit=True, bnb_4bit_compute_dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="load_in_8bit and load_in_4bit"):
        LlamaForCausalLM.from_pretrained(d, quantization_config={"load_in_8bit": True, "load_in_4bit": True})
    with pytest.raises(ValueError, match="bnb_4bit_quant_type"):
        LlamaForCausalLM.from_pretrained(d, quantization_config=SimpleNamespace(load_in_4bit=True,
                                                                                bnb_4bit_quant_type="fp8"))
    with pytest.raises(NotImplementedError, match="bnb_4bit_use_double_quant"):
        LlamaForCausalLM(None, {}, load_in_4bit=True, bnb_4bit_use_double_quant=True)
    # valid options get as far as the checkpoint directory, which holds no config.json
    with pytest.raises(Exception) as e:
        LlamaForCausalLM.from_pretrained(d, load_in_4bit=True, bnb_4bit_quant_type="nf4")
    assert not isinstance(e.value, (NotImplementedError, ValueError))


def test_peft_refuses_4bit_models():
    from seed_b200.peft import PeftModel

    with pytest.raises(NotImplementedError, match="load_in_4bit"):
        PeftModel.from_pretrained(SimpleNamespace(is_loaded_in_8bit=False, is_loaded_in_4bit=True), "/nonexistent")


# ---- C ABI -----------------------------------------------------------------------------------------------------------
def _lib():
    from seed_b200 import lib as L

    if not os.path.exists(L.LIB_PATH):
        pytest.skip("libseedb200.so not built")
    return L


def test_quant4_symbols_resolve():
    L = _lib()
    h = L.load()
    for sym in ("seedb200_quantize_4bit", "seedb200_dequantize_4bit", "seedb200_gemv_4bit",
                "seedb200_llama_create_4bit", "seedb200_llama_4bit_load_weight"):
        assert sym in L.EXPORTS and hasattr(h, sym)


def test_per_op_argument_checks():
    """argument checks come before any device work: fake pointers are never dereferenced"""
    L = _lib()
    h = L.load()
    p = 1 << 20
    assert h.seedb200_quantize_4bit(p, 96, 4, 96, 0, p, p, None) != 0
    assert "K=96 is not a multiple of the 4-bit blocksize 64" in h.seedb200_last_error().decode()
    assert h.seedb200_quantize_4bit(p, 128, 4, 128, 2, p, p, None) != 0
    assert "quant_type 2" in h.seedb200_last_error().decode()
    assert h.seedb200_dequantize_4bit(p, p, 4, 32, 1, p, 0, None) != 0
    assert "K=32" in h.seedb200_last_error().decode()
    assert h.seedb200_gemv_4bit(p, None, 1e-6, p, p, 7, p, None, 1, 64, 64, 0, None) != 0
    assert "quant_type 7" in h.seedb200_last_error().decode()
    assert h.seedb200_gemv_4bit(p, None, 1e-6, p, p, 1, p, None, 1, 64, 100, 0, None) != 0
    assert "K=100" in h.seedb200_last_error().decode()
    with pytest.raises(ValueError, match="bnb_4bit_quant_type"):
        L.quant4_type("nf8")


def _create(L, tensors, quant_type=1, hidden=256, ffn=256):
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
    cfg = L.LlamaConfig(hidden, 1, hidden // 128, 128, ffn, 64, 1, 32, 1e-6, 10000.0, 0)
    st = L.load().seedb200_llama_create_4bit(C.byref(cfg), arr, len(tensors), quant_type, C.byref(h))
    return st, L.load().seedb200_last_error().decode()


def _tensors(L, h=256, V=64):
    return [("model.embed_tokens.weight", L.DTYPE_F16, (V, h)), ("model.norm.weight", L.DTYPE_F16, (h,)),
            ("lm_head.weight", L.DTYPE_F16, (V, h)),
            ("model.layers.0.input_layernorm.weight", L.DTYPE_F16, (h,)),
            ("model.layers.0.post_attention_layernorm.weight", L.DTYPE_F16, (h,))]


def test_create_4bit_reports_bad_arguments():
    L = _lib()
    st, msg = _create(L, _tensors(L), quant_type=3)
    assert st != 0 and "quant_type 3" in msg, msg
    st, msg = _create(L, _tensors(L) + [("model.layers.0.mlp.up_proj.weight", L.DTYPE_F16, (256, 256))])
    assert st != 0 and "'model.layers.0.mlp.up_proj.weight' is a decoder linear" in msg, msg
    st, msg = _create(L, [x for x in _tensors(L) if x[0] != "model.norm.weight"])
    assert st != 0 and "missing weight 'model.norm.weight'" in msg, msg
    st, msg = _create(L, [(n, d, (s[0] + 1,) if n == "model.layers.0.input_layernorm.weight" else s)
                          for n, d, s in _tensors(L)])
    assert st != 0 and "input_layernorm.weight' must be fp16" in msg, msg
    st, msg = _create(L, _tensors(L), ffn=288)
    assert st != 0 and "ffn 288" in msg, msg
    # load_weight needs a handle: refused without one, by name
    assert L.load().seedb200_llama_4bit_load_weight(None, b"model.layers.0.mlp.up_proj.weight", 4096, 0, None) != 0
    assert "null argument" in L.load().seedb200_last_error().decode()
