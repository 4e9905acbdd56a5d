"""LoRA without a GPU: the restatement in tests/lora_ref.py, adapter-config parsing and key names, and the refusals of
the Python loader and of the C entry points."""
import ctypes as C
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lora_ref as R  # noqa: E402
from seed_b200 import peft as P  # noqa: E402

CFG = {"peft_type": "LORA", "r": 16, "lora_alpha": 32, "bias": "none", "fan_in_fan_out": False,
       "target_modules": ["q_proj", "v_proj", "k_proj", "o_proj", "gate_proj", "down_proj", "up_proj"],
       "modules_to_save": ["embed_tokens", "lm_head", "input_layernorm", "post_attention_layernorm", "norm"],
       "task_type": "CAUSAL_LM", "lora_dropout": 0.05}


@pytest.mark.parametrize("M,N,K,r", [(1, 64, 256, 1), (5, 128, 512, 16), (33, 96, 1024, 64)])
def test_restated_linear_matches_float64(M, N, K, r):
    g = torch.Generator().manual_seed(M * 1000 + r)
    x = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * 0.03).half()
    a = (torch.randn(r, K, generator=g) * 0.03).half()
    b = (torch.randn(N, r, generator=g) * 0.05).half()
    s = 32.0 / r
    y = R.linear(x, w, a, b, s).double()
    exact = x.double() @ w.double().T + s * (b.double() @ (a.double() @ x.double().T)).T
    # rounding points: base, t (propagated through B), u, c and y -- a few fp16 ulps of the operands' scale
    tb = (R.ulp(a.double() @ x.double().T).T.abs() @ b.double().abs().T) * s
    bound = 2 * R.ulp(exact) + 2 * R.ulp(x.double() @ w.double().T) + tb + 2 * R.ulp(y - (x.double() @ w.double().T))
    assert torch.all((y - exact).abs() <= bound)
    assert (y - exact).abs().max() > 0 or M == 1     # the bound is exercised, not vacuous


def test_restated_merge_matches_float64():
    g = torch.Generator().manual_seed(5)
    w = (torch.randn(64, 128, generator=g) * 0.03).half()
    a = (torch.randn(8, 128, generator=g) * 0.03).half()
    b = (torch.randn(64, 8, generator=g) * 0.05).half()
    m = R.merge(w, a, b, 4.0).double()
    exact = w.double() + 4.0 * (b.double() @ a.double())
    assert torch.all((m - exact).abs() <= R.ulp(exact) + 4.0 * R.ulp(b.double() @ a.double()) + R.ulp(m - w.double()))


def test_adapter_config_accepts_the_training_config():
    r, alpha, targets, save = P.check_adapter_config(CFG)
    assert (r, alpha) == (16, 32.0) and len(targets) == 7 and len(save) == 5


@pytest.mark.parametrize("field,value", [("use_dora", True), ("use_rslora", True), ("rank_pattern", {"q_proj": 8}),
                                         ("alpha_pattern", {"q_proj": 8}), ("bias", "all"), ("fan_in_fan_out", True),
                                         ("target_modules", ["q_proj", "lm_head"]), ("modules_to_save", ["score"]),
                                         ("target_modules", "q_proj|v_proj"), ("r", 65), ("peft_type", "IA3"),
                                         ("layers_to_transform", [0])])
def test_adapter_config_refusals_name_the_field(field, value):
    cfg = dict(CFG, **{field: value})
    with pytest.raises(ValueError, match=field if field != "target_modules" or isinstance(value, list) else "target"):
        P.check_adapter_config(cfg)


def _sd(prefix="base_model.model.", infix=""):
    a, b = torch.zeros(4, 8), torch.zeros(8, 4)
    sd = {}
    for l in range(2):
        for par, proj in (("self_attn", "q_proj"), ("mlp", "down_proj")):
            sd[f"{prefix}model.layers.{l}.{par}.{proj}.lora_A{infix}.weight"] = a
            sd[f"{prefix}model.layers.{l}.{par}.{proj}.lora_B{infix}.weight"] = b
    return sd


@pytest.mark.parametrize("infix", ["", ".default"])
def test_key_forms(infix):
    sd = _sd(infix=infix)
    sd["base_model.model.model.embed_tokens" + (".modules_to_save.default" if infix else "") + ".weight"] = torch.zeros(3, 8)
    sd["base_model.model.model.embed_tokens.original_module.weight"] = torch.zeros(3, 8)
    sd["base_model.model.lm_head.weight"] = torch.zeros(3, 8)
    lora, saved = P.split_adapter(sd, ("q_proj", "down_proj"), ("embed_tokens", "lm_head"))
    assert sorted(saved) == ["lm_head.weight", "model.embed_tokens.weight"]
    assert "model.layers.1.mlp.down_proj.lora_B.weight" in lora and len(lora) == 8


def test_loader_refusals():
    sd = _sd()
    del sd["base_model.model.model.layers.1.self_attn.q_proj.lora_B.weight"]
    with pytest.raises(ValueError, match="no matching lora_B"):
        P.split_adapter(sd, ("q_proj", "down_proj"), ())
    with pytest.raises(ValueError, match="not in the adapter's target_modules"):
        P.split_adapter(_sd(), ("q_proj",), ())
    sd = _sd()
    sd["base_model.model.model.layers.0.mlp.act_fn.weight"] = torch.zeros(1)
    with pytest.raises(ValueError, match="act_fn"):
        P.split_adapter(sd, ("q_proj", "down_proj"), ())
    sd = _sd()
    sd["base_model.model.model.norm.weight"] = torch.zeros(8)
    with pytest.raises(ValueError, match="modules_to_save"):
        P.split_adapter(sd, ("q_proj", "down_proj"), ())

    class Cfg:
        hidden_size, intermediate_size, num_hidden_layers, vocab_size = 8, 16, 2, 3
    lora, saved = P.split_adapter(_sd(), ("q_proj", "down_proj"), ())
    with pytest.raises(ValueError, match="down_proj.lora_A.weight: shape"):
        P.check_shapes(lora, saved, Cfg, 4)
    with pytest.raises(ValueError, match="different vocabulary"):
        P.check_shapes({}, {"model.embed_tokens.weight": torch.zeros(3, 8), "lm_head.weight": torch.zeros(4, 8)}, Cfg, 4)
    with pytest.raises(ValueError, match="resize_token_embeddings"):
        P.check_shapes({}, {"model.embed_tokens.weight": torch.zeros(4, 8), "lm_head.weight": torch.zeros(4, 8)}, Cfg, 4)
    P.check_shapes({}, {"model.embed_tokens.weight": torch.zeros(3, 8), "lm_head.weight": torch.zeros(3, 8)}, Cfg, 4)


def test_adapter_files_both_formats(tmp_path):
    from safetensors.torch import save_file

    for fmt in ("safetensors", "bin"):
        d = tmp_path / fmt
        d.mkdir()
        (d / "adapter_config.json").write_text(json.dumps(CFG))
        sd = {k: v.clone() for k, v in _sd().items()}
        if fmt == "bin":
            torch.save(sd, d / "adapter_model.bin")
        else:
            save_file(sd, str(d / "adapter_model.safetensors"))
        cfg, got = P.load_adapter_files(str(d))
        assert cfg["r"] == 16 and sorted(got) == sorted(sd)
    with pytest.raises(RuntimeError, match="neither"):
        (tmp_path / "empty").mkdir()
        (tmp_path / "empty" / "adapter_config.json").write_text("{}")
        P.load_adapter_files(str(tmp_path / "empty"))


def test_peft_model_refusals():
    class M:
        is_loaded_in_8bit = True
    with pytest.raises(NotImplementedError, match="is_trainable"):
        P.PeftModel.from_pretrained(M(), "x", is_trainable=True)
    with pytest.raises(NotImplementedError, match="load_in_8bit"):
        P.PeftModel.from_pretrained(M(), "x")
    from models.peft_model import get_peft_model_with_resize_embedding
    with pytest.raises(NotImplementedError, match="peft_config"):
        get_peft_model_with_resize_embedding(M(), peft_config={"r": 16})


def test_c_entry_points_refuse_bad_arguments():
    from seed_b200 import lib as L

    lib = L.load()
    fake = C.c_void_p(256)   # never dereferenced: the checks run first

    def err(status):
        assert status != 0
        return lib.seedb200_last_error().decode()

    assert "null" in err(lib.seedb200_llama_lora_load(None, None, 0, 16, 32.0))
    assert "null" in err(lib.seedb200_llama_lora_merge(None))
    assert "null" in err(lib.seedb200_llama_replace_weights(None, None, 0))
    assert "r_tot" in err(lib.seedb200_lora_shrink(fake, 64, None, 1e-6, fake, 5, 64, 193, fake, 193, None))
    assert "multiple of 8" in err(lib.seedb200_lora_shrink(fake, 60, None, 1e-6, fake, 5, 60, 16, fake, 16, None))
    op = L.LoraOperand(256, 16, 256, 65, 64, 1, 1, 2.0, None)
    assert "r 65" in err(lib.seedb200_gemv_lora(fake, fake, 64, fake, None, None, 1e-6, 1, 64, 64, 0, C.byref(op), None))
    op = L.LoraOperand(256, 16, 256, 16, 64, 1, 1, 2.0, None)
    assert "256" in err(lib.seedb200_gemv_lora(fake, fake, 64, fake, None, None, 1e-6, 1, 128, 64, 1, C.byref(op), None))
    d = L.GemmLoraDesc()
    d.gemm.M, d.gemm.N, d.gemm.K, d.gemm.bias = 8, 64, 64, 256
    d.lora = L.LoraOperand(256, 16, 256, 16, 64, 1, 1, 2.0, None)
    assert "epilogue" in err(lib.seedb200_gemm_lora(C.byref(d), None))
