"""PEFT's `PeftModel.from_pretrained` for unmerged LoRA adapters on seed_b200's LlamaForCausalLM (inference only).

The arithmetic is PEFT's `lora.Linear.forward` for an fp16 module in eval mode (include/seedb200.h states it): the
base product, then `fp16(base + fp16(fp16(B . fp16(A . x)) * s))` with s = lora_alpha / r, before the layer's residual
add or SiLU gate.  `modules_to_save` tensors replace the base model's embed_tokens, lm_head and norms outright.

Adapter layout: what peft's `get_peft_model_state_dict` writes for a LlamaForCausalLM --
`base_model.model.model.layers.N.<self_attn|mlp>.<proj>.lora_A.weight` / `.lora_B.weight` and, for `modules_to_save`,
`base_model.model.model.embed_tokens.weight`, `base_model.model.lm_head.weight`, ...  The `.default.` and
`.modules_to_save.default.` infixes of the in-memory module names are accepted too, and `.original_module.` entries are
ignored.  peft itself is not a dependency: this reading of the layout comes from peft's documented state-dict names
and has been checked against hand-written fixtures only, not against files peft wrote.

Refused, with a message naming the field: `use_dora`, `use_rslora`, a non-empty `rank_pattern` / `alpha_pattern`,
`bias != "none"`, `fan_in_fan_out`, `layers_to_transform`, target modules outside the seven decoder linears,
`modules_to_save` outside embed_tokens / lm_head / input_layernorm / post_attention_layernorm / norm, a lora_A without
its lora_B (or the reverse), shapes that do not match the model (a saved embed_tokens / lm_head must have the
model's vocabulary: resize_token_embeddings first), `is_trainable=True`, and int8 models.
"""
from __future__ import annotations

import json
import os
from typing import Dict, Tuple

import torch

LORA_TARGETS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
SAVE_MODULES = ("embed_tokens", "lm_head", "input_layernorm", "post_attention_layernorm", "norm")
_PARENT = {"q_proj": "self_attn", "k_proj": "self_attn", "v_proj": "self_attn", "o_proj": "self_attn",
           "gate_proj": "mlp", "up_proj": "mlp", "down_proj": "mlp"}


def check_adapter_config(cfg: dict) -> Tuple[int, float, tuple, tuple]:
    """adapter_config.json -> (r, lora_alpha, target_modules, modules_to_save); ValueError names a refused field."""
    if str(cfg.get("peft_type", "LORA")).upper() != "LORA":
        raise ValueError(f"peft_type: only LORA adapters are supported (got {cfg.get('peft_type')!r})")
    for flag in ("use_dora", "use_rslora", "fan_in_fan_out"):
        if cfg.get(flag):
            raise ValueError(f"{flag}=True is not supported")
    for pat in ("rank_pattern", "alpha_pattern"):
        if cfg.get(pat):
            raise ValueError(f"{pat} must be empty (got {cfg.get(pat)!r}): one r and lora_alpha for every module")
    if cfg.get("bias", "none") != "none":
        raise ValueError(f"bias={cfg.get('bias')!r} is not supported (only 'none')")
    if cfg.get("layers_to_transform") is not None:
        raise ValueError("layers_to_transform is not supported: every layer must carry the adapter")
    r = cfg.get("r")
    if not isinstance(r, int) or not 1 <= r <= 64:
        raise ValueError(f"r must be an integer in [1, 64] (got {r!r})")
    alpha = float(cfg.get("lora_alpha", 8))
    targets = cfg.get("target_modules")
    if isinstance(targets, str) or not targets:
        raise ValueError(f"target_modules must be a non-empty list of module names (got {targets!r})")
    bad = [t for t in targets if t not in LORA_TARGETS]
    if bad:
        raise ValueError(f"target_modules {bad} are not decoder linears of LLaMA ({', '.join(LORA_TARGETS)})")
    save = cfg.get("modules_to_save") or []
    bad = [m for m in save if m not in SAVE_MODULES]
    if bad:
        raise ValueError(f"modules_to_save {bad} are not supported ({', '.join(SAVE_MODULES)})")
    return r, alpha, tuple(targets), tuple(save)


def canonical_name(key: str):
    """adapter state-dict key -> ("lora" | "save", model-relative name), or None for an `.original_module.` entry"""
    if ".original_module." in key:
        return None
    name = key
    for prefix in ("base_model.model.",):
        if name.startswith(prefix):
            name = name[len(prefix):]
    name = name.replace(".modules_to_save.default.", ".").replace(".lora_A.default.", ".lora_A.")
    name = name.replace(".lora_B.default.", ".lora_B.")
    if ".lora_A." in name or ".lora_B." in name:
        return "lora", name
    return "save", name


def split_adapter(sd: Dict[str, torch.Tensor], targets: tuple, save: tuple):
    """-> (lora tensors, modules_to_save tensors) under the model's names; ValueError on unexpected keys"""
    lora, saved = {}, {}
    for key, t in sd.items():
        c = canonical_name(key)
        if c is None:
            continue
        kind, name = c
        parts = name.split(".")
        if kind == "lora":
            # model.layers.N.<parent>.<proj>.lora_X.weight
            ok = (len(parts) == 7 and parts[0] == "model" and parts[1] == "layers" and parts[2].isdigit()
                  and parts[4] in LORA_TARGETS and _PARENT[parts[4]] == parts[3] and parts[6] == "weight")
            if not ok:
                raise ValueError(f"{key}: not a lora_A / lora_B of a LLaMA decoder linear")
            if parts[4] not in targets:
                raise ValueError(f"{key}: {parts[4]} is not in the adapter's target_modules {list(targets)}")
            lora[name] = t
        else:
            module = parts[-2] if len(parts) >= 2 else ""
            if module not in SAVE_MODULES or parts[-1] != "weight":
                raise ValueError(f"{key}: not a LoRA tensor or a supported modules_to_save weight")
            if module not in save:
                raise ValueError(f"{key}: {module} is not in the adapter's modules_to_save {list(save)}")
            saved[name] = t
    for name in lora:
        other = name.replace(".lora_A.", ".lora_B.") if ".lora_A." in name else name.replace(".lora_B.", ".lora_A.")
        if other not in lora:
            raise ValueError(f"{name} has no matching {other.split('.')[-2]}")
    if not lora:
        raise ValueError("the adapter holds no lora_A / lora_B tensors")
    return lora, saved


def check_shapes(lora: Dict[str, torch.Tensor], saved: Dict[str, torch.Tensor], config, r: int) -> None:
    h, ffn, nl = config.hidden_size, config.intermediate_size, config.num_hidden_layers
    for name, t in lora.items():
        parts = name.split(".")
        layer, proj, ab = int(parts[2]), parts[4], parts[5]
        if layer >= nl:
            raise ValueError(f"{name}: the model has {nl} layers")
        n_out = ffn if proj in ("gate_proj", "up_proj") else h
        k_in = ffn if proj == "down_proj" else h
        want = (r, k_in) if ab == "lora_A" else (n_out, r)
        if tuple(t.shape) != want:
            raise ValueError(f"{name}: shape {tuple(t.shape)}, expected {want}")
    vocab = {n: t.shape[0] for n, t in saved.items() if n in ("model.embed_tokens.weight", "lm_head.weight")}
    for name, t in saved.items():
        want = (t.shape[0], h) if name in vocab else (h,)
        if tuple(t.shape) != want:
            raise ValueError(f"{name}: shape {tuple(t.shape)}, expected {want}")
    if len(set(vocab.values())) > 1:
        raise ValueError(f"embed_tokens and lm_head have different vocabulary sizes: {vocab}")
    for name, n in vocab.items():   # PEFT's load_state_dict refuses a size mismatch the same way
        if n != config.vocab_size:
            raise ValueError(f"{name}: {n} rows, but the model's vocabulary is {config.vocab_size} "
                             f"(call resize_token_embeddings({n}) first, as get_peft_model_with_resize_embedding does)")


def load_adapter_files(model_id: str):
    path = str(model_id)
    if not os.path.isdir(path):
        raise RuntimeError(f"{path} is not a local adapter directory (no network access)")
    with open(os.path.join(path, "adapter_config.json")) as f:
        cfg = json.load(f)
    st = os.path.join(path, "adapter_model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file

        sd = load_file(st)
    elif os.path.exists(os.path.join(path, "adapter_model.bin")):
        sd = torch.load(os.path.join(path, "adapter_model.bin"), map_location="cpu")
    else:
        raise RuntimeError(f"{path} holds neither adapter_model.safetensors nor adapter_model.bin")
    return cfg, sd


class PeftModel:
    """An unmerged LoRA adapter on a seed_b200 LlamaForCausalLM: forward / generate run the base kernels plus the
    LoRA shrink and expand kernels.  One adapter at a time, inference only."""

    def __init__(self, model, peft_config: dict, adapter_name: str = "default"):
        self.base_model = model
        self.peft_config = {adapter_name: peft_config}
        self.active_adapter = adapter_name

    @classmethod
    def from_pretrained(cls, model, model_id, adapter_name: str = "default", is_trainable: bool = False, **kwargs):
        if is_trainable:
            raise NotImplementedError("is_trainable=True: seed_b200 runs LoRA adapters for inference only")
        if getattr(model, "is_loaded_in_8bit", False):
            raise NotImplementedError("LoRA adapters on load_in_8bit models are not supported")
        if getattr(model, "is_loaded_in_4bit", False):
            raise NotImplementedError("LoRA adapters on load_in_4bit models are not supported")
        cfg, sd = load_adapter_files(model_id)
        r, alpha, targets, save = check_adapter_config(cfg)
        lora, saved = split_adapter(sd, targets, save)
        check_shapes(lora, saved, model.config, r)
        dev = model.device
        # adapter tensors arrive as fp32, bf16 or fp16 and are rounded to fp16 once, as the eval scripts' .half() does
        saved16 = {k: v.detach().to(device=dev, dtype=torch.float16).contiguous() for k, v in saved.items()}
        lora16 = {k: v.detach().to(device=dev, dtype=torch.float16).contiguous() for k, v in lora.items()}
        llm = model._llm
        # the adapter first: its load validates every tensor before anything changes, and the modules_to_save
        # tensors (validated above, same shapes as the model's) then cannot be refused
        llm.lora_load(lora16, r, alpha)
        model._lora_bytes = sum(t.numel() * 2 for t in lora16.values())
        if saved16:
            before = sum(llm._weights[k].numel() * 2 for k in saved16 if k in llm._weights)
            llm.replace_weights(saved16)
            model._weight_bytes += sum(t.numel() * 2 for t in saved16.values()) - before
            model._cache_len, model._cache_batch = 0, 0
        return cls(model, cfg, adapter_name)

    # ---- what the eval scripts call ------------------------------------------------------------------------
    def forward(self, *args, **kwargs):
        return self.base_model.forward(*args, **kwargs)

    __call__ = forward

    def generate(self, *args, **kwargs):
        return self.base_model.generate(*args, **kwargs)

    def compute_transition_scores(self, *args, **kwargs):
        return self.base_model.compute_transition_scores(*args, **kwargs)

    def prepare_inputs_for_generation(self, *args, **kwargs):
        return self.base_model.prepare_inputs_for_generation(*args, **kwargs)

    @property
    def config(self):
        return self.base_model.config

    @property
    def device(self):
        return self.base_model.device

    def eval(self):
        return self

    def half(self):
        return self

    def to(self, *args, **kwargs):
        self.base_model.to(*args, **kwargs)
        return self

    def get_memory_footprint(self) -> int:
        """device bytes of the weights the model holds: the base weights (with the modules_to_save tensors in place of
        the originals) plus the fp16 adapter.  PEFT's count also includes the `original_module` copy it keeps of each
        modules_to_save module; the originals are not kept here, so this is smaller by those bytes."""
        return int(self.base_model.get_memory_footprint() + getattr(self.base_model, "_lora_bytes", 0))

    def merge_and_unload(self):
        """PEFT's merge: W = fp16(W + fp16(fp16(B @ A) * s)) into the base weights (changed in place), adapter freed;
        returns the base LlamaForCausalLM, which then runs exactly the base kernels."""
        self.base_model._llm.lora_merge()
        self.base_model._lora_bytes = 0
        return self.base_model
