"""Host-side mirror of models/llama_xformer.py (LlamaForCausalLM) on top of libseedb200.

`forward()` keeps the reference signature and returns transformers' CausalLMOutputWithPast
(llama_xformer.py:661-743); `generate()` stands in for HF GenerationMixin (scripts/seed_llama_inference_8B.py:33):
by default one C call that keeps prefill, sampling and the graph-replayed decode steps on the device.

Reference behaviours kept on purpose (SURVEY.md section 7 "quirks"):
  * padding in `attention_mask` is ignored by attention -- the reference only tests `attention_mask.sum() == 0`
    to choose between a causal and an unmasked xformers call (llama_xformer.py:240-256);
  * q_len == 1 attends to the whole cache without a mask; q_len > 1 is causal;
  * logits are returned for every position in fp16.
`resize_token_embeddings` follows transformers 4.30.2; unmerged LoRA adapters are loaded through seed_b200/peft.py.
`load_in_8bit=True` runs the seven linear layers of every decoder layer as LLM.int8() (transformers' bitsandbytes
path, threshold `llm_int8_threshold`): int8 weights with per-row scales, per-call activation quantisation with fp16
outlier columns; embed_tokens, lm_head and the norms stay fp16 (include/seedb200.h states the arithmetic).
`load_in_4bit=True` runs the same seven linears as bitsandbytes 4-bit weights (`bnb_4bit_quant_type` "fp4" or "nf4",
blocks of 64 with an fp32 absmax): decode steps of up to 4 rows stream the packed codes through the 4-bit GEMV;
longer calls dequantise each linear into an fp16 scratch and run the fp16 GEMM, as bitsandbytes' MatMul4Bit does.
Differences: `past_key_values` are views of the handle's preallocated cache (no torch.cat per step);
`output_attentions` / `output_hidden_states` are not available (the reference's xformers path never computed
attention weights either).
"""
from __future__ import annotations

import glob
import json
import math
import os
from typing import List, Optional, Tuple, Union

import torch
import torch.nn as nn
from transformers.generation import GenerateBeamDecoderOnlyOutput, GenerateDecoderOnlyOutput
from transformers.generation.utils import GenerationMixin
from transformers.modeling_outputs import CausalLMOutputWithPast
from transformers.models.llama.configuration_llama import LlamaConfig

from . import lib as L


class _CudaView:
    def __init__(self, ptr: int, shape, strides_elems):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f2", "data": (ptr, False), "version": 3,
                                         "strides": tuple(s * 2 for s in strides_elems)}


_QUANTISED_LINEARS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def _is_quantised_linear(name: str) -> bool:
    """the decoder-layer nn.Linear weights transformers' load_in_8bit / load_in_4bit replace (lm_head stays fp16)"""
    parts = name.split(".")
    return ".layers." in name and len(parts) >= 2 and parts[-1] == "weight" and parts[-2] in _QUANTISED_LINEARS


_QUANT_DEFAULTS = {"load_in_8bit": False, "load_in_4bit": False, "llm_int8_threshold": 6.0,
                   "bnb_4bit_quant_type": "fp4", "bnb_4bit_compute_dtype": None, "bnb_4bit_use_double_quant": False}


def quant_options(quantization_config=None, **given) -> dict:
    """transformers 4.30.2's bitsandbytes options -> {load_in_8bit, llm_int8_threshold, load_in_4bit,
    bnb_4bit_quant_type}.  `given` holds the keywords the caller passed; `quantization_config` (a BitsAndBytesConfig,
    read by attribute, or a dict) replaces them, and passing both is an error, as in transformers.  Everything that
    cannot run here is refused by name before any weight is read or allocated."""
    unknown = set(given) - set(_QUANT_DEFAULTS)
    if unknown:
        raise TypeError(f"unknown quantisation options {sorted(unknown)}")
    if quantization_config is not None:
        if given:
            raise ValueError(f"pass either quantization_config or {sorted(given)}, not both")
        cfg = quantization_config

        def get(k):
            return cfg.get(k) if isinstance(cfg, dict) else getattr(cfg, k, None)

        given = {k: get(k) for k in _QUANT_DEFAULTS if get(k) is not None}
    o = dict(_QUANT_DEFAULTS)
    o.update(given)
    if o["load_in_8bit"] and o["load_in_4bit"]:
        raise ValueError("load_in_8bit and load_in_4bit are both True, and only one can be used at the same time")
    if o["bnb_4bit_use_double_quant"]:
        raise NotImplementedError("bnb_4bit_use_double_quant=True: double quantisation of the 4-bit absmax values is "
                                  "not supported")
    cd = o["bnb_4bit_compute_dtype"]
    if isinstance(cd, str):
        cd = getattr(torch, cd, cd)
    if cd not in (None, torch.float32, torch.float16):
        raise NotImplementedError(f"bnb_4bit_compute_dtype={o['bnb_4bit_compute_dtype']!r}: only None, torch.float32 "
                                  f"and torch.float16 are supported (they give the same fp16 result; bf16 does not)")
    if o["bnb_4bit_quant_type"] not in ("fp4", "nf4"):
        raise ValueError(f"bnb_4bit_quant_type must be 'fp4' or 'nf4' (got {o['bnb_4bit_quant_type']!r})")
    return {"load_in_8bit": bool(o["load_in_8bit"]), "llm_int8_threshold": float(o["llm_int8_threshold"]),
            "load_in_4bit": bool(o["load_in_4bit"]), "bnb_4bit_quant_type": o["bnb_4bit_quant_type"]}


def _one_device(device_map) -> torch.device:
    """device_map of HF from_pretrained -> the single device it names; no model parallelism here."""
    def dev(v):
        return torch.device(f"cuda:{v}") if isinstance(v, int) else torch.device(v)

    if isinstance(device_map, dict):
        devs = {dev(v) for v in device_map.values()}
        if len(devs) != 1:
            raise ValueError(f"device_map spans {len(devs)} devices; seed_b200 runs the model on one device")
        return devs.pop()
    if device_map == "auto":
        if torch.cuda.device_count() > 1:
            raise ValueError("device_map='auto' would span several GPUs; pass one device (e.g. 'cuda:0')")
        return torch.device("cuda:0")
    return dev(device_map)


def _linear_items(state_dict, names):
    """(name, tensor) of the quantised linears; a state dict that makes its tensors on demand (its items() is a generator)
    is walked again rather than indexed, so nothing is made twice at once"""
    if not names:
        return
    wanted = set(names)
    if isinstance(state_dict, dict) and type(state_dict).items is dict.items:
        for k in names:
            yield k, state_dict[k]
        return
    for k, v in state_dict.items():
        if k in wanted:
            yield k, v


class LlamaForCausalLM(nn.Module):
    def __init__(self, config: LlamaConfig, state_dict, device="cuda", max_batch: int = 1,
                 max_seq: Optional[int] = None, gemm_ctas: int = 0, load_in_8bit: bool = False,
                 llm_int8_threshold: float = 6.0, load_in_4bit: bool = False, bnb_4bit_quant_type: str = "fp4",
                 bnb_4bit_compute_dtype=None, bnb_4bit_use_double_quant: bool = False):
        super().__init__()
        q = quant_options(load_in_8bit=load_in_8bit, llm_int8_threshold=llm_int8_threshold, load_in_4bit=load_in_4bit,
                          bnb_4bit_quant_type=bnb_4bit_quant_type, bnb_4bit_compute_dtype=bnb_4bit_compute_dtype,
                          bnb_4bit_use_double_quant=bnb_4bit_use_double_quant)
        load_in_8bit, load_in_4bit = q["load_in_8bit"], q["load_in_4bit"]
        dev = torch.device(device)
        if dev.type != "cuda" or not torch.cuda.is_available():
            raise RuntimeError("LlamaForCausalLM (seed_b200) needs a CUDA device: there is no CPU path")
        self.config = config
        self._device = dev
        h, nl, nh = config.hidden_size, config.num_hidden_layers, config.num_attention_heads
        if getattr(config, "num_key_value_heads", nh) not in (None, nh):
            raise ValueError("grouped-query attention is not part of models/llama_xformer.py")
        self.max_batch = max_batch
        self.max_seq = max_seq or config.max_position_embeddings
        self.is_loaded_in_8bit = load_in_8bit
        self.is_loaded_in_4bit = load_in_4bit
        # With a quantised format the handle is made with the fp16 tensors only; then each linear goes to the device in
        # fp16, is quantised straight into the handle's int8 / 4-bit buffers, and is dropped before the next: device
        # memory stays at the quantised model plus one fp16 tensor.
        weights, linears = {}, []
        for k, v in state_dict.items():
            if "rotary_emb" in k:
                continue
            if (load_in_8bit or load_in_4bit) and _is_quantised_linear(k):
                linears.append(k)
                continue
            weights[k] = v.detach().to(device=dev, dtype=torch.float16).contiguous()
        # device bytes of the weights the handle owns or borrows (HF get_memory_footprint: no KV cache / workspace)
        self._weight_bytes = sum(t.numel() * t.element_size() for t in weights.values())
        self._llm = L.Llama(weights, hidden=h, layers=nl, heads=nh, ffn=config.intermediate_size,
                            vocab=config.vocab_size, max_batch=max_batch, max_seq=self.max_seq,
                            rms_eps=config.rms_norm_eps, gemm_ctas=gemm_ctas,
                            int8_threshold=q["llm_int8_threshold"] if load_in_8bit else None,
                            quant4=q["bnb_4bit_quant_type"] if load_in_4bit else None)
        for k, v in _linear_items(state_dict, linears):
            w16 = v.detach().to(device=dev, dtype=torch.float16)
            if w16.stride(-1) != 1 or (load_in_4bit and not w16.is_contiguous()):
                w16 = w16.contiguous()
            N, K = w16.shape
            if load_in_8bit:
                self._llm.int8_load_weight(k, w16)
                self._weight_bytes += N * K + 4 * N           # int8 values plus one fp32 scale per row
            else:
                self._llm.load_4bit_weight(k, w16)
                self._weight_bytes += N * K // 2 + 4 * (N * K // 64)   # packed codes plus one fp32 absmax per 64
            del w16, v     # stream-ordered: the allocator reuses this block only after the kernel has read it
        # q/k/v and gate/up were copied into fused layouts by the handle: drop our references to the originals
        for k in [k for k in self._llm._weights if any(s in k for s in ("q_proj", "k_proj", "v_proj", "gate_proj", "up_proj"))]:
            del self._llm._weights[k]
        del weights
        self._cache_len = 0          # tokens currently valid in the internal KV cache
        self._cache_batch = 0
        self._draws = 0              # Philox counter: sampling draws made so far (successive generate() calls differ)

    # ---- construction --------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, torch_dtype=torch.float16, device="cuda", device_map=None,
                        **kwargs):
        """HF checkpoint directory (config.json + *.safetensors or pytorch_model*.bin).  `load_in_8bit`,
        `llm_int8_threshold`, `load_in_4bit`, `bnb_4bit_quant_type`, `bnb_4bit_compute_dtype`,
        `bnb_4bit_use_double_quant`, a `quantization_config` holding them (attributes or a dict) and a single-device
        `device_map` are honoured as transformers does."""
        quant = quant_options(kwargs.pop("quantization_config", None),
                              **{k: kwargs.pop(k) for k in list(kwargs) if k in _QUANT_DEFAULTS})
        if device_map is not None:
            device = _one_device(device_map)
        path = str(pretrained_model_name_or_path)
        if not os.path.isdir(path):
            raise RuntimeError(f"{path} is not a local checkpoint directory (no network access)")
        if torch_dtype not in (torch.float16, "fp16", "float16", None):
            raise ValueError("seed_b200 implements the reference's fp16 LLaMA path (torch_dtype=fp16) only")
        with open(os.path.join(path, "config.json")) as f:
            config = LlamaConfig(**{k: v for k, v in json.load(f).items() if k not in ("architectures", "model_type")})
        sd = {}
        st_files = sorted(glob.glob(os.path.join(path, "*.safetensors")))
        if st_files:
            from safetensors.torch import load_file

            for fn in st_files:
                sd.update(load_file(fn))
        else:
            for fn in sorted(glob.glob(os.path.join(path, "pytorch_model*.bin"))):
                sd.update(torch.load(fn, map_location="cpu"))
        if not sd:
            raise RuntimeError(f"no weight files found under {path}")
        kwargs = {k: v for k, v in kwargs.items() if k in ("max_batch", "max_seq", "gemm_ctas")}
        return cls(config, sd, device=device, **kwargs, **quant)

    # ---- nn.Module conveniences ------------------------------------------------------------------
    @property
    def device(self):
        return self._device

    def eval(self):
        return self

    def get_memory_footprint(self) -> int:
        """device bytes of the model's weights; the KV cache and workspaces are excluded, as in transformers.  int8
        linears count their int8 values and fp32 scales, 4-bit linears their packed codes (half a byte per weight)
        and fp32 absmax values (one per 64 weights).  Counting the scales differs from transformers, which counts
        only the quantised parameters.  The 4-bit handle's fp16 dequantisation scratch (2 * ffn * hidden
        elements) is workspace and not counted."""
        return int(self._weight_bytes)

    def half(self):
        return self

    def resize_token_embeddings(self, new_num_tokens: Optional[int] = None) -> nn.Embedding:
        """transformers 4.30.2 PreTrainedModel.resize_token_embeddings (untied embeddings): embed_tokens and lm_head
        get `new_num_tokens` rows; the first min(old, new) rows are kept and new rows are drawn from
        N(0, config.initializer_range) (torch's default generator, fp32 draw rounded to fp16); config.vocab_size
        follows.  Resizing drops the handle's KV cache (the vocabulary-sized buffers are reallocated)."""
        old = self._llm._weights["model.embed_tokens.weight"]
        if new_num_tokens is None or int(new_num_tokens) == old.shape[0]:
            return nn.Embedding.from_pretrained(old, freeze=True)
        n = int(new_num_tokens)
        if n < 1:
            raise ValueError(f"new_num_tokens must be >= 1 (got {n})")
        std = float(getattr(self.config, "initializer_range", 0.02))
        keep = min(n, old.shape[0])
        new = {}
        for name in ("model.embed_tokens.weight", "lm_head.weight"):
            src = self._llm._weights[name]
            t = torch.empty((n, src.shape[1]), dtype=torch.float32, device=self._device).normal_(0.0, std).half()
            t[:keep] = src[:keep]
            new[name] = t
        self._llm.replace_weights(new)
        self._weight_bytes += 2 * (n - old.shape[0]) * old.shape[1] * 2
        self.config.vocab_size = n
        self._cache_len, self._cache_batch = 0, 0
        return nn.Embedding.from_pretrained(new["model.embed_tokens.weight"], freeze=True)

    def to(self, *args, **kwargs):
        tgt = kwargs.get("device", args[0] if args else None)
        if tgt is not None and not isinstance(tgt, torch.dtype) and torch.device(tgt).type != "cuda":
            raise RuntimeError("seed_b200 LLaMA weights cannot be moved off the GPU")
        return self

    # ---- KV cache plumbing -------------------------------------------------------------------------
    def _kv_tuple(self, B: int, length: int):
        H, D, ms = self._llm.heads, self._llm.head_dim, self.max_seq
        out = []
        for l in range(self._llm.layers):
            kp, vp = self._llm.kv_views(l)
            strides = (H * ms * D, ms * D, D, 1)
            k = torch.as_tensor(_CudaView(kp, (B, H, length, D), strides), device=self._device)
            v = torch.as_tensor(_CudaView(vp, (B, H, length, D), strides), device=self._device)
            out.append((k, v))
        return tuple(out)

    def _sync_past(self, past_key_values, B: int) -> int:
        """Make the internal cache hold `past_key_values`; returns past_len."""
        if past_key_values is None:
            self._cache_len, self._cache_batch = 0, B
            return 0
        past_len = int(past_key_values[0][0].shape[2])
        kp, _ = self._llm.kv_views(0)
        ours = (past_key_values[0][0].data_ptr() == kp and self._cache_batch == B and past_len <= self._cache_len)
        if not ours:   # foreign tensors (e.g. produced by the reference): copy them in
            for l, (k, v) in enumerate(past_key_values):
                self._llm.kv_load(l, k.to(self._device, torch.float16), v.to(self._device, torch.float16))
            self._cache_batch = B
        self._cache_len = past_len
        return past_len

    # ---- forward (llama_xformer.py:661-743) ------------------------------------------------------------
    def forward(self, input_ids: torch.LongTensor = None, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.LongTensor] = None,
                past_key_values: Optional[List[torch.FloatTensor]] = None,
                inputs_embeds: Optional[torch.FloatTensor] = None, labels: Optional[torch.LongTensor] = None,
                use_cache: Optional[bool] = None, output_attentions: Optional[bool] = None,
                output_hidden_states: Optional[bool] = None, return_dict: Optional[bool] = None,
                last_logits_only: bool = False) -> Union[Tuple, CausalLMOutputWithPast]:
        if output_attentions or output_hidden_states:
            raise NotImplementedError("output_attentions / output_hidden_states are not produced by the fused path")
        use_cache = use_cache if use_cache is not None else getattr(self.config, "use_cache", True)
        return_dict = return_dict if return_dict is not None else True
        if input_ids is not None and inputs_embeds is not None:
            raise ValueError("You cannot specify both decoder_input_ids and decoder_inputs_embeds at the same time")
        if input_ids is None and inputs_embeds is None:
            raise ValueError("You have to specify either decoder_input_ids or decoder_inputs_embeds")
        if input_ids is not None:
            input_ids = input_ids.to(self._device, torch.int64)
            B, S = input_ids.shape
        else:
            inputs_embeds = inputs_embeds.to(self._device, torch.float16)
            B, S = inputs_embeds.shape[:2]
        if B > self.max_batch:
            raise ValueError(f"batch {B} exceeds max_batch={self.max_batch} given at construction")
        past_len = self._sync_past(past_key_values, B)
        if past_len + S > self.max_seq:
            raise ValueError(f"sequence {past_len}+{S} exceeds max_seq={self.max_seq}")
        if position_ids is not None:
            position_ids = position_ids.to(self._device)
        logits = self._llm.forward(input_ids=input_ids, inputs_embeds=inputs_embeds, position_ids=position_ids,
                                   past_len=past_len, last_only=last_logits_only)
        self._cache_len = past_len + S
        loss = None
        if labels is not None:   # llama_xformer.py:720-731
            shift_logits = logits[..., :-1, :].contiguous().view(-1, self.config.vocab_size)
            shift_labels = labels[..., 1:].contiguous().view(-1).to(shift_logits.device)
            loss = nn.functional.cross_entropy(shift_logits.float(), shift_labels)
        past = self._kv_tuple(B, self._cache_len) if use_cache else None
        if not return_dict:
            out = (logits,) + ((past,) if past is not None else ())
            return ((loss,) + out) if loss is not None else out
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=past, hidden_states=None,
                                      attentions=None)

    __call__ = forward

    # ---- generation (stand-in for HF GenerationMixin.sample / greedy_search) -------------------------------
    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, attention_mask=None, inputs_embeds=None,
                                      **kwargs):
        """llama_xformer.py:745-776: last token only once a past exists; position_ids from the mask's cumsum."""
        if past_key_values:
            input_ids = input_ids[:, -1:]
        position_ids = kwargs.get("position_ids", None)
        if attention_mask is not None and position_ids is None:
            position_ids = attention_mask.long().cumsum(-1) - 1
            position_ids.masked_fill_(attention_mask == 0, 1)
            if past_key_values:
                position_ids = position_ids[:, -1].unsqueeze(-1)
        if inputs_embeds is not None and past_key_values is None:
            model_inputs = {"inputs_embeds": inputs_embeds}
        else:
            model_inputs = {"input_ids": input_ids}
        model_inputs.update({"position_ids": position_ids, "past_key_values": past_key_values,
                             "use_cache": kwargs.get("use_cache"), "attention_mask": attention_mask})
        return model_inputs

    def _next_seed(self, generator: Optional[torch.Generator], seed: Optional[int]) -> int:
        if seed is not None:
            return int(seed)
        if generator is not None:
            return int(generator.initial_seed())
        return int(torch.initial_seed())

    # GenerationConfig fields generate() honours, with the defaults used when neither it nor a kwarg sets them
    _GEN_DEFAULTS = {"max_new_tokens": 20, "do_sample": False, "temperature": 1.0, "top_p": 1.0, "num_beams": 1,
                     "length_penalty": 1.0, "early_stopping": False, "num_return_sequences": 1,
                     "top_k": 0, "repetition_penalty": 1.0, "no_repeat_ngram_size": 0, "min_length": 0,
                     "min_new_tokens": 0, "penalty_alpha": None, "output_scores": False,
                     "return_dict_in_generate": False, "output_attentions": False, "output_hidden_states": False}

    @staticmethod
    def _controls(opts) -> dict:
        """the logits processors / top_k warper settings, validated as transformers' classes do"""
        top_k, pen, n = int(opts["top_k"]), opts["repetition_penalty"], int(opts["no_repeat_ngram_size"])
        min_length, min_new = int(opts["min_length"]), int(opts["min_new_tokens"])
        if top_k < 0:
            raise ValueError(f"`top_k` has to be a non-negative integer, but is {top_k}")
        if not isinstance(pen, (int, float)) or not math.isfinite(pen) or not pen > 0:
            raise ValueError(f"`repetition_penalty` has to be a strictly positive float, but is {pen}")
        for name, v in (("no_repeat_ngram_size", n), ("min_length", min_length), ("min_new_tokens", min_new)):
            if v < 0:
                raise ValueError(f"`{name}` has to be a non-negative integer, but is {v}")
        return {"top_k": top_k, "repetition_penalty": float(pen), "no_repeat_ngram_size": n,
                "min_length": min_length, "min_new_tokens": min_new}

    @torch.no_grad()
    def generate(self, input_ids=None, inputs=None, max_new_tokens: Optional[int] = None,
                 do_sample: Optional[bool] = None, temperature: Optional[float] = None, top_p: Optional[float] = None,
                 num_beams: Optional[int] = None, eos_token_id=None, pad_token_id=None, attention_mask=None,
                 generator: Optional[torch.Generator] = None, seed: Optional[int] = None, use_graph: bool = True,
                 device_loop: Optional[bool] = None, generation_config=None, length_penalty: Optional[float] = None,
                 early_stopping=None, num_return_sequences: Optional[int] = None, top_k: Optional[int] = None,
                 repetition_penalty: Optional[float] = None, no_repeat_ngram_size: Optional[int] = None,
                 min_length: Optional[int] = None, min_new_tokens: Optional[int] = None,
                 penalty_alpha: Optional[float] = None, output_scores: Optional[bool] = None,
                 return_dict_in_generate: Optional[bool] = None, output_attentions: Optional[bool] = None,
                 output_hidden_states: Optional[bool] = None, **_):
        """Call pattern of scripts/seed_llama_inference_8B.py:33 (temperature=1.0, num_beams=1, max_new_tokens=512,
        top_p=0.5, do_sample=True); returns [B, S + n_new] like HF generate.

        Default path (`device_loop`): ONE C call -- prefill, on-device sampler, CUDA-graph-replayed decode steps
        (seedb200_llama_generate); no per-token host work.  With a padding `attention_mask` (position ids that are
        not past + arange) or more than one eos id, the loop runs from Python through
        `prepare_inputs_for_generation` exactly as HF drives the reference, still sampling with the device kernel.
        Sampled ids depend on the RNG (Philox keyed by `seed`, counter = draws made so far), not on torch's stream;
        logits are the parity contract.

        `num_beams` > 1 runs transformers 4.30.2's beam search (`do_sample=False`) or beam sampling (`do_sample=True`)
        on the device (seedb200_llama_beam_generate), with `length_penalty` and `early_stopping` (False / True /
        "never"); only an unpadded batch and one eos id.  B * num_beams rows must fit the handle: a model built with a
        smaller `max_batch` grows to it first, which drops the KV cache, so `past_key_values` returned by earlier
        forward() calls are no longer valid.
        `num_return_sequences` = n > 1 needs `do_sample=True` and returns [B * n, ...], prompt-major (row b * n + j is
        candidate j of prompt b), as transformers 4.30.2 does.  Sampling runs B * n rows in one device call
        (seedb200_llama_generate_n) that prefills each prompt once; beam sampling runs n independent searches per
        prompt, each returning its best hypothesis (seedb200_llama_beam_generate_n).  Both equal, token for token, the
        same call on `input_ids.repeat_interleave(n, 0)`, and grow the handle to B * n (times num_beams) rows as beams
        do.  With a padded mask or several eos ids the expanded batch runs through the per-token loop below.  Greedy,
        beam and contrastive search refuse n > 1.
        `top_k`, `repetition_penalty`, `no_repeat_ngram_size`, `min_length` and `min_new_tokens` act as transformers
        4.30.2's logits processors and TopK warper, on the device in every path (include/seedb200.h,
        seedb200_logits_params); the defaults turn them off.  Other generation keywords are ignored.
        `penalty_alpha` > 0 with `top_k` > 1, `num_beams=1` and `do_sample=False` runs transformers 4.30.2's contrastive
        search on the device (seedb200_llama_contrastive_generate): `top_k` is then the number of candidates (2..8,
        and it must be given: transformers' default of 50 would mean 50 cache rows), the processors above still
        apply, and B * top_k rows must fit the handle, which grows as for beams.  With `num_beams` > 1 or
        `do_sample=True` penalty_alpha is ignored, as in transformers.
        `return_dict_in_generate=True` returns transformers' GenerateDecoderOnlyOutput (GenerateBeamDecoderOnlyOutput
        with beams) instead of the tensor; with `output_scores=True` as well, greedy decoding, sampling and
        contrastive search fill `scores` as transformers 4.30.2 does (one fp16 [rows, V] tensor per step: the
        processed logits when greedy, the warped row with -inf off the kept tokens when sampling, the processed logits
        the candidates are taken from in contrastive search), written on the device by the kernel that holds the row (include/seedb200.h,
        seedb200_gen_outputs).  Every route (device loop, per-token loop, num_return_sequences) returns them.  Beam
        search and beam sampling fill `scores` (one [G * num_beams, V] tensor per BeamSearchScorer.process call: the
        processed fp16 log_softmax, warped without the beam score when sampling), `sequences_scores` and
        `beam_indices`, as 4.30.2 does.  `output_attentions` / `output_hidden_states` with
        return_dict_in_generate=True raise NotImplementedError, as forward() does.
        `generation_config` (a transformers GenerationConfig) supplies these fields and its eos / pad ids, and
        explicit keyword arguments override it, as in transformers."""
        given = {"max_new_tokens": max_new_tokens, "do_sample": do_sample, "temperature": temperature, "top_p": top_p,
                 "num_beams": num_beams, "length_penalty": length_penalty, "early_stopping": early_stopping,
                 "num_return_sequences": num_return_sequences, "top_k": top_k,
                 "repetition_penalty": repetition_penalty, "no_repeat_ngram_size": no_repeat_ngram_size,
                 "min_length": min_length, "min_new_tokens": min_new_tokens, "penalty_alpha": penalty_alpha,
                 "output_scores": output_scores, "return_dict_in_generate": return_dict_in_generate,
                 "output_attentions": output_attentions, "output_hidden_states": output_hidden_states}
        opts = dict(self._GEN_DEFAULTS)
        if generation_config is not None:
            for name in opts:
                v = getattr(generation_config, name, None)
                if v is not None:
                    opts[name] = v
            if eos_token_id is None:       # the config's own ids replace the model's, as in transformers
                eos_token_id = generation_config.eos_token_id if generation_config.eos_token_id is not None else -1
            if pad_token_id is None:
                pad_token_id = generation_config.pad_token_id
        opts.update({k: v for k, v in given.items() if v is not None})
        max_new_tokens, do_sample, temperature, top_p = (int(opts["max_new_tokens"]), bool(opts["do_sample"]),
                                                         float(opts["temperature"]), float(opts["top_p"]))
        num_beams = int(opts["num_beams"])
        return_dict = bool(opts["return_dict_in_generate"])
        for name in ("output_attentions", "output_hidden_states"):
            if return_dict and opts[name]:
                raise NotImplementedError(f"{name}=True: attention weights and hidden states are not produced by the "
                                          f"fused path")
        # transformers computes the scores with output_scores alone and drops them; here they are only made when
        # they are returned
        want_scores = return_dict and bool(opts["output_scores"])
        controls = self._controls(opts)
        n_ret = int(opts["num_return_sequences"])
        if n_ret < 1:
            raise ValueError(f"num_return_sequences must be >= 1 (got {n_ret})")
        if n_ret > 1 and not do_sample:
            raise NotImplementedError("num_return_sequences > 1 is supported with do_sample=True (sampling and beam "
                                      "sampling) only, not with greedy, beam or contrastive search")
        if num_beams < 1:
            raise ValueError(f"num_beams must be >= 1 (got {num_beams})")
        if input_ids is None:
            input_ids = inputs
        input_ids = input_ids.to(self._device, torch.int64)
        B, S = input_ids.shape
        if S + max_new_tokens > self.max_seq:
            max_new_tokens = self.max_seq - S          # HF stops at max_length; here the cache is the limit
            if max_new_tokens < 1:
                raise ValueError(f"prompt of {S} tokens leaves no room in max_seq={self.max_seq}")
        eos = eos_token_id if eos_token_id is not None else getattr(self.config, "eos_token_id", None)
        eos_list = list(eos) if isinstance(eos, (list, tuple)) else ([eos] if eos is not None else [])
        eos_list = [int(e) for e in eos_list if int(e) >= 0]      # a negative id disables the stop (fixed-length runs)
        pad = pad_token_id if pad_token_id is not None else (eos_list[0] if eos_list else 0)
        rng_seed = self._next_seed(generator, seed)
        offset = self._draws
        padded = attention_mask is not None and not bool(attention_mask.to(torch.bool).all())
        length_rules = controls["min_length"] > 0 or controls["min_new_tokens"] > 0
        if length_rules and len(eos_list) > 1:
            raise NotImplementedError("min_length / min_new_tokens with several eos_token_id values are not supported")
        alpha = opts["penalty_alpha"]
        if num_beams == 1 and not do_sample and alpha is not None and alpha > 0:
            top_k_given = top_k is not None or getattr(generation_config, "top_k", None) is not None
            if not top_k_given:
                raise ValueError("penalty_alpha > 0 selects contrastive search, which needs `top_k` (the number of "
                                 "candidates, 2..8): pass top_k explicitly")
            if controls["top_k"] > 1:
                return self._contrastive_generate(input_ids, max_new_tokens, controls["top_k"], float(alpha),
                                                  eos_list, pad, padded, use_graph, controls, return_dict,
                                                  want_scores)
        if num_beams > 1:
            out = self._beam_generate(input_ids, max_new_tokens, num_beams, do_sample, temperature, top_p,
                                      float(opts["length_penalty"]), opts["early_stopping"], eos_list, pad, padded,
                                      rng_seed, offset, use_graph, controls, n_ret, want_scores)
            return out if return_dict else out.sequences
        if device_loop is None:
            device_loop = (not padded) and len(eos_list) <= 1 and (B <= 4 or n_ret > 1)
        if device_loop:
            if padded or len(eos_list) > 1:
                raise ValueError("device_loop needs an unpadded batch and at most one eos id")
            self._reserve(B * n_ret)
            buf = L.scores_buffer(max_new_tokens, B * n_ret, self._llm.vocab, self._device) if want_scores else None
            new = self._llm.generate(input_ids, max_new_tokens, do_sample=do_sample, temperature=temperature,
                                     top_p=top_p, seed=rng_seed, offset=offset,
                                     eos_token_id=eos_list[0] if eos_list else -1, pad_token_id=pad,
                                     use_graph=use_graph, num_return_sequences=n_ret, scores=buf, **controls)
            self._draws += max_new_tokens
            self._cache_len, self._cache_batch = 0, 0       # the handle's cache now belongs to that generation
            seq = torch.cat([input_ids.repeat_interleave(n_ret, 0), new], dim=1)
            return self._decoder_output(seq, buf, new.shape[1]) if return_dict else seq
        # ---- HF-shaped loop (padding masks, several eos ids): one forward per token from Python ----
        if n_ret > 1:   # transformers' _expand_inputs_for_generation: every prompt n_ret times, prompt-major
            input_ids = input_ids.repeat_interleave(n_ret, 0)
            attention_mask = attention_mask.repeat_interleave(n_ret, 0) if attention_mask is not None else None
            B = input_ids.shape[0]
            self._reserve(B)
        mask = attention_mask.to(self._device) if attention_mask is not None else None
        buf = L.scores_buffer(max_new_tokens, B, self._llm.vocab, self._device) if want_scores else None
        seq, past = input_ids, None
        unfinished = torch.ones(B, dtype=torch.bool, device=self._device)
        for step in range(max_new_tokens):
            mi = self.prepare_inputs_for_generation(seq, past_key_values=past, attention_mask=mask, use_cache=True)
            out = self.forward(input_ids=mi["input_ids"], position_ids=mi["position_ids"],
                               past_key_values=mi["past_key_values"], use_cache=True, last_logits_only=True)
            past = out.past_key_values
            nxt = L.sample(out.logits[:, -1], do_sample=do_sample, temperature=temperature, top_p=top_p,
                           seed=rng_seed, offset=offset, step=step, history=seq, prompt_len=S,
                           eos_token_id=eos_list[0] if eos_list else -1,
                           scores_out=buf[step] if buf is not None else None, **controls)
            nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad))
            seq = torch.cat([seq, nxt[:, None]], dim=1)
            if mask is not None:
                mask = torch.cat([mask, mask.new_ones((B, 1))], dim=1)
            for e in eos_list:
                unfinished = unfinished & (nxt != e)
            if eos_list and not bool(unfinished.any()):
                break
        self._draws += max_new_tokens
        return self._decoder_output(seq, buf, seq.shape[1] - S) if return_dict else seq

    def _decoder_output(self, seq, buf, steps):
        """transformers' GenerateDecoderOnlyOutput; `scores` are views of the first `steps` steps of the scores
        buffer (None when none was made)"""
        scores = None if buf is None else tuple(buf[t, :, :self._llm.vocab] for t in range(steps))
        return GenerateDecoderOnlyOutput(sequences=seq, scores=scores)

    def compute_transition_scores(self, sequences: torch.Tensor, scores: Tuple[torch.Tensor],
                                  beam_indices: Optional[torch.Tensor] = None,
                                  normalize_logits: bool = False) -> torch.Tensor:
        """transformers' GenerationMixin.compute_transition_scores: the score of each generated token, gathered from
        the stacked `scores` (log_softmax over the vocabulary first when normalize_logits), beams followed through
        `beam_indices` (-1: past the hypothesis' end, scored 0).  The installed implementation is called: it is the
        algorithm of transformers 4.30.2 and reads only self.config."""
        return GenerationMixin.compute_transition_scores(self, sequences, scores, beam_indices=beam_indices,
                                                         normalize_logits=normalize_logits)

    def _reserve(self, rows):
        """grow the handle to `rows` rows; the cache is reallocated, so earlier past_key_values are void"""
        if rows > self.max_batch:
            self._llm.reserve_rows(rows)
            self.max_batch = rows

    def _beam_generate(self, input_ids, max_new_tokens, num_beams, do_sample, temperature, top_p, length_penalty,
                       early_stopping, eos_list, pad, padded, rng_seed, offset, use_graph, controls, n_ret=1,
                       want_scores=False):
        """-> GenerateBeamDecoderOnlyOutput; with want_scores its scores, sequences_scores and beam_indices are set"""
        if num_beams > 8:
            raise ValueError(f"num_beams={num_beams}: at most 8 beams (the scorer runs one CTA per sequence)")
        if padded:
            raise NotImplementedError("a padding attention_mask is not supported with num_beams > 1")
        if len(eos_list) > 1:
            raise NotImplementedError("several eos_token_id values are not supported with num_beams > 1")
        if early_stopping not in (False, True, "never"):
            raise ValueError(f"early_stopping must be False, True or 'never' (got {early_stopping!r})")
        if do_sample and temperature <= 0.0:
            raise ValueError(f"temperature must be > 0 when sampling (got {temperature})")
        B, S = input_ids.shape
        G = B * n_ret
        self._reserve(G * num_beams)
        buf = bi = None
        if want_scores:
            buf = L.scores_buffer(max_new_tokens, G * num_beams, self._llm.vocab, self._device)
            bi = torch.empty((G, S + max_new_tokens), dtype=torch.int64, device=self._device)
        res = self._llm.beam_generate(input_ids, max_new_tokens, num_beams, do_sample=do_sample,
                                      temperature=temperature if do_sample else 1.0, top_p=top_p,
                                      length_penalty=length_penalty, early_stopping=early_stopping, seed=rng_seed,
                                      offset=offset, eos_token_id=eos_list[0] if eos_list else -1,
                                      pad_token_id=pad, use_graph=use_graph, num_return_sequences=n_ret, scores=buf,
                                      beam_indices=bi, **controls)
        self._draws += max_new_tokens
        self._cache_len, self._cache_batch = 0, 0
        seq = torch.cat([input_ids.repeat_interleave(n_ret, 0), res[0]], dim=1)
        if not want_scores:     # 4.30.2 drops sequences_scores without output_scores
            return GenerateBeamDecoderOnlyOutput(sequences=seq)
        # len(scores): BeamSearchScorer.process calls, recorded on the device; it can exceed the generated width
        return GenerateBeamDecoderOnlyOutput(sequences=seq, sequences_scores=res[1],
                                             scores=tuple(buf[t, :, :self._llm.vocab] for t in range(res[2])),
                                             beam_indices=bi[:, :seq.shape[1]])


    def _contrastive_generate(self, input_ids, max_new_tokens, top_k, penalty_alpha, eos_list, pad, padded, use_graph,
                              controls, return_dict=False, want_scores=False):
        if top_k > 8:
            raise ValueError(f"top_k={top_k} with penalty_alpha: contrastive search takes at most 8 candidates")
        if not math.isfinite(penalty_alpha):
            raise ValueError(f"penalty_alpha must be finite (got {penalty_alpha})")
        if padded:
            raise NotImplementedError("a padding attention_mask is not supported with contrastive search")
        if len(eos_list) > 1:
            raise NotImplementedError("several eos_token_id values are not supported with contrastive search")
        B = input_ids.shape[0]
        self._reserve(B * top_k)
        buf = L.scores_buffer(max_new_tokens, B, self._llm.vocab, self._device) if want_scores else None
        new = self._llm.contrastive_generate(input_ids, max_new_tokens, top_k, penalty_alpha,
                                             eos_token_id=eos_list[0] if eos_list else -1, pad_token_id=pad,
                                             use_graph=use_graph, scores=buf,
                                             **{k: v for k, v in controls.items() if k != "top_k"})
        self._cache_len, self._cache_batch = 0, 0
        seq = torch.cat([input_ids, new], dim=1)
        return self._decoder_output(seq, buf, new.shape[1]) if return_dict else seq


def get_pretrained_llama_causal_model(pretrained_model_name_or_path=None, torch_dtype="fp16", **kwargs):
    """models/model_tools.py:5-18.  Like the reference, anything that is not one of the four dtype strings passes
    through unchanged (its `else: torch_dtype == torch.float32` is a no-op comparison), which is what lets
    scripts/seed_llama_inference_8B.py:77 call it with `torch_dtype=torch.float16`."""
    if torch_dtype in ("fp16", "float16"):
        torch_dtype = torch.float16
    elif torch_dtype in ("bf16", "bfloat16"):
        torch_dtype = torch.bfloat16
    kwargs.pop("low_cpu_mem_usage", None)
    return LlamaForCausalLM.from_pretrained(pretrained_model_name_or_path=pretrained_model_name_or_path,
                                            torch_dtype=torch_dtype, **kwargs)
