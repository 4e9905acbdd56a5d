"""Host-side mirror of models/llama_xformer.py (LlamaForCausalLM) on top of libseedb200.

`forward()` keeps the reference signature and returns transformers' CausalLMOutputWithPast
(llama_xformer.py:661-743); `generate()` stands in for HF GenerationMixin (scripts/seed_llama_inference_8B.py:33):
by default one C call that keeps prefill, sampling and the graph-replayed decode steps on the device.

Reference behaviours kept on purpose (SURVEY.md section 7 "quirks"):
  * padding in `attention_mask` is ignored by attention -- the reference only tests `attention_mask.sum() == 0`
    to choose between a causal and an unmasked xformers call (llama_xformer.py:240-256);
  * q_len == 1 attends to the whole cache without a mask; q_len > 1 is causal;
  * logits are returned for every position in fp16.
`load_in_8bit=True` runs the seven linear layers of every decoder layer as LLM.int8() (transformers' bitsandbytes
path, threshold `llm_int8_threshold`): int8 weights with per-row scales, per-call activation quantisation with fp16
outlier columns; embed_tokens, lm_head and the norms stay fp16 (include/seedb200.h states the arithmetic).
Differences: `past_key_values` are views of the handle's preallocated cache (no torch.cat per step);
`output_attentions` / `output_hidden_states` are not available (the reference's xformers path never computed
attention weights either).
"""
from __future__ import annotations

import glob
import json
import os
from typing import List, Optional, Tuple, Union

import torch
import torch.nn as nn
from transformers.modeling_outputs import CausalLMOutputWithPast
from transformers.models.llama.configuration_llama import LlamaConfig

from . import lib as L


class _CudaView:
    def __init__(self, ptr: int, shape, strides_elems):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f2", "data": (ptr, False), "version": 3,
                                         "strides": tuple(s * 2 for s in strides_elems)}


_INT8_LINEARS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def _is_int8_linear(name: str) -> bool:
    """the decoder-layer nn.Linear weights transformers' load_in_8bit replaces (lm_head is kept in fp16)"""
    parts = name.split(".")
    return ".layers." in name and len(parts) >= 2 and parts[-1] == "weight" and parts[-2] in _INT8_LINEARS


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
    """(name, tensor) of the int8 linears; a state dict that makes its tensors on demand (its items() is a generator)
    is walked again rather than indexed, so nothing is made twice at once"""
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
                 llm_int8_threshold: float = 6.0):
        super().__init__()
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
        self.is_loaded_in_8bit = bool(load_in_8bit)
        if load_in_8bit:
            # the handle is made with the fp16 tensors only; then each linear goes to the device in fp16, is quantised
            # straight into the handle's int8 buffers, and is dropped before the next: device memory stays at the
            # int8 model plus one fp16 tensor
            weights, linears = {}, []
            items = iter(state_dict.items())
            for k, v in items:
                if "rotary_emb" in k:
                    continue
                if _is_int8_linear(k):
                    linears.append(k)
                    continue
                weights[k] = v.detach().to(device=dev, dtype=torch.float16).contiguous()
            self._weight_bytes = sum(t.numel() * t.element_size() for t in weights.values())
            self._llm = L.Llama(weights, hidden=h, layers=nl, heads=nh, ffn=config.intermediate_size,
                                vocab=config.vocab_size, max_batch=max_batch, max_seq=self.max_seq,
                                rms_eps=config.rms_norm_eps, gemm_ctas=gemm_ctas,
                                int8_threshold=float(llm_int8_threshold))
            for k, v in _linear_items(state_dict, linears):
                w16 = v.detach().to(device=dev, dtype=torch.float16)
                if w16.stride(-1) != 1:
                    w16 = w16.contiguous()
                self._llm.int8_load_weight(k, w16)
                # int8 values plus one fp32 scale per row
                self._weight_bytes += w16.shape[0] * w16.shape[1] + 4 * w16.shape[0]
                del w16, v     # stream-ordered: the allocator reuses this block only after the kernel has read it
        else:
            weights = {k: v.detach().to(device=dev, dtype=torch.float16).contiguous() for k, v in state_dict.items()
                       if "rotary_emb" not in k}
            # device bytes of the weights the handle owns or borrows (HF get_memory_footprint: no KV cache / workspace)
            self._weight_bytes = sum(t.numel() * t.element_size() for t in weights.values())
            self._llm = L.Llama(weights, hidden=h, layers=nl, heads=nh, ffn=config.intermediate_size,
                                vocab=config.vocab_size, max_batch=max_batch, max_seq=self.max_seq,
                                rms_eps=config.rms_norm_eps, gemm_ctas=gemm_ctas)
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
        `llm_int8_threshold` and a single-device `device_map` are honoured as transformers does."""
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
        kwargs = {k: v for k, v in kwargs.items()
                  if k in ("max_batch", "max_seq", "gemm_ctas", "load_in_8bit", "llm_int8_threshold")}
        return cls(config, sd, device=device, **kwargs)

    # ---- nn.Module conveniences ------------------------------------------------------------------
    @property
    def device(self):
        return self._device

    def eval(self):
        return self

    def get_memory_footprint(self) -> int:
        """device bytes of the model's weights (int8 linears count their int8 values and fp32 scales); the KV cache
        and workspaces are excluded, as in transformers."""
        return int(self._weight_bytes)

    def half(self):
        return self

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
                     "length_penalty": 1.0, "early_stopping": False, "num_return_sequences": 1}

    @torch.no_grad()
    def generate(self, input_ids=None, inputs=None, max_new_tokens: Optional[int] = None,
                 do_sample: Optional[bool] = None, temperature: Optional[float] = None, top_p: Optional[float] = None,
                 num_beams: Optional[int] = None, eos_token_id=None, pad_token_id=None, attention_mask=None,
                 generator: Optional[torch.Generator] = None, seed: Optional[int] = None, use_graph: bool = True,
                 device_loop: Optional[bool] = None, generation_config=None, length_penalty: Optional[float] = None,
                 early_stopping=None, num_return_sequences: Optional[int] = None, **_):
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
        "never"); only `num_return_sequences=1`, an unpadded batch and one eos id.  B * num_beams rows must fit the
        handle: a model built with a smaller `max_batch` grows to it first, which drops the KV cache, so
        `past_key_values` returned by earlier forward() calls are no longer valid.
        `generation_config` (a transformers GenerationConfig) supplies these fields and its eos / pad ids, and
        explicit keyword arguments override it, as in transformers."""
        given = {"max_new_tokens": max_new_tokens, "do_sample": do_sample, "temperature": temperature, "top_p": top_p,
                 "num_beams": num_beams, "length_penalty": length_penalty, "early_stopping": early_stopping,
                 "num_return_sequences": num_return_sequences}
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
        if int(opts["num_return_sequences"]) != 1:
            raise NotImplementedError("num_return_sequences > 1 is not supported")
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
        if num_beams > 1:
            return self._beam_generate(input_ids, max_new_tokens, num_beams, do_sample, temperature, top_p,
                                       float(opts["length_penalty"]), opts["early_stopping"], eos_list, pad, padded,
                                       rng_seed, offset, use_graph)
        if device_loop is None:
            device_loop = (not padded) and len(eos_list) <= 1 and B <= 4
        if device_loop:
            if padded or len(eos_list) > 1 or B > 4:
                raise ValueError("device_loop needs an unpadded batch of <= 4 sequences and at most one eos id")
            new = self._llm.generate(input_ids, max_new_tokens, do_sample=do_sample, temperature=temperature,
                                     top_p=top_p, seed=rng_seed, offset=offset,
                                     eos_token_id=eos_list[0] if eos_list else -1, pad_token_id=pad,
                                     use_graph=use_graph)
            self._draws += max_new_tokens
            self._cache_len, self._cache_batch = 0, 0       # the handle's cache now belongs to that generation
            return torch.cat([input_ids, new], dim=1)
        # ---- HF-shaped loop (padding masks, several eos ids): one forward per token from Python ----
        mask = attention_mask.to(self._device) if attention_mask is not None else None
        seq, past = input_ids, None
        unfinished = torch.ones(B, dtype=torch.bool, device=self._device)
        for step in range(max_new_tokens):
            mi = self.prepare_inputs_for_generation(seq, past_key_values=past, attention_mask=mask, use_cache=True)
            out = self.forward(input_ids=mi["input_ids"], position_ids=mi["position_ids"],
                               past_key_values=mi["past_key_values"], use_cache=True, last_logits_only=True)
            past = out.past_key_values
            nxt = L.sample(out.logits[:, -1], do_sample=do_sample, temperature=temperature, top_p=top_p,
                           seed=rng_seed, offset=offset, step=step)
            nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad))
            seq = torch.cat([seq, nxt[:, None]], dim=1)
            if mask is not None:
                mask = torch.cat([mask, mask.new_ones((B, 1))], dim=1)
            for e in eos_list:
                unfinished = unfinished & (nxt != e)
            if eos_list and not bool(unfinished.any()):
                break
        self._draws += max_new_tokens
        return seq

    def _beam_generate(self, input_ids, max_new_tokens, num_beams, do_sample, temperature, top_p, length_penalty,
                       early_stopping, eos_list, pad, padded, rng_seed, offset, use_graph):
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
        B = input_ids.shape[0]
        if B * num_beams > self.max_batch:
            self._llm.reserve_rows(B * num_beams)       # the cache is reallocated: earlier past_key_values are void
            self.max_batch = B * num_beams
        new, _ = self._llm.beam_generate(input_ids, max_new_tokens, num_beams, do_sample=do_sample,
                                         temperature=temperature if do_sample else 1.0, top_p=top_p,
                                         length_penalty=length_penalty, early_stopping=early_stopping, seed=rng_seed,
                                         offset=offset, eos_token_id=eos_list[0] if eos_list else -1,
                                         pad_token_id=pad, use_graph=use_graph)
        self._draws += max_new_tokens
        self._cache_len, self._cache_batch = 0, 0
        return torch.cat([input_ids, new], dim=1)


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
