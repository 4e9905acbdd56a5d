"""ctypes binding of libseedb200.so (the C ABI declared in include/seedb200.h).

This is the binding a reference maintainer would add under models/ (see INTEGRATION.md): tensors are
passed as raw device pointers (`tensor.data_ptr()`) plus the current CUDA stream.  There is NO CPU or
PyTorch fallback: if the library is missing, cannot be loaded, or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libseedb200.so")

ACT_NONE, ACT_GELU, ACT_TANH, ACT_RELU = 0, 1, 2, 3
GEMM_COOPERATIVE, GEMM_PINGPONG = 1, 2     # enum seedb200_gemm_schedule (GemmDesc.wg_schedule; 0 = auto)
VQ_FP16, VQ_FP32 = 0, 1

# every symbol include/seedb200.h declares (tests check the library exports all of them)
EXPORTS = [
    "seedb200_version", "seedb200_last_error", "seedb200_launch_count", "seedb200_reset_launch_count",
    "seedb200_profile_begin", "seedb200_profile_end", "seedb200_set_option",
    "seedb200_gemm", "seedb200_layernorm", "seedb200_rmsnorm", "seedb200_attention", "seedb200_vq_argmin",
    "seedb200_patchify", "seedb200_rope_kv_append", "seedb200_embedding",
    "seedb200_encoder_create", "seedb200_encoder_destroy", "seedb200_encoder_encode",
    "seedb200_encoder_encode_host", "seedb200_encoder_detokenize", "seedb200_encoder_tap",
    "seedb200_llama_create", "seedb200_llama_destroy", "seedb200_llama_forward", "seedb200_llama_kv_ptrs",
    "seedb200_llama_kv_load", "seedb200_llama_tap",
    "seedb200_preprocess_create", "seedb200_preprocess_destroy", "seedb200_preprocess_run",
    "seedb200_preprocess_create_ex",
    "seedb200_gemv", "seedb200_decode_attention", "seedb200_decode_attention_workspace_bytes",
    "seedb200_sample", "seedb200_philox_uniform", "seedb200_image_ids_to_tokens", "seedb200_encoder_encode_tokens",
    "seedb200_llama_forward_ld", "seedb200_llama_generate", "seedb200_llama_generate_used_graph",
    "seedb200_row_stats", "seedb200_row_stats_from_moments", "seedb200_ln_fold_weights",
    "seedb200_gemm_plan", "seedb200_gemm_schedule_tile", "seedb200_gemm_plan_schedule", "seedb200_decode_attention_rope",
    "seedb200_int8_quantize_weight", "seedb200_int8_quantize_act", "seedb200_gemm_int8", "seedb200_gemv_int8",
    "seedb200_llama_create_int8", "seedb200_llama_int8_load_weight",
    "seedb200_beam_select", "seedb200_llama_beam_generate", "seedb200_llama_reserve_rows",
    "seedb200_decode_attention_lineage", "seedb200_decode_attention_rope_lineage",
    "seedb200_lora_shrink", "seedb200_gemm_lora", "seedb200_gemv_lora", "seedb200_llama_lora_load",
    "seedb200_llama_lora_merge", "seedb200_llama_replace_weights",
    "seedb200_quantize_4bit", "seedb200_dequantize_4bit", "seedb200_gemv_4bit", "seedb200_llama_create_4bit",
    "seedb200_llama_4bit_load_weight",
    "seedb200_sample_processed", "seedb200_llama_generate_processed", "seedb200_llama_beam_generate_processed",
    "seedb200_llama_contrastive_generate", "seedb200_contrastive_candidates", "seedb200_contrastive_rank",
    "seedb200_contrastive_context_init",
    "seedb200_llama_generate_n", "seedb200_llama_generate_n_processed", "seedb200_llama_beam_generate_n",
    "seedb200_llama_beam_generate_n_processed",
    "seedb200_sample_scores", "seedb200_llama_generate_ex", "seedb200_llama_contrastive_generate_ex",
    "seedb200_llama_beam_generate_ex",
]

DTYPE_F16, DTYPE_F32, DTYPE_I8 = 0, 1, 4
Q4_FP4, Q4_NF4 = 0, 1       # enum seedb200_quant4
_Q4_TYPES = {"fp4": Q4_FP4, "nf4": Q4_NF4}
_DTYPE_CODE = {torch.float16: DTYPE_F16, torch.float32: DTYPE_F32, torch.int8: DTYPE_I8}


class Tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("dtype", C.c_int32), ("ndim", C.c_int32),
                ("shape", C.c_int64 * 4)]


class GemmDesc(C.Structure):
    _fields_ = [("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
                ("A", C.c_void_p), ("lda", C.c_int64),
                ("W", C.c_void_p), ("ldw", C.c_int64),
                ("out", C.c_void_p), ("ldo", C.c_int64),
                ("bias", C.c_void_p),
                ("residual", C.c_void_p), ("ldr", C.c_int64),
                ("act", C.c_int32), ("mode", C.c_int32),
                ("row_group", C.c_int32), ("row_stride", C.c_int32), ("row_offset", C.c_int32),
                ("res_mod", C.c_int32), ("res_offset", C.c_int32),
                ("bn", C.c_int32), ("ctas", C.c_int32),
                ("ln_stats", C.c_void_p), ("ln_c", C.c_void_p), ("ln_b", C.c_void_p),
                ("row_moments", C.c_void_p), ("wg_schedule", C.c_int32)]


class GemmInt8Desc(C.Structure):
    _fields_ = [("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
                ("A", C.c_void_p), ("lda", C.c_int64), ("SCA", C.c_void_p),
                ("A16", C.c_void_p), ("lda16", C.c_int64),
                ("outliers", C.c_void_p), ("n_outliers", C.c_void_p),
                ("W", C.c_void_p), ("ldw", C.c_int64), ("SCB", C.c_void_p),
                ("out", C.c_void_p), ("ldo", C.c_int64),
                ("residual", C.c_void_p), ("ldr", C.c_int64),
                ("mode", C.c_int32), ("bn", C.c_int32), ("workspace", C.c_void_p)]


class LoraOperand(C.Structure):
    _fields_ = [("T", C.c_void_p), ("ldt", C.c_int64), ("B", C.c_void_p), ("r", C.c_int32), ("grp", C.c_int32),
                ("nsub", C.c_int32), ("mask", C.c_uint32), ("scale", C.c_float), ("workspace", C.c_void_p)]


class GemmLoraDesc(C.Structure):
    _fields_ = [("gemm", GemmDesc), ("lora", LoraOperand)]


class AttnDesc(C.Structure):
    _fields_ = [("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("o", C.c_void_p),
                ("q_bs", C.c_int64), ("q_hs", C.c_int64), ("q_ts", C.c_int64),
                ("k_bs", C.c_int64), ("k_hs", C.c_int64), ("k_ts", C.c_int64),
                ("v_bs", C.c_int64), ("v_hs", C.c_int64), ("v_ts", C.c_int64),
                ("o_bs", C.c_int64), ("o_hs", C.c_int64), ("o_ts", C.c_int64),
                ("batch", C.c_int32), ("heads", C.c_int32), ("nq", C.c_int32), ("nk", C.c_int32),
                ("head_dim", C.c_int32), ("causal", C.c_int32), ("scale", C.c_float)]


class EncoderConfig(C.Structure):
    _fields_ = [("vit_depth", C.c_int32), ("qformer_layers", C.c_int32), ("detok_depth", C.c_int32),
                ("n_codes", C.c_int32), ("max_batch", C.c_int32), ("vq_mode", C.c_int32),
                ("gemm_ctas", C.c_int32)]


class LlamaConfig(C.Structure):
    _fields_ = [("hidden", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32),
                ("ffn", C.c_int32), ("vocab", C.c_int32), ("max_batch", C.c_int32), ("max_seq", C.c_int32),
                ("rms_eps", C.c_float), ("rope_base", C.c_float), ("gemm_ctas", C.c_int32)]


class SampleParams(C.Structure):
    _fields_ = [("do_sample", C.c_int32), ("temperature", C.c_float), ("top_p", C.c_float), ("seed", C.c_uint64),
                ("offset", C.c_uint64)]


class BeamParams(C.Structure):
    _fields_ = [("num_beams", C.c_int32), ("do_sample", C.c_int32), ("temperature", C.c_float), ("top_p", C.c_float),
                ("length_penalty", C.c_double), ("early_stopping", C.c_int32), ("seed", C.c_uint64),
                ("offset", C.c_uint64)]


class LogitsParams(C.Structure):
    _fields_ = [("top_k", C.c_int32), ("repetition_penalty", C.c_float), ("no_repeat_ngram_size", C.c_int32),
                ("min_length", C.c_int32), ("min_new_tokens", C.c_int32)]


class ContrastiveParams(C.Structure):
    _fields_ = [("top_k", C.c_int32), ("penalty_alpha", C.c_double)]


class GenOutputs(C.Structure):
    _fields_ = [("scores", C.c_void_p), ("scores_pitch", C.c_int64), ("beam_indices", C.c_void_p),
                ("n_steps_out", C.c_int32)]


def scores_buffer(steps: int, rows: int, V: int, device) -> torch.Tensor:
    """the fp16 [steps, rows, pitch] buffer the scores outputs write: the pitch is V rounded up to a multiple of 8, so
    every row starts 16-byte aligned; callers see the [..., :V] view"""
    return torch.empty((steps, rows, (V + 7) // 8 * 8), dtype=torch.float16, device=device)


def logits_params(top_k: int = 0, repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0,
                  min_length: int = 0, min_new_tokens: int = 0) -> Optional[LogitsParams]:
    """seedb200_logits_params, or None when every control is neutral (the entry points then take their old path).
    Range checks are the C side's: it refuses bad values before any device work."""
    p = LogitsParams(int(top_k), float(repetition_penalty), int(no_repeat_ngram_size), int(min_length),
                     int(min_new_tokens))
    neutral = (p.top_k == 0 and p.repetition_penalty == 1.0 and p.no_repeat_ngram_size == 0 and p.min_length == 0
               and p.min_new_tokens == 0)
    return None if neutral else p


def _history_active(lp: Optional[LogitsParams], eos: int) -> bool:
    return lp is not None and (lp.repetition_penalty != 1.0 or lp.no_repeat_ngram_size > 0
                               or (eos >= 0 and (lp.min_length > 0 or lp.min_new_tokens > 0)))


# early_stopping of transformers' GenerationConfig -> seedb200_beam_params.early_stopping
EARLY_STOPPING = {False: 0, True: 1, "never": 2}


def beam_params(num_beams: int, do_sample: bool = False, temperature: float = 1.0, top_p: float = 1.0,
                length_penalty: float = 1.0, early_stopping=False, seed: int = 0, offset: int = 0) -> BeamParams:
    if early_stopping not in EARLY_STOPPING:
        raise ValueError(f"early_stopping must be False, True or 'never' (got {early_stopping!r})")
    return BeamParams(int(num_beams), int(bool(do_sample)), float(temperature), float(top_p), float(length_penalty),
                      EARLY_STOPPING[early_stopping], int(seed), int(offset))


_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the shared library (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m seed_b200.build` (needs nvcc, sm_90a). "
            "seed_b200 has no CPU or PyTorch fallback path.")
    lib = C.CDLL(LIB_PATH)
    lib.seedb200_version.restype = C.c_int
    lib.seedb200_last_error.restype = C.c_char_p
    lib.seedb200_launch_count.restype = C.c_int64
    lib.seedb200_reset_launch_count.restype = None
    lib.seedb200_profile_end.argtypes = [C.POINTER(C.c_double)]
    lib.seedb200_gemm.argtypes = [C.POINTER(GemmDesc), C.c_void_p]
    lib.seedb200_layernorm.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                       C.c_int, C.c_int, C.c_float, C.c_void_p]
    lib.seedb200_rmsnorm.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int,
                                     C.c_float, C.c_void_p]
    lib.seedb200_attention.argtypes = [C.POINTER(AttnDesc), C.c_void_p]
    lib.seedb200_vq_argmin.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                       C.c_void_p]
    lib.seedb200_patchify.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    lib.seedb200_rope_kv_append.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.seedb200_embedding.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                       C.c_int64, C.c_void_p]
    lib.seedb200_encoder_create.argtypes = [C.POINTER(EncoderConfig), C.POINTER(Tensor), C.c_int,
                                            C.POINTER(C.c_void_p)]
    lib.seedb200_encoder_destroy.argtypes = [C.c_void_p]
    lib.seedb200_encoder_destroy.restype = None
    lib.seedb200_preprocess_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
    lib.seedb200_preprocess_destroy.argtypes = [C.c_void_p]
    lib.seedb200_preprocess_destroy.restype = None
    lib.seedb200_preprocess_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.seedb200_encoder_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p]
    lib.seedb200_encoder_encode_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.seedb200_encoder_detokenize.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.seedb200_encoder_tap.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    lib.seedb200_encoder_tap.restype = C.c_int64
    lib.seedb200_llama_create.argtypes = [C.POINTER(LlamaConfig), C.POINTER(Tensor), C.c_int,
                                          C.POINTER(C.c_void_p)]
    lib.seedb200_llama_destroy.argtypes = [C.c_void_p]
    lib.seedb200_llama_destroy.restype = None
    lib.seedb200_llama_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.seedb200_llama_kv_ptrs.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
    lib.seedb200_llama_kv_load.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                           C.c_void_p]
    lib.seedb200_llama_tap.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    lib.seedb200_llama_tap.restype = C.c_int64
    lib.seedb200_row_stats.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    lib.seedb200_row_stats_from_moments.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    lib.seedb200_ln_fold_weights.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.seedb200_preprocess_create_ex.argtypes = [C.c_int] * 9 + [C.POINTER(C.c_void_p)]
    lib.seedb200_gemv.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float,
                                  C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.seedb200_decode_attention_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.seedb200_decode_attention_workspace_bytes.restype = C.c_int64
    lib.seedb200_decode_attention.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                              C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    lib.seedb200_sample.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.POINTER(SampleParams), C.c_uint64,
                                    C.c_void_p, C.c_void_p]
    lib.seedb200_philox_uniform.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32]
    lib.seedb200_philox_uniform.restype = C.c_float
    lib.seedb200_image_ids_to_tokens.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
                                                 C.c_int64, C.c_void_p]
    lib.seedb200_encoder_encode_tokens.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int64,
                                                   C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.seedb200_llama_forward_ld.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                              C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    lib.seedb200_llama_generate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(SampleParams),
                                            C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.c_void_p]
    lib.seedb200_llama_generate_used_graph.argtypes = [C.c_void_p]
    lib.seedb200_int8_quantize_weight.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                                  C.c_void_p]
    lib.seedb200_int8_quantize_act.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_float, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.seedb200_gemm_int8.argtypes = [C.POINTER(GemmInt8Desc), C.c_void_p]
    lib.seedb200_gemv_int8.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.seedb200_llama_create_int8.argtypes = [C.POINTER(LlamaConfig), C.POINTER(Tensor), C.c_int, C.c_float,
                                               C.POINTER(C.c_void_p)]
    lib.seedb200_llama_int8_load_weight.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.seedb200_beam_select.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                         C.POINTER(BeamParams), C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.seedb200_llama_beam_generate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                 C.POINTER(BeamParams), C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                                 C.POINTER(C.c_int), C.c_void_p, C.c_void_p]
    lib.seedb200_llama_reserve_rows.argtypes = [C.c_void_p, C.c_int]
    lib.seedb200_decode_attention_lineage.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                      C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                                      C.c_void_p, C.c_void_p]
    lib.seedb200_lora_shrink.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_int,
                                         C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
    lib.seedb200_gemm_lora.argtypes = [C.POINTER(GemmLoraDesc), C.c_void_p]
    lib.seedb200_gemv_lora.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_float, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(LoraOperand),
                                       C.c_void_p]
    lib.seedb200_llama_lora_load.argtypes = [C.c_void_p, C.POINTER(Tensor), C.c_int, C.c_int, C.c_float]
    lib.seedb200_llama_lora_merge.argtypes = [C.c_void_p]
    lib.seedb200_llama_replace_weights.argtypes = [C.c_void_p, C.POINTER(Tensor), C.c_int]
    lib.seedb200_quantize_4bit.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                           C.c_void_p]
    lib.seedb200_dequantize_4bit.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                             C.c_void_p]
    lib.seedb200_gemv_4bit.argtypes = [C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                       C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.seedb200_llama_create_4bit.argtypes = [C.POINTER(LlamaConfig), C.POINTER(Tensor), C.c_int, C.c_int,
                                               C.POINTER(C.c_void_p)]
    lib.seedb200_llama_4bit_load_weight.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.seedb200_sample_processed.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.POINTER(SampleParams),
                                              C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(LogitsParams), C.c_void_p,
                                              C.c_int64, C.c_int, C.c_int, C.c_int64]
    lib.seedb200_llama_generate_processed.argtypes = lib.seedb200_llama_generate.argtypes + [C.POINTER(LogitsParams)]
    lib.seedb200_llama_beam_generate_processed.argtypes = (lib.seedb200_llama_beam_generate.argtypes
                                                           + [C.POINTER(LogitsParams)])
    lib.seedb200_llama_contrastive_generate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                        C.POINTER(ContrastiveParams), C.c_int64, C.c_int64, C.c_int,
                                                        C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(LogitsParams)]
    lib.seedb200_llama_generate_n.argtypes = (lib.seedb200_llama_generate.argtypes[:5] + [C.c_int]
                                              + lib.seedb200_llama_generate.argtypes[5:])
    lib.seedb200_llama_generate_n_processed.argtypes = lib.seedb200_llama_generate_n.argtypes + [C.POINTER(LogitsParams)]
    lib.seedb200_llama_beam_generate_n.argtypes = (lib.seedb200_llama_beam_generate.argtypes[:5] + [C.c_int]
                                                   + lib.seedb200_llama_beam_generate.argtypes[5:])
    lib.seedb200_llama_beam_generate_n_processed.argtypes = (lib.seedb200_llama_beam_generate_n.argtypes
                                                             + [C.POINTER(LogitsParams)])
    lib.seedb200_sample_scores.argtypes = lib.seedb200_sample_processed.argtypes + [C.c_void_p, C.c_int64]
    lib.seedb200_llama_generate_ex.argtypes = (lib.seedb200_llama_generate_n_processed.argtypes
                                               + [C.POINTER(GenOutputs)])
    lib.seedb200_llama_beam_generate_ex.argtypes = (lib.seedb200_llama_beam_generate_n_processed.argtypes
                                                    + [C.POINTER(GenOutputs)])
    lib.seedb200_llama_contrastive_generate_ex.argtypes = (lib.seedb200_llama_contrastive_generate.argtypes
                                                           + [C.POINTER(GenOutputs)])
    lib.seedb200_contrastive_candidates.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                    C.c_void_p, C.c_void_p]
    lib.seedb200_contrastive_rank.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                              C.c_void_p, C.c_int, C.POINTER(ContrastiveParams), C.c_void_p,
                                              C.c_void_p, C.c_void_p]
    lib.seedb200_contrastive_context_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                                      C.c_void_p]
    _lib = lib
    return lib


def check(status: int, what: str) -> None:
    if status != 0:
        msg = load().seedb200_last_error()
        raise RuntimeError(f"{what} failed (status {status}): {msg.decode() if msg else '?'}")


def stream_ptr(device=None) -> int:
    """the CUDA stream torch considers current ON `device` (a tensor's / handle's device, not torch's current one)"""
    return torch.cuda.current_stream(device).cuda_stream


def on(device):
    """context: make `device` current for the C call.  Kernels are launched on, and cudaFuncSetAttribute /
    occupancy caches are keyed by, the CURRENT device, while tensors and handles may live on any cuda:N
    (reference pattern: tokenizer_device != llm_device, gradio_demo/seed_llama_flask.py:51-52)."""
    return torch.cuda.device(device)


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need_cuda_f16(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"{name}: expected a CUDA tensor; seed_b200 has no CPU path (got device {t.device})")
    if t.dtype != torch.float16:
        raise RuntimeError(f"{name}: expected float16, got {t.dtype}")


def launch_count() -> int:
    return int(load().seedb200_launch_count())


def reset_launch_count() -> None:
    load().seedb200_reset_launch_count()


def set_option(key: str, value: int) -> None:
    lib = load()
    lib.seedb200_set_option.argtypes = [C.c_char_p, C.c_int]
    check(lib.seedb200_set_option(key.encode(), int(value)), "seedb200_set_option")


def profile_begin() -> None:
    check(load().seedb200_profile_begin(), "seedb200_profile_begin")


def profile_end() -> dict:
    """-> {"gemm": {"launches", "ms", "flops"}, "attention": {...}} for the kernels launched since profile_begin()."""
    out = (C.c_double * 6)()
    check(load().seedb200_profile_end(out), "seedb200_profile_end")
    return {"gemm": {"launches": int(out[0]), "ms": out[1], "flops": out[2]},
            "attention": {"launches": int(out[3]), "ms": out[4], "flops": out[5]}}


# --------------------------------------------------------------------------------------------------
# per-op wrappers (used by the tests and by ncu runs)
# --------------------------------------------------------------------------------------------------
def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: int = ACT_NONE,
         residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, mode: int = 0,
         bn: int = 0, ctas: int = 0, row_group: int = 0, row_stride: int = 0, row_offset: int = 0,
         res_mod: int = 0, res_offset: int = 0, ln=None, row_moments: Optional[torch.Tensor] = None,
         wg_schedule: int = 0) -> torch.Tensor:
    """out = epilogue(a @ w.T); a [M,K], w [N,K] fp16 (nn.Linear layout).  ln = (stats [M,2] fp32, c [N] fp32,
    b [N] fp32) selects the LayerNorm-folded epilogue (w must then be the folded weight of ln_fold_weights).
    row_moments: float32 [M, N/64, 2] that receives (sum, sum of squares) per 64-column group of the output rows.
    wg_schedule: 0 = the planner's kernel, GEMM_COOPERATIVE / GEMM_PINGPONG force one (same results)."""
    _need_cuda_f16(a, "gemm.a"); _need_cuda_f16(w, "gemm.w")
    M, K = a.shape
    N = w.shape[0]
    n_out = N // 2 if mode == 1 else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.float16, device=a.device)
    d = GemmDesc()
    d.M, d.N, d.K = M, N, K
    d.A, d.lda = a.data_ptr(), a.stride(0)
    d.W, d.ldw = w.data_ptr(), w.stride(0)
    d.out, d.ldo = out.data_ptr(), out.stride(0)
    d.bias = _p(bias)
    d.residual = _p(residual)
    d.ldr = residual.stride(0) if residual is not None else 0
    d.act, d.mode = act, mode
    d.row_group, d.row_stride, d.row_offset = row_group, row_stride, row_offset
    d.res_mod, d.res_offset = res_mod, res_offset
    d.bn, d.ctas, d.wg_schedule = bn, ctas, wg_schedule
    if ln is not None:
        stats, cvec, bvec = ln
        for t in (stats, cvec, bvec):
            if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise RuntimeError("gemm: ln tensors must be contiguous CUDA float32")
        d.ln_stats, d.ln_c, d.ln_b = stats.data_ptr(), cvec.data_ptr(), bvec.data_ptr()
    if row_moments is not None:
        if (row_moments.dtype != torch.float32 or not row_moments.is_cuda or not row_moments.is_contiguous()
                or row_moments.numel() != M * (N // 64) * 2):
            raise RuntimeError("gemm: row_moments must be contiguous CUDA float32 [M, N/64, 2]")
        d.row_moments = row_moments.data_ptr()
    with on(a.device):
        check(load().seedb200_gemm(C.byref(d), stream_ptr(a.device)), "seedb200_gemm")
    return out


def layernorm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float) -> torch.Tensor:
    _need_cuda_f16(x, "layernorm.x")
    y = torch.empty_like(x)
    rows, cols = x.shape
    with on(x.device):
        check(load().seedb200_layernorm(x.data_ptr(), x.stride(0), w.data_ptr(), b.data_ptr(), y.data_ptr(),
                                        y.stride(0), rows, cols, eps, stream_ptr(x.device)), "seedb200_layernorm")
    return y


def row_stats(x: torch.Tensor, eps: float) -> torch.Tensor:
    """(mean, rstd) per row of x [rows, cols] fp16 -> float32 [rows, 2] (LayerNorm statistics, two-pass fp32)."""
    _need_cuda_f16(x, "row_stats.x")
    rows, cols = x.shape
    out = torch.empty((rows, 2), dtype=torch.float32, device=x.device)
    with on(x.device):
        check(load().seedb200_row_stats(x.data_ptr(), x.stride(0), rows, cols, eps, out.data_ptr(), stream_ptr(x.device)),
              "seedb200_row_stats")
    return out


def row_stats_from_moments(moments: torch.Tensor, cols: int, eps: float) -> torch.Tensor:
    """moments float32 [rows, cols/64, 2] (gemm(..., row_moments=)) -> (mean, rstd) float32 [rows, 2]."""
    rows = moments.shape[0]
    out = torch.empty((rows, 2), dtype=torch.float32, device=moments.device)
    with on(moments.device):
        check(load().seedb200_row_stats_from_moments(moments.data_ptr(), rows, cols, eps, out.data_ptr(),
                                                     stream_ptr(moments.device)), "seedb200_row_stats_from_moments")
    return out


def ln_fold_weights(w: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, bias: Optional[torch.Tensor] = None):
    """-> (W' = fp16(W diag(gamma)) [N,K], c [N] fp32 = row sums of W', b' [N] fp32 = W beta + bias)."""
    _need_cuda_f16(w, "ln_fold_weights.w")
    N, K = w.shape
    wf = torch.empty((N, K), dtype=torch.float16, device=w.device)
    c = torch.empty((N,), dtype=torch.float32, device=w.device)
    b = torch.empty((N,), dtype=torch.float32, device=w.device)
    with on(w.device):
        check(load().seedb200_ln_fold_weights(w.data_ptr(), w.stride(0), gamma.data_ptr(), beta.data_ptr(), _p(bias), N, K,
                                              wf.data_ptr(), c.data_ptr(), b.data_ptr(), stream_ptr(w.device)),
              "seedb200_ln_fold_weights")
    return wf, c, b


def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    _need_cuda_f16(x, "rmsnorm.x")
    y = torch.empty_like(x)
    rows, cols = x.shape
    with on(x.device):
        check(load().seedb200_rmsnorm(x.data_ptr(), x.stride(0), w.data_ptr(), y.data_ptr(), y.stride(0), rows, cols,
                                      eps, stream_ptr(x.device)), "seedb200_rmsnorm")
    return y


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, causal: bool = False) -> torch.Tensor:
    """q [B,H,Nq,D], k/v [B,H,Nk,D] (any strides with contiguous D) -> o [B,Nq,H,D] contiguous."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _need_cuda_f16(t, "attention." + n)
        if t.stride(3) != 1:
            raise RuntimeError("attention: head_dim must be contiguous")
    B, H, Nq, D = q.shape
    Nk = k.shape[2]
    o = torch.empty((B, Nq, H, D), dtype=torch.float16, device=q.device)
    d = AttnDesc()
    d.q, d.k, d.v, d.o = q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr()
    d.q_bs, d.q_hs, d.q_ts = q.stride(0), q.stride(1), q.stride(2)
    d.k_bs, d.k_hs, d.k_ts = k.stride(0), k.stride(1), k.stride(2)
    d.v_bs, d.v_hs, d.v_ts = v.stride(0), v.stride(1), v.stride(2)
    d.o_bs, d.o_hs, d.o_ts = o.stride(0), o.stride(2), o.stride(1)
    d.batch, d.heads, d.nq, d.nk, d.head_dim = B, H, Nq, Nk, D
    d.causal, d.scale = int(causal), scale
    with on(q.device):
        check(load().seedb200_attention(C.byref(d), stream_ptr(q.device)), "seedb200_attention")
    return o


def vq_argmin(z: torch.Tensor, codebook: torch.Tensor, mode: int = VQ_FP16) -> torch.Tensor:
    _need_cuda_f16(z, "vq.z"); _need_cuda_f16(codebook, "vq.codebook")
    z2 = z.reshape(-1, z.shape[-1]).contiguous()
    ids = torch.empty((z2.shape[0],), dtype=torch.int64, device=z.device)
    with on(z.device):
        check(load().seedb200_vq_argmin(z2.data_ptr(), codebook.data_ptr(), z2.shape[0], codebook.shape[0],
                                        z2.shape[1], mode, ids.data_ptr(), stream_ptr(z.device)), "seedb200_vq_argmin")
    return ids


def patchify(images: torch.Tensor, kpad: int = 592) -> torch.Tensor:
    _need_cuda_f16(images, "patchify.images")
    B = images.shape[0]
    images = images.contiguous()
    cols = torch.empty((B * 256, kpad), dtype=torch.float16, device=images.device)
    with on(images.device):
        check(load().seedb200_patchify(images.data_ptr(), B, cols.data_ptr(), kpad, stream_ptr(images.device)),
              "seedb200_patchify")
    return cols


def rope_kv_append(qkv: torch.Tensor, positions: Optional[torch.Tensor], B: int, S: int, H: int, D: int,
                   past_len: int, k_cache: torch.Tensor, v_cache: torch.Tensor) -> torch.Tensor:
    _need_cuda_f16(qkv, "rope.qkv")
    max_seq = k_cache.shape[2]
    q_out = torch.empty((B * S, H * D), dtype=torch.float16, device=qkv.device)
    with on(qkv.device):
        check(load().seedb200_rope_kv_append(qkv.data_ptr(), _p(positions), B, S, H, D, past_len, max_seq,
                                             q_out.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                             stream_ptr(qkv.device)), "seedb200_rope_kv_append")
    return q_out


def embedding(table: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    _need_cuda_f16(table, "embedding.table")
    flat = ids.reshape(-1).contiguous()
    out = torch.empty((flat.numel(), table.shape[1]), dtype=torch.float16, device=table.device)
    with on(table.device):
        check(load().seedb200_embedding(table.data_ptr(), table.stride(0), flat.data_ptr(), flat.numel(),
                                        table.shape[1], out.data_ptr(), out.stride(0), table.shape[0],
                                        stream_ptr(table.device)), "seedb200_embedding")
    return out


class Preprocess:
    """seedb200_preprocess plan: uint8 [n,H,W,3] (device) -> fp16 [n,3,S,S], bit-exact with torchvision + Pillow.
    `resize`/`crop` select the keep_ratio=True pipeline of models/transforms.py:6-9 (Resize(S) -> CenterCrop(S)):
    resize = (h, w) of the intermediate resample, crop = (top, left) of the S x S window inside it."""

    FILTERS = {"bilinear": 2, "bicubic": 3, 2: 2, 3: 3}

    def __init__(self, in_h: int, in_w: int, out_size: int = 224, filter="bilinear", max_batch: int = 256,
                 resize=None, crop=(0, 0), device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("seedb200 preprocessing needs a CUDA device: there is no CPU path")
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.in_h, self.in_w, self.out, self.max_batch = in_h, in_w, out_size, max_batch
        rh, rw = (out_size, out_size) if resize is None else resize
        self._h = C.c_void_p()
        with on(self.device):
            check(load().seedb200_preprocess_create_ex(in_h, in_w, rh, rw, crop[0], crop[1], out_size,
                                                       self.FILTERS[filter], max_batch, C.byref(self._h)),
                  "seedb200_preprocess_create_ex")

    def __call__(self, images_u8: torch.Tensor) -> torch.Tensor:
        if images_u8.dtype != torch.uint8 or not images_u8.is_cuda:
            raise RuntimeError("preprocess: expected a CUDA uint8 tensor [n,H,W,3]")
        if images_u8.device != self.device:
            raise RuntimeError(f"preprocess: plan lives on {self.device}, images on {images_u8.device}")
        if images_u8.dim() == 3:
            images_u8 = images_u8[None]
        n = images_u8.shape[0]
        if tuple(images_u8.shape[1:]) != (self.in_h, self.in_w, 3):
            raise ValueError(f"preprocess: plan is for {self.in_h}x{self.in_w}x3 images, got {tuple(images_u8.shape)}")
        images_u8 = images_u8.contiguous()
        out = torch.empty((n, 3, self.out, self.out), dtype=torch.float16, device=images_u8.device)
        with on(self.device):
            for i in range(0, n, self.max_batch):
                m = min(self.max_batch, n - i)
                check(load().seedb200_preprocess_run(self._h, images_u8[i:i + m].data_ptr(), m, out[i:i + m].data_ptr(),
                                                     stream_ptr(self.device)), "seedb200_preprocess_run")
        return out

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h:
            load().seedb200_preprocess_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def gemv(x: torch.Tensor, w: torch.Tensor, residual: Optional[torch.Tensor] = None,
         norm_w: Optional[torch.Tensor] = None, eps: float = 1e-6, mode: int = 0) -> torch.Tensor:
    """x [M<=4, K], w [N, K] -> [M, N] (mode 0) / [M, N/2] (mode 1: silu(gate) * up over 128-row blocks)."""
    _need_cuda_f16(x, "gemv.x"); _need_cuda_f16(w, "gemv.w")
    M, K = x.shape
    N = w.shape[0]
    out = torch.empty((M, N // 2 if mode == 1 else N), dtype=torch.float16, device=x.device)
    x = x.contiguous()
    with on(x.device):
        check(load().seedb200_gemv(x.data_ptr(), w.data_ptr(), w.stride(0), out.data_ptr(), _p(residual), _p(norm_w),
                                   eps, M, N, K, mode, stream_ptr(x.device)), "seedb200_gemv")
    return out


def lora_shrink(x: torch.Tensor, a: torch.Tensor, norm_w: Optional[torch.Tensor] = None,
                eps: float = 1e-6) -> torch.Tensor:
    """LoRA shrink: x [M, K], a [r_tot, K] -> t = fp16(x . a^T) [M, r_tot].  norm_w (M <= 4): x is RMS-normalised on
    the way in, as the fused-norm GEMV does."""
    _need_cuda_f16(x, "lora_shrink.x"); _need_cuda_f16(a, "lora_shrink.a")
    M, K = x.shape
    rtot = a.shape[0]
    a = a.contiguous()
    if M <= 4:
        x = x.contiguous()
    t = torch.empty((M, rtot), dtype=torch.float16, device=x.device)
    with on(x.device):
        check(load().seedb200_lora_shrink(x.data_ptr(), x.stride(0), _p(norm_w), eps, a.data_ptr(), M, K, rtot,
                                          t.data_ptr(), rtot, stream_ptr(x.device)), "seedb200_lora_shrink")
    return t


def lora_operand(t: torch.Tensor, b: torch.Tensor, r: int, grp: int, nsub: int, scale: float, mask: Optional[int] = None,
                 workspace: Optional[torch.Tensor] = None) -> LoraOperand:
    """t [M, r * nsub] (lora_shrink output), b [N, r] in the weight's fused row layout; output row n reads the t columns
    ((n // grp) % nsub) * r + [0, r).  The caller keeps t, b and workspace alive across the call."""
    for x, nm in ((t, "t"), (b, "b")):
        _need_cuda_f16(x, f"lora.{nm}")
    if not b.is_contiguous() or t.stride(1) != 1:
        raise RuntimeError("lora: b must be contiguous and t must have contiguous columns")
    return LoraOperand(t.data_ptr(), t.stride(0), b.data_ptr(), int(r), int(grp), int(nsub),
                       (1 << nsub) - 1 if mask is None else int(mask), float(scale), _p(workspace))


def gemm_lora(a: torch.Tensor, w: torch.Tensor, lora: LoraOperand, residual: Optional[torch.Tensor] = None,
              out: Optional[torch.Tensor] = None, mode: int = 0, bn: int = 0,
              workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gemm() (mode 0 with optional residual, or mode 1) with the LoRA branch of `lora` (see include/seedb200.h)."""
    _need_cuda_f16(a, "gemm_lora.a"); _need_cuda_f16(w, "gemm_lora.w")
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N // 2 if mode == 1 else N), dtype=torch.float16, device=a.device)
    if workspace is None and (mode == 1 or residual is not None):
        workspace = torch.empty((M, N), dtype=torch.float16, device=a.device)
    d = GemmLoraDesc()
    g = d.gemm
    g.M, g.N, g.K = M, N, K
    g.A, g.lda = a.data_ptr(), a.stride(0)
    g.W, g.ldw = w.data_ptr(), w.stride(0)
    g.out, g.ldo = out.data_ptr(), out.stride(0)
    g.residual = _p(residual)
    g.ldr = residual.stride(0) if residual is not None else 0
    g.mode, g.bn = mode, bn
    d.lora = lora
    d.lora.workspace = _p(workspace)
    with on(a.device):
        check(load().seedb200_gemm_lora(C.byref(d), stream_ptr(a.device)), "seedb200_gemm_lora")
    return out


def gemv_lora(x: torch.Tensor, w: torch.Tensor, lora: LoraOperand, residual: Optional[torch.Tensor] = None,
              norm_w: Optional[torch.Tensor] = None, eps: float = 1e-6, mode: int = 0,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gemv() with the LoRA expand in its epilogue (`lora`); x [M <= 4, K] dense, out dense rows."""
    _need_cuda_f16(x, "gemv_lora.x"); _need_cuda_f16(w, "gemv_lora.w")
    M, K = x.shape
    N = w.shape[0]
    x = x.contiguous()
    if out is None:
        out = torch.empty((M, N // 2 if mode == 1 else N), dtype=torch.float16, device=x.device)
    elif not out.is_contiguous():
        raise RuntimeError("gemv_lora: out must be contiguous")
    lo = LoraOperand.from_buffer_copy(lora)
    with on(x.device):
        check(load().seedb200_gemv_lora(x.data_ptr(), w.data_ptr(), w.stride(0), out.data_ptr(), _p(residual),
                                        _p(norm_w), eps, M, N, K, mode, C.byref(lo), stream_ptr(x.device)),
              "seedb200_gemv_lora")
    return out


def int8_quantize_weight(w: torch.Tensor):
    """LLM.int8() weight quantisation: fp16 [N,K] -> (CB int8 [N,K], SCB fp32 [N])."""
    _need_cuda_f16(w, "int8_quantize_weight.w")
    N, K = w.shape
    if w.stride(1) != 1:
        w = w.contiguous()
    cb = torch.empty((N, K), dtype=torch.int8, device=w.device)
    scb = torch.empty((N,), dtype=torch.float32, device=w.device)
    with on(w.device):
        check(load().seedb200_int8_quantize_weight(w.data_ptr(), w.stride(0), N, K, cb.data_ptr(), scb.data_ptr(),
                                                   stream_ptr(w.device)), "seedb200_int8_quantize_weight")
    return cb, scb


def int8_quantize_act(a: torch.Tensor, threshold: float = 6.0):
    """LLM.int8() activation quantisation: fp16 [M,K] -> (CA int8 [M,K], SCA fp32 [M], outliers int32 [K] (the
    first n entries are the outlier columns in ascending order), n int32 [1]) -- all on the device."""
    _need_cuda_f16(a, "int8_quantize_act.a")
    M, K = a.shape
    if a.stride(1) != 1:
        a = a.contiguous()
    ca = torch.empty((M, K), dtype=torch.int8, device=a.device)
    sca = torch.empty((M,), dtype=torch.float32, device=a.device)
    ol = torch.empty((K,), dtype=torch.int32, device=a.device)
    n = torch.empty((1,), dtype=torch.int32, device=a.device)
    with on(a.device):
        check(load().seedb200_int8_quantize_act(a.data_ptr(), a.stride(0), M, K, float(threshold), ca.data_ptr(),
                                                sca.data_ptr(), ol.data_ptr(), n.data_ptr(), stream_ptr(a.device)),
              "seedb200_int8_quantize_act")
    return ca, sca, ol, n


def gemm_int8(a: torch.Tensor, cb: torch.Tensor, scb: torch.Tensor, threshold: float = 6.0,
              residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, mode: int = 0,
              bn: int = 0) -> torch.Tensor:
    """linear8(a, (cb, scb)) by activation quantisation + the int8 wgmma GEMM; a fp16 [M,K], cb int8 [N,K]."""
    _need_cuda_f16(a, "gemm_int8.a")
    a = a.contiguous()
    M, K = a.shape
    N = cb.shape[0]
    ca, sca, ol, n = int8_quantize_act(a, threshold)
    if out is None:
        out = torch.empty((M, N // 2 if mode == 1 else N), dtype=torch.float16, device=a.device)
    d = GemmInt8Desc()
    d.M, d.N, d.K = M, N, K
    d.A, d.lda, d.SCA = ca.data_ptr(), K, sca.data_ptr()
    d.A16, d.lda16 = a.data_ptr(), K
    d.outliers, d.n_outliers = ol.data_ptr(), n.data_ptr()
    d.W, d.ldw, d.SCB = cb.data_ptr(), cb.stride(0), scb.data_ptr()
    d.out, d.ldo = out.data_ptr(), out.stride(0)
    d.residual, d.ldr = _p(residual), (residual.stride(0) if residual is not None else 0)
    d.mode, d.bn = mode, bn
    ws = torch.empty((M, N), dtype=torch.float16, device=a.device)
    d.workspace = ws.data_ptr()
    with on(a.device):
        check(load().seedb200_gemm_int8(C.byref(d), stream_ptr(a.device)), "seedb200_gemm_int8")
    return out


def gemv_int8(x: torch.Tensor, cb: torch.Tensor, scb: torch.Tensor, threshold: float = 6.0,
              residual: Optional[torch.Tensor] = None, norm_w: Optional[torch.Tensor] = None, eps: float = 1e-6,
              mode: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """linear8 for M <= 4 rows by the int8 GEMV (quantisation, and RMSNorm with norm_w, inside the kernel)."""
    _need_cuda_f16(x, "gemv_int8.x")
    x = x.contiguous()
    M, K = x.shape
    N = cb.shape[0]
    if out is None:
        out = torch.empty((M, N // 2 if mode == 1 else N), dtype=torch.float16, device=x.device)
    with on(x.device):
        check(load().seedb200_gemv_int8(x.data_ptr(), _p(norm_w), eps, float(threshold), cb.data_ptr(), scb.data_ptr(),
                                        out.data_ptr(), _p(residual), M, N, K, mode, stream_ptr(x.device)),
              "seedb200_gemv_int8")
    return out


def quant4_type(quant_type) -> int:
    """"fp4" / "nf4" (bitsandbytes' bnb_4bit_quant_type) or Q4_FP4 / Q4_NF4 -> the enum value"""
    if isinstance(quant_type, str):
        if quant_type not in _Q4_TYPES:
            raise ValueError(f"bnb_4bit_quant_type must be 'fp4' or 'nf4' (got {quant_type!r})")
        return _Q4_TYPES[quant_type]
    if quant_type not in (Q4_FP4, Q4_NF4):
        raise ValueError(f"4-bit quant type must be Q4_FP4 (0) or Q4_NF4 (1) (got {quant_type!r})")
    return int(quant_type)


def quantize_4bit(w: torch.Tensor, quant_type="fp4"):
    """bitsandbytes 4-bit quantisation (blocks of 64): fp16 [N,K] -> (packed uint8 [N, K/2], absmax fp32 [N, K/64])."""
    _need_cuda_f16(w, "quantize_4bit.w")
    qt = quant4_type(quant_type)
    N, K = w.shape
    if w.stride(1) != 1 or w.stride(0) % 8 != 0 or w.data_ptr() % 16 != 0:
        w = w.contiguous()
    packed = torch.empty((N, K // 2), dtype=torch.uint8, device=w.device)
    absmax = torch.empty((N, max(K // 64, 1)), dtype=torch.float32, device=w.device)
    with on(w.device):
        check(load().seedb200_quantize_4bit(w.data_ptr(), w.stride(0), N, K, qt, packed.data_ptr(), absmax.data_ptr(),
                                            stream_ptr(w.device)), "seedb200_quantize_4bit")
    return packed, absmax


def _need_q4(packed: torch.Tensor, absmax: torch.Tensor, K: int, what: str) -> None:
    N = packed.shape[0]
    if (not packed.is_cuda or packed.dtype != torch.uint8 or tuple(packed.shape) != (N, K // 2)
            or not packed.is_contiguous()):
        raise RuntimeError(f"{what}: packed must be a contiguous CUDA uint8 [N, K/2] = [{N}, {K // 2}] tensor")
    if (not absmax.is_cuda or absmax.dtype != torch.float32 or tuple(absmax.shape) != (N, K // 64)
            or not absmax.is_contiguous()):
        raise RuntimeError(f"{what}: absmax must be a contiguous CUDA float32 [N, K/64] = [{N}, {K // 64}] tensor")


def dequantize_4bit(packed: torch.Tensor, absmax: torch.Tensor, quant_type="fp4",
                    out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """packed uint8 [N, K/2] + absmax fp32 [N, K/64] -> W' fp16 [N, K]."""
    qt = quant4_type(quant_type)
    N, K = packed.shape[0], packed.shape[1] * 2
    _need_q4(packed, absmax, K, "dequantize_4bit")
    if out is None:
        out = torch.empty((N, K), dtype=torch.float16, device=packed.device)
    with on(packed.device):
        check(load().seedb200_dequantize_4bit(packed.data_ptr(), absmax.data_ptr(), N, K, qt, out.data_ptr(),
                                              out.stride(0), stream_ptr(packed.device)), "seedb200_dequantize_4bit")
    return out


def gemv_4bit(x: torch.Tensor, packed: torch.Tensor, absmax: torch.Tensor, quant_type="fp4",
              residual: Optional[torch.Tensor] = None, norm_w: Optional[torch.Tensor] = None, eps: float = 1e-6,
              mode: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gemv() on dequantize_4bit(packed, absmax), bit for bit, for M <= 4 rows without materialising W'."""
    _need_cuda_f16(x, "gemv_4bit.x")
    qt = quant4_type(quant_type)
    x = x.contiguous()
    M, K = x.shape
    N = packed.shape[0]
    _need_q4(packed, absmax, K, "gemv_4bit")
    if out is None:
        out = torch.empty((M, N // 2 if mode == 1 else N), dtype=torch.float16, device=x.device)
    with on(x.device):
        check(load().seedb200_gemv_4bit(x.data_ptr(), _p(norm_w), eps, packed.data_ptr(), absmax.data_ptr(), qt,
                                        out.data_ptr(), _p(residual), M, N, K, mode, stream_ptr(x.device)),
              "seedb200_gemv_4bit")
    return out


def decode_attention(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, kv_len: int,
                     scale: float) -> torch.Tensor:
    """q [B,H,D] against the first kv_len rows of caches [B,H,max_seq,D] -> [B, H*D]."""
    _need_cuda_f16(q, "decode_attention.q")
    B, H, D = q.shape
    max_seq = k_cache.shape[2]
    if not (k_cache.is_contiguous() and v_cache.is_contiguous() and q.is_contiguous()):
        raise RuntimeError("decode_attention: q and the caches must be contiguous")
    out = torch.empty((B, H * D), dtype=torch.float16, device=q.device)
    nbytes = int(load().seedb200_decode_attention_workspace_bytes(B, H, max_seq))
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=q.device)
    with on(q.device):
        check(load().seedb200_decode_attention(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr(),
                                               B, H, D, kv_len, max_seq, scale, ws.data_ptr(), stream_ptr(q.device)),
              "seedb200_decode_attention")
    return out


def decode_attention_lineage(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, slot: torch.Tensor,
                             kv_len: int, scale: float) -> torch.Tensor:
    """decode_attention where row b reads cached key / value p from cache row slot[b, p] (slot [B, max_seq] int32)."""
    _need_cuda_f16(q, "decode_attention_lineage.q")
    B, H, D = q.shape
    max_seq = k_cache.shape[2]
    if not (k_cache.is_contiguous() and v_cache.is_contiguous() and q.is_contiguous()):
        raise RuntimeError("decode_attention_lineage: q and the caches must be contiguous")
    if slot.dtype != torch.int32 or tuple(slot.shape) != (B, max_seq) or not slot.is_contiguous():
        raise RuntimeError("decode_attention_lineage: slot must be contiguous int32 [B, max_seq]")
    out = torch.empty((B, H * D), dtype=torch.float16, device=q.device)
    nbytes = int(load().seedb200_decode_attention_workspace_bytes(B, H, max_seq))
    ws = torch.empty((nbytes,), dtype=torch.uint8, device=q.device)
    with on(q.device):
        check(load().seedb200_decode_attention_lineage(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                                                       slot.data_ptr(), out.data_ptr(), B, H, D, kv_len, max_seq, scale,
                                                       ws.data_ptr(), stream_ptr(q.device)),
              "seedb200_decode_attention_lineage")
    return out


def decode_attention_rope_lineage(qkv: torch.Tensor, slot: torch.Tensor, H: int, past_len: int, k_cache: torch.Tensor,
                                  v_cache: torch.Tensor, scale: float) -> torch.Tensor:
    """decode_attention_rope where row b reads cached position p < past_len from cache row slot[b, p]"""
    _need_cuda_f16(qkv, "decode_attention_rope_lineage.qkv")
    B = qkv.shape[0]
    D = qkv.shape[1] // (3 * H)
    max_seq = k_cache.shape[2]
    if not (k_cache.is_contiguous() and v_cache.is_contiguous() and qkv.is_contiguous()):
        raise RuntimeError("decode_attention_rope_lineage: qkv and the caches must be contiguous")
    if slot.dtype != torch.int32 or tuple(slot.shape) != (B, max_seq) or not slot.is_contiguous():
        raise RuntimeError("decode_attention_rope_lineage: slot must be contiguous int32 [B, max_seq]")
    out = torch.empty((B, H * D), dtype=torch.float16, device=qkv.device)
    lib = load()
    lib.seedb200_decode_attention_rope_lineage.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                           C.c_float, C.c_void_p]
    with on(qkv.device):
        check(lib.seedb200_decode_attention_rope_lineage(qkv.data_ptr(), None, slot.data_ptr(), B, H, D, past_len,
                                                         max_seq, k_cache.data_ptr(), v_cache.data_ptr(),
                                                         out.data_ptr(), scale, stream_ptr(qkv.device)),
              "seedb200_decode_attention_rope_lineage")
    return out


def beam_select(logits: torch.Tensor, beam_scores: torch.Tensor, B: int, num_beams: int, first_step: bool = False,
                step: int = 0, **params):
    """Beam-search candidates of B sequences: logits [B*k, V] fp16 rows (or [B, V] with first_step: every beam reads
    its sequence's row), beam_scores [B*k] fp32 -> (scores [B, 2k] fp32, flat indices [B, 2k] int64)."""
    _need_cuda_f16(logits, "beam_select.logits")
    if logits.dim() != 2 or logits.stride(1) != 1:
        raise RuntimeError("beam_select: logits must be 2-D with contiguous rows")
    V = logits.shape[1]
    k = int(num_beams)
    if logits.shape[0] != (B if first_step else B * k):
        raise RuntimeError(f"beam_select: logits have {logits.shape[0]} rows")
    if beam_scores.dtype != torch.float32 or beam_scores.numel() != B * k or not beam_scores.is_contiguous():
        raise RuntimeError("beam_select: beam_scores must be contiguous fp32 [B*k]")
    ld = logits.stride(0)
    seq_ld, beam_ld = (ld, 0) if first_step else (k * ld, ld)
    bp = beam_params(k, **params)
    sc = torch.empty((B, 2 * k), dtype=torch.float32, device=logits.device)
    ix = torch.empty((B, 2 * k), dtype=torch.int32, device=logits.device)
    with on(logits.device):
        check(load().seedb200_beam_select(logits.data_ptr(), seq_ld, beam_ld, B, V, beam_scores.data_ptr(), C.byref(bp),
                                          int(step), sc.data_ptr(), ix.data_ptr(), stream_ptr(logits.device)),
              "seedb200_beam_select")
    return sc, ix.long()


def decode_attention_rope(qkv: torch.Tensor, positions: Optional[torch.Tensor], H: int, past_len: int,
                          k_cache: torch.Tensor, v_cache: torch.Tensor, scale: float) -> torch.Tensor:
    """RoPE + KV append + attention of one new token per sequence: qkv [B, 3*H*D] -> [B, H*D] (caches updated)."""
    _need_cuda_f16(qkv, "decode_attention_rope.qkv")
    B = qkv.shape[0]
    D = qkv.shape[1] // (3 * H)
    max_seq = k_cache.shape[2]
    if not (k_cache.is_contiguous() and v_cache.is_contiguous() and qkv.is_contiguous()):
        raise RuntimeError("decode_attention_rope: qkv and the caches must be contiguous")
    out = torch.empty((B, H * D), dtype=torch.float16, device=qkv.device)
    lib = load()
    lib.seedb200_decode_attention_rope.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]
    with on(qkv.device):
        check(lib.seedb200_decode_attention_rope(qkv.data_ptr(), _p(positions), B, H, D, past_len, max_seq,
                                                 k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr(), scale,
                                                 stream_ptr(qkv.device)), "seedb200_decode_attention_rope")
    return out


def sample(logits: torch.Tensor, do_sample: bool = False, temperature: float = 1.0, top_p: float = 1.0,
           seed: int = 0, offset: int = 0, step: int = 0, history: Optional[torch.Tensor] = None, top_k: int = 0,
           repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0, min_length: int = 0,
           min_new_tokens: int = 0, prompt_len: int = 0, eos_token_id: int = -1,
           scores_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """logits [B, V] fp16 (row stride free) -> next token per row, int64 [B].  The further controls are those of
    seedb200_logits_params; history [B, L] int64 (device) holds each row's input ids (prompt_len of them the prompt)
    and is needed by the penalty, n-gram and length controls.  `logits` is left unchanged.  scores_out (optional,
    fp16 [B, >= V] on the same device, rows 16-byte aligned and a multiple of 8 halves apart) receives each row's
    generation score, as seedb200_gen_outputs defines it (seedb200_sample_scores)."""
    _need_cuda_f16(logits, "sample.logits")
    if logits.dim() != 2 or logits.stride(1) != 1:
        raise RuntimeError("sample: logits must be [B, V] with contiguous rows")
    B, V = logits.shape
    out = torch.empty((B,), dtype=torch.int64, device=logits.device)
    sp = SampleParams(int(bool(do_sample)), float(temperature), float(top_p), int(seed), int(offset))
    lp = logits_params(top_k, repetition_penalty, no_repeat_ngram_size, min_length, min_new_tokens)
    if scores_out is not None:
        _need_cuda_f16(scores_out, "sample.scores_out")
        if scores_out.device != logits.device or scores_out.dim() != 2 or scores_out.shape[0] != B \
                or scores_out.shape[1] < V or scores_out.stride(1) != 1:
            raise RuntimeError(f"sample: scores_out must be [{B}, >= {V}] fp16 with contiguous rows on {logits.device}")
    if lp is None and scores_out is None:
        with on(logits.device):
            check(load().seedb200_sample(logits.data_ptr(), logits.stride(0), B, V, C.byref(sp), int(step),
                                         out.data_ptr(), stream_ptr(logits.device)), "seedb200_sample")
        return out
    hist, hist_len = None, 0
    if _history_active(lp, int(eos_token_id)):
        if history is None or history.dtype != torch.int64 or history.device != logits.device or history.dim() != 2 \
                or history.shape[0] != B:
            raise RuntimeError(f"sample: these controls need history [B, L] int64 on {logits.device}")
        hist = history if history.stride(1) == 1 else history.contiguous()
        hist_len = hist.shape[1]
        logits = logits.clone()                 # the processors rewrite the rows in place
    args = (logits.data_ptr(), logits.stride(0), B, V, C.byref(sp), int(step), out.data_ptr(),
            stream_ptr(logits.device), C.byref(lp) if lp is not None else None, _p(hist),
            hist.stride(0) if hist is not None else 0, hist_len, int(prompt_len), int(eos_token_id))
    with on(logits.device):
        if scores_out is None:
            check(load().seedb200_sample_processed(*args), "seedb200_sample_processed")
        else:
            check(load().seedb200_sample_scores(*args, scores_out.data_ptr(), scores_out.stride(0)),
                  "seedb200_sample_scores")
    return out


def contrastive_candidates(logits: torch.Tensor, top_k: int):
    """contrastive search's candidates of each row of logits [B, V] fp16 (row stride free): (ids [B, k] int64,
    probs [B, k] fp16), the k largest fp16 softmax probabilities, descending, ties to the lower id"""
    _need_cuda_f16(logits, "contrastive_candidates.logits")
    if logits.dim() != 2 or logits.stride(1) != 1:
        raise RuntimeError("contrastive_candidates: logits must be [B, V] with contiguous rows")
    B, V = logits.shape
    ids = torch.empty((B, int(top_k)), dtype=torch.int64, device=logits.device)
    probs = torch.empty((B, int(top_k)), dtype=torch.float16, device=logits.device)
    with on(logits.device):
        check(load().seedb200_contrastive_candidates(logits.data_ptr(), logits.stride(0), B, V, int(top_k),
                                                     ids.data_ptr(), probs.data_ptr(), stream_ptr(logits.device)),
              "seedb200_contrastive_candidates")
    return ids, probs


def contrastive_rank(context: torch.Tensor, p: int, cand_hidden: torch.Tensor, cand_probs: torch.Tensor,
                     penalty_alpha: float):
    """rank + select of B sequences: context [B, rows, H] fp16 (normalised, the first p rows valid; n(h_sel) is written
    at row p when p < rows), cand_hidden [B, k, H] fp16, cand_probs [B, k] fp16 -> (sel [B] int32, scores [B, k]
    fp32 holding the fp16 scores)"""
    for t, n in ((context, "context"), (cand_hidden, "cand_hidden"), (cand_probs, "cand_probs")):
        _need_cuda_f16(t, "contrastive_rank." + n)
        if not t.is_contiguous():
            raise RuntimeError(f"contrastive_rank: {n} must be contiguous")
    B, rows, H = context.shape
    k = cand_hidden.shape[1]
    if tuple(cand_hidden.shape) != (B, k, H) or tuple(cand_probs.shape) != (B, k):
        raise RuntimeError("contrastive_rank: cand_hidden must be [B, k, H] and cand_probs [B, k]")
    cp = ContrastiveParams(k, float(penalty_alpha))
    sel = torch.empty((B,), dtype=torch.int32, device=context.device)
    scores = torch.empty((B, k), dtype=torch.float32, device=context.device)
    with on(context.device):
        check(load().seedb200_contrastive_rank(context.data_ptr(), rows * H, rows, int(p), H, cand_hidden.data_ptr(),
                                               cand_probs.data_ptr(), B, C.byref(cp), sel.data_ptr(),
                                               scores.data_ptr(), stream_ptr(context.device)),
              "seedb200_contrastive_rank")
    return sel, scores


def contrastive_context_init(hidden_states: torch.Tensor, context: torch.Tensor) -> None:
    """hidden_states [B, S, H] fp16 -> rows [0, S) of context [B, rows, H], normalised"""
    _need_cuda_f16(hidden_states, "contrastive_context_init.hidden_states")
    _need_cuda_f16(context, "contrastive_context_init.context")
    if not (hidden_states.is_contiguous() and context.is_contiguous()):
        raise RuntimeError("contrastive_context_init: operands must be contiguous")
    B, S, H = hidden_states.shape
    with on(context.device):
        check(load().seedb200_contrastive_context_init(hidden_states.data_ptr(), B, S, H, context.data_ptr(),
                                                       context.shape[1] * H, stream_ptr(context.device)),
              "seedb200_contrastive_context_init")


def philox_uniform(seed: int, offset: int, row: int) -> float:
    return float(load().seedb200_philox_uniform(int(seed), int(offset), int(row)))


def image_ids_to_tokens(ids: torch.Tensor, image_id_shift: int, boi: int, eoi: int,
                        out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[n,32] int64 codebook ids (device) -> [n,34] LLaMA token ids; `out` may be a strided [n,>=34] view."""
    if not ids.is_cuda or ids.dtype != torch.int64:
        raise RuntimeError("image_ids_to_tokens: ids must be a CUDA int64 tensor")
    ids = ids.reshape(-1, 32).contiguous()
    n = ids.shape[0]
    if out is None:
        out = torch.empty((n, 34), dtype=torch.int64, device=ids.device)
    if out.dtype != torch.int64 or out.shape[0] != n or out.shape[1] < 34 or out.stride(1) != 1:
        raise RuntimeError("image_ids_to_tokens: out must be int64 [n, >=34] with contiguous rows")
    with on(ids.device):
        check(load().seedb200_image_ids_to_tokens(ids.data_ptr(), n, image_id_shift, boi, eoi, out.data_ptr(),
                                                  out.stride(0), stream_ptr(ids.device)), "seedb200_image_ids_to_tokens")
    return out


# --------------------------------------------------------------------------------------------------
# handles
# --------------------------------------------------------------------------------------------------
def _tensor_array(weights: Dict[str, torch.Tensor]):
    arr = (Tensor * len(weights))()
    keep = []
    dev = None
    for i, (name, t) in enumerate(weights.items()):
        if not t.is_cuda or t.dtype not in _DTYPE_CODE or not t.is_contiguous():
            raise RuntimeError(f"weight {name}: expected a contiguous CUDA float16, float32 or int8 tensor, got {t.dtype} "
                               f"on {t.device}")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise RuntimeError(f"weight {name} is on {t.device}, the others on {dev}: one handle, one device")
        b = name.encode()
        keep.append(b)
        arr[i].name = b
        arr[i].data = t.data_ptr()
        arr[i].dtype = _DTYPE_CODE[t.dtype]
        arr[i].ndim = min(t.dim(), 4)
        shp = list(t.shape)
        if len(shp) > 4:   # fold leading dims (conv weight [1408,3,14,14] has exactly 4)
            lead = 1
            for s in shp[:-3]:
                lead *= s
            shp = [lead] + shp[-3:]
        for j in range(4):
            arr[i].shape[j] = shp[j] if j < len(shp) else 1
    return arr, keep


class Encoder:
    """Owns a seedb200_encoder handle.  `weights` maps reference state-dict names to CUDA fp16 tensors."""

    def __init__(self, weights: Dict[str, torch.Tensor], vit_depth: int = 39, qformer_layers: int = 12,
                 detok_depth: int = 4, n_codes: int = 8192, max_batch: int = 256, vq_mode: int = VQ_FP16,
                 gemm_ctas: int = 0):
        lib = load()
        self._weights = dict(weights)   # keep the borrowed tensors alive
        arr, keep = _tensor_array(self._weights)
        self.device = next(iter(self._weights.values())).device
        cfg = EncoderConfig(vit_depth, qformer_layers, detok_depth, n_codes, max_batch, vq_mode, gemm_ctas)
        h = C.c_void_p()
        with on(self.device):   # the handle's workspace is allocated on the device that is current here
            check(lib.seedb200_encoder_create(C.byref(cfg), arr, len(self._weights), C.byref(h)),
                  "seedb200_encoder_create")
        self._h = h
        self.max_batch = max_batch

    def close(self) -> None:
        if getattr(self, "_h", None):
            load().seedb200_encoder_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check_dev(self, t: torch.Tensor, what: str) -> None:
        if t.device != self.device:
            raise RuntimeError(f"{what} is on {t.device}, the encoder handle on {self.device}")

    def encode(self, images: torch.Tensor, return_z: bool = False, return_query_up: bool = False):
        _need_cuda_f16(images, "encode.images")
        self._check_dev(images, "encode.images")
        images = images.contiguous()
        B = images.shape[0]
        ids = torch.empty((B, 32), dtype=torch.int64, device=images.device)
        z = torch.empty((B * 32, 32), dtype=torch.float16, device=images.device) if return_z else None
        qup = torch.empty((B, 32, 768), dtype=torch.float16, device=images.device) if return_query_up else None
        with on(self.device):
            check(load().seedb200_encoder_encode(self._h, images.data_ptr(), B, ids.data_ptr(), _p(z), _p(qup),
                                                 stream_ptr(self.device)), "seedb200_encoder_encode")
        return ids, z, qup

    def encode_tokens(self, images: torch.Tensor, image_id_shift: int, boi: int, eoi: int,
                      out: Optional[torch.Tensor] = None, return_ids: bool = False):
        """images -> [B,34] LLaMA token ids (`<img>` 32 shifted ids `</img>`) without leaving the device."""
        _need_cuda_f16(images, "encode_tokens.images")
        self._check_dev(images, "encode_tokens.images")
        images = images.contiguous()
        B = images.shape[0]
        if out is None:
            out = torch.empty((B, 34), dtype=torch.int64, device=images.device)
        if out.dtype != torch.int64 or out.shape[0] != B or out.shape[1] < 34 or out.stride(1) != 1:
            raise RuntimeError("encode_tokens: out must be int64 [B, >=34] with contiguous rows")
        ids = torch.empty((B, 32), dtype=torch.int64, device=images.device) if return_ids else None
        with on(self.device):
            check(load().seedb200_encoder_encode_tokens(self._h, images.data_ptr(), B, image_id_shift, boi, eoi,
                                                        out.data_ptr(), out.stride(0), _p(ids), stream_ptr(self.device)),
                  "seedb200_encoder_encode_tokens")
        return (out, ids) if return_ids else out

    def encode_host(self, images_pinned: torch.Tensor, ids_pinned: torch.Tensor) -> None:
        """Host (pinned) fp16 images -> host int64 ids; copies are enqueued on the current stream."""
        if images_pinned.is_cuda or ids_pinned.is_cuda:
            raise RuntimeError("encode_host takes host tensors")
        with on(self.device):
            check(load().seedb200_encoder_encode_host(self._h, images_pinned.data_ptr(), images_pinned.shape[0],
                                                      ids_pinned.data_ptr(), stream_ptr(self.device)),
                  "seedb200_encoder_encode_host")

    def detokenize(self, ids: torch.Tensor) -> torch.Tensor:
        if not ids.is_cuda or ids.dtype != torch.int64:
            raise RuntimeError("detokenize: ids must be a CUDA int64 tensor")
        self._check_dev(ids, "detokenize.ids")
        ids = ids.reshape(-1, 32).contiguous()
        B = ids.shape[0]
        out = torch.empty((B, 1024), dtype=torch.float16, device=ids.device)
        with on(self.device):
            check(load().seedb200_encoder_detokenize(self._h, ids.data_ptr(), B, out.data_ptr(), stream_ptr(self.device)),
                  "seedb200_encoder_detokenize")
        return out

    def tap(self, what: int, B: int) -> torch.Tensor:
        shape = {0: (B * 257, 1408), 1: (B * 32, 768), 2: (B * 257, 1408)}[what]
        out = torch.empty(shape, dtype=torch.float16, device=self.device)
        with on(self.device):
            n = load().seedb200_encoder_tap(self._h, what, out.data_ptr(), out.numel(), stream_ptr(self.device))
        if n != out.numel():
            raise RuntimeError(f"seedb200_encoder_tap({what}) returned {n}, expected {out.numel()}")
        return out


class Llama:
    """Owns a seedb200_llama handle.  `weights` uses the HF LLaMA state-dict names."""

    def __init__(self, weights: Dict[str, torch.Tensor], hidden: int, layers: int, heads: int, ffn: int, vocab: int,
                 max_batch: int = 1, max_seq: int = 4096, rms_eps: float = 1e-6, rope_base: float = 10000.0,
                 gemm_ctas: int = 0, int8_threshold: Optional[float] = None, quant4=None):
        """int8_threshold: None = fp16 weights (seedb200_llama_create); a float = LLM.int8() decoder linears given as
        int8 "<name>.weight" + fp32 "<name>.SCB" (seedb200_llama_create_int8), which the handle copies: only the
        fp16 tensors stay referenced after construction.  quant4 ("fp4" / "nf4"): bitsandbytes 4-bit decoder
        linears (seedb200_llama_create_4bit); `weights` then holds no decoder linear, and each is given to
        load_4bit_weight() before the model runs."""
        if int8_threshold is not None and quant4 is not None:
            raise ValueError("int8_threshold and quant4 are exclusive")
        lib = load()
        self._weights = dict(weights)
        arr, keep = _tensor_array(self._weights)
        self.device = next(iter(self._weights.values())).device
        cfg = LlamaConfig(hidden, layers, heads, hidden // heads, ffn, vocab, max_batch, max_seq, rms_eps,
                          rope_base, gemm_ctas)
        h = C.c_void_p()
        with on(self.device):
            if quant4 is not None:
                check(lib.seedb200_llama_create_4bit(C.byref(cfg), arr, len(self._weights), quant4_type(quant4),
                                                     C.byref(h)), "seedb200_llama_create_4bit")
            elif int8_threshold is None:
                check(lib.seedb200_llama_create(C.byref(cfg), arr, len(self._weights), C.byref(h)),
                      "seedb200_llama_create")
            else:
                check(lib.seedb200_llama_create_int8(C.byref(cfg), arr, len(self._weights), float(int8_threshold),
                                                     C.byref(h)), "seedb200_llama_create_int8")
        if int8_threshold is not None:
            self._weights = {k: v for k, v in self._weights.items() if v.dtype == torch.float16}
        self._h = h
        self.hidden, self.layers, self.heads, self.head_dim = hidden, layers, heads, hidden // heads
        self.ffn, self.vocab, self.max_batch, self.max_seq = ffn, vocab, max_batch, max_seq
        self.vpad = (vocab + 7) // 8 * 8      # logits row stride: 16-byte rows for the lm_head epilogue

    def close(self) -> None:
        if getattr(self, "_h", None):
            load().seedb200_llama_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, input_ids: Optional[torch.Tensor] = None, inputs_embeds: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.Tensor] = None, past_len: int = 0, last_only: bool = False,
                want_logits: bool = True) -> Optional[torch.Tensor]:
        if input_ids is not None:
            B, S = input_ids.shape
            input_ids = input_ids.contiguous()
        else:
            B, S = inputs_embeds.shape[:2]
            inputs_embeds = inputs_embeds.contiguous()
        if position_ids is not None:
            position_ids = position_ids.reshape(-1, S).expand(B, S).contiguous().long()
            # the reference indexes cos[position_ids] and fails on an out-of-range position (llama_xformer.py:157-158);
            # the kernel would clamp silently, so refuse here
            lo, hi = int(position_ids.min()), int(position_ids.max())
            if lo < 0 or hi >= max(self.max_seq, 4096):
                raise IndexError(f"position_ids outside the rotary table: [{lo}, {hi}]")
        logits = None
        if want_logits:
            # rows padded to a multiple of 8 halves (V = 40194 -> 40200); callers see the [..., :V] view
            full = torch.empty((B, 1 if last_only else S, self.vpad), dtype=torch.float16, device=self.device)
            logits = full[..., :self.vocab]
        with on(self.device):
            check(load().seedb200_llama_forward_ld(self._h, _p(input_ids), _p(inputs_embeds), _p(position_ids), B, S,
                                                   past_len, 1 if last_only else 0, _p(logits), self.vpad,
                                                   stream_ptr(self.device)), "seedb200_llama_forward_ld")
        return logits

    def generate(self, prompt_ids: torch.Tensor, max_new_tokens: int, do_sample: bool = False,
                 temperature: float = 1.0, top_p: float = 1.0, seed: int = 0, offset: int = 0,
                 eos_token_id: int = -1, pad_token_id: int = 0, use_graph: bool = True,
                 num_return_sequences: int = 1, scores: Optional[torch.Tensor] = None, **controls) -> torch.Tensor:
        """prompt [B,S] int64 (device) -> generated tokens [B * num_return_sequences, n] (n <= max_new_tokens; shorter
        only when every row hit eos), row b * num_return_sequences + j being sample j of prompt b.  Prefill + sampler
        + cached decode steps, all on the device; see seedb200_llama_generate_n.  Needs B * num_return_sequences <=
        max_batch (reserve_rows).  `controls`: the keywords of logits_params (top_k, repetition_penalty, ...).
        scores (optional): a scores_buffer(max_new_tokens, B * num_return_sequences, ...) that receives each step's
        generation scores (seedb200_llama_generate_ex); steps [0, n) are valid."""
        if not prompt_ids.is_cuda or prompt_ids.dtype != torch.int64 or prompt_ids.device != self.device:
            raise RuntimeError(f"generate: prompt_ids must be int64 on {self.device}")
        prompt_ids = prompt_ids.contiguous()
        B, S = prompt_ids.shape
        rs = int(num_return_sequences)
        out = torch.empty((B * max(rs, 1), max_new_tokens), dtype=torch.int64, device=self.device)
        sp = SampleParams(int(bool(do_sample)), float(temperature), float(top_p), int(seed), int(offset))
        lp = logits_params(**controls)
        n = C.c_int(0)
        args = (self._h, prompt_ids.data_ptr(), B, S, max_new_tokens, rs, C.byref(sp), int(eos_token_id),
                int(pad_token_id), int(bool(use_graph)), out.data_ptr(), C.byref(n), stream_ptr(self.device))
        with on(self.device):
            if scores is not None:
                o = self._outputs(scores, max_new_tokens, B * rs, "generate")
                check(load().seedb200_llama_generate_ex(*args, C.byref(lp) if lp is not None else None, C.byref(o)),
                      "seedb200_llama_generate_ex")
            elif lp is None:
                check(load().seedb200_llama_generate_n(*args), "seedb200_llama_generate_n")
            else:
                check(load().seedb200_llama_generate_n_processed(*args, C.byref(lp)),
                      "seedb200_llama_generate_n_processed")
        return out[:, :n.value]

    def beam_generate(self, prompt_ids: torch.Tensor, max_new_tokens: int, num_beams: int, do_sample: bool = False,
                      temperature: float = 1.0, top_p: float = 1.0, length_penalty: float = 1.0, early_stopping=False,
                      seed: int = 0, offset: int = 0, eos_token_id: int = -1, pad_token_id: int = 0,
                      use_graph: bool = True, num_return_sequences: int = 1, scores: Optional[torch.Tensor] = None,
                      beam_indices: Optional[torch.Tensor] = None, **controls):
        """prompt [B,S] int64 (device) -> (generated tokens [G, n] of the best hypothesis per search, fp32 scores [G]),
        G = B * num_return_sequences independent searches, prompt-major (beam sampling only when
        num_return_sequences > 1); see seedb200_llama_beam_generate_n.  Needs G * num_beams <= max_batch
        (reserve_rows).  `controls`: the keywords of logits_params.
        scores (optional): a scores_buffer(max_new_tokens, G * num_beams, ...) that receives each step's beam scores,
        with beam_indices (optional) an int64 [G, S + max_new_tokens] tensor (seedb200_llama_beam_generate_ex); the
        call then returns (tokens, scores [G], number of valid scores steps)."""
        if not prompt_ids.is_cuda or prompt_ids.dtype != torch.int64 or prompt_ids.device != self.device:
            raise RuntimeError(f"beam_generate: prompt_ids must be int64 on {self.device}")
        prompt_ids = prompt_ids.contiguous()
        B, S = prompt_ids.shape
        rs = int(num_return_sequences)
        G = B * max(rs, 1)
        out = torch.empty((G, max_new_tokens), dtype=torch.int64, device=self.device)
        scores_out, scores = scores, torch.empty((G,), dtype=torch.float32, device=self.device)
        bp = beam_params(num_beams, do_sample, temperature, top_p, length_penalty, early_stopping, seed, offset)
        lp = logits_params(**controls)
        n = C.c_int(0)
        args = (self._h, prompt_ids.data_ptr(), B, S, max_new_tokens, rs, C.byref(bp), int(eos_token_id),
                int(pad_token_id), int(bool(use_graph)), out.data_ptr(), C.byref(n), scores.data_ptr(),
                stream_ptr(self.device))
        with on(self.device):
            if scores_out is not None:
                o = self._outputs(scores_out, max_new_tokens, G * int(num_beams), "beam_generate")
                if beam_indices is not None:
                    if beam_indices.dtype != torch.int64 or beam_indices.device != self.device \
                            or tuple(beam_indices.shape) != (G, S + max_new_tokens) or not beam_indices.is_contiguous():
                        raise RuntimeError(f"beam_generate: beam_indices must be a contiguous int64 "
                                           f"[{G}, {S + max_new_tokens}] tensor on {self.device}")
                    o.beam_indices = beam_indices.data_ptr()
                check(load().seedb200_llama_beam_generate_ex(*args, C.byref(lp) if lp is not None else None,
                                                             C.byref(o)), "seedb200_llama_beam_generate_ex")
                return out[:, :n.value], scores, o.n_steps_out
            if lp is None:
                check(load().seedb200_llama_beam_generate_n(*args), "seedb200_llama_beam_generate_n")
            else:
                check(load().seedb200_llama_beam_generate_n_processed(*args, C.byref(lp)),
                      "seedb200_llama_beam_generate_n_processed")
        return out[:, :n.value], scores

    def contrastive_generate(self, prompt_ids: torch.Tensor, max_new_tokens: int, top_k: int, penalty_alpha: float,
                             eos_token_id: int = -1, pad_token_id: int = 0, use_graph: bool = True,
                             scores: Optional[torch.Tensor] = None, **controls) -> torch.Tensor:
        """prompt [B,S] int64 (device) -> generated tokens [B, n] of contrastive search (n < max_new_tokens only when
        every sequence hit eos); see seedb200_llama_contrastive_generate.  Needs B * top_k <= max_batch
        (reserve_rows).  `controls`: the processor keywords of logits_params (their top_k is not used).
        scores (optional): a scores_buffer(max_new_tokens, B, ...) that receives each step's processed logits
        (seedb200_llama_contrastive_generate_ex); steps [0, n) are valid."""
        if not prompt_ids.is_cuda or prompt_ids.dtype != torch.int64 or prompt_ids.device != self.device:
            raise RuntimeError(f"contrastive_generate: prompt_ids must be int64 on {self.device}")
        prompt_ids = prompt_ids.contiguous()
        B, S = prompt_ids.shape
        out = torch.empty((B, max_new_tokens), dtype=torch.int64, device=self.device)
        cp = ContrastiveParams(int(top_k), float(penalty_alpha))
        lp = logits_params(**dict(controls, top_k=0))
        n = C.c_int(0)
        args = (self._h, prompt_ids.data_ptr(), B, S, max_new_tokens, C.byref(cp), int(eos_token_id),
                int(pad_token_id), int(bool(use_graph)), out.data_ptr(), C.byref(n), stream_ptr(self.device),
                C.byref(lp) if lp is not None else None)
        with on(self.device):
            if scores is None:
                check(load().seedb200_llama_contrastive_generate(*args), "seedb200_llama_contrastive_generate")
            else:
                o = self._outputs(scores, max_new_tokens, B, "contrastive_generate")
                check(load().seedb200_llama_contrastive_generate_ex(*args, C.byref(o)),
                      "seedb200_llama_contrastive_generate_ex")
        return out[:, :n.value]

    def _outputs(self, scores: torch.Tensor, steps: int, rows: int, who: str) -> GenOutputs:
        """seedb200_gen_outputs over a scores_buffer(steps, rows, ...)"""
        if scores.dtype != torch.float16 or scores.device != self.device or scores.dim() != 3 \
                or tuple(scores.shape[:2]) != (steps, rows) or not scores.is_contiguous():
            raise RuntimeError(f"{who}: scores must be a contiguous fp16 [{steps}, {rows}, pitch] tensor on "
                               f"{self.device}")
        return GenOutputs(scores.data_ptr(), scores.stride(1), None, 0)

    def reserve_rows(self, rows: int) -> None:
        """grow every max_batch-sized buffer to `rows` rows (drops the cache contents and the captured graphs)"""
        with on(self.device):
            check(load().seedb200_llama_reserve_rows(self._h, int(rows)), "seedb200_llama_reserve_rows")
        self.max_batch = max(self.max_batch, int(rows))

    def int8_load_weight(self, name: str, w: torch.Tensor) -> None:
        """quantise the fp16 decoder linear `name` straight into the int8 handle's fused layout"""
        self._load_quantised("seedb200_llama_int8_load_weight", name, w)

    def load_4bit_weight(self, name: str, w: torch.Tensor) -> None:
        """quantise the fp16 decoder linear `name` straight into the 4-bit handle's fused layout"""
        self._load_quantised("seedb200_llama_4bit_load_weight", name, w)

    def _load_quantised(self, fn: str, name: str, w: torch.Tensor) -> None:
        # the C side reads the [N, K] rows its slot expects from the pointer it is given: the shape is checked here.
        # A name that is not a decoder linear passes through and is refused by the C side.
        _need_cuda_f16(w, name)
        if w.stride(1) != 1 or w.device != self.device:
            raise RuntimeError(f"{name}: expected rows with contiguous columns on {self.device}")
        lin = name.split(".")[-2] if name.count(".") >= 2 else ""
        N, K = {"q_proj": (self.hidden, self.hidden), "k_proj": (self.hidden, self.hidden),
                "v_proj": (self.hidden, self.hidden), "o_proj": (self.hidden, self.hidden),
                "gate_proj": (self.ffn, self.hidden), "up_proj": (self.ffn, self.hidden),
                "down_proj": (self.hidden, self.ffn)}.get(lin, tuple(w.shape))
        if tuple(w.shape) != (N, K):
            raise RuntimeError(f"{name}: expected shape [{N}, {K}], got {list(w.shape)}")
        with on(self.device):
            check(getattr(load(), fn)(self._h, name.encode(), w.data_ptr(), w.stride(0), stream_ptr(self.device)), fn)

    def lora_load(self, tensors: Dict[str, torch.Tensor], r: int, alpha: float) -> None:
        """copy a LoRA adapter ("model.layers.N.<...>.lora_A.weight" / ".lora_B.weight", fp16 on this device) into the
        handle; replaces an earlier one.  The tensors may be dropped afterwards."""
        arr, keep = _tensor_array(tensors)
        with on(self.device):
            check(load().seedb200_llama_lora_load(self._h, arr, len(tensors), int(r), float(alpha)),
                  "seedb200_llama_lora_load")

    def lora_merge(self) -> None:
        """add the loaded adapter into the weights (o_proj / down_proj are borrowed: changed in place) and drop it"""
        with on(self.device):
            check(load().seedb200_llama_lora_merge(self._h), "seedb200_llama_lora_merge")

    def replace_weights(self, tensors: Dict[str, torch.Tensor]) -> None:
        """re-point embed_tokens / lm_head (together when the vocabulary changes) and the norms; the handle borrows
        them, so they are kept referenced here"""
        arr, keep = _tensor_array(tensors)
        with on(self.device):
            check(load().seedb200_llama_replace_weights(self._h, arr, len(tensors)), "seedb200_llama_replace_weights")
        self._weights.update(tensors)
        if "model.embed_tokens.weight" in tensors:
            self.vocab = int(tensors["model.embed_tokens.weight"].shape[0])
            self.vpad = (self.vocab + 7) // 8 * 8

    @property
    def used_graph(self) -> int:
        return int(load().seedb200_llama_generate_used_graph(self._h))

    def kv_views(self, layer: int):
        k, v = C.c_void_p(), C.c_void_p()
        check(load().seedb200_llama_kv_ptrs(self._h, layer, C.byref(k), C.byref(v)), "seedb200_llama_kv_ptrs")
        return k.value, v.value

    def kv_load(self, layer: int, k: torch.Tensor, v: torch.Tensor) -> None:
        B, H, P, D = k.shape
        kc, vc = k.contiguous(), v.contiguous()   # keep BOTH alive across the call: two unnamed temporaries would
        # be freed immediately and the caching allocator hands the second one the first one's block
        with on(self.device):
            check(load().seedb200_llama_kv_load(self._h, layer, kc.data_ptr(), vc.data_ptr(), B, P,
                                                stream_ptr(self.device)), "seedb200_llama_kv_load")

    def tap_hidden(self, T: int) -> torch.Tensor:
        out = torch.empty((T, self.hidden), dtype=torch.float16, device=self.device)
        with on(self.device):
            n = load().seedb200_llama_tap(self._h, 0, out.data_ptr(), out.numel(), stream_ptr(self.device))
        if n != out.numel():
            raise RuntimeError(f"seedb200_llama_tap returned {n}, expected {out.numel()}")
        return out
