"""TEST INFRASTRUCTURE ONLY -- restatement of transformers 4.30.2 generate(num_return_sequences=n) for the two modes
that accept it on the device (include/seedb200.h, seedb200_llama_generate_n / seedb200_llama_beam_generate_n):

  sampling        _expand_inputs_for_generation(expand_size=n): row r = b * n + j is sample j of prompt b and draws
                  from Philox row r
  beam sampling   BeamSearchScorer(batch_size=B * n, num_beams=k) keeping one hypothesis, inputs expanded k * n
                  times: search g = b * n + j reads prompt b and draws from Philox sequence g; each search returns
                  its own best hypothesis (so n may exceed k)

Both are the n = 1 rule on prompt.repeat_interleave(n, 0), which is how they are stated here.
"""
from __future__ import annotations

from typing import Callable

import torch

import beam_ref as BR


def expand(prompt: torch.Tensor, n: int) -> torch.Tensor:
    """the prompt-major expansion of _expand_inputs_for_generation"""
    return prompt.repeat_interleave(n, dim=0)


def prompt_of(row: int, n: int) -> int:
    """the prompt a sampling row, or a beam-sample search, reads"""
    return row // n


def beam_sample_generate(step_logits: Callable, prompt: torch.Tensor, max_new_tokens: int, num_beams: int, n: int,
                         **kw):
    """beam_ref.beam_generate with do_sample=True over B * n searches; same return value, one row per search"""
    return BR.beam_generate(step_logits, expand(prompt, n), max_new_tokens, num_beams, do_sample=True, **kw)
