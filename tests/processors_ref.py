"""TEST INFRASTRUCTURE ONLY -- restatement of the generation controls of seedb200_logits_params (include/seedb200.h):
transformers 4.30.2's RepetitionPenalty, NoRepeatNGram, MinLength and MinNewTokensLength processors and TopK warper as
the reference runs them on CUDA with fp16 logits, and the greedy / sample / beam search / beam sample loops that apply
them.  tests/beam_ref.py supplies Philox, TopP and the beam hypotheses.

fp16 rounding: torch computes an fp16 tensor op with a Python scalar in fp32 and rounds once; its CUDA division by a
scalar multiplies by the fp32 reciprocal (tests/test_logits_processors_gpu.py pins that).
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch

import beam_ref as BR
from oracle import sampler_oracle as SO

NEUTRAL = {"top_k": 0, "repetition_penalty": 1.0, "no_repeat_ngram_size": 0, "min_length": 0, "min_new_tokens": 0}


def f32(x: float) -> torch.Tensor:
    return torch.tensor(x, dtype=torch.float32)


def scalar_div(v: torch.Tensor, d: float) -> torch.Tensor:
    """fp16 tensor / Python float on CUDA: fp16(float(v) * fp32(1 / fp32(d))) (fp32 rows: the same without rounding)"""
    return (v.float() * (f32(1.0) / f32(d))).to(v.dtype)


def process(scores: torch.Tensor, hist: List[int], S: int, eos: int, ctl: dict) -> torch.Tensor:
    """the four processors on one row (fp16 [V]) whose input ids are `hist` (prompt of S ids, then generated)"""
    x = scores.clone()
    V, L = x.shape[0], len(hist)
    p = float(ctl.get("repetition_penalty", 1.0))
    if p != 1.0:
        t = torch.tensor(sorted(set(hist)), dtype=torch.int64)
        v = x[t]
        x[t] = torch.where(v < 0, (v.float() * f32(p)).to(v.dtype), scalar_div(v, p))
    n = int(ctl.get("no_repeat_ngram_size", 0))
    if n > 0 and L + 1 >= n:
        tail = hist[L - n + 1:]
        for i in range(L - n + 1):
            if hist[i:i + n - 1] == tail and 0 <= hist[i + n - 1] < V:
                x[hist[i + n - 1]] = float("-inf")
    if eos is not None and eos >= 0:
        if L < int(ctl.get("min_length", 0)) or L - S < int(ctl.get("min_new_tokens", 0)):
            x[eos] = float("-inf")
    return x


def top_k_keep(values: torch.Tensor, k: int, min_keep: int) -> torch.Tensor:
    """TopKLogitsWarper in threshold form: every value >= the k'-th largest, k' = min(max(k, min_keep), V)"""
    if k <= 0:
        return torch.ones_like(values, dtype=torch.bool)
    kk = min(max(k, min_keep), values.shape[-1])
    thr = torch.sort(values.float(), descending=True).values[kk - 1]
    return values.float() >= thr


def sample_row(logits: torch.Tensor, hist: List[int], S: int, eos: int, ctl: dict, do_sample: bool,
               temperature: float = 1.0, top_p: float = 1.0, seed: int = 0, offset: int = 0, step: int = 0,
               row: int = 0):
    """one row of the sample / greedy path -> (token, draw margin, nucleus margin)"""
    x = process(logits, hist, S, eos, ctl)
    if not do_sample:
        return int(torch.argmax(x.float())), 1.0, 1.0
    key = x if temperature == 1.0 else scalar_div(x, temperature)
    keep = top_k_keep(key, int(ctl.get("top_k", 0)), 1).numpy()
    xs = x.float().numpy().astype(np.float64) / float(np.float32(temperature))
    xs = np.where(keep, xs, -np.inf)
    p = np.exp(xs - xs.max())
    p /= p.sum()
    nmargin = 1.0
    if top_p < 1.0:
        order = np.argsort(xs, kind="stable")
        cs = np.cumsum(p[order])
        rem = cs <= (1.0 - top_p)
        rem[-1:] = False
        kept = np.ones_like(rem)
        kept[order] = ~rem
        keep = keep & (xs >= xs[kept].min())
        nmargin = float(np.min(np.abs(cs[cs > 0] - (1.0 - top_p)))) if (cs > 0).any() else 1.0
    q = np.where(keep, p, 0.0)
    q /= q.sum()
    cdf = np.cumsum(q)
    u = float(SO.philox_uniform(seed, offset + step, row))
    tok = min(int(np.searchsorted(cdf, u, side="left")), len(q) - 1)
    while not keep[tok]:
        tok += 1
    dmargin = float(np.min(np.abs(np.concatenate([[0.0], cdf]) - u)))
    return tok, dmargin, nmargin


def generate(step_logits: Callable, prompt: torch.Tensor, max_new_tokens: int, ctl: dict, do_sample: bool = False,
             temperature: float = 1.0, top_p: float = 1.0, eos: Optional[int] = None, pad: int = 0, seed: int = 0,
             offset: int = 0):
    """greedy / sample loop: step_logits(ids [B, cur]) -> last-position logits [B, V].  Returns (sequences,
    smallest draw margin, smallest nucleus margin)."""
    ids = prompt.cpu().clone()
    B, S = ids.shape
    unfinished = torch.ones(B, dtype=torch.bool)
    dmin, nmin = 1.0, 1.0
    e = -1 if eos is None else eos
    for step in range(max_new_tokens):
        logits = step_logits(ids).cpu()
        nxt = torch.zeros(B, dtype=torch.int64)
        for b in range(B):
            t, dm, nm = sample_row(logits[b], ids[b].tolist(), S, e, ctl, do_sample, temperature, top_p, seed,
                                   offset, step, b)
            nxt[b], dmin, nmin = t, min(dmin, dm), min(nmin, nm)
        nxt = torch.where(unfinished, nxt, torch.full_like(nxt, pad))
        ids = torch.cat([ids, nxt[:, None]], dim=1)
        if eos is not None:
            unfinished &= nxt != eos
            if not bool(unfinished.any()):
                break
    return ids, dmin, nmin


def beam_select(s: torch.Tensor, k: int, top_k: int, do_sample: bool, temperature: float, top_p: float, seed: int,
                offset: int, step: int):
    """BR.select with top_k (min_tokens_to_keep 2) on w = s / T before TopP"""
    if not do_sample or top_k <= 0:
        return BR.select(s, k, do_sample, temperature, top_p, seed, offset, step)
    B, KV = s.shape
    V = KV // k
    scores, idx, kmargin, nmargin = [], [], [], 1.0
    for i in range(B):
        w = s[i] / temperature
        wr = w.view(k, V)
        keep_k = torch.stack([top_k_keep(wr[j], top_k, 2) for j in range(k)])
        wf = torch.where(keep_k, wr, torch.tensor(float("-inf")))
        keep, nm = BR.top_p_keep(wf, top_p)
        keep = keep & keep_k
        nmargin = min(nmargin, nm)
        u = BR.open_uniform(seed, offset + step, i, KV)
        key = torch.where(keep.reshape(-1), w + (-torch.log(-torch.log(u))), torch.tensor(-float("inf")))
        kn = key.numpy()
        order = BR._desc(kn)
        kmargin.append(float(kn[order[2 * k - 1]] - kn[order[2 * k]]) if KV > 2 * k else float("inf"))
        draws = order[:2 * k]
        o2 = np.lexsort((draws, -w.numpy()[draws]))
        draws = draws[o2]
        scores.append(w[draws])
        idx.append(torch.from_numpy(draws.copy()))
    return torch.stack(scores), torch.stack(idx), kmargin, nmargin


def beam_generate(step_logits: Callable, prompt: torch.Tensor, max_new_tokens: int, num_beams: int, ctl: dict,
                  do_sample: bool = False, temperature: float = 1.0, top_p: float = 1.0, length_penalty: float = 1.0,
                  early_stopping=False, eos: Optional[int] = None, pad: int = 0, seed: int = 0, offset: int = 0,
                  shared_history: bool = False):
    """BR.beam_generate with the processors on each beam row's fp16 log_softmax (its own sequence as history) and
    top_k in beam sampling.  Returns (sequences [B, width], smallest key margin, nucleus margin).  shared_history
    gives every beam row the history of its sequence's first beam instead (a wrong variant, for tests to contrast)."""
    k = num_beams
    B, S = prompt.shape
    max_length = S + max_new_tokens
    ids = prompt.cpu().repeat_interleave(k, dim=0)
    beam_scores = torch.zeros((B, k), dtype=torch.float32)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view(-1)
    hyps = [BR.Hyps(k, length_penalty, early_stopping, max_length) for _ in range(B)]
    done = [False] * B
    beam_idx, step, kmin, nmin = None, 0, float("inf"), 1.0
    e = -1 if eos is None else eos
    while True:
        cur_len = ids.shape[1]
        logits = step_logits(ids, beam_idx).cpu()
        V = logits.shape[-1]
        lp = BR.log_probs(logits).to(logits.dtype)
        hrow = [(r // k) * k if shared_history else r for r in range(B * k)]
        lp = torch.stack([process(lp[r], ids[hrow[r]].tolist(), S, e, ctl) for r in range(B * k)]).float()
        s = (lp + beam_scores[:, None]).view(B, k * V)
        sc, ix, km, nm = beam_select(s, k, int(ctl.get("top_k", 0)), do_sample, temperature, top_p, seed, offset,
                                     step)
        kmin, nmin = min([kmin] + km), min(nmin, nm)
        nb_s = torch.zeros((B, k), dtype=torch.float32)
        nb_t = torch.full((B, k), pad, dtype=torch.int64)
        nb_i = torch.zeros((B, k), dtype=torch.int64)
        for i in range(B):
            if done[i]:
                nb_i[i] = torch.arange(k) + i * k
                continue
            bi = 0
            for r in range(2 * k):
                f = int(ix[i, r])
                beam, tok = f // V, f % V
                if eos is not None and tok == eos:
                    if r >= k:
                        continue
                    hyps[i].add(ids[i * k + beam].tolist(), float(sc[i, r]))
                else:
                    nb_s[i, bi], nb_t[i, bi], nb_i[i, bi] = sc[i, r], tok, i * k + beam
                    bi += 1
                if bi == k:
                    break
            done[i] = done[i] or hyps[i].is_done(float(sc[i].max()), cur_len)
        beam_scores = nb_s.view(-1)
        beam_idx = nb_i.view(-1)
        ids = torch.cat([ids[beam_idx], nb_t.view(-1, 1)], dim=1)
        step += 1
        if all(done) or ids.shape[1] >= max_length:
            break
    for i in range(B):
        if not done[i]:
            for j in range(k):
                hyps[i].add(ids[i * k + j].tolist(), float(beam_scores[i * k + j]))
    best = [sorted(h.beams, key=lambda x: x[0])[-1][1] for h in hyps]
    width = min(max(len(h) for h in best) + 1, max_length)
    out = torch.full((B, width), pad, dtype=torch.int64)
    for i, h in enumerate(best):
        out[i, :len(h)] = torch.tensor(h)
        if len(h) < width and eos is not None:
            out[i, len(h)] = eos
    return out, kmin, nmin
