"""TEST INFRASTRUCTURE ONLY -- restatement of transformers 4.30.2 GenerationMixin.beam_search / beam_sample with
BeamSearchScorer(num_beam_hyps_to_keep=1) (requirements.txt:8), the arithmetic seedb200_llama_beam_generate follows.
include/seedb200.h (seedb200_beam_params) states the rules; tests/test_beam_cpu.py pins each one on a hand-worked case.

  init       beam_scores fp32: 0 for beam 0, -1e9 for beams 1..k-1
  step       lp = log_softmax(logits) in the logits' dtype (fp16: rounded); s = float(lp) + beam_score (fp32)
  greedy     top 2k of s over [k*V], descending, ties to the lowest flat index
  sampling   w = s / T; TopP per beam row (min_tokens_to_keep=2, every token tied with the least kept one stays);
             Gumbel-top-2k: key = w + (-log(-log u)) in fp32, u from Philox4x32-10 (seed; offset + step, sequence,
             1 + j), ((x >> 9) + 0.5) * 2^-23; draws sorted by w descending; the scorer receives w
  scorer     BeamSearchScorer.process / BeamHypotheses.add / is_done; finalize as 4.30.2
"""
from __future__ import annotations

from typing import Callable, List, Optional

import numpy as np
import torch

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = np.uint64(0xFFFFFFFF)


def philox_word(seed: int, offset: int, row: int, word3: np.ndarray) -> np.ndarray:
    """first output word of Philox4x32-10, counter (offset lo, offset hi, row, word3[...]), key = seed (vectorised)"""
    word3 = np.asarray(word3, dtype=np.uint64)
    c0 = np.full(word3.shape, offset & 0xFFFFFFFF, dtype=np.uint64)
    c1 = np.full(word3.shape, (offset >> 32) & 0xFFFFFFFF, dtype=np.uint64)
    c2 = np.full(word3.shape, row & 0xFFFFFFFF, dtype=np.uint64)
    c3 = word3 & MASK
    k0, k1 = seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & MASK, p1 >> np.uint64(32), p1 & MASK
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return c0


def open_uniform(seed: int, offset: int, row: int, n: int) -> torch.Tensor:
    """u_j, j < n: strictly inside (0, 1), exact in fp32"""
    x = philox_word(seed, offset, row, np.arange(n, dtype=np.uint64) + np.uint64(1))
    return torch.from_numpy(((x >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23).float()


def log_probs(logits: torch.Tensor) -> torch.Tensor:
    """log_softmax in the logits' dtype, returned as fp32"""
    if logits.dtype == torch.float16:
        return torch.log_softmax(logits.float(), dim=-1).half().float()
    return torch.log_softmax(logits.float(), dim=-1)


def top_p_keep(w: torch.Tensor, top_p: float, min_keep: int = 2):
    """TopPLogitsWarper on each row of w in threshold form (ties kept) -> (keep mask, boundary margin)"""
    keep = torch.ones_like(w, dtype=torch.bool)
    margin = 1.0
    if top_p >= 1.0:
        return keep, margin
    for r in range(w.shape[0]):
        x = w[r].double().numpy()
        p = np.exp(x - x.max())
        p /= p.sum()
        order = np.argsort(x, kind="stable")
        cs = np.cumsum(p[order])
        remove = cs <= (1.0 - top_p)
        remove[-min_keep:] = False
        kept = np.ones_like(remove)
        kept[order] = ~remove
        keep[r] = torch.from_numpy(x >= x[kept].min())
        margin = min(margin, float(np.min(np.abs(cs - (1.0 - top_p)))))
    return keep, margin


def _desc(v: np.ndarray) -> np.ndarray:
    """indices sorting v descending, ties to the lowest index"""
    return np.argsort(-v, kind="stable")


def select(s: torch.Tensor, k: int, do_sample: bool = False, temperature: float = 1.0, top_p: float = 1.0,
           seed: int = 0, offset: int = 0, step: int = 0):
    """s [B, k*V] fp32 -> (scores [B, 2k] fp32, flat indices [B, 2k], key margins [B], nucleus margin)"""
    B, KV = s.shape
    V = KV // k
    scores, idx, kmargin, nmargin = [], [], [], 1.0
    for i in range(B):
        if not do_sample:
            order = _desc(s[i].numpy())[:2 * k]
            scores.append(s[i][order]); idx.append(torch.from_numpy(order.copy())); kmargin.append(float("inf"))
            continue
        w = s[i] / temperature
        keep, nm = top_p_keep(w.view(k, V), top_p)
        nmargin = min(nmargin, nm)
        u = open_uniform(seed, offset + step, i, KV)
        key = torch.where(keep.reshape(-1), w + (-torch.log(-torch.log(u))), torch.tensor(-float("inf")))
        kn = key.numpy()
        order = _desc(kn)
        kmargin.append(float(kn[order[2 * k - 1]] - kn[order[2 * k]]) if KV > 2 * k else float("inf"))
        draws = order[:2 * k]
        ws = w.numpy()[draws]
        o2 = np.lexsort((draws, -ws))          # by w descending, ties to the lowest index
        draws = draws[o2]
        scores.append(w[draws]); idx.append(torch.from_numpy(draws.copy()))
    return torch.stack(scores), torch.stack(idx), kmargin, nmargin


class Hyps:
    """BeamHypotheses (4.30.2)"""

    def __init__(self, k: int, length_penalty: float, early_stopping, max_length: int):
        self.k, self.lp, self.es, self.max_length = k, length_penalty, early_stopping, max_length
        self.beams: List = []
        self.worst = 1e9

    def add(self, hyp: List[int], sum_logprobs: float) -> None:
        score = sum_logprobs / (len(hyp) ** self.lp)
        if len(self.beams) < self.k or score > self.worst:
            self.beams.append((score, list(hyp)))
            if len(self.beams) > self.k:
                srt = sorted([(sc, i) for i, (sc, _) in enumerate(self.beams)])
                del self.beams[srt[0][1]]
                self.worst = srt[1][0]
            else:
                self.worst = min(score, self.worst)

    def is_done(self, best: float, cur_len: int) -> bool:
        if len(self.beams) < self.k:
            return False
        if self.es is True:
            return True
        if self.es == "never" and self.lp > 0.0:
            return self.worst >= best / self.max_length ** self.lp
        return self.worst >= best / cur_len ** self.lp


def beam_generate(step_logits: Callable, prompt: torch.Tensor, max_new_tokens: int, num_beams: int,
                  do_sample: bool = False, temperature: float = 1.0, top_p: float = 1.0, length_penalty: float = 1.0,
                  early_stopping=False, eos: Optional[int] = None, pad: int = 0, seed: int = 0, offset: int = 0):
    """step_logits(input_ids [B*k, cur], beam_idx [B*k] or None) -> last-position logits [B*k, V] (fp16 or fp32).
    Returns (sequences [B, width], best scores [B] fp32, smallest key margin, nucleus margin,
    {"hyps_added": hypotheses the scorer accepted before finalize, "steps": steps run, "all_done": stopped early})."""
    k = num_beams
    B, S = prompt.shape
    max_length = S + max_new_tokens
    ids = prompt.cpu().repeat_interleave(k, dim=0)
    beam_scores = torch.zeros((B, k), dtype=torch.float32)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view(-1)
    hyps = [Hyps(k, length_penalty, early_stopping, max_length) for _ in range(B)]
    done = [False] * B
    beam_idx, step, kmin, nmin, added = None, 0, float("inf"), 1.0, 0
    while True:
        cur_len = ids.shape[1]
        logits = step_logits(ids, beam_idx).cpu()
        V = logits.shape[-1]
        s = (log_probs(logits) + beam_scores[:, None]).view(B, k * V)
        sc, ix, km, nm = select(s, k, do_sample, temperature, top_p, seed, offset, step)
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
                    added += 1
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
    stats = {"hyps_added": added, "steps": step, "all_done": all(done)}
    for i in range(B):
        if not done[i]:
            for j in range(k):
                hyps[i].add(ids[i * k + j].tolist(), float(beam_scores[i * k + j]))
    best, best_scores = [], torch.zeros(B, dtype=torch.float32)
    for i in range(B):
        srt = sorted(hyps[i].beams, key=lambda x: x[0])
        best.append(srt[-1][1])
        best_scores[i] = srt[-1][0]
    width = min(max(len(h) for h in best) + 1, max_length)
    out = torch.full((B, width), pad, dtype=torch.int64)
    for i, h in enumerate(best):
        out[i, :len(h)] = torch.tensor(h)
        if len(h) < width and eos is not None:
            out[i, len(h)] = eos
    return out, best_scores, kmin, nmin, stats
