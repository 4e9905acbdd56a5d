"""TEST INFRASTRUCTURE ONLY -- restatement of the `scores` transformers 4.30.2 returns from
generate(output_scores=True, return_dict_in_generate=True) in greedy decoding and sampling (include/seedb200.h,
seedb200_gen_outputs), built on tests/processors_ref.py.

  greedy_search (generation/utils.py, 4.30.2): next_tokens_scores = logits_processor(input_ids, next_token_logits);
                scores += (next_tokens_scores,)
  sample        next_token_scores = logits_processor(...); next_token_scores = logits_warper(input_ids,
                next_token_scores); scores += (next_token_scores,) -- Temperature (only when T != 1), TopK, TopP, each
                with filter_value -inf
  both          one entry per loop iteration; the loop ends once every row has finished, so len(scores) equals the
                generated width of `sequences`
"""
from __future__ import annotations

from typing import Callable, List

import numpy as np
import torch

import beam_ref as BR
import processors_ref as PR


def score_row(logits: torch.Tensor, hist: List[int], S: int, eos: int, ctl: dict, do_sample: bool,
              temperature: float = 1.0, top_p: float = 1.0):
    """one row's entry of `scores` (fp16 [V]) and the nucleus margin of its TopP boundary (1.0 without TopP): a
    kernel that sums in another order may legitimately keep or drop a token whose margin is ~1e-6"""
    x = PR.process(logits, hist, S, eos, ctl)
    if not do_sample:
        return x, 1.0
    key = x if temperature == 1.0 else PR.scalar_div(x, temperature)
    keep = PR.top_k_keep(key, int(ctl.get("top_k", 0)), 1).numpy()
    margin = 1.0
    if top_p < 1.0:
        xs = np.where(keep, key.float().numpy().astype(np.float64), -np.inf)
        p = np.exp(xs - xs.max())
        p /= p.sum()
        order = np.argsort(xs, kind="stable")
        cs = np.cumsum(p[order])
        rem = cs <= (1.0 - top_p)
        rem[-1:] = False
        kept = np.ones_like(rem)
        kept[order] = ~rem
        keep = keep & (xs >= xs[kept].min())          # threshold form: every token tied with the least kept one stays
        live = cs > 0
        margin = float(np.min(np.abs(cs[live] - (1.0 - top_p)))) if live.any() else 1.0
    return torch.where(torch.from_numpy(keep), key, torch.full_like(key, float("-inf"))), margin


def teacher_forced(step_logits: Callable, sequences: torch.Tensor, S: int, ctl: dict, do_sample: bool,
                   temperature: float = 1.0, top_p: float = 1.0, eos: int = -1):
    """`scores` of a finished generation: step t's entry from step_logits(sequences[:, :S + t]) (the last position's
    logits [B, V]) and each row's input ids.  Returns (tuple of [B, V], smallest nucleus margin)."""
    seq = sequences.cpu()
    out, mmin = [], 1.0
    for t in range(seq.shape[1] - S):
        logits = step_logits(seq[:, :S + t]).cpu()
        rows = []
        for b in range(seq.shape[0]):
            r, m = score_row(logits[b], seq[b, :S + t].tolist(), S, eos, ctl, do_sample, temperature, top_p)
            rows.append(r)
            mmin = min(mmin, m)
        out.append(torch.stack(rows))
    return tuple(out), mmin


# ---- beam search and beam sampling ---------------------------------------------------------------------------------
# beam_search (generation/utils.py, 4.30.2): scores += (next_token_scores_processed,) -- the processed fp16
#     log_softmax of each beam row, before `+ beam_scores[:, None]`
# beam_sample: scores += (logits_warper(input_ids, next_token_scores_processed),) -- the warpers (Temperature, TopK and
#     TopP with min_tokens_to_keep = 2, as _get_logits_warper builds them for num_beams > 1) on that row, not on the
#     `next_token_scores` the draws use
# BeamSearchScorer.process / finalize (beam_search.py, 4.30.2): a new beam's indices are beam_indices[batch_beam_idx] +
#     (batch_beam_idx,), and so are those of an eos hypothesis (one entry more than its tokens); finalize pads with -1
#     to the width of `sequences`
# len(scores): one entry per loop iteration; the loop ends after the iteration at which beam_scorer.is_done, or at
#     max_length


def beam_warp_row(lp: torch.Tensor, temperature: float, top_k: int, top_p: float):
    """beam_sample's warpers on one processed fp16 row (threshold form) -> (fp16 row, TopP boundary margin)"""
    v = lp if temperature == 1.0 else PR.scalar_div(lp, temperature)
    keep = PR.top_k_keep(v, top_k, 2)
    margin = 1.0
    if top_p < 1.0:
        vf = torch.where(keep, v.float(), torch.tensor(float("-inf")))
        kp, margin = BR.top_p_keep(vf[None], top_p, min_keep=2)
        keep = keep & kp[0]
    return torch.where(keep, v, torch.full_like(v, float("-inf"))), margin


def beam_generate(step_logits: Callable, prompt: torch.Tensor, max_new_tokens: int, num_beams: int, ctl: dict,
                  do_sample: bool = False, temperature: float = 1.0, top_p: float = 1.0, length_penalty: float = 1.0,
                  early_stopping=False, eos=None, pad: int = 0, seed: int = 0, offset: int = 0):
    """processors_ref.beam_generate with the outputs of return_dict_in_generate=True, output_scores=True.  Returns
    (sequences [B, width], scores (tuple of fp16 [B * k, V]), sequences_scores [B], beam_indices [B, width],
    smallest key margin, smallest TopP margin)."""
    k = num_beams
    B, S = prompt.shape
    max_length = S + max_new_tokens
    ids = prompt.cpu().repeat_interleave(k, dim=0)
    chains = [[] for _ in range(B * k)]
    beam_scores = torch.zeros((B, k), dtype=torch.float32)
    beam_scores[:, 1:] = -1e9
    beam_scores = beam_scores.view(-1)
    hyps = [BR.Hyps(k, length_penalty, early_stopping, max_length) for _ in range(B)]
    chain_of = {}                               # (search, score, hyp tokens) -> beam indices
    done = [False] * B
    beam_idx, step, kmin, nmin, scores = None, 0, float("inf"), 1.0, []
    e = -1 if eos is None else eos
    top_k = int(ctl.get("top_k", 0))
    while True:
        logits = step_logits(ids, beam_idx).cpu()
        V = logits.shape[-1]
        lp16 = BR.log_probs(logits).to(logits.dtype)
        lp16 = torch.stack([PR.process(lp16[r], ids[r].tolist(), S, e, ctl) for r in range(B * k)])
        if do_sample:
            rows = []
            for r in range(B * k):
                w, m = beam_warp_row(lp16[r], temperature, top_k, top_p)
                rows.append(w)
                nmin = min(nmin, m)
            scores.append(torch.stack(rows))
        else:
            scores.append(lp16.clone())
        s = (lp16.float() + beam_scores[:, None]).view(B, k * V)
        sc, ix, km, nm = PR.beam_select(s, k, top_k, do_sample, temperature, top_p, seed, offset, step)
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
                row = i * k + beam
                if eos is not None and tok == eos:
                    if r >= k:
                        continue
                    h = ids[row].tolist()
                    chain_of[(i, float(sc[i, r]) / (len(h) ** length_penalty), tuple(h))] = chains[row] + [row]
                    hyps[i].add(h, float(sc[i, r]))
                else:
                    nb_s[i, bi], nb_t[i, bi], nb_i[i, bi] = sc[i, r], tok, row
                    bi += 1
                if bi == k:
                    break
            done[i] = done[i] or hyps[i].is_done(float(sc[i].max()), ids.shape[1])
        beam_scores = nb_s.view(-1)
        beam_idx = nb_i.view(-1)
        chains = [chains[int(r)] + [int(r)] for r in beam_idx]
        ids = torch.cat([ids[beam_idx], nb_t.view(-1, 1)], dim=1)
        step += 1
        if all(done) or ids.shape[1] >= max_length:
            break
    for i in range(B):
        if not done[i]:
            for j in range(k):
                h = ids[i * k + j].tolist()
                chain_of[(i, float(beam_scores[i * k + j]) / (len(h) ** length_penalty), tuple(h))] = chains[i * k + j]
                hyps[i].add(h, float(beam_scores[i * k + j]))
    best = [sorted(h.beams, key=lambda x: x[0])[-1] for h in hyps]
    width = min(max(len(h) for _, h in best) + 1, max_length)
    out = torch.full((B, width), pad, dtype=torch.int64)
    indices = torch.full((B, width), -1, dtype=torch.int64)
    for i, (sc_h, h) in enumerate(best):
        out[i, :len(h)] = torch.tensor(h)
        if len(h) < width and eos is not None:
            out[i, len(h)] = eos
        c = chain_of[(i, sc_h, tuple(h))]
        indices[i, :len(c)] = torch.tensor(c, dtype=torch.int64)
    seq_scores = torch.tensor([sc_h for sc_h, _ in best], dtype=torch.float32)
    return out, tuple(scores), seq_scores, indices, kmin, nmin
