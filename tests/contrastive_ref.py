"""Restatement of contrastive search as transformers 4.30.2 runs it for the reference on CUDA in fp16
(GenerationMixin.contrastive_search + _ranking_fast), the contract of seedb200_llama_contrastive_generate
(include/seedb200.h, seedb200_contrastive_params).  transformers 4.30.2 is not installed (later releases moved contrastive
search to the Hub), so this file and its hand-worked cases in tests/test_contrastive_cpu.py are the statement.

Per sequence and step, at position p = S + t:
  logits  fp16 [V] -> the history processors of processors_ref.process (no warpers: top_k is the candidate count)
  probs   fp16(exp(x - max) * fp32(1 / sum)), max and sum in fp32         softmax(logits) of an fp16 tensor on CUDA
  (q_j, id_j), j < k: the k largest probs, descending, ties to the lower id  topk
  h_j     final RMSNorm output of candidate row j (hidden_states[-1]); logits_j its logits
  n(x)    fp16(float(x) / float(fp16(sqrt(sum float(x)^2))))               x / x.norm(dim=-1, keepdim=True)
  cos_ij  fp16(sum_d n(c_i)[d] n(h_j)[d]), fp32 accumulation (here float64, then one rounding)
  pen_j   max_i cos_ij, NaN propagating
  score_j fp16(fp16(fp32(1 - alpha) * q_j) - fp16(fp32(alpha) * pen_j))     1 - alpha in double, as Python computes it
  sel     argmax_j score_j, ties to the lower j, the first NaN wins           torch.max(dim=-1)
  token   id_sel, or pad once the sequence has finished
"""
from typing import Callable, List, Optional

import numpy as np
import torch

import processors_ref as PR


def softmax16(logits: torch.Tensor) -> torch.Tensor:
    """fp16 [..., V] -> fp16 probabilities: fp32 max and sum, torch's CUDA epilogue exp(x - max) * (1 / sum), one
    rounding"""
    x = logits.float()
    e = torch.exp(x - x.max(dim=-1, keepdim=True).values)
    return (e * (1.0 / e.sum(dim=-1, keepdim=True))).half()


def topk(probs: torch.Tensor, k: int):
    """the k largest of fp16 probs [V], descending, ties to the lower id -> (values fp16 [k], ids int64 [k])"""
    p = probs.float().numpy()
    order = np.lexsort((np.arange(p.shape[0]), -p))[:k]
    ids = torch.from_numpy(order.astype(np.int64))
    return probs[ids], ids


def normalise(x: torch.Tensor) -> torch.Tensor:
    """n(x) of fp16 rows [..., H]"""
    nrm = x.double().pow(2).sum(dim=-1, keepdim=True).sqrt().float().half()
    return (x.float() / nrm.float()).half()


def cosines(ctx_n: torch.Tensor, h_n: torch.Tensor) -> torch.Tensor:
    """fp16 [p, k] = fp16(n(c_i) . n(h_j)) of normalised fp16 rows"""
    return (ctx_n.double() @ h_n.double().T).half()


def nan_max(values: torch.Tensor) -> torch.Tensor:
    """max over dim 0 of [p, k], a NaN propagating"""
    m = values.float().max(dim=0).values
    return torch.where(torch.isnan(values.float()).any(dim=0), torch.full_like(m, float("nan")), m).half()


def c_prob(alpha: float) -> np.float32:
    """the scalar of (1.0 - alpha) * probs: Python's double 1 - alpha, rounded to fp32 (not 1 - fp32(alpha))"""
    return np.float32(1.0 - float(alpha))


def scores(q: torch.Tensor, pen: torch.Tensor, alpha: float) -> torch.Tensor:
    """fp16 [k] contrastive scores of fp16 probabilities q [k] and fp16 penalties pen [k]"""
    t1 = (torch.tensor(c_prob(alpha)) * q.float()).half()
    t2 = (torch.tensor(np.float32(alpha)) * pen.float()).half()
    return (t1.float() - t2.float()).half()


def select(sc: torch.Tensor) -> int:
    """torch.max(dim=-1) index: the largest score, ties to the lower index, the first NaN wins"""
    best = 0
    for j in range(1, sc.shape[0]):
        b, s = float(sc[best]), float(sc[j])
        if b != b:
            break
        if s != s or s > b:
            best = j
    return best


def rank(ctx_n: torch.Tensor, h: torch.Tensor, q: torch.Tensor, alpha: float):
    """one sequence: normalised context [p, H] fp16, candidates' raw h [k, H] fp16, probabilities q [k] fp16 ->
    (sel, scores fp16 [k], n(h) fp16 [k, H])"""
    hn = normalise(h)
    pen = nan_max(cosines(ctx_n, hn))
    sc = scores(q, pen, alpha)
    return select(sc), sc, hn


def gap(sc: torch.Tensor) -> float:
    """distance between the best and the second best score (inf for one finite score)"""
    v = sorted((float(x) for x in sc if x == x), reverse=True)
    return v[0] - v[1] if len(v) > 1 else float("inf")


def mode(num_beams: int = 1, do_sample: bool = False, top_k: Optional[int] = None,
         penalty_alpha: Optional[float] = None) -> str:
    """transformers 4.30.2 generate()'s mode selection over these four keywords"""
    if num_beams == 1 and not do_sample and top_k is not None and top_k > 1 and penalty_alpha is not None \
            and penalty_alpha > 0:
        return "contrastive"
    if num_beams == 1:
        return "sample" if do_sample else "greedy"
    return "beam_sample" if do_sample else "beam"


def generate(prefill: Callable, candidates_forward: Callable, prompt: torch.Tensor, max_new_tokens: int, k: int,
             alpha: float, ctl: dict, eos: Optional[int] = None, pad: int = 0, probs_fn: Callable = softmax16):
    """the contrastive_search loop.  prefill(prompt [B, S]) -> (last logits fp16 [B, V], hidden fp16 [B, S, H]);
    candidates_forward(step, ids [B, k]) -> (logits fp16 [B, k, V], h fp16 [B, k, H]), running the k candidates of
    every sequence on its selected past; its method on_select(step, sels) receives each step's selections.  Returns
    (new tokens [B, n], per-step top-2 score gaps [n][B], per-step k-th / (k+1)-th probability pairs [n][B])."""
    B, S = prompt.shape
    logits, hidden = prefill(prompt)
    ctx = [list(normalise(hidden[b])) for b in range(B)]
    seqs = [prompt[b].tolist() for b in range(B)]
    unfinished = [True] * B
    out, gaps, edges = [], [], []
    for t in range(max_new_tokens):
        ids = torch.empty((B, k), dtype=torch.int64)
        q = torch.empty((B, k), dtype=torch.float16)
        edge = []
        for b in range(B):
            row = PR.process(logits[b], seqs[b], S, -1 if eos is None else eos, dict(ctl, top_k=0))
            probs = probs_fn(row)
            q[b], ids[b] = topk(probs, k)
            nxt = topk(probs, k + 1)[0]
            edge.append((float(nxt[k - 1]), float(nxt[k])))
        cl, ch = candidates_forward(t, ids)
        toks, gp, sels = [], [], []
        for b in range(B):
            sel, sc, hn = rank(torch.stack(ctx[b]), ch[b], q[b], alpha)
            gp.append(gap(sc))
            sels.append(sel)
            ctx[b].append(hn[sel])
            tok = int(ids[b, sel]) if unfinished[b] else pad
            if eos is not None and tok == eos:
                unfinished[b] = False
            seqs[b].append(tok)
            toks.append(tok)
        logits = torch.stack([cl[b, sels[b]] for b in range(B)])
        candidates_forward.on_select(t, sels)
        out.append(toks)
        gaps.append(gp)
        edges.append(edge)
        if eos is not None and not any(unfinished):
            break
    return torch.tensor(out, dtype=torch.int64).T.reshape(B, -1), gaps, edges
