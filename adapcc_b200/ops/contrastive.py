"""Contrastive search (Su et al., "A Contrastive Framework for Neural Text Generation", 2022; HuggingFace's
``penalty_alpha`` + ``top_k``) evaluated in fp64: the CPU / non-bf16 path of ``GPT2DoubleHeads.contrastive_search``
and the reference the GPU tests compare ``contrastive_select_`` and ``contrastive_rerank_`` (csrc/ops_contrastive.cu)
against.

Row b has a *sequence* (its prompt without padding, then its chosen tokens) and a *context* ``C_b``: the final
hidden state at every position of that sequence (the prompt's from the prefill, then each chosen candidate's). Padding
is never part of the context, so a row's result does not depend on the other prompts of the batch. At each step, on the
fp32 logits ``l`` of the row's last position (DESIGN.md §4a):

1. the sequence bias and repetition controls, when on, are applied as in ``generate`` (``ops/repeats.py``); then, while
   ``step < min_new_tokens``, the ids in ``suppress_ids`` are removed;
2. the candidates are the ``top_k`` ids with the largest remaining logits, ranked by descending logit, ties to the
   lower id; ids at -inf are never candidates, and if fewer than ``top_k`` remain the missing slots are invalid;
3. candidate j gets ``p_j = exp(l_j - m) / sum_i exp(l_i - m)`` over the remaining ids;
4. ``h_j`` is the final hidden state of the sequence extended by candidate j (one decode step from the row's cache);
5. ``s_j = max over c in C_b of cos(h_j, c)``, a cosine with a zero-norm vector counting as 0;
6. ``score_j = (1 - alpha) p_j - alpha s_j``; the highest score wins, ties to the lower rank;
7. the winner's token is emitted and its hidden state appended to ``C_b`` (its keys and values become the cache's
   entry at that position). A stop id ends the row: the output gets -1 from there on. A row without a valid candidate
   emits id 0.

Ranking by logit with ties to the lower rank makes ``alpha = 0`` or ``top_k = 1`` exactly greedy decoding.
"""
from __future__ import annotations

import math
from typing import Dict, Sequence, Tuple

import numpy as np
import torch


def check_contrastive_args(who: str, top_k: int, penalty_alpha: float, max_k: int) -> None:
    """``ValueError`` unless ``1 <= top_k <= max_k`` and ``0 <= penalty_alpha <= 1``."""
    if int(top_k) != top_k or not 1 <= int(top_k) <= max_k:
        raise ValueError(f"{who}: top_k must be an integer in [1, {max_k}], got {top_k}")
    if not (isinstance(penalty_alpha, (int, float)) and math.isfinite(penalty_alpha) and 0 <= penalty_alpha <= 1):
        raise ValueError(f"{who}: penalty_alpha must be in [0, 1], got {penalty_alpha}")


def candidates_row(logits, top_k: int, step: int = 0, min_new: int = 0,
                   suppress_ids: Sequence[int] = ()) -> Tuple[np.ndarray, np.ndarray]:
    """Steps 1 (suppression) to 3 for one row of ``vocab`` fp32 logits: ``(ids, probs)``, int64 and fp64 [top_k],
    best first, -1 and 0 in invalid slots."""
    x = np.array(logits, dtype=np.float32).reshape(-1)
    if step < min_new:
        ids = np.array([i for i in suppress_ids if 0 <= i < x.size], dtype=np.int64)
        x[ids] = -np.inf
    ids, probs = np.full(top_k, -1, dtype=np.int64), np.zeros(top_k)
    live = np.flatnonzero(x > -np.inf)
    if live.size == 0:
        return ids, probs
    xd = x.astype(np.float64)
    m = xd[live].max()
    Z = np.exp(xd[live] - m).sum()
    order = live[np.argsort(-xd[live], kind="stable")][:top_k]    # live is ascending: ties keep the lower id first
    ids[:order.size] = order
    probs[:order.size] = np.exp(xd[order] - m) / Z
    return ids, probs


def max_cosine(h, ctx) -> np.ndarray:
    """Step 5: ``s_j = max_c cos(h_j, c)`` in fp64 for ``h`` [k, D] against ``ctx`` [n, D] (n >= 1); a zero norm gives
    cosine 0."""
    h = np.asarray(h, dtype=np.float64)
    c = np.asarray(ctx, dtype=np.float64)
    hn, cn = np.linalg.norm(h, axis=1), np.linalg.norm(c, axis=1)
    den = hn[:, None] * cn[None, :]
    cos = np.where(den > 0, (h @ c.T) / np.where(den > 0, den, 1.0), 0.0)
    return cos.max(axis=1)


def rerank_row(ids, probs, h, ctx, alpha: float) -> Dict[str, object]:
    """Steps 5 and 6 for one row: ``ids`` / ``probs`` from ``candidates_row``, ``h`` [k, D] the candidates' hidden states
    (invalid slots ignored), ``ctx`` [n, D]. Returns ``rank`` (the winner's slot; 0 without a valid candidate),
    ``token`` (its id; 0 without one), ``scores`` (fp64 [k], -inf in invalid slots) and ``sims`` (fp64 [k])."""
    ids = np.asarray(ids)
    valid = ids >= 0
    sims = np.zeros(ids.size)
    if valid.any():
        sims[valid] = max_cosine(np.asarray(h, dtype=np.float64)[valid], ctx)
    scores = np.where(valid, (1.0 - alpha) * np.asarray(probs, dtype=np.float64) - alpha * sims, -np.inf)
    rank = int(np.argmax(scores)) if valid.any() else 0                        # argmax: the first of equal scores
    return {"rank": rank, "token": int(ids[rank]) if valid.any() else 0, "scores": scores, "sims": sims}


def select_candidates(logits, vocab: int, top_k: int, step: int = 0, min_new: int = 0,
                      suppress_ids: Sequence[int] = (), done=None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Steps 1-3 for a batch: ``logits`` [B, >= vocab] (fp32 values), ``done`` [B] (rows that are done get no
    candidate). Returns ``(ids, probs)``: int64 [B, top_k] with -1 in invalid slots, fp64 [B, top_k]."""
    rows = torch.as_tensor(logits)[:, :vocab].detach().float().cpu().numpy()
    B = rows.shape[0]
    ids, probs = np.full((B, top_k), -1, dtype=np.int64), np.zeros((B, top_k))
    for b in range(B):
        if done is None or not bool(done[b]):
            ids[b], probs[b] = candidates_row(rows[b], top_k, step, min_new, suppress_ids)
    return torch.from_numpy(ids), torch.from_numpy(probs)
