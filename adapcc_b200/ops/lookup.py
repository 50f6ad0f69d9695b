"""Prompt-lookup speculative decoding for greedy generation (HuggingFace's ``prompt_lookup_num_tokens``): the CPU /
non-bf16 path of ``GPT2DoubleHeads.generate(..., prompt_lookup_num_tokens=k)`` and the reference the GPU tests compare
``lookup_accept_`` and ``lookup_draft_`` (csrc/ops_lookup.cu) against.

Row b has emitted ``e_b`` tokens. Its *sequence* ``s_b`` is its prompt without padding, then those tokens; the last
one, ``x_b``, is not in the KV cache yet, so ``lens[b] = len_b + e_b - 1`` (DESIGN.md §4a). Before the first token
``e_b = 0``, ``x_b`` is the prompt's last token and the prefill's logits at that position play the verify step's.

1. *Drafts.* A live row may take ``r_b = min(k, max_new_tokens - e_b - 1)`` drafts. For ``m = min(ngram, |s_b| - 1)``
   down to 1, take the earliest window ``i`` with ``s_b[i:i+m] == s_b[-m:]`` and ``i + m < |s_b|``; the drafts are
   ``s_b[i+m : min(i+m+r_b, |s_b|)]``. No match: no drafts. The row holds ``nq_b = 1 + #drafts`` real slots of the
   ``k + 1`` (``x_b``, then the drafts, at positions ``lens[b] + j``); a done row holds none.
2. *Verify.* One model step over the slots gives slot j's logits, and ``g_j`` is their arg-max, the lowest id on a tie
   (``sample_reference`` at temperature 0), with ``suppress_ids`` removed while ``e_b + j < min_new_tokens``.
3. *Acceptance.* ``a`` is the largest count with ``d_i == g_{i-1}`` for all ``i <= a``; the row emits
   ``d_1 .. d_a, g_a`` (that is ``g_0 .. g_a``) in order. Emission stops at the first stop id, which sets ``done`` and
   is not written to the output, or when ``e_b`` reaches ``max_new_tokens``, which sets ``done`` too. Every emitted id
   joins the sequence, and ``lens`` and ``e_b`` grow by the number emitted.

The sequence, the output, ``done`` and ``lens`` of a live row advance exactly as if plain greedy decoding had emitted
the same tokens one at a time, and given the same per-position logits the emitted tokens are the greedy ones. The cap
``r_b`` keeps the last slot at most at position ``max(lengths) + max_new_tokens - 2``, inside ``generate``'s cache.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch

from .sampling import reference_row


def check_lookup_args(who: str, k: int, ngram: int, max_k: int, max_ngram: int, temperature: float,
                      repetition_penalty: float, no_repeat_ngram_size: int) -> None:
    """``ValueError`` unless ``1 <= k <= max_k``, ``1 <= ngram <= max_ngram``, ``temperature == 0`` and both
    repetition controls are off."""
    if int(k) != k or not 1 <= int(k) <= max_k:
        raise ValueError(f"{who}: prompt_lookup_num_tokens must be an integer in [0, {max_k}], got {k}")
    if int(ngram) != ngram or not 1 <= int(ngram) <= max_ngram:
        raise ValueError(f"{who}: max_matching_ngram_size must be an integer in [1, {max_ngram}], got {ngram}")
    if temperature != 0:
        raise ValueError(f"{who}: prompt_lookup_num_tokens > 0 needs temperature == 0 (greedy), got {temperature}")
    if repetition_penalty != 1.0:
        raise ValueError(f"{who}: prompt_lookup_num_tokens > 0 cannot be combined with repetition_penalty != 1, got "
                         f"{repetition_penalty}")
    if no_repeat_ngram_size > 0:
        raise ValueError(f"{who}: prompt_lookup_num_tokens > 0 cannot be combined with no_repeat_ngram_size > 0, got "
                         f"{no_repeat_ngram_size}")


def draft_row(seq: Sequence[int], cap: int, ngram: int) -> List[int]:
    """Step 1 for one row: the drafts (at most ``cap``) of the sequence ``seq``."""
    seq = [int(t) for t in seq]
    n = len(seq)
    if cap <= 0:
        return []
    for m in range(min(ngram, n - 1), 0, -1):
        tail = seq[n - m:]
        for i in range(n - m):                      # i + m < n: the continuation is not empty
            if seq[i:i + m] == tail:
                return seq[i + m:min(i + m + cap, n)]
    return []


def greedy_token(logits, step: int, min_new: int = 0, suppress_ids: Sequence[int] = ()) -> int:
    """Step 2 for one slot: the arg-max of fp32 ``logits`` [vocab], lowest id on a tie, ``suppress_ids`` removed while
    ``step < min_new``; id 0 if no id is left."""
    return int(reference_row(logits, 0.0, 0, 1.0, 0, 0, step, min_new, suppress_ids)["token"])


def accept_row(g: Sequence[int], drafts: Sequence[int], emitted: int, max_new: int,
               stop_ids: Sequence[int] = (), accepted: Sequence[bool] = None) -> Tuple[List[int], bool]:
    """Step 3 for one row: the slots' arg-maxes ``g`` (one per real slot) and the drafts (one fewer) -> the emitted ids
    (a stop id included, as the last one) and whether the row is now done. ``accepted`` (rejection sampling,
    ``ops/assisted.py``): per draft whether it is accepted, in place of "equals the token just emitted"; the row emits
    the leading accepted drafts, then ``g[a]`` (the token a round that ends at slot a emits)."""
    stop = set(int(s) for s in stop_ids)
    out: List[int] = []
    e = int(emitted)
    for j, t in enumerate(g):
        ok = accepted is not None and j + 1 < len(g) and bool(accepted[j])
        t = int(drafts[j]) if ok else int(t)
        out.append(t)
        e += 1
        if t in stop or e >= max_new:
            return out, True
        if (not ok) if accepted is not None else (j + 1 < len(g) and int(drafts[j]) != t):
            break
    return out, False


def lookup_draft(seq: torch.Tensor, lens: torch.Tensor, emitted: torch.Tensor, done: torch.Tensor, k: int,
                 max_new: int, ngram: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``lookup_draft_`` for a batch on the host: ``seq`` [B, t_max] (row b's sequence is ``seq[b, :lens[b] + 1]``),
    ``lens``, ``emitted``, ``done`` [B]. Returns ``(ids, pos, nq)``: int64 [B·(k+1)] the step's input (slot 0 ``x_b``,
    then the drafts, 0 in a pad slot), int64 [B·(k+1)] positions ``lens[b] + j`` clamped to ``t_max - 1``, and int32
    [B] the real slots (0 for a done row)."""
    B, t_max = seq.shape
    S = int(k) + 1
    seq, lens, emitted, done = (t.cpu() for t in (seq, lens, emitted, done))
    ids = torch.zeros(B, S, dtype=torch.int64)
    nq = torch.zeros(B, dtype=torch.int32)
    L = lens.long().clamp(0, t_max - 1)
    pos = (L[:, None] + torch.arange(S)).clamp(max=t_max - 1)
    for b in range(B):
        if done[b]:
            continue
        s = seq[b, :int(L[b]) + 1].tolist()
        d = draft_row(s, min(int(k), int(max_new) - int(emitted[b]) - 1), ngram)
        ids[b, 0] = s[-1]
        ids[b, 1:1 + len(d)] = torch.tensor(d, dtype=torch.int64)
        nq[b] = 1 + len(d)
    return ids.reshape(-1), pos.reshape(-1), nq


def lookup_accept(logits: torch.Tensor, vocab: int, ids: torch.Tensor, nq: torch.Tensor, seq: torch.Tensor,
                  lens: torch.Tensor, emitted: torch.Tensor, done: torch.Tensor, tokens: torch.Tensor,
                  steps: torch.Tensor = None, min_new: int = 0, suppress_ids: Sequence[int] = (),
                  stop_ids: Sequence[int] = (), drawn=None, accepted=None) -> None:
    """``lookup_accept_`` for a batch on the host, in place on the CPU tensors ``seq`` [B, t_max], ``lens``,
    ``emitted``, ``done`` [B], ``tokens`` [B, max_new] (-1 where nothing is written) and ``steps`` [B] (verify steps
    per live row; None: not counted). ``logits`` [B·ls, >= vocab] holds ``ls`` slots per row (1 for the prefill's
    logits, k + 1 for a verify step), ``ids`` [B·(k+1)] the step's input and ``nq`` [B] its real slots (at most
    ``ls`` are used). ``drawn`` [B, ls] (``lookup_accept_drawn_``): the slots' tokens, already drawn
    (``ops/assisted.py``), in place of the arg-maxes of ``logits`` (which may then be None). ``accepted`` [B, ls]
    (``lookup_accept_drawn_(..., flagged=True)``): per slot whether its draft is accepted (``accept_row``), with
    ``drawn`` holding each slot's last token."""
    B, t_max = seq.shape
    ls = logits.shape[0] // B if drawn is None else drawn.shape[1]
    S = ids.numel() // B
    max_new = tokens.shape[1]
    stop = set(int(s) for s in stop_ids)
    rows = None if drawn is not None else logits[:, :vocab].detach().float().cpu().numpy().reshape(B, ls, vocab)
    ids = ids.cpu().reshape(B, S)
    for b in range(B):
        if done[b]:
            continue
        e, L = int(emitted[b]), int(lens[b])
        n = max(0, min(int(nq[b]), ls))
        g = ([int(drawn[b, j]) for j in range(n)] if drawn is not None
             else [greedy_token(rows[b, j], e + j, min_new, suppress_ids) for j in range(n)])
        out, fin = accept_row(g, ids[b, 1:n].tolist(), e, max_new, stop_ids,
                              None if accepted is None else [bool(accepted[b, j]) for j in range(n)])
        for i, t in enumerate(out):
            if L + 1 + i < t_max:
                seq[b, L + 1 + i] = t
            if t not in stop and e + i < max_new:          # a stop id can only be the last one emitted
                tokens[b, e + i] = t
        lens[b] = L + len(out)
        emitted[b] = e + len(out)
        if fin:
            done[b] = 1
        if steps is not None:
            steps[b] += 1


def mean_tokens_per_step(emitted: torch.Tensor, steps: torch.Tensor) -> float:
    """Tokens emitted by verify steps (all but each row's first) per verify step of a live row."""
    n = int(steps.sum())
    return float((emitted.long() - 1).clamp(min=0).sum()) / n if n else float("nan")
