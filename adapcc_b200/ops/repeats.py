"""The repetition controls of GPT-2 generation and beam search, the definition of ``penalize_repeats_``
(csrc/ops_repeats.cu) evaluated in fp32 with numpy: the CPU / non-bf16 path of ``GPT2DoubleHeads.generate`` and
``beam_search`` and the reference the GPU tests compare the kernel against, bit for bit.

Row r's *sequence* is its prompt (the first ``lengths[b]`` ids, without padding) followed by the tokens generated so
far; for a beam, the tokens of its own hypothesis. The definition applies to the row's fp32 logits ``l_i``,
``i < vocab``, before step 1 of ``ops/sampling.py`` or ``ops/beam.py`` (DESIGN.md §4a), in this order:

1. repetition penalty ``p > 0`` (1 = off): for every *distinct* id ``i < vocab`` in the sequence,
   ``l_i <- fl32(l_i * p)`` if ``l_i < 0`` and ``fl32(l_i / p)`` otherwise, with ``p`` rounded to fp32 once and each
   operation correctly rounded. Each id is penalised once however often it occurs; ids outside ``[0, vocab)`` are
   ignored. This is HuggingFace's ``RepetitionPenaltyLogitsProcessor``;
2. no-repeat n-grams ``n >= 1`` (0 = off): with ``L`` the sequence length, for every ``j`` with ``j + n - 1 < L`` and
   ``seq[j:j + n - 1] == seq[L - n + 1:L]``, ``l_{seq[j + n - 1]} <- -inf``. For ``n = 1`` every id of the sequence is
   banned; for ``L < n`` nothing is. This is HuggingFace's ``NoRepeatNGramLogitsProcessor`` on a decoder-only model:
   the prompt counts, and so do n-grams that cross from the prompt into the reply.

Ids at -inf are never candidates of the sampler or the beam selection. In beam search both controls act on the logits
before the log-softmax, so a beam's log-probabilities are renormalised over the ids that remain (as ``suppress_ids``
are); HuggingFace and fairseq process the log-probabilities after normalisation instead.
"""
from __future__ import annotations

import math
from typing import Sequence

import numpy as np
import torch


def check_repeat_args(who: str, penalty: float, ngram: int) -> None:
    """``ValueError`` unless ``penalty`` is finite and > 0 and ``ngram >= 0``."""
    if not (isinstance(penalty, (int, float)) and math.isfinite(penalty) and penalty > 0):
        raise ValueError(f"{who}: repetition_penalty must be a finite number > 0, got {penalty}")
    if int(ngram) != ngram or int(ngram) < 0:
        raise ValueError(f"{who}: no_repeat_ngram_size must be an integer >= 0, got {ngram}")


def banned_ngram_ids(seq: np.ndarray, n: int) -> np.ndarray:
    """Rule 2: the ids ``seq[j + n - 1]`` of every earlier n-gram whose first n - 1 ids equal the sequence's last
    n - 1 (all of them for n = 1, none for ``len(seq) < n``), out-of-range ids included."""
    L = seq.size
    if n < 1 or L < n:
        return seq[:0]
    win = np.lib.stride_tricks.sliding_window_view(seq, n)           # [L - n + 1, n]: every n-gram
    match = (win[:, :n - 1] == seq[L - n + 1:]).all(axis=1)
    return win[match, n - 1]


def penalize_repeats_reference(logits, seqs: Sequence, vocab: int, penalty: float, ngram: int) -> torch.Tensor:
    """Rules 1 and 2 for R rows: ``logits`` [R, >= vocab] (fp32 values), ``seqs`` R sequences (int lists, arrays or
    tensors). Returns a new fp32 tensor of the logits' shape on their device; columns from ``vocab`` on are copied."""
    t = logits if isinstance(logits, torch.Tensor) else torch.as_tensor(logits)
    x = t.detach().to(device="cpu", dtype=torch.float32).numpy().copy()
    if len(seqs) != x.shape[0]:
        raise ValueError(f"penalize_repeats_reference: {x.shape[0]} rows but {len(seqs)} sequences")
    p = np.float32(penalty)
    for r, s in enumerate(seqs):
        s = np.asarray(s.cpu() if isinstance(s, torch.Tensor) else s, dtype=np.int64).reshape(-1)
        row = x[r]
        if p != np.float32(1.0):
            ids = np.unique(s[(s >= 0) & (s < vocab)])
            v = row[ids]
            row[ids] = np.where(v < 0, v * p, v / p)
        if ngram > 0:
            ban = banned_ngram_ids(s, int(ngram))
            row[ban[(ban >= 0) & (ban < vocab)]] = -np.inf
    return torch.from_numpy(x).to(t.device if isinstance(logits, torch.Tensor) else "cpu")
