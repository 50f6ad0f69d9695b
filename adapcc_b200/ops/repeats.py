"""The repetition controls and sequence bias of GPT-2 generation and beam search, the definition of ``penalize_repeats_``
(csrc/ops_repeats.cu) evaluated in fp32 with numpy: the CPU / non-bf16 path of ``GPT2DoubleHeads.generate`` and
``beam_search`` and the reference the GPU tests compare the kernel against, bit for bit.

Row r's *sequence* is its prompt (the first ``lengths[b]`` ids, without padding) followed by the tokens generated so
far; for a beam, the tokens of its own hypothesis. The definition applies to the row's fp32 logits ``l_i``,
``i < vocab``, before step 1 of ``ops/sampling.py`` or ``ops/beam.py`` (DESIGN.md §4a), in this order:

0. sequence bias (a ``SequenceBias`` table shared by all rows; None: off). Each entry is a token sequence ``s`` of
   length ``m >= 1`` and an fp32 bias ``b``: HuggingFace's ``sequence_bias`` with its finite biases, then its
   ``bad_words_ids`` with ``b = -inf`` (a one-token bad word in ``stop_ids`` is dropped, so a row can still stop). An
   entry *applies* to a row whose sequence has length L when ``m = 1``, or when ``L >= m`` and
   ``seq[L - m + 1:L] == s[:m - 1]`` (HuggingFace ignores a sequence longer than the context, so a bad word whose
   prefix is the whole sequence so far, such as two ids after a one-token prompt, is not blocked). For every target id
   ``t`` with at least one applicable entry whose last id is t, the applicable biases are summed in fp32, each
   addition correctly rounded, in this order: t's length-1 ``sequence_bias`` entry, then its longer
   ``sequence_bias`` entries in the order given, then its bad words; then ``l_t <- fl32(l_t + sum)``. Other ids are
   unchanged. This is HuggingFace's ``SequenceBiasLogitsProcessor`` before, and ``NoBadWordsLogitsProcessor`` after,
   rules 1 and 2: -inf is unchanged by both rules and logits are never +inf, so applying the bad words here gives the
   same values. HuggingFace adds +0.0 to every id, so its -0.0 logits become +0.0; here ids without an applicable
   entry keep their bits;
1. repetition penalty ``p > 0`` (1 = off): for every *distinct* id ``i < vocab`` in the sequence,
   ``l_i <- fl32(l_i * p)`` if ``l_i < 0`` and ``fl32(l_i / p)`` otherwise, with ``p`` rounded to fp32 once and each
   operation correctly rounded. Each id is penalised once however often it occurs; ids outside ``[0, vocab)`` are
   ignored. This is HuggingFace's ``RepetitionPenaltyLogitsProcessor``;
2. no-repeat n-grams ``n >= 1`` (0 = off): with ``L`` the sequence length, for every ``j`` with ``j + n - 1 < L`` and
   ``seq[j:j + n - 1] == seq[L - n + 1:L]``, ``l_{seq[j + n - 1]} <- -inf``. For ``n = 1`` every id of the sequence is
   banned; for ``L < n`` nothing is. This is HuggingFace's ``NoRepeatNGramLogitsProcessor`` on a decoder-only model:
   the prompt counts, and so do n-grams that cross from the prompt into the reply.

Ids at -inf are never candidates of the sampler or the beam selection. In beam search all three rules act on the
logits before the log-softmax, so a beam's log-probabilities are renormalised over the ids that remain and the biased
values (as ``suppress_ids`` are); HuggingFace and fairseq process the log-probabilities after normalisation instead.
"""
from __future__ import annotations

import math
from numbers import Integral, Real
from typing import Optional, Sequence

import numpy as np
import torch


def check_repeat_args(who: str, penalty: float, ngram: int) -> None:
    """``ValueError`` unless ``penalty`` is finite and > 0 and ``ngram >= 0``."""
    if not (isinstance(penalty, (int, float)) and math.isfinite(penalty) and penalty > 0):
        raise ValueError(f"{who}: repetition_penalty must be a finite number > 0, got {penalty}")
    if int(ngram) != ngram or int(ngram) < 0:
        raise ValueError(f"{who}: no_repeat_ngram_size must be an integer >= 0, got {ngram}")


BIAS_MAX_ENTRIES = 1024      # sequence-bias entries per call, biases and bad words together
BIAS_MAX_LEN = 32            # ids per entry


class SequenceBias:
    """Rule 0's table, built by ``check_sequence_bias_args``: the distinct target ids ``targets`` int32 [U] and per
    target u its entries ``start[u]:start[u + 1]`` in the defined order; per entry e its prefix (the entry's first
    m - 1 ids) ``prefix[pre_off[e]:pre_off[e] + pre_len[e]]`` and its fp32 bias ``bias[e]``. ``tab`` is the int32
    array ``penalize_repeats_`` reads, ``[targets | start | pre_off | pre_len | prefixes]``, with ``pre_off`` counted
    from the start of ``tab``."""

    def __init__(self, per_target):
        """``per_target``: (target, [(prefix ids, bias), ...]) in order."""
        U = len(per_target)
        ents = [e for _, es in per_target for e in es]
        E = len(ents)
        self.targets = np.array([t for t, _ in per_target], dtype=np.int32)
        self.start = np.cumsum([0] + [len(es) for _, es in per_target]).astype(np.int32)
        self.pre_len = np.array([len(p) for p, _ in ents], dtype=np.int32)
        self.pre_off = (2 * U + 1 + 2 * E + np.cumsum(np.r_[0, self.pre_len[:-1]])).astype(np.int32)
        self.bias = np.array([b for _, b in ents], dtype=np.float32)
        self.tab = np.concatenate([self.targets, self.start, self.pre_off, self.pre_len,
                                   np.array([i for p, _ in ents for i in p], dtype=np.int32)]).astype(np.int32)
        self.max_id = int(max(self.tab[2 * U + 1 + 2 * E:].max(initial=-1), self.targets.max(initial=-1)))
        self._dev = {}

    @property
    def num_targets(self) -> int:
        """U, the distinct target ids."""
        return int(self.targets.size)

    @property
    def num_entries(self) -> int:
        """E, the entries of all targets."""
        return int(self.bias.size)

    def device_tensors(self, device):
        """``(tab int32, bias fp32)`` on ``device``, made once per device so that a captured graph keeps its
        pointers."""
        key = str(torch.device(device))
        if key not in self._dev:
            self._dev[key] = (torch.from_numpy(self.tab).to(device), torch.from_numpy(self.bias).to(device))
        return self._dev[key]

    def apply_row(self, row: np.ndarray, s: np.ndarray, vocab: int) -> None:
        """Rule 0 on one fp32 row in place, ``s`` the row's sequence."""
        L = s.size
        for u, t in enumerate(self.targets):
            total, hit = np.float32(0.0), False
            for e in range(self.start[u], self.start[u + 1]):
                m1 = int(self.pre_len[e])
                if m1 > 0 and (m1 >= L or not np.array_equal(
                        s[L - m1:], self.tab[self.pre_off[e]:self.pre_off[e] + m1])):
                    continue
                total = self.bias[e] if not hit else np.float32(total + self.bias[e])
                hit = True
            if hit and 0 <= t < vocab:
                row[t] = np.float32(row[t] + total)


def _id_seq(who: str, name: str, ids, vocab: int) -> tuple:
    if isinstance(ids, (str, bytes)) or not hasattr(ids, "__len__"):
        raise ValueError(f"{who}: each {name} entry must be a sequence of token ids, got {ids!r}")
    out = []
    for i in ids:
        if isinstance(i, bool) or not isinstance(i, Integral):
            raise ValueError(f"{who}: {name} ids must be integers, got {i!r} in {list(ids)}")
        if not 0 <= int(i) < vocab:
            raise ValueError(f"{who}: {name} ids must be in [0, vocab = {vocab}), got {int(i)} in {list(ids)}")
        out.append(int(i))
    if not 1 <= len(out) <= BIAS_MAX_LEN:
        raise ValueError(f"{who}: each {name} entry must have 1 to BIAS_MAX_LEN = {BIAS_MAX_LEN} ids, got "
                         f"{len(out)}")
    return tuple(out)


def check_sequence_bias_args(who: str, sequence_bias, bad_words_ids, vocab: int,
                             stop_ids: Sequence[int] = ()) -> Optional[SequenceBias]:
    """Rule 0's table from HuggingFace's ``sequence_bias`` (a dict ``{tuple(ids): bias}`` or a list of ``[ids, bias]``
    pairs) and ``bad_words_ids`` (a list of id lists); None when both are None or empty. ``ValueError`` naming
    ``who`` for an id outside ``[0, vocab)``, an empty or too long entry, a non-finite bias, a sequence listed twice in
    ``sequence_bias`` or more than ``BIAS_MAX_ENTRIES`` entries in all. A one-token bad word in ``stop_ids`` is
    dropped."""
    seq_entries, bad_entries = [], []
    if sequence_bias is not None:
        items = sequence_bias.items() if isinstance(sequence_bias, dict) else sequence_bias
        if isinstance(items, (str, bytes)) or not hasattr(items, "__iter__"):
            raise ValueError(f"{who}: sequence_bias must be a dict or a list of [ids, bias] pairs, got "
                             f"{type(sequence_bias).__name__}")
        seen = set()
        for item in items:
            if isinstance(item, (str, bytes)) or not hasattr(item, "__len__") or len(item) != 2:
                raise ValueError(f"{who}: each sequence_bias entry must be an [ids, bias] pair, got {item!r}")
            ids, b = item
            ids = _id_seq(who, "sequence_bias", ids, vocab)
            if isinstance(b, bool) or not isinstance(b, Real) or not math.isfinite(float(b)):
                raise ValueError(f"{who}: sequence_bias biases must be finite numbers, got {b!r} for {list(ids)}")
            if ids in seen:
                raise ValueError(f"{who}: sequence_bias lists {list(ids)} twice")
            seen.add(ids)
            seq_entries.append((ids, np.float32(b)))
    if bad_words_ids is not None:
        if isinstance(bad_words_ids, (str, bytes, dict)) or not hasattr(bad_words_ids, "__iter__"):
            raise ValueError(f"{who}: bad_words_ids must be a list of id lists, got {type(bad_words_ids).__name__}")
        stops = set(int(x) for x in stop_ids)
        for ids in bad_words_ids:
            ids = _id_seq(who, "bad_words_ids", ids, vocab)
            if not (len(ids) == 1 and ids[0] in stops):
                bad_entries.append((ids, np.float32(-np.inf)))
    n = len(seq_entries) + len(bad_entries)
    if n > BIAS_MAX_ENTRIES:
        raise ValueError(f"{who}: at most BIAS_MAX_ENTRIES = {BIAS_MAX_ENTRIES} sequence_bias and bad_words_ids "
                         f"entries in all, got {n}")
    if n == 0:
        return None
    # per target: its length-1 sequence_bias entry, its longer sequence_bias entries in order, then its bad words
    order = [e for e in seq_entries if len(e[0]) == 1] + [e for e in seq_entries if len(e[0]) > 1] + bad_entries
    per = {}
    for ids, b in order:
        per.setdefault(ids[-1], []).append((ids[:-1], b))
    return SequenceBias(list(per.items()))


def banned_ngram_ids(seq: np.ndarray, n: int) -> np.ndarray:
    """Rule 2: the ids ``seq[j + n - 1]`` of every earlier n-gram whose first n - 1 ids equal the sequence's last
    n - 1 (all of them for n = 1, none for ``len(seq) < n``), out-of-range ids included."""
    L = seq.size
    if n < 1 or L < n:
        return seq[:0]
    win = np.lib.stride_tricks.sliding_window_view(seq, n)           # [L - n + 1, n]: every n-gram
    match = (win[:, :n - 1] == seq[L - n + 1:]).all(axis=1)
    return win[match, n - 1]


def penalize_repeats_reference(logits, seqs: Sequence, vocab: int, penalty: float, ngram: int,
                               bias: Optional[SequenceBias] = None) -> torch.Tensor:
    """Rules 0 (with ``bias``), 1 and 2 for R rows: ``logits`` [R, >= vocab] (fp32 values), ``seqs`` R sequences (int
    lists, arrays or tensors). Returns a new fp32 tensor of the logits' shape on their device; columns from ``vocab``
    on are copied."""
    t = logits if isinstance(logits, torch.Tensor) else torch.as_tensor(logits)
    x = t.detach().to(device="cpu", dtype=torch.float32).numpy().copy()
    if len(seqs) != x.shape[0]:
        raise ValueError(f"penalize_repeats_reference: {x.shape[0]} rows but {len(seqs)} sequences")
    p = np.float32(penalty)
    for r, s in enumerate(seqs):
        s = np.asarray(s.cpu() if isinstance(s, torch.Tensor) else s, dtype=np.int64).reshape(-1)
        row = x[r]
        if bias is not None:
            bias.apply_row(row, s, vocab)
        if p != np.float32(1.0):
            ids = np.unique(s[(s >= 0) & (s < vocab)])
            v = row[ids]
            row[ids] = np.where(v < 0, v * p, v / p)
        if ngram > 0:
            ban = banned_ngram_ids(s, int(ngram))
            row[ban[(ban >= 0) & (ban < vocab)]] = -np.inf
    return torch.from_numpy(x).to(t.device if isinstance(logits, torch.Tensor) else "cpu")
