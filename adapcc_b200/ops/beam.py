"""The beam-search definition of ``beam_step_`` (csrc/ops_beam.cu) evaluated in fp64: the CPU / non-bf16 path of
``GPT2DoubleHeads.beam_search`` and the reference the GPU tests compare the kernels against.

For each item b there are K = ``num_beams`` beams; beam j has a running score ``s_j``, the sum of its tokens'
log-probabilities. At the start ``s = (0, -inf, ..., -inf)``: every beam starts from the same prompt, so only beam 0
is live. Per step, for every live beam row (DESIGN.md §4a):

1. while ``step < min_new`` the ids in ``suppress_ids`` are removed before anything else;
2. ``lp_i = (l_i - m) - log sum_j exp(l_j - m)`` over the remaining ids ``j < vocab``, from the fp32 logits; ``m`` is
   the row maximum;
3. a candidate ``(j, i)`` has score ``c = s_j + lp_i``;
4. candidates are ranked by descending ``c``, ties to the lower flat index ``j * V + i``; candidates at -inf are never
   taken;
5. walking the ranking, the first K candidates whose token is not in ``stop_ids`` become the new beams, in rank order
   (so the best live beam is beam 0); a stop candidate ranked before the K-th non-stop one is offered to the finished
   set; with fewer than K finite non-stop candidates the remaining beams are dead (-inf). Per row the best
   ``K + n_stop`` candidates decide this, which is what makes a bounded per-row selection exact;
6. the finished set keeps at most K hypotheses per item: one of L generated tokens (the stop token included) has the
   normalised score ``c / L ** length_penalty``; the set keeps the K best, the earlier insertion winning a tie;
7. an item is done when its set is full and no live beam can still beat the set's worst normalised score. A live sum
   can only fall (log-probabilities are <= 0), so its best reachable normalised score is ``s / max_new ** a`` for
   ``a = length_penalty > 0`` and ``s / (L + 1) ** a`` for ``a <= 0``: stopping early never changes the result;
8. items that reach ``max_new`` tokens without being done offer their live beams, in beam order, with
   ``L = max_new``. The result of an item is its best hypothesis: its tokens without the stop token, their number and
   the normalised score.

An item's result depends only on its prompt and the scalars, not on the other items.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch


class BeamReference:
    """The definition above for ``batch`` items, one step at a time, in fp64. ``step(logits)`` takes the beams'
    next-token logits [B·K, >= vocab] and returns ``(next_ids, parent)``: int64 [B·K] the new beams' tokens and the
    row (``b * K + j``) each continues. The state mirrors ``ops.BeamState``: ``scores`` [B, K], ``fin`` (per item a
    list of ``(normalised score, tokens, source beam)``, best first), ``done`` [B], ``hist_tok`` / ``hist_back``
    [max_new, B, K] and ``n_steps``. ``early_stop=False`` switches the done rule (7) off; the results must not change."""

    def __init__(self, batch: int, num_beams: int, max_new: int, vocab: int, length_penalty: float = 1.0,
                 stop_ids: Sequence[int] = (), suppress_ids: Sequence[int] = (), min_new: int = 0,
                 early_stop: bool = True):
        B, K = int(batch), int(num_beams)
        self.B, self.K, self.max_new, self.vocab = B, K, int(max_new), int(vocab)
        self.alpha = float(length_penalty)
        self.stop = set(int(i) for i in stop_ids)
        self.suppress = np.array(sorted(set(int(i) for i in suppress_ids if 0 <= int(i) < self.vocab)), dtype=np.int64)
        self.min_new, self.early_stop = int(min_new), bool(early_stop)
        self.scores = np.full((B, K), -np.inf)
        self.scores[:, 0] = 0.0
        self.fin: List[List[Tuple[float, int, int]]] = [[] for _ in range(B)]
        self.done = np.zeros(B, dtype=bool)
        self.hist_tok = np.full((self.max_new, B, K), -1, dtype=np.int64)
        self.hist_back = np.zeros((self.max_new, B, K), dtype=np.int64)
        self.n_steps = 0

    def penalty(self, L: int) -> float:
        """``L ** length_penalty``: the divisor of a hypothesis of L tokens."""
        return float(L) ** self.alpha

    def offer(self, b: int, score: float, n: int, src: int) -> None:
        """Rule 6: offer item b's finished set a hypothesis of normalised score ``score``, ``n`` tokens (without its
        stop token) and source beam ``src``."""
        fin = self.fin[b]
        if len(fin) == self.K and not score > fin[-1][0]:
            return
        p = len(fin)
        while p > 0 and fin[p - 1][0] < score:
            p -= 1
        fin.insert(p, (score, n, src))
        del fin[self.K:]

    def candidates(self, logits_row: np.ndarray, s: float, step: int) -> np.ndarray:
        """fp64 scores ``c_i = s + lp_i`` of one beam row (-inf for removed ids)."""
        x = np.array(logits_row[:self.vocab], dtype=np.float32).astype(np.float64)
        if step < self.min_new and self.suppress.size:
            x[self.suppress] = -np.inf
        if not np.isfinite(s) or not (x > -np.inf).any():
            return np.full(x.size, -np.inf)
        m = x.max()
        lse = np.log(np.exp(x - m).sum())
        return s + ((x - m) - lse)

    def ranking(self, b: int, logits: np.ndarray, step: int) -> List[Tuple[float, int, int]]:
        """Item b's finite candidates ``(c, j, i)`` in rank order, the best ``K + n_stop`` of each row (rule 5: the
        walk never reaches further into a row)."""
        K, V = self.K, self.vocab
        keep = K + len(self.stop)
        rows = []
        for j in range(K):
            c = self.candidates(logits[b * K + j], self.scores[b, j], step)
            ids = np.flatnonzero(c > -np.inf)
            if ids.size > keep:                                  # every id tied with the keep-th best stays in
                ids = ids[c[ids] >= np.partition(c[ids], ids.size - keep)[ids.size - keep]]
            ids = ids[np.lexsort((ids, -c[ids]))][:keep]
            rows.extend((float(c[i]), j * V + int(i)) for i in ids)
        rows.sort(key=lambda t: (-t[0], t[1]))
        return [(c, f // V, f % V) for c, f in rows]

    def step(self, logits) -> Tuple[torch.Tensor, torch.Tensor]:
        """One selection (rules 1-8) for every item that is not done; see the class docstring."""
        if isinstance(logits, torch.Tensor):
            logits = logits.detach().float().cpu().numpy()
        B, K = self.B, self.K
        step = self.n_steps
        if step >= self.max_new:
            raise ValueError(f"BeamReference: all {self.max_new} steps taken")
        nxt = np.zeros(B * K, dtype=np.int64)
        parent = np.arange(B * K, dtype=np.int64)
        L = step + 1
        for b in range(B):
            if self.done[b]:
                continue
            beams = []
            for c, j, i in self.ranking(b, logits, step):
                if len(beams) == K:
                    break
                if i in self.stop:
                    self.offer(b, c / self.penalty(L), L - 1, j)
                else:
                    beams.append((c, j, i))
            new = np.full(K, -np.inf)
            for k in range(K):
                if k < len(beams):
                    c, j, i = beams[k]
                    new[k], nxt[b * K + k], parent[b * K + k] = c, i, b * K + j
                    self.hist_tok[step, b, k], self.hist_back[step, b, k] = i, j
                else:
                    self.hist_tok[step, b, k], self.hist_back[step, b, k] = -1, k
            self.scores[b] = new
            if step == self.max_new - 1:
                for k in range(len(beams)):
                    self.offer(b, new[k] / self.penalty(self.max_new), self.max_new, k)
                self.done[b] = True
            elif not beams:
                self.done[b] = True
            elif self.early_stop and len(self.fin[b]) == K:
                reach = new[0] / self.penalty(self.max_new if self.alpha > 0 else L + 1)
                self.done[b] = not reach > self.fin[b][-1][0]
        self.n_steps += 1
        return torch.from_numpy(nxt), torch.from_numpy(parent)

    def result(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """``(tokens, n_new, scores)``: int64 [B, max_new] padded with -1, int64 [B], fp32 [B] of each item's best
        hypothesis (no tokens and -inf when an item has none)."""
        return best_hypotheses(self.fin, self.hist_tok, self.hist_back, self.max_new)


def best_hypotheses(fin, hist_tok, hist_back, max_new: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Each item's first finished hypothesis, its tokens followed back through the parent pointers. ``fin``: per item
    a best-first list of ``(normalised score, n, source beam)``; ``hist_tok`` / ``hist_back`` [max_new, B, K]."""
    B = len(fin)
    tokens = torch.full((B, max_new), -1, dtype=torch.int64)
    n_new = torch.zeros(B, dtype=torch.int64)
    scores = torch.full((B,), float("-inf"), dtype=torch.float32)
    for b in range(B):
        if not fin[b]:
            continue
        score, n, src = fin[b][0]
        r = int(src)
        for u in range(int(n) - 1, -1, -1):
            tokens[b, u] = int(hist_tok[u, b, r])
            r = int(hist_back[u, b, r])
        n_new[b], scores[b] = int(n), float(score)
    return tokens, n_new, scores
