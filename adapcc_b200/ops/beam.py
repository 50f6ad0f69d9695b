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

Beam sampling (``BeamSampleReference``, HuggingFace's ``_beam_search`` with ``do_sample=True``) keeps rules 1, 6 and
7 and replaces 2-5 and 8. With ``n_stop`` stop ids, ``min_keep = max(2, 1 + n_stop)`` and ``M = min_keep · K``; per
step, for every live beam row j of item b:

S1. suppression is rule 1 (the repetition controls act before it, as in greedy mode); ``lp_i`` is rule 2's
    log-softmax over the remaining ids;
S2. the filter is the sampler's steps 3-6a (``ops/sampling.py``'s ``keep``) with a minimum keep count: ``x_i =
    fl32(l_i / T)``; top-h keeps at least its ``min_keep`` first entries; top-k keeps the ``k' = max(k, min_keep)``
    largest values (``k > 0``); top-p keeps i iff the weight of the kept values strictly larger than ``x_i`` is ``<=
    p Z``, and always the ``min_keep`` largest values; min-p, typical, epsilon and eta each keep ``min_keep`` ids as
    well; tied values are kept or dropped together, except at top-h's cut (HuggingFace's warpers on ``lp / T`` with
    ``min_tokens_to_keep = min_keep``; HuggingFace's top-h has no keep count, and without one a step could offer
    fewer than M candidates);
S3. a kept id's candidate score is ``c = s_j + lp_i / T`` (the running sums are sums of warped log-probabilities);
    every other id is at -inf;
S4. the draw is an ordered sample without replacement of M candidates from the item's finite ``(j, i)`` with
    probability proportional to ``exp(c)`` (HuggingFace's ``multinomial(softmax(c), M)`` over the flattened K·V
    scores), by Gumbel-top-M: candidate ``(j, i)`` has the key ``g = c + G``, ``G = -log(-log u)``, ``u = ((w >> 8)
    + 0.5) 2^-24`` with ``w`` word ``i & 3`` of Philox4x32-10 at counter ``(i >> 2, j, step, 0)`` and key ``(seed
    mod 2^32, seed >> 32)`` of the item's seed; sorted by descending g, a tie to the lower flat index ``j·V + i``, the
    sample is the first M (all finite ones if there are fewer). A row's own M best keys decide the sample, which is
    what makes a bounded per-row selection exact, as in rule 5;
S5. a candidate finishes if its token is a stop id or the step is the last (``max_new - 1``). The first K draws that
    finish are offered in draw order: a stop id as in rule 6 (``c / L ** a``, L - 1 tokens, source beam j), otherwise
    with ``L = max_new`` and ``max_new`` tokens, its token recorded as the last step's history slot d (its draw index)
    with parent j. The new beams are the K largest-c (not g) drawn candidates that do not finish, in descending c,
    ties to the earlier draw; missing beams are dead. The last step has none, so the item is done.

Rules 6 and 7 are unchanged; the done rule stays exact because ``lp / T <= 0``. Item b's seed is ``seed + b`` for an
int ``seed`` or ``seeds[b]``; its result depends on its prompt, its seed and the scalars only.

Diverse (group) beam search (``GroupBeamReference``, Vijayakumar et al. 2016; HuggingFace 4.x's
``_group_beam_search`` with ``HammingDiversityLogitsProcessor``) splits an item's K beams into G = ``num_beam_groups``
groups of ``K_g = K / G``: group g owns beams ``g·K_g .. (g+1)·K_g - 1`` (rows ``b·K + j``), and each group's first
beam starts at 0, the others at -inf. With ``λ = fl32(diversity_penalty)``, per step the groups of an item that is not
done are processed in order g = 0 .. G-1, skipping done groups:

G1. rules 1 and 2 are unchanged (the repetition controls act before them);
G2. ``n_i`` is the number of this step's new beams of groups 0..g-1 of the item whose token is i (stop candidates,
    dead beams and groups done before this step count for nothing; a group that becomes done this step counts); a
    candidate scores ``c = s_j + lp_i - λ·n_i``, so the running sums and the finished scores include the penalty;
G3. rules 3-5 within the group, with K_g for K: its candidates only are ranked, its first K_g non-stop candidates
    become its beams in rank order, and a stop candidate ranked before the K_g-th non-stop one is offered to the
    group's finished set;
G4. rule 6 per (item, group): each set holds at most K_g hypotheses;
G5. rule 7 per group: a group is done when its set is full and its best live beam cannot beat its worst hypothesis
    (exact, because λ >= 0 only lowers sums); a done group's beams are dead; an item is done when all its groups are;
    rule 8 applies per group at ``max_new``;
G6. an item's hypotheses are the union of its groups' sets by descending normalised score, a tie to the lower group,
    then to the group's own order (``merge_finished_sets``).

G = 1 is the beam search above. Group 0 evolves exactly as a beam search of K_g beams on its rows. Per row the
best ``K + n_stop`` unpenalised candidates still decide the selection: at most ``g·K_g <= K - K_g`` tokens are
penalised, so a candidate past them ranks below at least ``K_g + n_stop`` of its row's candidates. Deliberate
differences from HuggingFace 4.x: the repetition controls act before the log-softmax, the done rule is the exact one,
and done groups add no pad tokens to the Hamming counts.

Stochastic beam search (``StochasticBeamReference``; Kool, van Hoof and Welling, ICML 2019, "Stochastic Beams and
Where to Find Them") draws K distinct replies without replacement from the law ``generate`` samples from. Per item b
there are K slots; a live slot j carries φ_j, the log-probability of its prefix, and G_j, its perturbed key. The item
also keeps a finished set of at most K entries ``(key, φ, n, src)`` and a threshold κ_b, which starts at -inf. At the
start slot 0 is live with φ = 0 and G_0 = the Gumbel (rule S4's transform) of word 0 of Philox4x32-10 at counter
``(0, 0, 0, 2)`` under the item's key; the other slots are dead. At step t (L = t + 1), for every live slot j:

R1. suppression below ``min_new`` is rule 1; the repetition controls and sequence bias act on the logits before it,
    as in ``generate``;
R2. ``x_i = fl32(l_i / T)``; the kept set is the sampler's (``ops/sampling.py`` steps 3a-6a: top-h, top-k, top-p,
    min-p, typical, epsilon, eta) with min_keep 1: ``keep(x, top_k, top_p, 1, ...)``, the filter ``generate`` draws
    from;
R3. for a kept i, ``lp'_i = (x_i - m) - log sum_kept exp(x_k - m)`` with m the largest kept x, and the child's
    log-probability is ``φ_ji = φ_j + lp'_i``: the per-step law is ``generate``'s, renormalised over the kept ids (beam
    sampling's ``s + lp / T`` is not renormalised; this rule differs on purpose);
R4. ``Gφ_ji = φ_ji + Gumbel(w)``, w word ``i & 3`` of Philox at counter ``(i >> 2, j, t, 1)`` (the last counter word
    separates this stream from beam sampling's);
R5. ``Z_j`` = the largest Gφ_ji over the kept i; the child's key is its Gumbel truncated at G_j:
    ``G̃_ji = G_j - max(v, 0) - log1p(exp(-|v|))`` with ``v = G_j - Gφ_ji + log1mexp(Gφ_ji - Z_j)``,
    ``log1mexp(a) = log(-expm1(a))`` for ``a > -ln 2`` and ``log1p(-exp(a))`` otherwise. ``log1mexp(0) = -inf``, so
    the row's best child keeps G_j exactly; in exact arithmetic ``G̃ = -log(exp(-G_j) - exp(-Z_j) + exp(-Gφ))``;
R6. each row offers its K + 1 best children by Gφ, a tie to the lower id; G̃ is monotone in Gφ within a row, so no
    child it does not offer could survive or be entry K + 1 of rule R7;
R7. the item's pool is its finished set and every row's offered children, ranked by descending key; on a tie a
    finished entry goes first, finished entries keep their set order and children go by the lower flat index
    ``j·V + i``. The first K survive, in rank order: a surviving child whose token is a stop id enters the finished
    set with ``n = L - 1`` tokens, φ including the stop token's lp' and ``src = j``; at ``t = max_new - 1`` every
    other surviving child takes history slot k in rank order, as a new beam would, and enters the set with ``n =
    max_new`` and ``src = k``; otherwise the other survivors become the new live beams in rank order (beam 0 the
    best). ``κ_b = max(κ_b, key of pool entry K + 1)`` when it exists: by R6 this is the largest key ever pruned, since
    a pruned node's largest descendant key is its own;
R8. the item is done when it has no live beam. Its results are its finished set, best (largest key) first.

Properties (``tests/test_stochastic_beam_cpu.py`` checks them):

P1. an item's first result is distributed exactly as the reply ``generate`` draws with the same temperature, top_k,
    top_p, truncation filters, stop / suppress / min_new, repetition settings, sequence bias and bad words and
    ``max_new_tokens`` (the same law, another random stream);
P2. its results are ``min(K, |support|)`` distinct sequences, a Gumbel-top-K sample without replacement from that law;
P3. κ = -inf if and only if the support holds at most K sequences;
P4. ``sum over results of f · exp(φ) / q``, ``q = -expm1(-exp(φ - κ))``, is unbiased for E[f] (priority sampling;
    Kool et al. §4); with κ = -inf, q = 1 and the sum is exact (``sbs_estimate``).

An item's result depends on its prompt, its seed and the scalars only.

``best_hypotheses(..., num_return_sequences=r)`` returns each item's first r finished hypotheses, best first, as rows
``b · r + q`` (HuggingFace's flattening); rows past an item's count have no tokens, ``n_new`` 0 and score -inf.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

from .sampling import check_filter_args, keep


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
        offer_finished(self.fin[b], self.K, score, n, src)

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
        V = self.vocab
        rows = [(c, j * V + i) for j in range(self.K) for c, i in self.row_best(b, j, logits, step)]
        rows.sort(key=lambda t: (-t[0], t[1]))
        return [(c, f // V, f % V) for c, f in rows]

    def row_best(self, b: int, j: int, logits: np.ndarray, step: int) -> List[Tuple[float, int]]:
        """Beam row j of item b: its best ``K + n_stop`` finite candidates ``(c, i)``, best first, ties to the lower
        id."""
        keep = self.K + len(self.stop)
        c = self.candidates(logits[b * self.K + j], self.scores[b, j], step)
        ids = np.flatnonzero(c > -np.inf)
        if ids.size > keep:                                      # every id tied with the keep-th best stays in
            ids = ids[c[ids] >= np.partition(c[ids], ids.size - keep)[ids.size - keep]]
        ids = ids[np.lexsort((ids, -c[ids]))][:keep]
        return [(float(c[i]), int(i)) for i in ids]

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

    def result(self, num_return_sequences: int = 1) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """``(tokens, n_new, scores)``: int64 [B·r, max_new] padded with -1, int64 [B·r], fp32 [B·r] of each item's r
        best hypotheses (no tokens and -inf past an item's count)."""
        return best_hypotheses(self.fin, self.hist_tok, self.hist_back, self.max_new, num_return_sequences)


def offer_finished(fin: List[Tuple[float, int, int]], cap: int, score: float, n: int, src: int, *extra) -> None:
    """Rule 6 on one finished set ``fin`` (best first) of at most ``cap`` hypotheses: ``(score, n, src, *extra)`` goes
    in after every entry with a score >= its own, unless the set is full and it does not beat the worst."""
    if len(fin) == cap and not score > fin[-1][0]:
        return
    p = len(fin)
    while p > 0 and fin[p - 1][0] < score:
        p -= 1
    fin.insert(p, (score, n, src) + extra)
    del fin[cap:]


def merge_finished_sets(sets: Sequence[Sequence[Tuple[float, int, int]]]) -> List[Tuple[float, int, int]]:
    """Rule G6: one item's finished hypotheses from its groups' sets (each best first, in group order) as one
    best-first list; a tie goes to the lower group, then to the group's own order. One set is returned as it is."""
    return sorted((h for fin in sets for h in fin), key=lambda h: -h[0])


class GroupBeamReference(BeamReference):
    """Diverse (group) beam search (rules G1-G6, see the module docstring) for ``batch`` items in fp64, with the
    interface of ``BeamReference``. ``fin[b][g]`` is group g's finished set, ``group_done`` [B, G] the groups' done
    flags (rule 7 per group) and ``result`` merges the sets (``merge_finished_sets``). ``early_stop=False`` keeps a
    done group selecting, its beams still counting for nothing in the Hamming counts: the results must not change."""

    def __init__(self, batch: int, num_beams: int, max_new: int, vocab: int, length_penalty: float = 1.0,
                 stop_ids: Sequence[int] = (), suppress_ids: Sequence[int] = (), min_new: int = 0,
                 early_stop: bool = True, num_beam_groups: int = 1, diversity_penalty: float = 0.0):
        super().__init__(batch, num_beams, max_new, vocab, length_penalty, stop_ids, suppress_ids, min_new,
                         early_stop)
        G, lam = int(num_beam_groups), float(diversity_penalty)
        if not 1 <= G <= self.K or self.K % G != 0 or not (np.isfinite(lam) and lam >= 0):
            raise ValueError(f"GroupBeamReference: need num_beam_groups dividing num_beams = {self.K} and a finite "
                             f"diversity_penalty >= 0, got {num_beam_groups}, {diversity_penalty}")
        self.G, self.Kg, self.lam = G, self.K // G, float(np.float32(lam))
        self.scores[:, ::self.Kg] = 0.0
        self.fin = [[[] for _ in range(G)] for _ in range(self.B)]
        self.group_done = np.zeros((self.B, G), dtype=bool)
        self.stopped = np.zeros((self.B, G), dtype=bool)   # the group selects no more (group_done with early_stop)

    def group_ranking(self, b: int, g: int, logits: np.ndarray, step: int,
                      taken: Sequence[int]) -> List[Tuple[float, int, int]]:
        """Group g of item b's candidates ``(c, j, i)`` in rank order (rule G2), ``taken``: the tokens of this step's
        counted new beams of the earlier groups."""
        V = self.vocab
        rows = []
        for j in range(g * self.Kg, (g + 1) * self.Kg):
            for c, i in self.row_best(b, j, logits, step):
                n = sum(t == i for t in taken)
                rows.append((c - self.lam * n if n else c, j * V + i))
        rows.sort(key=lambda t: (-t[0], t[1]))
        return [(c, f // V, f % V) for c, f in rows]

    def step(self, logits) -> Tuple[torch.Tensor, torch.Tensor]:
        """One step (rules G1-G5) for every item that is not done."""
        if isinstance(logits, torch.Tensor):
            logits = logits.detach().float().cpu().numpy()
        B, K, Kg = self.B, self.K, self.Kg
        step = self.n_steps
        if step >= self.max_new:
            raise ValueError(f"GroupBeamReference: all {self.max_new} steps taken")
        nxt = np.zeros(B * K, dtype=np.int64)
        parent = np.arange(B * K, dtype=np.int64)
        L, last = step + 1, step == self.max_new - 1
        for b in range(B):
            if self.done[b]:
                continue
            taken: List[int] = []
            for g in range(self.G):
                if self.stopped[b, g]:
                    continue
                j0, fin, counted = g * Kg, self.fin[b][g], not self.group_done[b, g]
                beams = []
                for c, j, i in self.group_ranking(b, g, logits, step, taken):
                    if len(beams) == Kg:
                        break
                    if i in self.stop:
                        offer_finished(fin, Kg, c / self.penalty(L), L - 1, j)
                    else:
                        beams.append((c, j, i))
                new = np.full(Kg, -np.inf)
                for k in range(Kg):
                    if k < len(beams):
                        c, j, i = beams[k]
                        new[k], nxt[b * K + j0 + k], parent[b * K + j0 + k] = c, i, b * K + j
                        self.hist_tok[step, b, j0 + k], self.hist_back[step, b, j0 + k] = i, j
                    else:
                        self.hist_tok[step, b, j0 + k], self.hist_back[step, b, j0 + k] = -1, j0 + k
                if last:
                    for k in range(len(beams)):
                        offer_finished(fin, Kg, new[k] / self.penalty(self.max_new), self.max_new, j0 + k)
                    self.group_done[b, g] = self.stopped[b, g] = True
                elif not beams:
                    self.group_done[b, g] = self.stopped[b, g] = True
                elif len(fin) == Kg:
                    reach = new[0] / self.penalty(self.max_new if self.alpha > 0 else L + 1)
                    self.group_done[b, g] |= not reach > fin[-1][0]
                    self.stopped[b, g] |= self.early_stop and self.group_done[b, g]
                if counted:                                      # this step's new beams count, even if now done
                    taken.extend(i for _, _, i in beams)
                self.scores[b, j0:j0 + Kg] = -np.inf if self.stopped[b, g] else new
            self.done[b] = bool(self.stopped[b].all())
        self.n_steps += 1
        return torch.from_numpy(nxt), torch.from_numpy(parent)

    def result(self, num_return_sequences: int = 1) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """``BeamReference.result`` of the merged finished sets (rule G6)."""
        return best_hypotheses([merge_finished_sets(f) for f in self.fin], self.hist_tok, self.hist_back,
                               self.max_new, num_return_sequences)


_MASK = np.uint64(0xFFFFFFFF)


def philox_words(c0: np.ndarray, c1: int, c2: int, c3: int, seed: int) -> np.ndarray:
    """Philox4x32-10 (``ops.sampling.philox4x32_10``) for the counters ``(c0[t], c1, c2, c3)`` and the key ``(seed mod
    2^32, seed >> 32)``, vectorised: uint64 [len(c0), 4], the four output words of each counter."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    n = len(c0)
    c = [np.asarray(c0, dtype=np.uint64) & _MASK] + [np.full(n, int(v) & 0xFFFFFFFF, dtype=np.uint64)
                                                     for v in (c1, c2, c3)]
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    w0, w1, s32 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85), np.uint64(32)
    for _ in range(10):
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> s32) ^ c[1] ^ k0, p1 & _MASK, (p0 >> s32) ^ c[3] ^ k1, p0 & _MASK]
        k0, k1 = (k0 + w0) & _MASK, (k1 + w1) & _MASK
    return np.stack(c, axis=1)


def gumbel(w: np.ndarray) -> np.ndarray:
    """``G = -log(-log u)`` in fp64 for ``u = ((w >> 8) + 0.5) 2^-24`` (rule S4)."""
    u = ((np.asarray(w, dtype=np.uint64) >> np.uint64(8)).astype(np.float64) + 0.5) * 2.0 ** -24
    return -np.log(-np.log(u))


def sample_keep(x: np.ndarray, top_k: int, top_p: float, min_keep: int) -> np.ndarray:
    """Rule S2's top-k / top-p on the fp32 values ``x = fl32(l / T)`` (-inf: removed): the bool mask of the kept ids,
    ``ops.sampling.keep`` with the truncation filters off."""
    return keep(x, top_k, top_p, min_keep)[0]


class BeamSampleReference(BeamReference):
    """Beam sampling (rules S1-S5 with 6 and 7, see the module docstring) for ``batch`` items in fp64, with the
    interface of ``BeamReference``. ``seeds``: one int per item (its Philox key). ``temperature > 0``, ``top_p`` and
    the truncation filters (``min_p``, ``typical_p``, ``epsilon_cutoff``, ``eta_cutoff``, ``top_h``; off at 0, 1, 0,
    0 and 0) are rounded to fp32, as the kernel takes them; ``top_k = 0`` is off."""

    def __init__(self, batch: int, num_beams: int, max_new: int, vocab: int, length_penalty: float = 1.0,
                 stop_ids: Sequence[int] = (), suppress_ids: Sequence[int] = (), min_new: int = 0,
                 early_stop: bool = True, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0,
                 seeds: Sequence[int] = (), min_p: float = 0.0, typical_p: float = 1.0, epsilon_cutoff: float = 0.0,
                 eta_cutoff: float = 0.0, top_h: float = 0.0):
        super().__init__(batch, num_beams, max_new, vocab, length_penalty, stop_ids, suppress_ids, min_new,
                         early_stop)
        if not temperature > 0 or int(top_k) < 0 or not 0 < top_p <= 1:
            raise ValueError(f"BeamSampleReference: need temperature > 0, top_k >= 0 and 0 < top_p <= 1, got "
                             f"{temperature}, {top_k}, {top_p}")
        check_filter_args("BeamSampleReference", min_p, typical_p, epsilon_cutoff, eta_cutoff, top_h)
        self.filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff,
                            top_h=top_h)
        self.seeds = [int(x) for x in seeds]
        if len(self.seeds) != self.B:
            raise ValueError(f"BeamSampleReference: need {self.B} seeds, got {len(self.seeds)}")
        self.T = float(np.float32(temperature))
        self.top_k, self.top_p = int(top_k), float(top_p)
        self.min_keep = max(2, 1 + len(self.stop))
        self.M = self.min_keep * self.K

    def row_candidates(self, b: int, j: int, logits_row: np.ndarray, step: int):
        """Rules S1-S4 for beam row j of item b: ``(ids, c, g)`` of its kept ids (fp64), in id order."""
        s = self.scores[b, j]
        x = np.array(logits_row[:self.vocab], dtype=np.float32)
        if step < self.min_new and self.suppress.size:
            x[self.suppress] = -np.inf
        fin = x > -np.inf
        if not np.isfinite(s) or not fin.any():
            return np.zeros(0, dtype=np.int64), np.zeros(0), np.zeros(0)
        xd = x.astype(np.float64)
        m = xd[fin].max()
        lp = (xd - m) - np.log(np.exp(xd[fin] - m).sum())
        ids = np.flatnonzero(keep((x / np.float32(self.T)).astype(np.float32), self.top_k, self.top_p,
                                  self.min_keep, **self.filters)[0])
        c = s + lp[ids] / self.T
        w = philox_words(ids >> 2, j, step, 0, self.seeds[b])[np.arange(ids.size), ids & 3]
        return ids, c, c + gumbel(w)

    def draws(self, b: int, logits: np.ndarray, step: int) -> List[Tuple[float, float, int, int]]:
        """Item b's sample (rule S4): ``(g, c, j, i)`` in draw order, at most M."""
        V = self.vocab
        g, c, flat = [], [], []
        for j in range(self.K):
            ids, cj, gj = self.row_candidates(b, j, logits[b * self.K + j], step)
            g.append(gj)
            c.append(cj)
            flat.append(j * V + ids)
        g, c, flat = np.concatenate(g), np.concatenate(c), np.concatenate(flat)
        order = np.lexsort((flat, -g))[:self.M]
        return [(float(g[o]), float(c[o]), int(flat[o]) // V, int(flat[o]) % V) for o in order]

    def step(self, logits) -> Tuple[torch.Tensor, torch.Tensor]:
        """One step (rules S1-S5, 6 and 7) for every item that is not done."""
        if isinstance(logits, torch.Tensor):
            logits = logits.detach().float().cpu().numpy()
        B, K = self.B, self.K
        step = self.n_steps
        if step >= self.max_new:
            raise ValueError(f"BeamSampleReference: all {self.max_new} steps taken")
        nxt = np.zeros(B * K, dtype=np.int64)
        parent = np.arange(B * K, dtype=np.int64)
        L, last = step + 1, step == self.max_new - 1
        for b in range(B):
            if self.done[b]:
                continue
            sample = self.draws(b, logits, step)
            finishes = [last or i in self.stop for _, _, _, i in sample]
            for d, (_, c, j, i) in enumerate(sample[:K]):
                if i in self.stop:
                    self.offer(b, c / self.penalty(L), L - 1, j)
                elif last:
                    self.offer(b, c / self.penalty(self.max_new), self.max_new, d)
            live = sorted((d for d in range(len(sample)) if not finishes[d]), key=lambda d: (-sample[d][1], d))[:K]
            new = np.full(K, -np.inf)
            for k in range(K):
                e = k if last else (live[k] if k < len(live) else -1)
                if 0 <= e < len(sample):
                    _, c, j, i = sample[e]
                    self.hist_tok[step, b, k], self.hist_back[step, b, k] = i, j
                    if not last:
                        new[k], nxt[b * K + k], parent[b * K + k] = c, i, b * K + j
                else:
                    self.hist_tok[step, b, k], self.hist_back[step, b, k] = -1, k
            self.scores[b] = new
            if last or not live:
                self.done[b] = True
            elif self.early_stop and len(self.fin[b]) == K:
                reach = new[0] / self.penalty(self.max_new if self.alpha > 0 else L + 1)
                self.done[b] = not reach > self.fin[b][-1][0]
        self.n_steps += 1
        return torch.from_numpy(nxt), torch.from_numpy(parent)


def best_hypotheses(fin, hist_tok, hist_back, max_new: int,
                    num_return_sequences: int = 1) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Each item's first ``num_return_sequences`` = r finished hypotheses, their tokens followed back through the
    parent pointers, as rows ``b * r + q``. ``fin``: per item a best-first list of ``(normalised score, n, source
    beam)``; ``hist_tok`` / ``hist_back`` [max_new, B, K]. Rows past an item's count: tokens -1, 0 and -inf."""
    B, R = len(fin), int(num_return_sequences)
    tokens = torch.full((B * R, max_new), -1, dtype=torch.int64)
    n_new = torch.zeros(B * R, dtype=torch.int64)
    scores = torch.full((B * R,), float("-inf"), dtype=torch.float32)
    for b in range(B):
        for q, (score, n, src) in enumerate(fin[b][:R]):
            row, r = b * R + q, int(src)
            for u in range(int(n) - 1, -1, -1):
                tokens[row, u] = int(hist_tok[u, b, r])
                r = int(hist_back[u, b, r])
            n_new[row], scores[row] = int(n), float(score)
    return tokens, n_new, scores


def start_keys(seeds: Sequence[int]) -> np.ndarray:
    """Rule R1's start: each item's G_0, the Gumbel of word 0 of Philox at counter ``(0, 0, 0, 2)``, in fp64."""
    return np.array([gumbel(philox_words(np.zeros(1, dtype=np.int64), 0, 0, 2, s)[0, 0]) for s in seeds])


def truncated_gumbel(G: float, gphi: np.ndarray, Z: float) -> np.ndarray:
    """Rule R5 in fp64: the keys of children with perturbed log-probabilities ``gphi`` (their largest ``Z``) of a beam
    with key ``G``."""
    a = np.asarray(gphi, dtype=np.float64) - Z
    with np.errstate(divide="ignore", invalid="ignore"):
        l1m = np.where(a > -np.log(2.0), np.log(-np.expm1(a)), np.log1p(-np.exp(a)))
    v = G - gphi + l1m
    return G - np.maximum(v, 0.0) - np.log1p(np.exp(-np.abs(v)))


class StochasticBeamReference(BeamReference):
    """Stochastic beam search (rules R1-R8, see the module docstring) for ``batch`` items in fp64, with the interface of
    ``BeamReference``. ``scores`` [B, K] are the live beams' φ, ``keys`` [B, K] their keys G, ``fin[b]`` item b's
    finished set as ``(key, n, src, φ)``, best first, and ``kappa`` [B] the thresholds. ``seeds``: one int per item;
    ``temperature > 0``, ``top_p`` and the truncation filters are rounded to fp32, as the kernels take them;
    ``top_k = 0`` is off."""

    def __init__(self, batch: int, num_beams: int, max_new: int, vocab: int, stop_ids: Sequence[int] = (),
                 suppress_ids: Sequence[int] = (), min_new: int = 0, temperature: float = 1.0, top_k: int = 0,
                 top_p: float = 1.0, seeds: Sequence[int] = (), min_p: float = 0.0, typical_p: float = 1.0,
                 epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0, top_h: float = 0.0):
        super().__init__(batch, num_beams, max_new, vocab, 1.0, stop_ids, suppress_ids, min_new)
        if not temperature > 0 or int(top_k) < 0 or not 0 < top_p <= 1:
            raise ValueError(f"StochasticBeamReference: need temperature > 0, top_k >= 0 and 0 < top_p <= 1, got "
                             f"{temperature}, {top_k}, {top_p}")
        check_filter_args("StochasticBeamReference", min_p, typical_p, epsilon_cutoff, eta_cutoff, top_h)
        self.filters = dict(min_p=min_p, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff, eta_cutoff=eta_cutoff,
                            top_h=top_h)
        self.seeds = [int(x) for x in seeds]
        if len(self.seeds) != self.B:
            raise ValueError(f"StochasticBeamReference: need {self.B} seeds, got {len(self.seeds)}")
        self.T = float(np.float32(temperature))
        self.top_k, self.top_p = int(top_k), float(top_p)
        self.keys = np.full((self.B, self.K), -np.inf)
        self.keys[:, 0] = start_keys(self.seeds)
        self.kappa = np.full(self.B, -np.inf)

    def children(self, b: int, j: int, logits_row: np.ndarray, step: int):
        """Rules R1-R6 for beam row j of item b: ``(ids, phi, gphi, key)`` of the children it offers, by descending
        Gφ (a tie to the lower id); empty for a dead beam."""
        empty = np.zeros(0, dtype=np.int64), np.zeros(0), np.zeros(0), np.zeros(0)
        x = (np.array(logits_row[:self.vocab], dtype=np.float32) / np.float32(self.T)).astype(np.float32)
        if step < self.min_new and self.suppress.size:
            x[self.suppress] = -np.inf
        if not np.isfinite(self.scores[b, j]) or not (x > -np.inf).any():
            return empty
        ids = np.flatnonzero(keep(x, self.top_k, self.top_p, 1, **self.filters)[0])
        xd = x[ids].astype(np.float64)
        m = xd.max()
        phi = self.scores[b, j] + ((xd - m) - np.log(np.exp(xd - m).sum()))
        w = philox_words(ids >> 2, j, step, 1, self.seeds[b])[np.arange(ids.size), ids & 3]
        gphi = phi + gumbel(w)
        order = np.lexsort((ids, -gphi))[:self.K + 1]
        return ids[order], phi[order], gphi[order], truncated_gumbel(self.keys[b, j], gphi[order], gphi.max())

    def step(self, logits) -> Tuple[torch.Tensor, torch.Tensor]:
        """One step (rules R1-R8) for every item that is not done."""
        if isinstance(logits, torch.Tensor):
            logits = logits.detach().float().cpu().numpy()
        B, K, V = self.B, self.K, self.vocab
        step = self.n_steps
        if step >= self.max_new:
            raise ValueError(f"StochasticBeamReference: all {self.max_new} steps taken")
        nxt = np.zeros(B * K, dtype=np.int64)
        parent = np.arange(B * K, dtype=np.int64)
        L, last = step + 1, step == self.max_new - 1
        for b in range(B):
            if self.done[b]:
                continue
            # pool entries (key, tie order, payload): finished entries first on a tie, then children by flat index
            pool = [(f[0], q, f) for q, f in enumerate(self.fin[b])]
            for j in range(K):
                ids, phi, _, key = self.children(b, j, logits[b * K + j], step)
                pool += [(float(key[e]), K + j * V + int(ids[e]), (j, int(ids[e]), float(phi[e])))
                         for e in range(ids.size)]
            pool.sort(key=lambda t: (-t[0], t[1]))
            if len(pool) > K:
                self.kappa[b] = max(self.kappa[b], pool[K][0])
            fin, beams = [], []
            for key, order, payload in pool[:K]:
                if order < K:
                    offer_finished(fin, K, *payload)
                    continue
                j, i, phi = payload
                if i in self.stop:
                    offer_finished(fin, K, key, L - 1, j, phi)
                    continue
                if last:
                    offer_finished(fin, K, key, self.max_new, len(beams), phi)
                beams.append((key, j, i, phi))
            self.fin[b] = fin
            self.scores[b], self.keys[b] = -np.inf, -np.inf
            for k in range(K):
                if k < len(beams):
                    key, j, i, phi = beams[k]
                    self.hist_tok[step, b, k], self.hist_back[step, b, k] = i, j
                    if not last:
                        self.scores[b, k], self.keys[b, k] = phi, key
                        nxt[b * K + k], parent[b * K + k] = i, b * K + j
                else:
                    self.hist_tok[step, b, k], self.hist_back[step, b, k] = -1, k
            self.done[b] = last or not beams
        self.n_steps += 1
        return torch.from_numpy(nxt), torch.from_numpy(parent)

    def result(self):
        """``stochastic_results`` of the finished sets: ``(tokens, n_new, log_probs, keys, kappa)``."""
        return stochastic_results(self.fin, self.hist_tok, self.hist_back, self.max_new, self.K, self.kappa)


def stochastic_results(fin, hist_tok, hist_back, max_new: int, K: int, kappa):
    """Each item's finished set ``(key, n, src, φ)`` (best first) as ``(tokens, n_new, log_probs, keys, kappa)``: rows
    ``b·K + q`` of int64 [B·K, max_new] padded with -1, int64 [B·K], fp32 [B·K] twice (rows past an item's count: no
    tokens, 0 and -inf), and fp32 [B]."""
    tokens, n_new, keys = best_hypotheses([[f[:3] for f in fb] for fb in fin], hist_tok, hist_back, max_new, K)
    _, _, log_probs = best_hypotheses([[(f[3], f[1], f[2]) for f in fb] for fb in fin], hist_tok, hist_back, max_new,
                                      K)
    return tokens, n_new, log_probs, keys, torch.as_tensor(np.asarray(kappa, dtype=np.float32))


def sbs_estimate(values: torch.Tensor, log_probs: torch.Tensor, kappa: torch.Tensor) -> torch.Tensor:
    """Property P4: per item, ``sum_q f_q · exp(φ_q) / q_q`` with ``q = -expm1(-exp(φ - κ))``, an unbiased estimate of
    E[f] under the reply law (exact when κ = -inf). ``values`` and ``log_probs`` are [B·K] (or [B, K]) in the row order
    of ``stochastic_beam_search``, ``kappa`` [B]; rows with φ = -inf count for nothing. Returns fp64 [B]."""
    kappa = kappa.double().reshape(-1)
    phi = log_probs.double().reshape(kappa.numel(), -1)
    f = values.double().reshape(phi.shape)
    live = phi > float("-inf")
    q = -torch.expm1(-torch.exp(phi - kappa[:, None]))
    w = torch.where(live, torch.exp(phi) / torch.where(live, q, torch.ones_like(q)), torch.zeros_like(q))
    return (torch.where(live, f, torch.zeros_like(f)) * w).sum(1)
