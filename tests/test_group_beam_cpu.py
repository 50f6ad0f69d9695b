"""Diverse (group) beam search on the CPU: the fp64 definition (``ops.beam.GroupBeamReference``) against plain beam
search, a hand-worked case, the Hamming penalty's effect, its done rule against running every step,
``GPT2DoubleHeads.beam_search(num_beam_groups=...)`` on the tiny model and the argument errors."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.beam import BeamReference, GroupBeamReference, merge_finished_sets  # noqa: E402


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _rows(*probs):
    with np.errstate(divide="ignore"):
        return np.log(np.array(probs, dtype=np.float64)).astype(np.float32)


def _random_steps(rng, B, K, V, n):
    steps = []
    for _ in range(n):
        logits = (rng.standard_normal((B * K, V)) * 2).astype(np.float32)
        logits[rng.random((B * K, V)) < 0.1] = -np.inf
        steps.append(logits)
    return steps


def _setting(rng):
    K = int(rng.choice([2, 4, 6]))
    G = int(rng.choice([g for g in (1, 2, 3, 6) if K % g == 0 and g <= K]))
    V, n = int(rng.integers(4, 14)), int(rng.integers(1, 7))
    stop = [int(x) for x in rng.choice(V, size=int(rng.integers(0, 3)), replace=False)]
    alpha = float(rng.choice([-1.0, 0.0, 0.5, 1.0, 2.0]))
    return dict(num_beams=K, max_new=n, vocab=V, length_penalty=alpha, stop_ids=stop,
                suppress_ids=stop[:1], min_new=int(rng.integers(0, 2))), G


def test_one_group_is_plain_beam_search():
    for trial in range(150):
        rng = np.random.default_rng(trial)
        kw, _ = _setting(rng)
        B = 3
        plain = BeamReference(B, **kw)
        group = GroupBeamReference(B, **kw, num_beam_groups=1)
        for logits in _random_steps(rng, B, kw["num_beams"], kw["vocab"], kw["max_new"]):
            live = ~plain.done.copy()
            a, b = plain.step(logits), group.step(logits)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), trial
            assert (plain.done == group.done).all() and (plain.hist_tok == group.hist_tok).all()
            assert (plain.hist_back == group.hist_back).all(), trial
            for i in range(B):
                assert plain.fin[i] == group.fin[i][0], trial
                if live[i] and not plain.done[i]:     # a done item's (group's) beams are dead in the group search
                    assert np.array_equal(plain.scores[i], group.scores[i]), trial
        for r in (1, kw["num_beams"]):
            assert all(torch.equal(x, y) for x, y in zip(plain.result(r), group.result(r))), trial


def test_group_zero_is_beam_search_with_its_beams():
    """Group 0 sees no penalty: it is BeamReference(K_g) fed the group-0 rows, step after step."""
    for trial in range(150):
        rng = np.random.default_rng(1000 + trial)
        kw, G = _setting(rng)
        if G == 1:
            G = kw["num_beams"]
        B, K = 2, kw["num_beams"]
        Kg = K // G
        group = GroupBeamReference(B, **kw, num_beam_groups=G, diversity_penalty=float(rng.choice([0.3, 2.0])))
        plain = BeamReference(B, **dict(kw, num_beams=Kg))
        rows = np.array([b * K + k for b in range(B) for k in range(Kg)])
        for logits in _random_steps(rng, B, K, kw["vocab"], kw["max_new"]):
            if plain.done.all():
                break
            live = ~plain.done.copy()
            gn, gp = group.step(logits)
            pn, pp = plain.step(logits[rows])
            for b in range(B):
                if not live[b]:
                    continue
                s = slice(b * K, b * K + Kg)
                assert gn[s].tolist() == pn[b * Kg:(b + 1) * Kg].tolist(), trial
                assert (gp[s] - b * K).tolist() == (pp[b * Kg:(b + 1) * Kg] - b * Kg).tolist(), trial
                assert group.fin[b][0] == plain.fin[b], trial
                assert bool(group.group_done[b, 0]) == bool(plain.done[b]), trial
                want = np.full(Kg, -np.inf) if plain.done[b] else plain.scores[b]
                assert np.array_equal(group.scores[b, :Kg], want), trial
                assert (group.hist_tok[group.n_steps - 1, b, :Kg] == plain.hist_tok[plain.n_steps - 1, b]).all()


def test_hand_worked_penalty_flips_group_one():
    # K = 2, G = 2: one beam per group, both starting from the prompt with the same next-token distribution
    row = _rows(0.1, 0.5, 0.3, 0.05, 0.05)
    logits = np.stack([row, row])
    lp = np.log([0.1, 0.5, 0.3, 0.05, 0.05])
    # lambda = 1: group 1's token 1 scores log 0.5 - 1 = -1.693 < log 0.3 = -1.204, so it takes token 2
    ref = GroupBeamReference(1, 2, 4, 5, num_beam_groups=2, diversity_penalty=1.0)
    nxt, parent = ref.step(logits)
    assert nxt.tolist() == [1, 2] and parent.tolist() == [0, 1]
    assert ref.scores[0].tolist() == pytest.approx([np.log(0.5), np.log(0.3)], abs=1e-6)
    # lambda = 0.2: -0.893 > -1.204, so group 1 takes token 1 too, with the penalty in its running sum
    ref = GroupBeamReference(1, 2, 4, 5, num_beam_groups=2, diversity_penalty=0.2)
    nxt, parent = ref.step(logits)
    assert nxt.tolist() == [1, 1] and parent.tolist() == [0, 1]
    assert ref.scores[0].tolist() == pytest.approx([lp[1], lp[1] - np.float32(0.2)], abs=1e-6)
    # a stop candidate pays the penalty too, and goes to its group's own finished set
    ref = GroupBeamReference(1, 2, 4, 5, stop_ids=[1], num_beam_groups=2, diversity_penalty=0.2)
    nxt, _ = ref.step(np.stack([_rows(0.1, 0.2, 0.6, 0.05, 0.05), _rows(0.1, 0.6, 0.2, 0.05, 0.05)]))
    # group 0: token 2 (0.6), token 1 (0.2, stop) ranks after it: not offered. Group 1: token 1 (stop, 0.6) first, then
    # token 2 at log 0.2 - 0.2 = -1.809 against token 0 at log 0.1 = -2.303, so token 2
    assert nxt.tolist() == [2, 2] and ref.fin[0][0] == [] and len(ref.fin[0][1]) == 1
    assert ref.fin[0][1][0][0] == pytest.approx(np.log(0.6), abs=1e-6) and ref.fin[0][1][0][1:] == (0, 1)
    assert ref.scores[0, 1] == pytest.approx(np.log(0.2) - np.float32(0.2), abs=1e-6)


def test_large_penalty_makes_the_groups_tokens_distinct():
    checked = 0
    for trial in range(60):
        rng = np.random.default_rng(2000 + trial)
        B, K, G, V, n = 2, 8, int(rng.choice([2, 4, 8])), 40, 6
        Kg = K // G
        ref = GroupBeamReference(B, K, n, V, num_beam_groups=G, diversity_penalty=1e6)
        for logits in _random_steps(rng, B, K, V, n):
            if ref.done.all():
                break
            was_done = ref.group_done.copy()
            ref.step(logits)
            t = ref.n_steps - 1
            for b in range(B):
                toks = [ref.hist_tok[t, b, g * Kg:(g + 1) * Kg] for g in range(G) if not was_done[b, g]]
                toks = [x[x >= 0] for x in toks]
                # with at least V - K finite ids per row left, every group found unpenalised candidates
                for g1 in range(len(toks)):
                    for g2 in range(g1):
                        assert not set(toks[g1].tolist()) & set(toks[g2].tolist()), (trial, t, b)
                        checked += 1
    assert checked > 0


def test_done_rule_is_exact():
    """Stopping a group early never changes any result: the same random logits with the done rule on and off."""
    stopped = 0
    for trial in range(300):
        runs = []
        for early in (True, False):
            rng = np.random.default_rng(3000 + trial)
            kw, G = _setting(rng)
            ref = GroupBeamReference(3, **kw, early_stop=early, num_beam_groups=G, diversity_penalty=0.7)
            for logits in _random_steps(rng, 3, kw["num_beams"], kw["vocab"], kw["max_new"]):
                ref.step(logits)
            runs.append(ref)
        K = runs[0].K
        for r in (1, K):
            assert all(torch.equal(a, b) for a, b in zip(runs[0].result(r), runs[1].result(r))), trial
        stopped += int(runs[0].group_done.sum())
    assert stopped > 0


def test_merge_order():
    sets = [[(-1.0, 3, 0), (-2.0, 2, 1)], [(-1.0, 4, 2), (-1.5, 1, 3)], []]
    assert merge_finished_sets(sets) == [(-1.0, 3, 0), (-1.0, 4, 2), (-1.5, 1, 3), (-2.0, 2, 1)]
    assert merge_finished_sets(sets[:1]) == sets[0]


def test_beam_search_groups_on_the_tiny_model(tiny):
    g = torch.Generator().manual_seed(7)
    V = tiny.cfg.vocab_size
    lengths = [6, 30, 17]
    ids = torch.randint(0, V, (3, 30), generator=g)
    tt = torch.randint(V - 5, V - 3, (3, 30), generator=g)
    kw = dict(num_beams=4, max_new_tokens=10, length_penalty=0.7, stop_ids=[int(ids[0, 0]), 77])
    # one group: the call without the new arguments
    want = tiny.beam_search(ids, lengths, tt, **kw, num_return_sequences=4)
    got = tiny.beam_search(ids, lengths, tt, **kw, num_return_sequences=4, num_beam_groups=1, diversity_penalty=0.0)
    assert all(torch.equal(a, b) for a, b in zip(want, got))
    div = dict(kw, num_beam_groups=2, diversity_penalty=1.5)
    tokens, n_new, scores = tiny.beam_search(ids, lengths, tt, **div, num_return_sequences=4)
    again = tiny.beam_search(ids, lengths, tt, **div, num_return_sequences=4)
    assert all(torch.equal(a, b) for a, b in zip((tokens, n_new, scores), again))
    assert not all(torch.equal(a, b) for a, b in zip(want, (tokens, n_new, scores)))
    for b, n in enumerate(lengths):
        alone = tiny.beam_search(ids[b:b + 1, :n], None, tt[b:b + 1, :n], **div, num_return_sequences=4)
        rows = slice(4 * b, 4 * b + 4)
        assert torch.equal(alone[0], tokens[rows]) and torch.equal(alone[1], n_new[rows]), b
        assert alone[2].tolist() == pytest.approx(scores[rows].tolist(), abs=1e-5)
        # the merged sets, best first: both groups' hypotheses, descending
        s = scores[rows]
        assert (s[:-1] >= s[1:]).all() and torch.isfinite(s).all(), b
        for q in range(4):
            k = int(n_new[4 * b + q])
            assert (tokens[4 * b + q, k:] == -1).all() and (tokens[4 * b + q, :k] >= 0).all()
    best = tiny.beam_search(ids, lengths, tt, **div)
    assert torch.equal(best[0], tokens[::4]) and torch.equal(best[2], scores[::4])


def test_beam_search_group_argument_errors(tiny):
    ids = torch.zeros(2, 10, dtype=torch.long)
    bad = [dict(num_beams=4, num_beam_groups=3, diversity_penalty=1.0),
           dict(num_beams=4, num_beam_groups=0),
           dict(num_beams=4, num_beam_groups=8, diversity_penalty=1.0),
           dict(num_beams=4, num_beam_groups=2),
           dict(num_beams=4, num_beam_groups=2, diversity_penalty=-1.0),
           dict(num_beams=4, num_beam_groups=2, diversity_penalty=float("inf")),
           dict(num_beams=4, num_beam_groups=2, diversity_penalty=float("nan")),
           dict(num_beams=4, num_beam_groups=2, diversity_penalty=1.0, do_sample=True),
           dict(num_beams=4, diversity_penalty=0.5)]
    for kw in bad:
        with pytest.raises(ValueError, match="beam_search"):
            tiny.beam_search(ids, **kw)
    from adapcc_b200.ops import BeamState

    for kw in (dict(groups=3), dict(groups=0), dict(groups=2, sample=True)):
        with pytest.raises(ValueError, match="BeamState"):
            BeamState(2, 4, 5, 1.0, "cpu", **kw)
    with pytest.raises(ValueError, match="GroupBeamReference"):
        GroupBeamReference(1, 4, 3, 5, num_beam_groups=3)


def test_beam_step_group_argument_errors():
    from adapcc_b200.ops import BeamState, beam_step_

    logits = torch.zeros(8, 16)
    st = BeamState(2, 4, 5, 1.0, "cpu", groups=2)
    assert st.fin_count.shape == (4,) and st.group_done.shape == (4,)
    assert st.scores.view(2, 4)[:, [0, 2]].eq(0).all() and st.scores.view(2, 4)[:, [1, 3]].eq(float("-inf")).all()
    for lam in (0.0, -0.5, float("inf")):
        with pytest.raises(ValueError, match="diversity_penalty"):
            beam_step_(logits, 16, st, diversity_penalty=lam)
    with pytest.raises(ValueError, match="diversity_penalty"):
        beam_step_(logits, 16, BeamState(2, 4, 5, 1.0, "cpu"), diversity_penalty=0.5)


def test_sample_replies_pass_groups_through(tiny):
    from adapcc_b200.eval import convai

    class Tok:
        special_ids = (507, 508, 509, 510, 511)
        pad_id = 511

        def encode(self, s):
            return [ord(c) % 500 for c in s]

        def decode(self, ids):
            return " ".join(str(i % 7) for i in ids)

    dialogs = [([[1, 2]], [[3, 4, 5]]), ([[6]], [[7], [8, 9]])]
    kw = dict(max_length=6, min_length=2, num_beams=4)
    replies = convai.sample_replies(tiny, Tok(), dialogs, **kw, num_beam_groups=2, diversity_penalty=2.0)
    assert len(replies) == 2 and all(2 <= len(r) <= 6 and not set(r) & set(Tok.special_ids) for r in replies)
    with pytest.raises(ValueError, match="diversity_penalty"):
        convai.sample_replies(tiny, Tok(), dialogs, **kw, num_beam_groups=2)
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    r = convai.evaluate_dialogs(tiny, Tok(), d, "f1", max_length=5, num_beams=2, num_beam_groups=2,
                                diversity_penalty=1.0)
    assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0
