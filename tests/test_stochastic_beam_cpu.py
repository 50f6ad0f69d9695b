"""Stochastic beam search on the CPU: the fp64 definition (``ops.beam.StochasticBeamReference``) on a hand-built
autoregressive logit table and on the tiny GPT-2, against the reply law of ``generate`` enumerated with the filter of
``ops/sampling.py`` (chi-square tests with fixed seeds), the truncated Gumbel, the estimator, the edge cases, the
argument errors and the build of the kernels (nvcc only, no device)."""
import os
import sys
from itertools import product

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.beam import StochasticBeamReference, sbs_estimate, truncated_gumbel  # noqa: E402
from adapcc_b200.ops.sampling import reference_row  # noqa: E402

V, STEPS, STOP = 4, 3, 3


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _table(seed=0, dead=()):
    """Logits [V] of every prefix of fewer than STEPS tokens; ids in ``dead`` at -inf after a prefix of that length."""
    rng = np.random.default_rng(seed)
    table = {}
    for n in range(STEPS):
        for pre in product(range(V), repeat=n):
            row = (rng.standard_normal(V) * 1.2).astype(np.float32)
            for t, i in dead:
                if t == n:
                    row[i] = -np.inf
            table[pre] = row
    return table


def _law(next_logits, n, kw, stop=(STOP,)):
    """Every reply of at most n tokens (the stop token excluded) and its probability under generate's draw:
    ``next_logits(prefix, t)`` gives the logits, the kept ids and weights are those of ops/sampling.py."""
    law, live = {}, {(): 1.0}
    for t in range(n):
        nxt = {}
        for pre, p in live.items():
            r = reference_row(next_logits(pre, t), kw.get("temperature", 1.0), kw.get("top_k", 0),
                              kw.get("top_p", 1.0), 0, 0, t, kw.get("min_new", 0), kw.get("suppress_ids", ()))
            e = np.where(r["kept"], r["e"], 0.0)
            for i in np.flatnonzero(r["kept"]):
                q = p * e[i] / e.sum()
                if int(i) in stop:
                    law[pre] = law.get(pre, 0.0) + q
                else:
                    nxt[pre + (int(i),)] = q
        live = nxt
    law.update(live)
    return law


def _run_table(table, B, K, seeds, **kw):
    ref = StochasticBeamReference(B, K, STEPS, V, stop_ids=[STOP], seeds=seeds, **kw)
    pre = [()] * (B * K)
    for _ in range(STEPS):
        logits = np.stack([table.get(p, np.zeros(V, dtype=np.float32)) for p in pre])
        nxt, parent = ref.step(logits)
        pre = [pre[int(parent[r])] + (int(nxt[r]),) for r in range(B * K)]
        if ref.done.all():
            break
    return ref


def _replies(tokens, n_new, B, K):
    return [[tuple(tokens[b * K + q, :int(n_new[b * K + q])].tolist()) for q in range(K)] for b in range(B)]


def _chi2(samples, law):
    from scipy.stats import chisquare

    N = len(samples)
    counts = {}
    for s in samples:
        counts[s] = counts.get(s, 0) + 1
    assert set(counts) <= set(law), set(counts) - set(law)
    big = [s for s in sorted(law, key=lambda s: -law[s]) if law[s] * N >= 5]
    got = [counts.get(s, 0) for s in big]
    want = [law[s] * N for s in big]
    rest = N - sum(want)
    if rest >= 1e-9 * N:
        got.append(N - sum(got))
        want.append(rest)
    return float(chisquare(got, np.array(want) * (N / sum(want))).pvalue)


def test_truncated_gumbel_identity_and_stable_form():
    rng = np.random.default_rng(0)
    for _ in range(200):
        gphi = rng.standard_normal(int(rng.integers(1, 40))) * 3 - 2
        G = float(rng.standard_normal() * 3)
        key = truncated_gumbel(G, gphi, gphi.max())
        assert abs(key.max() - G) <= 1e-12 and key[np.argmax(gphi)] == G
        assert (np.diff(key[np.argsort(gphi)]) >= 0).all()                  # monotone in gphi
        direct = -np.log(np.exp(-G) - np.exp(-gphi.max()) + np.exp(-gphi))
        ok = np.abs(gphi - gphi.max()) > 1e-3                               # where the direct form is accurate
        assert np.allclose(key[ok], direct[ok], rtol=0, atol=1e-9)
    # far in the tails the direct form overflows or cancels; the stable form stays finite and below G
    key = truncated_gumbel(40.0, np.array([-60.0, 0.0, 1e-9]), 1e-9)
    assert np.isfinite(key).all() and key[2] == 40.0 and (key[:2] < 40.0).all()


def test_first_result_follows_generate_law_on_the_table():
    """P1 and P2 on the table: 3000 items with their own seeds in one batched run."""
    table = _table(1)
    law = _law(lambda pre, t: table[pre], STEPS, {})
    B, K = 3000, 3
    ref = _run_table(table, B, K, list(range(7, 7 + B)))
    tokens, n_new, log_probs, keys, kappa = ref.result()
    rep = _replies(tokens, n_new, B, K)
    for b in range(B):
        assert len(set(rep[b])) == K and all(r in law for r in rep[b]), b        # distinct, min(K, |support|)
        k = keys[b * K:(b + 1) * K]
        assert (k[:-1] >= k[1:]).all()
        for q in range(K):
            assert float(log_probs[b * K + q]) == pytest.approx(np.log(law[rep[b][q]]), abs=1e-5)
    assert torch.isfinite(kappa).all()                                          # 40 sequences > K
    p = _chi2([r[0] for r in rep], law)
    print(f"table: {len(law)} sequences, first result vs generate's law: p = {p:.3g}")
    assert p > 1e-3


def test_estimator_exact_on_a_small_support_and_unbiased_otherwise():
    """P3 and P4: with K >= |support| kappa is -inf, the results are the support and the estimate is exact; with K
    smaller the mean estimate over seeds lies within 4 standard errors of the exact expectation."""
    small = _table(2, dead=[(0, 0), (0, 1), (1, 0), (1, 1), (2, 0), (2, 1)])   # ids 2 and the stop id 3 only
    law = _law(lambda pre, t: small[pre], STEPS, {})
    f = lambda s: len(s) + 2.0 * sum(1 for x in s if x == 2)                     # noqa: E731
    exact = sum(p * f(s) for s, p in law.items())
    B, K = 20, 8
    assert len(law) <= K
    tokens, n_new, log_probs, _, kappa = _run_table(small, B, K, list(range(B))).result()
    rep = _replies(tokens, n_new, B, K)
    vals = torch.tensor([[f(r) for r in rb] for rb in rep], dtype=torch.float64)
    assert torch.isinf(kappa).all() and (kappa < 0).all()
    for b in range(B):
        assert sorted(r for r, q in zip(rep[b], range(K)) if n_new[b * K + q] > 0 or log_probs[b * K + q] > -np.inf) \
            == sorted(law)
    assert sbs_estimate(vals, log_probs, kappa).tolist() == pytest.approx([exact] * B, rel=1e-6)  # fp32 phi
    table = _table(3)
    law = _law(lambda pre, t: table[pre], STEPS, {})
    exact = sum(p * f(s) for s, p in law.items())
    B, K = 2000, 4
    tokens, n_new, log_probs, _, kappa = _run_table(table, B, K, list(range(100, 100 + B))).result()
    rep = _replies(tokens, n_new, B, K)
    vals = torch.tensor([[f(r) for r in rb] for rb in rep], dtype=torch.float64)
    est = sbs_estimate(vals, log_probs, kappa).numpy()
    assert np.isfinite(kappa.numpy()).all()
    se = est.std(ddof=1) / np.sqrt(B)
    print(f"estimator: exact {exact:.4f}, mean {est.mean():.4f} +- {se:.4f}")
    assert abs(est.mean() - exact) <= 4 * se


def test_tiny_model_first_reply_follows_generate_law(tiny):
    """P1 and P2 through ``stochastic_beam_search`` on the tiny model: top_k = 3, 3 new tokens, a stop id."""
    prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 6), generator=torch.Generator().manual_seed(3))
    kw = dict(top_k=3, temperature=0.9)

    def next_logits(pre, t):
        with torch.no_grad():
            seq = torch.cat([prompt, torch.tensor([pre], dtype=torch.long)], 1) if pre else prompt
            return tiny.lm_logits(tiny.hidden(seq, None)[:, -1], tiny.wte.weight.float())[0, :tiny.cfg.vocab_size].numpy()

    first = next_logits((), 0)
    stop = int(np.argsort(-first)[1])                                   # the second most likely first token stops
    law = _law(next_logits, 3, kw, stop=(stop,))
    B, K = 1500, 2
    tokens, n_new, _, _, kappa = tiny.stochastic_beam_search(prompt.repeat(B, 1), num_beams=K, max_new_tokens=3,
                                                             stop_ids=[stop], seed=11, **kw)
    rep = _replies(tokens, n_new, B, K)
    assert all(len(set(r)) == K for r in rep) and torch.isfinite(kappa).all()
    p = _chi2([r[0] for r in rep], law)
    print(f"tiny model: {len(law)} sequences, first reply vs generate's law: p = {p:.3g}")
    assert p > 1e-3


def test_k1_top_k1_is_greedy(tiny):
    ids = torch.randint(0, tiny.cfg.vocab_size, (3, 9), generator=torch.Generator().manual_seed(4))
    want, wn = tiny.generate(ids, max_new_tokens=6, temperature=0.0)
    tokens, n_new, log_probs, _, kappa = tiny.stochastic_beam_search(ids, num_beams=1, max_new_tokens=6, top_k=1)
    assert torch.equal(tokens, want) and torch.equal(n_new, wn)
    assert log_probs.tolist() == [0.0] * 3 and torch.isinf(kappa).all()


def test_stop_and_max_new_follow_r7():
    # one row of three ids, the last a stop id: with K = 4 every sequence of the support finishes
    row = np.log(np.array([0.5, 0.3, 0.2], dtype=np.float64)).astype(np.float32)
    ref = StochasticBeamReference(1, 4, 2, 3, stop_ids=[2], seeds=[5])
    nxt, parent = ref.step(np.stack([row] * 4))
    assert sorted(nxt[:2].tolist()) == [0, 1] and parent.tolist() == [0, 0, 2, 3]
    assert [f[1:3] for f in ref.fin[0]] == [(0, 0)] and not ref.done[0]           # the stop id: n = L - 1, src = j
    assert ref.fin[0][0][3] == pytest.approx(np.log(0.2), abs=1e-6)
    ref.step(np.stack([row] * 4))
    assert ref.done[0] and np.isinf(ref.scores).all()
    fin = ref.fin[0]
    assert len(fin) == 4 and [f[0] for f in fin] == sorted((f[0] for f in fin), reverse=True)
    lengths = sorted(f[1] for f in fin)
    assert set(lengths) <= {0, 1, 2}                                             # stops at steps 0 and 1, or cut at 2
    tokens, n_new, log_probs, _, kappa = ref.result()
    got = {tuple(tokens[q, :int(n_new[q])].tolist()) for q in range(4)}
    assert len(got) == 4 and np.isfinite(float(kappa[0]))                       # support 1 + 2·3 = 7 > K
    for q in range(4):
        seq = tokens[q, :int(n_new[q])].tolist()
        lp = sum(np.log([0.5, 0.3, 0.2][i]) for i in seq) + (np.log(0.2) if len(seq) < 2 else 0.0)
        assert float(log_probs[q]) == pytest.approx(lp, abs=1e-6)


def test_suppression_and_repetition_controls(tiny):
    row = np.log(np.array([0.1, 0.1, 0.1, 0.6, 0.1])).astype(np.float32)
    ref = StochasticBeamReference(1, 2, 3, 5, suppress_ids=[3], min_new=1, seeds=[0])
    ids, phi, _, _ = ref.children(0, 0, row, 0)
    assert 3 not in ids.tolist() and phi.tolist() == pytest.approx([np.log(0.25)] * 3, abs=1e-6)
    assert 3 in ref.children(0, 0, row, 1)[0].tolist()
    ids = torch.randint(0, 20, (2, 10), generator=torch.Generator().manual_seed(8))
    tokens, n_new, _, _, _ = tiny.stochastic_beam_search(ids, num_beams=3, max_new_tokens=10, temperature=1.5,
                                                         top_k=8, seed=3, no_repeat_ngram_size=2,
                                                         repetition_penalty=1.5, suppress_ids=[5], min_new_tokens=4)
    for q in range(6):
        reply = tokens[q, :int(n_new[q])].tolist()
        assert 5 not in reply[:4]
        seq = ids[q // 3].tolist() + reply
        grams = [tuple(seq[t:t + 2]) for t in range(len(seq) - 1)]
        assert len(grams) == len(set(grams)), q


def test_items_alone_equal_items_in_a_batch_and_calls_repeat(tiny):
    g = torch.Generator().manual_seed(2)
    lengths = [5, 16, 11]
    ids = torch.randint(0, tiny.cfg.vocab_size, (3, 16), generator=g)
    kw = dict(num_beams=3, max_new_tokens=6, stop_ids=[int(ids[1, 2])], temperature=0.8, top_k=40, top_p=0.9)
    out = tiny.stochastic_beam_search(ids, lengths, seed=9, **kw)
    assert all(torch.equal(a, b) for a, b in zip(out, tiny.stochastic_beam_search(ids, lengths, seed=9, **kw)))
    seeds = torch.tensor([9, 10, 11], dtype=torch.int64)
    assert all(torch.equal(a, b) for a, b in zip(out, tiny.stochastic_beam_search(ids, lengths, seed=seeds, **kw)))
    for b, n in enumerate(lengths):
        one = tiny.stochastic_beam_search(ids[b:b + 1, :n], seed=9 + b, **kw)
        rows = slice(3 * b, 3 * b + 3)
        assert torch.equal(one[0], out[0][rows]) and torch.equal(one[1], out[1][rows]), b
        assert one[2].tolist() == pytest.approx(out[2][rows].tolist(), abs=1e-6)
        assert one[3].tolist() == pytest.approx(out[3][rows].tolist(), abs=1e-6)
        assert float(one[4][0]) == pytest.approx(float(out[4][b]), abs=1e-6)


def test_bad_arguments_name_the_argument(tiny):
    ids = torch.zeros(1, 6, dtype=torch.long)
    for kw, name in ((dict(temperature=0.0), "temperature"), (dict(temperature=-1.0), "temperature"),
                     (dict(top_k=-1), "top_k"), (dict(top_p=0.0), "top_p"), (dict(top_p=1.5), "top_p"),
                     (dict(num_beams=0), "num_beams"), (dict(num_beams=17), "num_beams"),
                     (dict(stop_ids=list(range(9))), "stop_ids"), (dict(suppress_ids=list(range(1025))), "suppress_ids"),
                     (dict(max_new_tokens=0), "max_new_tokens"), (dict(repetition_penalty=0.0), "repetition_penalty")):
        with pytest.raises(ValueError, match=name):
            tiny.stochastic_beam_search(ids, **kw)
    with pytest.raises(ValueError):
        StochasticBeamReference(1, 2, 3, 5, temperature=0.0, seeds=[0])
    with pytest.raises(ValueError):
        StochasticBeamReference(2, 2, 3, 5, seeds=[0])

