"""Beam sampling and n-best results on the CPU: the fp64 definition (``ops.beam.BeamSampleReference``) on hand cases
with the Philox words computed here, Gumbel-top-M against sequential sampling without replacement, HuggingFace's
``generate(do_sample=True, num_beams=K)`` by a chi-square test, ``num_return_sequences``, determinism, errors, the
ConvAI pass-through and the build of the sampled beam kernels (nvcc only, no device)."""
import math
import os
import sys
from itertools import permutations

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.beam import BeamSampleReference, sample_keep  # noqa: E402
from adapcc_b200.ops.sampling import philox4x32_10  # noqa: E402

NEG = -np.inf


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _rows(*probs):
    with np.errstate(divide="ignore"):
        return np.log(np.array(probs, dtype=np.float64)).astype(np.float32)


def _lp(row):
    x = np.asarray(row, dtype=np.float32).astype(np.float64)
    fin = x > -np.inf
    m = x[fin].max()
    return (x - m) - np.log(np.exp(x[fin] - m).sum())


def _g(c, j, i, step, seed):
    """Rule S4's key of candidate (j, i), from the scalar Philox of ops/sampling.py."""
    w = philox4x32_10((i >> 2, j, step, 0), (seed & 0xFFFFFFFF, seed >> 32))[i & 3]
    u = ((w >> 8) + 0.5) * 2.0 ** -24
    return c - math.log(-math.log(u))


def _draws(cands, step, seed, M):
    """The sample of candidates ``{(j, i): c}`` in draw order: ``[(j, i, c)]``."""
    keyed = sorted(cands.items(), key=lambda t: (-_g(t[1], t[0][0], t[0][1], step, seed), t[0]))
    return [(j, i, c) for (j, i), c in keyed[:M]]


def test_draws_follow_the_gumbel_keys_and_beams_go_by_c():
    row = _rows(0.3, 0.25, 0.2, 0.15, 0.06, 0.04)
    lp = _lp(row)
    seen = 0
    for seed in range(60):
        ref = BeamSampleReference(1, 2, 3, 6, seeds=[seed])
        sample = ref.draws(0, np.stack([row, row]), 0)
        want = _draws({(0, i): lp[i] for i in range(6)}, 0, seed, 4)
        assert [(j, i) for _, _, j, i in sample] == [(j, i) for j, i, _ in want], seed
        nxt, parent = ref.step(np.stack([row, row]))
        beams = sorted(range(4), key=lambda d: (-want[d][2], d))[:2]
        assert nxt.tolist() == [want[d][1] for d in beams] and parent.tolist() == [0, 0], seed
        assert ref.scores[0].tolist() == pytest.approx([want[d][2] for d in beams], abs=1e-12)
        seen += beams != [0, 1]                           # the draw order is not the beam order
    assert seen > 0


def test_stop_offered_only_among_the_first_k_draws():
    row = _rows(0.2, 0.2, 0.2, 0.15, 0.1, 0.15)
    lp = _lp(row)
    hits = {True: 0, False: 0}
    for seed in range(80):
        ref = BeamSampleReference(1, 2, 4, 6, stop_ids=[5], seeds=[seed])
        drawn = [i for _, i, _ in _draws({(0, i): lp[i] for i in range(6)}, 0, seed, 4)]
        place = drawn.index(5) if 5 in drawn else 9
        nxt, _ = ref.step(np.stack([row, row]))
        assert 5 not in nxt.tolist()
        if place < 2:
            assert ref.fin[0] == [(pytest.approx(lp[5], abs=1e-12), 0, 0)], seed
            hits[True] += 1
        else:
            assert ref.fin[0] == [], seed
            hits[False] += place < 4
    assert hits[True] > 0 and hits[False] > 0


def test_last_step_offers_the_first_k_draws():
    row = _rows(0.3, 0.25, 0.2, 0.15, 0.1)
    lp = _lp(row)
    for seed in range(10):
        ref = BeamSampleReference(1, 3, 1, 5, length_penalty=0.0, seeds=[seed])
        ref.step(np.stack([row] * 3))
        first = _draws({(0, i): lp[i] for i in range(5)}, 0, seed, 6)[:3]
        assert ref.done[0] and (ref.scores[0] == NEG).all()
        fin = sorted(ref.fin[0], key=lambda t: t[2])
        assert [(n, src) for _, n, src in fin] == [(1, 0), (1, 1), (1, 2)]
        assert [s for s, _, _ in fin] == pytest.approx([c for _, _, c in first], abs=1e-12)
        tokens, n_new, scores = ref.result(3)
        want = sorted(first, key=lambda t: -t[2])
        assert tokens[:, 0].tolist() == [i for _, i, _ in want] and n_new.tolist() == [1, 1, 1]


def test_min_keep_overrides_top_k_one_and_a_tiny_top_p():
    x = np.array([3.0, 2.5, 2.0, 1.0, -1.0], dtype=np.float32)
    assert np.flatnonzero(sample_keep(x, 1, 1.0, 2)).tolist() == [0, 1]
    assert np.flatnonzero(sample_keep(x, 1, 1.0, 3)).tolist() == [0, 1, 2]
    assert np.flatnonzero(sample_keep(x, 0, 1e-6, 2)).tolist() == [0, 1]
    assert np.flatnonzero(sample_keep(x, 4, 1e-6, 3)).tolist() == [0, 1, 2]
    tied = np.array([3.0, 2.0, 2.0, 1.0], dtype=np.float32)   # tied values are kept together
    assert np.flatnonzero(sample_keep(tied, 1, 1e-6, 2)).tolist() == [0, 1, 2]
    # through the definition: two stop ids make min_keep 3
    row = _rows(0.5, 0.2, 0.15, 0.1, 0.05)
    ref = BeamSampleReference(1, 2, 4, 5, stop_ids=[3, 4], top_k=1, seeds=[7])
    ids, c, _ = ref.row_candidates(0, 0, row, 0)
    assert ids.tolist() == [0, 1, 2] and c.tolist() == pytest.approx(_lp(row)[:3].tolist(), abs=1e-12)
    ref = BeamSampleReference(1, 2, 4, 5, top_p=0.01, temperature=0.5, seeds=[7])
    ids, c, _ = ref.row_candidates(0, 0, row, 0)
    assert ids.tolist() == [0, 1] and c.tolist() == pytest.approx((_lp(row)[:2] / 0.5).tolist(), abs=1e-12)


def test_dead_beams_on_a_tiny_vocabulary():
    row = _rows(0.5, 0.3, 0.2)
    ref = BeamSampleReference(1, 4, 3, 3, stop_ids=[2], seeds=[1])
    nxt, parent = ref.step(np.stack([row] * 4))
    # three candidates, one a stop id: two beams, the best c first; beams 2 and 3 are dead
    assert nxt.tolist()[:2] == [0, 1] and parent.tolist() == [0, 0, 2, 3]
    assert np.isfinite(ref.scores[0, :2]).all() and (ref.scores[0, 2:] == NEG).all()
    assert ref.hist_tok[0, 0, 2:].tolist() == [-1, -1] and ref.hist_back[0, 0, 2:].tolist() == [2, 3]


def test_suppression_below_min_new():
    row = _rows(0.1, 0.1, 0.1, 0.6, 0.1)
    ref = BeamSampleReference(1, 2, 3, 5, suppress_ids=[3], min_new=1, seeds=[0])
    ids, c, _ = ref.row_candidates(0, 0, row, 0)
    assert 3 not in ids.tolist() and c.tolist() == pytest.approx([np.log(0.25)] * 4, abs=1e-6)
    nxt, _ = ref.step(np.stack([row, row]))
    assert 3 not in nxt.tolist()
    assert 3 in ref.row_candidates(0, 0, row, 1)[0].tolist()


def test_gumbel_top_m_is_sequential_sampling_without_replacement():
    """Draw orders of the definition over 20 000 seeds against the exact Plackett-Luce probabilities."""
    from scipy.stats import chisquare

    row = _rows(0.35, 0.25, 0.2, 0.12, 0.08)
    w = np.exp(_lp(row))
    rows = np.stack([row, row])
    counts = {}
    n = 20000
    for seed in range(n):
        ref = BeamSampleReference(1, 2, 2, 5, seeds=[seed * 7919 + 3])
        key = tuple(i for _, _, _, i in ref.draws(0, rows, 0))
        counts[key] = counts.get(key, 0) + 1
    orders = list(permutations(range(5), 4))
    want = []
    for o in orders:
        p, left = 1.0, 1.0
        for i in o:
            p *= w[i] / left
            left -= w[i]
        want.append(p * n)
    got = [counts.get(o, 0) for o in orders]
    assert sum(got) == n
    p = chisquare(got, want).pvalue
    print(f"Gumbel-top-4 of 5 vs Plackett-Luce over {n} seeds: p = {p:.3f}")
    assert p > 1e-3


def _chi2_same(a, b):
    from scipy.stats import chi2_contingency

    keys = sorted(set(a) | set(b))
    ca, cb = {}, {}
    for x in a:
        ca[x] = ca.get(x, 0) + 1
    for x in b:
        cb[x] = cb.get(x, 0) + 1
    return float(chi2_contingency(np.array([[ca.get(k, 0) for k in keys], [cb.get(k, 0) for k in keys]]))[1])


@pytest.fixture(scope="module")
def hf(tiny):
    transformers = pytest.importorskip("transformers")
    cfg = tiny.cfg
    m = transformers.GPT2LMHeadModel(transformers.GPT2Config(
        vocab_size=cfg.vocab_size, n_positions=cfg.n_positions, n_embd=cfg.n_embd, n_layer=cfg.n_layer,
        n_head=cfg.n_head, layer_norm_epsilon=cfg.layer_norm_epsilon, activation_function="gelu_new")).eval()
    sd = {"transformer.wte.weight": tiny.wte.weight[:cfg.vocab_size], "transformer.wpe.weight": tiny.wpe.weight,
          "transformer.ln_f.weight": tiny.ln_f.weight, "transformer.ln_f.bias": tiny.ln_f.bias}
    for i, blk in enumerate(tiny.h):
        p = f"transformer.h.{i}."
        for ours, theirs in (("ln_1", "ln_1"), ("ln_2", "ln_2")):
            sd[p + theirs + ".weight"], sd[p + theirs + ".bias"] = getattr(blk, ours).weight, getattr(blk, ours).bias
        for ours, theirs in (("c_attn", "attn.c_attn"), ("c_proj", "attn.c_proj"), ("c_fc", "mlp.c_fc"),
                             ("c_proj2", "mlp.c_proj")):
            sd[p + theirs + ".weight"] = getattr(blk, ours).weight.t()
            sd[p + theirs + ".bias"] = getattr(blk, ours).bias
    missing, _ = m.load_state_dict({k: v.detach().clone() for k, v in sd.items()}, strict=False)
    assert not [k for k in missing if not k.endswith(("attn.bias", "masked_bias", "lm_head.weight"))], missing
    m.tie_weights()
    return m


# K, max_new, temperature, top_k, top_p: min_keep (2) dominates a small top_p; top_k = 5 > M = 4 makes the beams random
HF_SETTINGS = [(2, 2, 0.7, 0, 0.05), (2, 2, 1.0, 5, 1.0)]


@pytest.mark.parametrize("setting", HF_SETTINGS)
def test_beam_sampling_matches_huggingface(tiny, hf, setting):
    K, n, T, top_k, top_p = setting
    prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 8), generator=torch.Generator().manual_seed(11))
    runs = 300
    theirs, theirs_all, ours, ours_all = [], [], [], []
    with torch.no_grad():
        for s in range(runs):
            torch.manual_seed(s)
            out = hf.generate(prompt, attention_mask=torch.ones_like(prompt), num_beams=K, do_sample=True,
                              temperature=T, top_k=top_k, top_p=top_p, max_new_tokens=n, min_new_tokens=n,
                              eos_token_id=None, pad_token_id=0, length_penalty=0.0, early_stopping=False,
                              num_return_sequences=K)[:, 8:]
            theirs.append(tuple(out[0].tolist()))
            theirs_all.append(tuple(sorted(tuple(r) for r in out.tolist())))
            tokens, n_new, _ = tiny.beam_search(prompt, num_beams=K, max_new_tokens=n, length_penalty=0.0,
                                                do_sample=True, temperature=T, top_k=top_k, top_p=top_p,
                                                seed=1000 + s, num_return_sequences=K)
            assert n_new.tolist() == [n] * K
            ours.append(tuple(tokens[0].tolist()))
            ours_all.append(tuple(sorted(tuple(r) for r in tokens.tolist())))
    p1, pk = _chi2_same(theirs, ours), _chi2_same(theirs_all, ours_all)
    print(f"beam sampling vs HuggingFace {setting}: {len(set(ours))} outcomes, p = {p1:.3f}; "
          f"{len(set(ours_all))} n-best sets, p = {pk:.3f}")
    assert len(set(ours)) > 1 and p1 > 1e-3 and pk > 1e-3


def test_n_best_results(tiny, hf):
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, tiny.cfg.vocab_size, (3, 12), generator=g)
    kw = dict(num_beams=4, max_new_tokens=8, length_penalty=0.7, stop_ids=[int(ids[0, 0]), 77])
    for extra in ({}, dict(do_sample=True, temperature=0.9, top_k=30, seed=4)):
        one = tiny.beam_search(ids, **kw, **extra)
        assert all(torch.equal(a, b) for a, b in zip(one, tiny.beam_search(ids, **kw, **extra,
                                                                            num_return_sequences=1)))
        tokens, n_new, scores = tiny.beam_search(ids, **kw, **extra, num_return_sequences=4)
        assert tokens.shape == (12, 8) and n_new.shape == (12,) and scores.shape == (12,)
        for b in range(3):
            rows = slice(4 * b, 4 * b + 4)
            assert torch.equal(tokens[4 * b], one[0][b]) and int(n_new[4 * b]) == int(one[1][b])
            s = scores[rows]
            assert (s[:-1] >= s[1:]).all(), (b, s)
            for q in range(4 * b, 4 * b + 4):
                k = int(n_new[q])
                assert (tokens[q, k:] == -1).all() and (tokens[q, :k] >= 0).all()
    # greedy num_return_sequences = K against HuggingFace, in the configuration of the greedy comparison
    for trial, K in enumerate((2, 4)):
        prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 12), generator=g)
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), num_beams=K, do_sample=False,
                               length_penalty=0.0, max_new_tokens=10, min_new_tokens=10, eos_token_id=None,
                               pad_token_id=0, early_stopping=False, num_return_sequences=K)[:, 12:]
        tokens, _, _ = tiny.beam_search(prompt, num_beams=K, max_new_tokens=10, length_penalty=0.0,
                                        num_return_sequences=K)
        assert tokens.tolist() == want.tolist(), trial


def test_missing_hypotheses_are_padded():
    from adapcc_b200.ops.beam import best_hypotheses

    hist_tok = np.array([[[4, 5]], [[6, -1]]])
    hist_back = np.array([[[0, 0]], [[0, 1]]])
    tokens, n_new, scores = best_hypotheses([[(-1.0, 2, 0)]], hist_tok, hist_back, 2, 2)
    assert tokens.tolist() == [[4, 6], [-1, -1]] and n_new.tolist() == [2, 0]
    assert scores[0] == -1.0 and scores[1] == float("-inf")


def test_determinism_and_independence(tiny):
    g = torch.Generator().manual_seed(2)
    V = tiny.cfg.vocab_size
    lengths = [5, 16, 11]
    ids = torch.randint(0, V, (3, 16), generator=g)
    kw = dict(num_beams=3, max_new_tokens=7, length_penalty=1.0, stop_ids=[int(ids[1, 2])], do_sample=True,
              temperature=0.8, top_k=40, top_p=0.9, num_return_sequences=2)
    out = tiny.beam_search(ids, lengths, seed=9, **kw)
    assert all(torch.equal(a, b) for a, b in zip(out, tiny.beam_search(ids, lengths, seed=9, **kw)))
    seeds = torch.tensor([9, 10, 11], dtype=torch.int64)
    assert all(torch.equal(a, b) for a, b in zip(out, tiny.beam_search(ids, lengths, seed=seeds, **kw)))
    for b, n in enumerate(lengths):
        t1, n1, s1 = tiny.beam_search(ids[b:b + 1, :n], seed=9 + b, **kw)
        rows = slice(2 * b, 2 * b + 2)
        assert torch.equal(t1, out[0][rows]) and torch.equal(n1, out[1][rows]), b
        assert s1.tolist() == pytest.approx(out[2][rows].tolist(), abs=1e-6)
    other = tiny.beam_search(ids, lengths, seed=1234, **kw)
    assert not torch.equal(other[0], out[0])
    # do_sample=False ignores the sampling arguments
    greedy = tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=7)
    ignored = tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=7, temperature=0.1, top_k=2, top_p=0.3,
                               seed=77)
    assert all(torch.equal(a, b) for a, b in zip(greedy, ignored))


def test_bad_arguments_name_the_argument(tiny):
    ids = torch.zeros(1, 6, dtype=torch.long)
    for kw, name in ((dict(do_sample=True, temperature=0.0), "temperature"),
                     (dict(do_sample=True, temperature=-1.0), "temperature"),
                     (dict(num_return_sequences=0), "num_return_sequences"),
                     (dict(num_return_sequences=3), "num_return_sequences")):
        with pytest.raises(ValueError, match=name):
            tiny.beam_search(ids, num_beams=2, max_new_tokens=3, **kw)
    tiny.beam_search(ids, num_beams=2, max_new_tokens=3, temperature=0.0)      # ignored without do_sample
    with pytest.raises(ValueError):
        BeamSampleReference(1, 2, 3, 5, temperature=0.0, seeds=[0])
    with pytest.raises(ValueError):
        BeamSampleReference(2, 2, 3, 5, seeds=[0])


def test_repetition_controls_with_sampling(tiny):
    g = torch.Generator().manual_seed(8)
    ids = torch.randint(0, 20, (2, 10), generator=g)
    tokens, n_new, _ = tiny.beam_search(ids, num_beams=3, max_new_tokens=10, do_sample=True, temperature=1.5,
                                        top_k=8, seed=3, no_repeat_ngram_size=2, repetition_penalty=1.5,
                                        num_return_sequences=3)
    for q in range(6):
        seq = ids[q // 3].tolist() + tokens[q, :int(n_new[q])].tolist()
        grams = [tuple(seq[t:t + 2]) for t in range(len(seq) - 1)]
        assert len(grams) == len(set(grams)), q


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_sample_replies_and_evaluate_dialogs_pass_beam_sample(tiny, monkeypatch):
    from adapcc_b200.eval import convai

    dialogs = [([[1, 2]], [[3, 4, 5]]), ([[6]], [[7], [8, 9]])]
    calls = []
    real = tiny.beam_search

    def spy(*a, **kw):
        calls.append(kw)
        return real(*a, **kw)

    monkeypatch.setattr(tiny, "beam_search", spy)
    replies = convai.sample_replies(tiny, _Tok(), dialogs, max_length=6, min_length=2, num_beams=2, beam_sample=True,
                                    temperature=0.9, top_k=7, top_p=0.8, seeds=[5, 6])
    kw = calls[-1]
    assert kw["do_sample"] is True and (kw["temperature"], kw["top_k"], kw["top_p"]) == (0.9, 7, 0.8)
    assert kw["seed"].tolist() == [5, 6]
    assert len(replies) == 2 and all(2 <= len(r) <= 6 and not set(r) & set(_Tok.special_ids) for r in replies)
    convai.sample_replies(tiny, _Tok(), dialogs, max_length=6, num_beams=2)
    assert "do_sample" not in calls[-1]
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", batch_size=2, max_length=5, num_beams=2, beam_sample=True,
                                top_k=5)
    assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0 and calls[-1]["do_sample"] is True

