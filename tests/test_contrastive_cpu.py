"""Contrastive search on the CPU: the fp64 definition (ops/contrastive.py) on hand cases, ``GPT2DoubleHeads.
contrastive_search`` against greedy decoding, a brute-force uncached oracle, rows alone, the repetition controls and
argument errors, the ConvAI pass-through, and the contrastive kernels' build (nvcc only, no device)."""
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.contrastive import candidates_row, max_cosine, rerank_row, select_candidates  # noqa: E402

U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def test_alpha_zero_and_top_k_one_are_greedy():
    rng = np.random.default_rng(0)
    for _ in range(50):
        row = (rng.standard_normal(40) * 2).astype(np.float32)
        row[rng.integers(0, 40, 3)] = row[rng.integers(0, 40)]         # ties among the values
        want = int(np.argmax(row))                                      # the first maximum: the lower id
        ctx = rng.standard_normal((5, 8))
        for k, alpha in ((4, 0.0), (1, 0.7), (1, 1.0)):
            ids, probs = candidates_row(row, k)
            assert rerank_row(ids, probs, rng.standard_normal((k, 8)), ctx, alpha)["token"] == want


def test_candidates_ranked_by_logit_with_ties_to_the_lower_id():
    row = np.array([0.5, 2.0, -np.inf, 2.0, 1.0, 2.0], dtype=np.float32)
    ids, probs = candidates_row(row, 4)
    assert ids.tolist() == [1, 3, 5, 4]
    e = np.exp(np.array([0.5, 2.0, 2.0, 1.0, 2.0]) - 2.0)
    assert probs.tolist() == pytest.approx((np.array([1, 1, 1, np.exp(-1.0)]) / e.sum()).tolist(), abs=1e-15)
    # fewer live ids than k: the missing slots are invalid, and an invalid slot never wins
    ids, probs = candidates_row(np.array([-np.inf, 1.0, -np.inf, 0.0], dtype=np.float32), 4)
    assert ids.tolist() == [1, 3, -1, -1] and probs[2:].tolist() == [0.0, 0.0]
    h = np.array([[1.0, 0.0], [0.0, 1.0], [0.0, -1.0], [-1.0, 0.0]])
    r = rerank_row(ids, probs, h, np.array([[1.0, 0.0]]), 1.0)
    assert r["rank"] == 1 and r["token"] == 3 and r["scores"][2:].tolist() == [-np.inf, -np.inf]
    # no live id at all: id 0
    ids, probs = candidates_row(np.full(5, -np.inf, dtype=np.float32), 3)
    assert rerank_row(ids, probs, np.ones((3, 2)), np.ones((1, 2)), 0.5)["token"] == 0


def test_alpha_one_picks_the_least_similar_candidate():
    ids, probs = candidates_row(np.array([3.0, 2.0, 1.0, 0.0], dtype=np.float32), 3)
    ctx = np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])
    h = np.array([[2.0, 0.1, 0.0], [0.3, 0.3, 1.0], [0.0, 5.0, 0.0]])       # cosines ~1, ~0.39, 1
    r = rerank_row(ids, probs, h, ctx, 1.0)
    assert r["rank"] == 1 and r["token"] == 1
    assert r["sims"].tolist() == pytest.approx([2 / math.hypot(2, 0.1), 0.3 / math.sqrt(1.18), 1.0], abs=1e-12)


def test_equal_scores_go_to_the_lower_rank():
    ids = np.array([7, 3, 9])
    probs = np.array([0.3, 0.3, 0.1])
    h = np.array([[1.0, 1.0], [1.0, 1.0], [1.0, 0.1]])                   # the first two score exactly alike
    r = rerank_row(ids, probs, h, np.array([[1.0, 0.0]]), 0.5)
    assert r["scores"][0] == r["scores"][1] and r["rank"] == 0 and r["token"] == 7


def test_zero_norm_vectors_count_as_cosine_zero():
    ctx = np.array([[0.0, 0.0], [-1.0, 0.0]])
    sims = max_cosine(np.array([[0.0, 0.0], [1.0, 0.0], [-2.0, 0.0]]), ctx)
    assert sims.tolist() == [0.0, 0.0, 1.0]                              # 0 from the zero vector beats -1


def test_suppression_only_while_below_min_new():
    row = np.array([1.0, 5.0, 4.0, 3.0], dtype=np.float32)
    assert candidates_row(row, 2, step=0, min_new=1, suppress_ids=[1])[0].tolist() == [2, 3]
    assert candidates_row(row, 2, step=1, min_new=1, suppress_ids=[1])[0].tolist() == [1, 2]
    ids, _ = select_candidates(torch.from_numpy(np.stack([row, row])), 4, 2, done=torch.tensor([0, 1]))
    assert ids.tolist() == [[1, 2], [-1, -1]]                           # a done row gets no candidate


def test_alpha_zero_equals_greedy_generate_and_rows_alone(tiny):
    """alpha = 0 is greedy decoding. The candidates' hidden states come from a step at B·k rows rather than B; on the
    CPU those GEMMs give every row the same bits at either row count, so the tokens are equal, as is a row alone and
    the same row in a ragged batch (the GPU test allows near ties here and counts them)."""
    g = torch.Generator().manual_seed(1)
    V = tiny.cfg.vocab_size
    lengths = [5, 30, 17, 30]
    ids = torch.randint(0, V, (4, 30), generator=g)
    tt = torch.randint(V - 5, V - 3, (4, 30), generator=g)
    want, _ = tiny.generate(ids, lengths, tt, max_new_tokens=25, temperature=0.0)
    got, n_new = tiny.contrastive_search(ids, lengths, tt, top_k=4, penalty_alpha=0.0, max_new_tokens=25)
    differ = sum(not torch.equal(got[b], want[b]) for b in range(4))
    print(f"contrastive_search(alpha=0) vs generate(temperature=0): {differ} of 4 rows differ")
    assert differ == 0 and n_new.tolist() == [25] * 4
    kw = dict(top_k=5, penalty_alpha=0.6, max_new_tokens=20)
    tokens, _ = tiny.contrastive_search(ids, lengths, tt, **kw)
    again, _ = tiny.contrastive_search(ids, lengths, tt, **kw)
    assert torch.equal(tokens, again)
    for b, n in enumerate(lengths):
        alone, _ = tiny.contrastive_search(ids[b:b + 1, :n], None, tt[b:b + 1, :n], **kw)
        assert torch.equal(alone[0], tokens[b]), b


def _oracle(model, prompt, K, alpha, n):
    """Contrastive search with no cache at all: each step runs ``hidden`` over the whole sequence (the context and the
    logits) and over the sequence extended by each candidate (its hidden state), scored by the fp64 definition. Per
    step it also returns the slack its decision had: the gap between the two best scores and between the k-th and
    (k+1)-th logits."""
    seq = list(prompt)
    head = model.wte.weight.float()
    out, slack = [], []
    with torch.no_grad():
        for _ in range(n):
            hs = model.hidden(torch.tensor([seq]), None)[0]
            logits = model.lm_logits(hs[-1], head).numpy()
            ids, probs = candidates_row(logits, K)
            hc = np.stack([model.hidden(torch.tensor([seq + [int(c)]]), None)[0, -1].double().numpy() for c in ids])
            r = rerank_row(ids, probs, hc, hs.double().numpy(), alpha)
            sc = np.sort(r["scores"])[::-1]
            srt = np.sort(logits.astype(np.float64))[::-1]
            slack.append((sc[0] - sc[1], srt[K - 1] - srt[K], float(np.abs(hs.double().numpy()).max()),
                          float(probs.max())))
            out.append(r["token"])
            seq.append(r["token"])
    return out, slack


def test_against_a_brute_force_uncached_oracle(tiny):
    """Tokens equal the oracle's except at near ties. The bound: a hidden state is a chain of dot products of lengths
    D (attention projections), 4 D (MLP), T (attention) per layer and D (final LayerNorm); to first order its
    relative error is at most N u with N the sum of those lengths, on both paths. A cosine then moves by at most
    2 (2 N u) + (2 D + 4) u, a logit by at most 2 N u |h| |w| <= 2 N u sqrt(D) max|h| max|w| (Cauchy-Schwarz), and a
    probability p by p times twice that. Two scores closer than twice the resulting score error, or a k-th and
    (k+1)-th logit closer than twice the logit error, may decide the other way."""
    cfg = tiny.cfg
    D, Lyr = cfg.n_embd, cfg.n_layer
    g = torch.Generator().manual_seed(7)
    wmax = float(tiny.wte.weight.detach().abs().max())
    exempt = steps = 0
    for trial, (K, alpha, T) in enumerate(((4, 0.6, 12), (8, 0.4, 20), (3, 0.9, 7), (6, 0.6, 30))):
        prompt = torch.randint(0, cfg.vocab_size, (T,), generator=g).tolist()
        n = 12
        want, slack = _oracle(tiny, prompt, K, alpha, n)
        got, _ = tiny.contrastive_search(torch.tensor([prompt]), top_k=K, penalty_alpha=alpha, max_new_tokens=n)
        got = got[0].tolist()
        N = Lyr * (D + 4 * D + T + n) + D
        steps += n
        for i in range(n):
            if got[i] == want[i]:
                continue
            score_gap, logit_gap, hmax, pmax = slack[i]
            dl = 2 * N * U32 * math.sqrt(D) * hmax * wmax
            ds = 4 * N * U32 + (2 * D + 4) * U32
            tol = 2 * ((1 - alpha) * pmax * 2 * dl + alpha * ds)
            assert score_gap <= tol or logit_gap <= 2 * dl, (trial, i, got, want, slack[i], tol)
            exempt += 1
            break                                                      # the sequences differ from here on
    print(f"contrastive_search vs the uncached oracle: {steps} steps, {exempt} needed the near-tie exemption")
    assert exempt <= 1


def test_no_repeat_ngram_and_stop_ids(tiny):
    g = torch.Generator().manual_seed(3)
    V = tiny.cfg.vocab_size
    lengths = [8, 3, 20]
    ids = torch.randint(0, V, (3, 20), generator=g)
    for size in (1, 2, 3):
        tokens, n_new = tiny.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.3, max_new_tokens=30,
                                                no_repeat_ngram_size=size, repetition_penalty=1.3)
        for b, x in enumerate(lengths):
            seq = ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist()
            grams = [tuple(seq[j:j + size]) for j in range(len(seq) - size + 1)]
            assert len(grams) == len(set(grams)), (size, b)
    tokens, _ = tiny.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.5, max_new_tokens=12)
    stop = [int(tokens[0, 4]), int(tokens[1, 0])]
    t, n_new = tiny.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.5, max_new_tokens=12, stop_ids=stop)
    assert n_new.tolist()[:2] == [4, 0] and torch.equal(t[0, :4], tokens[0, :4]) and (t[0, 4:] == -1).all()
    t, _ = tiny.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.5, max_new_tokens=12, stop_ids=stop,
                                   suppress_ids=stop, min_new_tokens=12)
    assert not set(t.view(-1).tolist()) & set(stop) and (t >= 0).all()


def test_contrastive_search_rejects_bad_arguments(tiny):
    ids = torch.zeros(2, 10, dtype=torch.long)
    n_pos = tiny.cfg.n_positions
    bad = [dict(top_k=0), dict(top_k=17), dict(penalty_alpha=-0.1), dict(penalty_alpha=1.5),
           dict(penalty_alpha=float("nan")), dict(max_new_tokens=n_pos - 9), dict(max_new_tokens=0),
           dict(min_new_tokens=-1), dict(lengths=[3]), dict(lengths=[0, 4]), dict(repetition_penalty=0.0)]
    for kw in bad:
        with pytest.raises(ValueError):
            tiny.contrastive_search(ids, **kw)
    tiny.contrastive_search(ids, max_new_tokens=n_pos - 10, top_k=16, penalty_alpha=1.0)   # exactly fills the positions


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_sample_replies_with_contrastive_search(tiny):
    from adapcc_b200.eval import convai

    dialogs = [([[1, 2]], [[3, 4, 5]]), ([[6]], [[7], [8, 9]])]
    replies = convai.sample_replies(tiny, _Tok(), dialogs, max_length=6, min_length=2, top_k=4, penalty_alpha=0.6)
    assert len(replies) == 2 and all(2 <= len(r) <= 6 and not set(r) & set(_Tok.special_ids) for r in replies)
    assert convai.sample_replies(tiny, _Tok(), dialogs[1:], max_length=6, min_length=2, top_k=4,
                                 penalty_alpha=0.6) == replies[1:]
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, top_k=4, penalty_alpha=0.6)
    assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0


def test_build_log_shows_contrastive_select_and_rerank_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_contrastive\.cu", log)
    for kernel in ("cs_select_kernel", "cs_sim_kernel", "cs_commit_kernel", "cs_context_init_kernel",
                   "beam_rows_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
