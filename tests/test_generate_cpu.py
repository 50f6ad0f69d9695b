"""Batched sampled generation on the CPU: Philox against the Random123 known answers, the fp64 sampling definition
against the sort-based filter of ``sample_sequence``, ``GPT2DoubleHeads.generate`` on the tiny model, the batched
ConvAI F1 path, and the sampling kernels' build (nvcc only, no device)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.sampling import philox4x32_10, reference_row, sample_reference  # noqa: E402


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def test_philox_known_answers():
    # Random123's kat_vectors for philox4x32_10
    assert philox4x32_10((0, 0, 0, 0), (0, 0)) == (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)
    ones = 0xFFFFFFFF
    assert philox4x32_10((ones,) * 4, (ones, ones)) == (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)
    assert philox4x32_10((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0)) == \
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)


def _sort_filter(x, top_k, top_p):
    """The kept set of ``sample_sequence``'s filter (top-k by the k-th value, then the sort-based nucleus)."""
    logits = torch.tensor(x, dtype=torch.float64)[None]
    if top_k > 0:
        kth = torch.topk(logits, min(top_k, logits.shape[1])).values[:, -1:]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    if 0.0 < top_p < 1.0:
        srt, idx = torch.sort(logits, descending=True)
        cum = torch.softmax(srt, -1).cumsum(-1)
        drop = cum > top_p
        drop[:, 1:] = drop[:, :-1].clone()
        drop[:, 0] = False
        logits = logits.masked_fill(torch.zeros_like(drop).scatter(1, idx, drop), float("-inf"))
    return (logits[0] > float("-inf")).numpy()


def test_reference_keeps_the_sort_based_set_on_tie_free_logits():
    rng = np.random.default_rng(0)
    checked = 0
    for trial in range(300):
        V = int(rng.integers(2, 400))
        l = (rng.standard_normal(V) * rng.uniform(0.5, 6)).astype(np.float32)
        T = float(rng.choice([0.3, 0.7, 1.0, 1.7]))
        k = int(rng.choice([0, 1, 5, 40, V - 1, V]))
        p = float(rng.choice([0.05, 0.5, 0.9, 0.99, 1.0]))
        r = reference_row(l, T, k, p, seed=trial, pos=7)
        x = (l / np.float32(T)).astype(np.float32)
        if np.unique(x).size != V:                                   # tie-free rows only
            continue
        want = _sort_filter(x.astype(np.float64), k, p)
        # the nucleus rule compares a cumulative mass with p: skip rows where that mass sits at p within rounding
        tail = r["tail"][np.isfinite(r["tail"])] / r["Z"]
        if p < 1 and np.min(np.abs(tail - np.float32(p))) < 1e-9:
            continue
        assert np.array_equal(r["kept"], want), (trial, V, T, k, p)
        assert r["kept"][r["token"]]
        checked += 1
    assert checked > 280


def test_reference_hand_cases():
    l = np.array([1.0, 3.0, 2.0, 3.0, 2.0, 2.0, -1.0], dtype=np.float32)
    r = reference_row(l, 1.0, 3, 1.0, seed=1, pos=0)                 # ties at the 3rd value (2.0) are all kept
    assert r["kept"].tolist() == [False, True, True, True, True, True, False]
    for k, p in ((1, 1.0), (0, 1e-6), (2, 1e-6)):                     # only the maximum (both tied ones)
        assert reference_row(l, 0.7, k, p, seed=2, pos=3)["kept"].tolist() == [False, True, False, True] + [False] * 3
    assert reference_row(l, 0.7, 0, 1.0, seed=2, pos=3)["kept"].all()  # top_p = 1 keeps everything
    assert reference_row(l, 0.0, 0, 0.9, seed=0, pos=0)["token"] == 1   # greedy: lowest index on a tie
    sup = [1, 3]
    for pos in range(200):
        r = reference_row(l, 1.0, 0, 1.0, seed=5, pos=pos, step=0, min_new=1, suppress_ids=sup)
        assert r["token"] not in sup
        assert not r["kept"][sup].any()
    assert reference_row(l, 0.0, 0, 1.0, seed=0, pos=0, step=1, min_new=1, suppress_ids=sup)["token"] == 1
    one = np.full(9, -np.inf, dtype=np.float32)
    one[6] = -3.0
    assert reference_row(one, 0.8, 2, 0.5, seed=3, pos=1)["token"] == 6


def test_sample_reference_batch_stop_and_done():
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(4, 10, generator=g)
    logits[1, 7] = 50.0                                               # row 1 draws its stop id
    nxt, tok, done = sample_reference(logits, 10, 0.0, 0, 1.0, torch.arange(4), torch.zeros(4, dtype=torch.int32), 0,
                                      stop_ids=[7], done=torch.tensor([0, 0, 1, 0], dtype=torch.int32))
    assert tok[1] == -1 and done.tolist() == [0, 1, 1, 0] and nxt[1] == 7
    assert tok[2] == -1 and tok[0] == int(logits[0].argmax()) and tok[3] == int(logits[3].argmax())
    with pytest.raises(ValueError):
        sample_reference(logits, 10, -1.0, 0, 1.0, torch.arange(4), torch.zeros(4), 0)


def _argmax_uncached(model, ids, n):
    out = []
    for _ in range(n):
        h = model.hidden(ids, None)[:, -1]
        nxt = (h.float() @ model.wte.weight.float().t())[:, :model.cfg.vocab_size].argmax(-1, keepdim=True)
        ids = torch.cat([ids, nxt], 1)
        out.append(int(nxt))
    return out


def test_generate_top1_equals_uncached_argmax(tiny):
    g = torch.Generator().manual_seed(1)
    prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 20), generator=g)
    with torch.no_grad():
        want = _argmax_uncached(tiny, prompt, 25)
    for kw in (dict(top_k=1), dict(temperature=0.0)):
        tokens, n_new = tiny.generate(prompt, max_new_tokens=25, seed=3, **kw)
        assert tokens[0].tolist() == want and n_new.tolist() == [25]


def test_generate_row_alone_equals_row_in_ragged_batch_and_repeats(tiny):
    g = torch.Generator().manual_seed(2)
    V = tiny.cfg.vocab_size
    lengths = [5, 30, 17]
    ids = torch.randint(0, V, (3, 30), generator=g)
    tt = torch.randint(V - 5, V - 3, (3, 30), generator=g)
    kw = dict(max_new_tokens=30, temperature=0.9, top_k=50, top_p=0.95)
    tokens, n_new = tiny.generate(ids, lengths, tt, seed=11, **kw)
    again, _ = tiny.generate(ids, lengths, tt, seed=11, **kw)
    assert torch.equal(tokens, again) and n_new.tolist() == [30] * 3
    other, _ = tiny.generate(ids, lengths, tt, seed=12, **kw)
    assert not torch.equal(tokens, other)
    for b, n in enumerate(lengths):
        alone, _ = tiny.generate(ids[b:b + 1, :n], None, tt[b:b + 1, :n], seed=torch.tensor([11 + b]), **kw)
        assert torch.equal(alone[0], tokens[b]), b


def test_generate_stop_ids_pad_with_minus_one(tiny):
    V = tiny.cfg.vocab_size
    m = GPT2DoubleHeads(GPT2Config.tiny()).eval()
    m.load_state_dict(tiny.state_dict())
    prompt = torch.randint(0, V, (4, 8), generator=torch.Generator().manual_seed(3))
    tokens, _ = m.generate(prompt, max_new_tokens=16, temperature=1.0, top_p=1.0, seed=0)
    stop = int(tokens[2, 4])                                         # row 2 draws this id as its 5th token
    got, n_new = m.generate(prompt, max_new_tokens=16, temperature=1.0, top_p=1.0, seed=0, stop_ids=[stop])
    for b in range(4):
        row = tokens[b].tolist()
        k = row.index(stop) if stop in row else 16
        assert n_new[b] == k and got[b, :k].tolist() == row[:k] and (got[b, k:] == -1).all(), b
    assert n_new[2] <= 4
    # suppressed while fewer than min_new_tokens are out: the stop id cannot end the reply early
    got, n_new = m.generate(prompt, max_new_tokens=16, temperature=1.0, top_p=1.0, seed=0, stop_ids=[stop],
                            suppress_ids=[stop], min_new_tokens=6)
    assert (n_new >= 6).all()


def test_generate_rejects_bad_arguments(tiny):
    ids = torch.zeros(2, 10, dtype=torch.long)
    n_pos = tiny.cfg.n_positions
    bad = [dict(max_new_tokens=n_pos - 9), dict(temperature=-0.1), dict(top_k=-1), dict(top_p=0.0), dict(top_p=1.5),
           dict(max_new_tokens=0), dict(lengths=[3]), dict(lengths=[0, 4]), dict(lengths=[3, 11]),
           dict(seed=torch.zeros(3, dtype=torch.long)), dict(min_new_tokens=-1)]
    for kw in bad:
        with pytest.raises(ValueError):
            tiny.generate(ids, **kw)
    tiny.generate(ids, max_new_tokens=n_pos - 10)                  # exactly fills the positions


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_evaluate_dialogs_batched_f1_and_unchanged_sequential_path(tiny):
    from adapcc_b200.eval import convai

    dialogs = [{"personality": ["i like tea", "i run"],
                "utterances": [{"history": ["hello there"] * (j + 1), "candidates": ["x y", "1 2 3"]}
                               for j in range(3)]} for _ in range(3)]
    kw = dict(max_length=6, min_length=2, temperature=0.8, top_k=0, top_p=0.9)
    seq = convai.evaluate_dialogs(tiny, _Tok(), dialogs, "f1", seed=4, **kw)
    assert convai.evaluate_dialogs(tiny, _Tok(), dialogs, "f1", seed=4, batch_size=0, **kw) == seq
    a = convai.evaluate_dialogs(tiny, _Tok(), dialogs, "f1", seed=4, batch_size=4, **kw)
    b = convai.evaluate_dialogs(tiny, _Tok(), dialogs, "f1", seed=4, batch_size=3, **kw)
    assert a == b and a["examples"] == 9 and 0.0 <= a["f1"] <= 1.0
    replies = convai.sample_replies(tiny, _Tok(), [([[1, 2]], [[3, 4, 5]]), ([[6]], [[7], [8, 9]])], max_length=6,
                                    min_length=6, seeds=[1, 2])
    assert all(len(r) == 6 and not set(r) & set(_Tok.special_ids) for r in replies)


def test_build_log_shows_sampling_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_sample\.cu", log)
    for kernel in ("lm_head_logits_kernel", "sample_tokens_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
