"""Beam search on the CPU: the fp64 definition (ops/beam.py) on hand cases, its done rule against running every step,
``GPT2DoubleHeads.beam_search`` against exhaustive search, greedy decoding, items alone and HuggingFace's beam search,
the ConvAI reply path, and the beam kernels' build (nvcc only, no device)."""
import copy
import itertools
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.beam import BeamReference  # noqa: E402

NEG = -np.inf


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _rows(*probs):
    """fp32 logits rows from probabilities (log 0 = -inf)."""
    with np.errstate(divide="ignore"):
        return np.log(np.array(probs, dtype=np.float64)).astype(np.float32)


def _lp(row):
    x = np.asarray(row, dtype=np.float32).astype(np.float64)
    m = x.max()
    return (x - m) - np.log(np.exp(x - m).sum())


def test_stop_id_before_and_after_the_kth_beam():
    # ranked first: offered to the finished set, and the beams are the next two non-stop candidates
    ref = BeamReference(1, 2, 4, 6, stop_ids=[5])
    row = _rows(0.05, 0.2, 0.15, 0.05, 0.05, 0.5)
    nxt, parent = ref.step(np.stack([row, row]))
    assert nxt.tolist() == [1, 2] and parent.tolist() == [0, 0]
    assert len(ref.fin[0]) == 1 and ref.fin[0][0][1:] == (0, 0)
    assert ref.fin[0][0][0] == pytest.approx(_lp(row)[5], abs=1e-12)
    assert ref.scores[0].tolist() == pytest.approx([_lp(row)[1], _lp(row)[2]], abs=1e-12)
    # ranked after the second non-stop candidate: not offered
    ref = BeamReference(1, 2, 4, 6, stop_ids=[5])
    row = _rows(0.05, 0.4, 0.3, 0.05, 0.05, 0.15)
    assert ref.step(np.stack([row, row]))[0].tolist() == [1, 2] and ref.fin[0] == []
    # ranked between the first and the second: offered, and the second beam is the next candidate after it
    ref = BeamReference(1, 2, 4, 6, stop_ids=[5])
    row = _rows(0.05, 0.4, 0.1, 0.05, 0.05, 0.35)
    assert ref.step(np.stack([row, row]))[0].tolist() == [1, 2] and len(ref.fin[0]) == 1


def test_suppression_while_below_min_new():
    row = _rows(0.1, 0.1, 0.1, 0.6, 0.1)
    ref = BeamReference(1, 2, 3, 5, suppress_ids=[3], min_new=1)
    nxt, _ = ref.step(np.stack([row, row]))
    assert 3 not in nxt.tolist() and nxt.tolist() == [0, 1]
    # removed before the log-softmax: the remaining ids share all the mass
    assert ref.scores[0, 0] == pytest.approx(np.log(0.25), abs=1e-6)
    nxt, _ = ref.step(np.stack([row, row]))                  # step 1 >= min_new: id 3 is back
    assert nxt[0] == 3


@pytest.mark.parametrize("alpha", [-1.0, 0.0, 1.0, 2.0])
def test_length_penalty_orders_the_finished_set(alpha):
    ref = BeamReference(1, 2, 4, 4, length_penalty=alpha, stop_ids=[0])
    first = _rows(0.5, 0.25, 0.25, 1e-9)
    ref.step(np.stack([first, first]))                      # the stop id first: a hypothesis of L = 1
    assert ref.fin[0] == [(pytest.approx(np.log(0.5 / (0.5 + 0.5 + 1e-9)), abs=1e-6), 0, 0)]
    second = _rows(0.9, 0.05, 0.05, 1e-9)
    ref.step(np.stack([second, second]))                    # both rows' stop ids (tied), L = 2
    c1 = ref.candidates(first, 0.0, 0)[0]
    c2 = ref.candidates(first, 0.0, 0)[1] + _lp(second)[0]
    want = sorted([(c1, 0, 0), (c2 / 2.0 ** alpha, 1, 0), (c2 / 2.0 ** alpha, 1, 1)], key=lambda t: -t[0])
    # the K best by normalised score; of the two tied L = 2 hypotheses the earlier one (row 0) ranks first
    assert [(n, s) for _, n, s in ref.fin[0]] == [(n, s) for _, n, s in want[:2]]
    assert [t[0] for t in ref.fin[0]] == pytest.approx([t[0] for t in want[:2]], abs=1e-12)
    assert ref.fin[0][0][1] == (1 if alpha == 2.0 else 0)  # only a large enough penalty prefers the longer one


def test_dead_beams_on_a_tiny_vocabulary():
    ref = BeamReference(1, 4, 3, 3, stop_ids=[2])
    row = _rows(0.5, 0.3, 0.2)
    nxt, parent = ref.step(np.stack([row] * 4))
    # two non-stop candidates for four beams: beams 2 and 3 are dead and continue themselves
    assert nxt.tolist() == [0, 1, 0, 0] and parent.tolist() == [0, 0, 2, 3]
    assert np.isfinite(ref.scores[0, :2]).all() and (ref.scores[0, 2:] == NEG).all()
    nxt, parent = ref.step(np.stack([row] * 4))              # only rows 0 and 1 offer candidates: 4 of them
    assert parent.tolist() == [0, 0, 1, 1] and nxt.tolist() == [0, 1, 0, 1] and np.isfinite(ref.scores).all()


def _random_run(rng, early_stop):
    B, K = 3, int(rng.integers(1, 6))
    V, n = int(rng.integers(3, 12)), int(rng.integers(1, 7))
    stop = list(rng.choice(V, size=int(rng.integers(0, 3)), replace=False))
    alpha = float(rng.choice([-1.0, 0.0, 0.5, 1.0, 2.0]))
    ref = BeamReference(B, K, n, V, alpha, stop, [int(stop[0])] if stop else [], int(rng.integers(0, 2)),
                        early_stop=early_stop)
    steps = []
    for _ in range(n):
        logits = (rng.standard_normal((B * K, V)) * 2).astype(np.float32)
        logits[rng.random((B * K, V)) < 0.1] = -np.inf
        steps.append(logits)
    return ref, steps


def test_done_rule_is_exact():
    """Stopping an item early never changes its result: the same random logits with the done rule on and off."""
    stopped = 0
    for trial in range(400):
        runs = []
        for early in (True, False):
            ref, steps = _random_run(np.random.default_rng(trial), early)
            for logits in steps:
                ref.step(logits)
            runs.append(ref)
        on, off = runs[0].result(), runs[1].result()
        assert all(torch.equal(a, b) for a, b in zip(on, off)), trial
        stopped += int(runs[0].done.sum())
    assert stopped > 0


def test_beam_search_finds_the_best_of_all_sequences():
    """Vocabulary 4, 16 beams, 3 new tokens, no stop id: beam search keeps every prefix, so it must return the
    best of the 64 sequences, each scored by an uncached fp64 forward."""
    cfg = GPT2Config(vocab_size=4, n_positions=16, n_embd=32, n_layer=2, n_head=2, lm_chunk_rows=64)
    torch.manual_seed(3)
    m = GPT2DoubleHeads(cfg).eval()
    with torch.no_grad():
        m.wte.weight.mul_(20.0)                            # spread the 4-way distributions out
    prompt = torch.tensor([[1, 3, 0, 2, 2]])
    m64 = copy.deepcopy(m).double()
    head = m64.wte.weight[:4]
    seqs = list(itertools.product(range(4), repeat=3))
    scores = []
    with torch.no_grad():
        for s in seqs:
            ids = torch.cat([prompt, torch.tensor([s])], 1)
            lp = torch.log_softmax(m64.hidden(ids, None)[0, 4:7] @ head.t(), -1)
            scores.append(float(sum(lp[t, s[t]] for t in range(3))))
    order = np.argsort(scores)[::-1]
    assert scores[order[0]] - scores[order[1]] > 1e-3
    tokens, n_new, score = m.beam_search(prompt, num_beams=16, max_new_tokens=3, length_penalty=1.0)
    assert tokens[0].tolist() == list(seqs[order[0]]) and n_new.tolist() == [3]
    assert float(score[0]) == pytest.approx(scores[order[0]] / 3, abs=1e-4)


def test_beam_search_greedy_alone_and_repeatable(tiny):
    g = torch.Generator().manual_seed(1)
    V = tiny.cfg.vocab_size
    prompt = torch.randint(0, V, (1, 20), generator=g)
    want, _ = tiny.generate(prompt, max_new_tokens=25, temperature=0.0)
    tokens, n_new, _ = tiny.beam_search(prompt, num_beams=1, max_new_tokens=25)
    assert torch.equal(tokens, want) and n_new.tolist() == [25]
    lengths = [5, 30, 17]
    ids = torch.randint(0, V, (3, 30), generator=g)
    tt = torch.randint(V - 5, V - 3, (3, 30), generator=g)
    kw = dict(num_beams=4, max_new_tokens=12, length_penalty=0.7, stop_ids=[int(ids[0, 0]), 77])
    tokens, n_new, scores = tiny.beam_search(ids, lengths, tt, **kw)
    again = tiny.beam_search(ids, lengths, tt, **kw)
    assert all(torch.equal(a, b) for a, b in zip((tokens, n_new, scores), again))
    for b, n in enumerate(lengths):
        t1, n1, s1 = tiny.beam_search(ids[b:b + 1, :n], None, tt[b:b + 1, :n], **kw)
        assert torch.equal(t1[0], tokens[b]) and int(n1) == int(n_new[b]), b
        assert float(s1) == pytest.approx(float(scores[b]), abs=1e-5)
        k = int(n_new[b])
        assert (tokens[b, k:] == -1).all() and (tokens[b, :k] >= 0).all()
        assert not set(tokens[b, :k].tolist()) & set(kw["stop_ids"])


def test_beam_search_rejects_bad_arguments(tiny):
    ids = torch.zeros(2, 10, dtype=torch.long)
    n_pos = tiny.cfg.n_positions
    bad = [dict(num_beams=0), dict(num_beams=17), dict(stop_ids=list(range(9))), dict(max_new_tokens=n_pos - 9),
           dict(max_new_tokens=0), dict(min_new_tokens=-1), dict(lengths=[3]), dict(lengths=[0, 4]),
           dict(suppress_ids=list(range(1025)))]
    for kw in bad:
        with pytest.raises(ValueError):
            tiny.beam_search(ids, **kw)
    tiny.beam_search(ids, max_new_tokens=n_pos - 10, num_beams=2)         # exactly fills the positions


def test_beam_search_matches_huggingface(tiny):
    transformers = pytest.importorskip("transformers")
    cfg = tiny.cfg
    hf = transformers.GPT2LMHeadModel(transformers.GPT2Config(
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
    missing, _ = hf.load_state_dict({k: v.detach().clone() for k, v in sd.items()}, strict=False)
    assert not [k for k in missing if not k.endswith(("attn.bias", "masked_bias", "lm_head.weight"))], missing
    hf.tie_weights()
    g = torch.Generator().manual_seed(5)
    for trial in range(3):
        prompt = torch.randint(0, cfg.vocab_size, (1, 12), generator=g)
        K, n = (2, 4, 5)[trial], 10
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), num_beams=K, do_sample=False,
                               length_penalty=0.0, max_new_tokens=n, min_new_tokens=n, eos_token_id=None,
                               pad_token_id=0, early_stopping=False)[0, 12:]
        tokens, n_new, _ = tiny.beam_search(prompt, num_beams=K, max_new_tokens=n, length_penalty=0.0)
        assert tokens[0].tolist() == want.tolist(), trial


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_sample_replies_with_beams(tiny):
    from adapcc_b200.eval import convai

    dialogs = [([[1, 2]], [[3, 4, 5]]), ([[6]], [[7], [8, 9]])]
    replies = convai.sample_replies(tiny, _Tok(), dialogs, max_length=6, min_length=2, num_beams=2)
    assert len(replies) == 2 and all(2 <= len(r) <= 6 and not set(r) & set(_Tok.special_ids) for r in replies)
    again = convai.sample_replies(tiny, _Tok(), dialogs[1:], max_length=6, min_length=2, num_beams=2)
    assert again == replies[1:]
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", batch_size=2, max_length=5, num_beams=2)
    assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0


def test_build_log_shows_beam_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_beam\.cu", log)
    for kernel in ("beam_rows_kernel", "beam_select_kernel", "beam_sample_rows_kernel", "beam_sample_select_kernel",
                   "beam_stochastic_rows_kernel", "beam_stochastic_select_kernel", "kv_reorder_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
