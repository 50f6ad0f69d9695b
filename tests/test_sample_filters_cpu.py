"""The truncation filters of the sampler (min-p, typical, epsilon, eta) on the CPU: the fp64 definition in
``ops/sampling.py`` against HuggingFace's warpers and hand cases, ``GPT2DoubleHeads.generate`` on the tiny model
against an eager loop over the definition, argument errors, the ConvAI pass-through and the kernel's build (nvcc only,
no device)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.sampling import reference_row, sample_reference  # noqa: E402

OFF = dict(min_p=0.0, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0)
# each filter alone and chained, as (min_p, typical_p, epsilon_cutoff, eta_cutoff)
CONFIGS = [dict(min_p=0.05), dict(min_p=0.3), dict(typical_p=0.2), dict(typical_p=0.9), dict(epsilon_cutoff=3e-4),
           dict(epsilon_cutoff=0.02), dict(eta_cutoff=3e-4), dict(eta_cutoff=0.02),
           dict(min_p=0.02, typical_p=0.9, epsilon_cutoff=1e-3, eta_cutoff=1e-3),
           dict(min_p=0.1, typical_p=0.5, epsilon_cutoff=0.01, eta_cutoff=0.05)]
# a row is compared with HuggingFace only when no compared quantity sits within this relative margin of its threshold
REL = 1e-6


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _hf_kept(l32, T, f):
    """HuggingFace's chain: temperature (fp32, the same rounding as the definition's step 3), then min-p, typical,
    epsilon and eta in fp64."""
    lp = pytest.importorskip("transformers.generation.logits_process")
    scores = lp.TemperatureLogitsWarper(T)(None, torch.tensor(l32)[None]).double()
    f = {**OFF, **f}
    chain = []
    if f["min_p"] > 0:
        chain.append(lp.MinPLogitsWarper(f["min_p"]))
    if f["typical_p"] < 1:
        chain.append(lp.TypicalLogitsWarper(f["typical_p"]))
    if f["epsilon_cutoff"] > 0:
        chain.append(lp.EpsilonLogitsWarper(f["epsilon_cutoff"]))
    if f["eta_cutoff"] > 0:
        chain.append(lp.EtaLogitsWarper(f["eta_cutoff"]))
    for w in chain:
        scores = w(None, scores)
    return (scores[0] > float("-inf")).numpy()


def _near_threshold(r):
    """True if a filter decision of ``r`` sits within REL of its threshold: a compared quantity (other than the
    typical cut-off's own deviation) or, for typical, the weight that must reach p Z."""
    for name, f in r["filters"].items():
        q = f["q"][np.isfinite(f["q"])]
        if name == "typical":
            q = q[q != f["thr"]]
            if np.any(np.abs(f["G"] - f["pZ"]) <= REL * f["Z"]):
                return True
        if np.any(np.abs(q - f["thr"]) <= REL * max(abs(f["thr"]), 1e-300)):
            return True
    return False


def test_definition_keeps_huggingface_set_on_tie_free_rows():
    pytest.importorskip("transformers")
    rng = np.random.default_rng(0)
    checked = exempt = 0
    for trial in range(400):
        V = int(rng.integers(2, 600))
        l = (rng.standard_normal(V) * rng.uniform(0.5, 6)).astype(np.float32)
        T = float(rng.choice([0.5, 0.8, 1.0, 1.5]))
        if np.unique((l / np.float32(T)).astype(np.float32)).size != V:
            continue
        f = CONFIGS[trial % len(CONFIGS)]
        r = reference_row(l, T, 0, 1.0, seed=trial, pos=3, **f)
        if _near_threshold(r):
            exempt += 1
            continue
        assert np.array_equal(r["kept"], _hf_kept(l, T, f)), (trial, V, T, f)
        assert r["kept"][r["token"]]
        checked += 1
    print(f"filters vs HuggingFace: {checked} rows compared, {exempt} within {REL} of a threshold")
    assert checked >= 380


def test_typical_ties_in_deviation_are_kept_together():
    l = np.array([2.0, 0.0, 0.0, -3.0, 1.0], dtype=np.float32)      # ids 1 and 2 have the same deviation
    cut_at_tie = False
    for p in np.linspace(0.01, 0.99, 99):
        r = reference_row(l, 1.0, 0, 1.0, seed=0, pos=0, typical_p=float(p))
        assert r["kept"][1] == r["kept"][2], p
        d = r["filters"]["typical"]["q"]
        cut_at_tie |= bool(r["filters"]["typical"]["thr"] == d[1] and not r["kept"].all())
    assert cut_at_tie


def test_typical_drops_the_argmax_of_a_peaked_row_and_keeps_a_uniform_row():
    # p_0 = e^5 / (e^5 + 999) = 0.13 while the entropy (6.4) is close to the other ids' surprisal (7.05)
    l = np.zeros(1000, dtype=np.float32)
    l[0] = 5.0
    lp = pytest.importorskip("transformers.generation.logits_process")
    for seed in range(20):
        r = reference_row(l, 1.0, 0, 1.0, seed=seed, pos=seed, typical_p=0.8)
        assert not r["kept"][0] and r["kept"][1:].all() and r["token"] != 0
    hf = lp.TypicalLogitsWarper(0.8)(None, torch.tensor(l, dtype=torch.float64)[None])[0]
    assert hf[0] == float("-inf") and bool((hf[1:] > float("-inf")).all())
    flat = np.full(300, -1.5, dtype=np.float32)
    for p in (0.01, 0.5, 0.99):
        assert reference_row(flat, 0.7, 0, 1.0, seed=1, pos=2, typical_p=p)["kept"].all()


def test_epsilon_and_eta_fall_back_to_the_maximum():
    rng = np.random.default_rng(1)
    l = (rng.standard_normal(1000) * 0.1).astype(np.float32)
    l[[17, 400]] = 1.0                                              # tied maxima, both with p < 0.01
    r = reference_row(l, 1.0, 0, 1.0, seed=0, pos=0, epsilon_cutoff=0.01)
    assert np.flatnonzero(r["kept"]).tolist() == [17, 400]
    # eta's threshold sqrt(eta) exp(-H) is below p_max (H >= -log p_max), so the maximum always survives it
    for trial in range(50):
        x = (rng.standard_normal(500) * rng.uniform(0.1, 5)).astype(np.float32)
        r = reference_row(x, 1.0, 0, 1.0, seed=trial, pos=0, eta_cutoff=0.9)
        assert r["kept"][int(np.argmax(x))]
        assert r["filters"]["eta"]["thr"] <= np.nanmax(r["filters"]["eta"]["q"])
    # min-p keeps the maximum even at 1, with its ties
    x = np.array([0.5, 3.0, 3.0, 2.9], dtype=np.float32)
    assert reference_row(x, 1.0, 0, 1.0, seed=0, pos=0, min_p=1.0)["kept"].tolist() == [False, True, True, False]


def test_filters_at_their_off_values_equal_no_filter():
    rng = np.random.default_rng(2)
    for trial in range(30):
        l = (rng.standard_normal(257) * 3).astype(np.float32)
        for T, k, p in ((0.7, 0, 0.9), (1.0, 20, 1.0), (0.0, 0, 0.9)):
            a = reference_row(l, T, k, p, seed=trial, pos=trial)
            b = reference_row(l, T, k, p, seed=trial, pos=trial, **OFF)
            assert a["token"] == b["token"] and np.array_equal(a["kept"], b["kept"])
            if T > 0:
                assert np.array_equal(a["cum"], b["cum"]) and b["filters"] == {}
    # at temperature 0 the filters have no effect
    l = (rng.standard_normal(100) * 3).astype(np.float32)
    assert reference_row(l, 0.0, 0, 1.0, 0, 0, typical_p=0.1, eta_cutoff=0.5)["token"] == int(np.argmax(l))


def _eager_loop(model, ids, n, T, k, p, seed, f):
    """The definition on uncached fp32 logits, one row at a time."""
    out = []
    V = model.cfg.vocab_size
    head = model.wte.weight.float()
    for b in range(ids.shape[0]):
        seq, row = ids[b:b + 1], []
        for i in range(n):
            logits = (model.hidden(seq, None)[0, -1].float() @ head.t())[:V].numpy()
            t = reference_row(logits, T, k, p, seed + b, seq.shape[1], step=i, **f)["token"]
            row.append(t)
            seq = torch.cat([seq, torch.tensor([[t]])], 1)
        out.append(row)
    return out


@pytest.mark.parametrize("f", CONFIGS[:1] + CONFIGS[3:4] + CONFIGS[5:6] + CONFIGS[7:])
def test_generate_with_filters_equals_the_eager_definition(tiny, f):
    prompt = torch.randint(0, tiny.cfg.vocab_size, (3, 12), generator=torch.Generator().manual_seed(5))
    # the tiny model's logits spread by about 0.16, so a low temperature is what gives every filter ids to remove
    kw = dict(max_new_tokens=12, temperature=0.1, top_k=0, top_p=0.95, seed=21)
    tokens, n_new = tiny.generate(prompt, **kw, **f)
    with torch.no_grad():
        want = _eager_loop(tiny, prompt, 12, 0.1, 0, 0.95, 21, f)
    assert tokens.tolist() == want and n_new.tolist() == [12] * 3
    assert not torch.equal(tokens, tiny.generate(prompt, **kw)[0])


def test_generate_with_filters_off_equals_the_call_without_them(tiny):
    V = tiny.cfg.vocab_size
    ids = torch.randint(0, V, (3, 20), generator=torch.Generator().manual_seed(6))
    for kw in (dict(temperature=0.8, top_k=0, top_p=0.9), dict(temperature=1.0, top_k=30, top_p=1.0),
               dict(temperature=0.0)):
        a, na = tiny.generate(ids, [20, 7, 13], max_new_tokens=16, seed=3, **kw)
        b, nb = tiny.generate(ids, [20, 7, 13], max_new_tokens=16, seed=3, **kw, **OFF)
        assert torch.equal(a, b) and torch.equal(na, nb)
    # the filters do nothing at temperature 0
    g, _ = tiny.generate(ids, max_new_tokens=8, temperature=0.0, typical_p=0.2, min_p=0.5, eta_cutoff=0.3)
    assert torch.equal(g, tiny.generate(ids, max_new_tokens=8, temperature=0.0)[0])


def test_argument_errors_name_the_argument(tiny):
    from adapcc_b200.ops import sample_tokens_
    from adapcc_b200.ops.sampling import check_filter_args

    ids = torch.zeros(2, 10, dtype=torch.long)
    bad = [("min_p", -0.1), ("min_p", 1.5), ("min_p", float("nan")), ("typical_p", 0.0), ("typical_p", 1.01),
           ("typical_p", "x"), ("epsilon_cutoff", 1.0), ("epsilon_cutoff", -1e-3), ("eta_cutoff", 1.0),
           ("eta_cutoff", -0.5), ("eta_cutoff", None)]
    z = torch.zeros(2, dtype=torch.int64)
    for name, v in bad:
        with pytest.raises(ValueError, match=f"generate: {name} must be"):
            tiny.generate(ids, **{name: v})
        with pytest.raises(ValueError, match=f"generate: {name} must be"):   # also before the lookup path
            tiny.generate(ids, temperature=0.0, prompt_lookup_num_tokens=2, **{name: v})
        with pytest.raises(ValueError, match=f"sample_reference: {name} must be"):
            sample_reference(torch.zeros(2, 5), 5, 1.0, 0, 1.0, z, z, 0, **{name: v})
        with pytest.raises(ValueError, match=f"sample_tokens_: {name} must be"):
            sample_tokens_(torch.zeros(2, 5), 5, 1.0, 0, 1.0, z, z.int(), z[:1].int(), 0, None, None, z.int(), z,
                           z[:, None], **{name: v})
    for ok in (dict(min_p=1.0), dict(typical_p=1.0), dict(epsilon_cutoff=0.0), dict(eta_cutoff=0.999)):
        check_filter_args("x", **{**OFF, **ok})


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_convai_passes_the_filters_through(tiny, monkeypatch):
    from adapcc_b200.eval import convai

    f = dict(min_p=0.01, typical_p=0.7, epsilon_cutoff=1e-4, eta_cutoff=2e-4)
    seen = []
    generate = tiny.generate

    def spy(*args, **kw):
        seen.append({k: kw[k] for k in f})
        return generate(*args, **kw)

    monkeypatch.setattr(tiny, "generate", spy)
    dialogs = [([[1, 2, 3]], [[3, 4, 5, 1, 2]]), ([[6]], [[7], [8, 9, 7]])]
    got = convai.sample_replies(tiny, _Tok(), dialogs, max_length=8, min_length=2, seeds=[4, 5], **f)
    assert seen == [f] and len(got) == 2
    # any filter sends F1 through the batched path (one example at a time by default), like the repetition controls
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"] * (j + 1), "candidates": ["x y"]}
                                                          for j in range(3)]}]
    seen.clear()
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, temperature=0.9, top_p=0.95, typical_p=0.5)
    assert len(seen) == 3 and all(s["typical_p"] == 0.5 for s in seen)
    w = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, temperature=0.9, top_p=0.95, typical_p=0.5,
                                batch_size=1)
    assert r == w and r["examples"] == 3
    seen.clear()
    convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5)               # sequential path: no generate call
    assert seen == []


def test_build_log_shows_sampler_and_filters_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_sample\.cu", log)
    assert re.search(r"Compiling entry function '\w*sample_tokens_kernel\w*' for 'sm_90a'", log)
    for fn in ("sample_tokens_kernel", "filter_row"):
        names = set(re.findall(r"Function properties for (\w*%s\w*)" % fn, log))
        assert names, fn
        for name in names:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
