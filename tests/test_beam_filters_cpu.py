"""Top-h and the truncation filters in every sampled decoder, on the CPU: ``ops.sampling.keep`` against HuggingFace's
warpers with ``min_tokens_to_keep`` in {1, 2, 3}, alone and chained in HuggingFace's order; ``keep`` at min_keep 1 and
with the filters off against the sets the sampler and beam sampling kept before it; beam sampling with each filter
against HuggingFace's ``generate(num_beams=K, do_sample=True)`` by a chi-square test; stochastic beam search's first
reply against ``generate``'s filtered law on an enumerable table; the off values, argument errors, the ConvAI
pass-through and the build of the filtered row kernels (nvcc only, no device)."""
import os
import re
import sys
from itertools import product

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.beam import StochasticBeamReference, sample_keep  # noqa: E402
from adapcc_b200.ops.sampling import keep, reference_row  # noqa: E402

OFF = dict(min_p=0.0, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0, top_h=0.0)
# each filter alone, then chains with top-k / top-p, in HuggingFace's order
CONFIGS = [dict(top_h=0.3), dict(top_h=0.8), dict(top_h=0.97), dict(min_p=0.2), dict(typical_p=0.4),
           dict(epsilon_cutoff=0.02), dict(eta_cutoff=0.02),
           dict(top_h=0.6, top_k=40, top_p=0.9, min_p=0.02, typical_p=0.9, epsilon_cutoff=1e-3, eta_cutoff=1e-3),
           dict(top_h=0.9, top_k=8, top_p=0.6, min_p=0.1, typical_p=0.5, epsilon_cutoff=0.01, eta_cutoff=0.05)]
REL = 1e-6


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _hf_kept(x, f, min_keep):
    """HuggingFace's warpers on the temperature-scaled fp32 values ``x``, in ``_get_logits_processor``'s order."""
    lp = pytest.importorskip("transformers.generation.logits_process")
    f = {**OFF, "top_k": 0, "top_p": 1.0, **f}
    chain = []
    if f["top_h"] > 0:
        chain.append(lp.TopHLogitsWarper(f["top_h"]))
    if f["top_k"] > 0:
        chain.append(lp.TopKLogitsWarper(f["top_k"], min_tokens_to_keep=min_keep))
    if f["top_p"] < 1:
        chain.append(lp.TopPLogitsWarper(f["top_p"], min_tokens_to_keep=min_keep))
    if f["min_p"] > 0:
        chain.append(lp.MinPLogitsWarper(f["min_p"], min_tokens_to_keep=min_keep))
    if f["typical_p"] < 1:
        chain.append(lp.TypicalLogitsWarper(f["typical_p"], min_tokens_to_keep=min_keep))
    if f["epsilon_cutoff"] > 0:
        chain.append(lp.EpsilonLogitsWarper(f["epsilon_cutoff"], min_tokens_to_keep=min_keep))
    if f["eta_cutoff"] > 0:
        chain.append(lp.EtaLogitsWarper(f["eta_cutoff"], min_tokens_to_keep=min_keep))
    scores = torch.tensor(x, dtype=torch.float64)[None]
    for w in chain:
        scores = w(None, scores)
    return (scores[0] > float("-inf")).numpy()


def _near_threshold(info, top_p):
    """True if a decision of ``keep`` sits within REL of its threshold: the running sums on either side of top-h's
    cut, a top-p tail or a truncation filter's quantity. (At top_h = 1 the last running sum is H itself, so every
    row would sit on the threshold.)"""
    th = info.get("top_h")
    if th is not None:
        c0 = int((th["cum"] <= th["thr"]).sum())
        near = th["cum"][max(c0 - 1, 0):c0 + 1]
        if np.any(np.abs(near - th["thr"]) <= REL * max(th["thr"], 1e-300)):
            return True
    tail = info["tail"][np.isfinite(info["tail"])]
    if top_p < 1 and np.any(np.abs(tail - info["pZ"]) <= REL * info["Z"]):
        return True
    for name, f in info["filters"].items():
        q = f["q"][np.isfinite(f["q"])]
        if name == "typical":
            q = q[q != f["thr"]]
            if np.any(np.abs(f["G"] - f["pZ"]) <= REL * f["Z"]):
                return True
        if np.any(np.abs(q - f["thr"]) <= REL * max(abs(f["thr"]), 1e-300)):
            return True
    return False


@pytest.mark.parametrize("min_keep", [1, 2, 3])
def test_keep_equals_huggingface_warpers_on_tie_free_rows(min_keep):
    pytest.importorskip("transformers")
    rng = np.random.default_rng(min_keep)
    checked = exempt = floored = 0
    for trial in range(360):
        V = int(rng.integers(4, 400))
        x = (rng.standard_normal(V) * rng.uniform(0.5, 6)).astype(np.float32)
        if np.unique(x).size != V:
            continue
        f = dict(CONFIGS[trial % len(CONFIGS)])
        top_p = f.pop("top_p", 1.0)
        kept, info = keep(x, f.pop("top_k", 0), top_p, min_keep, **f)
        if _near_threshold(info, top_p):
            exempt += 1
            continue
        th = info.get("top_h")
        if th is not None and int((th["cum"] <= th["thr"]).sum()) < min_keep:
            # HuggingFace's top-h has no keep count; here it keeps its first min_keep entries
            assert th["c"] == min_keep and kept.sum() >= min_keep
            floored += 1
            continue
        f = dict(CONFIGS[trial % len(CONFIGS)])
        assert np.array_equal(kept, _hf_kept(x, f, min_keep)), (trial, V, f)
        assert kept.sum() >= min(min_keep, V)
        checked += 1
    print(f"keep vs HuggingFace, min_keep {min_keep}: {checked} rows compared, {exempt} within {REL} of a threshold, "
          f"{floored} where top-h's keep count decided")
    assert checked >= 250


def test_top_h_hand_cases():
    # p = (0.5, 0.25, 0.125, 0.125): h = (0.347, 0.347, 0.260, 0.260), H = 1.213
    x = np.log(np.array([0.125, 0.5, 0.125, 0.25])).astype(np.float32)
    assert np.flatnonzero(keep(x, top_h=0.6)[0]).tolist() == [1, 3]          # 0.693 <= 0.728 < 0.953
    assert np.flatnonzero(keep(x, top_h=0.2)[0]).tolist() == [1]             # the first entry always stays
    assert np.flatnonzero(keep(x, top_h=0.2, min_keep=3)[0]).tolist() == [0, 1, 3]   # tie at 0.125: the lower id
    kept, info = keep(x, top_h=1.0)
    assert kept.sum() >= 3 and info["top_h"]["c"] == kept.sum()
    # only the 100 largest values are looked at
    y = np.concatenate([np.zeros(100), np.full(50, -0.5)]).astype(np.float32)
    assert np.flatnonzero(keep(y, top_h=1.0)[0]).max() < 100


def _old_sample_keep(x, top_k, top_p, min_keep):
    """Rule S2's kept set as beam sampling computed it before ``keep`` existed."""
    cand = x > -np.inf
    kept = cand.copy()
    n = int(cand.sum())
    if n == 0:
        return kept
    desc = np.sort(x[cand].astype(np.float64))[::-1]
    k = max(int(top_k), min_keep) if top_k > 0 else 0
    if 0 < k < n:
        kept &= x >= desc[k - 1]
    p = float(np.float32(top_p))
    if p < 1.0:
        xd = x.astype(np.float64)
        m = xd[kept].max()
        e = np.where(kept, np.exp(np.where(kept, xd - m, 0.0)), 0.0)
        order = np.argsort(-xd[kept], kind="stable")
        vals, csum = xd[kept][order], np.cumsum(e[kept][order])
        first = np.searchsorted(-vals, -vals, side="left")
        tail = np.full(x.size, np.inf)
        tail[np.flatnonzero(kept)[order]] = np.where(first > 0, csum[np.maximum(first - 1, 0)], 0.0)
        keep_p = ~(tail > p * float(e.sum()))
        keep_p |= x >= (desc[min_keep - 1] if min_keep < n else -np.inf)
        kept &= keep_p
    return kept


def test_keep_with_filters_off_is_the_old_top_k_top_p_set():
    rng = np.random.default_rng(5)
    for trial in range(300):
        V = int(rng.integers(1, 80))
        x = np.round(rng.standard_normal(V) * 2, 1).astype(np.float32)             # ties on purpose
        x[rng.random(V) < 0.1] = -np.inf
        k, p, mk = int(rng.integers(0, 6)), float(rng.choice([1.0, 0.9, 0.5, 1e-6])), int(rng.integers(1, 4))
        want = _old_sample_keep(x, k, p, mk)
        assert np.array_equal(keep(x, k, p, mk)[0], want), trial
        assert np.array_equal(sample_keep(x, k, p, mk), want), trial
        if mk == 1 and (x > -np.inf).any():
            assert np.array_equal(reference_row(x, 1.0, k, p, 0, 0)["kept"], want), trial


def test_off_values_change_no_set():
    rng = np.random.default_rng(6)
    for trial in range(100):
        x = (rng.standard_normal(int(rng.integers(2, 300))) * 3).astype(np.float32)
        for mk in (1, 2, 3):
            a, b = keep(x, 5, 0.8, mk)[0], keep(x, 5, 0.8, mk, **OFF)[0]
            assert np.array_equal(a, b)


# K, max_new, temperature, and one filter: the filters bite at temperature 0.5 on the tiny model
HF_FILTERS = [dict(min_p=0.4), dict(typical_p=0.3), dict(epsilon_cutoff=0.02), dict(eta_cutoff=0.05),
              dict(top_h=0.4)]


def _chi2_same(a, b):
    from scipy.stats import chi2_contingency

    keys = sorted(set(a) | set(b))
    if len(keys) < 2:
        return 1.0
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
        for name in ("ln_1", "ln_2"):
            sd[p + name + ".weight"], sd[p + name + ".bias"] = getattr(blk, name).weight, getattr(blk, name).bias
        for ours, theirs in (("c_attn", "attn.c_attn"), ("c_proj", "attn.c_proj"), ("c_fc", "mlp.c_fc"),
                             ("c_proj2", "mlp.c_proj")):
            sd[p + theirs + ".weight"] = getattr(blk, ours).weight.t()
            sd[p + theirs + ".bias"] = getattr(blk, ours).bias
    missing, _ = m.load_state_dict({k: v.detach().clone() for k, v in sd.items()}, strict=False)
    assert not [k for k in missing if not k.endswith(("attn.bias", "masked_bias", "lm_head.weight"))], missing
    m.tie_weights()
    return m


@pytest.mark.parametrize("f", HF_FILTERS)
def test_beam_sampling_with_filters_matches_huggingface(tiny, hf, f):
    K, n, T = 2, 2, 0.5
    prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 8), generator=torch.Generator().manual_seed(11))
    theirs, ours = [], []
    with torch.no_grad():
        for s in range(300):
            torch.manual_seed(s)
            out = hf.generate(prompt, attention_mask=torch.ones_like(prompt), num_beams=K, do_sample=True,
                              temperature=T, top_k=0, top_p=1.0, max_new_tokens=n, min_new_tokens=n,
                              eos_token_id=None, pad_token_id=0, length_penalty=0.0, early_stopping=False, **f)
            theirs.append(tuple(out[0, 8:].tolist()))
            tokens, n_new, _ = tiny.beam_search(prompt, num_beams=K, max_new_tokens=n, length_penalty=0.0,
                                                do_sample=True, temperature=T, seed=1000 + s, **f)
            ours.append(tuple(tokens[0].tolist()))
    p = _chi2_same(theirs, ours)
    print(f"beam sampling with {f} vs HuggingFace: {len(set(ours))} outcomes, p = {p:.3f}")
    assert len(set(ours)) > 1 and p > 1e-3


V, STEPS, STOP = 5, 3, 4


def _table(seed):
    rng = np.random.default_rng(seed)
    return {pre: (rng.standard_normal(V) * 1.5).astype(np.float32)
            for n in range(STEPS) for pre in product(range(V), repeat=n)}


def _law(table, f):
    """Every reply and its probability under generate's filtered draw (ops/sampling.py)."""
    law, live = {}, {(): 1.0}
    for t in range(STEPS):
        nxt = {}
        for pre, p in live.items():
            r = reference_row(table[pre], 1.0, 0, 1.0, 0, 0, **f)
            e = np.where(r["kept"], r["e"], 0.0)
            for i in np.flatnonzero(r["kept"]):
                q = p * e[i] / e.sum()
                if int(i) == STOP:
                    law[pre] = law.get(pre, 0.0) + q
                else:
                    nxt[pre + (int(i),)] = q
        live = nxt
    law.update(live)
    return law


@pytest.mark.parametrize("f", [dict(top_h=0.7), dict(min_p=0.05, eta_cutoff=0.01), dict(epsilon_cutoff=0.05)])
def test_stochastic_first_reply_follows_generate_filtered_law(f):
    from scipy.stats import chisquare

    table = _table(3)
    law = _law(table, f)
    assert 5 < len(law) < len(_law(table, {}))                                 # the filters bite, and leave a choice
    B, K = 2000, 2
    ref = StochasticBeamReference(B, K, STEPS, V, stop_ids=[STOP], seeds=list(range(5, 5 + B)), **f)
    pre = [()] * (B * K)
    for _ in range(STEPS):
        logits = np.stack([table.get(p, np.zeros(V, dtype=np.float32)) for p in pre])
        nxt, parent = ref.step(logits)
        pre = [pre[int(parent[r])] + (int(nxt[r]),) for r in range(B * K)]
        if ref.done.all():
            break
    tokens, n_new, log_probs, _, _ = ref.result()
    first = [tuple(tokens[b * K, :int(n_new[b * K])].tolist()) for b in range(B)]
    for b in range(B):
        assert first[b] in law and float(log_probs[b * K]) == pytest.approx(np.log(law[first[b]]), abs=1e-5)
    seqs = sorted(law)
    got = np.array([sum(1 for s in first if s == q) for q in seqs], dtype=np.float64)
    p = float(chisquare(got, np.array([law[q] for q in seqs]) * B).pvalue)
    print(f"stochastic beam search with {f}: {len(law)} sequences, first reply vs generate's law: p = {p:.3g}")
    assert p > 1e-3


def test_filters_at_off_values_equal_calls_without_them(tiny):
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, tiny.cfg.vocab_size, (2, 10), generator=g)
    a = tiny.generate(ids, max_new_tokens=6, temperature=0.9, top_k=20, seed=3)
    b = tiny.generate(ids, max_new_tokens=6, temperature=0.9, top_k=20, seed=3, **OFF)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    kw = dict(num_beams=3, max_new_tokens=5, temperature=0.8, top_p=0.9, seed=4, stop_ids=[7])
    a = tiny.beam_search(ids, do_sample=True, **kw)
    b = tiny.beam_search(ids, do_sample=True, **kw, **OFF)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    a = tiny.stochastic_beam_search(ids, **kw)
    b = tiny.stochastic_beam_search(ids, **kw, **OFF)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    # without do_sample the filters are ignored, as top-k and top-p are
    a = tiny.beam_search(ids, num_beams=3, max_new_tokens=5)
    b = tiny.beam_search(ids, num_beams=3, max_new_tokens=5, min_p=0.5, top_h=0.3, typical_p=0.2)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_filters_change_the_sampled_decoders(tiny):
    ids = torch.randint(0, tiny.cfg.vocab_size, (4, 10), generator=torch.Generator().manual_seed(3))
    kw = dict(num_beams=3, max_new_tokens=6, temperature=1.5, seed=4)
    assert not torch.equal(tiny.beam_search(ids, do_sample=True, **kw)[0],
                           tiny.beam_search(ids, do_sample=True, top_h=0.2, **kw)[0])
    assert not torch.equal(tiny.stochastic_beam_search(ids, **kw)[0],
                           tiny.stochastic_beam_search(ids, min_p=0.5, **kw)[0])
    gk = dict(max_new_tokens=8, temperature=1.5, top_p=1.0, seed=5)
    assert not torch.equal(tiny.generate(ids, **gk)[0], tiny.generate(ids, top_h=0.2, **gk)[0])


def test_argument_errors_name_the_argument(tiny):
    from adapcc_b200.ops.sampling import check_filter_args

    ids = torch.zeros(2, 10, dtype=torch.long)
    bad = [("top_h", -0.1), ("top_h", 1.5), ("top_h", float("nan")), ("top_h", "x"), ("min_p", 2.0),
           ("typical_p", 0.0), ("epsilon_cutoff", 1.0), ("eta_cutoff", -1.0)]
    for name, v in bad:
        with pytest.raises(ValueError, match=f"beam_search: {name} must be"):
            tiny.beam_search(ids, do_sample=True, **{name: v})
        with pytest.raises(ValueError, match=f"stochastic_beam_search: {name} must be"):
            tiny.stochastic_beam_search(ids, **{name: v})
    for name, v in bad[:4]:
        with pytest.raises(ValueError, match=f"generate: {name} must be"):
            tiny.generate(ids, **{name: v})
        with pytest.raises(ValueError, match=f"generate: {name} must be"):   # before the lookup path
            tiny.generate(ids, temperature=0.0, prompt_lookup_num_tokens=2, **{name: v})
    check_filter_args("x", **{**OFF, "top_h": 1.0})
    # group beam sampling stays unsupported
    with pytest.raises(ValueError, match="num_beam_groups > 1 needs do_sample=False"):
        tiny.beam_search(ids, num_beams=4, num_beam_groups=2, diversity_penalty=0.5, do_sample=True, min_p=0.1)


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_convai_passes_the_filters_to_beam_sampling(tiny, monkeypatch):
    from adapcc_b200.eval import convai

    f = dict(min_p=0.01, typical_p=0.7, epsilon_cutoff=1e-4, eta_cutoff=2e-4, top_h=0.9)
    seen = []
    beam_search = tiny.beam_search

    def spy(*args, **kw):
        seen.append({k: kw.get(k) for k in f})
        return beam_search(*args, **kw)

    monkeypatch.setattr(tiny, "beam_search", spy)
    dialogs = [([[1, 2, 3]], [[3, 4, 5, 1, 2]]), ([[6]], [[7], [8, 9, 7]])]
    got = convai.sample_replies(tiny, _Tok(), dialogs, max_length=6, min_length=2, seeds=[4, 5], num_beams=2,
                                beam_sample=True, **f)
    assert seen == [f] and len(got) == 2
    seen.clear()
    convai.sample_replies(tiny, _Tok(), dialogs, max_length=6, num_beams=2, **f)   # not sampled: no filters
    assert seen == [{k: None for k in f}]


def test_build_log_shows_filtered_row_kernels_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    for fn in ("sample_tokens_kernel", "sample_slots_kernel", "spec_slots_kernel", "beam_sample_rows_kernel",
               "beam_stochastic_rows_kernel", "top_h_row", "filter_row"):
        names = set(re.findall(r"Function properties for (\w*%s\w*)" % fn, log))
        assert names, fn
        for name in names:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
        if fn.endswith("_kernel"):                     # 1024-thread CTAs: at most 64 registers each
            regs = re.search(r"Compiling entry function '\w*%s\w*' for 'sm_90a'\n.*\n.*\n.*Used (\d+) registers"
                             % fn, log)
            assert regs and int(regs.group(1)) <= 64, (fn, regs and regs.group(0))
