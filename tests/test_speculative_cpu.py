"""Rejection-sampling verification of assisted generation on the CPU (``assistant_verification="rejection"``,
``ops/assisted.py``): the definition against HuggingFace's ``_speculative_sampling``, its acceptance rate, the joint
distribution of ``generate``'s tokens against plain sampling, hand cases, argument errors, the ConvAI and example
pass-through, and the new kernel's build (nvcc only, no device)."""
import os
import re
import runpy
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.assisted import draw_slot, spec_slot, spec_slots  # noqa: E402
from adapcc_b200.ops.lookup import lookup_accept, mean_tokens_per_step  # noqa: E402
from adapcc_b200.ops.sampling import philox4x32_10, uniform  # noqa: E402

SEEDS = 20000


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


@pytest.fixture(scope="module")
def noisy(tiny):
    """The target's weights plus noise: a draft close to, but not equal to, the target."""
    m = GPT2DoubleHeads(GPT2Config.tiny()).eval()
    g = torch.Generator().manual_seed(9)
    m.load_state_dict({k: v + 0.3 * v.std() * torch.randn(v.shape, generator=g) if v.is_floating_point() and v.numel() > 1
                       else v for k, v in tiny.state_dict().items()})
    return m


def _chi2_same(a, b):
    """p-value of the two-sample chi-square test that the outcome lists ``a`` and ``b`` come from one distribution."""
    from scipy.stats import chi2_contingency

    keys = sorted(set(a) | set(b))
    ca, cb = {}, {}
    for x in a:
        ca[x] = ca.get(x, 0) + 1
    for x in b:
        cb[x] = cb.get(x, 0) + 1
    return float(chi2_contingency(np.array([[ca.get(k, 0) for k in keys], [cb.get(k, 0) for k in keys]]))[1])


def _round(P, Q, drafts, seed, L=11):
    """(accepted count, last token) of one round of the definition on fixed log-probability rows: P [k+1, V] the
    model's slots, Q [k, V] the draft's steps."""
    for j, d in enumerate(drafts):
        r = spec_slot(P[j], Q[j], d, 1.0, 0, 1.0, seed, L, 0, j)
        if not r["accept"]:
            return j, r["t"]
    return len(drafts), spec_slot(P[len(drafts)], None, 0, 1.0, 0, 1.0, seed, L, 0, len(drafts))["g"]


def _rows(V, k, seed):
    g = np.random.default_rng(seed)
    P = g.dirichlet(np.full(V, 0.7), k + 1)
    Q = np.clip(P[:k] + g.normal(0, 0.15, (k, V)), 0.01, None)
    Q /= Q.sum(1, keepdims=True)
    return P, Q


def test_philox_words():
    """``uniform``'s words are Philox4x32-10's outputs; word 0 is the existing draw."""
    w = philox4x32_10((5, 0, 0, 0), (7, 0))
    for i in range(4):
        assert uniform(7, 5, i) == (w[i] >> 8) * 2.0 ** -24
    assert uniform(7, 5) == uniform(7, 5, 0)


def test_definition_matches_huggingface_speculative_sampling():
    hf = pytest.importorskip("transformers.generation.utils")
    V, k = 6, 3
    P, Q = _rows(V, k, 0)
    drafts = [int(np.random.default_rng(1 + j).choice(V, p=Q[j])) for j in range(k)]
    lp, lq = np.log(P).astype(np.float32), np.log(Q).astype(np.float32)
    cand = torch.tensor([[0] + drafts])
    new_logits, cand_logits = torch.from_numpy(lp)[None], torch.from_numpy(lq)[None]
    theirs = []
    for s in range(SEEDS):
        torch.manual_seed(s)
        tok, n = hf._speculative_sampling(cand, cand_logits, k, new_logits, False)
        theirs.append((int(n), int(tok[0, -1])))
    ours = [_round(lp, lq, drafts, s) for s in range(SEEDS)]
    p = _chi2_same(theirs, ours)
    print(f"HuggingFace vs definition: p = {p:.3g}, {len(set(ours))} outcomes")
    assert p > 1e-3


def test_acceptance_rate_is_the_overlap():
    V = 8
    P, Q = _rows(V, 1, 5)
    lp, lq = np.log(P).astype(np.float32), np.log(Q).astype(np.float32)
    want = float(np.minimum(P[0], Q[0]).sum())
    hits = 0
    for s in range(SEEDS):
        d = draw_slot(lq[0], 1.0, 0, 1.0, s, 11, 0, 0)                  # the draft's own draw of d_1
        hits += spec_slot(lp[0], lq[0], d, 1.0, 0, 1.0, s, 11, 0, 0)["accept"]
    sigma = (want * (1 - want) / SEEDS) ** 0.5
    print(f"acceptance {hits / SEEDS:.4f}, overlap {want:.4f}")
    assert abs(hits / SEEDS - want) <= 4 * sigma


def _joint(model, draft, seed, **kw):
    ids = torch.tensor([[5, 17, 3, 9]]).repeat(4000, 1)
    extra = {} if draft is None else dict(assistant_model=draft, num_assistant_tokens=2,
                                          assistant_verification="rejection")
    tok, _ = model.generate(ids, max_new_tokens=4, temperature=1.0, top_k=4, top_p=1.0, seed=seed, **extra, **kw)
    return [tuple(r[:3]) for r in tok.tolist()]


def test_generate_tokens_are_distributed_as_plain_sampling(tiny, noisy):
    """Token 1 comes from the prefill, tokens 2 and 3 from accepted drafts or residual draws; their joint distribution
    (at most 64 outcomes) matches plain sampling's. Independent seeds for the two samples."""
    ours = _joint(tiny, noisy, 0)
    plain = _joint(tiny, None, 1 << 20)
    st = tiny.assist_stats
    p = _chi2_same(ours, plain)
    print(f"rejection vs plain: p = {p:.3g}, {len(set(ours))} outcomes, "
          f"{mean_tokens_per_step(st['emitted'], st['steps']):.2f} tokens per step")
    assert p > 1e-3


# ---- hand cases ------------------------------------------------------------------------------------------------------
def test_equal_distributions_accept_every_draft():
    g = np.random.default_rng(2)
    for s in range(200):
        l = (g.standard_normal(50) * 2).astype(np.float32)
        kw = dict(min_p=0.01) if s % 2 else {}
        d = draw_slot(l, 0.8, 10, 0.9, s, 4, 0, 0, **kw)
        assert spec_slot(l, l, d, 0.8, 10, 0.9, s, 4, 0, 0, **kw)["accept"]


def test_a_draft_the_model_cannot_draw_is_never_accepted_nor_emitted():
    q = np.zeros(20, dtype=np.float32)
    q[7] = 3.0                                                          # the draft prefers id 7
    p = np.linspace(0, 1, 20).astype(np.float32)
    p[7] = -np.inf                                                      # the model never draws it
    for s in range(300):
        r = spec_slot(p, q, 7, 1.0, 0, 1.0, s, 4, 0, 0)
        assert not r["accept"] and r["t"] != 7 and r["P"][7] == 0
    p[7] = 0.0                                                          # outside the model's top-k: P = 0 as well
    for s in range(300):
        r = spec_slot(p, q, 7, 1.0, 5, 1.0, s, 4, 0, 0)
        assert not r["accept"] and r["t"] != 7


def test_cap_and_stop_ids_among_drafts():
    B, k, V = 3, 3, 30
    S = k + 1
    g = torch.Generator().manual_seed(0)
    logits = torch.randn(B * S, V, generator=g)
    ql = logits.view(B, S, V)[:, :k].clone()                            # Q = P: every real draft is accepted
    lens, emitted = torch.tensor([4, 4, 4]), torch.tensor([1, 1, 1])
    done, nq = torch.tensor([0, 0, 1]), torch.tensor([4, 2, 0])         # row 1: r = 1; row 2: done
    ids = torch.zeros(B, S, dtype=torch.int64)
    for b in range(2):
        for j in range(k):
            ids[b, j + 1] = draw_slot(ql[b, j].numpy(), 1.0, 0, 1.0, 3 + b, 4, 1, j)
    gd, acc, last = spec_slots(logits, ql, V, 1.0, 0, 1.0, [3, 4, 5], lens, emitted, done, nq, ids.view(-1))
    assert acc[0, :3].tolist() == [1, 1, 1] and acc[1].tolist() == [1, 0, 0, 0] and (gd[2] == -1).all()
    assert last[0, 3] == gd[0, 3] and last[1, 1] == gd[1, 1] and gd[1, 2] == -1   # past the cap: nothing decided
    seq = torch.zeros(B, 40, dtype=torch.int32)
    tokens = torch.full((B, 20), -1, dtype=torch.int64)
    steps = torch.zeros(B, dtype=torch.int32)
    stop = [int(ids[0, 2])] if int(ids[0, 2]) != int(ids[0, 1]) else []
    lookup_accept(None, V, ids.view(-1), nq, seq, lens, emitted, done, tokens, steps, stop_ids=stop,
                  drawn=torch.from_numpy(last), accepted=torch.from_numpy(acc))
    if stop:                                                            # a stop id among the accepted drafts ends row 0
        assert tokens[0, 1:4].tolist() == [int(ids[0, 1]), -1, -1] and int(done[0]) == 1 and int(emitted[0]) == 3
    assert tokens[1, 1:3].tolist() == [int(ids[1, 1]), int(gd[1, 1])] and int(emitted[1]) == 3
    assert int(done[1]) == 0 and int(steps[2]) == 0


def test_temperature_zero_is_the_greedy_path(tiny, noisy):
    ids, lengths = torch.randint(0, 40, (4, 12), generator=torch.Generator().manual_seed(3)), [12, 5, 9, 1]
    kw = dict(max_new_tokens=20, temperature=0.0, assistant_model=noisy, num_assistant_tokens=3)
    want, n_want = tiny.generate(ids, lengths, **kw)
    st = {key: v.clone() if torch.is_tensor(v) else v for key, v in tiny.assist_stats.items()}
    got, n_got = tiny.generate(ids, lengths, assistant_verification="rejection", **kw)
    assert torch.equal(got, want) and torch.equal(n_got, n_want)
    assert set(tiny.assist_stats) == set(st)
    for key, v in st.items():
        assert torch.equal(tiny.assist_stats[key], v) if torch.is_tensor(v) else tiny.assist_stats[key] == v


def test_rejection_accepts_at_least_as_much_as_coupled(tiny, noisy):
    ids = torch.randint(0, 40, (6, 10), generator=torch.Generator().manual_seed(4))
    rates = {}
    for rule in ("coupled", "rejection"):
        tiny.generate(ids, max_new_tokens=30, temperature=0.9, top_p=0.95, seed=7, assistant_model=noisy,
                      num_assistant_tokens=4, assistant_verification=rule)
        rates[rule] = mean_tokens_per_step(tiny.assist_stats["emitted"], tiny.assist_stats["steps"])
    print(rates)
    assert rates["rejection"] >= rates["coupled"]


def test_stop_and_suppressed_ids_with_min_new_tokens(tiny, noisy):
    ids = torch.randint(0, 40, (5, 8), generator=torch.Generator().manual_seed(6))
    kw = dict(max_new_tokens=20, temperature=1.0, top_k=8, seed=2, assistant_model=noisy, num_assistant_tokens=3,
              assistant_verification="rejection")
    free, _ = tiny.generate(ids, **kw)
    stop = sorted({int(free[0, 4]), int(free[1, 2])})
    got, n_got = tiny.generate(ids, stop_ids=stop, suppress_ids=stop, min_new_tokens=3, **kw)
    for b in range(5):
        row = got[b, :int(n_got[b])].tolist()
        assert -1 not in row and not set(row[:3]) & set(stop) and not set(row) & set(stop)
        assert (got[b, int(n_got[b]):] == -1).all()


# ---- arguments and pass-through --------------------------------------------------------------------------------------
def test_bad_verification_is_rejected_before_anything_runs(tiny, noisy, monkeypatch):
    from adapcc_b200.eval import convai

    ids = torch.zeros(2, 5, dtype=torch.long)
    calls = []
    monkeypatch.setattr(GPT2DoubleHeads, "hidden", lambda *a, **k: calls.append(1))
    for kw in (dict(assistant_model=noisy, assistant_verification="speculative"),
               dict(assistant_model=noisy, assistant_verification=None),
               dict(assistant_verification="rejection"),
               dict(assistant_verification="rejection", prompt_lookup_num_tokens=2, temperature=0.0)):
        with pytest.raises(ValueError, match="assistant_verification"):
            tiny.generate(ids, **kw)
    dialogs = [([[1, 2, 3]], [[3, 4, 5, 1, 2]])]
    with pytest.raises(ValueError, match="assistant_verification"):
        convai.sample_replies(tiny, _Tok(), dialogs, max_length=4, num_beams=2, assistant_verification="rejection")
    with pytest.raises(ValueError, match="assistant_verification"):
        convai.evaluate_dialogs(tiny, _Tok(), [], "f1", assistant_verification="nope")
    assert not calls
    monkeypatch.undo()
    tiny.generate(ids, max_new_tokens=3, assistant_model=noisy, assistant_verification="coupled")


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_convai_and_example_pass_the_rule_through(tiny, noisy, monkeypatch):
    from adapcc_b200 import eval as ev
    from adapcc_b200.eval import convai

    seen = []
    generate = GPT2DoubleHeads.generate

    def spy(self, *a, **kw):
        seen.append(kw.get("assistant_verification"))
        return generate(self, *a, **kw)

    monkeypatch.setattr(GPT2DoubleHeads, "generate", spy)
    dialogs = [([[1, 2, 3]], [[3, 4, 5, 1, 2]]), ([[6]], [[7], [8, 9, 7]])]
    kw = dict(max_length=8, min_length=2, seeds=[4, 5], assistant_model=noisy, num_assistant_tokens=3)
    got = convai.sample_replies(tiny, _Tok(), dialogs, assistant_verification="rejection", **kw)
    assert seen == ["rejection"] and len(got) == 2
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, assistant_model=noisy, num_assistant_tokens=2,
                            assistant_verification="rejection")
    assert seen[-1] == "rejection"
    monkeypatch.undo()
    # the example's flag reaches evaluate_dialogs
    calls = []
    monkeypatch.setattr(ev, "load_model_from_checkpoint", lambda *a, **k: (tiny, _Tok()))
    monkeypatch.setattr(ev, "evaluate_dialogs", lambda *a, **k: calls.append(k) or {})
    for flag in ("rejection", "coupled"):
        monkeypatch.setattr(sys, "argv", ["eval_gpt2_convai.py", "--model_checkpoint", "m.pt", "--eval_type", "f1",
                                          "--assistant_checkpoint", "d.pt", "--assistant_verification", flag,
                                          "--synthetic_dialogs", "8", "--device", "cpu"])
        runpy.run_path(os.path.join(ROOT, "examples", "eval_gpt2_convai.py"), run_name="__main__")
        assert calls[-1]["assistant_verification"] == flag


def test_build_log_shows_spec_slots_kernel_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    for src in ("ops_sample", "ops_lookup"):
        assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*%s\.cu" % src, log)
    for kernel in ("spec_slots_kernel", "sample_slots_kernel", "sample_tokens_kernel", "lk_accept_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
