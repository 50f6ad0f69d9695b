"""Diverse (group) beam search on the GPU: ``beam_step_`` on a ``BeamState(..., groups=G)`` against the fp64 definition
(``ops.beam.GroupBeamReference``) with the near-tie exemption of test_gpu_beam.py widened by the penalty's roundings,
group 0 against plain ``beam_step_`` bit for bit, items alone, ``num_beam_groups=1`` against the call without it, and
GPT-2 small against an eager loop of the definition."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # unit roundoff of fp32


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _tol(V, cs, lam, K):
    """test_gpu_beam.py's bound on two candidate scores c = s + ((l - m) - logf(Z)) (M = 1 + max |c|), plus the
    penalty's two roundings per score: fl32(lam * n) within u lam K and fl32(c - that) within u M."""
    M = 1.0 + max(abs(c) for c in cs) if cs else 1.0
    return 2.0 * (4.0 * M + math.ceil(V / 512) + 14) * U32 + 2.0 * (lam * K + M) * U32


def _near(vals, tol):
    v = np.sort(np.asarray([x for x in vals if np.isfinite(x)], dtype=np.float64))
    d = np.diff(v)
    return bool(((d > 0) & (d <= tol)).any())


def _spy(ref, K, n_stop):
    """Record each group ranking the reference walks per item: ``(g, its first K·(K + n_stop) scores, the score of
    its first non-stop candidate or None)``."""
    seen = {}
    orig = ref.group_ranking

    def spy(b, g, logits, step, taken):
        r = orig(b, g, logits, step, taken)
        s0 = next((c for c, _, i in r if i not in ref.stop), None)
        seen.setdefault(b, []).append((g, [c for c, _, _ in r[:K * (K + n_stop)]], s0))
        return r

    ref.group_ranking = spy
    return seen


def _check_step(dev, B, K, G, V, step, max_new, alpha, lam, stop, suppress, min_new, seed):
    from adapcc_b200.ops import BeamState, beam_step_
    from adapcc_b200.ops.beam import GroupBeamReference

    rng = np.random.default_rng(seed)
    Kg = K // G
    st = BeamState(B, K, max_new, alpha, dev, groups=G)
    scores = -np.abs(rng.standard_normal((B, G, Kg)) * 3 * (step + 1)).astype(np.float32)
    scores = -np.sort(-scores, axis=2)
    if step == 0:
        scores[:, :, 1:] = -np.inf
    scores[rng.random((B, G, Kg)) < 0.1] = -np.inf                   # some dead beams
    gdone = rng.random((B, G)) < 0.15                                 # some done groups: dead rows
    scores[gdone] = -np.inf
    scores = scores.reshape(B, K)
    logits = (rng.standard_normal((B * K, V)) * 3).astype(np.float32)
    for b in range(0, B, 3):                                         # planted ties: within a row, across rows and
        r = b * K                                                    # across groups (rows 0 and Kg of the item)
        top = np.argsort(-logits[r])[:6]
        logits[r, top[2]] = logits[r, top[1]]
        logits[r + Kg] = logits[r]
        scores[b, Kg] = scores[b, 0]
        if Kg > 1:
            logits[r + 1] = logits[r]
            scores[b, 1] = scores[b, 0]
    fin_count = rng.integers(0, Kg + 1, (B, G))
    fin_score = -np.sort(np.abs(rng.standard_normal((B, G, Kg)) * 4), axis=2).astype(np.float32)
    fin_n = rng.integers(0, max(1, step), (B, G, Kg)).astype(np.int32)
    fin_src = rng.integers(0, K, (B, G, Kg)).astype(np.int32)
    st.scores.copy_(torch.from_numpy(scores.reshape(-1)))
    st.step.fill_(step)
    st.group_done.copy_(torch.from_numpy(gdone.astype(np.int32).reshape(-1)))
    st.fin_count.copy_(torch.from_numpy(fin_count.astype(np.int32).reshape(-1)))
    st.fin_score.copy_(torch.from_numpy(fin_score.reshape(B, K)))
    st.fin_n.copy_(torch.from_numpy(fin_n.reshape(B, K)))
    st.fin_src.copy_(torch.from_numpy(fin_src.reshape(B, K)))
    i32 = dict(dtype=torch.int32, device=dev)
    beam_step_(torch.from_numpy(logits).to(dev), V, st, min_new, torch.tensor(suppress, **i32) if suppress else None,
               torch.tensor(stop, **i32) if stop else None, diversity_penalty=lam)
    torch.cuda.synchronize()
    ref = GroupBeamReference(B, K, max_new, V, alpha, stop, suppress, min_new, num_beam_groups=G,
                             diversity_penalty=lam)
    ref.scores = scores.astype(np.float64)
    ref.n_steps = step
    ref.group_done[:] = gdone
    ref.stopped[:] = gdone
    for b in range(B):
        for g in range(G):
            ref.fin[b][g] = [(float(fin_score[b, g, k]), int(fin_n[b, g, k]), int(fin_src[b, g, k]))
                             for k in range(fin_count[b, g])]
    seen = _spy(ref, K, len(stop))
    nxt, parent = ref.step(logits)
    got = dict(nxt=st.next_ids.cpu().view(B, K), parent=st.parent.cpu().view(B, K), scores=st.scores.cpu().view(B, K),
               done=st.done.cpu(), gdone=st.group_done.cpu().view(B, G), count=st.fin_count.cpu().view(B, G),
               fs=st.fin_score.cpu().view(B, G, Kg), fn=st.fin_n.cpu().view(B, G, Kg),
               src=st.fin_src.cpu().view(B, G, Kg), ht=st.hist_tok.cpu()[step].view(B, K),
               hb=st.hist_back.cpu()[step].view(B, K))
    assert int(st.step) == step + 1
    exempt = 0
    for b in range(B):
        rankings = seen.get(b, [])
        allc = [c for _, r, _ in rankings for c in r] + [float(s) for s in scores[b] if np.isfinite(s)]
        tol = _tol(V, allc, ref.lam, K)
        same = (got["nxt"][b].tolist() == nxt.view(B, K)[b].tolist()
                and got["parent"][b].tolist() == parent.view(B, K)[b].tolist()
                and int(got["done"][b]) == int(ref.done[b])
                and got["gdone"][b].tolist() == ref.group_done[b].astype(int).tolist()
                and np.allclose(got["scores"][b].double().numpy(), ref.scores[b], rtol=0, atol=tol))
        if same and not ref.done[b] and not all(gdone[b]):
            live = [g for g in range(G) if not gdone[b, g]]
            same = (got["ht"][b].view(G, Kg)[live].tolist() == ref.hist_tok[step, b].reshape(G, Kg)[live].tolist()
                    and got["hb"][b].view(G, Kg)[live].tolist()
                    == ref.hist_back[step, b].reshape(G, Kg)[live].tolist())
        for g in range(G):
            fin = ref.fin[b][g]
            same = same and (int(got["count"][b, g]) == len(fin)
                             and [(int(got["fn"][b, g, k]), int(got["src"][b, g, k])) for k in range(len(fin))]
                             == [f[1:] for f in fin]
                             and np.allclose(got["fs"][b, g, :len(fin)].double().numpy(), [f[0] for f in fin],
                                             rtol=0, atol=4 * tol))
        if same:
            continue
        # the only allowed cause: two decision values (ranked candidates, normalised scores, a done bound) within the
        # fp32 error of each other
        pens = [ref.penalty(L) for L in range(1, max_new + 1)]
        lp = 4 * tol / min(pens)
        near = any(_near(r, tol) for _, r, _ in rankings)
        for g in range(G):
            fin = ref.fin[b][g]
            near = near or _near([f[0] for f in fin] + [float(x) for x in fin_score[b, g, :fin_count[b, g]]], lp)
        for g, _, s0 in rankings:                                   # the done bound of each group that selected
            fin = ref.fin[b][g]
            if s0 is not None and len(fin) == Kg:
                near = near or _near([fin[-1][0], s0 / pens[-1 if alpha > 0 else min(step + 1, max_new - 1)]], lp)
        assert near, (B, K, G, V, step, b, got["nxt"][b].tolist(), nxt.view(B, K)[b].tolist())
        exempt += 1
    return B, exempt


CASES = [  # B, K, G, V, step, max_new, alpha, lambda, stop, suppress, min_new
    (32, 16, 2, 50262, 2, 16, 1.0, 0.5, [50256, 11, 13, 30, 0, 1, 2, 3], list(range(50257, 50262)), 3),
    (32, 16, 4, 50262, 0, 8, -0.5, 2.0, [50256], list(range(50257, 50262)), 1),
    (32, 16, 8, 50262, 5, 8, 2.0, 0.25, [50256, 7], [], 0),
    (32, 16, 16, 50262, 1, 4, 0.7, 1.0, [50256, 5, 6, 7], [5, 6], 2),
    (512, 4, 2, 3001, 3, 20, 1.0, 0.5, [7, 11], [], 0),
    (512, 8, 4, 1003, 6, 8, 0.0, 3.0, [1, 2, 3, 4, 5, 6, 7, 8], [], 0),
    (384, 6, 3, 64, 1, 4, 0.7, 0.01, [3, 9], [3, 9], 2),
    (400, 2, 2, 700, 0, 8, 1.0, 1e-3, [0], [], 0),
]


def test_group_beam_step_matches_fp64_definition(dev):
    items = exempt = 0
    for i, case in enumerate(CASES):
        n, e = _check_step(dev, *case, seed=i)
        items += n
        exempt += e
    print(f"group beam_step vs fp64: {items} items, {exempt} exempt")
    assert items >= 1800 and exempt <= items // 50


def _as_bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def test_group_zero_is_plain_beam_step_bit_for_bit(dev):
    """Group 0 of a G-group step against beam_step_ with K / G beams on the same rows, step after step: every state
    tensor as int bits (a done group's scores are -inf)."""
    from adapcc_b200.ops import BeamState, beam_step_

    B, K, V, n = 6, 8, 50257, 10
    g = torch.Generator(device=dev).manual_seed(5)
    stop = torch.tensor([11, 50256], dtype=torch.int32, device=dev)
    sup = torch.tensor([5, 6, 11], dtype=torch.int32, device=dev)
    for G in (2, 4, 8):
        Kg = K // G
        rows = torch.tensor([b * K + k for b in range(B) for k in range(Kg)], device=dev)
        full = BeamState(B, K, n, 0.6, dev, groups=G)
        plain = BeamState(B, Kg, n, 0.6, dev)
        for t in range(n):
            lg = torch.randn(B * K, V, device=dev, generator=g) * 4
            lg[:, 11] += 6.0                                         # the stop id competes
            beam_step_(lg, V, full, 2, sup, stop, diversity_penalty=0.75)
            beam_step_(lg[rows].contiguous(), V, plain, 2, sup, stop)
            torch.cuda.synchronize()
            fs, ps = full.scores.view(B, K)[:, :Kg], plain.scores.view(B, Kg)
            gd = full.group_done.view(B, G)[:, 0]
            assert torch.equal(gd, plain.done), (G, t)
            want = torch.where(plain.done[:, None].bool(), torch.full_like(ps, float("-inf")), ps)
            assert torch.equal(_as_bits(fs), _as_bits(want)), (G, t)
            base_f = torch.arange(B, device=dev)[:, None] * K
            base_p = torch.arange(B, device=dev)[:, None] * Kg
            assert torch.equal(full.next_ids.view(B, K)[:, :Kg], plain.next_ids.view(B, Kg)), (G, t)
            assert torch.equal(full.parent.view(B, K)[:, :Kg] - base_f, plain.parent.view(B, Kg) - base_p), (G, t)
            assert torch.equal(full.hist_tok.view(n, B, K)[:, :, :Kg], plain.hist_tok.view(n, B, Kg)), (G, t)
            assert torch.equal(full.hist_back.view(n, B, K)[:, :, :Kg], plain.hist_back.view(n, B, Kg)), (G, t)
            for name in ("fin_score", "fin_n", "fin_src"):
                a, p = getattr(full, name).view(B, G, Kg)[:, 0], getattr(plain, name).view(B, Kg)
                assert torch.equal(_as_bits(a), _as_bits(p)), (G, t, name)
            assert torch.equal(full.fin_count.view(B, G)[:, 0], plain.fin_count), (G, t)
            assert int(full.step) == int(plain.step) == t + 1
        assert int(full.fin_count.sum()) > 0 and int(full.group_done.sum()) > 0, G


def test_group_beam_step_item_alone_equals_item_in_batch(dev):
    from adapcc_b200.ops import BeamState, beam_step_

    B, K, G, V, n = 6, 8, 4, 50257, 8
    g = torch.Generator(device=dev).manual_seed(3)
    stop = torch.tensor([11, 50256], dtype=torch.int32, device=dev)
    sup = torch.tensor([5, 6, 11], dtype=torch.int32, device=dev)
    steps = [torch.randn(B * K, V, device=dev, generator=g) * 4 for _ in range(n)]
    for lg in steps:
        lg[:, 11] += 6.0
    full = BeamState(B, K, n, 0.6, dev, groups=G)
    alone = [BeamState(1, K, n, 0.6, dev, groups=G) for _ in range(B)]
    for lg in steps:
        beam_step_(lg, V, full, 2, sup, stop, diversity_penalty=0.5)
        for b in range(B):
            beam_step_(lg[b * K:(b + 1) * K].contiguous(), V, alone[b], 2, sup, stop, diversity_penalty=0.5)
    torch.cuda.synchronize()
    for b in range(B):
        a = alone[b]
        rows, grp = slice(b * K, (b + 1) * K), slice(b * G, (b + 1) * G)
        assert torch.equal(full.scores[rows].view(torch.int32), a.scores.view(torch.int32)), b
        assert torch.equal(full.next_ids[rows], a.next_ids) and torch.equal(full.parent[rows] - b * K, a.parent), b
        assert torch.equal(full.hist_tok[:, rows], a.hist_tok) and torch.equal(full.hist_back[:, rows], a.hist_back)
        assert torch.equal(full.fin_score[b].view(torch.int32), a.fin_score[0].view(torch.int32)), b
        assert torch.equal(full.fin_n[b], a.fin_n[0]) and torch.equal(full.fin_src[b], a.fin_src[0]), b
        assert torch.equal(full.fin_count[grp], a.fin_count) and torch.equal(full.group_done[grp], a.group_done), b
        assert int(full.done[b]) == int(a.done[0]), b
    assert int(full.fin_count.sum()) > 0


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def test_one_group_equals_the_call_without_groups(dev):
    from adapcc_b200.runtime.native import load_library

    lib = load_library(build_if_missing=False)
    m = _gpt2_small(dev)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(4)
    ids = torch.randint(0, V, (4, 50), device=dev, generator=g)
    kw = dict(num_beams=8, max_new_tokens=16, stop_ids=[int(ids[0, 3])], num_return_sequences=8)
    c0 = lib.adapcc_launch_count()
    want = m.beam_search(ids, [50, 7, 31, 2], **kw)
    c1 = lib.adapcc_launch_count()
    got = m.beam_search(ids, [50, 7, 31, 2], **kw, num_beam_groups=1, diversity_penalty=0.0)
    c2 = lib.adapcc_launch_count()
    assert all(torch.equal(_as_bits(a), _as_bits(b)) for a, b in zip(want, got))
    assert c2 - c1 == c1 - c0 > 0


def _graph_against_eager(dev, B, K, G, n, alpha, lam, lengths, ngram, seed):
    """The graph path against an eager loop of the same decode step and LM head, selecting with GroupBeamReference in
    fp64 (after penalize_repeats_reference on each beam's own sequence when ``ngram`` > 0) and reordering the cache by
    torch indexing. An item may differ only if one of its group rankings had two candidates within the bound."""
    from adapcc_b200.ops import lm_head_logits_
    from adapcc_b200.ops.beam import GroupBeamReference
    from adapcc_b200.ops.repeats import penalize_repeats_reference

    m = _gpt2_small(dev, seed=seed)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(seed + 10)
    T = max(lengths)
    ids = torch.randint(0, 400 if ngram else V, (B, T), device=dev, generator=g)
    stop = [int(ids[0, 0]), int(ids[1, 1])]
    kw = dict(num_beams=K, max_new_tokens=n, length_penalty=alpha, stop_ids=stop, num_beam_groups=G,
              diversity_penalty=lam, num_return_sequences=K, no_repeat_ngram_size=ngram)
    tokens, n_new, scores = m.beam_search(ids, lengths, **kw)
    again = m.beam_search(ids, lengths, **kw)
    assert all(torch.equal(_as_bits(a), _as_bits(b)) for a, b in zip((tokens, n_new, scores), again))
    w = m.wte.weight
    with torch.no_grad():
        last = torch.tensor(lengths, device=dev) - 1
        pre = m.new_cache(B, T)
        h = m.hidden(ids, None, cache=pre, lengths=lengths)[torch.arange(B, device=dev), last]
        cache = m.new_cache(B * K, T + n)
        cache.reset([x for x in lengths for _ in range(K)], T)
        cache.k[:, :, :, :T].copy_(pre.k.repeat_interleave(K, dim=1))
        cache.v[:, :, :, :T].copy_(pre.v.repeat_interleave(K, dim=1))
        h = h.repeat_interleave(K, dim=0).contiguous()
        ref = GroupBeamReference(B, K, n, V, alpha, stop, num_beam_groups=G, diversity_penalty=lam)
        seen = _spy(ref, K, len(stop))
        logits = torch.empty(B * K, w.shape[0], dtype=torch.float32, device=dev)
        seqs = [ids[r // K, :lengths[r // K]].tolist() for r in range(B * K)]
        for i in range(n):
            if i:
                h = m.decode_step(nxt.to(dev), None, cache)
                seqs = [seqs[int(pr)] + [int(t)] for pr, t in zip(parent, nxt)]
            lm_head_logits_(h, w, logits)
            lc = (penalize_repeats_reference(logits, seqs, V, 1.0, ngram) if ngram else logits).cpu().numpy()
            nxt, parent = ref.step(lc)
            rows = parent.to(dev)
            cache.k.copy_(cache.k[:, rows])
            cache.v.copy_(cache.v[:, rows])
            if ref.done.all():
                break
    rt, rn, rs = ref.result(K)
    exempt = 0
    for b in range(B):
        r = slice(b * K, (b + 1) * K)
        if torch.equal(tokens[r].cpu(), rt[r]) and torch.equal(n_new[r].cpu(), rn[r]):
            assert scores[r].cpu().tolist() == pytest.approx(rs[r].tolist(), abs=1e-3), b
            continue
        near = any(_near(cs, _tol(V, cs, ref.lam, K)) for _, cs, _ in seen.get(b, []))
        fs = [f[0] for fin in ref.fin[b] for f in fin]              # the merge order of the groups' hypotheses
        near = near or _near(fs, 4 * _tol(V, fs, ref.lam, K))
        assert near, b
        exempt += 1
    print(f"group beam_search (G={G}, ngram={ngram}) graph vs eager fp64 loop: {B} items, {exempt} exempt")
    assert exempt <= B // 2


def test_group_beam_search_graph_equals_eager_reference_loop(dev):
    _graph_against_eager(dev, 6, 8, 4, 20, 0.8, 0.5, [64, 17, 120, 40, 5, 99], 0, seed=1)


def test_group_beam_search_with_ngram_blocking_graph_equals_eager_reference_loop(dev):
    _graph_against_eager(dev, 6, 8, 4, 16, 1.0, 1.5, [30, 9, 64, 2, 50, 41], 3, seed=2)
