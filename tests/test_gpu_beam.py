"""Beam search on the GPU: ``kv_reorder_`` against a torch gather, ``beam_step_`` against the fp64 definition
(ops/beam.py) with a derived exemption bound for near ties, and ``GPT2DoubleHeads.beam_search`` on GPT-2 small."""
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


def _reorder_want(k, parent, prompt_len, lens, max_new):
    want = k.clone()
    for r, p in enumerate(parent.tolist()):
        if p == r:
            continue
        lo, hi = int(prompt_len[r]), min(int(lens[r]), int(prompt_len[r]) + max_new)
        want[:, r, :, lo:hi] = k[:, p, :, lo:hi]
    return want


def test_kv_reorder_against_torch_gather(dev):
    from adapcc_b200.ops import kv_reorder_, kv_reorder_scratch_numel

    L, R, H, t_max, Dh, max_new = 3, 12, 2, 48, 64, 16
    g = torch.Generator(device=dev).manual_seed(0)
    k = torch.randn(L, R, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16)
    v = torch.randn(L, R, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16)
    prompt_len = torch.tensor([5, 5, 5, 5, 9, 9, 9, 9, 14, 14, 14, 14], dtype=torch.int32, device=dev)
    lens = prompt_len + torch.tensor([0, 1, 3, 16, 7, 7, 7, 7, 2, 2, 2, 2], dtype=torch.int32, device=dev)
    scratch = torch.empty(kv_reorder_scratch_numel(k, max_new), dtype=torch.bfloat16, device=dev)
    maps = {"permutation": [1, 0, 3, 2, 6, 4, 5, 7, 11, 10, 9, 8],
            "cycle": [3, 0, 1, 2, 5, 6, 7, 4, 9, 10, 11, 8],
            "many_to_one": [0, 0, 0, 0, 4, 4, 5, 5, 8, 8, 8, 8],
            "identity": list(range(R))}
    for name, pm in maps.items():
        parent = torch.tensor(pm, dtype=torch.int32, device=dev)
        kk, vv = k.clone(), v.clone()
        kv_reorder_(kk, vv, parent, prompt_len, lens, max_new, scratch)
        torch.cuda.synchronize()
        assert torch.equal(kk.view(torch.int16), _reorder_want(k, parent, prompt_len, lens, max_new).view(torch.int16))
        assert torch.equal(vv.view(torch.int16), _reorder_want(v, parent, prompt_len, lens, max_new).view(torch.int16))
        # the prompt region and the rows that keep their own parent are untouched
        for r in range(R):
            if pm[r] == r:
                assert torch.equal(kk[:, r], k[:, r]), (name, r)
            assert torch.equal(kk[:, r, :, :int(prompt_len[r])], k[:, r, :, :int(prompt_len[r])]), (name, r)
    # a graph replay equals an eager launch
    parent = torch.tensor(maps["cycle"], dtype=torch.int32, device=dev)
    eager_k, eager_v = k.clone(), v.clone()
    kv_reorder_(eager_k, eager_v, parent, prompt_len, lens, max_new, scratch)
    kk, vv = k.clone(), v.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        kv_reorder_(kk, vv, parent, prompt_len, lens, max_new, scratch)
    kk.copy_(k)
    vv.copy_(v)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(kk.view(torch.int16), eager_k.view(torch.int16))
    assert torch.equal(vv.view(torch.int16), eager_v.view(torch.int16))
    with pytest.raises(ValueError, match="kv_reorder_"):
        kv_reorder_(k, v, parent, prompt_len, lens, max_new, scratch[:10])


def _tol(V, cs):
    """fp32 error bound of a candidate score c = s + ((l - m) - logf(Z)) against its fp64 value. Each of the three
    operations rounds once (u |result|, each result bounded by M = 1 + max |c|, |s|, |l - m|, log Z). Z is a sum of
    at most C = ceil(V / 512) terms per thread, 5 + 5 shuffle levels, each term within 2 ulp (expf) and a rounded
    argument: relative error (C + 14) u, which logf passes on as an absolute error, plus one rounding of log Z.
    So |c32 - c64| <= (4 M + C + 14) u; two candidates closer than twice that may swap."""
    M = 1.0 + max(abs(c) for c in cs) if cs else 1.0
    return 2.0 * (4.0 * M + math.ceil(V / 512) + 14) * U32


def _near(vals, tol):
    v = np.sort(np.asarray([x for x in vals if np.isfinite(x)], dtype=np.float64))
    d = np.diff(v)
    return bool(((d > 0) & (d <= tol)).any())


def _check_step(dev, B, K, V, step, max_new, alpha, stop, suppress, min_new, seed):
    from adapcc_b200.ops import BeamState, beam_step_
    from adapcc_b200.ops.beam import BeamReference

    rng = np.random.default_rng(seed)
    st = BeamState(B, K, max_new, alpha, dev)
    scores = -np.abs(rng.standard_normal((B, K)) * 3 * (step + 1)).astype(np.float32)
    scores.sort(axis=1)
    scores = scores[:, ::-1].copy()
    if step == 0:
        scores[:, 1:] = -np.inf
    scores[rng.random((B, K)) < 0.1] = -np.inf                      # some dead beams
    logits = (rng.standard_normal((B * K, V)) * 3).astype(np.float32)
    for b in range(0, B, 3):                                         # planted ties: within a row, and across rows
        r = b * K
        top = np.argsort(-logits[r])[:6]
        logits[r, top[2]] = logits[r, top[1]]
        if K > 1:
            logits[r + 1] = logits[r]
            scores[b, 1] = scores[b, 0]
    fin_count = rng.integers(0, K + 1, B)
    fin_score = np.sort(-np.abs(rng.standard_normal((B, K)) * 4), axis=1)[:, ::-1].astype(np.float32).copy()
    fin_n = rng.integers(0, max(1, step), (B, K)).astype(np.int32)
    fin_src = rng.integers(0, K, (B, K)).astype(np.int32)
    st.scores.copy_(torch.from_numpy(scores.reshape(-1)))
    st.step.fill_(step)
    st.fin_count.copy_(torch.from_numpy(fin_count.astype(np.int32)))
    st.fin_score.copy_(torch.from_numpy(fin_score))
    st.fin_n.copy_(torch.from_numpy(fin_n))
    st.fin_src.copy_(torch.from_numpy(fin_src))
    i32 = dict(dtype=torch.int32, device=dev)
    lt = torch.from_numpy(logits).to(dev)
    beam_step_(lt, V, st, min_new, torch.tensor(suppress, **i32) if suppress else None,
               torch.tensor(stop, **i32) if stop else None)
    torch.cuda.synchronize()
    ref = BeamReference(B, K, max_new, V, alpha, stop, suppress, min_new)
    ref.scores = scores.astype(np.float64)
    ref.n_steps = step
    for b in range(B):
        ref.fin[b] = [(float(fin_score[b, k]), int(fin_n[b, k]), int(fin_src[b, k])) for k in range(fin_count[b])]
    rank = [ref.ranking(b, logits, step)[:K * (K + len(stop))] for b in range(B)]
    nxt, parent = ref.step(logits)
    got = dict(nxt=st.next_ids.cpu().view(B, K), parent=st.parent.cpu().view(B, K), scores=st.scores.cpu().view(B, K),
               done=st.done.cpu(), count=st.fin_count.cpu(), fs=st.fin_score.cpu(), fn=st.fin_n.cpu(),
               src=st.fin_src.cpu())
    assert int(st.step) == step + 1
    exempt = 0
    for b in range(B):
        cs = [c for c, _, _ in rank[b]]
        tol = _tol(V, cs + [float(s) for s in scores[b] if np.isfinite(s)])
        fin = ref.fin[b]
        same = (got["nxt"][b].tolist() == nxt.view(B, K)[b].tolist()
                and got["parent"][b].tolist() == parent.view(B, K)[b].tolist()
                and int(got["count"][b]) == len(fin) and int(got["done"][b]) == int(ref.done[b])
                and [(int(got["fn"][b, k]), int(got["src"][b, k])) for k in range(len(fin))] == [f[1:] for f in fin]
                and np.allclose(got["fs"][b, :len(fin)].double().numpy(), [f[0] for f in fin], rtol=0, atol=4 * tol)
                and np.allclose(got["scores"][b].double().numpy(), ref.scores[b], rtol=0, atol=tol, equal_nan=True))
        if same:
            continue
        # the only allowed cause: two decision values (ranked candidates, normalised scores, the done bound) within
        # the fp32 error of each other
        pens = [ref.penalty(L) for L in range(1, max_new + 1)]
        near = (_near(cs, tol) or _near([f[0] for f in fin] + [float(x) for x in fin_score[b, :fin_count[b]]],
                                        4 * tol / min(pens))
                or (len(fin) == K and _near([fin[-1][0], ref.scores[b, 0] / pens[-1 if alpha > 0 else min(step + 1,
                                                                                                    max_new - 1)]],
                                            4 * tol / min(pens))))
        assert near, (B, K, V, step, b, got["nxt"][b].tolist(), nxt.view(B, K)[b].tolist())
        exempt += 1
    return B, exempt


CASES = [  # B, K, V, step, max_new, alpha, stop, suppress, min_new
    (512, 4, 3001, 3, 20, 1.0, [7, 11], [], 0),
    (256, 1, 3001, 0, 10, 0.0, [], [5, 6], 1),
    (128, 16, 1003, 5, 8, 2.0, [1, 2, 3, 4, 5, 6, 7, 8], [], 0),
    (32, 8, 50262, 2, 16, -0.5, [50256], list(range(50257, 50262)), 3),
    (512, 2, 700, 7, 8, 1.0, [0], [], 0),
    (400, 5, 64, 1, 4, 0.7, [3, 9], [3, 9], 2),
]


def test_beam_step_matches_fp64_definition(dev):
    items = exempt = 0
    for i, case in enumerate(CASES):
        n, e = _check_step(dev, *case, seed=i)
        items += n
        exempt += e
    print(f"beam_step vs fp64: {items} items, {exempt} exempt")
    assert items >= 1800 and exempt <= items // 50


def test_beam_step_item_alone_equals_item_in_batch(dev):
    """Selection of a batch, step after step, against each item run alone on the same logits: every output bit."""
    from adapcc_b200.ops import BeamState, beam_step_

    B, K, V, n = 6, 4, 50257, 6
    g = torch.Generator(device=dev).manual_seed(3)
    stop = torch.tensor([11, 50256], dtype=torch.int32, device=dev)
    sup = torch.tensor([5, 6, 11], dtype=torch.int32, device=dev)
    steps = [torch.randn(B * K, V, device=dev, generator=g) * 4 for _ in range(n)]
    for lg in steps:
        lg[:, 11] += 6.0                                             # the stop id competes
    full = BeamState(B, K, n, 0.6, dev)
    alone = [BeamState(1, K, n, 0.6, dev) for _ in range(B)]
    for lg in steps:
        beam_step_(lg, V, full, 2, sup, stop)
        for b in range(B):
            beam_step_(lg[b * K:(b + 1) * K].contiguous(), V, alone[b], 2, sup, stop)
    torch.cuda.synchronize()
    for b in range(B):
        a = alone[b]
        rows = slice(b * K, (b + 1) * K)
        assert torch.equal(full.scores[rows].view(torch.int32), a.scores.view(torch.int32)), b
        assert torch.equal(full.next_ids[rows], a.next_ids) and torch.equal(full.parent[rows] - b * K, a.parent), b
        assert torch.equal(full.hist_tok[:, rows], a.hist_tok) and torch.equal(full.hist_back[:, rows], a.hist_back)
        assert torch.equal(full.fin_score[b].view(torch.int32), a.fin_score[0].view(torch.int32)), b
        assert torch.equal(full.fin_n[b], a.fin_n[0]) and torch.equal(full.fin_src[b], a.fin_src[0]), b
        assert int(full.fin_count[b]) == int(a.fin_count[0]) and int(full.done[b]) == int(a.done[0]), b
    assert int(full.fin_count.sum()) > 0


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def test_beam_search_gpt2_small(dev):
    from adapcc_b200.ops import LM_HEAD_MAX_ROWS

    m = _gpt2_small(dev)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(4)
    prompt = torch.randint(0, V, (1, 200), device=dev, generator=g)
    want, _ = m.generate(prompt, max_new_tokens=32, temperature=0.0)
    tokens, n_new, _ = m.beam_search(prompt, num_beams=1, max_new_tokens=32)
    assert torch.equal(tokens, want) and n_new.tolist() == [32]
    lengths = [200, 37, 128, 1, 64, 199, 150, 90]
    ids = torch.randint(0, V, (8, 200), device=dev, generator=g)
    tt = torch.randint(V - 5, V - 3, (8, 200), device=dev, generator=g)
    stop = [int(want[0, 3]), V - 1]
    kw = dict(num_beams=4, max_new_tokens=24, length_penalty=1.0, stop_ids=stop)
    tokens, n_new, scores = m.beam_search(ids, lengths, tt, **kw)
    again = m.beam_search(ids, lengths, tt, **kw)
    assert all(torch.equal(a, b) for a, b in zip((tokens, n_new, scores), again))
    # an item alone: the prefill and the decode step's cuBLAS GEMMs round differently at other row counts (a 1-token
    # prompt alone runs a GEMV), so its logits are not the same bits as in the batch and a near tie between two
    # hypotheses may go the other way; test_beam_step_item_alone_equals_item_in_batch shows that the beam kernels
    # themselves are per item, bit for bit. Here: scores within 5 % (bf16 activations computed by GEMMs of another
    # shape drift apart by about 1 % over 24 tokens) and, where the tokens differ, hypotheses that near ties let swap.
    differ = 0
    for b, n in enumerate(lengths):
        t1, n1, s1 = m.beam_search(ids[b:b + 1, :n], None, tt[b:b + 1, :n], **kw)
        assert float(s1) == pytest.approx(float(scores[b]), rel=5e-2), b
        differ += not (torch.equal(t1[0], tokens[b]) and int(n1) == int(n_new[b]))
    print(f"beam_search items alone vs in a ragged batch of 8: {differ} with other tokens (near-tied hypotheses)")
    assert differ <= len(lengths) // 2
    with pytest.raises(ValueError, match="beam rows"):
        m.beam_search(ids[:, :10], num_beams=LM_HEAD_MAX_ROWS // 8 + 1)


def test_beam_search_graph_equals_eager_reference_loop(dev):
    """The graph path against an eager loop of the same decode step and LM head, with the selection done by
    ops/beam.py in fp64 and the cache reordered by torch indexing. An item may differ only if one of its steps had two
    candidates within the fp32 bound of each other."""
    from adapcc_b200.ops import lm_head_logits_
    from adapcc_b200.ops.beam import BeamReference

    m = _gpt2_small(dev, seed=1)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(9)
    B, K, n, alpha = 6, 4, 20, 0.8
    lengths = [64, 17, 120, 40, 5, 99]
    ids = torch.randint(0, V, (B, 120), device=dev, generator=g)
    stop = [int(ids[0, 0]), int(ids[1, 1])]
    tokens, n_new, scores = m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha,
                                          stop_ids=stop)
    w = m.wte.weight
    with torch.no_grad():
        last = torch.tensor(lengths, device=dev) - 1
        pre = m.new_cache(B, 120)
        h = m.hidden(ids, None, cache=pre, lengths=lengths)[torch.arange(B, device=dev), last]
        cache = m.new_cache(B * K, max(lengths) + n)
        cache.reset([x for x in lengths for _ in range(K)], 120)
        cache.k[:, :, :, :120].copy_(pre.k.repeat_interleave(K, dim=1))
        cache.v[:, :, :, :120].copy_(pre.v.repeat_interleave(K, dim=1))
        h = h.repeat_interleave(K, dim=0).contiguous()
        ref = BeamReference(B, K, n, V, alpha, stop)
        logits = torch.empty(B * K, w.shape[0], dtype=torch.float32, device=dev)
        near = np.zeros(B, dtype=bool)
        for i in range(n):
            if i:
                h = m.decode_step(nxt.to(dev), None, cache)
            lm_head_logits_(h, w, logits)
            lc = logits.cpu().numpy()
            for b in range(B):
                if not ref.done[b]:
                    cs = [c for c, _, _ in ref.ranking(b, lc, i)[:K * (K + len(stop))]]
                    near[b] |= _near(cs, _tol(V, cs))
            nxt, parent = ref.step(lc)
            rows = parent.to(dev)
            cache.k.copy_(cache.k[:, rows])
            cache.v.copy_(cache.v[:, rows])
            if ref.done.all():
                break
    rt, rn, rs = ref.result()
    exempt = 0
    for b in range(B):
        if torch.equal(tokens[b].cpu(), rt[b]) and int(n_new[b]) == int(rn[b]):
            assert float(scores[b]) == pytest.approx(float(rs[b]), abs=1e-3), b
            continue
        assert near[b], b
        exempt += 1
    print(f"beam_search graph vs eager fp64 loop: {B} items, {exempt} exempt")
    assert exempt <= B // 2
