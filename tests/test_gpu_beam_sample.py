"""Beam sampling on the GPU: the sampled ``beam_step_`` against the fp64 definition (``ops.beam.BeamSampleReference``)
with the same Philox words and a derived exemption bound for near ties, graph replay against an eager loop of the same
kernels, items alone, GPT-2 small against an eager loop of the definition, ``num_return_sequences`` on the native path
and a row that reaches ``n_positions``."""
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


def _tol_c(V, s, lp_max, T):
    """fp32 error bound of c = s + ((l - m) - logf(Z)) / T against fp64: the greedy bound of test_gpu_beam.py on the
    log-probability (Z a sum of ceil(V / 512) terms per thread and 5 + 5 shuffle levels, each within 2 ulp), carried
    through the division by T (one more rounding) and the addition of s (one rounding)."""
    lp_err = (3.0 * (1.0 + lp_max) + math.ceil(V / 512) + 14) * U32
    return lp_err / T + 2.0 * U32 * (abs(s) + lp_max / T + 1.0)


def _tol_g(tol_c, g):
    """c's bound plus G = -logf(-logf(u)) or -logf(-log1pf(u - 1)): the inner result within 1 ulp (relative), which
    the outer log turns into an absolute error, the outer within 1 ulp of |G| <= 17.4, and the rounding of c + G."""
    return tol_c + 2.0 * U32 + 2.0 * 17.4 * U32 + U32 * (abs(g) + 1.0)


def _decode_key(k):
    k = int(k) & 0xFFFFFFFFFFFFFFFF
    hi, lo = k >> 32, k & 0xFFFFFFFF
    u = (hi & 0x7FFFFFFF) if hi & 0x80000000 else (~hi & 0xFFFFFFFF)
    return float(np.array([u], dtype=np.uint32).view(np.float32)[0]), 0xFFFFFFFF - lo


def _near(vals, tol):
    v = np.sort(np.asarray([x for x in vals if np.isfinite(x)], dtype=np.float64))
    return bool(((np.diff(v) >= 0) & (np.diff(v) <= tol)).any())


def _item_near(ref, b, logits, step, V):
    """Whether item b's step had two of its M + 1 largest keys g, or two drawn scores c, within twice their fp32 bound
    of each other (the only way the kernel may order them differently), and that bound."""
    K, T = ref.K, ref.T
    gs, tg = [], 0.0
    for j in range(K):
        ids, c, g = ref.row_candidates(b, j, logits[b * K + j], step)
        gs += g.tolist()
        if ids.size:
            s = float(ref.scores[b, j])
            tc = _tol_c(V, s, float(np.max(np.abs(c - s) * T)), T)
            tg = max(tg, _tol_g(tc, float(np.max(np.abs(g)))))
    top = sorted(gs, reverse=True)[:ref.M + 1]
    cs = [c for _, c, _, _ in ref.draws(b, logits, step)]
    return _near(top, 2 * tg) or _near(cs, 2 * tg), tg


def _check_step(dev, B, K, V, step, max_new, alpha, stop, suppress, min_new, T, top_k, top_p, seed):
    from adapcc_b200.ops import BeamState, beam_step_
    from adapcc_b200.ops.beam import BeamSampleReference

    rng = np.random.default_rng(seed)
    st = BeamState(B, K, max_new, alpha, dev, sample=True)
    scores = -np.abs(rng.standard_normal((B, K)) * 3 * (step + 1)).astype(np.float32)
    scores = -np.sort(-scores, axis=1)
    if step == 0:
        scores[:, 1:] = -np.inf
    scores[rng.random((B, K)) < 0.1] = -np.inf
    logits = (rng.standard_normal((B * K, V)) * 3).astype(np.float32)
    fin_count = rng.integers(0, K + 1, B)
    fin_score = np.sort(-np.abs(rng.standard_normal((B, K)) * 4), axis=1)[:, ::-1].astype(np.float32).copy()
    fin_n = rng.integers(0, max(1, step), (B, K)).astype(np.int32)
    fin_src = rng.integers(0, K, (B, K)).astype(np.int32)
    seeds = rng.integers(0, 2 ** 62, B)
    st.scores.copy_(torch.from_numpy(scores.reshape(-1)))
    st.step.fill_(step)
    st.fin_count.copy_(torch.from_numpy(fin_count.astype(np.int32)))
    st.fin_score.copy_(torch.from_numpy(fin_score))
    st.fin_n.copy_(torch.from_numpy(fin_n))
    st.fin_src.copy_(torch.from_numpy(fin_src))
    i32 = dict(dtype=torch.int32, device=dev)
    beam_step_(torch.from_numpy(logits).to(dev), V, st, min_new, torch.tensor(suppress, **i32) if suppress else None,
               torch.tensor(stop, **i32) if stop else None, temperature=T, top_k=top_k, top_p=top_p,
               seeds=torch.from_numpy(seeds).to(dev))
    torch.cuda.synchronize()
    ref = BeamSampleReference(B, K, max_new, V, alpha, stop, suppress, min_new, temperature=T, top_k=top_k,
                              top_p=top_p, seeds=seeds.tolist())
    ref.scores = scores.astype(np.float64)
    ref.n_steps = step
    for b in range(B):
        ref.fin[b] = [(float(fin_score[b, k]), int(fin_n[b, k]), int(fin_src[b, k])) for k in range(fin_count[b])]
    M = ref.M
    cand = st.cand.view(-1)[:B * K * M].view(B * K, M).cpu().numpy()          # packed [B·K, M]
    cand_c = st.cand_c.view(-1)[:B * K * M].view(B * K, M).cpu().numpy()
    kept_exempt = 0
    for b in range(B):
        for j in range(K):
            ids, c, g = ref.row_candidates(b, j, logits[b * K + j], step)
            r = b * K + j
            got = [(_decode_key(k), float(cc)) for k, cc in zip(cand[r], cand_c[r]) if k != 0]
            got_ids = [i for (_, i), _ in got]
            lp_max = float(np.max(np.abs(c - scores[b, j]) * T)) if ids.size else 0.0
            tc = _tol_c(V, float(scores[b, j]), lp_max, T)
            where = {int(i): n for n, i in enumerate(ids)}
            if ids.size <= M and set(got_ids) != set(ids.tolist()):
                assert top_p < 1, (b, j)                          # only a top-p boundary may round the other way
                kept_exempt += 1
            for (gk, i), cc in got:
                if i in where:
                    assert abs(cc - c[where[i]]) <= tc, (b, j, i, cc, c[where[i]], tc)
                    assert abs(gk - g[where[i]]) <= _tol_g(tc, gk), (b, j, i, gk, g[where[i]])
    near = {b: _item_near(ref, b, logits, step, V) for b in range(B)}
    nxt, parent = ref.step(logits)
    got = dict(nxt=st.next_ids.cpu().view(B, K), parent=st.parent.cpu().view(B, K), done=st.done.cpu(),
               count=st.fin_count.cpu(), fs=st.fin_score.cpu(), fn=st.fin_n.cpu(), src=st.fin_src.cpu(),
               tok=st.hist_tok[step].cpu().view(B, K), back=st.hist_back[step].cpu().view(B, K))
    assert int(st.step) == step + 1
    exempt = 0
    for b in range(B):
        fin = ref.fin[b]
        same = (got["nxt"][b].tolist() == nxt.view(B, K)[b].tolist()
                and got["parent"][b].tolist() == parent.view(B, K)[b].tolist()
                and got["tok"][b].tolist() == ref.hist_tok[step, b].tolist()
                and got["back"][b].tolist() == ref.hist_back[step, b].tolist()
                and int(got["count"][b]) == len(fin) and int(got["done"][b]) == int(ref.done[b])
                and [(int(got["fn"][b, k]), int(got["src"][b, k])) for k in range(len(fin))] == [f[1:] for f in fin]
                and np.allclose(got["fs"][b, :len(fin)].double().numpy(), [f[0] for f in fin], rtol=1e-5, atol=1e-5))
        if same:
            continue
        # the only allowed causes: two keys g (the draw order) or two scores c (the beam order, the offers) within
        # their fp32 bounds of each other, or two normalised scores of the finished set
        tie, tg = near[b]
        pens = [ref.penalty(L) for L in range(1, max_new + 1)]
        tie = tie or _near([f[0] for f in fin] + [float(x) for x in fin_score[b, :fin_count[b]]], 4 * tg / min(pens))
        assert tie, (B, K, V, step, b, got["nxt"][b].tolist(), nxt.view(B, K)[b].tolist())
        exempt += 1
    return B, exempt, kept_exempt


CASES = [  # B, K, V, step, max_new, alpha, stop, suppress, min_new, T, top_k, top_p
    (256, 1, 3001, 0, 10, 0.0, [], [5, 6], 1, 1.0, 0, 1.0),
    (256, 4, 3001, 3, 20, 1.0, [7, 11], [], 0, 0.7, 50, 1.0),
    (128, 4, 50257, 2, 16, -0.5, [50256], list(range(50257 - 5, 50257)), 3, 1.3, 0, 0.9),
    (64, 16, 1003, 5, 8, 2.0, [1, 2, 3, 4, 5, 6, 7, 8], [], 0, 0.9, 40, 0.8),
    (64, 16, 700, 7, 8, 1.0, [], [], 0, 1.0, 3, 0.05),
    (256, 4, 64, 1, 4, 0.7, [3, 9], [3, 9], 2, 2.0, 0, 1.0),
]


def test_beam_sample_step_matches_fp64_definition(dev):
    items = exempt = kept_exempt = 0
    for i, case in enumerate(CASES):
        n, e, k = _check_step(dev, *case, seed=i)
        items += n
        exempt += e
        kept_exempt += k
    print(f"beam_sample_step vs fp64: {items} items, {exempt} exempt (near ties), {kept_exempt} rows with a kept set "
          f"rounded at the top-p boundary")
    assert items >= 1000 and exempt <= items // 50 and kept_exempt <= items // 50


def test_beam_sample_step_item_alone_equals_item_in_batch(dev):
    from adapcc_b200.ops import BeamState, beam_step_

    B, K, V, n = 6, 4, 50257, 6
    g = torch.Generator(device=dev).manual_seed(3)
    stop = torch.tensor([11, 50256], dtype=torch.int32, device=dev)
    sup = torch.tensor([5, 6, 11], dtype=torch.int32, device=dev)
    seeds = torch.arange(100, 100 + B, dtype=torch.int64, device=dev)
    steps = [torch.randn(B * K, V, device=dev, generator=g) * 4 for _ in range(n)]
    for lg in steps:
        lg[:, 11] += 6.0
    kw = dict(temperature=0.8, top_k=30, top_p=0.95)
    full = BeamState(B, K, n, 0.6, dev, sample=True)
    alone = [BeamState(1, K, n, 0.6, dev, sample=True) for _ in range(B)]
    for lg in steps:
        beam_step_(lg, V, full, 2, sup, stop, seeds=seeds, **kw)
        for b in range(B):
            beam_step_(lg[b * K:(b + 1) * K].contiguous(), V, alone[b], 2, sup, stop, seeds=seeds[b:b + 1], **kw)
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


def _eager(m, ids, lengths, K, n, alpha, stop, seeds, kw, select):
    """The native beam_search's loop without the graph: prefill, the K-row cache, LM head, then ``select(logits, i)``
    returning the parents; the caller decides how a step selects."""
    from adapcc_b200.ops import lm_head_logits_

    dev, B, T = ids.device, ids.shape[0], ids.shape[1]
    w = m.wte.weight
    last = torch.tensor(lengths, device=dev) - 1
    pre = m.new_cache(B, T)
    h = m.hidden(ids, None, cache=pre, lengths=lengths)[torch.arange(B, device=dev), last]
    cache = m.new_cache(B * K, max(lengths) + n)
    cache.reset([x for x in lengths for _ in range(K)], T)
    cache.k[:, :, :, :T].copy_(pre.k.repeat_interleave(K, dim=1))
    cache.v[:, :, :, :T].copy_(pre.v.repeat_interleave(K, dim=1))
    h = h.repeat_interleave(K, dim=0).contiguous()
    logits = torch.empty(B * K, w.shape[0], dtype=torch.float32, device=dev)
    nxt = None
    for i in range(n):
        if i:
            h = m.decode_step(nxt.to(dev), None, cache)
        lm_head_logits_(h, w, logits)
        nxt, rows, stop_now = select(logits, i, cache)
        if rows is not None:
            cache.k.copy_(cache.k[:, rows])
            cache.v.copy_(cache.v[:, rows])
        if stop_now:
            break


def test_graph_equals_eager_loop_of_the_same_kernels(dev):
    from adapcc_b200.ops import BeamState, beam_step_, kv_reorder_, kv_reorder_scratch_numel
    from adapcc_b200.ops.beam import best_hypotheses

    m = _gpt2_small(dev, seed=1)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(9)
    B, K, n, alpha = 6, 4, 20, 0.8
    lengths = [64, 17, 120, 40, 5, 99]
    ids = torch.randint(0, V, (B, 120), device=dev, generator=g)
    stop = [int(ids[0, 0]), int(ids[1, 1])]
    kw = dict(temperature=0.9, top_k=40, top_p=0.95)
    seeds = torch.arange(7, 7 + B, dtype=torch.int64)
    out = m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha, stop_ids=stop,
                        do_sample=True, seed=seeds, num_return_sequences=K, **kw)
    again = m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha, stop_ids=stop,
                          do_sample=True, seed=seeds, num_return_sequences=K, **kw)
    assert all(torch.equal(a, b) for a, b in zip(out, again))
    st = BeamState(B, K, n, alpha, dev, sample=True)
    stop_t = torch.tensor(stop, dtype=torch.int32, device=dev)
    sd = seeds.to(dev)

    def select(logits, i, cache):
        if i == 0:
            select.prompt_len = cache.lens.clone()
            select.scratch = torch.empty(kv_reorder_scratch_numel(cache.k, n), dtype=cache.k.dtype, device=dev)
        beam_step_(logits, V, st, 0, None, stop_t, seeds=sd, **kw)
        kv_reorder_(cache.k, cache.v, st.parent, select.prompt_len, cache.lens, n, select.scratch)
        return st.next_ids, None, False

    with torch.no_grad():
        _eager(m, ids, lengths, K, n, alpha, stop, seeds, kw, select)
    count = st.fin_count.cpu().tolist()
    fin = [list(zip(st.fin_score.cpu().tolist()[b], st.fin_n.cpu().tolist()[b],
                    st.fin_src.cpu().tolist()[b]))[:count[b]] for b in range(B)]
    want = best_hypotheses(fin, st.hist_tok.view(n, B, K).cpu().numpy(), st.hist_back.view(n, B, K).cpu().numpy(),
                           n, K)
    assert torch.equal(out[0].cpu(), want[0]) and torch.equal(out[1].cpu(), want[1])
    assert torch.equal(out[2].cpu().view(torch.int32), want[2].view(torch.int32))
    # n-best on the native path: the CPU path's semantics
    for b in range(B):
        s = out[2][b * K:(b + 1) * K].cpu()
        assert (s[:-1] >= s[1:]).all() and int(out[1][b * K]) > 0, b
        for q in range(b * K, (b + 1) * K):
            k = int(out[1][q])
            assert (out[0][q, k:] == -1).all() and (out[0][q, :k] >= 0).all()
            assert k == 0 or float(out[2][q]) > float("-inf")
    first = m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha, stop_ids=stop,
                          do_sample=True, seed=seeds, **kw)
    assert torch.equal(first[0], out[0][::K]) and torch.equal(first[1], out[1][::K])


def test_gpt2_small_against_the_fp64_definition(dev):
    """The graph path against an eager loop of the same decode step and LM head with the selection done by
    BeamSampleReference in fp64 and the cache reordered by torch indexing. An item may differ only if one of its steps
    had two keys or two scores within the fp32 bound of each other."""
    from adapcc_b200.ops.beam import BeamSampleReference

    m = _gpt2_small(dev, seed=2)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(5)
    B, K, n, alpha = 4, 4, 16, 1.0
    lengths = [50, 17, 90, 33]
    ids = torch.randint(0, V, (B, 90), device=dev, generator=g)
    stop = [int(ids[0, 3])]
    kw = dict(temperature=0.8, top_k=50, top_p=0.9)
    tokens, n_new, scores = m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha,
                                          stop_ids=stop, do_sample=True, seed=21, **kw)
    ref = BeamSampleReference(B, K, n, V, alpha, stop, temperature=kw["temperature"], top_k=kw["top_k"],
                              top_p=kw["top_p"], seeds=[21 + b for b in range(B)])
    near = np.zeros(B, dtype=bool)

    def select(logits, i, cache):
        lc = logits.cpu().numpy()
        for b in range(B):
            if not ref.done[b]:
                near[b] |= _item_near(ref, b, lc, i, V)[0]
        nxt, parent = ref.step(lc)
        return nxt, parent.to(dev), bool(ref.done.all())

    with torch.no_grad():
        _eager(m, ids, lengths, K, n, alpha, stop, None, kw, select)
    rt, rn, rs = ref.result()
    exempt = 0
    for b in range(B):
        if torch.equal(tokens[b].cpu(), rt[b]) and int(n_new[b]) == int(rn[b]):
            assert float(scores[b]) == pytest.approx(float(rs[b]), abs=1e-3), b
            continue
        assert near[b], b
        exempt += 1
    print(f"beam sampling graph vs eager fp64 loop: {B} items, {exempt} exempt")
    assert exempt <= B // 2


def test_row_reaching_n_positions_and_vocabulary_limit(dev):
    from adapcc_b200.ops import SAMPLE_MAX_VOCAB, BeamState, beam_step_

    m = _gpt2_small(dev, seed=3)
    V, P = m.cfg.vocab_size, m.cfg.n_positions
    g = torch.Generator(device=dev).manual_seed(6)
    ids = torch.randint(0, V, (2, P - 8), device=dev, generator=g)
    tokens, n_new, scores = m.beam_search(ids, [P - 8, 30], num_beams=4, max_new_tokens=8, do_sample=True, seed=1,
                                          top_k=20, num_return_sequences=2)
    assert tokens.shape == (4, 8) and (n_new > 0).all() and torch.isfinite(scores).all()
    st = BeamState(1, 2, 4, 1.0, dev, sample=True)
    big = torch.zeros(2, SAMPLE_MAX_VOCAB + 64, device=dev)
    with pytest.raises(ValueError, match="vocab"):
        beam_step_(big, SAMPLE_MAX_VOCAB + 1, st, seeds=torch.zeros(1, dtype=torch.int64, device=dev))
    with pytest.raises(ValueError, match="sample=True"):
        beam_step_(big, 100, BeamState(1, 2, 4, 1.0, dev), seeds=torch.zeros(1, dtype=torch.int64, device=dev))
