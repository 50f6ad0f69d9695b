"""Stochastic beam search on the GPU: one stochastic ``beam_step_`` against the fp64 definition
(``ops.beam.StochasticBeamReference``) with an exemption for near ties, graph replay against an eager loop of the
same kernels, GPT-2 small against an eager loop of the definition, the first reply's law on the tiny bf16 model by a
chi-square test, items alone against items in a batch, and the limits."""
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


def _tol_phi(V, phi):
    """fp32 bound of phi = phi_j + ((x - m) - logf(Z)): Z a fixed-order sum of ceil(V / 1024) terms per thread and
    5 + 5 shuffle levels of expf values (each within 2 ulp), then three roundings of values up to |phi|."""
    return (2.0 * (np.ceil(V / 1024) + 10) + 4.0) * U32 + 4.0 * U32 * (abs(phi) + 1.0)


def _tol_key(V, phi, key, amp=0.0):
    """phi's bound plus the Gumbel (inner and outer log within 1 ulp of |G| <= 17.4) gives Gphi's; the truncation adds a
    few ulp of values up to |key| + 40 and carries the errors of Gphi and Z through a = Gphi - Z with the gain ``amp``
    = |d key / d a| (``_gain``), which is large where a child's Gphi is close to the row's best."""
    g = _tol_phi(V, phi) + 40.0 * U32 + U32 * (abs(phi) + 20.0)
    return g * (1.0 + 2.0 * amp) + 8.0 * U32 * (abs(key) + 40.0)


def _gain(G, gphi):
    """|d key / d a| of rule R5 at a = Gphi - Z: sigmoid(v) / expm1(-a) (0 for the row's best child)."""
    a = gphi - gphi.max()
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        l1m = np.where(a > -np.log(2.0), np.log(-np.expm1(a)), np.log1p(-np.exp(a)))
        v = G - gphi + l1m
        out = 1.0 / (1.0 + np.exp(-v)) / np.expm1(-a)
    return np.where(a < 0, out, 0.0)


def _row_tols(V, ref, b, j, phi, gphi, key):
    if not gphi.size:
        return np.zeros(1)
    return np.array([_tol_key(V, float(p), float(k), float(g))
                     for p, k, g in zip(phi, key, _gain(ref.keys[b, j], gphi))])


def _decode(k):
    k = int(k) & 0xFFFFFFFFFFFFFFFF
    return 0xFFFFFFFF - (k & 0xFFFFFFFF)


def _near(vals, tol):
    v = np.sort(np.asarray([x for x in vals if np.isfinite(x)], dtype=np.float64))
    return bool((np.diff(v) <= tol).any())


def _item_near(ref, b, logits, step, V):
    """Whether two of item b's children (Gphi within a row) or two of its pool's K + 2 largest keys lie within twice
    their fp32 bound of each other: the only way the kernels may order them differently."""
    K = ref.K
    keys, tol = [f[0] for f in ref.fin[b]], 0.0
    for j in range(K):
        ids, phi, gphi, key = ref.children(b, j, logits[b * K + j], step)
        if ids.size:
            tol = max(tol, float(_row_tols(V, ref, b, j, phi, gphi, key).max()))
            if _near(gphi, 2 * tol):
                return True, tol
            keys += key.tolist()
    top = sorted(keys, reverse=True)[:K + 2]
    tol = max([tol] + [_tol_key(V, 0.0, k) for k in top])
    return _near(top, 2 * tol), tol


def _check_step(dev, B, K, V, step, max_new, stop, suppress, min_new, T, top_k, top_p, seed):
    from adapcc_b200.ops import BeamState, beam_step_
    from adapcc_b200.ops.beam import StochasticBeamReference

    rng = np.random.default_rng(seed)
    seeds = rng.integers(0, 2 ** 62, B)
    st = BeamState(B, K, max_new, 1.0, dev, seeds=torch.from_numpy(seeds))
    phi = -np.sort(np.abs(rng.standard_normal((B, K)) * 3 * (step + 1)), axis=1).astype(np.float32)
    keys = np.sort(rng.standard_normal((B, K)) * 2 + 1, axis=1)[:, ::-1].astype(np.float32).copy()
    if step == 0:
        phi[:, 1:] = -np.inf
    phi[rng.random((B, K)) < 0.1] = -np.inf
    keys[~np.isfinite(phi)] = -np.inf
    logits = (rng.standard_normal((B * K, V)) * 3).astype(np.float32)
    fin_count = rng.integers(0, K + 1, B)
    fin_key = np.sort(rng.standard_normal((B, K)) * 2 - 1, axis=1)[:, ::-1].astype(np.float32).copy()
    fin_phi = -np.abs(rng.standard_normal((B, K)) * 5).astype(np.float32)
    fin_n = rng.integers(0, max(1, step), (B, K)).astype(np.int32)
    fin_src = rng.integers(0, K, (B, K)).astype(np.int32)
    kappa = np.where(rng.random(B) < 0.5, -np.inf, rng.standard_normal(B) * 2 - 4).astype(np.float32)
    st.scores.copy_(torch.from_numpy(phi.reshape(-1)))
    st.keys.copy_(torch.from_numpy(keys.reshape(-1)))
    st.step.fill_(step)
    st.fin_count.copy_(torch.from_numpy(fin_count.astype(np.int32)))
    for t, a in ((st.fin_score, fin_key), (st.fin_phi, fin_phi), (st.fin_n, fin_n), (st.fin_src, fin_src),
                 (st.kappa, kappa)):
        t.copy_(torch.from_numpy(a))
    i32 = dict(dtype=torch.int32, device=dev)
    beam_step_(torch.from_numpy(logits).to(dev), V, st, min_new, torch.tensor(suppress, **i32) if suppress else None,
               torch.tensor(stop, **i32) if stop else None, temperature=T, top_k=top_k, top_p=top_p)
    torch.cuda.synchronize()
    ref = StochasticBeamReference(B, K, max_new, V, stop, suppress, min_new, temperature=T, top_k=top_k, top_p=top_p,
                                  seeds=seeds.tolist())
    ref.scores, ref.keys, ref.kappa = phi.astype(np.float64), keys.astype(np.float64), kappa.astype(np.float64)
    ref.n_steps = step
    for b in range(B):
        ref.fin[b] = [(float(fin_key[b, k]), int(fin_n[b, k]), int(fin_src[b, k]), float(fin_phi[b, k]))
                      for k in range(fin_count[b])]
    cand = st.cand.view(-1)[:B * K * (K + 1)].view(B * K, K + 1).cpu().numpy()          # packed [B·K, K + 1]
    ck, cp = st.cand_key.cpu().numpy(), st.cand_phi.cpu().numpy()
    rows_exempt = 0
    for b in range(B):
        for j in range(K):
            ids, rphi, gphi, rkey = ref.children(b, j, logits[b * K + j], step)
            r = b * K + j
            got = [(_decode(k), float(ck[r, e]), float(cp[r, e])) for e, k in enumerate(cand[r]) if k != 0]
            tols = _row_tols(V, ref, b, j, rphi, gphi, rkey)
            if [i for i, _, _ in got] != ids.tolist():
                assert _near(gphi, 2 * tols.max()) or top_p < 1, (b, j)   # near ties, or a top-p boundary rounded
                rows_exempt += 1
            where = {int(i): e for e, i in enumerate(ids)}
            for i, k, p in got:
                if i in where:
                    e = where[i]
                    assert abs(p - rphi[e]) <= _tol_phi(V, rphi[e]), (b, j, i, p, rphi[e])
                    assert abs(k - rkey[e]) <= tols[e], (b, j, i, k, rkey[e], tols[e])
    near = {b: _item_near(ref, b, logits, step, V) for b in range(B)}
    nxt, parent = ref.step(logits)
    got = dict(nxt=st.next_ids.cpu().view(B, K), parent=st.parent.cpu().view(B, K), done=st.done.cpu(),
               count=st.fin_count.cpu(), fk=st.fin_score.cpu(), fp=st.fin_phi.cpu(), fn=st.fin_n.cpu(),
               src=st.fin_src.cpu(), tok=st.hist_tok[step].cpu().view(B, K), back=st.hist_back[step].cpu().view(B, K),
               kappa=st.kappa.cpu(), phi=st.scores.cpu().view(B, K), keys=st.keys.cpu().view(B, K))
    assert int(st.step) == step + 1
    exempt = 0
    for b in range(B):
        fin = ref.fin[b]
        vals = [f[0] for f in fin] + [f[3] for f in fin] + ref.scores[b].tolist() + ref.keys[b].tolist()
        big = max([abs(x) for x in vals + [float(ref.kappa[b])] if np.isfinite(x)] + [0.0])
        tol = 2 * max(_tol_key(V, big, big), near[b][1])
        same = (got["nxt"][b].tolist() == nxt.view(B, K)[b].tolist()
                and got["parent"][b].tolist() == parent.view(B, K)[b].tolist()
                and got["tok"][b].tolist() == ref.hist_tok[step, b].tolist()
                and got["back"][b].tolist() == ref.hist_back[step, b].tolist()
                and int(got["count"][b]) == len(fin) and int(got["done"][b]) == int(ref.done[b])
                and [(int(got["fn"][b, k]), int(got["src"][b, k])) for k in range(len(fin))] == [f[1:3] for f in fin]
                and np.allclose(got["fk"][b, :len(fin)].double().numpy(), [f[0] for f in fin], rtol=0, atol=tol)
                and np.allclose(got["fp"][b, :len(fin)].double().numpy(), [f[3] for f in fin], rtol=0, atol=tol)
                and np.allclose(got["kappa"][b].double().numpy(), ref.kappa[b], rtol=0, atol=tol)
                and np.allclose(got["phi"][b].double().numpy(), ref.scores[b], rtol=0, atol=tol)
                and np.allclose(got["keys"][b].double().numpy(), ref.keys[b], rtol=0, atol=tol))
        if same:
            continue
        assert near[b][0], (B, K, V, step, b, got["nxt"][b].tolist(), nxt.view(B, K)[b].tolist())
        exempt += 1
    return B, exempt, rows_exempt


CASES = [  # B, K, V, step, max_new, stop, suppress, min_new, T, top_k, top_p
    (64, 1, 3001, 0, 10, [], [5, 6], 1, 1.0, 0, 1.0),
    (16, 4, 50257, 0, 8, [50256], [], 0, 1.0, 0, 1.0),                     # B·K = 64 at GPT-2's vocabulary
    (16, 4, 50257, 3, 16, [50256], list(range(50257 - 5, 50257)), 5, 1.3, 0, 0.9),
    (128, 4, 3001, 2, 20, [7, 11], [], 0, 0.7, 50, 1.0),
    (64, 16, 1003, 5, 8, [1, 2, 3, 4, 5, 6, 7, 8], [], 0, 0.9, 40, 0.8),
    (64, 16, 700, 7, 8, [], [], 0, 1.0, 3, 0.05),                          # the last step; few kept ids
    (256, 8, 12, 1, 4, [3, 9], [3, 9], 2, 2.0, 0, 1.0),                    # fewer children than K + 1 per row
]


def test_stochastic_step_matches_fp64_definition(dev):
    items = exempt = rows_exempt = 0
    for i, case in enumerate(CASES):
        n, e, r = _check_step(dev, *case, seed=i)
        items += n
        exempt += e
        rows_exempt += r
    print(f"stochastic beam step vs fp64: {items} items, {exempt} exempt (near ties), {rows_exempt} rows with "
          f"another offered set (near ties or a top-p boundary)")
    assert exempt <= items // 20 and rows_exempt <= items // 20


def test_step_item_alone_equals_item_in_batch(dev):
    from adapcc_b200.ops import BeamState, beam_step_

    B, K, V, n = 6, 4, 50257, 6
    g = torch.Generator(device=dev).manual_seed(3)
    stop = torch.tensor([11, 50256], dtype=torch.int32, device=dev)
    sup = torch.tensor([5, 6, 11], dtype=torch.int32, device=dev)
    seeds = torch.arange(100, 100 + B, dtype=torch.int64)
    steps = [torch.randn(B * K, V, device=dev, generator=g) * 4 for _ in range(n)]
    for lg in steps:
        lg[:, 11] += 6.0
    kw = dict(temperature=0.8, top_k=30, top_p=0.95)
    full = BeamState(B, K, n, 1.0, dev, seeds=seeds)
    alone = [BeamState(1, K, n, 1.0, dev, seeds=seeds[b:b + 1]) for b in range(B)]
    for lg in steps:
        beam_step_(lg, V, full, 2, sup, stop, **kw)
        for b in range(B):
            beam_step_(lg[b * K:(b + 1) * K].contiguous(), V, alone[b], 2, sup, stop, **kw)
    torch.cuda.synchronize()
    bits = lambda t: t.view(torch.int32)                                   # noqa: E731
    for b in range(B):
        a, rows = alone[b], slice(b * K, (b + 1) * K)
        assert torch.equal(bits(full.scores[rows]), bits(a.scores)) and torch.equal(bits(full.keys[rows]), bits(a.keys))
        assert torch.equal(full.next_ids[rows], a.next_ids) and torch.equal(full.parent[rows] - b * K, a.parent), b
        assert torch.equal(full.hist_tok[:, rows], a.hist_tok) and torch.equal(full.hist_back[:, rows], a.hist_back)
        for x, y in ((full.fin_score, a.fin_score), (full.fin_phi, a.fin_phi)):
            assert torch.equal(bits(x[b]), bits(y[0])), b
        assert torch.equal(full.fin_n[b], a.fin_n[0]) and torch.equal(full.fin_src[b], a.fin_src[0]), b
        assert int(full.fin_count[b]) == int(a.fin_count[0]) and int(full.done[b]) == int(a.done[0]), b
        assert torch.equal(bits(full.kappa[b:b + 1]), bits(a.kappa)), b
    assert int(full.fin_count.sum()) > 0


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def _eager(m, ids, lengths, K, n, select):
    """The native decoder's loop without the graph: prefill, the K-row cache, LM head, then ``select(logits, i,
    cache)`` returning ``(next ids, rows to gather or None, stop)``."""
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
    from adapcc_b200.ops.beam import stochastic_results

    m = _gpt2_small(dev, seed=1)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(9)
    B, K, n = 6, 4, 20
    lengths = [64, 17, 120, 40, 5, 99]
    ids = torch.randint(0, V, (B, 120), device=dev, generator=g)
    stop = [int(ids[0, 0]), int(ids[1, 1])]
    kw = dict(temperature=0.9, top_k=40, top_p=0.95)
    seeds = torch.arange(7, 7 + B, dtype=torch.int64)
    out = m.stochastic_beam_search(ids, lengths, num_beams=K, max_new_tokens=n, stop_ids=stop, seed=seeds, **kw)
    again = m.stochastic_beam_search(ids, lengths, num_beams=K, max_new_tokens=n, stop_ids=stop, seed=seeds, **kw)
    assert all(torch.equal(a, b) for a, b in zip(out, again))
    st = BeamState(B, K, n, 1.0, dev, seeds=seeds)
    stop_t = torch.tensor(stop, dtype=torch.int32, device=dev)
    Vm = m.cfg.vocab_size

    def select(logits, i, cache):
        if i == 0:
            select.prompt_len = cache.lens.clone()
            select.scratch = torch.empty(kv_reorder_scratch_numel(cache.k, n), dtype=cache.k.dtype, device=dev)
        beam_step_(logits, Vm, st, 0, None, stop_t, **kw)
        kv_reorder_(cache.k, cache.v, st.parent, select.prompt_len, cache.lens, n, select.scratch)
        return st.next_ids, None, False

    with torch.no_grad():
        _eager(m, ids, lengths, K, n, select)
    count = st.fin_count.cpu().tolist()
    cols = [x.cpu().tolist() for x in (st.fin_score, st.fin_n, st.fin_src, st.fin_phi)]
    fin = [list(zip(*(c[b] for c in cols)))[:count[b]] for b in range(B)]
    want = stochastic_results(fin, st.hist_tok.view(n, B, K).cpu().numpy(), st.hist_back.view(n, B, K).cpu().numpy(),
                              n, K, st.kappa.cpu().numpy())
    assert torch.equal(out[0].cpu(), want[0]) and torch.equal(out[1].cpu(), want[1])
    for q in (2, 3, 4):
        assert torch.equal(out[q].cpu().view(torch.int32), want[q].view(torch.int32)), q
    for b in range(B):
        rows = [tuple(out[0][q, :int(out[1][q])].tolist()) for q in range(b * K, (b + 1) * K)]
        k = out[3][b * K:(b + 1) * K].cpu()
        assert len(set(rows)) == K and (k[:-1] >= k[1:]).all(), b          # K distinct replies, best key first


def test_gpt2_small_against_the_fp64_definition(dev):
    """The graph path against an eager loop of the same decode step and LM head with the selection done by
    StochasticBeamReference in fp64 and the cache reordered by torch indexing. An item may differ only if one of its
    steps had a near tie."""
    from adapcc_b200.ops.beam import StochasticBeamReference

    m = _gpt2_small(dev, seed=2)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(5)
    B, K, n = 4, 8, 16
    lengths = [50, 17, 90, 33]
    ids = torch.randint(0, V - 5, (B, 90), device=dev, generator=g)
    stop = [int(ids[0, 3])]
    kw = dict(temperature=0.8, top_k=50, top_p=0.9)
    tokens, n_new, log_probs, keys, kappa = m.stochastic_beam_search(ids, lengths, num_beams=K, max_new_tokens=n,
                                                                     stop_ids=stop, seed=21, **kw)
    ref = StochasticBeamReference(B, K, n, V, stop, seeds=[21 + b for b in range(B)], **kw)
    near = np.zeros(B, dtype=bool)

    def select(logits, i, cache):
        lc = logits.cpu().numpy()
        for b in range(B):
            if not ref.done[b]:
                near[b] |= _item_near(ref, b, lc, i, V)[0]
        nxt, parent = ref.step(lc)
        return nxt, parent.to(dev), bool(ref.done.all())

    with torch.no_grad():
        _eager(m, ids, lengths, K, n, select)
    rt, rn, rlp, rk, rkap = ref.result()
    exempt = 0
    for b in range(B):
        rows = slice(b * K, (b + 1) * K)
        if torch.equal(tokens[rows].cpu(), rt[rows]) and torch.equal(n_new[rows].cpu(), rn[rows]):
            assert log_probs[rows].cpu().tolist() == pytest.approx(rlp[rows].tolist(), abs=1e-3), b
            assert keys[rows].cpu().tolist() == pytest.approx(rk[rows].tolist(), abs=1e-3), b
            assert float(kappa[b]) == pytest.approx(float(rkap[b]), abs=1e-3), b
            continue
        assert near[b], b
        exempt += 1
    print(f"stochastic beam search graph vs eager fp64 loop: {B} items, {exempt} exempt")
    assert exempt <= B // 2


def test_first_reply_law_on_the_tiny_bf16_model(dev):
    """P1 on the native path: the first reply of 64-item batches (distinct seeds) against the law of generate's draw,
    enumerated from the same bf16 model's logits with the filter of ops/sampling.py."""
    from scipy.stats import chisquare

    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.ops import lm_head_logits_
    from adapcc_b200.ops.sampling import reference_row

    torch.manual_seed(4)
    m = GPT2DoubleHeads(GPT2Config.tiny()).to(device=dev, dtype=torch.bfloat16).eval()
    V, n, top_k, T = m.cfg.vocab_size, 3, 3, 1.0
    prompt = torch.randint(0, V, (1, 6), generator=torch.Generator().manual_seed(1)).to(dev)
    law = {(): 1.0}
    w = m.wte.weight
    with torch.no_grad():
        for t in range(n):
            nxt = {}
            for pre, p in law.items():
                seq = torch.cat([prompt, torch.tensor([pre], dtype=torch.long, device=dev)], 1) if pre else prompt
                h = m.hidden(seq, None)[:, -1].contiguous()
                lg = torch.empty(1, w.shape[0], dtype=torch.float32, device=dev)
                lm_head_logits_(h, w, lg)
                r = reference_row(lg[0, :V].cpu().numpy(), T, top_k, 1.0, 0, 0)
                e = np.where(r["kept"], r["e"], 0.0)
                for i in np.flatnonzero(r["kept"]):
                    nxt[pre + (int(i),)] = p * e[i] / e.sum()
            law = nxt
    K, B, calls = 2, 32, 40
    counts = {}
    for c in range(calls):
        tokens, n_new, _, _, _ = m.stochastic_beam_search(prompt.repeat(B, 1), num_beams=K, max_new_tokens=n,
                                                          top_k=top_k, temperature=T, seed=1000 + c * B)
        for b in range(B):
            first = tuple(tokens[b * K, :int(n_new[b * K])].tolist())
            counts[first] = counts.get(first, 0) + 1
            second = tuple(tokens[b * K + 1, :int(n_new[b * K + 1])].tolist())
            assert second != first and second in law
    N = B * calls
    assert set(counts) <= set(law)
    seqs = sorted(law, key=lambda s: -law[s])
    big = [s for s in seqs if law[s] * N >= 5]
    got = [counts.get(s, 0) for s in big] + [N - sum(counts.get(s, 0) for s in big)]
    want = [law[s] * N for s in big] + [N - sum(law[s] * N for s in big)]
    if want[-1] < 5:
        got, want = got[:-2] + [got[-2] + got[-1]], want[:-2] + [want[-2] + want[-1]]
    p = chisquare(got, want).pvalue
    print(f"tiny bf16 stochastic beam search, first reply vs generate's law: {len(law)} sequences, p = {p:.3g}")
    assert p > 1e-3


def test_limits_raise_before_launch(dev):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.ops import SAMPLE_MAX_VOCAB, BeamState, beam_step_
    from adapcc_b200.runtime.native import load_library

    lib = load_library(build_if_missing=False)
    m = _gpt2_small(dev, seed=3)
    ids = torch.zeros(13, 8, dtype=torch.long, device=dev)
    before = lib.adapcc_launch_count()
    with pytest.raises(ValueError, match="beam rows"):
        m.stochastic_beam_search(ids, num_beams=5)                        # 13 x 5 = 65 rows
    tokens, n_new, _, _, _ = m.stochastic_beam_search(ids[:8, :4], num_beams=8, max_new_tokens=2)   # 64 rows run
    assert tokens.shape == (64, 2) and (n_new == 2).all()
    torch.manual_seed(0)
    big = GPT2DoubleHeads(GPT2Config(vocab_size=SAMPLE_MAX_VOCAB + 8, n_positions=64, n_embd=64, n_layer=1, n_head=4,
                                     lm_chunk_rows=64)).to(device=dev, dtype=torch.bfloat16).eval()
    before = lib.adapcc_launch_count()
    with pytest.raises(ValueError, match="vocab"):
        big.stochastic_beam_search(ids[:2], num_beams=2, max_new_tokens=3)
    assert lib.adapcc_launch_count() == before
    st = BeamState(1, 2, 4, 1.0, dev, seeds=torch.zeros(1, dtype=torch.int64))
    lg = torch.zeros(2, SAMPLE_MAX_VOCAB + 64, device=dev)
    with pytest.raises(ValueError, match="vocab"):
        beam_step_(lg, SAMPLE_MAX_VOCAB + 1, st)
    with pytest.raises(ValueError, match="seeds"):
        beam_step_(lg, 100, st, seeds=torch.zeros(1, dtype=torch.int64, device=dev))
