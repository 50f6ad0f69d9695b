"""The sampler's truncation filters (min-p, typical, epsilon, eta) on the GPU: ``sample_tokens_`` against the fp64
definition (ops/sampling.py) with derived exemption bounds, edge cases, the distribution of the draws, bit-identity
with the filters off, graph and batch invariance, and ``GPT2DoubleHeads.generate`` on GPT-2 small."""
import ctypes
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # unit roundoff of fp32
OFF = dict(min_p=0.0, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


class _State:
    def __init__(self, dev, B, max_new=4, step=0, seeds=None, pos=None):
        self.seeds = seeds if seeds is not None else torch.arange(B, dtype=torch.int64, device=dev) * 7919 + 3
        self.pos = pos if pos is not None else torch.arange(B, dtype=torch.int32, device=dev) % 977
        self.step = torch.full((1,), step, dtype=torch.int32, device=dev)
        self.done = torch.zeros(B, dtype=torch.int32, device=dev)
        self.next_ids = torch.full((B,), -5, dtype=torch.int64, device=dev)
        self.tokens = torch.full((B, max_new), -7, dtype=torch.int64, device=dev)


def _sample(logits, vocab, T, k, p, st, min_new=0, suppress=(), stop=(), **f):
    from adapcc_b200.ops import sample_tokens_

    dev = logits.device
    sup = torch.tensor(list(suppress), dtype=torch.int32, device=dev) if suppress else None
    stp = torch.tensor(list(stop), dtype=torch.int32, device=dev) if stop else None
    sample_tokens_(logits, vocab, T, k, p, st.seeds, st.pos, st.step, min_new, sup, stp, st.done, st.next_ids,
                   st.tokens, **f)
    return st


def _logits(dev, B, V, seed, scale=3.0):
    g = torch.Generator(device=dev).manual_seed(seed)
    l = torch.randn(B, V, device=dev, generator=g) * scale
    srt = torch.sort(l, dim=1, descending=True)
    for r in range(0, B, 2):                         # tied values among the top ones and deeper in the row
        idx = srt.indices[r]
        l[r, idx[3]] = l[r, idx[2]]
        l[r, idx[min(V - 1, 200)]] = l[r, idx[min(V - 1, 199)]]
    return l


def _near(r, V):
    """The kernel may pick another token only where a decision sits at its threshold within the fp32 error.

    e_i = expf(x_i - m) is within (4 + |y_i|) u of the exact weight (y = x - m rounded, expf within 2 ulp). A sum
    over any subset of the ids kept by top-k has at most C + 72 roundings on any path (C = ceil(V / 1024) per
    thread, the shuffle trees, the warp partials and up to 32 chained bisection sums), so its error is at most
    errZ = (C + 74) u Z + 2 sum of the weight errors, Z the top-k weight. mu = s1 / Z_K adds the error of s1 (the same
    argument over e_i |y_i|, and one rounding of y per term) and of the division. Each threshold adds a few roundings
    (the product with Z, sqrtf and expf). Every bound below is twice the sum of the errors of the two compared sides."""
    if "e" not in r:
        return False
    C = math.ceil(V / 1024)
    S = (C + 74) * U32
    e = r["e"]
    ya = np.where(e > 0, -np.log(np.maximum(e, 1e-300)), 0.0)
    errZ = S * r["Z"] + 2 * float(((4 + ya) * U32 * e).sum())
    A = float((e * ya).sum())
    err_s1 = S * A + 2 * float(((5 + ya) * U32 * e * ya).sum())
    for name, f in r["filters"].items():
        q = f["q"]
        live = np.isfinite(q)
        if name == "min_p":
            if np.any(np.abs(q[live] - f["thr"]) <= 2 * ((4 + ya[live]) * U32 * q[live] + U32 * f["thr"])):
                return True
            continue
        ZK, mu = f["Z"], f["mu"]
        err_mu = err_s1 / ZK + abs(mu) * errZ / ZK + U32 * abs(mu)
        if name == "typical":
            err_d = lambda d: err_mu + U32 * (3 * d + 2 * abs(mu))   # noqa: E731
            other = live & (q != f["thr"])
            if np.any(np.abs(q[other] - f["thr"]) <= 2 * (err_d(q[other]) + err_d(f["thr"]))):
                return True
            if np.any(np.abs(f["G"] - f["pZ"]) <= 2 * (2 * errZ + U32 * f["pZ"])):
                return True
            continue
        rel_thr = errZ / ZK + 2 * U32 + (err_mu + 3 * U32 if name == "eta" else 0.0)
        if np.any(np.abs(q[live] - f["thr"]) <= 2 * ((4 + ya[live]) * U32 * q[live] + rel_thr * f["thr"])):
            return True
    return bool((np.abs(r["cum"][r["kept"]] - r["target"]) <= S * r["Z"] + 2 * float(((4 + ya) * U32 * e).sum())).any()
                or (r["pZ"] < r["Z"] and (np.abs(r["tail"][np.isfinite(r["tail"])] - r["pZ"])
                                          <= S * r["Z"] + 2 * float(((4 + ya) * U32 * e).sum())).any()))


CASES = [(0.7, 0, 1.0, dict(min_p=0.05)), (1.0, 0, 1.0, dict(typical_p=0.9)), (0.8, 0, 1.0, dict(typical_p=0.3)),
         (1.0, 0, 1.0, dict(epsilon_cutoff=3e-4)), (1.0, 0, 1.0, dict(eta_cutoff=3e-4)),
         (0.9, 50, 0.95, dict(min_p=0.02, typical_p=0.9, epsilon_cutoff=1e-4, eta_cutoff=1e-4)),
         (1.2, 200, 0.9, dict(typical_p=0.5, eta_cutoff=1e-3)), (0.7, 0, 0.9, dict(min_p=0.1, epsilon_cutoff=1e-3))]


def test_sampler_with_filters_matches_fp64_definition(dev):
    from adapcc_b200.ops.sampling import reference_row

    rows = exempt = 0
    for ci, (T, k, p, f) in enumerate(CASES):
        for V, B in ((3001, 128), (50262, 64)):
            l = _logits(dev, B, V + 5, seed=300 + 10 * ci + V % 7)
            st = _sample(l, V, T, k, p, _State(dev, B), **f)
            torch.cuda.synchronize()
            got = st.next_ids.cpu().tolist()
            lc, seeds, pos = l.cpu().numpy(), st.seeds.cpu().tolist(), st.pos.cpu().tolist()
            for b in range(B):
                r = reference_row(lc[b, :V], T, k, p, seeds[b], pos[b], **f)
                rows += 1
                if got[b] != r["token"]:
                    assert _near(r, V), (T, k, p, f, V, b, got[b], r["token"])
                    exempt += 1
    print(f"filtered sampler vs fp64: {rows} rows, {exempt} exempt near a threshold")
    assert rows >= 1500 and exempt <= rows // 50


def test_filter_edge_cases(dev):
    from adapcc_b200.ops.sampling import reference_row

    every = dict(min_p=0.3, typical_p=0.2, epsilon_cutoff=0.5, eta_cutoff=0.5)
    V = 1500
    one = torch.full((3, V), float("-inf"), device=dev)
    one[:, 77] = 5.0                                             # a single finite logit survives every filter
    assert _sample(one, V, 0.9, 5, 0.3, _State(dev, 3), **every).next_ids.tolist() == [77] * 3
    # uniform rows: typical keeps everything (every deviation is 0), the draw is the definition's
    B = 256
    flat = torch.full((B, V), 1.25, device=dev)
    st = _sample(flat, V, 0.8, 0, 1.0, _State(dev, B), typical_p=0.3, eta_cutoff=1e-4)
    torch.cuda.synchronize()
    seeds, pos = st.seeds.cpu().tolist(), st.pos.cpu().tolist()
    for b in range(B):
        r = reference_row(flat[b].cpu().numpy(), 0.8, 0, 1.0, seeds[b], pos[b], typical_p=0.3, eta_cutoff=1e-4)
        assert r["kept"].all() and (int(st.next_ids[b]) == r["token"] or _near(r, V)), b
    assert len(set(st.next_ids.tolist())) > B // 2
    # typical drops the arg-max of a peaked row: p_0 = 0.13, the others are closer to the entropy
    peak = torch.zeros(B, 1000, device=dev)
    peak[:, 0] = 5.0
    st = _sample(peak, 1000, 1.0, 0, 1.0, _State(dev, B), typical_p=0.8)
    assert int((st.next_ids == 0).sum()) == 0 and len(set(st.next_ids.tolist())) > B // 2
    # suppressed ids are never drawn while step < min_new, with the filters applied to what remains
    l = torch.full((B, V), -20.0, device=dev)
    l[:, :4] = 10.0
    st = _sample(l, V, 1.0, 0, 1.0, _State(dev, B, step=0), min_new=1, suppress=(0, 1, 2), **every)
    assert int((st.next_ids == 3).sum()) == B
    st = _sample(l, V, 1.0, 0, 1.0, _State(dev, B, step=1), min_new=1, suppress=(0, 1, 2), typical_p=0.9)
    torch.cuda.synchronize()
    assert set(st.next_ids.tolist()) <= {0, 1, 2, 3} and len(set(st.next_ids.tolist())) == 4
    # done rows draw nothing
    st = _State(dev, 4, max_new=3, step=1)
    st.done[[1, 3]] = 1
    st.tokens[1] = 123
    _sample(_logits(dev, 4, V, seed=5), V, 0.9, 0, 0.9, st, **every)
    torch.cuda.synchronize()
    assert st.tokens[1].tolist() == [123, -1, 123] and int(st.tokens[3, 1]) == -1
    assert st.next_ids[[1, 3]].tolist() == [0, 0] and st.done.tolist() == [0, 1, 0, 1]
    assert bool((st.tokens[[0, 2], 1] >= 0).all())


@pytest.mark.parametrize("f", [dict(typical_p=0.5), dict(eta_cutoff=0.02)])
def test_filtered_draws_chi_square(dev, f):
    from scipy.stats import chisquare

    from adapcc_b200.ops.sampling import reference_row

    V, n, B = 40, 1 << 16, 4096
    base = torch.linspace(2.0, -3.0, V, device=dev)
    base[5] = base[4]                                            # a tie inside the kept set
    T = 0.8
    counts = np.zeros(V)
    for c in range(n // B):
        pos = torch.arange(c * B, (c + 1) * B, dtype=torch.int32, device=dev)
        st = _State(dev, B, seeds=torch.full((B,), 4242, dtype=torch.int64, device=dev), pos=pos)
        _sample(base.expand(B, V).contiguous(), V, T, 0, 1.0, st, **f)
        counts += np.bincount(st.next_ids.cpu().numpy(), minlength=V)
    r = reference_row(base.cpu().numpy(), T, 0, 1.0, 0, 0, **f)
    assert not _near({**r, "cum": np.full(V, np.inf)}, V)        # the kept set is not at a threshold
    kept = r["kept"]
    assert 3 < int(kept.sum()) < V - 3
    prob = np.where(kept, r["e"], 0.0) / r["Zp"]
    assert counts[~kept].sum() == 0
    stat = chisquare(counts[kept], prob[kept] * n)
    assert stat.pvalue > 1e-3, stat


def test_filters_off_give_the_same_bits(dev):
    from adapcc_b200.ops import _lib, _ptr, _stream

    V, B = 50262, 64
    for T, k, p in ((0.7, 0, 0.9), (1.0, 40, 0.95), (0.0, 0, 1.0)):
        l = _logits(dev, B, V, seed=int(T * 10) + k)
        a = _sample(l, V, T, k, p, _State(dev, B, max_new=2))
        b = _sample(l, V, T, k, p, _State(dev, B, max_new=2), **OFF)
        c = _State(dev, B, max_new=2)                            # the C entry point without the filter arguments
        rc = _lib().adapcc_sample_tokens(_ptr(l), V, V, B, ctypes.c_float(T), k, ctypes.c_float(p), _ptr(c.seeds),
                                         _ptr(c.pos), _ptr(c.step), 0, None, 0, None, 0, _ptr(c.done),
                                         _ptr(c.next_ids), _ptr(c.tokens), 2, _stream())
        assert rc == 0
        torch.cuda.synchronize()
        assert torch.equal(a.tokens, b.tokens) and torch.equal(a.tokens, c.tokens) and int(c.step) == 1


def test_filtered_sampler_graph_equals_eager_and_rows_do_not_depend_on_batch(dev):
    V, B = 50262, 16
    f = dict(min_p=0.01, typical_p=0.9, epsilon_cutoff=1e-4, eta_cutoff=1e-4)
    l = _logits(dev, B, V, seed=21)
    st = _State(dev, B, max_new=8)
    for _ in range(8):
        _sample(l, V, 0.9, 40, 0.95, st, **f)
        st.pos += 1
    eager = st.tokens.clone()
    st = _State(dev, B, max_new=8)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _sample(l, V, 0.9, 40, 0.95, st, **f)
    torch.cuda.current_stream().wait_stream(s)
    st.step.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _sample(l, V, 0.9, 40, 0.95, st, **f)
        st.pos.add_(1)
    for _ in range(8):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager, st.tokens) and int(st.step) == 8
    full = _State(dev, B, max_new=1)
    _sample(l, V, 0.9, 0, 0.9, full, **f)
    for b in (0, 5, 15):
        alone = _State(dev, 1, max_new=1, seeds=full.seeds[b:b + 1].clone(), pos=full.pos[b:b + 1].clone())
        _sample(l[b:b + 1].contiguous(), V, 0.9, 0, 0.9, alone, **f)
        assert int(alone.next_ids[0]) == int(full.next_ids[b]), b


# random GPT-2 weights give flat rows (entropy near log V), where eta's threshold sqrt(eta) exp(-H) needs a large eta
# to reach the ids' probabilities
@pytest.mark.parametrize("f", [dict(min_p=0.05), dict(typical_p=0.9), dict(epsilon_cutoff=3e-4),
                               dict(eta_cutoff=0.3),
                               dict(min_p=0.02, typical_p=0.8, epsilon_cutoff=1e-4, eta_cutoff=1e-4)])
def test_generate_gpt2_small_with_filters_equals_host_loop(dev, f):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.ops import lm_head_logits_
    from adapcc_b200.ops.sampling import reference_row

    torch.manual_seed(0)
    m = GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(8)
    lengths = [90, 37, 64, 1, 80, 12]
    B, n = len(lengths), 24
    ids = torch.randint(0, V, (B, 90), device=dev, generator=g)
    T, k, p = 0.5, 0, 0.9
    tokens, n_new = m.generate(ids, lengths, max_new_tokens=n, temperature=T, top_k=k, top_p=p, seed=77, **f)
    assert n_new.tolist() == [n] * B
    # the same steps eagerly: the LM head kernel's logits at every step, fed the tokens generate drew
    w = m.wte.weight
    cache = m.new_cache(B, max(lengths) + n)
    last = torch.tensor(lengths, device=dev) - 1
    exempt = 0
    with torch.no_grad():
        h = m.hidden(ids, None, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last]
        logits = torch.empty(B, w.shape[0], dtype=torch.float32, device=dev)
        for i in range(n):
            if i:
                h = m.decode_step(tokens[:, i - 1].contiguous(), None, cache)
            lm_head_logits_(h, w, logits)
            lc, pos = logits[:, :V].cpu().numpy(), cache.lens.cpu().tolist()
            for b in range(B):
                r = reference_row(lc[b], T, k, p, 77 + b, pos[b], **f)
                if r["token"] != int(tokens[b, i]):
                    assert _near(r, V), (f, b, i)
                    exempt += 1
    print(f"generate {f}: {B * n} draws, {exempt} exempt near a threshold")
    assert exempt <= B * n // 20
    assert not torch.equal(tokens, m.generate(ids, lengths, max_new_tokens=n, temperature=T, top_k=k, top_p=p,
                                              seed=77)[0])
