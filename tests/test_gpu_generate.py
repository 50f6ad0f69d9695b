"""Sampled generation on the GPU: the bf16 LM-head kernel against fp64, the sampling kernel against the fp64
definition (ops/sampling.py) with a derived exemption bound, its edge cases, distribution and repeatability, and
``GPT2DoubleHeads.generate`` on GPT-2 small."""
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


def _head(h, w):
    from adapcc_b200.ops import lm_head_logits_

    out = torch.full((h.shape[0], w.shape[0]), float("nan"), dtype=torch.float32, device=h.device)
    return lm_head_logits_(h, w, out)


@pytest.mark.parametrize("V", [50304, 1003])
def test_lm_head_against_fp64_and_batch_invariant(dev, V):
    """Every product of two bf16 values is exact in fp32. A lane adds its D / 32 products in order with fused
    multiply-adds and a 5-level shuffle tree adds the lanes, so each output is a sum of D exact terms evaluated with
    at most D / 32 + 5 roundings on any path: |err| <= (D / 32 + 6) u32 sum_d |h_d w_d| (the +1 covers the bound's
    first-order slack)."""
    g = torch.Generator(device=dev).manual_seed(V)
    D = 768
    w = (torch.randn(V, D, device=dev, generator=g) * 0.05).to(torch.bfloat16)
    hb = torch.randn(64, D, device=dev, generator=g).to(torch.bfloat16)
    single = torch.stack([_head(hb[b:b + 1], w)[0] for b in range(64)])
    for B in (1, 7, 8, 64):
        h = hb[:B]
        out = _head(h, w)
        torch.cuda.synchronize()
        ref = h.double() @ w.double().t()
        bound = (D / 32 + 6) * U32 * (h.double().abs() @ w.double().abs().t())
        assert bool(((out.double() - ref).abs() <= bound).all()), (B, float((out.double() - ref).abs().max()))
        assert torch.equal(out.view(torch.int32), single[:B].view(torch.int32)), B
    # a strided h (rows of a wider buffer) gives the same bits
    wide = torch.zeros(8, D + 64, dtype=torch.bfloat16, device=dev)
    wide[:, :D] = hb[:8]
    assert torch.equal(_head(wide[:, :D], w).view(torch.int32), single[:8].view(torch.int32))
    with pytest.raises(ValueError, match="lm_head_logits_"):
        _head(torch.zeros(65, D, dtype=torch.bfloat16, device=dev), w)


class _State:
    def __init__(self, dev, B, max_new=4, step=0, seeds=None, pos=None):
        self.seeds = seeds if seeds is not None else torch.arange(B, dtype=torch.int64, device=dev) * 7919 + 3
        self.pos = pos if pos is not None else torch.arange(B, dtype=torch.int32, device=dev) % 977
        self.step = torch.full((1,), step, dtype=torch.int32, device=dev)
        self.done = torch.zeros(B, dtype=torch.int32, device=dev)
        self.next_ids = torch.full((B,), -5, dtype=torch.int64, device=dev)
        self.tokens = torch.full((B, max_new), -7, dtype=torch.int64, device=dev)


def _sample(logits, vocab, T, k, p, st, min_new=0, suppress=(), stop=()):
    from adapcc_b200.ops import sample_tokens_

    dev = logits.device
    sup = torch.tensor(list(suppress), dtype=torch.int32, device=dev) if suppress else None
    stp = torch.tensor(list(stop), dtype=torch.int32, device=dev) if stop else None
    sample_tokens_(logits, vocab, T, k, p, st.seeds, st.pos, st.step, min_new, sup, stp, st.done, st.next_ids,
                   st.tokens)
    return st


def _logits(dev, B, V, seed, scale=3.0, ties=True):
    g = torch.Generator(device=dev).manual_seed(seed)
    l = torch.randn(B, V, device=dev, generator=g) * scale
    if ties:
        # plant ties at the places thresholds fall: among the top values, and deeper where top-k / top-p cut
        srt = torch.sort(l, dim=1, descending=True)
        for r in range(0, B, 2):
            idx = srt.indices[r]
            j = int(torch.randint(0, min(V - 1, 60), (1,), generator=torch.Generator().manual_seed(seed + r)))
            l[r, idx[j + 1]] = l[r, idx[j]]
            l[r, idx[min(V - 1, 20)]] = l[r, idx[min(V - 1, 19)]]
    return l


def _margin_ok(r, V):
    """The kernel may pick another token only where a decision quantity sits at its threshold within the fp32 error.

    Weights: x - m is rounded (u32 |x - m| relative in the exponent) and expf is within 2 ulp, so each e_i is within
    (4 + |x_i - m|) u32 relative. Sums: a thread adds at most C = ceil(V / 1024) terms in order, a 5-level shuffle tree
    and 32 warp partials follow, the bisection chains at most 32 further partial sums and the prefix adds one offset:
    at most C + 72 roundings per path, so every sum S is within (C + 72) u32 S plus the weight errors. p Z and u Z' each
    add one rounding."""
    if "e" not in r:
        return False
    C = math.ceil(V / 1024)
    xm = np.where(r["e"] > 0, -np.log(np.maximum(r["e"], 1e-300)), 0.0)
    weight_err = float(((4 + xm) * U32 * r["e"]).sum())
    bound = (C + 74) * U32 * r["Z"] + 2 * weight_err
    tail = r["tail"][np.isfinite(r["tail"])]
    near_p = r["pZ"] < r["Z"] and bool((np.abs(tail - r["pZ"]) <= bound).any())
    near_draw = bool((np.abs(r["cum"][r["kept"]] - r["target"]) <= bound).any())
    return near_p or near_draw


CASES = [(0.7, 0, 0.9), (1.0, 20, 1.0), (0.8, 50, 0.95), (1.3, 0, 0.5), (0.5, 3, 0.99), (1.0, 0, 1.0),
         (0.9, 200, 0.7), (2.0, 1, 0.9)]


def test_sampler_matches_fp64_definition(dev):
    from adapcc_b200.ops.sampling import reference_row

    rows = exempt = 0
    for ci, (T, k, p) in enumerate(CASES):
        for V, B in ((3001, 384), (50262, 64)):
            l = _logits(dev, B, V + 5, seed=100 * ci + V % 7)
            st = _sample(l, V, T, k, p, _State(dev, B))
            torch.cuda.synchronize()
            got = st.next_ids.cpu().tolist()
            lc, seeds, pos = l.cpu().numpy(), st.seeds.cpu().tolist(), st.pos.cpu().tolist()
            for b in range(B):
                r = reference_row(lc[b, :V], T, k, p, seeds[b], pos[b])
                rows += 1
                if got[b] != r["token"]:
                    assert _margin_ok(r, V), (T, k, p, V, b, got[b], r["token"])
                    exempt += 1
    print(f"sampler vs fp64: {rows} rows, {exempt} exempt")
    assert rows >= 3000 and exempt <= rows // 100


def test_sampler_edge_cases(dev):
    V = 1500                                                    # not a multiple of the 1024-thread block
    l = _logits(dev, 6, V, seed=9, ties=False)
    l[1] = float("-inf")
    l[1, 1234] = -2.0                                            # a single finite logit
    l[2, [17, 900, 1400]] = 40.0                                 # greedy ties: the lowest index wins
    st = _State(dev, 6, max_new=3, step=1)
    st.done[4] = 1
    st.tokens[4] = 123
    _sample(l, V, 0.0, 0, 0.9, st)
    torch.cuda.synchronize()
    assert int(st.next_ids[1]) == 1234 and int(st.next_ids[2]) == 17
    assert st.tokens[:, 1].tolist() == [int(l[0].argmax()), 1234, 17, int(l[3].argmax()), -1, int(l[5].argmax())]
    assert st.tokens[4].tolist() == [123, -1, 123] and st.done.tolist() == [0, 0, 0, 0, 1, 0]
    assert (st.tokens[:, [0, 2]][[0, 1, 2, 3, 5]] == -7).all() and int(st.step) == 2
    # sampled: the single finite logit is drawn at any k and p; suppressed ids are never drawn while step < min_new;
    # a stop id ends the row
    B = 512
    l = torch.full((B, V), -20.0, device=dev)
    l[:, :4] = 10.0
    st = _State(dev, B, step=0)
    _sample(l, V, 1.0, 0, 1.0, st, min_new=1, suppress=(0, 1, 2))
    torch.cuda.synchronize()
    assert int((st.next_ids == 3).sum()) == B                   # id 3 holds all but 1500 e^-30 of the remaining mass
    st = _State(dev, B, step=1)
    _sample(l, V, 1.0, 0, 1.0, st, min_new=1, suppress=(0, 1, 2), stop=(0,))
    torch.cuda.synchronize()
    stopped = st.next_ids == 0
    assert 0 < int(stopped.sum()) < B
    assert torch.equal(st.done.bool(), stopped) and bool((st.tokens[stopped, 1] == -1).all())
    assert torch.equal(st.tokens[~stopped, 1], st.next_ids[~stopped])
    one = torch.full((3, V), float("-inf"), device=dev)
    one[:, 77] = 5.0
    st = _sample(one, V, 0.9, 5, 0.3, _State(dev, 3))
    assert st.next_ids.tolist() == [77] * 3
    with pytest.raises(ValueError, match="sample_tokens_"):
        _sample(torch.zeros(2, 60000, device=dev), 60000, 1.0, 0, 0.9, _State(dev, 2))
    for T, k, p in ((-1.0, 0, 0.9), (1.0, -1, 0.9), (1.0, 0, 0.0), (1.0, 0, 1.1)):
        with pytest.raises(ValueError, match="sample_tokens_"):
            _sample(torch.zeros(2, 100, device=dev), 100, T, k, p, _State(dev, 2))


def test_sampler_distribution_chi_square(dev):
    from scipy.stats import chisquare

    from adapcc_b200.ops.sampling import reference_row

    V, n = 40, 1 << 16
    base = torch.linspace(2.0, -3.0, V, device=dev)
    base[5] = base[4]                                            # a tie inside the nucleus
    T, k, p = 0.8, 12, 0.9
    counts = np.zeros(V)
    B = 4096
    for c in range(n // B):
        pos = torch.arange(c * B, (c + 1) * B, dtype=torch.int32, device=dev)
        st = _State(dev, B, seeds=torch.full((B,), 12345, dtype=torch.int64, device=dev), pos=pos)
        _sample(base.expand(B, V).contiguous(), V, T, k, p, st)
        counts += np.bincount(st.next_ids.cpu().numpy(), minlength=V)
    r = reference_row(base.cpu().numpy(), T, k, p, 0, 0)
    prob = np.where(r["kept"], r["e"], 0.0) / r["Zp"]
    assert counts[~r["kept"]].sum() == 0
    stat = chisquare(counts[r["kept"]], prob[r["kept"]] * n)
    assert stat.pvalue > 1e-3, stat


def test_sampler_repeatable_and_graph_equals_eager(dev):
    V, B = 50262, 16
    l = _logits(dev, B, V, seed=21)
    runs = []
    for _ in range(2):
        st = _State(dev, B, max_new=8)
        for _ in range(8):
            _sample(l, V, 0.9, 40, 0.9, st)
            st.pos += 1
        runs.append(st.tokens.clone())
    st = _State(dev, B, max_new=8)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _sample(l, V, 0.9, 40, 0.9, st)
    torch.cuda.current_stream().wait_stream(s)
    st.step.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _sample(l, V, 0.9, 40, 0.9, st)
        st.pos.add_(1)
    for _ in range(8):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], st.tokens) and int(st.step) == 8


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def test_generate_gpt2_small(dev):
    from adapcc_b200.models.gpt2 import DecodeGraph

    m = _gpt2_small(dev)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(4)
    # top_k = 1 follows the existing cached greedy loop (DecodeGraph + fp32 head arg-max) up to the first near tie
    prompt = torch.randint(0, V, (1, 200), device=dev, generator=g)
    tokens, n_new = m.generate(prompt, max_new_tokens=32, top_k=1, seed=5)
    assert n_new.tolist() == [32]
    cache = m.new_cache(1)
    head = m.wte.weight.float()
    with torch.no_grad():
        h = m.hidden(prompt, None, cache=cache)[:, -1]
        step = DecodeGraph(m, cache, token_types=False)
        for i in range(32):
            logits = (h.float() @ head.t())[0, :V]
            top2 = torch.topk(logits, 2).values
            if float(top2[0] - top2[1]) < 0.1:
                break
            assert int(tokens[0, i]) == int(logits.argmax()), i
            h = step(tokens[0, i:i + 1])
    # ragged batch of 8: each row draws what it draws alone, up to its first near tie of the sampling decision
    lengths = [200, 37, 128, 1, 64, 199, 150, 90]
    ids = torch.randint(0, V, (8, 200), device=dev, generator=g)
    tt = torch.randint(V - 5, V - 3, (8, 200), device=dev, generator=g)
    kw = dict(max_new_tokens=40, temperature=0.8, top_k=0, top_p=0.9)
    tokens, _ = m.generate(ids, lengths, tt, seed=77, **kw)
    again, _ = m.generate(ids, lengths, tt, seed=77, **kw)
    assert torch.equal(tokens, again)
    from adapcc_b200.ops.sampling import reference_row

    for b, n in enumerate(lengths):
        alone, _ = m.generate(ids[b:b + 1, :n], None, tt[b:b + 1, :n], seed=torch.tensor([77 + b]), **kw)
        k = 0
        while k < 40 and int(alone[0, k]) == int(tokens[b, k]):
            k += 1
        if k == 40:
            continue
        # the bf16 GEMMs of a padded batch may round differently from the row alone: the first differing draw must
        # be a near tie, a decision quantity within 2 % of the mass of its threshold
        seq = torch.cat([ids[b, :n], tokens[b, :k]])[None]
        types = torch.cat([tt[b, :n], tt[b, n - 1].expand(k)])[None]
        with torch.no_grad():
            logits = (m.hidden(seq, types)[0, -1].float() @ head.t())[:V].cpu().numpy()
        r = reference_row(logits, 0.8, 0, 0.9, 77 + b, n + k)
        tail = r["tail"][np.isfinite(r["tail"])]
        near = (np.abs(r["cum"][r["kept"]] - r["target"]).min() <= 0.02 * r["Zp"]
                or np.abs(tail - r["pZ"]).min() <= 0.02 * r["Z"])
        assert near, (b, k)
    # a stop id ends rows with -1 padding
    stop = int(tokens[3, 5])
    got, n_new = m.generate(ids, lengths, tt, seed=77, stop_ids=[stop], **kw)
    for b in range(8):
        k = int(n_new[b])
        assert (got[b, k:] == -1).all() and (got[b, :k] >= 0).all() and stop not in got[b, :k].tolist()
    assert int(n_new[3]) <= 5
