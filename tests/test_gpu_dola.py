"""DoLa layer contrast on the GPU: the two kernels against the fp64 definition (ops/dola.py) with error bounds derived
from their fp32 order of operations, their batch invariance, graph capture and repeatability, and
``GPT2DoubleHeads.generate(dola_layers=)`` on GPT-2 small (random init, bf16) against an eager loop of the model's own
pieces and against the fp64 decision."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # unit roundoff of fp32
TINY = 2.0 ** -148        # twice the smallest fp32 subnormal: what an underflowing exp or product can lose


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _run(x, vocab, B, C):
    """(scores buffer, the kernel's JS [C, B]) of ``dola_contrast_`` on a copy of ``x``."""
    from adapcc_b200.ops import dola_contrast_, dola_work_numel

    out = x.clone()
    work = torch.full((dola_work_numel(B, C),), float("nan"), dtype=torch.float32, device=x.device)
    dola_contrast_(out, vocab, B, C, work)
    return out, work.view(C + 1, B, 4)[:C, :, 0]


def _lsm_err(x, C):
    """fp64 (log-softmax l, its error bound, the log-sum's error bound) of the rows x [..., V] as the kernel computes
    them (csrc/ops_dola.cu). The maximum m is exact. d_i = fl(x_i - m) is within |d_i| u; expf is within 2 ulp, so
    e_i = expf(d_i) is within (4 + |d_i|) u e_i. S adds positive terms with at most C + 10 roundings on any path
    (C = ceil(vocab / 1024) in a thread, 5 shuffle levels over lanes, 5 over warps): |dS| <= (C + 10) u S +
    sum (4 + |d_i|) u e_i. logf is within 1 ulp, so |d log S| <= |dS| / S + 2 u |log S|, and l_i = fl(d_i - log S) is
    within |d_i| u + |d log S| + |l_i| u."""
    d = x - x.max(-1, keepdim=True).values
    e = d.exp()
    S = e.sum(-1, keepdim=True)
    dS = (C + 10) * U32 * S + ((4 + d.abs()) * U32 * e).sum(-1, keepdim=True)
    dlog = dS / S + 2 * U32 * S.log().abs()
    lsm = d - S.log()
    return lsm, d.abs() * U32 + dlog + lsm.abs() * U32, dlog


def _bounds(f, q, vocab):
    """Per-element score bounds [C, B, V] (lf_i - lq_j,i of every candidate j), JS bounds [C, B], and lf, its error,
    and the threshold's error [B] for the kept set; f [B, V], q [C, B, V] fp64.

    Scores: fl(lf - lq) is within err_lf + err_lq + |lf - lq| u. JS: pf = expf(lf) is within (err_lf + 4 u) pf plus
    an absolute TINY where it underflows; M = fl(0.5 fl(pf + pq)) within r_M M + TINY, r_M = max of the two plus u.
    The term t1 = fl(M fl(log M - lf)) is within e_M |log M - lf| + e_M + M (2 u |log M| + err_lf) + M |log M - lf| u +
    |t1| u + TINY (1 + |log M - lf|), t2 alike; the sums add at most C + 10 roundings of partial sums of |t|, the means
    one more and JS = fl(0.5 fl(KL1 + KL2)) another. A factor 1.05 covers the second-order terms."""
    Cn = math.ceil(vocab / 1024)
    lf, ef, dlog_f = _lsm_err(f, Cn)
    lq, eq, _ = _lsm_err(q, Cn)
    score_b = 1.05 * (ef[None] + eq + (lf[None] - lq).abs() * U32) + 1e-30
    pf, pq = lf.exp()[None], lq.exp()
    M = 0.5 * (pf + pq)
    rM = torch.maximum(ef[None] + 4 * U32, eq + 4 * U32) + U32
    eM = rM * M + TINY
    lm = torch.where(M > 0, M.log(), torch.zeros_like(M))
    js_err = 0.0
    js = 0.0
    for l, e in ((lf[None], ef[None]), (lq, eq)):
        gap = (lm - l).abs()
        t = torch.where(M > 0, M * (lm - l), torch.zeros_like(M))
        dt = eM * gap + eM + M * (2 * U32 * lm.abs() + e) + M * gap * U32 + t.abs() * U32 + TINY * (1 + gap)
        err_sum = dt.sum(-1) + (Cn + 10) * U32 * t.abs().sum(-1)
        kl = t.sum(-1) / vocab
        js = js + 0.5 * kl
        js_err = js_err + 0.5 * (err_sum / vocab + kl.abs() * U32)
    js_b = 1.05 * (js_err + 2 * js.abs() * U32) + 1e-30
    thr = lf.max(-1).values + float(np.float32(math.log(0.1)))
    thr_err = dlog_f[..., 0] + 2 * thr.abs() * U32
    return score_b, js_b, lf, ef, thr, thr_err


def _check(x, vocab, B, C):
    """Run the kernel on x [(1 + C)·B, ld] and check it against the fp64 definition; returns the number of rows
    whose choice sat inside the JS bound."""
    from adapcc_b200.ops.dola import dola_js_reference, dola_scores_reference

    out, js_k = _run(x, vocab, B, C)
    torch.cuda.synchronize()
    ld = x.shape[1]
    # candidate rows and padding columns are never written
    assert torch.equal(out[B:].view(torch.int32), x[B:].view(torch.int32))
    assert torch.equal(out[:B, vocab:].view(torch.int32), x[:B, vocab:].view(torch.int32))
    f, q = x[:B, :vocab].double(), x[B:, :vocab].double().view(C, B, vocab)
    score_b, js_b, lf, ef, thr, thr_err = _bounds(f, q, vocab)
    near = 0
    if C > 1:
        js_ref = dola_js_reference(x[:B].cpu(), x[B:].view(C, B, ld).cpu(), vocab).to(x.device)
        assert bool(((js_k.double() - js_ref).abs() <= js_b).all()), float(((js_k.double() - js_ref).abs() - js_b).max())
        chosen_k = js_k.argmax(0)                                           # the first maximum, as the kernel picks
        chosen_r = js_ref.argmax(0)
        for b in range(B):
            ck, cr = int(chosen_k[b]), int(chosen_r[b])
            if ck != cr:
                assert js_ref[cr, b] - js_ref[ck, b] <= js_b[cr, b] + js_b[ck, b], (b, ck, cr)
                near += 1
    else:
        chosen_k = torch.zeros(B, dtype=torch.int64, device=x.device)
    rows = torch.arange(B, device=x.device)
    base = x[B:].view(C, B, ld)[chosen_k, rows]
    ref, _ = dola_scores_reference(x[:B], base[None], vocab)
    got = out[:B, :vocab].double()
    kept_k, kept_r = torch.isfinite(got), torch.isfinite(ref)
    margin = (lf - thr[:, None]).abs() <= ef + thr_err[:, None]
    assert bool((kept_k == kept_r)[~margin].all())
    assert bool(kept_k.any(1).all())                                        # the arg-max of lf is always kept
    both = kept_k & kept_r
    sb = score_b[chosen_k, rows]
    assert bool(((got - ref).abs() <= sb)[both].all()), float(((got - ref).abs() - sb)[both].max())
    return near


def _logits(dev, B, C, ld, seed, large=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn((1 + C) * B, ld, device=dev, generator=g) * 4
    x[B::3] *= 3                                                # candidates of several sharpnesses
    x[1::4, :5] += 30.0                                         # spikes that hold nearly all the mass
    if large:                                                   # raw residual streams through the head
        x[B:] = x[B:] * 60 + 400
    return x


@pytest.mark.parametrize("vocab,ld", [(50257, 50304), (1000, 1010), (7, 8)])
@pytest.mark.parametrize("C", [1, 2, 3, 16])
def test_kernels_against_fp64_definition(dev, vocab, ld, C):
    near = 0
    for B in (1, 5, 64):
        for large in (False, True):
            x = _logits(dev, B, C, ld, seed=B * 31 + C + vocab + large, large=large)
            x[:, vocab:] = float("nan")                         # padding columns: never read, never written
            near += _check(x, vocab, B, C)
    assert near <= 2


def test_duplicate_candidates_and_a_candidate_equal_to_the_final_row(dev):
    V, ld, B, C = 50257, 50304, 5, 4
    x = _logits(dev, B, C, ld, seed=3)
    view = x[B:].view(C, B, ld)
    view[2] = view[0]                                           # a duplicate: bit-equal JS, the first one wins ties
    view[3] = x[:B]                                             # the final row itself: JS within its bound of 0
    _check(x, V, B, C)
    _, js = _run(x, V, B, C)
    assert torch.equal(js[0].view(torch.int32), js[2].view(torch.int32))
    f, q = x[:B, :V].double(), x[B:, :V].double().view(C, B, V)
    js_b = _bounds(f, q, V)[1]
    assert bool((js[3].double().abs() <= js_b[3]).all())
    # every candidate a copy of one row: the choice is the first
    y = _logits(dev, B, C, ld, seed=4)
    yv = y[B:].view(C, B, ld)
    for j in range(1, C):
        yv[j] = yv[0]
    _, js = _run(y, V, B, C)
    assert int((js.argmax(0) != 0).sum()) == 0


def test_rows_alone_graph_replay_and_repeat_runs_are_bit_identical(dev):
    from adapcc_b200.ops import dola_contrast_, dola_work_numel

    V, ld, B, C = 50257, 50264, 16, 3
    x = _logits(dev, B, C, ld, seed=5, large=True)
    out, _ = _run(x, V, B, C)
    again, _ = _run(x, V, B, C)
    assert torch.equal(out.view(torch.int32), again.view(torch.int32))
    xv = x[B:].view(C, B, ld)
    for b in range(B):
        alone, _ = _run(torch.cat([x[b:b + 1], xv[:, b]]), V, 1, C)
        assert torch.equal(alone[0].view(torch.int32), out[b].view(torch.int32)), b
    sub, _ = _run(torch.cat([x[:7], xv[:, :7].reshape(C * 7, ld)]), V, 7, C)
    assert torch.equal(sub[:7].view(torch.int32), out[:7].view(torch.int32))
    buf = x.clone()
    work = torch.empty(dola_work_numel(B, C), dtype=torch.float32, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dola_contrast_(buf, V, B, C, work)                      # warm-up
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        dola_contrast_(buf, V, B, C, work)
    for _ in range(2):
        buf.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(buf.view(torch.int32), out.view(torch.int32))


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


@pytest.fixture(scope="module")
def small(dev):
    return _gpt2_small(dev)


def _inputs(dev, V, B=6, seed=4):
    g = torch.Generator(device=dev).manual_seed(seed)
    lengths = [90, 17, 64, 1, 40, 77][:B]
    ids = torch.randint(0, V - 5, (B, 90), device=dev, generator=g)
    tt = torch.randint(V - 5, V - 3, (B, 90), device=dev, generator=g)
    return ids, lengths, tt


@torch.no_grad()
def _eager(m, ids, lengths, tt, layers, n, temperature=0.0, top_k=0, top_p=1.0, seed=0, penalty=1.0, kv=None,
           keep=None):
    """``generate(dola_layers=layers)`` as an eager loop of the model's pieces: the prefill with the streams tapped,
    then per token the LM head on the final and tapped rows (at most 64 per launch), the contrast, the repetition
    penalty, the sampler and one tapped decode step. ``keep`` collects each step's head logits before the contrast."""
    from adapcc_b200.models.gpt2 import _Taps
    from adapcc_b200.ops import (LM_HEAD_MAX_ROWS, dola_contrast_, dola_work_numel, lm_head_logits_,
                                 penalize_repeats_, sample_tokens_)
    from adapcc_b200.ops.dola import dola_candidate_layers

    dev, V, D = ids.device, m.cfg.vocab_size, m.cfg.n_embd
    B, T = ids.shape
    C = dola_candidate_layers(m.cfg.n_layer, layers)
    cache = m.new_cache(B, max(lengths) + n, kv)
    last = torch.tensor(lengths, device=dev) - 1
    rows = torch.arange(B, device=dev)
    w = m.wte.weight
    hbuf = torch.empty((1 + len(C)) * B, D, dtype=w.dtype, device=dev)
    taps = _Taps(C, hbuf[B:].view(len(C), B, D), last)
    h = m.hidden(ids, tt, cache=cache, lengths=lengths, taps=taps)[rows, last]
    tt_new = None if tt is None else tt[rows, last]
    logits = torch.empty(hbuf.shape[0], w.shape[0], dtype=torch.float32, device=dev)
    work = torch.empty(dola_work_numel(B, len(C)), dtype=torch.float32, device=dev)
    next_ids = torch.zeros(B, dtype=torch.int64, device=dev)
    tokens = torch.full((B, n), -1, dtype=torch.int64, device=dev)
    done = torch.zeros(B, dtype=torch.int32, device=dev)
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    seeds = seed + torch.arange(B, dtype=torch.int64, device=dev)
    empty = torch.zeros(0, dtype=torch.int32, device=dev)
    seq = torch.zeros(B, cache.t_max, dtype=torch.int32, device=dev)
    seq[:, :T] = ids
    prompt_len = torch.tensor(lengths, dtype=torch.int32, device=dev)
    for i in range(n):
        if i:
            h = m.decode_step(next_ids, tt_new, cache, taps=taps)
        hbuf[:B].copy_(h)
        for s in range(0, hbuf.shape[0], LM_HEAD_MAX_ROWS):
            lm_head_logits_(hbuf[s:s + LM_HEAD_MAX_ROWS], w, logits[s:s + LM_HEAD_MAX_ROWS])
        if keep is not None:
            keep.append(logits.clone())
        dola_contrast_(logits, V, B, len(C), work)
        if penalty != 1.0:
            penalize_repeats_(logits[:B], V, seq, prompt_len, cache.lens, step, next_ids, None, 1, penalty, 0)
        sample_tokens_(logits[:B], V, temperature, top_k, top_p, seeds, cache.lens, step, 0, empty, empty, done,
                       next_ids, tokens)
    return tokens


LAYERS = ["low", "high", [0, 4, 11, 4]]


@pytest.mark.parametrize("layers", LAYERS)
def test_generate_graph_equals_eager_native_loop(dev, small, layers):
    m, V = small, small.cfg.vocab_size
    ids, lengths, tt = _inputs(dev, V)
    n = 20
    for kw in (dict(temperature=0.0), dict(temperature=0.9, top_k=50, top_p=0.9, seed=31)):
        for extra in (dict(), dict(penalty=1.3), dict(penalty=1.3, kv="fp8_e4m3")):
            want = _eager(m, ids, lengths, tt, layers, n, **kw, **extra)
            got, n_new = m.generate(ids, lengths, tt, max_new_tokens=n, dola_layers=layers,
                                    repetition_penalty=extra.get("penalty", 1.0), kv_cache_dtype=extra.get("kv"),
                                    top_k=kw.get("top_k", 0), top_p=kw.get("top_p", 1.0), seed=kw.get("seed", 0),
                                    temperature=kw["temperature"])
            assert torch.equal(got, want), (layers, kw, extra)
            assert n_new.tolist() == [n] * len(lengths)
    kw = dict(max_new_tokens=n, temperature=1.0, top_p=1.0, seed=5)
    assert not torch.equal(m.generate(ids, lengths, tt, **kw)[0], m.generate(ids, lengths, tt, dola_layers=layers,
                                                                             **kw)[0])


def test_generate_tokens_are_the_fp64_decision(dev, small):
    """Greedy: each emitted token is the arg-max of the fp64 DoLa scores of the kernel's own head logits, unless the
    fp64 choice of layer sits within the JS bound or the kernel's pick is within the two entries' score bounds of the
    fp64 maximum; a few such exemptions are allowed."""
    from adapcc_b200.ops.dola import dola_candidate_layers, dola_js_reference, dola_scores_reference

    m, V = small, small.cfg.vocab_size
    ids, lengths, tt = _inputs(dev, V, seed=9)
    n, B = 16, ids.shape[0]
    exempt = 0
    for layers in LAYERS:
        C = len(dola_candidate_layers(m.cfg.n_layer, layers))
        keep = []
        tokens = _eager(m, ids, lengths, tt, layers, n, keep=keep)
        for i, lg in enumerate(keep):
            f, q = lg[:B, :V].double(), lg[B:, :V].double().view(C, B, V)
            score_b, js_b = _bounds(f, q, V)[:2]
            ref, chosen = dola_scores_reference(lg[:B], lg[B:].view(C, B, -1), V)
            js = dola_js_reference(lg[:B], lg[B:].view(C, B, -1), V).to(dev) if C > 1 else None
            for b in range(B):
                c = int(chosen[b])
                if js is not None:
                    others = [j for j in range(C) if j != c]
                    if any(js[c, b] - js[j, b] <= js_b[c, b] + js_b[j, b] for j in others):
                        exempt += 1
                        continue
                t, best = int(tokens[b, i]), int(ref[b].argmax())
                if t != best:
                    assert bool(torch.isfinite(ref[b, t])), (layers, i, b)
                    assert ref[b, best] - ref[b, t] <= score_b[c, b, best] + score_b[c, b, t], (layers, i, b)
                    exempt += 1
    assert exempt <= 4


def test_off_is_plain_generate_with_the_same_launches(dev, small):
    from adapcc_b200.runtime.native import load_library

    lib = load_library(build_if_missing=False)
    m, V = small, small.cfg.vocab_size
    ids, lengths, tt = _inputs(dev, V)
    for kw in (dict(temperature=0.0), dict(temperature=0.8, top_p=0.9, seed=3, repetition_penalty=1.2)):
        counts, outs = [], []
        for extra in ({}, dict(dola_layers=None)):
            torch.cuda.synchronize()
            c0 = lib.adapcc_launch_count()
            outs.append(m.generate(ids, lengths, tt, max_new_tokens=16, **kw, **extra))
            torch.cuda.synchronize()
            counts.append(lib.adapcc_launch_count() - c0)
        assert all(torch.equal(a, b) for a, b in zip(*outs)) and counts[0] == counts[1], (kw, counts)


def _near_tie(lg, C, V, a, b, tol=0.05):
    """Whether ids ``a`` and ``b`` are a near tie of the greedy DoLa decision on one row's head logits ``lg``
    [1 + C, ld] (the final row, then the candidates'): the top two JS within ``tol`` of the larger, either id's lf
    within ``tol`` of the kept set's threshold, or both kept with scores within ``tol``."""
    from adapcc_b200.ops.dola import LN_TENTH, dola_js_reference, dola_scores_reference

    f, q = lg[:1], lg[1:].view(C, 1, -1)
    if C > 1:
        js = dola_js_reference(f, q, V)[:, 0].sort(descending=True).values
        if float(js[0] - js[1]) <= tol * float(js[0]):
            return True
    lf = torch.log_softmax(f[0, :V].double(), -1).cpu()
    thr = float(lf.max()) + LN_TENTH
    if any(abs(float(lf[i]) - thr) <= tol for i in (a, b)):
        return True
    ref = dola_scores_reference(f, q, V)[0][0].cpu()
    return bool(torch.isfinite(ref[a]) and torch.isfinite(ref[b]) and abs(float(ref[a] - ref[b])) <= tol)


def test_row_limit_with_three_candidates(dev, small):
    m, V = small, small.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(1)
    ids = torch.randint(0, V, (65, 8), device=dev, generator=g)
    n = 4
    tokens, n_new = m.generate(ids[:64], max_new_tokens=n, dola_layers="low", temperature=0.0)
    assert tokens.shape == (64, n) and n_new.tolist() == [n] * 64
    assert torch.equal(tokens, m.generate(ids[:64], max_new_tokens=n, dola_layers="low", temperature=0.0)[0])
    # A row alone gives the same tokens up to its first near tie. The head and the DoLa kernels give a row the same
    # bits whatever the batch (test_rows_alone_graph_replay_and_repeat_runs_are_bit_identical), but the prefill's and
    # the decode step's bf16 cuBLAS GEMMs round differently at other row counts, as in plain generate
    # (tests/test_gpu_generate.py), and DoLa's scores of a random-init model hold many near ties.
    for b in range(3):
        keep = []
        alone = _eager(m, ids[b:b + 1], [8], None, "low", n, keep=keep)
        k = 0
        while k < n and int(alone[0, k]) == int(tokens[b, k]):
            k += 1
        if k < n:
            assert _near_tie(keep[k], 3, V, int(alone[0, k]), int(tokens[b, k])), (b, k)
    with pytest.raises(ValueError, match="at most 64 rows"):
        m.generate(ids, max_new_tokens=4, dola_layers="low")
