"""Classifier-free guidance on the GPU: the mix kernel against the fp64 definition (ops/guidance.py) with an error bound
derived from its fp32 reduction order, its batch invariance and graph capture, and ``GPT2DoubleHeads.generate`` with
guidance on GPT-2 small (random init, bf16) against an eager loop of the same native ops and against the fp64
decision."""
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


def _mix(logits, vocab, B, scale):
    from adapcc_b200.ops import guidance_mix_

    out = logits.clone()
    guidance_mix_(out, vocab, B, scale)
    return out


def _bound(cond, uncond, vocab, scale):
    """The kernel's error against the fp64 definition, from its order of operations (csrc/ops_guidance.cu), per element.

    Per row: the maximum m is exact. d_i = fl(x_i - m) is within |d_i| u; expf is within 2 ulp (4 u relative), so
    e_i = expf(d_i) is within (4 + |d_i|) u e_i. S adds positive terms with at most C + 10 roundings on any path
    (C = ceil(vocab / 1024) in a thread, 5 shuffle levels over lanes, 5 over warps): |dS| <= (C + 10) u S +
    sum (4 + |d_i|) u e_i. logf is within 1 ulp (2 u |log S|), so |d log S| <= |dS| / S + 2 u |log S|. Then
    l_i = fl(d_i - log S) is within |d_i| u + |d log S| + |l_i| u, and the three roundings of
    fl(fl(g fl(lc - lu)) + lu) add |lc - lu| u (times |g|), |g (lc - lu)| u and |s| u. A factor 1.01 covers the
    second-order terms."""
    C = math.ceil(vocab / 1024)
    errs, logs = [], []
    for x in (cond, uncond):
        x = x[:, :vocab].double()
        d = x - x.max(1, keepdim=True).values
        e = d.exp()
        S = e.sum(1, keepdim=True)
        dS = (C + 10) * U32 * S + ((4 + d.abs()) * U32 * e).sum(1, keepdim=True)
        dlog = dS / S + 2 * U32 * S.log().abs()
        lsm = d - S.log()
        errs.append(d.abs() * U32 + dlog + lsm.abs() * U32)
        logs.append(lsm)
    (ec, eu), (lc, lu) = errs, logs
    g = float(np.float32(scale))
    s = g * (lc - lu) + lu
    e_diff = ec + eu + (lc - lu).abs() * U32
    return 1.01 * (abs(g) * e_diff + (g * (lc - lu)).abs() * U32 + eu + s.abs() * U32) + 1e-30


def _wide(dev, B, ld, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(2 * B, ld, device=dev, generator=g) * 8
    x[::3] *= 4                                                # a wide spread: e^-200 next to 1
    x[1::4, :7] += 60.0                                        # spikes that hold nearly all the mass
    return x


@pytest.mark.parametrize("vocab,ld", [(50257, 50304), (1003, 1010)])
def test_kernel_against_fp64_definition(dev, vocab, ld):
    from adapcc_b200.ops.guidance import guided_scores_reference

    for B in (1, 7, 32):
        x = _wide(dev, B, ld, seed=B + vocab)
        x[:, vocab:] = float("nan")                                # padding columns: never read, never written
        for scale in (1.5, 3.0, 0.0, -1.0, 0.37):
            out = _mix(x, vocab, B, scale)
            torch.cuda.synchronize()
            assert torch.equal(out[B:].view(torch.int32), x[B:].view(torch.int32)), (B, scale)
            assert torch.equal(out[:B, vocab:].view(torch.int32), x[:B, vocab:].view(torch.int32)), (B, scale)
            ref = guided_scores_reference(x[:B], x[B:], vocab, scale).cpu()
            bound = _bound(x[:B].cpu(), x[B:].cpu(), vocab, scale)
            err = (out[:B, :vocab].cpu().double() - ref).abs()
            assert bool((err <= bound).all()), (B, scale, float((err - bound).max()))


def test_kernel_rows_do_not_depend_on_the_batch_and_graph_equals_eager(dev):
    V, ld, B = 50257, 50264, 32
    x = _wide(dev, B, ld, seed=5)
    out = _mix(x, V, B, 2.5)
    for b in range(B):
        alone = _mix(torch.stack([x[b], x[B + b]]), V, 1, 2.5)
        assert torch.equal(alone[0].view(torch.int32), out[b].view(torch.int32)), b
    sub = _mix(torch.cat([x[:7], x[B:B + 7]]), V, 7, 2.5)
    assert torch.equal(sub[:7].view(torch.int32), out[:7].view(torch.int32))
    from adapcc_b200.ops import guidance_mix_

    buf = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        guidance_mix_(buf, V, B, 2.5)                              # warm-up
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        guidance_mix_(buf, V, B, 2.5)
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
    neg_lengths = [30, 1, 45, 12, 8, 50][:B]
    neg = torch.randint(0, V - 5, (B, 50), device=dev, generator=g)
    neg_tt = torch.randint(V - 5, V - 3, (B, 50), device=dev, generator=g)
    return ids, lengths, tt, neg, neg_lengths, neg_tt


@torch.no_grad()
def _eager(m, ids, lengths, tt, neg, neg_lengths, neg_tt, n, scale, temperature=0.0, top_k=0, top_p=1.0, seed=0,
           min_new=0, suppress=(), stop=(), penalty=1.0, keep=None):
    """``generate`` with guidance as an eager loop of the native ops: the stacked prefill, then per token LM head,
    guidance mix, repetition penalty, sampler and one decode step of all 2B rows. ``keep`` collects each step's
    LM-head logits of the 2B rows (before the mix)."""
    from adapcc_b200.ops import guidance_mix_, lm_head_logits_, penalize_repeats_, sample_tokens_

    dev, V = ids.device, m.cfg.vocab_size
    B, T = ids.shape
    Tn = neg.shape[1]
    x = torch.zeros(2 * B, max(T, Tn), dtype=ids.dtype, device=dev)
    y = torch.zeros_like(x)
    x[:B, :T], x[B:, :Tn], y[:B, :T], y[B:, :Tn] = ids, neg, tt, neg_tt
    lens = list(lengths) + list(neg_lengths)
    cache = m.new_cache(2 * B, max(lens) + n)
    h = m.hidden(x, y, cache=cache, lengths=lens)[torch.arange(2 * B, device=dev), torch.tensor(lens, device=dev) - 1]
    tt_new = tt[torch.arange(B, device=dev), torch.tensor(lengths, device=dev) - 1].repeat(2)
    w = m.wte.weight
    logits = torch.empty(2 * B, w.shape[0], dtype=torch.float32, device=dev)
    next_ids = torch.zeros(2 * B, dtype=torch.int64, device=dev)
    tokens = torch.full((B, n), -1, dtype=torch.int64, device=dev)
    done = torch.zeros(B, dtype=torch.int32, device=dev)
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    seeds = seed + torch.arange(B, dtype=torch.int64, device=dev)
    sup, stp = (torch.tensor(list(v), dtype=torch.int32, device=dev) for v in (suppress, stop))
    seq = torch.zeros(B, cache.t_max, dtype=torch.int32, device=dev)
    seq[:, :T] = ids
    prompt_len = torch.tensor(lengths, dtype=torch.int32, device=dev)
    for i in range(n):
        if i:
            h = m.decode_step(next_ids, tt_new, cache)
        lm_head_logits_(h, w, logits)
        if keep is not None:
            keep.append(logits.clone())
        guidance_mix_(logits, V, B, scale)
        if penalty != 1.0:
            penalize_repeats_(logits[:B], V, seq, prompt_len, cache.lens[:B], step, next_ids[:B], None, 1, penalty, 0)
        sample_tokens_(logits[:B], V, temperature, top_k, top_p, seeds, cache.lens[:B], step, min_new, sup, stp, done,
                       next_ids[:B], tokens)
        next_ids[B:].copy_(next_ids[:B])
    return tokens


def test_generate_graph_equals_eager_native_loop(dev, small):
    m, V = small, small.cfg.vocab_size
    ids, lengths, tt, neg, neg_lengths, neg_tt = _inputs(dev, V)
    n = 24
    for kw in (dict(temperature=0.0), dict(temperature=0.9, top_k=50, top_p=0.9, seed=31)):
        for extra in (dict(), dict(penalty=1.3, min_new=6, suppress=(V - 1, V - 2), stop=(V - 1, 13))):
            want = _eager(m, ids, lengths, tt, neg, neg_lengths, neg_tt, n, 1.5, **kw, **extra)
            got, n_new = m.generate(ids, lengths, tt, max_new_tokens=n, guidance_scale=1.5, negative_prompt_ids=neg,
                                    negative_lengths=neg_lengths, negative_token_type_ids=neg_tt,
                                    repetition_penalty=extra.get("penalty", 1.0), min_new_tokens=extra.get("min_new", 0),
                                    suppress_ids=extra.get("suppress", ()), stop_ids=extra.get("stop", ()),
                                    top_k=kw.get("top_k", 0), top_p=kw.get("top_p", 1.0), seed=kw.get("seed", 0),
                                    temperature=kw["temperature"])
            assert torch.equal(got, want), (kw, extra)
            assert n_new.tolist() == (want >= 0).sum(1).tolist()


def test_generate_tokens_are_the_fp64_decision(dev, small):
    """Greedy: each emitted token is the arg-max of the fp64 guided scores of the kernel's own LM-head logits, unless
    the kernel's pick is within the two entries' derived mix bounds of the fp64 maximum."""
    from adapcc_b200.ops.guidance import guided_scores_reference

    m, V = small, small.cfg.vocab_size
    ids, lengths, tt, neg, neg_lengths, neg_tt = _inputs(dev, V, seed=9)
    n, B = 20, ids.shape[0]
    exempt = 0
    for scale in (1.5, 3.0, -0.5):
        keep = []
        tokens = _eager(m, ids, lengths, tt, neg, neg_lengths, neg_tt, n, scale, keep=keep)
        for i, lg in enumerate(keep):
            lg = lg.cpu()
            ref = guided_scores_reference(lg[:B], lg[B:], V, scale)
            bound = _bound(lg[:B], lg[B:], V, scale)
            for b in range(B):
                t, best = int(tokens[b, i]), int(ref[b].argmax())
                if t != best:
                    assert ref[b, best] - ref[b, t] <= bound[b, best] + bound[b, t], (scale, i, b)
                    exempt += 1
    assert exempt <= 3


def test_scale_one_is_plain_generate_with_no_extra_launch(dev, small):
    from adapcc_b200.runtime.native import load_library

    lib = load_library(build_if_missing=False)
    m, V = small, small.cfg.vocab_size
    ids, lengths, tt, neg, neg_lengths, neg_tt = _inputs(dev, V)
    for kw in (dict(temperature=0.0), dict(temperature=0.8, top_p=0.9, seed=3, repetition_penalty=1.2)):
        counts, outs = [], []
        for extra in ({}, dict(guidance_scale=1.0, negative_prompt_ids=neg, negative_lengths=neg_lengths,
                               negative_token_type_ids=neg_tt)):
            torch.cuda.synchronize()
            c0 = lib.adapcc_launch_count()
            outs.append(m.generate(ids, lengths, tt, max_new_tokens=16, **kw, **extra))
            torch.cuda.synchronize()
            counts.append(lib.adapcc_launch_count() - c0)
        assert all(torch.equal(a, b) for a, b in zip(*outs)) and counts[0] == counts[1], (kw, counts)


def test_row_and_cache_limits(dev, small):
    m, V = small, small.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(1)
    ids = torch.randint(0, V, (33, 8), device=dev, generator=g)
    tokens, n_new = m.generate(ids[:32], max_new_tokens=4, guidance_scale=2.0)
    assert tokens.shape == (32, 4) and n_new.tolist() == [4] * 32
    with pytest.raises(ValueError, match="at most 64 rows with guidance"):
        m.generate(ids, max_new_tokens=4, guidance_scale=2.0)
    # a row that ends at n_positions: every token is generated, as in plain generate; one position more is an error
    n = 6
    prompt = torch.randint(0, V, (2, m.cfg.n_positions - n), device=dev, generator=g)
    plain, plain_n = m.generate(prompt, max_new_tokens=n, temperature=0.0)
    got, got_n = m.generate(prompt, max_new_tokens=n, temperature=0.0, guidance_scale=1.5, negative_prompt_ids=prompt,
                            negative_lengths=[m.cfg.n_positions - n, 3])
    assert plain_n.tolist() == got_n.tolist() == [n, n]
    with pytest.raises(ValueError, match="n_positions"):
        m.generate(prompt[:, :5], max_new_tokens=n, guidance_scale=1.5,
                   negative_prompt_ids=torch.zeros(2, m.cfg.n_positions - n + 1, dtype=torch.long, device=dev))
