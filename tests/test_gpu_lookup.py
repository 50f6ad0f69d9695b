"""Prompt-lookup decoding on the GPU: ``verify_attention_`` bit for bit against sequential ``decode_attention_``
launches, ``lookup_draft_``, ``lookup_argmax_`` and ``lookup_accept_`` exactly against the definition (ops/lookup.py),
graph replay against eager launches, and ``GPT2DoubleHeads.generate(..., prompt_lookup_num_tokens=k)`` on GPT-2
small with random weights against plain greedy ``generate``, with a near-tie allowance calibrated in the test."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


@pytest.mark.parametrize("k", [1, 2, 4, 15])
def test_verify_attention_bit_exact_against_sequential_decode_attention(dev, k):
    from adapcc_b200.ops import decode_attention_, decode_attention_work_numel, verify_attention_

    H, Dh, t_max = 12, 64, 200
    D, S = H * Dh, k + 1
    lens = torch.tensor([0, 63, 64, 65, t_max - k - 1, 64, 10], dtype=torch.int32, device=dev)
    B = lens.numel()
    g = torch.Generator(device=dev).manual_seed(k)
    k0 = torch.randn(B, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16)
    v0 = torch.randn(B, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16)
    qkv = (torch.randn(B * S, 3 * D, device=dev, generator=g) * 2).to(torch.bfloat16)
    work = torch.empty(decode_attention_work_numel(B * S, H, Dh, t_max), dtype=torch.float32, device=dev)
    for nq_rows in ([S] * B, [S, 1, max(1, k), S, S, 0, (k + 2) // 2]):
        nq = torch.tensor(nq_rows, dtype=torch.int32, device=dev)
        kc, vc = k0.clone(), v0.clone()
        out = torch.full((B * S, D), 7.0, dtype=torch.bfloat16, device=dev)
        verify_attention_(qkv, kc, vc, lens, nq, k, out, work)
        # slot j of every row through decode_attention_ at lens + j on a cache that holds slots 0..j-1; pad slots get
        # a length outside the cache, which decode_attention_ leaves alone with a zero output
        kr, vr = k0.clone(), v0.clone()
        want = torch.empty(B, S, D, dtype=torch.bfloat16, device=dev)
        w2 = torch.empty(decode_attention_work_numel(B, H, Dh, t_max), dtype=torch.float32, device=dev)
        for j in range(S):
            lj = torch.where(j < nq, lens + j, torch.full_like(lens, -1)).contiguous()
            o = torch.empty(B, D, dtype=torch.bfloat16, device=dev)
            decode_attention_(qkv.view(B, S, 3 * D)[:, j], kr, vr, lj, o, w2)
            want[:, j] = o
        torch.cuda.synchronize()
        assert torch.equal(_bits(out), _bits(want.view(B * S, D))), (k, nq_rows)
        assert torch.equal(_bits(kc), _bits(kr)) and torch.equal(_bits(vc), _bits(vr)), (k, nq_rows)
        # exactly the real slots' positions changed
        changed = (kc != k0).any(-1).any(1) | (vc != v0).any(-1).any(1)                     # [B, t_max]
        for b in range(B):
            real = set(range(int(lens[b]), int(lens[b]) + nq_rows[b]))
            assert set(torch.nonzero(changed[b]).flatten().tolist()) <= real, (b, nq_rows)
        # a graph replay equals the eager launch
        kg, vg = k0.clone(), v0.clone()
        again = torch.zeros_like(out)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            verify_attention_(qkv, kg, vg, lens, nq, k, again, work)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(again), _bits(out)) and torch.equal(_bits(kg), _bits(kc))


def _state(dev, B, k, n, t_max, ngram, seed):
    """A LookupState mid-generation: ragged rows with planted repeats, some near max_new, one done."""
    from adapcc_b200.ops import LookupState

    rng = np.random.default_rng(seed)
    st = LookupState(B, k, n, t_max, ngram, dev)
    seq = rng.integers(0, 6, (B, t_max)).astype(np.int32)
    lens = rng.integers(0, t_max - n, B).astype(np.int32)
    emitted = rng.integers(0, n, B).astype(np.int32)
    emitted[0], emitted[1] = n - 1, n - 2                                # no room for drafts / room for one
    for b in range(B):                                                   # plant the tail earlier in the row
        L, m = int(lens[b]), int(rng.integers(1, 4))
        if L >= 2 * m + 2:
            i = int(rng.integers(0, L - 2 * m))
            seq[b, i:i + m] = seq[b, L + 1 - m:L + 1]
    done = np.zeros(B, dtype=np.int32)
    done[2] = 1
    st.seq.copy_(torch.from_numpy(seq))
    st.emitted.copy_(torch.from_numpy(emitted))
    st.done.copy_(torch.from_numpy(done))
    return st, torch.from_numpy(lens).to(dev)


def test_lookup_draft_exact_against_the_definition(dev):
    from adapcc_b200.ops import lookup_draft_
    from adapcc_b200.ops.lookup import lookup_draft

    for seed, (B, k, ngram) in enumerate(((8, 4, 2), (5, 15, 4), (16, 1, 1), (6, 7, 3))):
        st, lens = _state(dev, B, k, 24, 120, ngram, seed)
        ids, pos, nq = lookup_draft(st.seq.cpu(), lens.cpu(), st.emitted.cpu(), st.done.cpu(), k, 24, ngram)
        lookup_draft_(st, lens)
        torch.cuda.synchronize()
        assert torch.equal(st.ids.cpu(), ids) and torch.equal(st.pos.cpu(), pos) and torch.equal(st.nq.cpu(), nq)
        assert int((nq > 1).sum()) >= 2, nq                              # drafts were found


@pytest.mark.parametrize("first", [False, True])
def test_lookup_argmax_and_accept_exact_against_the_definition(dev, first):
    from adapcc_b200.ops import lookup_accept_, lookup_argmax_, lookup_draft_
    from adapcc_b200.ops.lookup import greedy_token, lookup_accept

    B, k, n, t_max, V, ld = 8, 4, 24, 120, 1000, 1024
    S = k + 1
    st, lens = _state(dev, B, k, n, t_max, 2, 3)
    lookup_draft_(st, lens)
    rng = np.random.default_rng(1)
    ls = 1 if first else S
    logits = rng.standard_normal((B * ls, ld)).astype(np.float32)
    logits[:, V:] = 100.0                                                # beyond vocab: never read
    em = st.emitted.cpu().numpy()
    ids = st.ids.cpu().view(B, S).numpy().copy()
    stop, suppress, min_new = [], [17, 18], 12
    for b in range(B):
        for j in range(ls):
            row = logits[b * ls + j]
            t = int(rng.integers(0, V))
            row[t] = 9.0
            if (b + j) % 3 == 0:
                row[t + 1 if t + 1 < V else t - 1] = 9.0                 # a tie among the leading logits
            if b == 4 and j == 1:
                row[17] = 11.0                                           # a suppressed id on top
            g = greedy_token(row[:V], int(em[b]) + j, min_new, suppress)
            if j + 1 < S and (b % 4 != 3 or j < 1):                      # the next draft equals it, mostly
                ids[b, j + 1] = g
            if b == 5 and j == 1:
                stop.append(g)                                           # a stop id among the accepted drafts
    if not first:
        st.ids.copy_(torch.from_numpy(ids).view(-1))
    else:
        st.nq.fill_(1)
    want = {name: getattr(st, name).cpu().clone() for name in ("seq", "emitted", "done", "tokens", "steps")}
    wl = lens.cpu().clone()
    lookup_accept(torch.from_numpy(logits), V, st.ids.cpu(), st.nq.cpu(), want["seq"], wl, want["emitted"],
                  want["done"], want["tokens"], None if first else want["steps"], min_new, suppress, stop)
    dl = lens.clone()
    lookup_argmax_(torch.from_numpy(logits).to(dev), V, st, min_new,
                   torch.tensor(suppress, dtype=torch.int32, device=dev))
    lookup_accept_(st, dl, torch.tensor(stop, dtype=torch.int32, device=dev), count=not first)
    torch.cuda.synchronize()
    for name, t in want.items():
        assert torch.equal(getattr(st, name).cpu(), t), name
    assert torch.equal(dl.cpu(), wl)
    grown = (want["emitted"] - torch.from_numpy(em)).tolist()
    print(f"tokens emitted per row: {grown}")
    if not first:
        assert max(grown) >= 3 and int(want["done"].sum()) >= 2


# ---- GPT-2 small, random weights -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpt2(dev):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def _prompts(V, dev, B=8, T=96, seed=0):
    """Ragged prompts that repeat phrases of themselves, as dialogue histories do."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (B, T), generator=g)
    for b in range(B):
        phrase = ids[b, :12].clone()
        for start in range(24, T - 12, 30):
            ids[b, start:start + 12] = phrase
    lengths = [T, 40, 77, T, 13, 60, T - 1, 31][:B]
    return ids.to(dev), lengths


@torch.no_grad()
def _calibrate(model, ids, lengths, tokens, k):
    """Plain greedy's per-position logits [B, n, V] (eager decode steps over ``tokens``) and delta: the largest logit
    difference between them and verify steps at B·(k+1) rows fed ``tokens`` as drafts, all of which are accepted."""
    from adapcc_b200.models.gpt2 import VerifyKV
    from adapcc_b200.ops import decode_attention_work_numel, lm_head_logits_

    dev, W, V = ids.device, model.wte.weight, model.cfg.vocab_size
    B, n = tokens.shape
    S, t_max = k + 1, max(lengths) + n
    last = torch.tensor(lengths, device=dev) - 1
    toks = torch.cat([ids[torch.arange(B, device=dev), last][:, None], tokens.clamp(min=0)], 1)
    logits = torch.empty(B * S, W.shape[0], dtype=torch.float32, device=dev)
    cache = model.new_cache(B, t_max)
    h = model.hidden(ids, None, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last]
    plain = torch.empty(B, n, V, dtype=torch.float32, device=dev)
    lm_head_logits_(h, W, logits[:B])
    plain[:, 0] = logits[:B, :V]
    for i in range(1, n):
        lm_head_logits_(model.decode_step(toks[:, i], None, cache), W, logits[:B])
        plain[:, i] = logits[:B, :V]
    cache = model.new_cache(B, t_max)
    model.hidden(ids, None, cache=cache, lengths=lengths)
    work = torch.empty(decode_attention_work_numel(B * S, model.cfg.n_head, 64, t_max), dtype=torch.float32,
                       device=dev)
    delta, e = 0.0, 1
    while e < n:
        nq = min(S, n - e)
        slot = torch.zeros(B, S, dtype=torch.int64, device=dev)
        slot[:, :nq] = toks[:, e:e + nq]
        pos = (cache.lens.long()[:, None] + torch.arange(S, device=dev)).clamp(max=t_max - 1)
        nqt = torch.full((B,), nq, dtype=torch.int32, device=dev)
        hv = model._verify_hidden(slot.view(-1), pos.view(-1), None, VerifyKV(cache, S, nqt, work))
        lm_head_logits_(hv, W, logits)
        got = logits.view(B, S, -1)[:, :nq, :V]
        delta = max(delta, float((got - plain[:, e:e + nq]).abs().max()))
        cache.lens.add_(nq)
        e += nq
    return plain, delta


def _check_rule(got, want, plain, delta, what):
    differ = 0
    for b in range(got.shape[0]):
        if torch.equal(got[b], want[b]):
            continue
        differ += 1
        i = int(torch.nonzero(got[b] != want[b])[0])
        top2 = torch.topk(plain[b, i], 2).values
        assert float(top2[0] - top2[1]) <= 2 * delta, (what, b, i, float(top2[0] - top2[1]), delta)
    return differ


@pytest.mark.parametrize("k", [2, 4, 7])
def test_gpt2_small_lookup_generate_against_greedy(gpt2, dev, k):
    V, n = gpt2.cfg.vocab_size, 48
    ids, lengths = _prompts(V, dev)
    want, n_want = gpt2.generate(ids, lengths, max_new_tokens=n, temperature=0.0)
    got, n_got = gpt2.generate(ids, lengths, max_new_tokens=n, temperature=0.0, prompt_lookup_num_tokens=k)
    st = gpt2.lookup_stats
    per_step = float((st["emitted"] - 1).sum()) / float(st["steps"].sum())
    again, _ = gpt2.generate(ids, lengths, max_new_tokens=n, temperature=0.0, prompt_lookup_num_tokens=k)
    assert torch.equal(again, got)
    plain, delta = _calibrate(gpt2, ids, lengths, want, k)
    differ = _check_rule(got, want, plain, delta, "batch")
    print(f"k = {k}: delta {delta:.3g}, {differ} of 8 rows differ, {per_step:.2f} tokens per verify step, "
          f"{st['replays']} replays for {int(st['steps'].max())} steps of the longest row")
    assert per_step > 1.0 and torch.equal(n_got, n_want)
    # rows alone follow the same rule against plain greedy of the row alone
    for b in (1, 4, 6):
        row = ids[b:b + 1, :lengths[b]]
        w1, _ = gpt2.generate(row, max_new_tokens=n, temperature=0.0)
        g1, _ = gpt2.generate(row, max_new_tokens=n, temperature=0.0, prompt_lookup_num_tokens=k)
        p1, d1 = _calibrate(gpt2, row, [lengths[b]], w1, k)
        _check_rule(g1, w1, p1, d1, f"row {b} alone")


def test_too_many_verify_rows_raise_before_launching(gpt2, dev):
    ids = torch.zeros(9, 8, dtype=torch.long, device=dev)
    with pytest.raises(ValueError, match="verify rows"):
        gpt2.generate(ids, temperature=0.0, prompt_lookup_num_tokens=7)
