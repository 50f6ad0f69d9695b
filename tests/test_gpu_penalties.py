"""Frequency / presence penalties and context n-gram blocking on the GPU: rules 2 and 4 of ``penalize_repeats_``
against the definition (ops/repeats.py) bit for bit, alone and with the other rules, at step 0 and after, with and
without parent maps; the same bits with the new rules off; a row alone against the same row in a batch and graph
replay against eager launches; and ``generate``, ``beam_search``, ``stochastic_beam_search`` and
``contrastive_search`` on GPT-2 small against eager loops with the reference."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # unit roundoff of fp32
V, LD, T_MAX = 50257, 50304, 1024
ALONE = [dict(frequency=0.7), dict(presence=1.25), dict(frequency=-0.3, presence=-2.0), dict(frequency=1e-3),
         dict(context_ngram=1), dict(context_ngram=3)]
ALL = dict(frequency=0.5, presence=0.375, context_ngram=2)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _logits(rng, R):
    """fp32 [R, LD] with +-0, subnormals and -inf planted among the low ids the sequences use."""
    x = (rng.standard_normal((R, LD)) * 4).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-40, -1e-40, -np.inf, -np.inf, 3e-39, -0.0], dtype=np.float32)
    for r in range(R):
        x[r, rng.choice(64, size=special.size, replace=False)] = special
    return x


def _sequences(rng, R, lens):
    """Sequences over 4, 64 or all ids by row (the first two heavily duplicated), padded with -7 past lens."""
    seq = np.full((R, T_MAX), -7, dtype=np.int32)
    for r in range(R):
        L = int(lens[r])
        seq[r, :L] = rng.integers(0, [4, 64, V][r % 3], L)
    return seq


def _run(dev, logits, seq, prompt_len, lens, step, ids, parent, group, p, n, table=None, **kw):
    from adapcc_b200.ops import penalize_repeats_

    i32 = dict(dtype=torch.int32, device=dev)
    t = dict(logits=torch.from_numpy(logits).to(dev), seq=torch.from_numpy(seq).to(dev),
             prompt_len=torch.as_tensor(prompt_len, **i32), lens=torch.as_tensor(lens, **i32),
             step=torch.tensor([step], **i32), ids=torch.as_tensor(ids, dtype=torch.int64, device=dev),
             parent=None if parent is None else torch.as_tensor(parent, **i32))
    penalize_repeats_(t["logits"], V, t["seq"], t["prompt_len"], t["lens"], t["step"], t["ids"], t["parent"], group,
                      p, n, table, **kw)
    torch.cuda.synchronize()
    return t


def _want(logits, seq, prompt_len, lens, p, n, table=None, **kw):
    from adapcc_b200.ops.repeats import penalize_repeats_reference

    return penalize_repeats_reference(torch.from_numpy(logits), [seq[r, :int(x)] for r, x in enumerate(lens)], V, p,
                                      n, table, prompt_lens=[int(x) for x in prompt_len], **kw)


def _table(rng, seq, lens):
    from adapcc_b200.ops.repeats import check_sequence_bias_args

    sb, bad = {}, []
    for r in range(min(seq.shape[0], 40)):
        L = int(lens[r])
        m = int(rng.integers(1, 4))
        if L >= m:
            sb[tuple(seq[r, L - m + 1:L].tolist()) + (int(rng.integers(0, 64)),)] = float(rng.standard_normal() * 3)
        bad.append([int(rng.integers(0, 64))])
    return check_sequence_bias_args("test", sb, bad, V)


def test_kernel_matches_reference_bit_for_bit(dev):
    rng = np.random.default_rng(0)
    rows = 0
    changed = {}
    for R, step in ((1, 0), (1, 3), (8, 0), (8, 5), (33, 2), (64, 0), (64, 9)):
        lens = rng.integers(1, T_MAX + 1, R)
        lens[0] = T_MAX
        prompt_len = rng.integers(0, lens + 1)
        prompt_len[0] = 1                                        # 1023 generated ids
        if R > 1:
            lens[-1], prompt_len[-1] = 1, 1
            prompt_len[1] = lens[1]                              # an empty generated region
        logits, seq = _logits(rng, R), _sequences(rng, R, lens)
        ids = rng.integers(0, 4, R)                               # in every row's alphabet
        want_seq = seq.copy()
        if step:
            want_seq[np.arange(R), lens - 1] = ids
        cases = ALONE + [ALL]
        for kw in cases:
            got = _run(dev, logits, seq, prompt_len, lens, step, ids, None, 1, 1.0, 0, **kw)
            want = _want(logits, want_seq, prompt_len, lens, 1.0, 0, **kw)
            assert torch.equal(got["seq"].cpu(), torch.from_numpy(want_seq))
            assert torch.equal(_bits(got["logits"]), _bits(want)), (R, step, kw)
            key = tuple(sorted(kw.items()))
            changed[key] = changed.get(key, 0) + int((_bits(want) != _bits(torch.from_numpy(logits))).sum())
        # everything on together, with a sequence-bias table, the penalty and the n-gram ban
        table = _table(rng, want_seq, lens)
        got = _run(dev, logits, seq, prompt_len, lens, step, ids, None, 1, 1.3, 3, table, **ALL)
        assert torch.equal(_bits(got["logits"]), _bits(_want(logits, want_seq, prompt_len, lens, 1.3, 3, table,
                                                              **ALL))), (R, step)
        rows += R * (len(cases) + 1)
    assert all(c > 0 for c in changed.values()), changed          # every rule changed something
    print(f"penalize_repeats_ with frequency / presence / context n-grams vs reference: {rows} rows, every bit equal")


def test_new_rules_off_give_the_same_bits(dev):
    rng = np.random.default_rng(3)
    R = 24
    lens = rng.integers(2, T_MAX + 1, R)
    prompt_len = lens // 2
    logits, seq = _logits(rng, R), _sequences(rng, R, lens)
    ids = rng.integers(0, 64, R)
    table = _table(rng, seq, lens)
    for p, n, tab in ((1.0, 0, None), (1.2, 2, None), (0.8, 0, table), (1.0, 3, table)):
        base = _run(dev, logits, seq, prompt_len, lens, 4, ids, None, 1, p, n, tab)
        off = _run(dev, logits, seq, prompt_len, lens, 4, ids, None, 1, p, n, tab, frequency=0.0, presence=-0.0,
                   context_ngram=0)
        assert torch.equal(_bits(off["logits"]), _bits(base["logits"])) and torch.equal(off["seq"], base["seq"])


def test_parent_maps(dev):
    rng = np.random.default_rng(1)
    for K in (1, 8, 16):
        G = max(1, 64 // K)
        R = G * K
        prompt_len = np.repeat([T_MAX - 200 - 7 * (g % 5) for g in range(G)], K)
        lens = prompt_len + np.repeat([200 - g % 3 for g in range(G)], K)
        cycle = [g * K + (k + 1) % K for g in range(G) for k in range(K)]
        many = [g * K + (K - 1 if k % 2 else 0) for g in range(G) for k in range(K)]
        for parent in (cycle, many):
            logits, seq = _logits(rng, R), _sequences(rng, R, lens)
            for g in range(G):
                seq[g * K:(g + 1) * K, :prompt_len[g * K]] = seq[g * K, :prompt_len[g * K]]
            ids = rng.integers(0, 64, R)
            want_seq = seq.copy()
            for r, pr in enumerate(parent):
                lo, hi = int(prompt_len[r]), int(lens[r]) - 1
                want_seq[r, lo:hi] = seq[pr, lo:hi]
                want_seq[r, hi] = ids[r]
            for kw in (dict(frequency=0.7), dict(presence=-1.5), dict(context_ngram=2), ALL):
                got = _run(dev, logits, seq, prompt_len, lens, 7, ids, parent, K, 1.0, 0, **kw)
                assert torch.equal(got["seq"].cpu(), torch.from_numpy(want_seq)), K
                want = _want(logits, want_seq, prompt_len, lens, 1.0, 0, **kw)
                assert torch.equal(_bits(got["logits"]), _bits(want)), (K, kw)
            table = _table(rng, want_seq, lens)
            got = _run(dev, logits, seq, prompt_len, lens, 7, ids, parent, K, 1.3, 3, table, **ALL)
            assert torch.equal(_bits(got["logits"]), _bits(_want(logits, want_seq, prompt_len, lens, 1.3, 3, table,
                                                                  **ALL))), K


def test_row_alone_equals_row_in_batch_and_graph_equals_eager(dev):
    from adapcc_b200.ops import penalize_repeats_

    rng = np.random.default_rng(2)
    R, K = 16, 8
    lens = rng.integers(100, T_MAX + 1, R)
    prompt_len = lens - 90
    logits, seq = _logits(rng, R), _sequences(rng, R, lens)
    ids = rng.integers(0, 64, R)
    full = _run(dev, logits, seq, prompt_len, lens, 3, ids, None, 1, 0.7, 2, **ALL)
    for r in range(R):
        one = _run(dev, logits[r:r + 1].copy(), seq[r:r + 1].copy(), prompt_len[r:r + 1], lens[r:r + 1], 3,
                   ids[r:r + 1], None, 1, 0.7, 2, **ALL)
        assert torch.equal(_bits(one["logits"][0]), _bits(full["logits"][r])), r
    prompt_len = np.repeat(prompt_len[::K], K)
    lens = np.repeat(lens[::K], K)
    parent = [g * K + (k + 3) % K for g in range(R // K) for k in range(K)]
    eager = _run(dev, logits, seq, prompt_len, lens, 3, ids, parent, K, 1.0, 0, **ALL)
    t = _run(dev, logits, seq, prompt_len, lens, 0, ids, parent, K, 1.0, 0, **ALL)
    t["step"].fill_(3)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        penalize_repeats_(t["logits"], V, t["seq"], t["prompt_len"], t["lens"], t["step"], t["ids"], t["parent"], K,
                          1.0, 0, **ALL)
    t["logits"].copy_(torch.from_numpy(logits))
    t["seq"].copy_(torch.from_numpy(seq))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(t["logits"]), _bits(eager["logits"])) and torch.equal(t["seq"], eager["seq"])


# ---- GPT-2 small ---------------------------------------------------------------------------------------------------
CONTROLS = dict(frequency_penalty=0.5, presence_penalty=0.5, context_no_repeat_ngram_size=3)
REF = dict(frequency=0.5, presence=0.5, context_ngram=3)


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def _prompts(dev, B, T, seed):
    """Right-padded prompts over 300 ids, each with a repeated stretch, so the context block has n-grams to refuse."""
    g = torch.Generator(device=dev).manual_seed(seed)
    ids = torch.randint(0, 300, (B, T), device=dev, generator=g)
    ids[:, 3:9] = ids[:, 0:1]
    return ids


def copied_ngrams(full, P, m):
    grams = {tuple(full[j:j + m]) for j in range(P - m + 1)}
    return [t for t in range(max(P, m), len(full)) if tuple(full[t - m + 1:t + 1]) in grams]


def _check_op(logits, before, vocab, seq, lens, prompt_len, rows):
    """The op's output equals the reference on the sequences the op keeps, bit for bit."""
    from adapcc_b200.ops.repeats import penalize_repeats_reference

    L, P = lens.cpu().tolist(), prompt_len.cpu().tolist()
    want = penalize_repeats_reference(before, [seq[r, :L[r]].cpu() for r in range(rows)], vocab, 1.0, 0,
                                      prompt_lens=P, **REF)
    assert torch.equal(_bits(logits), _bits(want))


@pytest.mark.parametrize("mode", ["greedy", "sampled", "guided"])
def test_generate_graph_equals_eager_loop(dev, mode):
    """``generate`` (graph replay) against an eager loop of the same kernels: the same tokens, and at every step of
    the loop the op's output equals the reference bit for bit."""
    from adapcc_b200.ops import guidance_mix_, lm_head_logits_, penalize_repeats_, sample_tokens_

    m = _gpt2_small(dev, seed=2)
    Vv = m.cfg.vocab_size                      # GPT-2's 50257 ids and the dialogue special tokens
    B, n = 6, 24
    lengths = [90, 17, 64, 9, 120, 33]
    ids = _prompts(dev, B, 120, 5)
    temp, scale = (0.0, 1.0) if mode == "greedy" else (1.0, 1.5 if mode == "guided" else 1.0)
    kw = dict(max_new_tokens=n, temperature=temp, top_p=0.95, seed=11, guidance_scale=scale)
    free, _ = m.generate(ids, lengths, **kw)
    tokens, n_new = m.generate(ids, lengths, **kw, **CONTROLS)
    assert not torch.equal(tokens, free)
    w = m.wte.weight
    with torch.no_grad():
        if mode == "guided":
            ids_all, _, lengths_all, _ = m._guidance_rows(ids, None, lengths, torch.tensor(lengths, device=dev) - 1,
                                                          None, None, [1] * B, None)
        else:
            ids_all, lengths_all = ids, lengths
        R = len(lengths_all)
        cache = m.new_cache(R, max(lengths_all) + n)
        last = torch.tensor(lengths_all, device=dev) - 1
        h = m.hidden(ids_all, None, cache=cache, lengths=lengths_all)[torch.arange(R, device=dev), last]
        logits = torch.empty(R, w.shape[0], dtype=torch.float32, device=dev)
        next_ids = torch.zeros(R, dtype=torch.int64, device=dev)
        done = torch.zeros(B, dtype=torch.int32, device=dev)
        step = torch.zeros(1, dtype=torch.int32, device=dev)
        seeds = 11 + torch.arange(B, dtype=torch.int64, device=dev)
        seq = torch.zeros(B, cache.t_max, dtype=torch.int32, device=dev)
        seq[:, :ids.shape[1]] = ids
        prompt_len = cache.lens[:B].clone()
        want = torch.full((B, n), -1, dtype=torch.int64, device=dev)
        empty = torch.zeros(0, dtype=torch.int32, device=dev)
        for i in range(n):
            if i:
                h = m.decode_step(next_ids, None, cache)
            lm_head_logits_(h, w, logits)
            if mode == "guided":
                guidance_mix_(logits, Vv, B, scale)
            before = logits[:B].clone()
            penalize_repeats_(logits[:B], Vv, seq, prompt_len, cache.lens[:B], step, next_ids[:B], None, 1, 1.0, 0,
                              **REF)
            _check_op(logits[:B], before, Vv, seq, cache.lens[:B], prompt_len, B)
            sample_tokens_(logits[:B], Vv, temp, 0, 0.95, seeds, cache.lens[:B], step, 0, empty, empty, done,
                           next_ids[:B], want)
            if mode == "guided":
                next_ids[B:].copy_(next_ids[:B])
    assert torch.equal(tokens, want), mode
    for b, x in enumerate(lengths):
        full = ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist()
        assert not copied_ngrams(full, x, 3), (mode, b)


@pytest.mark.parametrize("mode", ["greedy", "sampled", "groups", "stochastic"])
def test_beam_decoders_graph_equal_eager_loop(dev, mode):
    """``beam_search`` (greedy, sampled, groups) and ``stochastic_beam_search`` (graph replay) against an eager loop of
    the same kernels (``penalize_repeats_`` with a parent map, ``beam_step_``, ``kv_reorder_``): bit-identical
    results; at every step of the loop the op's output equals the reference on the sequences it keeps."""
    from adapcc_b200.ops import (BeamState, beam_step_, kv_reorder_, kv_reorder_scratch_numel, lm_head_logits_,
                                 penalize_repeats_)
    from adapcc_b200.ops.beam import best_hypotheses, merge_finished_sets, stochastic_results

    m = _gpt2_small(dev, seed=1)
    Vv = m.cfg.vocab_size
    B, K, n, alpha = 4, 8 if mode != "groups" else 16, 16, 0.8
    lengths = [64, 17, 120, 40]
    ids = _prompts(dev, B, 120, 9)
    seeds = torch.arange(7, 7 + B, dtype=torch.int64)
    scalars = dict(temperature=0.9, top_k=40, top_p=0.95)
    if mode == "stochastic":
        call = lambda **kw: m.stochastic_beam_search(ids, lengths, num_beams=K, max_new_tokens=n, seed=seeds,  # noqa
                                                     **scalars, **kw)
        st = BeamState(B, K, n, 1.0, dev, seeds=seeds.to(dev))
        step_kw = scalars
    else:
        extra = dict(greedy={}, sampled=dict(do_sample=True, seed=seeds, **scalars),
                     groups=dict(num_beam_groups=4, diversity_penalty=0.7))[mode]
        call = lambda **kw: m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha,  # noqa
                                          num_return_sequences=K, **extra, **kw)
        st = BeamState(B, K, n, alpha, dev, sample=mode == "sampled", groups=4 if mode == "groups" else 1)
        step_kw = (dict(seeds=seeds.to(dev), **scalars) if mode == "sampled" else
                   dict(diversity_penalty=0.7 if mode == "groups" else 0.0))
    free = call()
    out = call(**CONTROLS)
    assert not torch.equal(out[0], free[0])
    w = m.wte.weight
    with torch.no_grad():
        T = ids.shape[1]
        last = torch.tensor(lengths, device=dev) - 1
        pre = m.new_cache(B, T)
        h = m.hidden(ids, None, cache=pre, lengths=lengths)[torch.arange(B, device=dev), last]
        cache = m.new_cache(B * K, max(lengths) + n)
        cache.reset([x for x in lengths for _ in range(K)], T)
        cache.k[:, :, :, :T].copy_(pre.k.repeat_interleave(K, dim=1))
        cache.v[:, :, :, :T].copy_(pre.v.repeat_interleave(K, dim=1))
        h = h.repeat_interleave(K, dim=0).contiguous()
        prompt_len = cache.lens.clone()
        seq = torch.zeros(B * K, cache.t_max, dtype=torch.int32, device=dev)
        seq[:, :T] = ids.repeat_interleave(K, dim=0)
        scratch = torch.empty(kv_reorder_scratch_numel(cache.k, n), dtype=cache.k.dtype, device=dev)
        logits = torch.empty(B * K, w.shape[0], dtype=torch.float32, device=dev)
        for i in range(n):
            if i:
                h = m.decode_step(st.next_ids, None, cache)
            lm_head_logits_(h, w, logits)
            before = logits.clone()
            penalize_repeats_(logits, Vv, seq, prompt_len, cache.lens, st.step, st.next_ids, st.parent, K, 1.0, 0,
                              **REF)
            _check_op(logits, before, Vv, seq, cache.lens, prompt_len, B * K)
            beam_step_(logits, Vv, st, 0, None, None, **step_kw)
            kv_reorder_(cache.k, cache.v, st.parent, prompt_len, cache.lens, n, scratch)
    hist_tok, hist_back = st.hist_tok.view(n, B, K).cpu().numpy(), st.hist_back.view(n, B, K).cpu().numpy()
    if mode == "stochastic":
        fin = [sets[0] for sets in st.finished()]
        want = stochastic_results(fin, hist_tok, hist_back, n, K, st.kappa.cpu().numpy())
    else:
        fin = [merge_finished_sets(sets) for sets in st.finished()]
        want = best_hypotheses(fin, hist_tok, hist_back, n, K)
    assert torch.equal(out[0].cpu(), want[0]) and torch.equal(out[1].cpu(), want[1]), mode
    for q in range(2, len(want)):
        assert torch.equal(out[q].cpu().view(torch.int32), want[q].view(torch.int32)), (mode, q)
    for q in range(B * K):
        b = q // K
        full = ids[b, :lengths[b]].tolist() + out[0][q, :int(out[1][q])].tolist()
        assert not copied_ngrams(full, lengths[b], 3), (mode, q)


def test_contrastive_search_graph_equals_eager_reference_loop(dev):
    """Contrastive search with the new controls against the eager loop of the same model calls, the reference on each
    row's sequence and ops/contrastive.py in fp64; a row may differ only after a near tie of its scores."""
    from adapcc_b200.models.gpt2 import CandidateKV
    from adapcc_b200.ops import ContrastiveState, lm_head_logits_
    from adapcc_b200.ops.contrastive import rerank_row, select_candidates
    from adapcc_b200.ops.repeats import penalize_repeats_reference

    m = _gpt2_small(dev)
    cfg = m.cfg
    Vv, Lr, H, D = cfg.vocab_size, cfg.n_layer, cfg.n_head, cfg.n_embd
    lengths = [200, 37, 128, 9, 64, 199, 150, 90]
    B, K, alpha, n = 8, 4, 0.6, 24
    ids = _prompts(dev, B, 200, 4)
    free, _ = m.contrastive_search(ids, lengths, top_k=K, penalty_alpha=alpha, max_new_tokens=n)
    got, n_new = m.contrastive_search(ids, lengths, top_k=K, penalty_alpha=alpha, max_new_tokens=n, **CONTROLS)
    tol = 2 * (alpha * (2 * D + 4) * U32 + (1 - alpha) * (math.ceil(Vv / 512) + 20) * U32 + 4 * U32)
    with torch.no_grad():
        t_max = max(lengths) + n
        cache = m.new_cache(B, t_max)
        hs = m.hidden(ids, None, cache=cache, lengths=lengths)
        ctx = [hs[b, :x].double().cpu().numpy() for b, x in enumerate(lengths)]
        h = hs[torch.arange(B, device=dev), torch.tensor(lengths, device=dev) - 1].contiguous()
        st = ContrastiveState(B, K, n, t_max, Lr, H, D // H, dev)
        cand = CandidateKV(cache, K, st.side, st.work)
        logits = torch.empty(B, m.wte.weight.shape[0], dtype=torch.float32, device=dev)
        tokens = torch.full((B, n), -1, dtype=torch.int64)
        done = np.zeros(B, dtype=bool)
        near = np.zeros(B, dtype=bool)
        rows = torch.arange(B, device=dev)
        seqs = [ids[b, :x].tolist() for b, x in enumerate(lengths)]
        for i in range(n):
            lm_head_logits_(h, m.wte.weight, logits)
            lc = penalize_repeats_reference(logits, seqs, Vv, 1.0, 0, prompt_lens=lengths, **REF)
            cid, probs = select_candidates(lc, Vv, K, i, 0, (), done)
            hc = m._candidate_hidden(cid.clamp(min=0).reshape(-1).to(dev), None, cand)
            hk = hc.view(B, K, D).double().cpu().numpy()
            pick = []
            for b in range(B):
                r = rerank_row(cid[b].numpy(), probs[b].numpy(), hk[b], ctx[b], alpha)
                sc = np.sort(r["scores"][np.isfinite(r["scores"])])[::-1]
                near[b] |= sc.size > 1 and sc[0] - sc[1] <= tol
                pick.append(b * K + r["rank"])
                tokens[b, i] = r["token"]
                seqs[b].append(int(r["token"]))
                ctx[b] = np.concatenate([ctx[b], hk[b, r["rank"]][None]])
            pick = torch.tensor(pick, device=dev)
            pos = cache.lens.long()
            cache.k[:, rows, :, pos] = st.side[:, 0, pick].view(Lr, B, H, D // H).transpose(0, 1)
            cache.v[:, rows, :, pos] = st.side[:, 1, pick].view(Lr, B, H, D // H).transpose(0, 1)
            cache.advance()
            h = hc[pick].contiguous()
    exempt = 0
    for b, x in enumerate(lengths):
        assert not copied_ngrams(ids[b, :x].tolist() + got[b, :int(n_new[b])].tolist(), x, 3), b
        if torch.equal(got[b].cpu(), tokens[b]):
            continue
        assert near[b], (b, got[b].tolist(), tokens[b].tolist())
        exempt += 1
    print(f"contrastive_search with the penalties, graph vs eager fp64 loop: {B} rows, {exempt} exempt")
    assert exempt <= 2 and not torch.equal(got, free)
