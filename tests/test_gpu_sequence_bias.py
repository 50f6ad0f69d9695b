"""Sequence bias and bad-word blocking on the GPU: rule 0 of ``penalize_repeats_`` against the definition
(ops/repeats.py) bit for bit, alone and with the penalty and n-gram rules, with and without parent maps, a row alone
against the same row in a batch, graph replay against eager launches, and ``generate``, ``beam_search``,
``stochastic_beam_search`` and ``contrastive_search`` on GPT-2 small against eager loops with the reference."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24          # unit roundoff of fp32
V, LD, T_MAX = 50257, 50304, 1024


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
    """fp32 [R, LD] with +-0, subnormals and -inf planted among the low ids the sequences and tables use."""
    x = (rng.standard_normal((R, LD)) * 4).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-40, -1e-40, 1.4e-45, -np.inf, 3e-39, -2e-38], dtype=np.float32)
    for r in range(R):
        x[r, rng.choice(64, size=special.size, replace=False)] = special
    return x


def _sequences(rng, R, lens):
    seq = np.full((R, T_MAX), -7, dtype=np.int32)                  # padding beyond lens, never read
    for r in range(R):
        L = int(lens[r])
        seq[r, :L] = rng.integers(0, [8, 64, V][r % 3], L)
    return seq


def _table(rng, seq, lens, n_entries, max_len):
    """A random table of ``n_entries`` entries of 1 to ``max_len`` ids, most of them planted on some row's tail (so
    they apply), with repeated targets, finite biases of every size and bad words."""
    from adapcc_b200.ops.repeats import check_sequence_bias_args

    R = seq.shape[0]
    sb, bad = {}, []
    while len(sb) + len(bad) < n_entries:
        m = int(rng.integers(1, max_len + 1))
        r = int(rng.integers(0, R))
        L = int(lens[r])
        if rng.random() < 0.7 and L >= m:
            pre = seq[r, L - m + 1:L].tolist()
        else:
            pre = rng.integers(0, 8, m - 1).tolist()
        s = tuple(pre) + (int(rng.integers(0, 48)),)
        if rng.random() < 0.15:
            bad.append(list(s))
        elif s not in sb:
            sb[s] = float(rng.choice([rng.standard_normal() * 3, rng.standard_normal() * 1e30, 2.0 ** -30]))
    return check_sequence_bias_args("test", sb, bad, V)


def _run(dev, logits, seq, prompt_len, lens, step, ids, parent, group, p, n, table):
    from adapcc_b200.ops import penalize_repeats_

    i32 = dict(dtype=torch.int32, device=dev)
    t = dict(logits=torch.from_numpy(logits).to(dev), seq=torch.from_numpy(seq).to(dev),
             prompt_len=torch.as_tensor(prompt_len, **i32), lens=torch.as_tensor(lens, **i32),
             step=torch.tensor([step], **i32), ids=torch.as_tensor(ids, dtype=torch.int64, device=dev),
             parent=None if parent is None else torch.as_tensor(parent, **i32))
    penalize_repeats_(t["logits"], V, t["seq"], t["prompt_len"], t["lens"], t["step"], t["ids"], t["parent"], group,
                      p, n, table)
    torch.cuda.synchronize()
    return t


def _want(logits, seq, lens, p, n, table):
    from adapcc_b200.ops.repeats import penalize_repeats_reference

    return penalize_repeats_reference(torch.from_numpy(logits), [seq[r, :int(x)] for r, x in enumerate(lens)], V, p, n,
                                      table)


def test_kernel_matches_reference_bit_for_bit(dev):
    from adapcc_b200.ops.repeats import BIAS_MAX_ENTRIES, BIAS_MAX_LEN

    rng = np.random.default_rng(0)
    rows = 0
    for R, n_entries, max_len, p, n in ((1, 1, 1, 1.0, 0), (1, 64, 4, 1.0, 0), (8, 64, 4, 1.3, 2),
                                        (8, BIAS_MAX_ENTRIES, BIAS_MAX_LEN, 1.0, 0), (33, 300, 8, 0.7, 3),
                                        (64, BIAS_MAX_ENTRIES, 4, 2.0, 1), (64, 200, BIAS_MAX_LEN, 1.0, 4)):
        lens = rng.integers(1, T_MAX + 1, R)
        lens[0] = T_MAX
        if R > 1:
            lens[-1] = 1
        logits, seq = _logits(rng, R), _sequences(rng, R, lens)
        table = _table(rng, seq, lens, n_entries, max_len)
        got = _run(dev, logits, seq, lens, lens, 0, np.zeros(R), None, 1, p, n, table)
        want = _want(logits, seq, lens, p, n, table)
        assert torch.equal(_bits(got["logits"]), _bits(want)), (R, n_entries, max_len, p, n)
        changed = int((_bits(want) != _bits(torch.from_numpy(logits))).sum())
        assert changed > 0
        rows += R
    # with *step > 0 the consumed token is appended first, and rule 0 sees it
    R = 24
    lens = rng.integers(40, T_MAX + 1, R)
    logits, seq = _logits(rng, R), _sequences(rng, R, lens)
    ids = rng.integers(0, 64, R)
    seq2 = seq.copy()
    seq2[np.arange(R), lens - 1] = ids
    table = _table(rng, seq2, lens, 500, 6)
    got = _run(dev, logits, seq, lens - 1, lens, 5, ids, None, 1, 1.3, 3, table)
    assert torch.equal(got["seq"].cpu(), torch.from_numpy(seq2))
    assert torch.equal(_bits(got["logits"]), _bits(_want(logits, seq2, lens, 1.3, 3, table)))
    print(f"penalize_repeats_ with sequence bias vs reference: {rows + R} rows, every bit equal")


def test_parent_maps(dev):
    rng = np.random.default_rng(1)
    for K in (1, 2, 4, 7, 16):
        G = max(1, 64 // K)
        R = G * K
        prompt_len = np.repeat([T_MAX - 40 - g % 5 for g in range(G)], K)
        lens = prompt_len + np.repeat([40 - g % 3 for g in range(G)], K)
        for parent in ([g * K + (k + 1) % K for g in range(G) for k in range(K)],
                       [g * K + K - 1 for g in range(G) for k in range(K)]):
            logits, seq = _logits(rng, R), _sequences(rng, R, lens)
            for g in range(G):
                seq[g * K:(g + 1) * K, :prompt_len[g * K]] = seq[g * K, :prompt_len[g * K]]
            ids = rng.integers(0, 64, R)
            want_seq = seq.copy()
            for r, pr in enumerate(parent):
                lo, hi = int(prompt_len[r]), int(lens[r]) - 1
                want_seq[r, lo:hi] = seq[pr, lo:hi]
                want_seq[r, hi] = ids[r]
            table = _table(rng, want_seq, lens, 400, 12)           # planted on the reordered rows' tails
            for p, n in ((1.0, 0), (1.3, 3)):
                got = _run(dev, logits, seq, prompt_len, lens, 7, ids, parent, K, p, n, table)
                assert torch.equal(got["seq"].cpu(), torch.from_numpy(want_seq)), K
                assert torch.equal(_bits(got["logits"]), _bits(_want(logits, want_seq, lens, p, n, table))), (K, p)


def test_row_alone_equals_row_in_batch_and_graph_equals_eager(dev):
    from adapcc_b200.ops import penalize_repeats_

    rng = np.random.default_rng(2)
    R, K = 16, 4
    lens = rng.integers(100, T_MAX + 1, R)
    prompt_len = lens - 10
    logits, seq = _logits(rng, R), _sequences(rng, R, lens)
    ids = rng.integers(0, 64, R)
    table = _table(rng, seq, lens, 700, 10)
    full = _run(dev, logits, seq, prompt_len, lens, 3, ids, None, 1, 0.7, 2, table)
    for r in range(R):
        one = _run(dev, logits[r:r + 1].copy(), seq[r:r + 1].copy(), prompt_len[r:r + 1], lens[r:r + 1], 3,
                   ids[r:r + 1], None, 1, 0.7, 2, table)
        assert torch.equal(_bits(one["logits"][0]), _bits(full["logits"][r])), r
    parent = [g * K + (k + 1) % K for g in range(R // K) for k in range(K)]
    eager = _run(dev, logits, seq, prompt_len, lens, 3, ids, parent, K, 1.0, 0, table)
    t = _run(dev, logits, seq, prompt_len, lens, 0, ids, parent, K, 1.0, 0, table)
    t["step"].fill_(3)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        penalize_repeats_(t["logits"], V, t["seq"], t["prompt_len"], t["lens"], t["step"], t["ids"], t["parent"], K,
                          1.0, 0, table)
    t["logits"].copy_(torch.from_numpy(logits))
    t["seq"].copy_(torch.from_numpy(seq))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(t["logits"]), _bits(eager["logits"])) and torch.equal(t["seq"], eager["seq"])


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def occurrences(full, start, banned):
    """Every banned sequence in ``full`` whose last id is at a position t >= start where the rule applies: t >= m, the
    sequence before it at least as long as the entry (so not one that starts at position 0)."""
    return [(t, tuple(s)) for s in banned for t in range(max(start, len(s)), len(full))
            if tuple(full[t - len(s) + 1:t + 1]) == tuple(s)]


def _options(free, ids, lengths):
    """A bias and bad words that act on the unbiased replies ``free``: bigrams of the replies banned (one crossing
    the prompt / reply boundary), ids pushed down after their predecessors and one pushed up everywhere."""
    bias, bad = {}, []
    for b, x in enumerate(lengths):
        full = ids[b, :x].tolist() + free[b].tolist()
        bad.append(full[x - 1:x + 1])
        bad.append(full[x + 4:x + 6])
        bias.setdefault(tuple(full[x + 1:x + 3]), -4.0)
        bias.setdefault(tuple(full[x + 7:x + 10]), -1.5)
    bias[(int(free[0, 12]),)] = 2.5
    return bias, bad


def test_generate_graph_equals_eager_reference_loop(dev):
    """Greedy ``generate`` with a bias and bad words against an eager loop of the same decode step and LM head with
    the reference: the same fp32 values give the same arg-max, so the tokens must agree up to exact near ties."""
    from adapcc_b200.ops import lm_head_logits_
    from adapcc_b200.ops.repeats import check_sequence_bias_args, penalize_repeats_reference

    m = _gpt2_small(dev, seed=2)
    Vv = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(5)
    B, n = 6, 24
    lengths = [90, 17, 64, 5, 120, 33]
    ids = torch.randint(0, 200, (B, 120), device=dev, generator=g)
    free, _ = m.generate(ids, lengths, max_new_tokens=n, temperature=0.0)
    bias, bad = _options(free, ids, lengths)
    table = check_sequence_bias_args("test", bias, bad, Vv)
    tokens, n_new = m.generate(ids, lengths, max_new_tokens=n, temperature=0.0, sequence_bias=bias,
                               bad_words_ids=bad, repetition_penalty=1.2)
    assert n_new.tolist() == [n] * B and not torch.equal(tokens, free)
    w = m.wte.weight
    exempt = 0
    with torch.no_grad():
        cache = m.new_cache(B, max(lengths) + n)
        last = torch.tensor(lengths, device=dev) - 1
        h = m.hidden(ids, None, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last]
        logits = torch.empty(B, w.shape[0], dtype=torch.float32, device=dev)
        seqs = [ids[b, :x].tolist() for b, x in enumerate(lengths)]
        for i in range(n):
            if i:
                h = m.decode_step(tokens[:, i - 1].contiguous(), None, cache)
                for b in range(B):
                    seqs[b].append(int(tokens[b, i - 1]))
            lm_head_logits_(h, w, logits)
            lc = penalize_repeats_reference(logits, seqs, Vv, 1.2, 0, table)[:, :Vv]
            for b in range(B):
                want, got = int(lc[b].argmax()), int(tokens[b, i])
                if want != got:                                   # the same fp32 values give the same arg-max
                    top = float(lc[b, want])
                    assert top - float(lc[b, got]) <= 4 * U32 * (1 + abs(top)), (b, i, want, got)
                    exempt += 1
    print(f"generate with sequence bias, graph vs eager reference loop: {B * n} tokens, {exempt} exempt")
    assert exempt <= B * n // 50
    for b, x in enumerate(lengths):
        assert not occurrences(ids[b, :x].tolist() + tokens[b].tolist(), x, bad), b
    assert any(occurrences(ids[b, :x].tolist() + free[b].tolist(), x, bad) for b, x in enumerate(lengths))
    # sampled, guided: the ban holds there too
    for seed in (1, 2):
        t, k = m.generate(ids, lengths, max_new_tokens=n, temperature=1.0, top_p=1.0, seed=seed,
                          guidance_scale=1.5 if seed == 2 else 1.0, bad_words_ids=bad, sequence_bias=bias)
        for b, x in enumerate(lengths):
            assert not occurrences(ids[b, :x].tolist() + t[b, :int(k[b])].tolist(), x, bad), (seed, b)


def _tol(Vv, cs):
    """The fp32 error bound of a beam candidate score of test_gpu_beam.py."""
    M = 1.0 + max(abs(c) for c in cs) if cs else 1.0
    return 2.0 * (4.0 * M + math.ceil(Vv / 512) + 14) * U32


def _near(vals, tol):
    v = np.sort(np.asarray([x for x in vals if np.isfinite(x)], dtype=np.float64))
    d = np.diff(v)
    return bool(((d > 0) & (d <= tol)).any())


def test_beam_search_graph_equals_eager_reference_loop(dev):
    """Beam search with a bias and bad words against an eager loop of the same decode step and LM head, the reference
    on each beam's own sequence, ops/beam.py in fp64 and torch reordering. An item may differ only if one of its steps
    had two candidates within the fp32 bound of each other."""
    from adapcc_b200.ops import lm_head_logits_
    from adapcc_b200.ops.beam import BeamReference
    from adapcc_b200.ops.repeats import check_sequence_bias_args, penalize_repeats_reference

    m = _gpt2_small(dev, seed=1)
    Vv = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(9)
    B, K, n, alpha = 6, 4, 20, 0.8
    lengths = [64, 17, 120, 40, 5, 99]
    ids = torch.randint(0, 300, (B, 120), device=dev, generator=g)
    free = m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha)[0]
    bias, bad = _options(free, ids, lengths)
    table = check_sequence_bias_args("test", bias, bad, Vv)
    tokens, n_new, scores = m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha,
                                          sequence_bias=bias, bad_words_ids=bad)
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
        ref = BeamReference(B, K, n, Vv, alpha, ())
        logits = torch.empty(B * K, w.shape[0], dtype=torch.float32, device=dev)
        seqs = [ids[r // K, :lengths[r // K]].tolist() for r in range(B * K)]
        near = np.zeros(B, dtype=bool)
        for i in range(n):
            if i:
                h = m.decode_step(nxt.to(dev), None, cache)
                seqs = [seqs[int(pr)] + [int(t)] for pr, t in zip(parent, nxt)]
            lm_head_logits_(h, w, logits)
            lc = penalize_repeats_reference(logits, seqs, Vv, 1.0, 0, table).cpu().numpy()
            for b in range(B):
                if not ref.done[b]:
                    cs = [c for c, _, _ in ref.ranking(b, lc, i)[:K * K]]
                    near[b] |= _near(cs, _tol(Vv, cs))
            nxt, parent = ref.step(lc)
            rows = parent.to(dev)
            cache.k.copy_(cache.k[:, rows])
            cache.v.copy_(cache.v[:, rows])
            if ref.done.all():
                break
    rt, rn, rs = ref.result()
    exempt = 0
    for b in range(B):
        k = int(n_new[b])
        assert not occurrences(ids[b, :lengths[b]].tolist() + tokens[b, :k].tolist(), lengths[b], bad), b
        if torch.equal(tokens[b].cpu(), rt[b]) and k == int(rn[b]):
            assert float(scores[b]) == pytest.approx(float(rs[b]), abs=1e-3), b
            continue
        assert near[b], b
        exempt += 1
    print(f"beam_search with sequence bias, graph vs eager fp64 loop: {B} items, {exempt} exempt")
    assert exempt <= B // 2
    assert not torch.equal(tokens, free)


def test_stochastic_beam_search_graph_equals_eager_loop_of_the_same_kernels(dev):
    """The native decoder's graph against an eager loop of the same kernels (``penalize_repeats_`` with the table,
    ``beam_step_``, ``kv_reorder_``): bit-identical results. At every step the op's output also equals the reference
    on the sequences the op keeps, bit for bit."""
    from adapcc_b200.ops import (BeamState, beam_step_, kv_reorder_, kv_reorder_scratch_numel, lm_head_logits_,
                                 penalize_repeats_)
    from adapcc_b200.ops.beam import stochastic_results
    from adapcc_b200.ops.repeats import check_sequence_bias_args, penalize_repeats_reference

    m = _gpt2_small(dev, seed=1)
    Vv = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(9)
    B, K, n = 6, 4, 20
    lengths = [64, 17, 120, 40, 5, 99]
    ids = torch.randint(0, 300, (B, 120), device=dev, generator=g)
    kw = dict(temperature=0.9, top_k=40, top_p=0.95)
    seeds = torch.arange(7, 7 + B, dtype=torch.int64)
    free = m.stochastic_beam_search(ids, lengths, num_beams=K, max_new_tokens=n, seed=seeds, **kw)[0]
    bias, bad = _options(free[::K], ids, lengths)
    table = check_sequence_bias_args("test", bias, bad, Vv)
    out = m.stochastic_beam_search(ids, lengths, num_beams=K, max_new_tokens=n, seed=seeds, sequence_bias=bias,
                                   bad_words_ids=bad, **kw)
    st = BeamState(B, K, n, 1.0, dev, seeds=seeds)
    w = m.wte.weight
    checked = 0
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
                              table)
            L = cache.lens.cpu().tolist()
            want = penalize_repeats_reference(before, [seq[r, :L[r]].cpu() for r in range(B * K)], Vv, 1.0, 0, table)
            assert torch.equal(_bits(logits), _bits(want)), i
            checked += B * K
            beam_step_(logits, Vv, st, 0, None, None, **kw)
            kv_reorder_(cache.k, cache.v, st.parent, prompt_len, cache.lens, n, scratch)
    count = st.fin_count.cpu().tolist()
    cols = [x.cpu().tolist() for x in (st.fin_score, st.fin_n, st.fin_src, st.fin_phi)]
    fin = [list(zip(*(c[b] for c in cols)))[:count[b]] for b in range(B)]
    want = stochastic_results(fin, st.hist_tok.view(n, B, K).cpu().numpy(), st.hist_back.view(n, B, K).cpu().numpy(),
                              n, K, st.kappa.cpu().numpy())
    assert torch.equal(out[0].cpu(), want[0]) and torch.equal(out[1].cpu(), want[1])
    for q in (2, 3, 4):
        assert torch.equal(out[q].cpu().view(torch.int32), want[q].view(torch.int32)), q
    for q in range(B * K):
        b = q // K
        full = ids[b, :lengths[b]].tolist() + out[0][q, :int(out[1][q])].tolist()
        assert not occurrences(full, lengths[b], bad), q
    print(f"stochastic_beam_search with sequence bias: graph equals the eager loop; {checked} rows of the op equal "
          "the reference")


def test_contrastive_search_graph_equals_eager_reference_loop(dev):
    """Contrastive search with a bias and bad words against the eager loop of the same model calls, the reference on
    each row's sequence and ops/contrastive.py in fp64; a row may differ only after a near tie of its scores."""
    from adapcc_b200.models.gpt2 import CandidateKV
    from adapcc_b200.ops import ContrastiveState, lm_head_logits_
    from adapcc_b200.ops.contrastive import rerank_row, select_candidates
    from adapcc_b200.ops.repeats import check_sequence_bias_args, penalize_repeats_reference

    m = _gpt2_small(dev)
    cfg = m.cfg
    Vv, Lr, H, D = cfg.vocab_size, cfg.n_layer, cfg.n_head, cfg.n_embd
    g = torch.Generator(device=dev).manual_seed(4)
    lengths = [200, 37, 128, 1, 64, 199, 150, 90]
    B, K, alpha, n = 8, 4, 0.6, 24
    ids = torch.randint(0, 300, (B, 200), device=dev, generator=g)
    free, _ = m.contrastive_search(ids, lengths, top_k=K, penalty_alpha=alpha, max_new_tokens=n)
    bias, bad = _options(free, ids, lengths)
    table = check_sequence_bias_args("test", bias, bad, Vv)
    got, n_new = m.contrastive_search(ids, lengths, top_k=K, penalty_alpha=alpha, max_new_tokens=n,
                                      sequence_bias=bias, bad_words_ids=bad)
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
            lc = penalize_repeats_reference(logits, seqs, Vv, 1.0, 0, table)
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
        assert not occurrences(ids[b, :x].tolist() + got[b, :int(n_new[b])].tolist(), x, bad), b
        if torch.equal(got[b].cpu(), tokens[b]):
            continue
        assert near[b], (b, got[b].tolist(), tokens[b].tolist())
        exempt += 1
    print(f"contrastive_search with sequence bias, graph vs eager fp64 loop: {B} rows, {exempt} exempt")
    assert exempt <= 2 and not torch.equal(got, free)
