"""Repetition controls on the GPU: ``penalize_repeats_`` against the definition (ops/repeats.py) bit for bit, its
sequence update and group reorder against a torch gather, a row alone against the same row in a batch, graph replay
against eager launches, and ``generate`` / ``beam_search`` on GPT-2 small against eager loops of the same decode step
and LM head with the reference processor and the fp64 sampling and beam definitions."""
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
    """fp32 [R, LD] with +-0, subnormals and -inf planted among the low ids the sequences repeat."""
    x = (rng.standard_normal((R, LD)) * 4).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-40, -1e-40, 1.4e-45, -np.inf, 3e-39, -2e-38], dtype=np.float32)
    for r in range(R):
        cols = rng.choice(64, size=special.size, replace=False)
        x[r, cols] = special
    return x


def _sequences(rng, R, lens):
    """int32 [R, T_MAX]: random ids, small alphabets and copied segments (so every n has matches), a few ids outside
    the vocabulary, and a copy of an earlier stretch at the end of some rows."""
    seq = np.full((R, T_MAX), -7, dtype=np.int32)                  # padding beyond lens, never read
    for r in range(R):
        L = int(lens[r])
        hi = [8, 64, V][r % 3]
        s = rng.integers(0, hi, L)
        if L > 20 and r % 2 == 0:                                   # the tail repeats an earlier stretch
            j = int(rng.integers(0, L - 12))
            s[L - 8:] = s[j:j + 8]
        s[rng.random(L) < 0.01] = V + int(rng.integers(0, 40))      # ids >= vocab (< ld) are ignored
        s[rng.random(L) < 0.005] = -1
        seq[r, :L] = s
    return seq


def _run(dev, logits, seq, prompt_len, lens, step, ids, parent, group, p, n):
    from adapcc_b200.ops import penalize_repeats_

    i32 = dict(dtype=torch.int32, device=dev)
    t = dict(logits=torch.from_numpy(logits).to(dev), seq=torch.from_numpy(seq).to(dev),
             prompt_len=torch.as_tensor(prompt_len, **i32), lens=torch.as_tensor(lens, **i32),
             step=torch.tensor([step], **i32), ids=torch.as_tensor(ids, dtype=torch.int64, device=dev),
             parent=None if parent is None else torch.as_tensor(parent, **i32))
    penalize_repeats_(t["logits"], V, t["seq"], t["prompt_len"], t["lens"], t["step"], t["ids"], t["parent"], group,
                      p, n)
    torch.cuda.synchronize()
    return t


def _want(logits, seq, lens, p, n):
    from adapcc_b200.ops.repeats import penalize_repeats_reference

    return penalize_repeats_reference(torch.from_numpy(logits), [seq[r, :int(x)] for r, x in enumerate(lens)], V, p, n)


PN = [(0.7, 1), (1.3, 2), (2.0, 3), (1.0, 4), (1.3, 8), (0.7, 0), (2.0, 1), (1.0, 3)]


def test_kernel_matches_reference_bit_for_bit(dev):
    rng = np.random.default_rng(0)
    rows = 0
    for R in (1, 2, 7, 33, 64):
        for p, n in PN:
            lens = rng.integers(1, T_MAX + 1, R)
            lens[0], lens[-1] = T_MAX, max(1, n - 1)                 # a full row and a row shorter than n
            logits, seq = _logits(rng, R), _sequences(rng, R, lens)
            got = _run(dev, logits, seq, lens, lens, 0, np.zeros(R), None, 1, p, n)
            assert torch.equal(got["seq"].cpu(), torch.from_numpy(seq))            # step 0: the prompt as stored
            want = _want(logits, seq, lens, p, n)
            assert torch.equal(_bits(got["logits"]), _bits(want)), (R, p, n)
            rows += R
    # with *step > 0 the consumed token is appended first, at lens - 1
    R = 24
    lens = rng.integers(2, T_MAX + 1, R)
    logits, seq = _logits(rng, R), _sequences(rng, R, lens)
    ids = rng.integers(0, 64, R)
    got = _run(dev, logits, seq, lens - 1, lens, 5, ids, None, 1, 1.3, 3)
    seq[np.arange(R), lens - 1] = ids
    assert torch.equal(got["seq"].cpu(), torch.from_numpy(seq))
    assert torch.equal(_bits(got["logits"]), _bits(_want(logits, seq, lens, 1.3, 3)))
    print(f"penalize_repeats_ vs reference: {rows + R} rows, every bit equal")


def _maps(K, G):
    out = {"identity": [g * K + k for g in range(G) for k in range(K)],
           "swap": [g * K + (k ^ 1 if (k ^ 1) < K else k) for g in range(G) for k in range(K)],
           "cycle": [g * K + (k + 1) % K for g in range(G) for k in range(K)],
           "all_from_one": [g * K + K - 1 for g in range(G) for k in range(K)]}
    return out


def test_group_reorder_against_torch_gather(dev):
    rng = np.random.default_rng(1)
    for K in range(1, 17):
        G = max(1, 64 // K)
        R = G * K
        gen = np.repeat([40 - g % 3 for g in range(G)], K)             # generated regions that end near t_max
        prompt_len = np.repeat([T_MAX - 40 - g % 5 for g in range(G)], K)
        lens = prompt_len + gen
        for name, parent in _maps(K, G).items():
            logits, seq = _logits(rng, R), _sequences(rng, R, lens)
            for g in range(G):                                       # every row of an item shares its prompt
                seq[g * K:(g + 1) * K, :prompt_len[g * K]] = seq[g * K, :prompt_len[g * K]]
            ids = rng.integers(0, 64, R)
            got = _run(dev, logits, seq, prompt_len, lens, 7, ids, parent, K, 1.3, 3)
            src = torch.from_numpy(seq)
            want = src.clone()
            for r, pr in enumerate(parent):
                lo, hi = int(prompt_len[r]), int(lens[r]) - 1
                want[r, lo:hi] = src[pr, lo:hi]
                want[r, hi] = int(ids[r])
            assert torch.equal(got["seq"].cpu(), want), (K, name)
            assert torch.equal(_bits(got["logits"]), _bits(_want(logits, want.numpy(), lens, 1.3, 3))), (K, name)


def test_row_alone_equals_row_in_batch_and_graph_equals_eager(dev):
    from adapcc_b200.ops import penalize_repeats_

    rng = np.random.default_rng(2)
    R, K = 16, 4
    lens = rng.integers(100, T_MAX + 1, R)
    prompt_len = lens - 10
    logits, seq = _logits(rng, R), _sequences(rng, R, lens)
    ids = rng.integers(0, 64, R)
    full = _run(dev, logits, seq, prompt_len, lens, 3, ids, None, 1, 0.7, 2)
    for r in range(R):
        one = _run(dev, logits[r:r + 1].copy(), seq[r:r + 1].copy(), prompt_len[r:r + 1], lens[r:r + 1], 3,
                   ids[r:r + 1], None, 1, 0.7, 2)
        assert torch.equal(_bits(one["logits"][0]), _bits(full["logits"][r])), r
        assert torch.equal(one["seq"][0], full["seq"][r]), r
    # a graph replay with a parent map equals an eager launch
    parent = _maps(K, R // K)["cycle"]
    eager = _run(dev, logits, seq, prompt_len, lens, 3, ids, parent, K, 1.3, 3)
    t = _run(dev, logits, seq, prompt_len, lens, 0, ids, parent, K, 1.3, 3)           # step 0: a no-op on seq
    t["step"].fill_(3)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        penalize_repeats_(t["logits"], V, t["seq"], t["prompt_len"], t["lens"], t["step"], t["ids"], t["parent"], K,
                          1.3, 3)
    t["logits"].copy_(torch.from_numpy(logits))
    t["seq"].copy_(torch.from_numpy(seq))
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(_bits(t["logits"]), _bits(eager["logits"])) and torch.equal(t["seq"], eager["seq"])


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def repeated_ngram(full, start, n):
    for t in range(max(start, n - 1), len(full)):
        gram = full[t - n + 1:t + 1]
        if any(full[j:j + n] == gram for j in range(t - n + 1)):
            return t
    return None


def _margin_ok(r, Vv):
    """A sampled token may differ from the fp64 definition only where a decision quantity sits at its threshold within
    the sampler's fp32 error (the bound of test_gpu_generate.py: C + 74 roundings per sum plus the weight errors)."""
    if "e" not in r:
        return False
    C = math.ceil(Vv / 1024)
    xm = np.where(r["e"] > 0, -np.log(np.maximum(r["e"], 1e-300)), 0.0)
    bound = (C + 74) * U32 * r["Z"] + 2 * float(((4 + xm) * U32 * r["e"]).sum())
    tail = r["tail"][np.isfinite(r["tail"])]
    return ((r["pZ"] < r["Z"] and bool((np.abs(tail - r["pZ"]) <= bound).any()))
            or bool((np.abs(r["cum"][r["kept"]] - r["target"]) <= bound).any()))


def test_generate_graph_equals_eager_reference_loop(dev, monkeypatch):
    """The graph path against an eager loop of the same decode step and LM head, the reference processor and the fp64
    sampling definition, fed the graph's own tokens so that every step is compared. Greedy steps must agree exactly
    (arg-max of the same fp32 values); a sampled step may differ only at a near tie of its decision."""
    import adapcc_b200.ops as ops
    from adapcc_b200.ops import lm_head_logits_
    from adapcc_b200.ops.repeats import penalize_repeats_reference
    from adapcc_b200.ops.sampling import reference_row

    m = _gpt2_small(dev, seed=2)
    Vv = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(5)
    B, n, p, ng = 6, 24, 1.3, 3
    lengths = [90, 17, 64, 5, 120, 33]
    ids = torch.randint(0, 200, (B, 120), device=dev, generator=g)          # a small alphabet: repeats in prompts
    w = m.wte.weight
    for temperature, top_p in ((0.0, 1.0), (0.9, 0.9)):
        tokens, n_new = m.generate(ids, lengths, max_new_tokens=n, temperature=temperature, top_p=top_p, seed=40,
                                   repetition_penalty=p, no_repeat_ngram_size=ng)
        assert n_new.tolist() == [n] * B
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
                lc = penalize_repeats_reference(logits, seqs, Vv, p, ng).cpu().numpy()
                pos = cache.lens.cpu().tolist()
                for b in range(B):
                    r = reference_row(lc[b, :Vv], temperature, 0, top_p, 40 + b, pos[b], i)
                    got = int(tokens[b, i])
                    if r["token"] == got:
                        continue
                    if temperature == 0:                             # the same fp32 values give the same arg-max
                        top = float(lc[b, r["token"]])
                        assert top - float(lc[b, got]) <= 4 * U32 * (1 + abs(top)), (b, i, r["token"], got)
                    else:
                        assert _margin_ok(r, Vv), (b, i)
                    exempt += 1
        print(f"generate (T={temperature}) graph vs eager reference loop: {B * n} tokens, {exempt} exempt")
        assert exempt <= B * n // 50
        for b, x in enumerate(lengths):
            full = ids[b, :x].tolist() + tokens[b].tolist()
            assert repeated_ngram(full, x, ng) is None, b
    # with the defaults the op is not called, and the tokens are those of a call that never mentions the options
    want, _ = m.generate(ids, lengths, max_new_tokens=8, temperature=0.0)
    monkeypatch.setattr(ops, "penalize_repeats_", None)
    got, _ = m.generate(ids, lengths, max_new_tokens=8, temperature=0.0, repetition_penalty=1.0,
                        no_repeat_ngram_size=0)
    assert torch.equal(got, want)


def _tol(Vv, cs):
    """The fp32 error bound of a beam candidate score of test_gpu_beam.py: |c32 - c64| <= (4 M + C + 14) u with
    M = 1 + max |c| and C = ceil(V / 512) terms per thread; two candidates closer than twice that may swap."""
    M = 1.0 + max(abs(c) for c in cs) if cs else 1.0
    return 2.0 * (4.0 * M + math.ceil(Vv / 512) + 14) * U32


def _near(vals, tol):
    v = np.sort(np.asarray([x for x in vals if np.isfinite(x)], dtype=np.float64))
    d = np.diff(v)
    return bool(((d > 0) & (d <= tol)).any())


def test_beam_search_graph_equals_eager_reference_loop(dev):
    """The pattern of test_gpu_beam.py: beam search with both controls against an eager loop of the same decode step
    and LM head, the reference processor on each beam's own sequence, ops/beam.py in fp64 and torch reordering. An item
    may differ only if one of its steps had two candidates within the fp32 bound of each other."""
    from adapcc_b200.ops import lm_head_logits_
    from adapcc_b200.ops.beam import BeamReference
    from adapcc_b200.ops.repeats import penalize_repeats_reference

    m = _gpt2_small(dev, seed=1)
    Vv = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(9)
    B, K, n, alpha, p, ng = 6, 4, 20, 0.8, 1.2, 3
    lengths = [64, 17, 120, 40, 5, 99]
    ids = torch.randint(0, 300, (B, 120), device=dev, generator=g)
    stop = [int(ids[0, 0]), int(ids[1, 1])]
    tokens, n_new, scores = m.beam_search(ids, lengths, num_beams=K, max_new_tokens=n, length_penalty=alpha,
                                          stop_ids=stop, repetition_penalty=p, no_repeat_ngram_size=ng)
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
        ref = BeamReference(B, K, n, Vv, alpha, stop)
        logits = torch.empty(B * K, w.shape[0], dtype=torch.float32, device=dev)
        seqs = [ids[r // K, :lengths[r // K]].tolist() for r in range(B * K)]
        near = np.zeros(B, dtype=bool)
        for i in range(n):
            if i:
                h = m.decode_step(nxt.to(dev), None, cache)
                seqs = [seqs[int(pr)] + [int(t)] for pr, t in zip(parent, nxt)]
            lm_head_logits_(h, w, logits)
            lc = penalize_repeats_reference(logits, seqs, Vv, p, ng).cpu().numpy()
            for b in range(B):
                if not ref.done[b]:
                    cs = [c for c, _, _ in ref.ranking(b, lc, i)[:K * (K + len(stop))]]
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
        full = ids[b, :lengths[b]].tolist() + tokens[b, :k].tolist()
        assert repeated_ngram(full, lengths[b], ng) is None, b
        if torch.equal(tokens[b].cpu(), rt[b]) and k == int(rn[b]):
            assert float(scores[b]) == pytest.approx(float(rs[b]), abs=1e-3), b
            continue
        assert near[b], b
        exempt += 1
    print(f"beam_search with repetition controls, graph vs eager fp64 loop: {B} items, {exempt} exempt")
    assert exempt <= B // 2
