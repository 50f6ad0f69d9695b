"""Green-list watermarking on the GPU: ``watermark_`` and ``watermark_count_`` against the definition (ops/watermark.py)
bit for bit and count for count, a row alone against the same row in a batch, graph replay against eager launches, the
four decoders on GPT-2 small against eager loops with the reference, the exact all-green property, detection power and
false alarms bounded by binomial tails, and the launches a watermark adds to a replay."""
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
    """fp32 [R, LD] with +-0, subnormals and -inf planted at 256 random ids per row, so many of them are green."""
    x = (rng.standard_normal((R, LD)) * 4).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-40, -1e-40, 1.4e-45, -np.inf, 3e-39, -2e-38], dtype=np.float32)
    for r in range(R):
        x[r, rng.choice(LD, size=256, replace=False)] = np.resize(special, 256)
    return x


def _run(dev, logits, seq, lens, cfg):
    from adapcc_b200.ops import watermark_

    t = dict(logits=torch.from_numpy(logits).to(dev), seq=torch.from_numpy(seq).to(dev),
             lens=torch.as_tensor(lens, dtype=torch.int32, device=dev))
    watermark_(t["logits"], V, t["seq"], t["lens"], cfg)
    torch.cuda.synchronize()
    return t


def test_kernel_matches_reference_bit_for_bit(dev):
    from adapcc_b200.ops.watermark import watermark_reference

    rng = np.random.default_rng(0)
    rows = i = 0
    for scheme in ("lefthash", "selfhash"):
        for w in (1, 2, 3, 8):
            for gamma in (0.1, 0.25, 0.5, 0.9):
                R = (1, 8, 33, 64)[i % 4]
                delta = (2.0, -3.5, 1e30, 1e-3)[(i // 4) % 4]
                i += 1
                cfg = dict(seeding_scheme=scheme, context_width=w, greenlist_ratio=gamma, bias=delta,
                           hashing_key=int(rng.integers(0, 2 ** 63)) * 2 + 1)
                need = w - (scheme == "selfhash")                                # the length the rule needs
                lens = rng.integers(0, T_MAX + 1, R)
                lens[0] = T_MAX
                if R > 1:
                    lens[1] = need                                               # just long enough
                    lens[-1] = max(need - 1, 0)                                  # shorter, when anything is
                seq = rng.integers(0, V, (R, T_MAX)).astype(np.int32)
                logits = _logits(rng, R)
                got = _run(dev, logits, seq, lens, cfg)
                want = watermark_reference(torch.from_numpy(logits), [seq[r, :int(x)] for r, x in enumerate(lens)],
                                           V, cfg)
                assert torch.equal(_bits(got["logits"]), _bits(want)), cfg
                changed = (_bits(want) != _bits(torch.from_numpy(logits))).sum(1)
                assert int(changed[0]) > 0 and (R == 1 or need == 0 or int(changed[-1]) == 0)
                rows += R
    print(f"watermark_ vs reference: {rows} rows of {V} ids, every bit equal")


def test_row_alone_equals_row_in_batch_and_graph_equals_eager(dev):
    from adapcc_b200.ops import watermark_

    rng = np.random.default_rng(2)
    R = 16
    for cfg in (dict(context_width=2), dict(seeding_scheme="selfhash", context_width=4, greenlist_ratio=0.5)):
        lens = rng.integers(1, T_MAX + 1, R)
        logits, seq = _logits(rng, R), rng.integers(0, V, (R, T_MAX)).astype(np.int32)
        full = _run(dev, logits, seq, lens, cfg)
        for r in range(R):
            one = _run(dev, logits[r:r + 1].copy(), seq[r:r + 1].copy(), lens[r:r + 1], cfg)
            assert torch.equal(_bits(one["logits"][0]), _bits(full["logits"][r])), r
        t = dict(logits=torch.from_numpy(logits).to(dev), seq=torch.from_numpy(seq).to(dev),
                 lens=torch.as_tensor(lens, dtype=torch.int32, device=dev))
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            watermark_(t["logits"], V, t["seq"], t["lens"], cfg)
        t["logits"].copy_(torch.from_numpy(logits))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(t["logits"]), _bits(full["logits"]))
        # the graph reads the lengths and sequences on the device: new ones give the eager result for them
        lens2 = rng.integers(1, T_MAX + 1, R)
        t["lens"].copy_(torch.as_tensor(lens2, dtype=torch.int32))
        t["logits"].copy_(torch.from_numpy(logits))
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(t["logits"]), _bits(_run(dev, logits, seq, lens2, cfg)["logits"]))


def test_count_kernel_matches_reference_exactly(dev):
    from adapcc_b200.ops import watermark_count_
    from adapcc_b200.ops.watermark import watermark_counts_reference

    rng = np.random.default_rng(3)
    B, T = 64, 1024
    for cfg in (dict(), dict(context_width=3, greenlist_ratio=0.5), dict(seeding_scheme="selfhash"),
                dict(seeding_scheme="selfhash", context_width=4, hashing_key=2 ** 64 - 1)):
        ids = np.stack([rng.integers(0, (4, 50, V)[b % 3], T) for b in range(B)]).astype(np.int32)  # repeats too
        lens = rng.integers(0, T + 1, B)
        lens[0] = T
        starts = rng.integers(0, 40, B)
        starts[:4] = 0
        for ignore in (False, True):
            got = watermark_count_(torch.from_numpy(ids).to(dev), torch.as_tensor(lens, dtype=torch.int32, device=dev),
                                   torch.as_tensor(starts, dtype=torch.int32, device=dev), cfg, ignore)
            want = watermark_counts_reference(ids, lens, starts, cfg, ignore)
            assert np.array_equal(got.cpu().numpy(), want), (cfg, ignore)
            assert want[:, 1].sum() > 0
    print("watermark_count_ vs reference: every count equal")


# ---- the decoders on GPT-2 small --------------------------------------------------------------------------------------
WM = dict(bias=3.0, context_width=2)
WM_BEAM = dict(bias=2.0, seeding_scheme="selfhash", context_width=2, greenlist_ratio=0.5)


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def _prompts(dev, B, T, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(0, 300, (B, T), device=dev, generator=g)


def _check_op(logits, before, Vv, seq, lens, rows, wm, penalty=1.0):
    """The ops' output equals the reference rules on the sequences the repetition op keeps, bit for bit."""
    from adapcc_b200.ops.repeats import penalize_repeats_reference
    from adapcc_b200.ops.watermark import watermark_reference

    L = lens.cpu().tolist()
    seqs = [seq[r, :L[r]].cpu() for r in range(rows)]
    want = watermark_reference(penalize_repeats_reference(before, seqs, Vv, penalty, 0), seqs, Vv, wm)
    assert torch.equal(_bits(logits), _bits(want))


@pytest.mark.parametrize("mode", ["greedy", "sampled", "guided", "fp8"])
def test_generate_graph_equals_eager_loop(dev, mode):
    """``generate`` (graph replay) against an eager loop of the same kernels: the same tokens, and at every step of
    the loop the ops' output equals the reference bit for bit."""
    from adapcc_b200.ops import guidance_mix_, lm_head_logits_, penalize_repeats_, sample_tokens_, watermark_

    m = _gpt2_small(dev, seed=2)

    Vv = m.cfg.vocab_size                      # GPT-2's 50257 ids and the dialogue special tokens
    B, n = 6, 24
    lengths = [90, 17, 64, 9, 120, 1]
    ids = _prompts(dev, B, 120, 5)
    temp, scale = (0.0, 1.0) if mode == "greedy" else (1.0, 1.5 if mode == "guided" else 1.0)
    penalty = 1.2 if mode == "guided" else 1.0
    kv = "fp8_e4m3" if mode == "fp8" else None
    kw = dict(max_new_tokens=n, temperature=temp, top_p=0.95, seed=11, guidance_scale=scale, kv_cache_dtype=kv,
              repetition_penalty=penalty)
    free, _ = m.generate(ids, lengths, **kw)
    tokens, n_new = m.generate(ids, lengths, **kw, watermarking_config=WM)
    assert not torch.equal(tokens, free)
    w = m.wte.weight
    with torch.no_grad():
        if mode == "guided":
            ids_all, _, lengths_all, _ = m._guidance_rows(ids, None, lengths, torch.tensor(lengths, device=dev) - 1,
                                                          None, None, [1] * B, None)
        else:
            ids_all, lengths_all = ids, lengths
        R = len(lengths_all)
        cache = m.new_cache(R, max(lengths_all) + n, kv)
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
            penalize_repeats_(logits[:B], Vv, seq, prompt_len, cache.lens[:B], step, next_ids[:B], None, 1, penalty,
                              0)
            watermark_(logits[:B], Vv, seq, cache.lens[:B], WM)
            _check_op(logits[:B], before, Vv, seq, cache.lens[:B], B, WM, penalty)
            sample_tokens_(logits[:B], Vv, temp, 0, 0.95, seeds, cache.lens[:B], step, 0, empty, empty, done,
                           next_ids[:B], want)
            if mode == "guided":
                next_ids[B:].copy_(next_ids[:B])
    assert torch.equal(tokens, want), mode


@pytest.mark.parametrize("mode", ["greedy", "sampled", "groups", "stochastic"])
def test_beam_decoders_graph_equal_eager_loop(dev, mode):
    """``beam_search`` (greedy, sampled, groups) and ``stochastic_beam_search`` (graph replay) against an eager loop of
    the same kernels (``penalize_repeats_`` keeping each beam's sequence through the parent map, ``watermark_``,
    ``beam_step_``, ``kv_reorder_``): bit-identical results; at every step the ops' output equals the reference."""
    from adapcc_b200.ops import (BeamState, beam_step_, kv_reorder_, kv_reorder_scratch_numel, lm_head_logits_,
                                 penalize_repeats_, watermark_)
    from adapcc_b200.ops.beam import best_hypotheses, merge_finished_sets, stochastic_results

    m = _gpt2_small(dev, seed=1)

    Vv = m.cfg.vocab_size                      # GPT-2's 50257 ids and the dialogue special tokens
    B, K, n, alpha = 4, 8 if mode != "groups" else 16, 16, 0.8
    lengths = [64, 17, 120, 1]
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
    out = call(watermarking_config=WM_BEAM)
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
            penalize_repeats_(logits, Vv, seq, prompt_len, cache.lens, st.step, st.next_ids, st.parent, K, 1.0, 0)
            watermark_(logits, Vv, seq, cache.lens, WM_BEAM)
            _check_op(logits, before, Vv, seq, cache.lens, B * K, WM_BEAM)
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


def test_contrastive_search_graph_equals_eager_reference_loop(dev):
    """Contrastive search with a watermark against the eager loop of the same model calls, the reference rules on each
    row's sequence and ops/contrastive.py in fp64; a row may differ only after a near tie of its scores."""
    from adapcc_b200.models.gpt2 import CandidateKV
    from adapcc_b200.ops import ContrastiveState, lm_head_logits_
    from adapcc_b200.ops.contrastive import rerank_row, select_candidates
    from adapcc_b200.ops.watermark import watermark_reference

    m = _gpt2_small(dev)

    Vv = m.cfg.vocab_size                      # GPT-2's 50257 ids and the dialogue special tokens
    cfg = m.cfg
    Lr, H, D = cfg.n_layer, cfg.n_head, cfg.n_embd
    lengths = [200, 37, 128, 9, 64, 199, 150, 1]
    B, K, alpha, n = 8, 4, 0.6, 24
    wm = dict(bias=2.5)
    ids = _prompts(dev, B, 200, 4)
    free, _ = m.contrastive_search(ids, lengths, top_k=K, penalty_alpha=alpha, max_new_tokens=n)
    got, n_new = m.contrastive_search(ids, lengths, top_k=K, penalty_alpha=alpha, max_new_tokens=n,
                                      watermarking_config=wm)
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
            lc = watermark_reference(logits, seqs, Vv, wm)
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
    for b in range(B):
        if torch.equal(got[b].cpu(), tokens[b]):
            continue
        assert near[b], (b, got[b].tolist(), tokens[b].tolist())
        exempt += 1
    print(f"contrastive_search with a watermark, graph vs eager fp64 loop: {B} rows, {exempt} exempt")
    assert exempt <= 2 and not torch.equal(got, free)


def _scored(ids, lengths, tokens, n_new):
    """[B, T + n] prompts followed by their replies, the full lengths and the prompt lengths (where scoring starts)."""
    seqs = [ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist() for b, x in enumerate(lengths)]
    T = max(map(len, seqs))
    return (torch.tensor([s + [0] * (T - len(s)) for s in seqs], device=ids.device), [len(s) for s in seqs],
            list(lengths))


def test_large_bias_makes_every_scored_token_green(dev):
    from adapcc_b200.ops.watermark import detect_watermark

    m = _gpt2_small(dev, seed=4)

    lengths = [40, 3, 1, 25]
    ids = _prompts(dev, 4, 40, 1)
    for wm in (dict(bias=1e4), dict(bias=1e4, seeding_scheme="selfhash", context_width=4),
               dict(bias=1e4, context_width=3, greenlist_ratio=0.1)):
        tokens, n_new = m.generate(ids, lengths, max_new_tokens=32, temperature=0.0, watermarking_config=wm)
        x, L, P = _scored(ids, lengths, tokens, n_new)
        det = detect_watermark(x, wm, lengths=L, scored_from=P)
        assert (det.num_tokens_scored > 0).all() and np.array_equal(det.num_green_tokens, det.num_tokens_scored), wm


def test_detection_power_and_false_alarms(dev):
    """Sampled ``generate`` at δ = 4, γ = 0.25 is flagged (z > 3) in all 32 rows of 64 tokens; without the watermark,
    scored with ``ignore_repeated_ngrams``, at most the number of rows a binomial tail allows. Each bound holds with
    probability at least 1 - 1e-6 under its stated model."""
    from scipy.stats import binom

    from adapcc_b200.ops.watermark import check_watermark_args, detect_watermark

    wm = check_watermark_args("test", dict(bias=4.0, greenlist_ratio=0.25))
    g, B, n = wm.gamma_eff, 32, 64
    m = _gpt2_small(dev, seed=5)
    Vv = m.cfg.vocab_size                      # GPT-2's 50257 ids and the dialogue special tokens
    lengths = [16] * B
    ids = _prompts(dev, B, 16, 2)
    # The model: GPT-2 small with seeded random weights favours the ids already in its context (tied embeddings) and
    # is close to uniform over the others (checked below at the first step). With no_repeat_ngram_size=1 banning
    # those ids, a token's unbiased green mass is at least gamma / 2 and its green probability under the bias at least
    # p_min.
    with torch.no_grad():
        logits = m.lm_logits(m.hidden(ids, None)[:, -1], m.wte.weight.float())[:, :Vv]
        logits[torch.arange(B, device=dev)[:, None], ids] = -math.inf
        p = torch.softmax(logits, -1)
    assert float(p.max()) < 1e-3
    G = g / 2
    p_min = G * math.exp(4.0) / (G * math.exp(4.0) + 1 - G)
    need = math.floor(3 * math.sqrt(n * g * (1 - g)) + g * n) + 1          # the fewest greens with z > 3 at n = 64
    assert B * binom.cdf(need - 1, n, p_min) <= 1e-6
    tokens, n_new = m.generate(ids, lengths, max_new_tokens=n, temperature=1.0, top_p=1.0, seed=3,
                               no_repeat_ngram_size=1, watermarking_config=wm)
    x, L, P = _scored(ids, lengths, tokens, n_new)
    det = detect_watermark(x, wm, lengths=L, scored_from=P)
    assert (det.num_tokens_scored == n).all() and det.prediction.all(), det.z_score
    # Without it each distinct n-gram is green with probability gamma_eff independently; a row with k distinct n-grams
    # is flagged with probability q(k) = P(Binomial(k, gamma_eff) >= the fewest greens with z > 3), at most q.
    q = max(binom.sf(math.floor(3 * math.sqrt(k * g * (1 - g)) + g * k), k, g) for k in range(1, n + 1))
    allowed = next(a for a in range(B + 1) if binom.sf(a, B, q) <= 1e-6)
    free, k_new = m.generate(ids, lengths, max_new_tokens=n, temperature=1.0, top_p=1.0, seed=3,
                             no_repeat_ngram_size=1)
    x, L, P = _scored(ids, lengths, free, k_new)
    det = detect_watermark(x, wm, lengths=L, scored_from=P, ignore_repeated_ngrams=True)
    assert int(det.prediction.sum()) <= allowed, (det.z_score, allowed)
    print(f"detection: 32 / 32 watermarked rows flagged (min z {det.z_score.min():.2f} unmarked); "
          f"{int(det.prediction.sum())} unmarked rows flagged, {allowed} allowed")


def test_launches_per_replay(dev):
    """A watermark adds one launch per decode step (``watermark_``) when a repetition control already runs, two when
    none does (``penalize_repeats_`` keeps the sequences); the head runs once eagerly for the first token and once in
    the graph capture (replays are not host launches). With ``watermarking_config=None`` nothing changes."""
    from adapcc_b200.runtime.native import load_library

    lib = load_library(build_if_missing=False)
    m = _gpt2_small(dev, seed=6)
    ids = _prompts(dev, 4, 20, 3)

    def launches(n, **kw):
        c0 = lib.adapcc_launch_count()
        m.generate(ids, max_new_tokens=n, temperature=0.0, **kw)
        torch.cuda.synchronize()
        return lib.adapcc_launch_count() - c0

    base = launches(12)
    assert launches(12, watermarking_config=None) == base
    assert launches(12, watermarking_config=WM) - base == 2 * 2
    rep = launches(12, repetition_penalty=1.3)
    assert launches(12, repetition_penalty=1.3, watermarking_config=WM) - rep == 2 * 1
    for call in (lambda **kw: m.beam_search(ids, num_beams=4, max_new_tokens=8, **kw),
                 lambda **kw: m.contrastive_search(ids, max_new_tokens=8, **kw)):
        c0 = lib.adapcc_launch_count()
        call()
        c1 = lib.adapcc_launch_count()
        call(watermarking_config=WM)
        c2 = lib.adapcc_launch_count()
        assert (c2 - c1) - (c1 - c0) == 2 * 2
