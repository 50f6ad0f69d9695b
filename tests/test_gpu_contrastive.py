"""Contrastive search on the GPU: ``cand_attention_`` bit for bit against ``decode_attention_`` on k-fold copies,
``contrastive_select_`` and ``contrastive_rerank_`` against the fp64 definition (ops/contrastive.py) with derived
near-tie bounds, the context append and KV commit against torch indexing, graph replay against eager launches, a row
alone against the same row in a batch, and ``GPT2DoubleHeads.contrastive_search`` on GPT-2 small with random weights."""
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


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def test_cand_attention_bit_exact_against_decode_attention_on_copies(dev):
    from adapcc_b200.ops import cand_attention_, decode_attention_, decode_attention_work_numel

    H, Dh, t_max = 12, 64, 200
    D = H * Dh
    lens = torch.tensor([0, 63, 64, 65, t_max - 1], dtype=torch.int32, device=dev)
    B = lens.numel()
    g = torch.Generator(device=dev).manual_seed(0)
    kc = torch.randn(B, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16)
    vc = torch.randn(B, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16)
    k0, v0 = kc.clone(), vc.clone()
    for K in (1, 2, 4, 16):
        qkv = (torch.randn(B * K, 3 * D, device=dev, generator=g) * 2).to(torch.bfloat16)
        out = torch.empty(B * K, D, dtype=torch.bfloat16, device=dev)
        side_k, side_v = torch.empty_like(out), torch.empty_like(out)
        work = torch.empty(decode_attention_work_numel(B * K, H, Dh, t_max), dtype=torch.float32, device=dev)
        cand_attention_(qkv, kc, vc, lens, K, out, side_k, side_v, work)
        kx, vx = kc.repeat_interleave(K, 0).contiguous(), vc.repeat_interleave(K, 0).contiguous()
        want = torch.empty_like(out)
        decode_attention_(qkv, kx, vx, lens.repeat_interleave(K).contiguous(), want, work)
        torch.cuda.synchronize()
        assert torch.equal(_bits(out), _bits(want)), K
        assert torch.equal(_bits(kc), _bits(k0)) and torch.equal(_bits(vc), _bits(v0)), K     # the cache is read only
        assert torch.equal(_bits(side_k), _bits(qkv[:, D:2 * D])) and torch.equal(_bits(side_v), _bits(qkv[:, 2 * D:]))
        # a graph replay equals the eager launch
        again = torch.zeros_like(out)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cand_attention_(qkv, kc, vc, lens, K, again, side_k, side_v, work)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(_bits(again), _bits(out)), K
    with pytest.raises(ValueError, match="top_k"):
        cand_attention_(qkv, kc, vc, lens, 17, out, side_k, side_v, work)


def _p_tol(V):
    """fp32 error of p = expf(l - m) / Z against fp64 (relative): Z sums at most C = ceil(V / 512) terms per thread and
    5 + 5 shuffle levels, each term within 2 ulp (expf of a rounded argument); then one expf and one division."""
    return (math.ceil(V / 512) + 20) * U32


def test_select_against_fp64_with_planted_ties(dev):
    from adapcc_b200.ops import ContrastiveState, contrastive_select_
    from adapcc_b200.ops.contrastive import select_candidates

    B, V = 40, 50257
    rng = np.random.default_rng(1)
    logits = (rng.standard_normal((B, V + 7)) * 3).astype(np.float32)
    for b in range(0, B, 3):                                          # planted ties among the leaders
        top = np.argsort(-logits[b, :V])[:6]
        logits[b, top[3]] = logits[b, top[1]]
        logits[b, top[4]] = logits[b, top[1]]
    logits[5, :V] = -np.inf                                           # no candidate at all
    logits[6, :V] = -np.inf
    logits[6, [3, 9]] = [1.0, 1.0]                                    # fewer than k candidates
    sup = [int(np.argmax(logits[b, :V])) for b in (1, 2)] + [50256]
    done = np.zeros(B, dtype=np.int32)
    done[[7, 20]] = 1
    lt = torch.from_numpy(logits).to(dev)
    for K, step, min_new in ((4, 0, 1), (16, 2, 1), (1, 0, 0)):
        st = ContrastiveState(B, K, 8, 16, 1, 1, 8, dev)
        st.step.fill_(step)
        st.done.copy_(torch.from_numpy(done))
        contrastive_select_(lt, V, st, min_new, torch.tensor(sup, dtype=torch.int32, device=dev))
        ids, probs = select_candidates(logits, V, K, step, min_new, sup, done)
        torch.cuda.synchronize()
        assert torch.equal(st.cand_tok.cpu().view(B, K).long(), ids), K
        assert torch.equal(st.next_ids.cpu().view(B, K), ids.clamp(min=0)), K
        p = st.cand_p.cpu().view(B, K).double()
        assert torch.allclose(p, probs, rtol=_p_tol(V), atol=0), (K, float((p - probs).abs().max()))
        # a row alone equals the same row in the batch, bit for bit
        one = ContrastiveState(1, K, 8, 16, 1, 1, 8, dev)
        one.step.fill_(step)
        contrastive_select_(lt[1:2].contiguous(), V, one, min_new, torch.tensor(sup, dtype=torch.int32, device=dev))
        assert torch.equal(one.cand_tok, st.cand_tok.view(B, K)[1]) and torch.equal(
            _bits(one.cand_p), _bits(st.cand_p.view(B, K)[1]))


def _s_tol(D):
    """fp32 error of a cosine against fp64: the dot product of D terms by fma chains and a shuffle tree is within
    D u |h| |c| (Cauchy-Schwarz), each norm within (D / 2 + 1) u relative, the product and the division one rounding
    each: |cos32 - cos64| <= (2 D + 4) u."""
    return (2 * D + 4) * U32


def _rerank_case(dev, B, K, D, t_max, seed):
    """A state with a random context (some zero vectors, a candidate equal to a context vector), candidates and
    probabilities, and caches; returns what the fp64 reference needs."""
    from adapcc_b200.ops import ContrastiveState

    n_layer, H = 2, D // 64
    rng = np.random.default_rng(seed)
    g = torch.Generator(device=dev).manual_seed(seed)
    st = ContrastiveState(B, K, 6, t_max, n_layer, H, 64, dev)
    lens = torch.from_numpy(rng.integers(1, t_max, B).astype(np.int32))
    lens[0], lens[-1] = 1, t_max - 1
    st.ctx.copy_(torch.randn(B, t_max, D, device=dev, generator=g).to(torch.bfloat16))
    st.ctx[1, 0].zero_()                                              # zero-norm context vector
    hc = torch.randn(B * K, D, device=dev, generator=g).to(torch.bfloat16)
    hc[2 * K + 1] = st.ctx[2, 0]                                      # cosine 1 with the context
    hc[3 * K].zero_()                                                 # zero-norm candidate
    st.ctx_norm.copy_(st.ctx.double().norm(dim=-1).float())
    tok = torch.from_numpy(rng.integers(0, 50000, B * K).astype(np.int32))
    tok.view(B, K)[4, K // 2:] = -1                                   # invalid slots
    tok.view(B, K)[5] = -1                                            # no candidate
    p = torch.from_numpy(np.sort(rng.random((B, K)), axis=1)[:, ::-1].astype(np.float32).copy())
    p.view(B, K)[6, :] = p.view(B, K)[6, 0]                           # tied probabilities
    st.cand_tok.copy_(tok)
    st.cand_p.copy_(p.reshape(-1))
    st.side.copy_(torch.randn(st.side.shape, device=dev, generator=g).to(torch.bfloat16))
    kc = torch.randn(n_layer, B, H, t_max, 64, device=dev, generator=g).to(torch.bfloat16)
    vc = torch.randn_like(kc.float()).to(torch.bfloat16)
    return st, hc, lens.to(dev), kc, vc


def _clone_state(st):
    import copy

    c = copy.copy(st)
    for name in ("step", "done", "next_ids", "cand_tok", "cand_p", "tokens", "win_ids", "win_h", "ctx", "ctx_norm",
                 "side", "sim", "work"):
        setattr(c, name, getattr(st, name).clone())
    return c


@pytest.mark.parametrize("alpha", [0.0, 0.6, 1.0])
def test_rerank_and_commit(dev, alpha):
    from adapcc_b200.ops import contrastive_rerank_
    from adapcc_b200.ops.contrastive import rerank_row

    B, K, D, t_max = 12, 8, 768, 300
    st, hc, lens, kc, vc = _rerank_case(dev, B, K, D, t_max, seed=int(alpha * 10))
    st.done[7] = 1
    stop_id = int(st.cand_tok[8 * K])
    stop = torch.tensor([stop_id], dtype=torch.int32, device=dev)
    s0, lens0, k0, v0 = _clone_state(st), lens.clone(), kc.clone(), vc.clone()
    contrastive_rerank_(hc, st, alpha, kc, vc, lens, stop)
    torch.cuda.synchronize()
    tok, p = s0.cand_tok.cpu().view(B, K).numpy(), s0.cand_p.cpu().view(B, K).numpy()
    hk = hc.view(B, K, D).double().cpu().numpy()
    tol = 2 * (alpha * _s_tol(D) + 4 * U32)
    exempt = 0
    for b in range(B):
        n = int(lens0[b])
        ref = rerank_row(tok[b], p[b], hk[b], s0.ctx[b, :n].double().cpu().numpy(), alpha)
        w = int(st.win_ids[b])
        rank = ref["rank"]
        if w != ref["token"]:
            sc = np.sort(ref["scores"][np.isfinite(ref["scores"])])[::-1]
            assert sc.size > 1 and sc[0] - sc[1] <= tol, (b, w, ref)
            exempt += 1
            rank = int(np.flatnonzero(tok[b] == w)[0])
        r = b * K + rank
        # the sims the kernel found, against fp64
        sims = st.sim.view(B, -1, K)[b].max(0).values.double().cpu().numpy()
        valid = tok[b] >= 0
        assert np.allclose(np.maximum(sims[valid], -1), ref["sims"][valid], atol=_s_tol(D), rtol=0), b
        # the append, the KV commit and the lengths, against torch indexing
        assert torch.equal(_bits(st.ctx[b, n]), _bits(hc[r])) and torch.equal(_bits(st.win_h[b]), _bits(hc[r])), b
        assert float(st.ctx_norm[b, n]) == pytest.approx(float(hc[r].double().norm()), rel=(D / 2 + 2) * U32, abs=0)
        assert torch.equal(_bits(st.ctx[b, :n]), _bits(s0.ctx[b, :n])) and torch.equal(
            _bits(st.ctx[b, n + 1:]), _bits(s0.ctx[b, n + 1:])), b
        want_k, want_v = k0[:, b].clone(), v0[:, b].clone()
        want_k[:, :, n] = s0.side[:, 0, r].view(-1, D // 64, 64)
        want_v[:, :, n] = s0.side[:, 1, r].view(-1, D // 64, 64)
        assert torch.equal(_bits(kc[:, b]), _bits(want_k)) and torch.equal(_bits(vc[:, b]), _bits(want_v)), b
        assert int(lens[b]) == n + 1
        emitted = int(st.tokens[b, 0])
        if b == 7:
            assert emitted == -1 and w == ref["token"]                 # a row already done emits nothing
        elif w == stop_id:
            assert emitted == -1 and int(st.done[b]) == 1
        else:
            assert emitted == w and int(st.done[b]) == 0
    assert int(st.win_ids[5]) == 0                                    # no candidate: id 0
    assert int(st.step) == 1
    print(f"contrastive_rerank_ vs fp64 (alpha {alpha}): {B} rows, {exempt} exempt")
    assert exempt <= 1

    # a graph replay equals the eager launch, and a row alone equals the same row in the batch, bit for bit
    st2, lens2, k2, v2 = _clone_state(s0), lens0.clone(), k0.clone(), v0.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        contrastive_rerank_(hc, st2, alpha, k2, v2, lens2, stop)
    graph.replay()
    torch.cuda.synchronize()
    for name in ("tokens", "done", "win_ids", "win_h", "ctx", "ctx_norm", "sim", "step"):
        assert torch.equal(_bits(getattr(st2, name)) if getattr(st2, name).dtype in (torch.bfloat16, torch.float32)
                           else getattr(st2, name), _bits(getattr(st, name)) if getattr(st, name).dtype in (
                               torch.bfloat16, torch.float32) else getattr(st, name)), name
    assert torch.equal(_bits(k2), _bits(kc)) and torch.equal(lens2, lens)
    from adapcc_b200.ops import ContrastiveState
    b = 2
    one = ContrastiveState(1, K, 6, t_max, 2, D // 64, 64, dev)
    one.ctx.copy_(s0.ctx[b:b + 1])
    one.ctx_norm.copy_(s0.ctx_norm[b:b + 1])
    one.cand_tok.copy_(s0.cand_tok.view(B, K)[b])
    one.cand_p.copy_(s0.cand_p.view(B, K)[b])
    one.side.copy_(s0.side[:, :, b * K:(b + 1) * K])
    k1, v1, l1 = k0[:, b:b + 1].contiguous(), v0[:, b:b + 1].contiguous(), lens0[b:b + 1].clone()
    contrastive_rerank_(hc[b * K:(b + 1) * K].contiguous(), one, alpha, k1, v1, l1, stop)
    torch.cuda.synchronize()
    assert int(one.win_ids[0]) == int(st.win_ids[b]) and int(one.tokens[0, 0]) == int(st.tokens[b, 0])
    assert torch.equal(_bits(one.ctx[0]), _bits(st.ctx[b])) and torch.equal(_bits(one.ctx_norm[0]),
                                                                             _bits(st.ctx_norm[b]))
    assert torch.equal(_bits(one.sim.view(-1, K)), _bits(st.sim.view(B, -1, K)[b]))
    assert torch.equal(_bits(k1[:, 0]), _bits(kc[:, b]))


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


@torch.no_grad()
def _eager_reference(m, ids, lengths, K, alpha, n, stop=()):
    """The native path's model calls run eagerly (the same kernels, so the same hidden states and logits), with the
    selection and re-ranking done by ops/contrastive.py in fp64 and the commit by torch indexing. Returns the tokens
    and, per row, whether some step had two candidate scores within the derived fp32 bound of each other."""
    from adapcc_b200.models.gpt2 import CandidateKV
    from adapcc_b200.ops import ContrastiveState, lm_head_logits_
    from adapcc_b200.ops.contrastive import rerank_row, select_candidates

    dev = ids.device
    B, T = ids.shape
    cfg = m.cfg
    V, L, H, D = cfg.vocab_size, cfg.n_layer, cfg.n_head, cfg.n_embd
    t_max = max(lengths) + n
    cache = m.new_cache(B, t_max)
    hs = m.hidden(ids, None, cache=cache, lengths=lengths)
    ctx = [hs[b, :x].double().cpu().numpy() for b, x in enumerate(lengths)]
    h = hs[torch.arange(B, device=dev), torch.tensor(lengths, device=dev) - 1].contiguous()
    st = ContrastiveState(B, K, n, t_max, L, H, D // H, dev)
    cand = CandidateKV(cache, K, st.side, st.work)
    logits = torch.empty(B, m.wte.weight.shape[0], dtype=torch.float32, device=dev)
    tokens = torch.full((B, n), -1, dtype=torch.int64)
    done = np.zeros(B, dtype=bool)
    near = np.zeros(B, dtype=bool)
    tol = 2 * (alpha * _s_tol(D) + (1 - alpha) * _p_tol(V) + 4 * U32)
    rows = torch.arange(B, device=dev)
    for i in range(n):
        lm_head_logits_(h, m.wte.weight, logits)
        cid, probs = select_candidates(logits, V, K, i, 0, (), done)
        hc = m._candidate_hidden(cid.clamp(min=0).reshape(-1).to(dev), None, cand)
        hk = hc.view(B, K, D).double().cpu().numpy()
        pick = []
        for b in range(B):
            r = rerank_row(cid[b].numpy(), probs[b].numpy(), hk[b], ctx[b], alpha)
            sc = np.sort(r["scores"][np.isfinite(r["scores"])])[::-1]
            near[b] |= (not done[b]) and sc.size > 1 and sc[0] - sc[1] <= tol
            pick.append(b * K + r["rank"])
            if not done[b]:
                if r["token"] in stop:
                    done[b] = True
                else:
                    tokens[b, i] = r["token"]
            ctx[b] = np.concatenate([ctx[b], hk[b, r["rank"]][None]])
        pick = torch.tensor(pick, device=dev)
        pos = cache.lens.long()
        cache.k[:, rows, :, pos] = st.side[:, 0, pick].view(L, B, H, D // H).transpose(0, 1)
        cache.v[:, rows, :, pos] = st.side[:, 1, pick].view(L, B, H, D // H).transpose(0, 1)
        cache.advance()
        h = hc[pick].contiguous()
    return tokens, near


def test_contrastive_search_gpt2_small(dev):
    from adapcc_b200.ops import LM_HEAD_MAX_ROWS

    m = _gpt2_small(dev)
    V = m.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(4)
    lengths = [200, 37, 128, 1, 64, 199, 150, 90]
    ids = torch.randint(0, V, (8, 200), device=dev, generator=g)
    n = 32
    # alpha = 0 is greedy decoding; the candidates' hidden states come from GEMMs at B·k rows rather than B, so a
    # near tie between the two best logits may go the other way after the rows' states drift apart in their last bits
    want, _ = m.generate(ids, lengths, max_new_tokens=n, temperature=0.0)
    got, n_new = m.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.0, max_new_tokens=n)
    differ = sum(not torch.equal(got[b], want[b]) for b in range(8))
    print(f"contrastive_search(alpha=0) vs greedy generate: {differ} of 8 rows differ (near-tied logits)")
    assert differ <= 2 and n_new.tolist() == [n] * 8
    # alpha = 0.6 against the eager fp64 loop on the same model calls
    for K in (4, 8):
        got, _ = m.contrastive_search(ids, lengths, top_k=K, penalty_alpha=0.6, max_new_tokens=n)
        again, _ = m.contrastive_search(ids, lengths, top_k=K, penalty_alpha=0.6, max_new_tokens=n)
        assert torch.equal(got, again)
        ref, near = _eager_reference(m, ids, lengths, K, 0.6, n)
        exempt = 0
        for b in range(8):
            if torch.equal(got[b].cpu(), ref[b]):
                continue
            assert near[b], (K, b, got[b].tolist(), ref[b].tolist())
            exempt += 1
        print(f"contrastive_search(alpha=0.6, k={K}) graph vs eager fp64 loop: 8 rows, {exempt} exempt")
        assert exempt <= 2
    # a row alone: same tokens as in the batch up to near ties (GEMMs at other row counts round differently)
    got, _ = m.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.6, max_new_tokens=n)
    differ = 0
    for b in (0, 3, 6):
        t1, _ = m.contrastive_search(ids[b:b + 1, :lengths[b]], top_k=4, penalty_alpha=0.6, max_new_tokens=n)
        differ += not torch.equal(t1[0], got[b])
    print(f"contrastive_search rows alone vs in a ragged batch of 8: {differ} of 3 with other tokens")
    assert differ <= 1
    # stop ids and the repetition controls on the graph path
    stop = [int(got[0, 5])]
    t, k = m.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.6, max_new_tokens=n, stop_ids=stop,
                                no_repeat_ngram_size=2)
    for b in range(8):
        row = t[b, :int(k[b])].tolist()
        assert (t[b, int(k[b]):] == -1).all() and stop[0] not in row
        seq = ids[b, :lengths[b]].tolist() + row
        grams = [tuple(seq[j:j + 2]) for j in range(len(seq) - 1)]
        assert len(grams) == len(set(grams)), b
    with pytest.raises(ValueError, match="rows"):
        m.contrastive_search(torch.zeros(LM_HEAD_MAX_ROWS + 1, 4, dtype=torch.long, device=dev))
