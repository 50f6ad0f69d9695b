"""Rejection-sampling verification of assisted generation on the GPU (``assistant_verification="rejection"``): the
draft weights of ``sample_slots_(..., weights=True)`` and ``spec_slots_``'s decisions against the fp64 definition
(ops/assisted.py) with exemptions derived from the fp32 error, ``generate`` on GPT-2 small exactly against an eager
loop of the same kernels, and the distribution of the tiny model's tokens against plain sampling."""
import math

import numpy as np
import pytest
import torch

from test_gpu_assisted import MODES, _slot_state, models  # noqa: F401  (models: GPT-2 small and its three drafts)
from test_gpu_lookup import _prompts
from test_gpu_sample_filters import U32, _near

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _split(mode):
    kw = dict(mode)
    return kw.pop("temperature"), kw.pop("top_k"), kw.pop("top_p"), kw


# ---- fp32 error bounds -----------------------------------------------------------------------------------------------
def _cut_near(r, V):
    """The kept set of row ``r`` may differ from the kernel's: a top-p or filter decision sits at its threshold within
    the fp32 error (``_near`` of the sampler tests, without its draw)."""
    return "e" in r and _near(dict(r, cum=np.array([np.inf]), kept=np.array([True]), target=0.0), V)


def _weight_err(r, V):
    """Per-id bounds on the kernel's weight ``expf(x - m)`` and on its total Z' (``_near``'s argument: the weight is
    within (4 + |y|) u, a sum over the kept ids has at most C + 74 roundings on any path)."""
    e, kept = r["e"], r["kept"]
    ya = np.where(e > 0, -np.log(np.maximum(e, 1e-300)), 0.0)
    we = (4 + ya) * U32 * e
    return we, (math.ceil(V / 1024) + 74) * U32 * r["Zp"] + 2 * float(we[kept].sum())


def _prob_err(r, V):
    """Per-id bound on the kernel's probability ``weight / Z'`` (one more rounding for the division)."""
    if "e" not in r:
        return np.zeros(V)
    from adapcc_b200.ops.assisted import filtered_probs

    we, ez = _weight_err(r, V)
    P = filtered_probs(r)
    return np.where(r["kept"], we / r["Zp"] + P * (ez / r["Zp"] + 2 * U32), 0.0)


def _accept_near(r, d, V):
    eP, eQ = _prob_err(r["rp"], V), _prob_err(r["rq"], V)
    vq = r["v"] * r["Q"][d]
    return abs(vq - r["P"][d]) <= 2 * (r["v"] * eQ[d] + eP[d]) + 2 * U32 * vq


def _residual_near(r, V):
    """The residual draw may differ where a prefix of rho lies within its error of u' sum(rho)."""
    err = _prob_err(r["rp"], V) + _prob_err(r["rq"], V)
    bound = 2 * ((math.ceil(V / 1024) + 74) * U32 * float(r["cum"][-1]) + float(err.sum()))
    live = (r["rho"] > 0) | (err > 0)
    return bool((np.abs(r["cum"][live] - r["target"]) <= bound).any()) or float(r["cum"][-1]) <= bound


def _decisions(P, Q, d, T, tk, tp, seed, L, e, j, min_new, sup, kw, acc, last, V):
    """The fp64 decision of one slot against the kernel's ``acc`` / ``last``: 0 equal, 1 exempt (asserts the bound)."""
    from adapcc_b200.ops.assisted import spec_slot

    r = spec_slot(P, Q, d, T, tk, tp, seed, L, e, j, min_new, sup, **kw)
    ok_a, ok_t = bool(acc) == r["accept"], int(last) == r["t"]
    if ok_a and ok_t:
        return 0
    cut = _cut_near(r["rp"], V) or _cut_near(r["rq"], V)
    assert cut or ok_a or _accept_near(r, d, V), ("accept", j, r["accept"], r["v"], r["P"][d], r["Q"][d])
    assert cut or ok_t or _residual_near(r, V), ("residual", j, int(last), r["t"], float(r["cum"][-1]))
    return 1


# ---- the kernels against the definition ------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", range(len(MODES)))
def test_draft_weights_against_fp64_and_tokens_unchanged(dev, mode):
    from adapcc_b200.ops import AssistState, sample_slots_, sample_tokens_
    from adapcc_b200.ops.sampling import reference_row

    T, tk, tp, kw = _split(MODES[mode])
    B, k, V, ld, n = 12, 4, 50262, 50304, 30
    st, lens = _slot_state(dev, B, k, n, 10 + mode)
    wst = AssistState(B, k, n, 300, dev, V)
    for name in ("emitted", "nq", "done"):
        getattr(wst, name).copy_(getattr(st, name))
    g = torch.Generator(device=dev).manual_seed(20 + mode)
    logits = torch.randn(B, ld, device=dev, generator=g) * 3
    seeds = torch.arange(B, dtype=torch.int64, device=dev) * 13 + 5
    sup = torch.tensor([int(i) for i in logits[:, :V].argmax(1)[:3]], dtype=torch.int32, device=dev)
    if T == 0:
        with pytest.raises(ValueError, match="weights"):
            sample_slots_(logits, V, T, tk, tp, seeds, wst, lens, 0, 3, sup, draft=True, weights=True, **kw)
        return
    rows = exempt = 0
    nq, em, done = st.nq.cpu(), st.emitted.cpu(), st.done.cpu()
    for j in range(k):
        sample_slots_(logits, V, T, tk, tp, seeds, st, lens, j, 3, sup, draft=True, **kw)
        sample_slots_(logits, V, T, tk, tp, seeds, wst, lens, j, 3, sup, draft=True, weights=True, **kw)
        assert torch.equal(st.ids, wst.ids) and torch.equal(st.d_in, wst.d_in), (mode, j)   # the same bits
        q, zq = wst.q[:, j].cpu().double().numpy(), wst.zq[:, j].cpu().double().numpy()
        ids = st.ids.view(B, k + 1)[:, j + 1].cpu()
        lc = logits[:, :V].cpu().numpy()
        for b in range(B):
            if done[b] or j + 1 >= nq[b]:
                continue
            step = torch.tensor([int(em[b]) + j], dtype=torch.int32, device=dev)
            pos = (lens[b:b + 1] + j + 1).contiguous()
            nxt = torch.zeros(1, dtype=torch.int64, device=dev)
            sample_tokens_(logits[b:b + 1], V, T, tk, tp, seeds[b:b + 1], pos, step, 3, sup, None,
                           torch.zeros(1, dtype=torch.int32, device=dev), nxt,
                           torch.zeros(1, 1, dtype=torch.int64, device=dev), **kw)
            assert int(nxt) == int(ids[b])
            r = reference_row(lc[b], T, tk, tp, int(seeds[b]), int(lens[b]) + j + 1, int(em[b]) + j, 3,
                              sup.tolist(), **kw)
            rows += 1
            if _cut_near(r, V) and not np.array_equal(q[b] > 0, r["kept"] & (r["e"] > 0)):
                exempt += 1
                continue
            we, ez = _weight_err(r, V)
            assert (q[b][~r["kept"]] == 0).all(), (mode, j, b)                  # exactly 0 off the survivors
            assert (np.abs(q[b] - np.where(r["kept"], r["e"], 0.0)) <= 2 * we + 1e-45).all(), (mode, j, b)
            assert abs(zq[b] - r["Zp"]) <= 2 * ez, (mode, j, b, zq[b], r["Zp"])
    print(f"mode {mode}: {rows} draft weight rows against fp64, {exempt} exempt near a cut")
    assert rows >= 10 and exempt <= rows // 10


@pytest.mark.parametrize("mode", range(len(MODES)))
def test_spec_slots_against_the_definition(dev, mode):
    from adapcc_b200.ops import AssistState, sample_slots_, spec_slots_

    T, tk, tp, kw = _split(MODES[mode])
    B, k, V, ld, n = 48, 4, 50262, 50304, 30
    S = k + 1
    decisions = exempt = 0
    for rep, noise in enumerate((0.0, 0.02, 0.2, 1.0, 4.0)):
        base, lens = _slot_state(dev, B, k, n, 40 + rep)
        st = AssistState(B, k, n, 300, dev, V)
        for name in ("emitted", "nq", "done"):
            getattr(st, name).copy_(getattr(base, name))
        g = torch.Generator(device=dev).manual_seed(100 * mode + rep)
        P = torch.randn(B * S, ld, device=dev, generator=g) * 3
        Q = P.view(B, S, ld)[:, :k] + noise * torch.randn(B, k, ld, device=dev, generator=g)
        seeds = torch.arange(B, dtype=torch.int64, device=dev) * 7 + rep
        sup = torch.tensor([int(i) for i in P[:4, :V].argmax(1)], dtype=torch.int32, device=dev)
        if T == 0:
            with pytest.raises(ValueError, match="temperature > 0"):
                spec_slots_(P, V, T, tk, tp, seeds, st, lens, 2, sup, **kw)
            return
        for j in range(k):
            sample_slots_(Q[:, j].contiguous(), V, T, tk, tp, seeds, st, lens, j, 2, sup, draft=True, weights=True,
                          **kw)
        st.g.fill_(-3)
        spec_slots_(P, V, T, tk, tp, seeds, st, lens, 2, sup, **kw)
        g_spec = st.g.clone()
        st.g.fill_(-3)
        sample_slots_(P, V, T, tk, tp, seeds, st, lens, 0, 2, sup, **kw)
        assert torch.equal(g_spec, st.g), (mode, noise)                        # g: the same bits as sample_slots_
        acc, last = st.acc.view(B, S).cpu(), st.last.view(B, S).cpu()
        ids, g_all = st.ids.view(B, S).cpu(), st.g.view(B, S).cpu()
        nq, em, done = st.nq.cpu(), st.emitted.cpu(), st.done.cpu()
        Pc, Qc = P[:, :V].cpu().numpy().reshape(B, S, V), Q[:, :, :V].cpu().numpy()
        for b in range(B):
            if done[b]:
                continue
            m = int(nq[b])
            assert int(last[b, m - 1]) == int(g_all[b, m - 1])                # the last real slot: g
            for j in range(m - 1):
                decisions += 1
                exempt += _decisions(Pc[b, j], Qc[b, j], int(ids[b, j + 1]), T, tk, tp, int(seeds[b]), int(lens[b]),
                                     int(em[b]), j, 2, sup.tolist(), kw, acc[b, j], last[b, j], V)
    print(f"mode {mode}: {decisions} decisions against fp64, {exempt} exempt")
    assert decisions >= 300 and exempt <= decisions // 100


# ---- GPT-2 small, random weights -------------------------------------------------------------------------------------
@torch.no_grad()
def _eager_rejection(model, draft, ids, lengths, k, n, mode, seeds, min_new=0, suppress=(), stop=(), check=False):
    """Rejection-sampling assisted generation run eagerly with the same kernels as ``generate``'s graph (the draft's
    decode steps with ``sample_slots_(..., weights=True)``, the verify step, ``spec_slots_``), launched one by one,
    with the round set-up, the counters and the acceptance kept on the host (``assist_round``, ``lookup_accept``).
    With ``check``, every decision is also compared with the fp64 definition on the same logits. Returns ``(tokens,
    emitted, steps, decisions, exempt)``."""
    from adapcc_b200.models.gpt2 import KVCache, VerifyKV
    from adapcc_b200.ops import (AssistState, decode_attention_work_numel, lm_head_logits_, sample_slots_,
                                 sample_tokens_, spec_slots_)
    from adapcc_b200.ops.assisted import assist_round
    from adapcc_b200.ops.lookup import lookup_accept

    T, tk, tp, kw = _split(mode)
    dev, W, dW, V = ids.device, model.wte.weight, draft.wte.weight, model.cfg.vocab_size
    B, Tp = ids.shape
    S, t_max, dc = k + 1, max(lengths) + n, draft.cfg
    sup = torch.tensor(list(suppress), dtype=torch.int32, device=dev)
    last_pos = torch.tensor(lengths, device=dev) - 1
    cache = model.new_cache(B, t_max)
    h = model.hidden(ids, None, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last_pos]
    dcache = KVCache(dc.n_layer, B, dc.n_head, t_max + k, dc.n_embd // dc.n_head, dW.dtype, dev)
    draft.hidden(ids, None, cache=dcache, lengths=lengths)
    work = torch.empty(decode_attention_work_numel(B * S, model.cfg.n_head, model.cfg.n_embd // model.cfg.n_head,
                                                   t_max), dtype=torch.float32, device=dev)
    logits = torch.empty(B * S, W.shape[0], dtype=torch.float32, device=dev)
    dlogits = torch.empty(B, dW.shape[0], dtype=torch.float32, device=dev)
    st = AssistState(B, k, n, t_max, dev, V)                         # the kernels' buffers only
    seq = torch.zeros(B, t_max, dtype=torch.int32)
    seq[:, :Tp] = ids.cpu()
    lens = torch.tensor(lengths, dtype=torch.int32) - 1
    emitted, done, steps = (torch.zeros(B, dtype=torch.int32) for _ in range(3))
    tokens = torch.full((B, n), -1, dtype=torch.int64)
    lm_head_logits_(h, W, logits[:B])
    zero = torch.zeros(1, dtype=torch.int32, device=dev)
    nxt, tok = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, 1, dtype=torch.int64, device=dev)
    g0 = []
    for b in range(B):
        sample_tokens_(logits[b:b + 1], V, T, tk, tp, seeds[b:b + 1], lens[b:b + 1].to(dev) + 1,
                       torch.zeros(1, dtype=torch.int32, device=dev), min_new, sup, None, zero, nxt, tok, **kw)
        g0.append([int(nxt)])
    lookup_accept(None, V, torch.zeros(B * S, dtype=torch.int64), torch.ones(B, dtype=torch.int32), seq, lens,
                  emitted, done, tokens, None, stop_ids=stop, drawn=torch.tensor(g0))
    decisions = exempt = 0
    while not bool(done.all()):
        slots, pos, nq, d_in, d_pos = assist_round(seq, lens, emitted, done, k, n, dc.n_positions)
        for name, v in (("nq", nq), ("emitted", emitted), ("done", done), ("ids", slots), ("d_in", d_in)):
            getattr(st, name).copy_(v)
        L = lens.to(dev)
        dcache.lens.copy_(lens)
        qrows = []
        for j in range(S):
            hd = draft._blocks(draft._embed(st.d_in.clone(), None, d_pos[j].to(dev)), dcache)
            dcache.lens.add_(1)
            if j < k:
                lm_head_logits_(hd, dW, dlogits)
                qrows.append(dlogits[:, :V].cpu().numpy() if check else None)
                sample_slots_(dlogits, V, T, tk, tp, seeds, st, L, j, min_new, sup, draft=True, weights=True, **kw)
        slots = st.ids.cpu()
        cache.lens.copy_(lens)
        hv = model._verify_hidden(st.ids, pos.to(dev), None, VerifyKV(cache, S, nq.to(dev), work))
        lm_head_logits_(hv, W, logits)
        spec_slots_(logits, V, T, tk, tp, seeds, st, L, min_new, sup, **kw)
        acc, last = st.acc.view(B, S).cpu(), st.last.view(B, S).cpu()
        if check:
            Pc = logits[:, :V].cpu().numpy().reshape(B, S, V)
            for b in range(B):
                for j in range(0 if done[b] else int(nq[b]) - 1):
                    decisions += 1
                    exempt += _decisions(Pc[b, j], qrows[j][b], int(slots[b * S + j + 1]), T, tk, tp, int(seeds[b]),
                                         int(lens[b]), int(emitted[b]), j, min_new, list(suppress), kw, acc[b, j],
                                         last[b, j], V)
        lookup_accept(None, V, slots, nq, seq, lens, emitted, done, tokens, steps, stop_ids=stop, drawn=last,
                      accepted=acc)
    return tokens, emitted, steps, decisions, exempt


@pytest.mark.parametrize("mode", [1, 2, 3])
def test_gpt2_small_rejection_generate_exact_against_eager_kernels(models, dev, mode):
    gpt2 = models["self"]
    V, n, k = gpt2.cfg.vocab_size, 24, 4
    ids, lengths = _prompts(V, dev)
    seeds = torch.arange(8, dtype=torch.int64, device=dev) * 29 + 3
    plain, _ = gpt2.generate(ids, lengths, max_new_tokens=n, seed=seeds, **MODES[mode])
    stop, suppress = [int(plain[0, 7]), int(plain[5, 3])], [int(plain[5, 3]), int(plain[2, 0])]
    gk = dict(MODES[mode], max_new_tokens=n, seed=seeds, stop_ids=stop, suppress_ids=suppress, min_new_tokens=5)
    total = ex = 0
    for name, draft in models.items():
        got, n_got = gpt2.generate(ids, lengths, assistant_model=draft, num_assistant_tokens=k,
                                   assistant_verification="rejection", **gk)
        stats = {key: v.cpu() for key, v in gpt2.assist_stats.items() if key != "replays"}
        want, emitted, steps, dec, exm = _eager_rejection(gpt2, draft, ids, lengths, k, n, MODES[mode], seeds, 5,
                                                          suppress, stop, check=True)
        assert torch.equal(got.cpu(), want), (mode, name)
        assert torch.equal(stats["emitted"], emitted) and torch.equal(stats["steps"], steps), (mode, name)
        assert torch.equal(n_got.cpu(), (want >= 0).sum(1))
        total, ex = total + dec, ex + exm
        print(f"mode {mode}, draft {name}: equal to the eager kernels, "
              f"{float((emitted - 1).sum()) / float(steps.sum()):.2f} tokens per verify step, {dec} decisions, "
              f"{exm} exempt against fp64")
    assert ex <= max(1, total // 100)


def test_gpt2_small_rejection_at_temperature_zero_is_coupled(models, dev):
    gpt2 = models["self"]
    ids, lengths = _prompts(gpt2.cfg.vocab_size, dev)
    for name in ("cut", "other"):
        kw = dict(max_new_tokens=24, temperature=0.0, assistant_model=models[name], num_assistant_tokens=3)
        want, _ = gpt2.generate(ids, lengths, **kw)
        st = {key: v.clone() if torch.is_tensor(v) else v for key, v in gpt2.assist_stats.items()}
        got, _ = gpt2.generate(ids, lengths, assistant_verification="rejection", **kw)
        assert torch.equal(got, want), name
        for key, v in st.items():
            assert torch.equal(gpt2.assist_stats[key], v) if torch.is_tensor(v) else gpt2.assist_stats[key] == v


def test_gpt2_small_rejection_row_reaching_n_positions_runs_clean(models, dev):
    gpt2 = models["self"]
    n, k = 12, 7
    N = gpt2.cfg.n_positions
    ids = torch.randint(0, 50000, (2, N - n), generator=torch.Generator().manual_seed(9)).to(dev)
    lengths = [N - n, 100]
    seeds = torch.tensor([3, 4], dtype=torch.int64, device=dev)
    for name in ("self", "other"):
        got, n_got = gpt2.generate(ids, lengths, assistant_model=models[name], num_assistant_tokens=k,
                                   max_new_tokens=n, seed=seeds, assistant_verification="rejection", **MODES[1])
        torch.cuda.synchronize()
        want, _, _, _, _ = _eager_rejection(gpt2, models[name], ids, lengths, k, n, MODES[1], seeds)
        assert torch.equal(got.cpu(), want) and int(n_got[0]) == n, name


def test_gpt2_small_self_draft_accepts_more_under_rejection(models, dev):
    gpt2 = models["self"]
    ids, lengths = _prompts(gpt2.cfg.vocab_size, dev)
    rates = {}
    for rule in ("coupled", "rejection"):
        gpt2.generate(ids, lengths, max_new_tokens=40, seed=5, assistant_model=gpt2, num_assistant_tokens=4,
                      assistant_verification=rule, **MODES[1])
        st = gpt2.assist_stats
        rates[rule] = float((st["emitted"] - 1).sum()) / float(st["steps"].sum())
    print(f"self draft, k = 4, B = 8, tokens per verify step: {rates}")
    assert rates["rejection"] > rates["coupled"]


def test_tiny_bf16_tokens_are_distributed_as_plain_sampling(dev):
    from scipy.stats import chi2_contingency

    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(0)
    tiny = GPT2DoubleHeads(GPT2Config.tiny()).eval()
    noisy = GPT2DoubleHeads(GPT2Config.tiny()).eval()
    g = torch.Generator().manual_seed(9)
    noisy.load_state_dict({key: v + 0.3 * v.std() * torch.randn(v.shape, generator=g)
                           if v.is_floating_point() and v.numel() > 1 else v for key, v in tiny.state_dict().items()})
    tiny, noisy = (m.to(device=dev, dtype=torch.bfloat16) for m in (tiny, noisy))
    B, N = 20, 4000
    prompt = torch.tensor([[5, 17, 3, 9]], device=dev).repeat(B, 1)
    kw = dict(max_new_tokens=4, temperature=1.0, top_k=4, top_p=1.0)
    out = {}
    for rule, base in (("rejection", 0), ("plain", 1 << 20)):
        rows = []
        for c in range(N // B):
            seed = torch.arange(B, dtype=torch.int64, device=dev) + base + c * B
            extra = {} if rule == "plain" else dict(assistant_model=noisy, num_assistant_tokens=2,
                                                    assistant_verification="rejection")
            tok, _ = tiny.generate(prompt, seed=seed, **kw, **extra)
            rows += [tuple(r[:3]) for r in tok.tolist()]
        out[rule] = rows
    keys = sorted(set(out["rejection"]) | set(out["plain"]))
    table = np.array([[rows.count(x) for x in keys] for rows in out.values()])
    p = float(chi2_contingency(table)[1])
    print(f"tiny bf16 on the device, rejection vs plain: p = {p:.3g}, {len(keys)} outcomes")
    assert p > 1e-3
