"""Assisted generation on the GPU: ``sample_slots_`` bit for bit against ``sample_tokens_`` row by row,
``assist_round_`` and ``lookup_accept_`` on drawn tokens exactly against the definition (ops/assisted.py,
ops/lookup.py), and ``GPT2DoubleHeads.generate(..., assistant_model=draft)`` on GPT-2 small with random weights,
with three drafts: greedy and sampled exactly against the definition evaluated eagerly with the same compute (host
counters and acceptance, one ``sample_tokens_`` call per slot), and greedy against plain ``generate`` up to near
ties."""
import numpy as np
import pytest
import torch

from test_gpu_lookup import _calibrate, _prompts

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


MODES = [dict(temperature=0.0, top_k=0, top_p=1.0),
         dict(temperature=0.7, top_k=0, top_p=0.9),
         dict(temperature=1.0, top_k=50, top_p=0.95, min_p=0.02, typical_p=0.9, eta_cutoff=0.001),
         dict(temperature=1.3, top_k=0, top_p=1.0, epsilon_cutoff=0.0003)]


def _slot_state(dev, B, k, n, seed, t_max=300):
    from adapcc_b200.ops import AssistState

    rng = np.random.default_rng(seed)
    st = AssistState(B, k, n, t_max, dev)
    st.emitted.copy_(torch.from_numpy(rng.integers(0, 6, B).astype(np.int32)))
    nq = rng.integers(1, k + 2, B).astype(np.int32)
    nq[0] = k + 1
    done = np.zeros(B, dtype=np.int32)
    done[2] = 1
    nq[2] = 0
    st.nq.copy_(torch.from_numpy(nq))
    st.done.copy_(torch.from_numpy(done))
    lens = torch.from_numpy(rng.integers(5, 200, B).astype(np.int32)).to(dev)
    return st, lens


@pytest.mark.parametrize("mode", range(len(MODES)))
def test_sample_slots_bit_exact_against_sample_tokens(dev, mode):
    from adapcc_b200.ops import sample_slots_, sample_tokens_

    kw = dict(MODES[mode])
    B, k, V, ld, n = 7, 4, 50262, 50304, 30
    S = k + 1
    st, lens = _slot_state(dev, B, k, n, mode)
    g = torch.Generator(device=dev).manual_seed(mode)
    logits = torch.randn(B * S, ld, device=dev, generator=g) * 3
    logits[:, V:] = 1e4                                                  # beyond vocab: never read
    sup_ids = [int(i) for i in logits[:, :V].argmax(1)[:4]]             # the best ids of some rows are suppressed
    sup = torch.tensor(sup_ids, dtype=torch.int32, device=dev)
    seeds = torch.arange(B, dtype=torch.int64, device=dev) * 977 + (1 << 33)
    min_new = 3
    st.g.fill_(-7)
    sample_slots_(logits, V, kw.pop("temperature"), kw.pop("top_k"), kw.pop("top_p"), seeds, st, lens, 0, min_new,
                  sup, **kw)
    kw = dict(MODES[mode])
    T, tk, tp = kw.pop("temperature"), kw.pop("top_k"), kw.pop("top_p")
    got = st.g.view(B, S).cpu()
    nq, em, done = st.nq.cpu(), st.emitted.cpu(), st.done.cpu()
    drawn = 0
    for b in range(B):
        for j in range(S):
            if done[b] or j >= nq[b]:
                assert int(got[b, j]) == -7, (b, j)                      # pad slots and done rows untouched
                continue
            step = torch.tensor([int(em[b]) + j], dtype=torch.int32, device=dev)
            pos = (lens[b:b + 1] + j + 1).contiguous()
            nxt, tok = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, 1, dtype=torch.int64, device=dev)
            sample_tokens_(logits[b * S + j:b * S + j + 1], V, T, tk, tp, seeds[b:b + 1], pos, step, min_new, sup,
                           None, torch.zeros(1, dtype=torch.int32, device=dev), nxt, tok, **kw)
            assert int(got[b, j]) == int(nxt), (mode, b, j)
            drawn += 1
    # draft draws: one logits row per row at draft step j, into ids[b, j + 1] and the draft's next input
    for j in range(k):
        st.ids.fill_(-5)
        st.d_in.fill_(-5)
        sample_slots_(logits[j::S].contiguous(), V, T, tk, tp, seeds, st, lens, j, min_new, sup, draft=True, **kw)
        ids, d_in = st.ids.view(B, S).cpu(), st.d_in.cpu()
        for b in range(B):
            if done[b] or j + 1 >= nq[b]:
                assert int(ids[b, j + 1]) == 0 and int(d_in[b]) == 0
            else:
                assert int(ids[b, j + 1]) == int(got[b, j]) == int(d_in[b]), (mode, b, j)
            assert (ids[b, :j + 1] == -5).all() and (ids[b, j + 2:] == -5).all()
    with pytest.raises(ValueError, match="one logits row per row"):    # draft j + 1 needs draft j: one at a time
        sample_slots_(logits[:2 * B], V, T, tk, tp, seeds, st, lens, 0, min_new, sup, draft=True, **kw)
    print(f"mode {mode}: {drawn} slots drawn bit-exact")


def test_round_and_accept_on_drawn_tokens_exact_against_the_definition(dev):
    from adapcc_b200.ops import assist_round_, lookup_accept_, sample_slots_
    from adapcc_b200.ops.assisted import assist_round, draw_slots
    from adapcc_b200.ops.lookup import lookup_accept

    B, k, n, t_max, V, n_pos = 8, 4, 24, 120, 1000, 110
    S = k + 1
    rng = np.random.default_rng(3)
    st, _ = _slot_state(dev, B, k, n, 3, t_max)
    st.seq.copy_(torch.from_numpy(rng.integers(0, V, (B, t_max)).astype(np.int32)))
    em = rng.integers(0, n - 1, B).astype(np.int32)
    em[0], em[1] = n - 1, n - 2                                          # no room for drafts / room for one
    st.emitted.copy_(torch.from_numpy(em))
    lens = torch.from_numpy(rng.integers(0, t_max - n, B).astype(np.int32))
    lens[3] = t_max - 1                                                  # positions past the cache are clamped
    lens = lens.to(dev)
    d_lens = torch.zeros(B, dtype=torch.int32, device=dev)
    want = assist_round(st.seq.cpu(), lens.cpu(), st.emitted.cpu(), st.done.cpu(), k, n, n_pos)
    assist_round_(st, lens, d_lens, n_pos)
    torch.cuda.synchronize()
    for name, w in zip(("ids", "pos", "nq", "d_in", "d_pos"), want):
        assert torch.equal(getattr(st, name).cpu(), w), name
    assert torch.equal(d_lens, lens)
    # drafts that mostly equal the target's draws, then the draws and acceptance against the definition
    logits = torch.from_numpy(rng.standard_normal((B * S, 1024)).astype(np.float32) * 2)
    seeds = torch.arange(B, dtype=torch.int64) + 40
    host = draw_slots(logits, V, 0.8, 0, 0.9, seeds.tolist(), lens.cpu(), st.emitted.cpu(), st.done.cpu(),
                      st.nq.cpu())
    ids = st.ids.cpu().view(B, S)
    for b in range(B):
        for j in range(1, S):
            ids[b, j] = int(host[b, j - 1]) if (b % 4 != 3 or j < 2) and host[b, j - 1] >= 0 else 0
    st.ids.copy_(ids.view(-1))
    stop = [int(host[5, 1])] if host[5, 1] >= 0 else []
    ld = logits.to(dev)
    sample_slots_(ld, V, 0.8, 0, 0.9, seeds.to(dev), st, lens)
    names = ("seq", "emitted", "done", "tokens", "steps")
    w = {name: getattr(st, name).cpu().clone() for name in names}
    wl = lens.cpu().clone()
    lookup_accept(None, V, st.ids.cpu(), st.nq.cpu(), w["seq"], wl, w["emitted"], w["done"], w["tokens"],
                  w["steps"], stop_ids=stop, drawn=torch.from_numpy(host))
    lookup_accept_(st, lens, torch.tensor(stop, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    for name in names:
        assert torch.equal(getattr(st, name).cpu(), w[name]), name
    assert torch.equal(lens.cpu(), wl)
    grown = (w["emitted"] - torch.from_numpy(em)).tolist()
    print(f"tokens emitted per row: {grown}")
    assert max(grown) >= 3


# ---- GPT-2 small, random weights -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models(dev):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(0)
    target = GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()
    cut = GPT2DoubleHeads(GPT2Config(n_layer=2)).to(device=dev, dtype=torch.bfloat16).eval()
    cut.load_state_dict({k: v for k, v in target.state_dict().items()
                         if not k.startswith("h.") or k.split(".")[1] in ("0", "1")})
    torch.manual_seed(77)
    other = GPT2DoubleHeads(GPT2Config(n_layer=2)).to(device=dev, dtype=torch.bfloat16).eval()
    return {"self": target, "cut": cut, "other": other}


@torch.no_grad()
def _eager_assisted(model, draft, ids, lengths, k, n, mode, seeds, min_new=0, suppress=(), stop=()):
    """The definition (ops/assisted.py) run eagerly on the GPU, with the native path's compute: the draft's decode steps
    at B rows, the model's verify steps at B·(k+1) rows, and the LM head, all launched one by one as ``generate``'s
    graph launches them. The round set-up, counters, steps and acceptance are computed on the host
    (``assist_round``, ``lookup_accept``), and each slot is drawn by its own ``sample_tokens_`` call with the counter
    ``lens + j + 1`` and step ``emitted + j`` computed here. Returns ``(tokens, emitted, steps)``."""
    from adapcc_b200.models.gpt2 import KVCache, VerifyKV
    from adapcc_b200.ops import decode_attention_work_numel, lm_head_logits_, sample_tokens_
    from adapcc_b200.ops.assisted import assist_round
    from adapcc_b200.ops.lookup import lookup_accept

    kw = dict(mode)
    T, tk, tp = kw.pop("temperature"), kw.pop("top_k"), kw.pop("top_p")
    dev, W, dW, V = ids.device, model.wte.weight, draft.wte.weight, model.cfg.vocab_size
    B, Tp = ids.shape
    S, t_max, dc = k + 1, max(lengths) + n, draft.cfg
    sup = torch.tensor(list(suppress), dtype=torch.int32, device=dev)
    zero = torch.zeros(1, dtype=torch.int32, device=dev)
    nxt, tok = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, 1, dtype=torch.int64, device=dev)

    def draw(row, b, L, e, j):                     # the token at sequence index L + j + 1, step e + j
        pos = torch.tensor([L + j + 1], dtype=torch.int32, device=dev)
        step = torch.tensor([e + j], dtype=torch.int32, device=dev)
        sample_tokens_(row, V, T, tk, tp, seeds[b:b + 1], pos, step, min_new, sup, None, zero, nxt, tok, **kw)
        return int(nxt)

    last = torch.tensor(lengths, device=dev) - 1
    cache = model.new_cache(B, t_max)
    h = model.hidden(ids, None, cache=cache, lengths=lengths)[torch.arange(B, device=dev), last]
    dcache = KVCache(dc.n_layer, B, dc.n_head, t_max + k, dc.n_embd // dc.n_head, dW.dtype, dev)
    draft.hidden(ids, None, cache=dcache, lengths=lengths)
    work = torch.empty(decode_attention_work_numel(B * S, model.cfg.n_head, model.cfg.n_embd // model.cfg.n_head,
                                                   t_max), dtype=torch.float32, device=dev)
    logits = torch.empty(B * S, W.shape[0], dtype=torch.float32, device=dev)
    dlogits = torch.empty(B, dW.shape[0], dtype=torch.float32, device=dev)
    seq = torch.zeros(B, t_max, dtype=torch.int32)
    seq[:, :Tp] = ids.cpu()
    lens = torch.tensor(lengths, dtype=torch.int32) - 1
    emitted, done, steps = (torch.zeros(B, dtype=torch.int32) for _ in range(3))
    tokens = torch.full((B, n), -1, dtype=torch.int64)
    lm_head_logits_(h, W, logits[:B])
    g = torch.tensor([[draw(logits[b:b + 1], b, int(lens[b]), 0, 0)] for b in range(B)])
    lookup_accept(None, V, torch.zeros(B * S, dtype=torch.int64), torch.ones(B, dtype=torch.int32), seq, lens,
                  emitted, done, tokens, None, stop_ids=stop, drawn=g)
    while not bool(done.all()):
        slots, pos, nq, d_in, d_pos = assist_round(seq, lens, emitted, done, k, n, dc.n_positions)
        slots = slots.view(B, S)
        dcache.lens.copy_(lens)
        for j in range(S):
            hd = draft._blocks(draft._embed(d_in.to(dev), None, d_pos[j].to(dev)), dcache)
            dcache.lens.add_(1)
            if j < k:
                lm_head_logits_(hd, dW, dlogits)
                d_in = torch.tensor([draw(dlogits[b:b + 1], b, int(lens[b]), int(emitted[b]), j)
                                     if not done[b] and j + 1 < nq[b] else 0 for b in range(B)])
                slots[:, j + 1] = d_in
        cache.lens.copy_(lens)
        hv = model._verify_hidden(slots.reshape(-1).to(dev), pos.to(dev), None, VerifyKV(cache, S, nq.to(dev), work))
        lm_head_logits_(hv, W, logits)
        g = torch.full((B, S), -1, dtype=torch.int64)
        for b in range(B):
            for j in range(int(nq[b]) if not done[b] else 0):
                g[b, j] = draw(logits[b * S + j:b * S + j + 1], b, int(lens[b]), int(emitted[b]), j)
        lookup_accept(None, V, slots.reshape(-1), nq, seq, lens, emitted, done, tokens, steps, stop_ids=stop,
                      drawn=g)
    return tokens, emitted, steps


@pytest.mark.parametrize("mode", range(len(MODES)))
def test_gpt2_small_assisted_generate_exact_against_eager_definition(models, dev, mode):
    """The graph-replayed native path against the definition evaluated eagerly with the same compute: every token,
    every row's emitted count and verify steps equal, with each draft, stop and suppressed ids and min_new_tokens; no
    row is exempt."""
    gpt2 = models["self"]
    V, n, k = gpt2.cfg.vocab_size, 32, 4
    ids, lengths = _prompts(V, dev)
    seeds = torch.arange(8, dtype=torch.int64, device=dev) * 31 + 17
    plain, _ = gpt2.generate(ids, lengths, max_new_tokens=n, seed=seeds, **MODES[mode])
    stop, suppress = [int(plain[0, 9]), int(plain[5, 3])], [int(plain[5, 3]), int(plain[2, 0])]
    gk = dict(MODES[mode], max_new_tokens=n, seed=seeds, stop_ids=stop, suppress_ids=suppress, min_new_tokens=5)
    for name, draft in models.items():
        got, n_got = gpt2.generate(ids, lengths, assistant_model=draft, num_assistant_tokens=k, **gk)
        st = {key: v.cpu() for key, v in gpt2.assist_stats.items() if key != "replays"}
        want, emitted, steps = _eager_assisted(gpt2, draft, ids, lengths, k, n, MODES[mode], seeds, 5, suppress, stop)
        assert torch.equal(got.cpu(), want), (mode, name)
        assert torch.equal(st["emitted"], emitted) and torch.equal(st["steps"], steps), (mode, name)
        assert torch.equal(n_got.cpu(), (want >= 0).sum(1))
        per_step = float((emitted - 1).sum()) / float(steps.sum())
        print(f"mode {mode}, draft {name}: tokens equal to the eager definition, {per_step:.2f} tokens per verify "
              f"step, {int((want >= 0).sum())} tokens, {int((n_got < n).sum())} rows stopped early")
        if name == "self" and mode == 0:
            assert per_step > 2.0                                        # greedy: the draft is the target
    # rows alone: the same, and a row's tokens do not depend on the batch it was generated in
    for b in (1, 4):
        row = ids[b:b + 1, :lengths[b]]
        g1, _ = gpt2.generate(row, assistant_model=models["cut"], num_assistant_tokens=k,
                              **dict(gk, seed=seeds[b:b + 1]))
        w1, _, _ = _eager_assisted(gpt2, models["cut"], row, [lengths[b]], k, n, MODES[mode], seeds[b:b + 1], 5,
                                   suppress, stop)
        assert torch.equal(g1.cpu(), w1), (mode, b)


def _check_greedy(got, want, plain, delta, what):
    """Rows equal to plain greedy ``generate``, or first different at a near tie of the two best logits (within
    2·delta, the measured verify-vs-decode logit difference); returns the exempt rows."""
    exempt = 0
    for b in range(got.shape[0]):
        if torch.equal(got[b], want[b]):
            continue
        i = int(torch.nonzero(got[b] != want[b])[0])
        top2 = torch.topk(plain[b, i], 2).values
        assert float(top2[0] - top2[1]) <= 2 * delta, (what, b, i, float(top2[0] - top2[1]), delta)
        exempt += 1
    return exempt


def test_gpt2_small_greedy_assisted_generate_against_plain(models, dev):
    """Greedy assisted generation against plain greedy ``generate``: the verify step's GEMMs run at B·(k+1) rows, so
    rows may differ at near ties only, and at most 2 of 8."""
    gpt2 = models["self"]
    V, n, k = gpt2.cfg.vocab_size, 40, 4
    ids, lengths = _prompts(V, dev)
    want, n_want = gpt2.generate(ids, lengths, max_new_tokens=n, temperature=0.0)
    plain, delta = _calibrate(gpt2, ids, lengths, want, k)
    for name, draft in models.items():
        got, n_got = gpt2.generate(ids, lengths, max_new_tokens=n, temperature=0.0, assistant_model=draft,
                                   num_assistant_tokens=k)
        again, _ = gpt2.generate(ids, lengths, max_new_tokens=n, temperature=0.0, assistant_model=draft,
                                 num_assistant_tokens=k)
        assert torch.equal(again, got), name                              # graph replay equals a second run
        exempt = _check_greedy(got, want, plain, delta, name)
        print(f"draft {name}: delta {delta:.3g}, {exempt} of 8 rows exempt")
        assert exempt <= 2 and torch.equal(n_got, n_want)


def test_row_reaching_n_positions_runs_clean(models, dev):
    gpt2 = models["self"]
    n, k = 12, 7
    N = gpt2.cfg.n_positions
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, 50000, (2, N - n), generator=g).to(dev)
    lengths = [N - n, 100]
    seeds = torch.tensor([3, 4], dtype=torch.int64, device=dev)
    for mode in (0, 1):
        for name in ("self", "other"):
            got, n_got = gpt2.generate(ids, lengths, assistant_model=models[name], num_assistant_tokens=k,
                                       max_new_tokens=n, seed=seeds, **MODES[mode])
            torch.cuda.synchronize()
            want, _, _ = _eager_assisted(gpt2, models[name], ids, lengths, k, n, MODES[mode], seeds)
            assert torch.equal(got.cpu(), want) and int(n_got[0]) == n, (mode, name)
