"""The fp8 (e4m3) KV cache on the GPU: ``kv_quantize_`` and the stores of the fp8 ``decode_attention_`` bit for bit
against ``ops/kvcache.py``; the fp8 decode attention bit for bit against the bf16 op on a bf16 cache holding the
dequantized values; the fp8 ``kv_reorder_`` against torch indexing; and GPT-2 small generating on an fp8 cache."""
import pytest
import torch

pytestmark = pytest.mark.gpu

FP8_NAN = 0x7F            # an e4m3 NaN byte: a sentinel the kernels must neither read nor overwrite
LENS = [0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1022, 1023]     # as in test_gpu_decode.py


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.uint8) if t.dtype == torch.uint8 else \
        t.view(torch.int16)


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _hard_values(dev, B, T, n_vec, Dh, seed):
    """bf16 [B, T, n_vec * Dh] of mixed magnitudes: normal, tiny (bf16 subnormals) and huge vectors, and at every
    third position vectors of e4m3 ties."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, T, n_vec, Dh, device=dev, generator=g)
    mag = torch.tensor([1.0, 1e-3, 1e-30, 1e30, 2.0 ** -120, 3e4], device=dev)
    x = x * mag[torch.randint(0, len(mag), (B, T, n_vec, 1), device=dev, generator=g)]
    # amax = 255 gives e = 0, and each of the first eight values lies halfway between two e4m3 neighbours (or is 255)
    ties = torch.tensor([136.0, 152.0, 9.5, 10.5, 2.0 ** -10, 3 * 2.0 ** -10, -200.0, 255.0], device=dev)
    x[:, ::3, :, :8] = ties
    x[:, ::3, :, 8:] = 0.0
    x[:, ::3, :, -1] = 255.0
    return x.reshape(B, T, n_vec * Dh).to(torch.bfloat16)


@pytest.mark.parametrize("H,Dh", [(12, 64), (4, 16), (4, 128)])
def test_kv_quantize_matches_reference(dev, H, Dh):
    from adapcc_b200.ops import kv_quantize_
    from adapcc_b200.ops.kvcache import quantize

    B, t_max = 3, 160
    D = H * Dh
    for T in (1, 5, 64, 131, 160):
        x = _hard_values(dev, B, T, 3 * H, Dh, seed=T)
        x[0, 0, D + 3] = float("nan")                    # a non-finite key vector: NaN scale, zero bytes
        x[1, T - 1, 2 * D] = float("inf")
        kc = torch.full((B, H, t_max, Dh), FP8_NAN, dtype=torch.uint8, device=dev)
        vc = kc.clone()
        ks = torch.full((B, H, t_max), float("nan"), device=dev)
        vs = ks.clone()
        kv_quantize_(x, kc, vc, ks, vs)
        torch.cuda.synchronize()
        for off, c, s in ((D, kc, ks), (2 * D, vc, vs)):
            q, sc = quantize(x[:, :, off:off + D].view(B, T, H, Dh).transpose(1, 2).cpu())     # on the CPU
            assert _same(c[:, :, :T].cpu(), q), (T, off)
            assert _same(s[:, :, :T].cpu(), sc), (T, off)
            assert bool((c[:, :, T:] == FP8_NAN).all()) and bool(s[:, :, T:].isnan().all()), T
        assert bool(ks[0, 0, 0].isnan()) and bool((kc[0, 0, 0] == 0).all())
        assert bool(vs[1, 0, T - 1].isnan())


def _fp8_inputs(dev, lens, H, Dh, t_max, seed):
    """qkv; an fp8 cache with the quantized random vectors below lens[b] and NaN sentinels from lens[b] on; the bf16
    cache holding its dequantized values (the same sentinels)."""
    from adapcc_b200.ops.kvcache import dequantize, quantize

    g = torch.Generator(device=dev).manual_seed(seed)
    B = len(lens)
    qkv = torch.randn(B, 3 * H * Dh, device=dev, generator=g)
    qkv[:, :H * Dh] *= 2.0
    qkv = qkv.to(torch.bfloat16)
    lens_t = torch.tensor(lens, dtype=torch.int32, device=dev)
    beyond = torch.arange(t_max, device=dev)[None, :] >= lens_t[:, None].long()
    out = []
    for _ in range(2):
        q, s = quantize(torch.randn(B, H, t_max, Dh, device=dev, generator=g).to(torch.bfloat16))
        q[beyond[:, None, :, None].expand_as(q)] = FP8_NAN
        s[beyond[:, None, :].expand_as(s)] = float("nan")
        out += [q, s, dequantize(q, s).to(torch.bfloat16)]
    kq, ks, kb, vq, vs, vb = out
    return qkv, lens_t, kq, ks, vq, vs, kb, vb


def _attend(qkv, lens, kc, vc, ks=None, vs=None):
    from adapcc_b200.ops import decode_attention_, decode_attention_work_numel

    B, H, t_max, Dh = kc.shape
    out = torch.full((B, H * Dh), float("nan"), dtype=torch.bfloat16, device=kc.device)
    work = torch.empty(decode_attention_work_numel(B, H, Dh, t_max), dtype=torch.float32, device=kc.device)
    return decode_attention_(qkv, kc, vc, lens, out, work, k_scale=ks, v_scale=vs)


@pytest.mark.parametrize("H,Dh", [(12, 64), (4, 16), (4, 128)])
def test_fp8_decode_attention_is_bf16_on_dequantized_cache(dev, H, Dh):
    from adapcc_b200.ops.kvcache import quantize

    t_max, D = 1024, H * Dh
    qkv, lens, kq, ks, vq, vs, kb, vb = _fp8_inputs(dev, LENS, H, Dh, t_max, seed=H + Dh)
    k8, s8, v8, w8 = kq.clone(), ks.clone(), vq.clone(), vs.clone()
    out8 = _attend(qkv, lens, k8, v8, s8, w8)
    out16 = _attend(qkv, lens, kb.clone(), vb.clone())
    torch.cuda.synchronize()
    assert _same(out8, out16)
    # the new k / v at lens[b], quantized; nothing else changed
    rows = torch.arange(len(LENS), device=dev)
    pos = lens.long()
    for new, c0, s0, c, s in ((qkv[:, D:2 * D], kq, ks, k8, s8), (qkv[:, 2 * D:], vq, vs, v8, w8)):
        q, sc = quantize(new.view(-1, H, Dh).cpu())
        q, sc = q.to(dev), sc.to(dev)
        assert _same(c[rows, :, pos], q) and _same(s[rows, :, pos], sc)
        c0, s0 = c0.clone(), s0.clone()
        c0[rows, :, pos], s0[rows, :, pos] = q, sc
        assert _same(c, c0) and _same(s, s0)
    # repeatable, and each row alone gives its bits in the batch
    again = _attend(qkv, lens, kq.clone(), vq.clone(), ks.clone(), vs.clone())
    assert _same(again, out8)
    for b in (0, 3, 9, 12):
        one = _attend(qkv[b:b + 1], lens[b:b + 1], kq[b:b + 1].clone(), vq[b:b + 1].clone(), ks[b:b + 1].clone(),
                      vs[b:b + 1].clone())
        assert _same(one[0], out8[b]), b
    # graph replay equals an eager launch
    from adapcc_b200.ops import decode_attention_, decode_attention_work_numel

    B = len(LENS)
    k8, s8, v8, w8 = kq.clone(), ks.clone(), vq.clone(), vs.clone()
    out = torch.empty(B, D, dtype=torch.bfloat16, device=dev)
    work = torch.empty(decode_attention_work_numel(B, H, Dh, t_max), dtype=torch.float32, device=dev)
    decode_attention_(qkv, k8, v8, lens, out, work, k_scale=s8, v_scale=w8)     # warm-up
    k8.copy_(kq), s8.copy_(ks), v8.copy_(vq), w8.copy_(vs)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        decode_attention_(qkv, k8, v8, lens, out, work, k_scale=s8, v_scale=w8)
    k8.copy_(kq), s8.copy_(ks), v8.copy_(vq), w8.copy_(vs)
    out.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert _same(out, out8)


def test_fp8_decode_attention_argument_checks(dev):
    qkv, lens, kq, ks, vq, vs, kb, vb = _fp8_inputs(dev, [3, 5], 4, 16, 64, seed=0)
    for kw in (dict(k_scale=ks), dict(v_scale=vs), dict(k_scale=ks, v_scale=vs[:, :, :10].contiguous())):
        with pytest.raises(ValueError, match="decode_attention_"):
            _attend(qkv, lens, kq, vq, kw.get("k_scale"), kw.get("v_scale"))
    with pytest.raises(ValueError, match="decode_attention_"):
        _attend(qkv, lens, kq, vq)                      # a uint8 cache without scales
    with pytest.raises(ValueError, match="decode_attention_"):
        _attend(qkv, lens, kb, vb, ks, vs)              # scales with a bf16 cache


def _reorder_want(k, parent, prompt_len, lens, max_new):
    want = k.clone()
    for r, p in enumerate(parent.tolist()):
        if p == r:
            continue
        lo, hi = int(prompt_len[r]), min(int(lens[r]), int(prompt_len[r]) + max_new)
        want[:, r, :, lo:hi] = k[:, p, :, lo:hi]
    return want


def test_fp8_kv_reorder_against_torch_indexing(dev):
    from adapcc_b200.ops import kv_reorder_, kv_reorder_scratch_numel

    L, R, H, t_max, Dh, max_new = 3, 12, 2, 48, 64, 16
    g = torch.Generator(device=dev).manual_seed(0)
    parts = [torch.randint(0, 256, (L, R, H, t_max, Dh), dtype=torch.uint8, device=dev, generator=g) for _ in range(2)]
    parts += [torch.randn(L, R, H, t_max, device=dev, generator=g) for _ in range(2)]
    prompt_len = torch.tensor([5, 5, 5, 5, 9, 9, 9, 9, 14, 14, 14, 14], dtype=torch.int32, device=dev)
    lens = prompt_len + torch.tensor([0, 1, 3, 16, 7, 7, 7, 7, 2, 2, 2, 2], dtype=torch.int32, device=dev)
    scratch = torch.empty(kv_reorder_scratch_numel(parts[0], max_new, fp8=True), dtype=torch.uint8, device=dev)
    maps = {"permutation": [1, 0, 3, 2, 6, 4, 5, 7, 11, 10, 9, 8],
            "cycle": [3, 0, 1, 2, 5, 6, 7, 4, 9, 10, 11, 8],
            "many_to_one": [0, 0, 0, 0, 4, 4, 5, 5, 8, 8, 8, 8],
            "identity": list(range(R))}
    for name, pm in maps.items():
        parent = torch.tensor(pm, dtype=torch.int32, device=dev)
        k, v, ks, vs = (t.clone() for t in parts)
        kv_reorder_(k, v, parent, prompt_len, lens, max_new, scratch, k_scale=ks, v_scale=vs)
        torch.cuda.synchronize()
        for got, t0 in zip((k, v, ks, vs), parts):
            assert _same(got, _reorder_want(t0, parent, prompt_len, lens, max_new)), name
    parent = torch.tensor(maps["cycle"], dtype=torch.int32, device=dev)
    eager = [t.clone() for t in parts]
    kv_reorder_(*eager[:2], parent, prompt_len, lens, max_new, scratch, k_scale=eager[2], v_scale=eager[3])
    k, v, ks, vs = (t.clone() for t in parts)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        kv_reorder_(k, v, parent, prompt_len, lens, max_new, scratch, k_scale=ks, v_scale=vs)
    for t, t0 in zip((k, v, ks, vs), parts):
        t.copy_(t0)
    graph.replay()
    torch.cuda.synchronize()
    assert all(_same(a, b) for a, b in zip((k, v, ks, vs), eager))
    with pytest.raises(ValueError, match="kv_reorder_"):
        kv_reorder_(k, v, parent, prompt_len, lens, max_new, scratch[:10], k_scale=ks, v_scale=vs)
    with pytest.raises(ValueError, match="kv_reorder_"):
        kv_reorder_(k, v, parent, prompt_len, lens, max_new, scratch, k_scale=ks)


# ---- GPT-2 small ---------------------------------------------------------------------------------------------------
def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


@pytest.fixture(scope="module")
def small(dev):
    return _gpt2_small(dev, seed=3)


def test_teacher_forced_fp8_cache_is_bf16_cache_of_dequantized_values(dev, small):
    """Each step: the bf16 cache is overwritten with the fp8 cache's dequantized contents, then both decode the same
    token; the hidden states have the same bits."""
    from adapcc_b200.ops.kvcache import dequantize

    m, V = small, small.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(1)
    B, T, n = 4, 40, 12
    lengths = [40, 7, 23, 1]
    ids = torch.randint(0, V, (B, T + n), device=dev, generator=g)
    c8, cb = m.new_cache(B, T + n, "fp8_e4m3"), m.new_cache(B, T + n)
    with torch.no_grad():
        h8 = m.hidden(ids[:, :T], None, cache=c8, lengths=lengths)
        hb = m.hidden(ids[:, :T], None, cache=cb, lengths=lengths)
        assert _same(h8, hb)                            # the prefill attends to the unquantized keys and values
        for i in range(n):
            cb.k.copy_(dequantize(c8.k, c8.k_scale).to(torch.bfloat16))
            cb.v.copy_(dequantize(c8.v, c8.v_scale).to(torch.bfloat16))
            x = ids[:, T + i]
            h8, hb = m.decode_step(x, None, c8), m.decode_step(x, None, cb)
            assert _same(h8, hb), i


@torch.no_grad()                                        # as generate: the decode-path MLP, not the training GEMMs
def _eager_generate(m, ids, lengths, n, temperature, seed, guided):
    """``generate`` on an fp8 cache as an eager loop of decode_step and the native head, guidance mix and sampler.
    With ``guided`` the negative prompt is each row's last prompt token and the scale 1.5."""
    from adapcc_b200.ops import guidance_mix_, lm_head_logits_, sample_tokens_

    dev, V = ids.device, m.cfg.vocab_size
    B, T = ids.shape
    rows = torch.arange(B, device=dev)
    last = torch.tensor(lengths, device=dev) - 1
    if guided:
        x = torch.zeros(2 * B, T, dtype=ids.dtype, device=dev)
        x[:B], x[B:, 0] = ids, ids[rows, last]
        lens = list(lengths) + [1] * B
    else:
        x, lens = ids, list(lengths)
    R = len(lens)
    cache = m.new_cache(R, max(lens) + n, "fp8_e4m3")
    h = m.hidden(x, None, cache=cache, lengths=lens)[torch.arange(R, device=dev), torch.tensor(lens, device=dev) - 1]
    w = m.wte.weight
    logits = torch.empty(R, w.shape[0], dtype=torch.float32, device=dev)
    next_ids = torch.zeros(R, dtype=torch.int64, device=dev)
    tokens = torch.full((B, n), -1, dtype=torch.int64, device=dev)
    done = torch.zeros(B, dtype=torch.int32, device=dev)
    step = torch.zeros(1, dtype=torch.int32, device=dev)
    seeds = seed + torch.arange(B, dtype=torch.int64, device=dev)
    none = torch.zeros(0, dtype=torch.int32, device=dev)
    for i in range(n):
        if i:
            h = m.decode_step(next_ids, None, cache)
        lm_head_logits_(h, w, logits)
        if guided:
            guidance_mix_(logits, V, B, 1.5)
        sample_tokens_(logits[:B], V, temperature, 0, 0.9, seeds, cache.lens[:B], step, 0, none, none, done,
                       next_ids[:B], tokens)
        if guided:
            next_ids[B:].copy_(next_ids[:B])
    return tokens


@pytest.mark.parametrize("temperature,guided", [(0.0, False), (0.8, False), (0.0, True), (0.8, True)])
def test_generate_fp8_graph_equals_eager_loop(dev, small, temperature, guided):
    m, V = small, small.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(2)
    lengths = [96, 17, 60, 1, 33]
    ids = torch.randint(0, V, (len(lengths), 96), device=dev, generator=g)
    n = 24
    kw = dict(max_new_tokens=n, temperature=temperature, top_p=0.9, seed=11, kv_cache_dtype="fp8_e4m3")
    if guided:
        kw["guidance_scale"] = 1.5
    tokens, n_new = m.generate(ids, lengths, **kw)
    again, _ = m.generate(ids, lengths, **kw)
    assert torch.equal(tokens, again)
    want = _eager_generate(m, ids, lengths, n, temperature, 11, guided)
    assert torch.equal(tokens, want)
    assert n_new.tolist() == [n] * len(lengths)


def test_beam_search_fp8_graph_equals_eager_loop(dev, small):
    import numpy as np

    from adapcc_b200.ops import BeamState, beam_step_, kv_reorder_, kv_reorder_scratch_numel, lm_head_logits_
    from adapcc_b200.ops.beam import best_hypotheses, merge_finished_sets

    m, V = small, small.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(5)
    B, K, n, T = 4, 4, 20, 80
    lengths = [80, 12, 47, 1]
    ids = torch.randint(0, V, (B, T), device=dev, generator=g)
    stop = [int(ids[0, 0])]
    kw = dict(num_beams=K, max_new_tokens=n, stop_ids=stop, kv_cache_dtype="fp8_e4m3")
    got = m.beam_search(ids, lengths, **kw)
    again = m.beam_search(ids, lengths, **kw)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    w = m.wte.weight
    with torch.no_grad():
        last = torch.tensor(lengths, device=dev) - 1
        pre = m.new_cache(B, T, "fp8_e4m3")
        h = m.hidden(ids, None, cache=pre, lengths=lengths)[torch.arange(B, device=dev), last]
        cache = m.new_cache(B * K, max(lengths) + n, "fp8_e4m3")
        cache.reset([x for x in lengths for _ in range(K)], T)
        for dst, src in zip(cache.parts, pre.parts):
            dst[:, :, :, :T].copy_(src.repeat_interleave(K, dim=1))
        h = h.repeat_interleave(K, dim=0).contiguous()
        st = BeamState(B, K, n, 1.0, dev)
        logits = torch.empty(B * K, w.shape[0], dtype=torch.float32, device=dev)
        sup = torch.zeros(0, dtype=torch.int32, device=dev)
        stp = torch.tensor(stop, dtype=torch.int32, device=dev)
        prompt_len = cache.lens.clone()
        scratch = torch.empty(kv_reorder_scratch_numel(cache.k, n, fp8=True), dtype=torch.uint8, device=dev)
        for i in range(n):
            if i:
                h = m.decode_step(st.next_ids, None, cache)
            lm_head_logits_(h, w, logits)
            beam_step_(logits, V, st, 0, sup, stp)
            kv_reorder_(cache.k, cache.v, st.parent, prompt_len, cache.lens, n, scratch, k_scale=cache.k_scale,
                        v_scale=cache.v_scale)
            if bool(st.done.all()):
                break
    fin = [merge_finished_sets(sets) for sets in st.finished()]
    want = best_hypotheses(fin, st.hist_tok.view(n, B, K).cpu().numpy(), st.hist_back.view(n, B, K).cpu().numpy(),
                           n, 1)
    for a, b in zip(got, want):
        assert np.array_equal(a.cpu().numpy(), b.cpu().numpy() if torch.is_tensor(b) else np.asarray(b))


def test_beam_search_one_beam_is_greedy_generate_fp8(dev, small):
    m, V = small, small.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(6)
    prompt = torch.randint(0, V, (1, 150), device=dev, generator=g)
    want, _ = m.generate(prompt, max_new_tokens=32, temperature=0.0, kv_cache_dtype="fp8_e4m3")
    tokens, n_new, _ = m.beam_search(prompt, num_beams=1, max_new_tokens=32, kv_cache_dtype="fp8_e4m3")
    assert torch.equal(tokens, want) and n_new.tolist() == [32]


def test_stochastic_beam_search_fp8_repeatable(dev, small):
    m, V = small, small.cfg.vocab_size
    g = torch.Generator(device=dev).manual_seed(7)
    ids = torch.randint(0, V, (3, 50), device=dev, generator=g)
    kw = dict(num_beams=4, max_new_tokens=16, temperature=0.9, top_k=50, seed=3, kv_cache_dtype="fp8_e4m3")
    a = m.stochastic_beam_search(ids, [50, 9, 31], **kw)
    b = m.stochastic_beam_search(ids, [50, 9, 31], **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert int((a[1] > 0).sum()) > 0
