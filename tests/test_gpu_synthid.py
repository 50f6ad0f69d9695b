"""SynthID Text watermarking on the GPU: the sampler's SynthID instantiation against the fp64 definition
(``ops.sampling.reference_row``), skipped and repeated steps against the plain sampler bit for bit, a row alone against
the same row in a batch, ``generate`` on GPT-2 small (graph replay) against eager loops of the same kernels,
``synthid_count_`` and the g-values against the reference and HuggingFace exactly, detection power and false alarms,
and the launches per replay."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

V, LD = 50257, 50304
KEYS9 = [654, 400, 836, 123, 340, 443, 597, 160, 57]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def _logits(rng, R):
    """fp32 [R, LD] with +-0, subnormals and -inf planted at 256 random ids per row."""
    x = (rng.standard_normal((R, LD)) * 2).astype(np.float32)
    special = np.array([0.0, -0.0, 1e-40, -1e-40, 1.4e-45, -np.inf, 3e-39, -2e-38], dtype=np.float32)
    for r in range(R):
        x[r, rng.choice(LD, size=256, replace=False)] = np.resize(special, 256)
    return x


def _sample(dev, logits, gen, temperature, top_k, top_p, seeds, pos, synthid):
    """One ``sample_tokens_`` call at step t = gen.shape[1] with the rows' reply columns so far in ``tokens``."""
    from adapcc_b200.ops import sample_tokens_

    B, t = gen.shape
    tokens = torch.full((B, t + 1), -1, dtype=torch.int64, device=dev)
    tokens[:, :t] = torch.from_numpy(gen).to(dev)
    nxt = torch.zeros(B, dtype=torch.int64, device=dev)
    sample_tokens_(torch.from_numpy(logits).to(dev), V, temperature, top_k, top_p,
                   torch.as_tensor(seeds, dtype=torch.int64, device=dev),
                   torch.as_tensor(pos, dtype=torch.int32, device=dev), torch.tensor([t], dtype=torch.int32, device=dev),
                   0, None, None, torch.zeros(B, dtype=torch.int32, device=dev), nxt, tokens, synthid=synthid)
    torch.cuda.synchronize()
    assert torch.equal(tokens[:, t], nxt)
    return nxt.cpu().numpy()


@pytest.mark.parametrize("temperature,top_k,top_p", [(0.0, 0, 1.0), (1.0, 50, 1.0), (0.9, 0, 0.9), (1.0, 0, 1.0)])
def test_kernel_matches_reference(dev, temperature, top_k, top_p):
    """Tokens equal the fp64 reference's, except where the reference's target lies within fp32 rounding of a prefix
    boundary (sampled) or the two p' values are within fp32 rounding (greedy)."""
    from adapcc_b200.ops.sampling import reference_row
    from adapcc_b200.ops.synthid import check_synthid_args, synthid_flags

    rng = np.random.default_rng(int(temperature * 10) + top_k)
    near = 0
    for m, n in ((9, 5), (30, 3)):
        cfg = check_synthid_args("t", dict(ngram_len=n, keys=[int(k) for k in rng.integers(-2 ** 63, 2 ** 63, m)]))
        R, t = 8, 12
        logits = _logits(rng, R)
        gen = rng.integers(0, V, (R, t))
        seeds, pos = rng.integers(0, 2 ** 62, R), rng.integers(0, 1000, R)
        got = _sample(dev, logits, gen, temperature, top_k, top_p, seeds, pos, cfg)
        for r in range(R):
            assert synthid_flags(gen[r], cfg)[0] == "watermarked"
            ref = reference_row(logits[r, :V], temperature, top_k, top_p, int(seeds[r]), int(pos[r]), t, synthid=cfg,
                                generated=gen[r])
            k, want = int(got[r]), ref["token"]
            if k == want:
                continue
            near += 1
            q = ref["synthid_p"]
            if temperature == 0:
                assert abs(q[k] - q[want]) <= 1e-5 * q[want], (r, k, want)
            else:
                lo = min(k, want)
                assert abs(ref["cum"][lo] - ref["target"]) <= 1e-5 * ref["Zp"], (r, k, want)
    assert near <= 2, near


def test_skipped_and_repeated_steps_equal_the_plain_sampler(dev):
    from adapcc_b200.ops.synthid import check_synthid_args, synthid_flags

    rng = np.random.default_rng(7)
    R = 8
    for temperature, top_k in ((0.0, 0), (1.0, 50), (1.0, 0)):
        cfg = check_synthid_args("t", dict(ngram_len=4, keys=KEYS9, skip_first_ngram_calls=True,
                                           context_history_size=6))
        logits = _logits(rng, R)
        seeds, pos = rng.integers(0, 2 ** 62, R), rng.integers(0, 1000, R)
        for gen, kind in ((rng.integers(0, V, (R, 2)), "skipped"),
                          (np.tile([3, 4, 5, 3, 4, 5, 3, 4, 5], (R, 1)), "repeated")):
            assert all(synthid_flags(g, cfg)[0] == kind for g in gen)
            on = _sample(dev, logits, gen, temperature, top_k, 1.0, seeds, pos, cfg)
            off = _sample(dev, logits, gen, temperature, top_k, 1.0, seeds, pos, None)
            assert np.array_equal(on, off), kind
        gen = rng.integers(0, V, (R, 9))
        on = _sample(dev, logits, gen, temperature, top_k, 1.0, seeds, pos, cfg)
        off = _sample(dev, logits, gen, temperature, top_k, 1.0, seeds, pos, None)
        assert not np.array_equal(on, off)


def test_row_alone_equals_row_in_batch(dev):
    from adapcc_b200.ops.synthid import check_synthid_args

    rng = np.random.default_rng(8)
    cfg = check_synthid_args("t", dict(ngram_len=3, keys=KEYS9))
    R, t = 8, 20
    logits, gen = _logits(rng, R), rng.integers(0, V, (R, t))
    seeds, pos = rng.integers(0, 2 ** 62, R), rng.integers(0, 1000, R)
    for temperature, top_k, top_p in ((0.0, 0, 1.0), (1.0, 50, 0.9)):
        full = _sample(dev, logits, gen, temperature, top_k, top_p, seeds, pos, cfg)
        for r in range(R):
            one = _sample(dev, logits[r:r + 1].copy(), gen[r:r + 1], temperature, top_k, top_p, seeds[r:r + 1],
                          pos[r:r + 1], cfg)
            assert one[0] == full[r], r


def test_count_kernel_matches_reference_and_huggingface(dev):
    from adapcc_b200.ops import synthid_count_
    from adapcc_b200.ops.synthid import check_synthid_args, synthid_counts_reference, synthid_mask_reference

    rng = np.random.default_rng(3)
    B, T = 64, 1024
    for cfg in (dict(ngram_len=5, keys=KEYS9), dict(ngram_len=2, keys=[-1, 2 ** 63 - 1], context_history_size=7,
                                                    sampling_table_size=1000, sampling_table_seed=9)):
        cfg = check_synthid_args("t", cfg)
        ids = np.stack([rng.integers(0, (4, 50, V)[b % 3], T) for b in range(B)]).astype(np.int32)
        lens = rng.integers(0, T + 1, B)
        lens[:2] = T
        starts = rng.integers(0, 40, B)
        starts[:4] = 0
        i32 = dict(dtype=torch.int32, device=dev)
        for eos in (None, 3):
            got, g, mask = synthid_count_(torch.from_numpy(ids).to(dev), torch.as_tensor(lens, **i32),
                                          torch.as_tensor(starts, **i32), cfg, eos, with_g_values=True)
            want = synthid_counts_reference(ids, lens, starts, cfg, eos)
            assert np.array_equal(got.cpu().numpy(), want), (cfg, eos)
            gw, mw = synthid_mask_reference(ids, lens, starts, cfg, eos)
            assert np.array_equal(g.cpu().numpy(), gw) and np.array_equal(mask.cpu().numpy(), mw)
            assert want[:, 0].sum() > 0 and want[:, 1:].sum() > 0
        lp = pytest.importorskip("transformers.generation.logits_process")
        hf = lp.SynthIDTextWatermarkLogitsProcessor(cfg.ngram_len, list(cfg.keys), cfg.sampling_table_size,
                                                    cfg.sampling_table_seed, cfg.context_history_size, "cpu")
        x = torch.from_numpy(ids[:8]).long()
        _, g, mask = synthid_count_(torch.from_numpy(ids[:8]).to(dev), torch.full((8,), T, **i32),
                                    torch.zeros(8, **i32), cfg, 3, with_g_values=True)
        assert np.array_equal(g.cpu().numpy(), hf.compute_g_values(x).numpy())
        hm = hf.compute_context_repetition_mask(x) * hf.compute_eos_token_mask(x, 3)[:, cfg.ngram_len - 1:]
        assert np.array_equal(mask.cpu().numpy(), hm.numpy())


# ---- generate on GPT-2 small ------------------------------------------------------------------------------------------
SID = dict(ngram_len=4, keys=KEYS9)


def _gpt2_small(dev, seed=0):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(seed)
    return GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()


def _prompts(dev, B, T, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(0, 300, (B, T), device=dev, generator=g)


@pytest.mark.parametrize("mode", ["greedy", "sampled", "guided", "fp8"])
def test_generate_graph_equals_eager_loop(dev, mode):
    from adapcc_b200.ops import guidance_mix_, lm_head_logits_, sample_tokens_

    m = _gpt2_small(dev, seed=2)
    Vv = m.cfg.vocab_size
    B, n = 6, 24
    lengths = [90, 17, 64, 9, 120, 1]
    ids = _prompts(dev, B, 120, 5)
    temp, scale = (0.0, 1.0) if mode == "greedy" else (1.0, 1.5 if mode == "guided" else 1.0)
    kv = "fp8_e4m3" if mode == "fp8" else None
    kw = dict(max_new_tokens=n, temperature=temp, top_k=50 if mode == "sampled" else 0, top_p=0.95, seed=11,
              guidance_scale=scale, kv_cache_dtype=kv)
    free, _ = m.generate(ids, lengths, **kw)
    tokens, _ = m.generate(ids, lengths, **kw, watermarking_config=SID)
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
        want = torch.full((B, n), -1, dtype=torch.int64, device=dev)
        empty = torch.zeros(0, dtype=torch.int32, device=dev)
        for i in range(n):
            if i:
                h = m.decode_step(next_ids, None, cache)
            lm_head_logits_(h, w, logits)
            if mode == "guided":
                guidance_mix_(logits, Vv, B, scale)
            sample_tokens_(logits[:B], Vv, temp, kw["top_k"], 0.95, seeds, cache.lens[:B], step, 0, empty, empty, done,
                           next_ids[:B], want, synthid=SID)
            if mode == "guided":
                next_ids[B:].copy_(next_ids[:B])
    assert torch.equal(tokens, want), mode


def test_detection_power_and_false_alarms(dev):
    """Sampled 64-token replies of GPT-2 small (seeded random weights: near-uniform next-token distributions, where
    the tournament's signal is strongest) with m = 9 layers: at least 90 % are flagged at z > 4. Unwatermarked replies
    are flagged at most as often as a binomial tail allows with a per-row rate of ten times the normal tail at 4 (the
    margin covers the independence approximation of z); the bound holds with probability >= 1 - 1e-6."""
    from scipy.stats import binom, norm

    from adapcc_b200.ops.synthid import detect_synthid

    B, n = 32, 64
    m = _gpt2_small(dev, seed=5)
    ids = _prompts(dev, B, 16, 2)
    kw = dict(max_new_tokens=n, temperature=1.0, top_p=1.0, seed=3)
    tokens, n_new = m.generate(ids, **kw, watermarking_config=SID)
    assert (n_new == n).all()
    det = detect_synthid(tokens, SID, z_threshold=4.0)
    rate = float(det.prediction.mean())
    print(f"detection: {int(det.prediction.sum())} / {B} flagged at z > 4, mean z {np.nanmean(det.z_score):.2f}, "
          f"mean weighted score {np.nanmean(det.weighted_mean_score):.4f}")
    assert rate >= 0.9, det.z_score
    q = 10 * norm.sf(4.0)
    allowed = next(a for a in range(B + 1) if binom.sf(a, B, q) <= 1e-6)
    free, _ = m.generate(ids, **kw)
    det0 = detect_synthid(free, SID, z_threshold=4.0)
    assert int(det0.prediction.sum()) <= allowed, (det0.z_score, allowed)
    print(f"false alarms: {int(det0.prediction.sum())} of {B} unmarked rows, {allowed} allowed; "
          f"mean z {np.nanmean(det0.z_score):.2f}")


def test_launches_per_replay(dev):
    """SynthID runs inside the sampler's launch: ``generate`` issues as many launches with it as without."""
    from adapcc_b200.runtime.native import load_library

    lib = load_library(build_if_missing=False)
    m = _gpt2_small(dev, seed=6)
    ids = _prompts(dev, 4, 20, 3)

    def launches(**kw):
        c0 = lib.adapcc_launch_count()
        m.generate(ids, max_new_tokens=12, temperature=1.0, **kw)
        torch.cuda.synchronize()
        return lib.adapcc_launch_count() - c0

    assert launches(watermarking_config=SID) == launches()
