"""Green-list watermarking on the CPU: the keyed hash against a scalar loop over ``philox4x32_10``, the statistics of
the green lists, what the lefthash and selfhash lists depend on, detector counts on hand-built sequences, the four
decoders' CPU paths against explicit loops with ``watermark_reference``, the exact all-green property of greedy
decoding at a large bias, argument errors, the ConvAI pass-through and the build log."""
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.sampling import philox4x32_10  # noqa: E402
from adapcc_b200.ops.watermark import (TAG_CTX, TAG_GREEN, TAG_SELF, WatermarkingConfig,  # noqa: E402
                                       check_watermark_args, detect_watermark, green_ids, watermark_counts_reference,
                                       watermark_reference)

M32 = 0xFFFFFFFF


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _bits(t):
    return t.contiguous().view(torch.int32)


# ---- the definition in Python integers ------------------------------------------------------------------------------
def _green_scalar(v, s0, s1, theta):
    return philox4x32_10((v, 0, 0, TAG_GREEN), (s0, s1))[0] < theta


def _left_seed_scalar(seq, cfg):
    s0, s1 = cfg.hashing_key & M32, cfg.hashing_key >> 32
    for i in range(1, cfg.context_width + 1):
        s0, s1 = philox4x32_10((seq[-i], i, 0, TAG_CTX), (s0, s1))[:2]
    return s0, s1


def _self_green_scalar(v, win, cfg):
    k = (cfg.hashing_key & M32, cfg.hashing_key >> 32)

    def h(x):
        x, y = philox4x32_10((x, v, 0, TAG_SELF), k)[:2]
        return (y << 32) | x

    m = min(h(x) for x in list(win) + [v])
    return _green_scalar(v, m & M32, m >> 32, cfg.threshold)


def _scalar_mask(seq, vocab, cfg):
    w = cfg.context_width
    if cfg.selfhash:
        win = seq[len(seq) - w + 1:] if w > 1 else []
        return np.array([_self_green_scalar(v, win, cfg) for v in range(vocab)])
    s0, s1 = _left_seed_scalar(seq, cfg)
    return np.array([_green_scalar(v, s0, s1, cfg.threshold) for v in range(vocab)])


def test_vectorised_green_test_equals_scalar_philox_loop():
    rng = np.random.default_rng(0)
    for scheme, w, gamma, key in (("lefthash", 1, 0.25, 15485863), ("lefthash", 3, 0.5, 2 ** 64 - 1),
                                  ("selfhash", 1, 0.25, 7), ("selfhash", 4, 0.1, 2 ** 40 + 3),
                                  ("lefthash", 8, 0.9, 0)):
        cfg = check_watermark_args("t", dict(seeding_scheme=scheme, context_width=w, greenlist_ratio=gamma,
                                             hashing_key=key))
        for _ in range(2):
            seq = rng.integers(0, 50257, 12).tolist()
            got = green_ids(seq, 300, cfg)
            assert np.array_equal(got, _scalar_mask(seq, 300, cfg)), (scheme, w)


def test_green_counts_are_binomial():
    cfg = check_watermark_args("t", WatermarkingConfig(greenlist_ratio=0.25))
    V, g = 50257, cfg.gamma_eff
    sd = math.sqrt(V * g * (1 - g))
    counts = [int(green_ids([t], V, cfg).sum()) for t in range(200)]
    assert all(abs(c - V * g) <= 6 * sd for c in counts), (min(counts), max(counts))
    assert len(set(counts)) > 100                                  # 200 different lists, not one
    assert abs(np.mean(counts) - V * g) <= 6 * sd / math.sqrt(200)


def test_lefthash_depends_only_on_the_last_w_ids():
    rng = np.random.default_rng(1)
    for w in (1, 2, 5):
        cfg = check_watermark_args("t", dict(context_width=w))
        tail = rng.integers(0, 1000, w).tolist()
        ref = green_ids(tail, 2000, cfg)
        for _ in range(3):
            assert np.array_equal(green_ids(rng.integers(0, 1000, 7).tolist() + tail, 2000, cfg), ref)
        other = list(tail)
        other[0] += 1                                              # the oldest id of the window counts
        assert not np.array_equal(green_ids(other, 2000, cfg), ref)
        assert green_ids(tail[1:], 2000, cfg) is None              # shorter than w: no list, the row is unchanged


def test_selfhash_at_width_one_ignores_the_context():
    cfg = check_watermark_args("t", dict(seeding_scheme="selfhash", context_width=1))
    ref = green_ids([], 3000, cfg)
    for seq in ([5], [9, 1, 2], list(range(40))):
        assert np.array_equal(green_ids(seq, 3000, cfg), ref)
    wide = check_watermark_args("t", dict(seeding_scheme="selfhash", context_width=3))
    assert green_ids([4], 3000, wide) is None
    assert not np.array_equal(green_ids([4, 5], 3000, wide), green_ids([4, 6], 3000, wide))


def test_reference_bias_rule():
    cfg = check_watermark_args("t", dict(bias=1.5, context_width=2))
    V, LD = 700, 704
    x = np.random.default_rng(2).standard_normal((3, LD)).astype(np.float32) * 4
    x[0, :8] = [0.0, -0.0, 1e-40, -1e-40, -np.inf, 3e38, -3e38, 1.4e-45]
    seqs = [[3, 9, 1], [4], [7, 7]]
    out = watermark_reference(torch.from_numpy(x), seqs, V, cfg).numpy()
    assert np.array_equal(out[:, V:].view(np.int32), x[:, V:].view(np.int32))      # columns from vocab on
    assert np.array_equal(out[1].view(np.int32), x[1].view(np.int32))              # too short: unchanged
    for r in (0, 2):
        g = _scalar_mask(seqs[r], V, cfg)
        assert np.array_equal(out[r, :V][~g].view(np.int32), x[r, :V][~g].view(np.int32))
        assert np.array_equal(out[r, :V][g], (x[r, :V][g] + np.float32(1.5)).astype(np.float32))
    assert out[0, 4] == -np.inf


# ---- detection ------------------------------------------------------------------------------------------------------
def _pos_green(seq, j, cfg):
    w = cfg.context_width
    if cfg.selfhash:
        return _self_green_scalar(seq[j], seq[j - w + 1:j] if w > 1 else [], cfg)
    return _green_scalar(seq[j], *_left_seed_scalar(seq[:j], cfg), cfg.threshold)


def test_detector_counts_on_hand_built_sequences():
    a, b, c, d = 11, 22, 33, 44
    rows = [[a, b, a, b, a, b, c, d], [a, b, c, a, b, c, 0, 0], [d, d, d, d, d, 0, 0, 0], [c, 0, 0, 0, 0, 0, 0, 0]]
    lengths = [8, 6, 5, 1]
    for scheme, w in (("lefthash", 1), ("lefthash", 2), ("selfhash", 1), ("selfhash", 2)):
        cfg = check_watermark_args("t", dict(seeding_scheme=scheme, context_width=w))
        first = w - int(cfg.selfhash)
        n_gram = w + 1 - int(cfg.selfhash)
        for starts in ([0, 0, 0, 0], [3, 2, 0, 1]):
            for ignore in (False, True):
                want = []
                for r, L, st in zip(rows, lengths, starts):
                    pos = list(range(max(st, first), L))
                    if ignore:                                     # the hand list of first occurrences
                        seen, keep = set(), []
                        for j in pos:
                            if tuple(r[j - n_gram + 1:j + 1]) not in seen:
                                seen.add(tuple(r[j - n_gram + 1:j + 1]))
                                keep.append(j)
                        pos = keep
                    want.append((len(pos), sum(_pos_green(r, j, cfg) for j in pos)))
                got = watermark_counts_reference(np.array(rows), lengths, starts, cfg, ignore)
                assert [tuple(x) for x in got.tolist()] == want, (scheme, w, starts, ignore)
        # the distinct n-grams of the rows, counted by hand for lefthash w = 1 (bigrams) from position 0
        if (scheme, w) == ("lefthash", 1):
            got = watermark_counts_reference(np.array(rows), lengths, [0] * 4, cfg, True)[:, 0].tolist()
            assert got == [4, 3, 1, 0]        # (a,b) (b,a) (b,c) (c,d); (a,b) (b,c) (c,a); (d,d); none
            got = watermark_counts_reference(np.array(rows), lengths, [0] * 4, cfg, False)[:, 0].tolist()
            assert got == [7, 5, 4, 0]


def test_detect_watermark_statistics():
    cfg = WatermarkingConfig()
    rng = np.random.default_rng(3)
    ids = torch.from_numpy(rng.integers(0, 50257, (4, 40)))
    det = detect_watermark(ids, cfg, lengths=[40, 30, 1, 0], scored_from=[0, 5, 0, 0])
    counts = watermark_counts_reference(ids, [40, 30, 1, 0], [0, 5, 0, 0], cfg)
    assert det.num_tokens_scored.tolist() == [39, 25, 0, 0] == counts[:, 0].tolist()
    assert det.num_green_tokens.tolist() == counts[:, 1].tolist()
    g = cfg.gamma_eff
    for r in range(2):
        n, k = det.num_tokens_scored[r], det.num_green_tokens[r]
        z = (k - g * n) / math.sqrt(n * g * (1 - g))
        assert det.z_score[r] == z and det.p_value[r] == 0.5 * math.erfc(z / math.sqrt(2))
        assert det.green_fraction[r] == k / n and det.prediction[r] == (z > 3.0)
    assert np.isnan(det.z_score[2:]).all() and not det.prediction[2:].any()
    # a fully green text is flagged
    seq = [5]
    cfg1 = check_watermark_args("t", cfg)
    for _ in range(30):
        seq.append(int(np.flatnonzero(green_ids(seq, 500, cfg1))[0]))
    det = detect_watermark(torch.tensor([seq]), cfg, z_threshold=4.0)
    assert det.num_green_tokens[0] == det.num_tokens_scored[0] == 30 and det.prediction[0]


# ---- the decoders -------------------------------------------------------------------------------------------------
WMS = (dict(bias=3.0), dict(bias=2.0, seeding_scheme="selfhash", context_width=3, greenlist_ratio=0.5),
       WatermarkingConfig(bias=1.0, context_width=2, hashing_key=2 ** 63 + 5))


def test_greedy_generate_equals_uncached_reference_loop(tiny):
    """Teacher-forced on ``generate``'s own tokens: at every step the arg-max of the uncached model's logits after the
    reference rules is the token ``generate`` chose (up to a near tie of the two paths' fp32 logits)."""
    from adapcc_b200.ops.repeats import penalize_repeats_reference

    g = torch.Generator().manual_seed(5)
    V, n = tiny.cfg.vocab_size, 14
    lengths = [12, 5, 1]
    ids = torch.randint(0, V, (3, 12), generator=g)
    free, _ = tiny.generate(ids, lengths, max_new_tokens=n, temperature=0.0)
    for wm in WMS:
        for rp in (1.0, 1.3):
            tokens, n_new = tiny.generate(ids, lengths, max_new_tokens=n, temperature=0.0, watermarking_config=wm,
                                          repetition_penalty=rp)
            assert n_new.tolist() == [n] * 3
            for b, x in enumerate(lengths):
                seq = ids[b, :x].tolist()
                for i in range(n):
                    with torch.no_grad():
                        logits = tiny.lm_logits(tiny.hidden(torch.tensor([seq]), None)[0, -1])[None]
                    lc = penalize_repeats_reference(logits, [seq], V, rp, 0)
                    lc = watermark_reference(lc, [seq], V, wm)[0]
                    want, got = int(lc.argmax()), int(tokens[b, i])
                    if want != got:
                        assert float(lc[want] - lc[got]) <= 1e-4, (wm, b, i, want, got)
                    seq.append(got)
            assert not torch.equal(tokens, free), wm


def _decoders(tiny, ids, lengths, n=10, **kw):
    out = []
    out.append(("generate", *tiny.generate(ids, lengths, max_new_tokens=n, temperature=1.0, top_p=1.0, seed=3, **kw)))
    out.append(("generate greedy", *tiny.generate(ids, lengths, max_new_tokens=n, temperature=0.0, **kw)))
    out.append(("generate guided", *tiny.generate(ids, lengths, max_new_tokens=n, temperature=1.0, seed=3,
                                                  guidance_scale=1.5, **kw)))
    out.append(("beam", *tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=n, num_return_sequences=3,
                                          **kw)))
    out.append(("beam sampled", *tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=n, do_sample=True, seed=5,
                                                  **kw)))
    out.append(("beam groups", *tiny.beam_search(ids, lengths, num_beams=4, num_beam_groups=2, diversity_penalty=0.5,
                                                 max_new_tokens=n, **kw)))
    out.append(("stochastic beam", *tiny.stochastic_beam_search(ids, lengths, num_beams=3, max_new_tokens=n, seed=2,
                                                                **kw)))
    out.append(("contrastive", *tiny.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.6, max_new_tokens=n,
                                                        **kw)))
    return out


def test_every_decoder_equals_its_loop_with_the_reference_rule(tiny, monkeypatch):
    """Each decoder's CPU path with a watermark against the same eager loop run without it, the reference rule applied
    explicitly after the repetition rules to every row's own sequence (a zero sequence bias keeps the rule pass on):
    every output equal, bit for bit."""
    import adapcc_b200.models.gpt2 as gpt2

    g = torch.Generator().manual_seed(7)
    lengths = [9, 4, 1]
    ids = torch.randint(0, tiny.cfg.vocab_size, (3, 9), generator=g)
    free = _decoders(tiny, ids, lengths)
    orig = gpt2.penalize_repeats_reference
    for wm in WMS:
        got = _decoders(tiny, ids, lengths, watermarking_config=wm)
        seen = []

        def explicit(logits, seqs, vocab, *a, _wm=wm, **k):
            seen.append(len(seqs))
            return watermark_reference(orig(logits, seqs, vocab, *a, **k), seqs, vocab, _wm)

        monkeypatch.setattr(gpt2, "penalize_repeats_reference", explicit)
        want = _decoders(tiny, ids, lengths, sequence_bias={(0,): 0.0})
        monkeypatch.setattr(gpt2, "penalize_repeats_reference", orig)
        assert seen
        changed = 0
        for (name, *a), (_, *b), (_, *f) in zip(got, want, free):
            assert all(torch.equal(_bits(x) if x.is_floating_point() else x,
                                   _bits(y) if y.is_floating_point() else y) for x, y in zip(a, b)), (wm, name)
            changed += not torch.equal(a[0], f[0])
        assert changed >= 6, wm


def test_large_bias_makes_every_scored_token_green(tiny):
    """Greedy decoding with δ larger than the range of the logits: every id it picks is green, so the detector finds
    g = n, over the reply with the prompt as context, for every scheme."""
    g = torch.Generator().manual_seed(11)
    lengths = [10, 3, 1, 6]
    ids = torch.randint(0, tiny.cfg.vocab_size, (4, 10), generator=g)
    for wm in (dict(bias=1e4), dict(bias=1e4, seeding_scheme="selfhash", context_width=4),
               dict(bias=1e4, context_width=3, greenlist_ratio=0.1)):
        for call in (lambda: tiny.generate(ids, lengths, max_new_tokens=16, temperature=0.0, watermarking_config=wm),
                     lambda: tiny.contrastive_search(ids, lengths, max_new_tokens=16, watermarking_config=wm)):
            tokens, n_new = call()
            seqs = [ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist() for b, x in enumerate(lengths)]
            T = max(map(len, seqs))
            det = detect_watermark(torch.tensor([s + [0] * (T - len(s)) for s in seqs]), wm,
                                   lengths=[len(s) for s in seqs], scored_from=lengths)
            assert (det.num_tokens_scored > 0).all()
            assert np.array_equal(det.num_green_tokens, det.num_tokens_scored), wm


def test_argument_errors(tiny):
    ids = torch.zeros(2, 5, dtype=torch.long)
    cases = [(dict(greenlist_ratio=0.0), "greenlist_ratio"), (dict(greenlist_ratio=1.0), "greenlist_ratio"),
             (dict(greenlist_ratio=1e-12), "greenlist_ratio"), (dict(greenlist_ratio=1 - 1e-12), "greenlist_ratio"),
             (dict(greenlist_ratio="0.5"), "greenlist_ratio"), (dict(greenlist_ratio=float("nan")), "greenlist_ratio"),
             (dict(bias=float("inf")), "bias"), (dict(bias=1e39), "bias"), (dict(bias=None), "bias"),
             (dict(seeding_scheme="minhash"), "seeding_scheme"), (dict(context_width=0), "context_width"),
             (dict(context_width=9), "context_width"), (dict(context_width=1.5), "context_width"),
             (dict(context_width=True), "context_width"), (dict(hashing_key=-1), "hashing_key"),
             (dict(hashing_key=2 ** 64), "hashing_key"), (dict(hashing_key=1.0), "hashing_key"),
             (dict(colour="green"), "unknown keys")]
    for kw, name in cases:
        for wm in (kw, None if "colour" in kw else WatermarkingConfig(**kw)):
            if wm is None:
                continue
            for call in (lambda: tiny.generate(ids, max_new_tokens=2, watermarking_config=wm),
                         lambda: tiny.beam_search(ids, num_beams=2, max_new_tokens=2, watermarking_config=wm),
                         lambda: tiny.stochastic_beam_search(ids, num_beams=2, max_new_tokens=2,
                                                             watermarking_config=wm),
                         lambda: tiny.contrastive_search(ids, max_new_tokens=2, watermarking_config=wm),
                         lambda: detect_watermark(ids, wm)):
                with pytest.raises(ValueError, match=name):
                    call()
    for bad in ("lefthash", 3, [1]):
        with pytest.raises(ValueError, match="watermarking_config"):
            tiny.generate(ids, max_new_tokens=2, watermarking_config=bad)
    # both forms are accepted and mean the same thing; an empty dict is the defaults
    a = tiny.generate(ids, max_new_tokens=3, temperature=0.0, watermarking_config=dict(bias=5.0, context_width=2))
    b = tiny.generate(ids, max_new_tokens=3, temperature=0.0,
                      watermarking_config=WatermarkingConfig(bias=5.0, context_width=2))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert check_watermark_args("t", {}) == WatermarkingConfig()
    # with prompt lookup or an assistant
    with pytest.raises(ValueError, match="cannot be combined with prompt_lookup_num_tokens or assistant_model"):
        tiny.generate(ids, max_new_tokens=2, temperature=0.0, prompt_lookup_num_tokens=2, watermarking_config={})
    with pytest.raises(ValueError, match="cannot be combined with prompt_lookup_num_tokens or assistant_model"):
        tiny.generate(ids, max_new_tokens=2, assistant_model=tiny, watermarking_config={})
    # the detector's own arguments
    for kw, name in ((dict(lengths=[6, 1]), "lengths"), (dict(scored_from=-1), "scored_from"),
                     (dict(scored_from=[0]), "scored_from"), (dict(ignore_repeated_ngrams=1), "ignore_repeated"),
                     (dict(z_threshold=float("nan")), "z_threshold")):
        with pytest.raises(ValueError, match=name):
            detect_watermark(ids, {}, **kw)
    with pytest.raises(ValueError, match="input_ids"):
        detect_watermark(ids[0], {})
    with pytest.raises(ValueError, match="config"):
        detect_watermark(ids, None)
    # the ops validate before they load or launch anything
    from adapcc_b200.ops import watermark_, watermark_count_

    i32 = dict(dtype=torch.int32)
    with pytest.raises(ValueError, match="watermark_: bias"):
        watermark_(torch.zeros(2, 8), 8, torch.zeros(2, 4, **i32), torch.ones(2, **i32), dict(bias=float("nan")))
    with pytest.raises(ValueError, match="watermark_: seq"):
        watermark_(torch.zeros(2, 8), 8, torch.zeros(2, 2000, **i32), torch.ones(2, **i32), {})
    with pytest.raises(ValueError, match="watermark_count_: ids"):
        watermark_count_(torch.zeros(2, 4), torch.ones(2, **i32), torch.zeros(2, **i32), {})


def test_defaults_run_nothing_new(tiny, monkeypatch):
    import adapcc_b200.models.gpt2 as gpt2

    def boom(*a, **k):
        raise AssertionError("the watermark ran while off")

    ids = torch.randint(0, tiny.cfg.vocab_size, (2, 9), generator=torch.Generator().manual_seed(0))
    want = tiny.generate(ids, max_new_tokens=6, temperature=0.0)
    monkeypatch.setattr(gpt2, "watermark_reference", boom)
    monkeypatch.setattr(gpt2, "penalize_repeats_reference", boom)
    got = tiny.generate(ids, max_new_tokens=6, temperature=0.0, watermarking_config=None)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    with pytest.raises(AssertionError):
        tiny.generate(ids, max_new_tokens=2, watermarking_config={})


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_convai_passes_the_watermark_through(tiny, monkeypatch):
    from adapcc_b200.eval import convai

    wm = dict(bias=8.0, context_width=1)
    seen = []
    for name in ("generate", "beam_search", "contrastive_search"):
        orig = getattr(tiny, name)

        def spy(*a, _orig=orig, _name=name, **k):
            seen.append((_name, k.get("watermarking_config")))
            return _orig(*a, **k)
        monkeypatch.setattr(tiny, name, spy)
    dialogs = [([[1, 2]], [[3, 4, 5, 3, 4]]), ([[6]], [[7], [8, 9]])]
    for extra in (dict(num_beams=0), dict(num_beams=2), dict(penalty_alpha=0.5, top_k=3)):
        assert len(convai.sample_replies(tiny, _Tok(), dialogs, max_length=6, no_sample=True,
                                         watermarking_config=wm, **extra)) == 2
    assert seen == [("generate", wm), ("beam_search", wm), ("contrastive_search", wm)]
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]},
                                                        {"history": ["hi", "so"], "candidates": ["a", "b c"]}]}]
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", watermarking_config=wm, max_length=12, min_length=12)
    assert r["examples"] == 2 and 0.0 <= r["f1"] <= 1.0
    assert r["watermark_z"] > 2 and r["watermark_detected"] >= 0.5
    assert "watermark_z" not in convai.evaluate_dialogs(tiny, _Tok(), d, "f1", batch_size=2)


def test_example_has_the_flags():
    src = open(os.path.join(ROOT, "examples", "eval_gpt2_convai.py")).read()
    for flag in ("--watermark_bias", "--watermark_ratio", "--watermark_scheme", "--watermark_context_width"):
        assert f'"{flag}"' in src


def test_build_log_shows_watermark_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_watermark\.cu", log)
    for kernel in ("watermark_kernel", "watermark_count_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
