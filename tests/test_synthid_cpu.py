"""SynthID Text watermarking on the CPU: the table, g-values and masks against HuggingFace's processor, the fp64
tournament against its ``update_scores``, the skipped and repeated steps against its ``__call__`` state, greedy
``generate`` against HuggingFace's, the tournament's unbiasedness, argument errors, the ConvAI report and the build
log."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.sampling import reference_row  # noqa: E402
from adapcc_b200.ops.synthid import (SynthIDTextWatermarkingConfig, accumulate, check_synthid_args,  # noqa: E402
                                     detect_synthid, g_values, sampling_table, synthid_counts_reference, synthid_flags,
                                     synthid_g_values, synthid_mask_reference, synthid_scores, tournament)

KEYS = (654, 400, 836, 123, 340, 443, 597, 160, 57)


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _hf_processor(cfg):
    lp = pytest.importorskip("transformers.generation.logits_process")
    return lp.SynthIDTextWatermarkLogitsProcessor(
        ngram_len=cfg.ngram_len, keys=list(cfg.keys), sampling_table_size=cfg.sampling_table_size,
        sampling_table_seed=cfg.sampling_table_seed, context_history_size=cfg.context_history_size, device="cpu",
        skip_first_ngram_calls=cfg.skip_first_ngram_calls)


@pytest.mark.parametrize("n,keys,size,hist", [(5, KEYS, 2 ** 16, 1024), (3, (-7, 2 ** 63 - 1, -2 ** 63), 1000, 4),
                                              (2, (1,), 37, 2)])
def test_table_g_values_and_masks_match_huggingface(n, keys, size, hist):
    cfg = check_synthid_args("t", SynthIDTextWatermarkingConfig(n, keys, hist, 3, size))
    hf = _hf_processor(cfg)
    assert np.array_equal(hf.sampling_table.numpy(), sampling_table(cfg))
    g = torch.Generator().manual_seed(n)
    ids = torch.randint(0, 30, (4, 60), generator=g)
    ids[1, 20:35] = ids[1, :15]                                   # repeated contexts
    ids[2, 40] = 5                                                # an EOS
    gm, mask = synthid_mask_reference(ids, [60] * 4, [0] * 4, cfg, eos_token_id=5)
    assert np.array_equal(hf.compute_g_values(ids).numpy(), gm)
    want = hf.compute_context_repetition_mask(ids).numpy() * hf.compute_eos_token_mask(ids, 5).numpy()[:, n - 1:]
    assert np.array_equal(want, mask)
    gt, mt = synthid_g_values(ids, cfg, eos_token_id=5)
    assert torch.equal(gt, torch.from_numpy(gm)) and torch.equal(mt, torch.from_numpy(mask))


def test_tournament_matches_update_scores():
    hf = _hf_processor(check_synthid_args("t", SynthIDTextWatermarkingConfig(4, KEYS)))
    g = torch.Generator().manual_seed(1)
    scores = torch.randn(3, 500, generator=g) * 3
    scores[:, 100:200] = -float("inf")
    gv = torch.randint(0, 2, (3, 500, 9), generator=g)
    want = torch.exp(hf.update_scores(scores, gv.float()))
    for b in range(3):
        p = torch.softmax(scores[b].double(), 0).numpy()
        got = tournament(p, gv[b].numpy())
        np.testing.assert_allclose(got, want[b].double().numpy(), rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("skip,hist", [(False, 1024), (True, 1024), (True, 3), (False, 2)])
def test_skipped_and_repeated_steps_follow_the_processor(skip, hist):
    cfg = check_synthid_args("t", SynthIDTextWatermarkingConfig(3, KEYS[:3], hist, skip_first_ngram_calls=skip))
    hf = _hf_processor(cfg)
    g = torch.Generator().manual_seed(int(skip) * 10 + hist)
    B, V, steps = 3, 6, 40
    prompt = torch.randint(0, V, (B, 4), generator=g)
    gen = torch.randint(0, V, (B, steps), generator=g)
    gen[1] = gen[1] % 2                                           # a row that repeats its contexts often
    seen = {"skipped", "repeated", "watermarked"}
    kinds = set()
    for t in range(steps):
        ids = torch.cat([prompt, gen[:, :t]], 1)
        scores = torch.randn(B, V, generator=g)
        out = hf(ids, scores.clone())
        for b in range(B):
            kind, _ = synthid_flags(gen[b, :t], cfg)
            kinds.add(kind)
            assert torch.equal(out[b], scores[b]) == (kind != "watermarked"), (t, b, kind)
    assert kinds <= seen and "watermarked" in kinds and "repeated" in kinds
    assert ("skipped" in kinds) == skip


def test_greedy_generate_matches_huggingface(tiny):
    transformers = pytest.importorskip("transformers")
    from test_repeats_cpu import _hf_model

    _, hf = _hf_model(tiny)
    n = 24
    g = torch.Generator().manual_seed(3)
    for trial, (ng, keys, skip) in enumerate([(5, KEYS, False), (3, KEYS[:4], True), (2, (11, 12), False)]):
        prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 10), generator=g)
        hf_cfg = transformers.SynthIDTextWatermarkingConfig(ngram_len=ng, keys=list(keys),
                                                            skip_first_ngram_calls=skip)
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), do_sample=False, max_new_tokens=n,
                               min_new_tokens=n, eos_token_id=None, pad_token_id=0,
                               watermarking_config=hf_cfg)[0, prompt.shape[1]:]
        cfg = dict(ngram_len=ng, keys=list(keys), skip_first_ngram_calls=skip)
        got, _ = tiny.generate(prompt, max_new_tokens=n, temperature=0, watermarking_config=cfg)
        plain, _ = tiny.generate(prompt, max_new_tokens=n, temperature=0)
        assert torch.equal(got[0], want), trial
        assert not torch.equal(got[0], plain[0]), trial


def test_reference_row_steps():
    cfg = check_synthid_args("t", SynthIDTextWatermarkingConfig(3, KEYS))
    g = np.random.default_rng(0)
    x = g.standard_normal(300).astype(np.float32)
    gen = [5, 6, 7, 8]
    off = reference_row(x, 0.8, 50, 0.9, seed=4, pos=9)
    on = reference_row(x, 0.8, 50, 0.9, seed=4, pos=9, synthid=cfg, generated=gen)
    assert on["synthid"] == "watermarked"
    assert np.array_equal(on["p"] > 0, off["kept"]) and np.isclose(on["synthid_p"].sum(), 1.0)
    assert set(np.flatnonzero(on["synthid_p"] > 0)) <= set(np.flatnonzero(off["kept"]))
    rep = reference_row(x, 0.8, 50, 0.9, seed=4, pos=9, synthid=cfg, generated=[1, 2, 1, 2, 1])
    assert rep["synthid"] == "repeated" and rep["token"] == off["token"] and "synthid_p" not in rep


def test_tournament_is_unbiased_over_keys():
    g = np.random.default_rng(1)
    V, trials = 12, 3000
    p = g.dirichlet(np.ones(V))
    acc = np.zeros(V)
    for t in range(trials):
        keys = tuple(int(k) for k in g.integers(-2 ** 62, 2 ** 62, 4))
        cfg = check_synthid_args("t", SynthIDTextWatermarkingConfig(2, keys, sampling_table_seed=t % 5))
        gv = g_values(np.uint64(int(accumulate(1, [7]))), np.arange(V), cfg)
        acc += tournament(p, gv)
    mean = acc / trials
    # p'_i lies in [0, 2^4 p_i]; a binomial-style bound of 5 sigma on its mean with variance <= E[p'^2] <= 16 p_i^2
    sigma = np.sqrt(16 * p ** 2 / trials)
    assert np.all(np.abs(mean - p) < 5 * sigma + 1e-12), (mean, p)


def test_detection_statistics():
    cfg = check_synthid_args("t", SynthIDTextWatermarkingConfig(2, (1, 2, 3)))
    out = synthid_scores([[10, 10, 0, 5], [0, 0, 0, 0]], 0.5)
    w = np.linspace(10, 1, 3) * 3 / np.linspace(10, 1, 3).sum()
    assert out.mean_score[0] == pytest.approx(15 / 30)
    assert out.weighted_mean_score[0] == pytest.approx((10 * w[0] + 5 * w[2]) / 30)
    assert out.z_score[0] == pytest.approx(0.0) and np.isnan(out.z_score[1]) and not out.prediction[1]
    ids = torch.tensor([[1, 2, 3, 4, 1, 2, 9, 0], [5, 6, 7, 8, 9, 10, 11, 12]])
    c = synthid_counts_reference(ids, [7, 8], [0, 3], cfg)
    gv, mask = synthid_mask_reference(ids, [7, 8], [0, 3], cfg)
    assert list(mask[0]) == [1, 1, 1, 1, 0, 0, 0] and list(mask[1]) == [0, 0, 1, 1, 1, 1, 1]
    assert list(c[:, 0]) == [4, 5] and np.array_equal(c[:, 1:], (gv * mask[:, :, None]).sum(1))
    det = detect_synthid(ids, cfg, lengths=[7, 8], scored_from=[0, 3])
    assert list(det.num_tokens_scored) == [4, 5]


def test_argument_errors(tiny):
    good = dict(ngram_len=3, keys=[1, 2])
    for bad, what in [(dict(good, ngram_len=1), "ngram_len"), (dict(good, ngram_len=17), "ngram_len"),
                      (dict(good, keys=[]), "keys"), (dict(good, keys=list(range(65))), "keys"),
                      (dict(good, keys=[2 ** 63]), "int64"), (dict(good, context_history_size=0), "context_history"),
                      (dict(good, sampling_table_size=2 ** 24 + 1), "sampling_table_size"),
                      (dict(good, sampling_table_size=0), "sampling_table_size"),
                      (dict(good, sampling_table_seed=2 ** 64), "sampling_table_seed"),
                      (dict(good, debug_mode=True), "debug_mode"), (dict(good, colour=1), "unknown"),
                      (dict(keys=[1]), "ngram_len")]:
        with pytest.raises(ValueError, match=what):
            check_synthid_args("t", bad)
    prompt = torch.tensor([[1, 2, 3]])
    for name, extra in (("beam_search", {}), ("stochastic_beam_search", {}),
                        ("contrastive_search", dict(penalty_alpha=0.5, top_k=3))):
        with pytest.raises(ValueError, match="SynthID"):
            getattr(tiny, name)(prompt, max_new_tokens=2, watermarking_config=good, **extra)
    with pytest.raises(ValueError, match="unknown keys"):
        tiny.generate(prompt, max_new_tokens=2, watermarking_config=dict(colour="green"))
    with pytest.raises(ValueError, match="watermarking_config"):
        tiny.generate(prompt, max_new_tokens=2, prompt_lookup_num_tokens=2, temperature=0, watermarking_config=good)
    with pytest.raises(ValueError, match="ngram_len"):
        detect_synthid(torch.tensor([[1, 2]]), good)


def test_convai_reports_synthid_score(tiny):
    from adapcc_b200.eval import convai
    from test_watermark_cpu import _Tok

    cfg = dict(ngram_len=2, keys=list(KEYS))
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]},
                                                        {"history": ["hi", "so"], "candidates": ["a", "b c"]}]}]
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", watermarking_config=cfg, max_length=12, min_length=12)
    assert r["examples"] == 2 and 0.0 <= r["f1"] <= 1.0
    assert 0.0 <= r["synthid_score"] <= 1.0 and 0.0 <= r["synthid_detected"] <= 1.0
    assert "watermark_z" not in r


def test_build_log_shows_synthid_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_synthid\.cu", log)
    for kernel in ("synthid_count_kernel", "sample_tokens_synthid_kernel", "synthid_tournament"):
        hits = re.findall(r"(?:Compiling entry function|Function properties for) '?(\w*%s\w*)" % kernel, log)
        assert hits, kernel
        for name in set(hits):
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
