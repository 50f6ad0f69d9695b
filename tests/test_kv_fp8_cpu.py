"""The fp8 (e4m3) KV cache without a GPU: the reference quantizer of ``ops/kvcache.py``, the cache plumbing of the tiny
model against a full-precision cache holding the dequantized values, the decoders on an fp8 cache, the argument
errors, and the build log of the fp8 kernels."""
import os
import re

import pytest
import torch

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
from adapcc_b200.ops.kvcache import dequantize, quantize

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP8 = "fp8_e4m3"


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def test_scales_are_powers_of_two_that_put_amax_in_128_256():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(200, 64, generator=g) * torch.logspace(-35, 35, 200)[:, None]
    x = x.to(torch.bfloat16)
    q, s = quantize(x)
    m, e = torch.frexp(s.double())
    assert bool((m == 0.5).all())                            # exact powers of two
    amax = x.double().abs().amax(-1)
    r = amax / s.double()
    assert bool(((r >= 128) & (r < 256)).all())
    # the read value is within half an e4m3 step of x, and exact in bf16
    d = dequantize(q, s)
    assert bool(((d.double() - x.double()).abs() <= amax[:, None] * 2.0 ** -4).all())
    assert torch.equal(d.to(torch.bfloat16).float(), d)


def test_ties_round_to_even_and_grid_values_round_trip():
    # amax 255: e = 0, so the values are quantized as they are
    x = torch.tensor([[136.0, 152.0, 9.5, 10.5, 2.0 ** -10, 3 * 2.0 ** -10, -200.0, 255.0]])
    q, s = quantize(x.to(torch.bfloat16))
    assert float(s) == 1.0
    assert dequantize(q, s).tolist() == [[128.0, 160.0, 10.0, 10.0, 0.0, 2.0 ** -8, -192.0, 256.0]]
    # every finite e4m3 value times a power of two comes back exactly when the vector's amax sets that power
    grid = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).float()
    grid = grid[torch.isfinite(grid) & (grid.abs() < 256)]
    for p in (-20, 0, 9):
        x = torch.cat([grid, torch.tensor([240.0])]) * 2.0 ** p      # 240: amax in [128, 256)
        q, s = quantize(x.to(torch.bfloat16)[None])
        assert float(s) == 2.0 ** p and torch.equal(dequantize(q, s)[0], x)


def test_zero_and_non_finite_vectors():
    x = torch.zeros(3, 16, dtype=torch.bfloat16)
    x[1, 4] = float("nan")
    x[2, 0] = float("-inf")
    x[2, 1] = 1.0
    q, s = quantize(x)
    assert float(s[0]) == 1.0 and bool((q == 0).all())
    assert bool(s[1:].isnan().all())
    assert bool(dequantize(q, s)[1:].isnan().all())


def test_teacher_forced_fp8_cache_is_full_cache_of_dequantized_values(tiny):
    """Before every step the full-precision cache is overwritten with the fp8 cache's dequantized contents; both then
    decode the same token and give the same hidden states."""
    m = tiny
    g = torch.Generator().manual_seed(1)
    B, T, n = 3, 9, 8
    lengths = [9, 4, 1]
    ids = torch.randint(0, m.cfg.vocab_size, (B, T + n), generator=g)
    c8, cf = m.new_cache(B, T + n, FP8), m.new_cache(B, T + n)
    assert c8.k.dtype == torch.uint8 and c8.k_scale.shape == c8.k.shape[:4] and cf.k_scale is None
    with torch.no_grad():
        assert torch.equal(m.hidden(ids[:, :T], None, cache=c8, lengths=lengths),
                           m.hidden(ids[:, :T], None, cache=cf, lengths=lengths))
        for full, q, s in ((cf.k, c8.k, c8.k_scale), (cf.v, c8.v, c8.v_scale)):   # every prefill position quantized
            assert all(torch.equal(x, y) for x, y in zip(quantize(full[:, :, :, :T]), (q[:, :, :, :T], s[..., :T])))
        for i in range(n):
            cf.k.copy_(dequantize(c8.k, c8.k_scale))
            cf.v.copy_(dequantize(c8.v, c8.v_scale))
            x = ids[:, T + i]
            assert torch.equal(m.decode_step(x, None, c8), m.decode_step(x, None, cf)), i


def test_decoders_run_on_an_fp8_cache(tiny):
    m = tiny
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, m.cfg.vocab_size, (3, 8), generator=g)
    lengths = [8, 3, 5]
    for kw in (dict(temperature=0.0), dict(temperature=0.8, top_k=20, min_p=0.05), dict(guidance_scale=1.5),
               dict(repetition_penalty=1.2, no_repeat_ngram_size=2, bad_words_ids=[[5]])):
        tokens, n_new = m.generate(ids, lengths, max_new_tokens=6, kv_cache_dtype=FP8, **kw)
        again, _ = m.generate(ids, lengths, max_new_tokens=6, kv_cache_dtype=FP8, **kw)
        assert tokens.shape == (3, 6) and torch.equal(tokens, again)
    for kw in (dict(), dict(do_sample=True, temperature=0.9), dict(num_beam_groups=2, diversity_penalty=0.5)):
        tokens, n_new, scores = m.beam_search(ids, lengths, num_beams=4, max_new_tokens=6, kv_cache_dtype=FP8, **kw)
        assert tokens.shape == (3, 6) and bool(torch.isfinite(scores).all())
    out = m.stochastic_beam_search(ids, lengths, num_beams=3, max_new_tokens=5, kv_cache_dtype=FP8)
    assert out[0].shape == (9, 5)
    greedy, _ = m.generate(ids[:1], max_new_tokens=6, temperature=0.0, kv_cache_dtype=FP8)
    beam1, _, _ = m.beam_search(ids[:1], num_beams=1, max_new_tokens=6, kv_cache_dtype=FP8)
    assert torch.equal(greedy, beam1)


def test_rejected_combinations(tiny):
    m = tiny
    ids = torch.randint(0, m.cfg.vocab_size, (2, 6))
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        m.generate(ids, max_new_tokens=3, kv_cache_dtype="fp8")
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        m.beam_search(ids, max_new_tokens=3, kv_cache_dtype="int8")
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        m.stochastic_beam_search(ids, max_new_tokens=3, kv_cache_dtype=torch.float8_e4m3fn)
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        m.generate(ids, max_new_tokens=3, temperature=0.0, prompt_lookup_num_tokens=2, kv_cache_dtype=FP8)
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        m.generate(ids, max_new_tokens=3, assistant_model=m, kv_cache_dtype=FP8)
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        m.contrastive_search(ids, max_new_tokens=3, kv_cache_dtype=FP8)
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        m.new_cache(2, 8, "e5m2")


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_convai_passes_the_cache_dtype_through(tiny):
    from adapcc_b200.eval import convai

    dialogs = [([[1, 2]], [[3, 4, 5]]), ([[6]], [[7], [8, 9]])]
    for kw in (dict(no_sample=True), dict(num_beams=2)):
        replies = convai.sample_replies(tiny, _Tok(), dialogs, max_length=5, kv_cache_dtype=FP8, **kw)
        assert len(replies) == 2
    with pytest.raises(ValueError, match="kv_cache_dtype"):
        convai.sample_replies(tiny, _Tok(), dialogs, max_length=5, penalty_alpha=0.6, kv_cache_dtype=FP8)
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, kv_cache_dtype=FP8)
    assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0


def test_build_log_shows_fp8_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    for pattern in (r"decode_attn_split_kernelILb0EhE\w*", r"kv_quantize_kernel\w*", r"kv_reorder_kernelILb0ELb1E\w*",
                    r"kv_reorder_kernelILb1ELb1E\w*"):
        hits = re.findall(r"Compiling entry function '(\w*%s)' for 'sm_90a'" % pattern, log)
        assert hits, pattern
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
