"""Incremental (KV-cached) GPT-2 decoding on the CPU: the cached path against the uncached model, the sampling loops
against their uncached form, the guards, and the decode kernels' build (nvcc only, no device)."""
import os
import re
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, sample_sequence  # noqa: E402


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def test_teacher_forced_decode_matches_full_recompute(tiny):
    m, cfg = tiny, tiny.cfg
    g = torch.Generator().manual_seed(1)
    lengths = [1, 17, 40]
    B, T = len(lengths), max(lengths)
    ids = torch.randint(0, cfg.vocab_size, (B, T), generator=g)
    tt = torch.randint(cfg.vocab_size - 5, cfg.vocab_size - 3, (B, T), generator=g)
    prefix = [(ids[b, :n].clone(), tt[b, :n].clone()) for b, n in enumerate(lengths)]
    cache = m.new_cache(B)
    with torch.no_grad():
        h = m.hidden(ids, tt, cache=cache, lengths=lengths)
        for b, (pi, pt) in enumerate(prefix):
            want = m.hidden(pi[None], pt[None])[:, -1]
            assert torch.allclose(h[b, lengths[b] - 1], want[0], atol=1e-5, rtol=0), b
        assert cache.host_lens == lengths and cache.lens.tolist() == lengths
        for step in range(20):
            nid = torch.randint(0, cfg.vocab_size, (B,), generator=g)
            ntt = torch.randint(cfg.vocab_size - 5, cfg.vocab_size - 3, (B,), generator=g)
            h = m.decode_step(nid, ntt, cache)
            assert h.shape == (B, cfg.n_embd)
            for b in range(B):
                pi, pt = prefix[b]
                prefix[b] = (torch.cat([pi, nid[b:b + 1]]), torch.cat([pt, ntt[b:b + 1]]))
                want = m.hidden(prefix[b][0][None], prefix[b][1][None])[0, -1]
                err = float((h[b] - want).abs().max())
                assert err <= 1e-5, (step, b, err)
        assert cache.host_lens == [n + 20 for n in lengths] and cache.lens.tolist() == cache.host_lens


def _greedy_uncached(model, ids, tt, n, reply_type=None):
    """The generation loop as it was before the cache: the whole (windowed) prefix through the model per token."""
    out = []
    for _ in range(n):
        w = slice(max(0, ids.shape[1] - model.cfg.n_positions), None)
        h = model.hidden(ids[:, w], tt[:, w] if tt is not None else None)
        nxt = (h[:, -1].float() @ model.wte.weight.float().t())[:, :model.cfg.vocab_size].argmax(-1, keepdim=True)
        ids = torch.cat([ids, nxt], 1)
        if tt is not None:
            tt = torch.cat([tt, torch.full_like(nxt, reply_type)], 1)
        out.append(int(nxt))
    return out


@pytest.mark.parametrize("prompt_len", [9, 50])
def test_greedy_sample_sequence_matches_uncached_loop(tiny, prompt_len):
    # 50 + 25 tokens crosses n_positions = 64 mid-generation: the window slides and the loop leaves the cache
    m, cfg = tiny, tiny.cfg
    g = torch.Generator().manual_seed(prompt_len)
    prompt = torch.randint(0, cfg.vocab_size, (1, prompt_len), generator=g)
    tt = torch.full_like(prompt, cfg.vocab_size - 4)
    rt = cfg.vocab_size - 5
    with torch.no_grad():
        want = _greedy_uncached(m, prompt, tt, 25, rt)
    got = sample_sequence(m, prompt, tt, max_new_tokens=25, top_k=1, top_p=1.0, reply_type=rt)
    assert got[0].tolist() == want
    with torch.no_grad():
        want = _greedy_uncached(m, prompt, None, 25)
    assert sample_sequence(m, prompt, None, max_new_tokens=25, top_k=1, top_p=1.0)[0].tolist() == want


def _reply_uncached(model, tokenizer, persona, history, max_length):
    """``sample_reply(no_sample=True)`` as it was before the cache."""
    from adapcc_b200.data.personachat import build_input_from_segments

    special = set(tokenizer.special_ids)
    out = []
    for _ in range(max_length):
        inst = build_input_from_segments(persona, history, out, tokenizer, with_eos=False, max_len=model.cfg.n_positions)
        h = model.hidden(torch.tensor(inst.input_ids)[None], torch.tensor(inst.token_type_ids)[None])[0, -1]
        probs = F.softmax((h.float() @ model.wte.weight.float().t())[:model.cfg.vocab_size] / 0.7, dim=-1)
        nxt = int(torch.argmax(probs))
        if nxt in special:
            break
        out.append(nxt)
    return out


class _Tok:
    special_ids = (507, 508, 509, 510, 511)


def test_greedy_sample_reply_matches_uncached_loop_through_truncation():
    from adapcc_b200.data.personachat import build_input_from_segments
    from adapcc_b200.eval.convai import sample_reply

    torch.manual_seed(2)
    m = GPT2DoubleHeads(GPT2Config.tiny()).eval()
    g = torch.Generator().manual_seed(5)
    tok = _Tok()
    # special tokens end a reply; keep them out of the arg-max so the reply runs its full length
    with torch.no_grad():
        m.wte.weight[507:] = 0
    persona = [torch.randint(0, 500, (6,), generator=g).tolist()]
    history = [torch.randint(0, 500, (n,), generator=g).tolist() for n in (12, 10, 14, 9, 5)]
    first = build_input_from_segments(persona, history, [], tok, with_eos=False, max_len=m.cfg.n_positions)
    assert len(first.input_ids) >= m.cfg.n_positions - 6          # truncation drops history turns during the reply
    with torch.no_grad():
        want = _reply_uncached(m, tok, persona, history, 30)
    got = sample_reply(m, tok, persona, history, max_length=30, no_sample=True)
    assert len(want) == 30 and got == want
    last = build_input_from_segments(persona, history, want, tok, with_eos=False, max_len=m.cfg.n_positions)
    assert len(last.input_ids) < len(first.input_ids) + len(want)                  # history turns were dropped


def test_full_cache_raises(tiny):
    m, cfg = tiny, tiny.cfg
    cache = m.new_cache(2, t_max=5)
    ids = torch.randint(0, cfg.vocab_size, (2, 4))
    with torch.no_grad():
        m.hidden(ids, None, cache=cache, lengths=[4, 3])
    m.decode_step(ids[:, 0], None, cache)                 # row 0 reaches t_max = 5
    with pytest.raises(ValueError, match="full"):
        m.decode_step(ids[:, 0], None, cache)
    assert cache.host_lens == [5, 4] and cache.lens.tolist() == [5, 4]
    with pytest.raises(ValueError):
        m.hidden(torch.zeros(2, 6, dtype=torch.long), None, cache=cache)         # longer than t_max
    with pytest.raises(ValueError):
        m.decode_step(ids[0, :1], None, cache)                                     # wrong batch
    with pytest.raises(ValueError):
        m.new_cache(1, t_max=cfg.n_positions + 1)


def test_decode_attention_rejects_bad_arguments():
    from adapcc_b200.ops import decode_attention_

    B, H, t, Dh = 2, 4, 16, 16
    bf = torch.bfloat16

    def args(**kw):
        a = dict(qkv=torch.zeros(B, 3 * H * Dh, dtype=bf), k_cache=torch.zeros(B, H, t, Dh, dtype=bf),
                 v_cache=torch.zeros(B, H, t, Dh, dtype=bf), lens=torch.zeros(B, dtype=torch.int32),
                 out=torch.zeros(B, H * Dh, dtype=bf), work=torch.zeros(4096))
        a.update(kw)
        return a

    bad = [
        dict(qkv=torch.zeros(B, 3 * H * Dh)),                                        # fp32 qkv
        dict(k_cache=torch.zeros(B, H, t, Dh)),                                      # fp32 cache
        dict(out=torch.zeros(B, H * Dh, dtype=torch.float16)),
        dict(v_cache=torch.zeros(B, H, t + 1, Dh, dtype=bf)),                        # caches disagree
        dict(k_cache=torch.zeros(B, H, Dh, t, dtype=bf).transpose(2, 3), v_cache=torch.zeros(B, H, Dh, t, dtype=bf).transpose(2, 3)),
        dict(qkv=torch.zeros(B, 3 * H * Dh + 8, dtype=bf)),                          # wrong width
        dict(qkv=torch.zeros(3 * H * Dh, B, dtype=bf).t()),                           # strided columns
        dict(out=torch.zeros(B + 1, H * Dh, dtype=bf)),
        dict(lens=torch.zeros(B, dtype=torch.int64)),
        dict(lens=torch.zeros(B + 1, dtype=torch.int32)),
        dict(work=torch.zeros(4096, dtype=torch.float64)),
        {},                                                                          # everything on the CPU
    ]
    for kw in bad:
        with pytest.raises(ValueError, match="decode_attention_"):
            decode_attention_(**args(**kw))


def test_build_log_shows_decode_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert "ops_decode.cu" in log and "arch=compute_90a,code=sm_90a" in log
    for kernel in ("decode_attn_split_kernel", "decode_attn_combine_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        if kernel == "decode_attn_split_kernel":     # both variants: K / V read from global memory, and staged
            assert any("ILb0E" in h for h in hits) and any("ILb1E" in h for h in hits), hits
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
