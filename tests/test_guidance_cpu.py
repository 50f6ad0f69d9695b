"""Classifier-free guidance on the CPU: the fp64 definition (ops/guidance.py) against HuggingFace's processor,
``generate`` on the tiny model against HuggingFace's ``generate(guidance_scale=...)``, guidance off at scale 1, a
negative prompt equal to the prompt, the argument errors, the ConvAI pass-through and the kernel's build (nvcc only,
no device)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.guidance import guided_scores_reference  # noqa: E402
from test_repeats_cpu import _hf_model, _Tok  # noqa: E402

U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


@pytest.mark.parametrize("scale", [0.0, 0.5, 1.5, 3.0, -1.0])
def test_reference_matches_huggingface_processor(scale):
    lp = pytest.importorskip("transformers.generation.logits_process")
    from transformers.modeling_outputs import CausalLMOutputWithPast

    R, V = 6, 1000
    g = torch.Generator().manual_seed(int(10 * scale) + 100)
    cond = torch.randn(R, V, generator=g) * 4
    uncond = torch.randn(R, V, generator=g) * 4

    def stub(input_ids, **kw):                      # the negative prompt's forward: the given logits
        return CausalLMOutputWithPast(logits=uncond[:, None])

    proc = lp.UnbatchedClassifierFreeGuidanceLogitsProcessor(scale, stub)
    want = proc(torch.zeros(R, 3, dtype=torch.long), cond.clone()).double()
    got = guided_scores_reference(cond, uncond, V, scale)
    lc, lu = torch.log_softmax(cond.double(), -1), torch.log_softmax(uncond.double(), -1)
    # HuggingFace's fp32 log-softmaxes are each within a few roundings of |x| + |logsumexp|; the mix adds three
    tol = 16 * U32 * ((abs(scale) + 1) * (lc.abs() + lu.abs() + cond.abs().double() + uncond.abs().double() + 10)
                      + got.abs())
    assert bool(((got - want).abs() <= tol).all()), float((got - want).abs().max())


def test_reference_keeps_only_the_vocabulary_and_rounds_the_scale():
    cond, uncond = torch.randn(2, 9), torch.randn(2, 9)
    got = guided_scores_reference(cond, uncond, 7, 0.1)
    assert got.shape == (2, 7) and got.dtype == torch.float64
    lc = torch.log_softmax(cond[:, :7].double(), -1)
    lu = torch.log_softmax(uncond[:, :7].double(), -1)
    assert torch.allclose(got, float(np.float32(0.1)) * (lc - lu) + lu, rtol=0, atol=1e-12)
    assert torch.allclose(guided_scores_reference(cond, uncond, 7, 0.0), lu, rtol=0, atol=1e-12)


@pytest.mark.parametrize("scale", [1.5, 3.0, 0.0, -1.0])
def test_tiny_greedy_matches_huggingface(tiny, scale):
    _, hf = _hf_model(tiny)
    g = torch.Generator().manual_seed(int(10 * scale) + 7)
    n = 16
    for trial, (neg_len, p) in enumerate([(0, 1.0), (5, 1.0), (0, 1.3), (9, 1.5)]):
        prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 12), generator=g)
        neg = torch.randint(0, tiny.cfg.vocab_size, (1, neg_len), generator=g) if neg_len else None
        extra = {} if neg is None else dict(negative_prompt_ids=neg, negative_prompt_attention_mask=torch.ones_like(neg))
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), do_sample=False, max_new_tokens=n,
                               min_new_tokens=n, eos_token_id=None, pad_token_id=0, guidance_scale=scale,
                               repetition_penalty=p, **extra)[0, 12:]
        tokens, _ = tiny.generate(prompt, max_new_tokens=n, temperature=0.0, guidance_scale=scale,
                                  negative_prompt_ids=neg, repetition_penalty=p)
        assert tokens[0].tolist() == want.tolist(), (trial, scale, neg_len, p)


def _batch(V, seed=3):
    g = torch.Generator().manual_seed(seed)
    lengths = [12, 5, 9]
    ids = torch.randint(0, V - 5, (3, 12), generator=g)
    tt = torch.randint(V - 5, V - 3, (3, 12), generator=g)
    return ids, lengths, tt


def test_scale_one_is_off(tiny, monkeypatch):
    import adapcc_b200.models.gpt2 as gpt2
    import adapcc_b200.ops as ops

    V = tiny.cfg.vocab_size
    ids, lengths, tt = _batch(V)
    neg = torch.randint(0, V, (3, 4), generator=torch.Generator().manual_seed(1))
    for kw in (dict(temperature=0.0), dict(temperature=0.9, top_k=20, top_p=0.9, seed=11)):
        want = tiny.generate(ids, lengths, tt, max_new_tokens=8, **kw)

        def boom(*a, **k):
            raise AssertionError("guidance ran at scale 1")
        with monkeypatch.context() as mp:
            mp.setattr(gpt2, "guided_scores_reference", boom)
            mp.setattr(ops, "guidance_mix_", boom)
            for extra in ({}, dict(negative_prompt_ids=neg, negative_lengths=[4, 1, 2])):
                got = tiny.generate(ids, lengths, tt, max_new_tokens=8, guidance_scale=1.0, **extra, **kw)
                assert all(torch.equal(a, b) for a, b in zip(got, want)), kw
    # and it runs at any other scale
    with pytest.raises(AssertionError, match="guidance ran"):
        monkeypatch.setattr(gpt2, "guided_scores_reference", boom)
        tiny.generate(ids, lengths, tt, max_new_tokens=2, guidance_scale=1.0001)


def test_negative_prompt_equal_to_prompt_gives_plain_tokens(tiny):
    """lc = lu, so the scores are the log-softmax of the logits: the same arg-max and the same distribution as the
    plain logits. Only the rounding of ``x - m`` differs, so a draw may differ only at a near tie: a decision quantity
    within 2 % of the mass of its threshold (the rule of tests/test_gpu_generate.py)."""
    from adapcc_b200.ops.sampling import reference_row

    V = tiny.cfg.vocab_size
    ids, lengths, tt = _batch(V)
    head = tiny.wte.weight.float()
    for kw in (dict(temperature=0.0), dict(temperature=0.8, top_k=0, top_p=0.9, seed=5)):
        for scale in (2.0, -0.5):
            plain, _ = tiny.generate(ids, lengths, tt, max_new_tokens=12, **kw)
            got, _ = tiny.generate(ids, lengths, tt, max_new_tokens=12, guidance_scale=scale, negative_prompt_ids=ids,
                                   negative_lengths=lengths, negative_token_type_ids=tt, **kw)
            for b, x in enumerate(lengths):
                k = 0
                while k < 12 and int(plain[b, k]) == int(got[b, k]):
                    k += 1
                if k == 12:
                    continue
                seq = torch.cat([ids[b, :x], plain[b, :k]])[None]
                types = torch.cat([tt[b, :x], tt[b, x - 1].expand(k)])[None]
                with torch.no_grad():
                    logits = (tiny.hidden(seq, types)[0, -1].float() @ head.t())[:V].numpy()
                if kw["temperature"] == 0.0:
                    top2 = np.sort(logits)[-2:]
                    assert top2[1] - top2[0] <= 1e-5 * max(1.0, abs(top2[1])), (b, k)
                    continue
                r = reference_row(logits, 0.8, 0, 0.9, 5 + b, x + k)
                tail = r["tail"][np.isfinite(r["tail"])]
                assert (np.abs(r["cum"][r["kept"]] - r["target"]).min() <= 0.02 * r["Zp"]
                        or np.abs(tail - r["pZ"]).min() <= 0.02 * r["Z"]), (b, k)


def test_guided_rows_depend_on_their_own_prompts_only(tiny):
    V = tiny.cfg.vocab_size
    ids, lengths, tt = _batch(V)
    neg = torch.randint(0, V - 5, (3, 6), generator=torch.Generator().manual_seed(2))
    kw = dict(max_new_tokens=10, temperature=0.9, top_p=0.95, guidance_scale=1.7, repetition_penalty=1.2)
    both, _ = tiny.generate(ids, lengths, tt, seed=torch.tensor([4, 5, 6]), negative_prompt_ids=neg,
                            negative_lengths=[6, 2, 4], **kw)
    for b, (x, nl) in enumerate(zip(lengths, [6, 2, 4])):
        alone, _ = tiny.generate(ids[b:b + 1, :x], None, tt[b:b + 1, :x], seed=torch.tensor([4 + b]),
                                 negative_prompt_ids=neg[b:b + 1, :nl], **kw)
        assert torch.equal(alone[0], both[b]), b


def test_argument_errors(tiny):
    V = tiny.cfg.vocab_size
    ids, lengths, tt = _batch(V)
    neg = torch.zeros(3, 4, dtype=torch.long)
    cases = [
        (dict(guidance_scale=float("nan")), "guidance_scale"),
        (dict(guidance_scale=float("inf")), "guidance_scale"),
        (dict(guidance_scale=-float("inf")), "guidance_scale"),
        (dict(guidance_scale=1e39), "guidance_scale"),
        (dict(guidance_scale=None), "guidance_scale"),
        (dict(guidance_scale=2.0, negative_prompt_ids=neg, negative_lengths=[4, 0, 1]), "negative_lengths"),
        (dict(guidance_scale=2.0, negative_prompt_ids=neg, negative_lengths=[4, 5, 1]), "negative_lengths"),
        (dict(guidance_scale=2.0, negative_prompt_ids=neg, negative_lengths=[4, 1]), "negative_lengths"),
        (dict(guidance_scale=2.0, negative_prompt_ids=neg[:2]), "negative_prompt_ids"),
        (dict(guidance_scale=2.0, negative_lengths=[1, 1, 1]), "negative_prompt_ids"),
        (dict(guidance_scale=2.0, negative_prompt_ids=neg, negative_token_type_ids=neg[:, :3]),
         "negative_token_type_ids"),
        (dict(guidance_scale=2.0, negative_prompt_ids=torch.zeros(3, 60, dtype=torch.long), max_new_tokens=5),
         "n_positions"),
        (dict(guidance_scale=2.0, prompt_lookup_num_tokens=3, temperature=0.0), "prompt_lookup_num_tokens"),
        (dict(guidance_scale=0.5, assistant_model=tiny), "assistant_model"),
    ]
    for kw, match in cases:
        kw = dict(dict(max_new_tokens=4), **kw)
        with pytest.raises(ValueError, match=match):
            tiny.generate(ids, lengths, tt, **kw)
    with pytest.raises(ValueError, match="token_type_ids"):        # negative types need the prompts' types
        tiny.generate(ids, lengths, None, guidance_scale=2.0, negative_prompt_ids=neg, negative_token_type_ids=neg)
    # 60 + 4 fits n_positions = 64, 60 + 5 does not
    long_neg = torch.zeros(3, 60, dtype=torch.long)
    tiny.generate(ids, lengths, tt, max_new_tokens=4, guidance_scale=2.0, negative_prompt_ids=long_neg)


def test_guidance_mix_op_validates_before_launching():
    from adapcc_b200.ops import guidance_mix_

    good = dict(logits=torch.zeros(4, 10), vocab=10, B=2, scale=1.5)
    for kw in (dict(scale=float("nan")), dict(scale=1e39), dict(vocab=11), dict(vocab=0), dict(B=3), dict(B=0),
               dict(logits=torch.zeros(4, 10, dtype=torch.float64)), dict(logits=torch.zeros(10, 4).t()), {}):
        with pytest.raises(ValueError, match="guidance_mix_"):
            guidance_mix_(**dict(good, **kw))               # {} : CPU tensors are refused too


def test_convai_passes_guidance_through(tiny, monkeypatch):
    from adapcc_b200.data.personachat import build_input_from_segments
    from adapcc_b200.eval import convai

    tok = _Tok()
    seen = []
    orig = tiny.generate

    def spy(*a, **k):
        seen.append(k)
        return orig(*a, **k)
    monkeypatch.setattr(tiny, "generate", spy)
    dialogs = [([[1, 2], [3]], [[3, 4, 5, 3, 4]]), ([[6]], [[7], [8, 9]])]
    replies = convai.sample_replies(tiny, tok, dialogs, max_length=6, no_sample=True, guidance_scale=1.5,
                                    guidance_negative="no_persona")
    assert len(replies) == 2
    k = seen[-1]
    assert k["guidance_scale"] == 1.5
    bos = tok.special_ids[0]
    for b, (_, history) in enumerate(dialogs):
        inst = build_input_from_segments([], history, [], tok, with_eos=False, max_len=tiny.cfg.n_positions - 6)
        n = k["negative_lengths"][b]
        assert n == len(inst.input_ids) and inst.input_ids[0] == bos
        assert k["negative_prompt_ids"][b, :n].tolist() == inst.input_ids
        assert k["negative_token_type_ids"][b, :n].tolist() == inst.token_type_ids
    # [bos] + history + the reply's speaker token: the prompt's layout with the persona tokens gone
    sp1, sp2 = tok.special_ids[2], tok.special_ids[3]
    assert k["negative_prompt_ids"][1, :k["negative_lengths"][1]].tolist() == [bos, sp1, 7, sp2, 8, 9, sp1]
    assert k["negative_token_type_ids"][1, :7].tolist() == [sp1, sp2, sp2, sp1, sp1, sp1, sp2]
    # the default negative prompt is generate's own (the last prompt token)
    convai.sample_replies(tiny, tok, dialogs, max_length=6, no_sample=True, guidance_scale=1.5)
    assert seen[-1]["guidance_scale"] == 1.5 and "negative_prompt_ids" not in seen[-1]
    convai.sample_replies(tiny, tok, dialogs, max_length=6, no_sample=True)
    assert "guidance_scale" not in seen[-1]
    for kw in (dict(num_beams=2), dict(penalty_alpha=0.6), dict(prompt_lookup_num_tokens=2),
               dict(assistant_model=tiny), dict(guidance_negative="persona")):
        with pytest.raises(ValueError, match="sample_replies"):
            convai.sample_replies(tiny, tok, dialogs, max_length=6, no_sample=True, guidance_scale=1.5, **kw)
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    n_calls = len(seen)
    for neg in ("last_token", "no_persona"):
        r = convai.evaluate_dialogs(tiny, tok, d, "f1", guidance_scale=2.0, guidance_negative=neg, max_length=6)
        assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0
    assert len(seen) == n_calls + 2 and seen[-1]["guidance_scale"] == 2.0 and "negative_prompt_ids" in seen[-1]


def test_build_log_shows_guidance_kernel_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_guidance\.cu", log)
    hits = re.findall(r"Compiling entry function '(\w*guidance_mix_kernel\w*)' for 'sm_90a'", log)
    assert hits
    for name in hits:
        props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                          r"(\d+) bytes spill loads" % name, log)
        assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
