"""Prompt-lookup decoding on the CPU: the draft rule (ops/lookup.py) against HuggingFace's
``PromptLookupCandidateGenerator`` and on hand cases, the acceptance rule on hand cases, ``GPT2DoubleHeads.generate(...,
prompt_lookup_num_tokens=k)`` against plain greedy ``generate`` and HuggingFace's prompt lookup, argument errors, the
ConvAI pass-through, and the lookup kernels' build (nvcc only, no device)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.lookup import accept_row, draft_row, lookup_accept, lookup_draft  # noqa: E402


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _hf_model(tiny):
    transformers = pytest.importorskip("transformers")
    cfg = tiny.cfg
    hf = transformers.GPT2LMHeadModel(transformers.GPT2Config(
        vocab_size=cfg.vocab_size, n_positions=cfg.n_positions, n_embd=cfg.n_embd, n_layer=cfg.n_layer,
        n_head=cfg.n_head, layer_norm_epsilon=cfg.layer_norm_epsilon, activation_function="gelu_new")).eval()
    sd = {"transformer.wte.weight": tiny.wte.weight[:cfg.vocab_size], "transformer.wpe.weight": tiny.wpe.weight,
          "transformer.ln_f.weight": tiny.ln_f.weight, "transformer.ln_f.bias": tiny.ln_f.bias}
    for i, blk in enumerate(tiny.h):
        p = f"transformer.h.{i}."
        for ours, theirs in (("ln_1", "ln_1"), ("ln_2", "ln_2")):
            sd[p + theirs + ".weight"], sd[p + theirs + ".bias"] = getattr(blk, ours).weight, getattr(blk, ours).bias
        for ours, theirs in (("c_attn", "attn.c_attn"), ("c_proj", "attn.c_proj"), ("c_fc", "mlp.c_fc"),
                             ("c_proj2", "mlp.c_proj")):
            sd[p + theirs + ".weight"] = getattr(blk, ours).weight.t()
            sd[p + theirs + ".bias"] = getattr(blk, ours).bias
    missing, _ = hf.load_state_dict({k: v.detach().clone() for k, v in sd.items()}, strict=False)
    assert not [k for k in missing if not k.endswith(("attn.bias", "masked_bias", "lm_head.weight"))], missing
    hf.tie_weights()
    return transformers, hf


# ---- the draft rule ------------------------------------------------------------------------------------------------
def test_draft_rule_equals_huggingface_prompt_lookup():
    transformers = pytest.importorskip("transformers")
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator

    rng = np.random.default_rng(0)
    checked = 0                                                         # an eos id that never occurs: no cut
    for trial in range(400):
        n = int(rng.integers(1, 40))
        seq = rng.integers(0, int(rng.integers(2, 12)), n)
        if n > 6 and trial % 2:                                         # a planted repeat of the tail
            m = int(rng.integers(1, 5))
            i = int(rng.integers(0, n - m))
            seq[i:i + m] = seq[n - m:]
        for ngram in (1, 2, 3, 4):
            for cap in (1, 3, 7):
                gen = PromptLookupCandidateGenerator(torch.tensor([-1]), num_output_tokens=cap,
                                                     max_matching_ngram_size=ngram, max_length=10 ** 6)
                out, _ = gen.get_candidates(torch.tensor([seq.tolist()]))
                want = out[0, n:].tolist()
                assert draft_row(seq.tolist(), cap, ngram) == want, (seq.tolist(), ngram, cap)
                checked += bool(want)
    assert checked > 500


def test_draft_rule_hand_cases():
    assert draft_row([1, 2, 3, 4], 4, 2) == []                         # no match
    assert draft_row([5], 4, 3) == []                                  # shorter than any n-gram with a continuation
    assert draft_row([7, 7], 4, 3) == [7]                              # m = min(3, |s| - 1) = 1
    # the earliest match wins, and a longer n-gram before a shorter one
    assert draft_row([1, 2, 9, 1, 2, 8, 1, 2], 2, 2) == [9, 1]
    assert draft_row([3, 2, 5, 1, 2, 6, 2], 3, 2) == [5, 1, 2]         # no 2-gram (6, 2): the 1-gram (2) at 1
    assert draft_row([4, 1, 2, 3, 1, 2], 9, 2) == [3, 1, 2]            # the continuation is cut by the sequence end
    assert draft_row([4, 1, 2, 3, 1, 2], 2, 2) == [3, 1]               # ... and by the cap
    assert draft_row([4, 1, 2, 3, 1, 2], 0, 2) == []                   # no room left under max_new_tokens
    seq = torch.tensor([[4, 1, 2, 3, 1, 2, 0, 0], [4, 1, 2, 3, 1, 2, 0, 0], [1, 1, 1, 0, 0, 0, 0, 0]],
                       dtype=torch.int32)
    ids, pos, nq = lookup_draft(seq, torch.tensor([5, 5, 2]), torch.tensor([1, 8, 1]), torch.tensor([0, 0, 1]), 3,
                                10, 2)
    # row 0: r = min(3, 10 - 1 - 1) = 3; row 1: r = min(3, 10 - 8 - 1) = 1; row 2: done
    assert ids.tolist() == [2, 3, 1, 2, 2, 3, 0, 0, 0, 0, 0, 0] and nq.tolist() == [4, 2, 0]
    assert pos.tolist() == [5, 6, 7, 7, 5, 6, 7, 7, 2, 3, 4, 5]


# ---- the acceptance rule -------------------------------------------------------------------------------------------
def _logits(best, V=10):
    """fp32 logits [len(best), V] whose arg-max in row j is best[j]."""
    x = np.zeros((len(best), V), dtype=np.float32)
    for j, t in enumerate(best):
        x[j, t] = 5.0
    return torch.from_numpy(x)


def _accept(best, drafts, e=1, max_new=20, L=3, stop=(), suppress=(), min_new=0, done=0, k=None):
    k = len(best) - 1 if k is None else k
    B = 1
    seq = torch.zeros(B, 40, dtype=torch.int32)
    lens, emitted, dn = (torch.tensor([v], dtype=torch.int32) for v in (L, e, done))
    tokens = torch.full((B, max_new), -1, dtype=torch.int64)
    steps = torch.zeros(B, dtype=torch.int32)
    ids = torch.zeros(k + 1, dtype=torch.int64)
    ids[1:1 + len(drafts)] = torch.tensor(drafts, dtype=torch.int64)
    logits = torch.full((k + 1, 10), -1.0)
    logits[:len(best)] = _logits(best)
    lookup_accept(logits, 10, ids, torch.tensor([len(best)], dtype=torch.int32), seq, lens, emitted, dn, tokens, steps,
                  min_new, suppress, stop)
    return tokens[0].tolist(), int(lens), int(emitted), int(dn), seq[0, L + 1:L + 6].tolist(), int(steps)


def test_acceptance_all_drafts_and_none():
    # a = k: every draft equals the previous slot's arg-max, so k + 1 tokens come out
    tok, L, e, done, seq, steps = _accept([4, 5, 6, 7], [4, 5, 6])
    assert tok[1:5] == [4, 5, 6, 7] and (L, e, done, steps) == (7, 5, 0, 1) and seq[:4] == [4, 5, 6, 7]
    # a = 0: the first draft differs, so only g_0 comes out
    tok, L, e, done, _, _ = _accept([4, 5, 6, 7], [3, 5, 6])
    assert tok[1:3] == [4, -1] and (L, e, done) == (4, 2, 0)
    # a = 1, then a rejection
    tok, L, e, _, _, _ = _accept([4, 5, 6, 7], [4, 9, 6])
    assert tok[1:4] == [4, 5, -1] and (L, e) == (5, 3)
    assert accept_row([4, 5], [4], 0, 20) == ([4, 5], False)


def test_acceptance_stop_inside_the_accepted_drafts():
    tok, L, e, done, seq, _ = _accept([4, 5, 6, 7], [4, 5, 6], stop=[5])
    assert tok[1:4] == [4, -1, -1] and done == 1 and (L, e) == (5, 3) and seq[:2] == [4, 5]


def test_acceptance_suppressed_draft_during_min_new():
    # slot 1's best id 5 is suppressed while e + 1 < min_new: its arg-max falls to the next id, so draft 2 (= 5) fails
    logits_best = [4, 5, 6]
    tok, L, e, done, _, _ = _accept(logits_best, [4, 5], e=1, min_new=3, suppress=[5])
    assert tok[1:4] == [4, 0, -1] and (L, e, done) == (5, 3, 0)
    # from e + 1 >= min_new on the id may be chosen again
    tok, *_ = _accept(logits_best, [4, 5], e=2, min_new=3, suppress=[5])
    assert tok[2:5] == [4, 5, 6]


def test_acceptance_max_new_cap_and_done_row():
    tok, L, e, done, _, _ = _accept([4, 5, 6, 7], [4, 5, 6], e=2, max_new=4)
    assert tok == [-1, -1, 4, 5] and done == 1 and (L, e) == (5, 4)
    tok, L, e, done, seq, steps = _accept([4, 5, 6, 7], [4, 5, 6], done=1)
    assert tok == [-1] * 20 and (L, e, done, steps) == (3, 1, 1, 0) and seq == [0] * 5


# ---- the model -----------------------------------------------------------------------------------------------------
def _ragged(V, seed=1, alphabet=24):
    g = torch.Generator().manual_seed(seed)
    lengths = [5, 30, 17, 30, 1]
    ids = torch.randint(0, alphabet, (5, 30), generator=g)             # a small alphabet: the prompts repeat
    tt = torch.randint(V - 5, V - 3, (5, 30), generator=g)
    return ids, lengths, tt


@pytest.mark.parametrize("k", [1, 3, 8])
def test_lookup_generate_equals_greedy_generate(tiny, k):
    V = tiny.cfg.vocab_size
    ids, lengths, tt = _ragged(V)
    want, n_want = tiny.generate(ids, lengths, tt, max_new_tokens=25, temperature=0.0)
    got, n_got = tiny.generate(ids, lengths, tt, max_new_tokens=25, temperature=0.0, prompt_lookup_num_tokens=k)
    assert torch.equal(got, want) and torch.equal(n_got, n_want)
    st = tiny.lookup_stats
    per_step = float((st["emitted"] - 1).sum()) / float(st["steps"].sum())
    print(f"k = {k}: {per_step:.2f} tokens per verify step")
    assert per_step >= 1.0
    # stop and suppressed ids, min_new_tokens, another n-gram size
    stop = [int(want[0, 6]), int(want[1, 2]), int(want[3, 0])]
    kw = dict(max_new_tokens=25, temperature=0.0, stop_ids=stop, suppress_ids=stop[2:], min_new_tokens=3)
    want, n_want = tiny.generate(ids, lengths, tt, **kw)
    got, n_got = tiny.generate(ids, lengths, tt, prompt_lookup_num_tokens=k, max_matching_ngram_size=3, **kw)
    assert torch.equal(got, want) and torch.equal(n_got, n_want)
    assert n_want.min() < 25


def test_lookup_generate_equals_huggingface_prompt_lookup(tiny):
    _, hf = _hf_model(tiny)                                             # its eos id lies outside the vocabulary
    g = torch.Generator().manual_seed(5)
    n = 30
    for trial, (k, ngram) in enumerate([(1, 2), (3, 2), (8, 3), (4, 1)]):
        prompt = torch.randint(0, 16, (1, 12), generator=g)
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), do_sample=False, max_new_tokens=n,
                               eos_token_id=tiny.cfg.vocab_size, pad_token_id=0, prompt_lookup_num_tokens=k,
                               max_matching_ngram_size=ngram)[0, 12:]
        tokens, _ = tiny.generate(prompt, max_new_tokens=n, temperature=0.0, prompt_lookup_num_tokens=k,
                                  max_matching_ngram_size=ngram)
        assert tokens[0].tolist() == want.tolist(), (trial, k, ngram)


def test_lookup_generate_rejects_bad_arguments(tiny):
    from adapcc_b200.ops import LOOKUP_MAX_TOKENS

    ids = torch.zeros(2, 10, dtype=torch.long)
    bad = [(dict(prompt_lookup_num_tokens=2, temperature=0.7), "temperature"),
           (dict(prompt_lookup_num_tokens=2, repetition_penalty=1.2), "repetition_penalty"),
           (dict(prompt_lookup_num_tokens=2, no_repeat_ngram_size=2), "no_repeat_ngram_size"),
           (dict(prompt_lookup_num_tokens=-1), "prompt_lookup_num_tokens"),
           (dict(prompt_lookup_num_tokens=LOOKUP_MAX_TOKENS + 1), "prompt_lookup_num_tokens"),
           (dict(prompt_lookup_num_tokens=2, max_matching_ngram_size=0), "max_matching_ngram_size"),
           (dict(prompt_lookup_num_tokens=2, max_new_tokens=0), "max_new_tokens")]
    for kw, name in bad:
        kw.setdefault("temperature", 0.0)
        with pytest.raises(ValueError, match=name):
            tiny.generate(ids, **kw)
    tiny.generate(ids, temperature=0.0, prompt_lookup_num_tokens=LOOKUP_MAX_TOKENS, max_new_tokens=5)


def test_too_many_verify_rows_on_the_native_path(monkeypatch):
    """The 64-row limit of the native LM head bounds B·(k+1); it is checked before anything is launched, so a bf16
    model that only claims to be on CUDA shows it."""
    from adapcc_b200.ops import LM_HEAD_MAX_ROWS

    model = GPT2DoubleHeads(GPT2Config.tiny()).to(torch.bfloat16).eval()
    monkeypatch.setattr(type(model.wte.weight), "is_cuda", property(lambda self: True), raising=False)
    ids = torch.zeros(9, 4, dtype=torch.long)
    assert 9 * 8 > LM_HEAD_MAX_ROWS >= 8 * 8
    with pytest.raises(ValueError, match=r"verify rows \(batch x \(prompt_lookup_num_tokens \+ 1\)\).*9 x 8"):
        model.generate(ids, temperature=0.0, prompt_lookup_num_tokens=7)


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_sample_replies_with_prompt_lookup(tiny):
    from adapcc_b200.eval import convai

    dialogs = [([[1, 2, 3]], [[3, 4, 5, 1, 2]]), ([[6]], [[7], [8, 9, 7]])]
    want = convai.sample_replies(tiny, _Tok(), dialogs, max_length=8, min_length=2, no_sample=True)
    got = convai.sample_replies(tiny, _Tok(), dialogs, max_length=8, min_length=2, no_sample=True,
                                prompt_lookup_num_tokens=3)
    assert got == want and tiny.lookup_stats["steps"].numel() == 2
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, no_sample=True, prompt_lookup_num_tokens=2)
    w = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, no_sample=True, batch_size=1)
    assert r == w


def test_build_log_shows_lookup_accept_and_draft_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_lookup\.cu", log)
    for kernel in ("lk_argmax_kernel", "lk_accept_kernel", "lk_draft_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
