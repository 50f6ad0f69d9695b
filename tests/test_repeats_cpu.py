"""Repetition penalty and no-repeat n-gram blocking on the CPU: the definition (ops/repeats.py) on hand cases and
against HuggingFace's logits processors, ``generate`` and ``beam_search`` against HuggingFace's greedy and beam search
with the same options, the no-repeat property of their outputs, argument errors, the ConvAI pass-through and the
kernel's build (nvcc only, no device)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.repeats import banned_ngram_ids, penalize_repeats_reference  # noqa: E402

INF = float("inf")


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _bits(t):
    return t.contiguous().view(torch.int32)


def repeated_ngram(full, start, n):
    """The first position t >= start whose n-gram ending at t occurs earlier in ``full`` (None if there is none)."""
    for t in range(max(start, n - 1), len(full)):
        gram = full[t - n + 1:t + 1]
        if any(full[j:j + n] == gram for j in range(t - n + 1)):
            return t
    return None


def test_penalty_hand_cases():
    row = torch.tensor([[2.0, -2.0, 0.5, 3.0, 0.0, -0.0, -INF, INF]])
    out = penalize_repeats_reference(row, [[0, 0, 1, 0, 4, 5, 6, 7, 1]], 8, 2.0, 0)[0]
    # every id once, however often it occurs: negative values multiplied, the others divided
    assert out[:4].tolist() == [1.0, -4.0, 0.5, 3.0]
    assert out[4].item() == 0.0 and not torch.signbit(out[4]) and torch.signbit(out[5])   # +-0 keep their sign
    assert out[6].item() == -INF and out[7].item() == INF
    # the penalty rounds to fp32 once and every operation is correctly rounded
    x = np.float32(-0.3)
    got = penalize_repeats_reference(torch.tensor([[float(x)]]), [[0]], 1, 1.1, 0)[0, 0].item()
    assert got == float(x * np.float32(1.1))
    # penalty 1 leaves every bit alone
    assert torch.equal(_bits(penalize_repeats_reference(row, [[0, 1, 4, 5]], 8, 1.0, 0)), _bits(row))


def test_ids_outside_the_vocabulary_are_ignored():
    row = torch.arange(1.0, 9.0).reshape(1, 8)                 # ld 8, vocab 4
    out = penalize_repeats_reference(row, [[-1, 5, 600, 2, 5, 600]], 4, 2.0, 1)[0]
    assert out.tolist() == [1.0, 2.0, -INF, 4.0, 5.0, 6.0, 7.0, 8.0]


def test_ngram_hand_cases():
    s = np.array
    assert sorted(banned_ngram_ids(s([3, 1, 3, 2]), 1).tolist()) == [1, 2, 3, 3]       # n = 1: the whole sequence
    assert banned_ngram_ids(s([1, 2]), 3).size == 0                                    # L < n: nothing
    assert banned_ngram_ids(s([1, 2, 1]), 3).size == 0                                 # the tail (2, 1) never seen
    assert banned_ngram_ids(s([1, 1]), 2).tolist() == [1]
    assert banned_ngram_ids(s([5, 6, 5, 7, 5]), 2).tolist() == [6, 7]
    # prompt (4, 9), reply (3, 4, 9): the n-gram (4, 9, 3) crosses the boundary and bans 3
    row = torch.zeros(1, 10)
    out = penalize_repeats_reference(row, [[4, 9, 3, 4, 9]], 10, 1.0, 3)[0]
    assert torch.isinf(out).nonzero().flatten().tolist() == [3]
    # penalty first, then bans: a banned id stays at -inf
    out = penalize_repeats_reference(torch.full((1, 4), -1.0), [[0, 1, 0]], 4, 1.5, 2)[0]
    assert out.tolist() == [-1.5, -INF, -1.0, -1.0]


def test_reference_matches_huggingface_processors():
    lp = pytest.importorskip("transformers.generation.logits_process")
    g = torch.Generator().manual_seed(0)
    for trial in range(40):
        R, L, V = 6, int(torch.randint(1, 40, (1,), generator=g)), 300
        logits = torch.randn(R, V, generator=g) * 5
        logits[torch.rand(R, V, generator=g) < 0.05] = 0.0
        logits[torch.rand(R, V, generator=g) < 0.02] = -INF
        hi = [8, 40, V][trial % 3]                                   # small id ranges plant repeats
        ids = torch.randint(0, hi, (R, L), generator=g)
        p = [0.7, 1.2, 1.3, 2.0, 1.0][trial % 5]
        n = [0, 1, 2, 3, 4, 8][trial % 6]
        want = logits.clone()
        if p != 1.0:
            want = lp.RepetitionPenaltyLogitsProcessor(p)(ids, want)
        if n:
            want = lp.NoRepeatNGramLogitsProcessor(n)(ids, want)
        got = penalize_repeats_reference(logits, list(ids), V, p, n)
        assert torch.equal(_bits(got), _bits(want)), (trial, p, n)


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


def test_greedy_generate_matches_huggingface(tiny):
    _, hf = _hf_model(tiny)
    g = torch.Generator().manual_seed(7)
    n = 30
    for trial, (p, ng) in enumerate([(1.3, 0), (1.0, 2), (1.5, 3), (0.8, 1), (2.0, 4)]):
        prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 12), generator=g)
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), do_sample=False, max_new_tokens=n,
                               min_new_tokens=n, eos_token_id=None, pad_token_id=0, repetition_penalty=p,
                               no_repeat_ngram_size=ng)[0, 12:]
        tokens, _ = tiny.generate(prompt, max_new_tokens=n, temperature=0.0, repetition_penalty=p,
                                  no_repeat_ngram_size=ng)
        assert tokens[0].tolist() == want.tolist(), (trial, p, ng)


def test_beam_search_matches_huggingface_with_renormalised_bans(tiny):
    transformers, hf = _hf_model(tiny)

    class Renormalise(transformers.LogitsProcessor):
        """HF bans after its log-softmax; normalising again gives the renormalised ban of ops/repeats.py."""

        def __call__(self, input_ids, scores):
            return torch.log_softmax(scores, dim=-1)

    g = torch.Generator().manual_seed(11)
    for trial, (K, ng) in enumerate([(2, 1), (4, 2), (5, 3), (3, 2)]):
        prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 12), generator=g)
        prompt[0, 6:9] = prompt[0, :3]                           # a planted repeat inside the prompt
        n = 12
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), num_beams=K, do_sample=False,
                               length_penalty=0.0, max_new_tokens=n, min_new_tokens=n, eos_token_id=None,
                               pad_token_id=0, early_stopping=False, no_repeat_ngram_size=ng,
                               logits_processor=transformers.LogitsProcessorList([Renormalise()]))[0, 12:]
        tokens, _, _ = tiny.beam_search(prompt, num_beams=K, max_new_tokens=n, length_penalty=0.0,
                                        no_repeat_ngram_size=ng)
        assert tokens[0].tolist() == want.tolist(), (trial, K, ng)


def test_no_ngram_repeats_in_outputs(tiny):
    g = torch.Generator().manual_seed(3)
    V = tiny.cfg.vocab_size
    lengths = [20, 7, 14]
    ids = torch.randint(0, 6, (3, 20), generator=g)                  # six ids: repeats everywhere in the prompts
    for n in (1, 2, 3):
        outs = []
        for seed in range(4):
            tokens, n_new = tiny.generate(ids, lengths, max_new_tokens=5 if n == 1 else 16, temperature=1.0,
                                          top_k=0, top_p=1.0, seed=seed * 10, no_repeat_ngram_size=n,
                                          repetition_penalty=1.2, stop_ids=[V - 1])
            outs.append((tokens, n_new))
        outs.append(tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=16, no_repeat_ngram_size=n)[:2])
        for tokens, n_new in outs:
            for b, x in enumerate(lengths):
                full = ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist()
                assert repeated_ngram(full, x, n) is None, (n, b, full)
    # without blocking the same prompts do repeat: the property is not vacuous
    tokens, n_new = tiny.generate(ids, lengths, max_new_tokens=16, temperature=0.0)
    assert any(repeated_ngram(ids[b, :x].tolist() + tokens[b].tolist(), x, 2) is not None
               for b, x in enumerate(lengths))


def test_defaults_run_nothing_new(tiny, monkeypatch):
    import adapcc_b200.models.gpt2 as gpt2
    import adapcc_b200.ops as ops

    def boom(*a, **k):
        raise AssertionError("repetition controls ran with their defaults")

    ids = torch.randint(0, tiny.cfg.vocab_size, (2, 9), generator=torch.Generator().manual_seed(0))
    want = tiny.generate(ids, max_new_tokens=6, temperature=0.0)
    want_beam = tiny.beam_search(ids, num_beams=3, max_new_tokens=6)
    monkeypatch.setattr(gpt2, "penalize_repeats_reference", boom)
    monkeypatch.setattr(ops, "penalize_repeats_", boom)
    got = tiny.generate(ids, max_new_tokens=6, temperature=0.0, repetition_penalty=1.0, no_repeat_ngram_size=0)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    got = tiny.beam_search(ids, num_beams=3, max_new_tokens=6)
    assert all(torch.equal(a, b) for a, b in zip(got, want_beam))
    with pytest.raises(AssertionError):
        tiny.generate(ids, max_new_tokens=2, no_repeat_ngram_size=2)


def test_argument_errors(tiny):
    from adapcc_b200.ops import penalize_repeats_

    ids = torch.zeros(2, 5, dtype=torch.long)
    for kw in (dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=float("nan")),
               dict(repetition_penalty=INF), dict(no_repeat_ngram_size=-1), dict(no_repeat_ngram_size=1.5)):
        with pytest.raises(ValueError, match="repetition_penalty|no_repeat_ngram_size"):
            tiny.generate(ids, max_new_tokens=2, **kw)
        with pytest.raises(ValueError, match="repetition_penalty|no_repeat_ngram_size"):
            tiny.beam_search(ids, max_new_tokens=2, **kw)
    # the op validates before it loads or launches anything
    R, T = 4, 16
    i32 = dict(dtype=torch.int32)
    good = dict(logits=torch.zeros(R, 10), vocab=10, seq=torch.zeros(R, T, **i32), prompt_len=torch.ones(R, **i32),
                lens=torch.ones(R, **i32), step=torch.zeros(1, **i32), ids=torch.zeros(R, dtype=torch.int64),
                parent=None, group=1, penalty=1.2, ngram=2)
    bad = [dict(penalty=0.0), dict(penalty=float("nan")), dict(ngram=-1), dict(vocab=11), dict(group=3),
           dict(group=17), dict(logits=torch.zeros(R, 10, dtype=torch.float64)), dict(seq=torch.zeros(R, T)),
           dict(seq=torch.zeros(R, 1025, **i32)), dict(lens=torch.ones(R + 1, **i32)),
           dict(ids=torch.zeros(R, **i32)), dict(parent=torch.zeros(R, dtype=torch.int64)), {}]
    for kw in bad:
        with pytest.raises(ValueError, match="penalize_repeats_"):
            penalize_repeats_(**dict(good, **kw))          # {} : CPU tensors are refused too


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_convai_passes_the_options_through(tiny, monkeypatch):
    from adapcc_b200.eval import convai

    seen = []
    for name in ("generate", "beam_search"):
        orig = getattr(tiny, name)

        def spy(*a, _orig=orig, _name=name, **k):
            seen.append((_name, k.get("repetition_penalty"), k.get("no_repeat_ngram_size")))
            return _orig(*a, **k)
        monkeypatch.setattr(tiny, name, spy)
    dialogs = [([[1, 2]], [[3, 4, 5, 3, 4]]), ([[6]], [[7], [8, 9]])]
    kw = dict(max_length=6, repetition_penalty=1.4, no_repeat_ngram_size=2)
    for beams in (0, 2):
        replies = convai.sample_replies(tiny, _Tok(), dialogs, num_beams=beams, no_sample=True, **kw)
        assert len(replies) == 2
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    # the sequential path has no repetition controls: with them on, f1 goes through the batched path
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", **kw)
    assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", num_beams=2, **kw)
    assert r["examples"] == 1
    assert seen == [("generate", 1.4, 2), ("beam_search", 1.4, 2), ("generate", 1.4, 2), ("beam_search", 1.4, 2)]


def test_build_log_shows_repeats_kernel_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_repeats\.cu", log)
    hits = re.findall(r"Compiling entry function '(\w*repeats_kernel\w*)' for 'sm_90a'", log)
    assert hits
    for name in hits:
        props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                          r"(\d+) bytes spill loads" % name, log)
        assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
