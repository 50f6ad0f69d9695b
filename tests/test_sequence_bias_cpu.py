"""Sequence bias and bad-word blocking on the CPU: rule 0 of the definition (ops/repeats.py) on hand cases and against
HuggingFace's processor chain, ``generate`` and ``beam_search`` against HuggingFace's greedy and beam search with the
same options, the no-banned-sequence property of every decoder, the defaults, argument errors and the ConvAI
pass-through."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.repeats import (BIAS_MAX_ENTRIES, BIAS_MAX_LEN, check_sequence_bias_args,  # noqa: E402
                                     penalize_repeats_reference)

INF = float("inf")


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _bits(t):
    return t.contiguous().view(torch.int32)


def _bits_pos_zero(t):
    """Bits with -0.0 mapped to +0.0: HuggingFace adds +0.0 to every id."""
    return _bits(torch.where(t == 0, torch.zeros_like(t), t))


def _ref(logits, seqs, vocab, sequence_bias=None, bad_words_ids=None, stop_ids=(), penalty=1.0, ngram=0):
    table = check_sequence_bias_args("test", sequence_bias, bad_words_ids, vocab, stop_ids)
    return penalize_repeats_reference(torch.as_tensor(logits, dtype=torch.float32), seqs, vocab, penalty, ngram,
                                      table)


def occurrences(full, start, banned):
    """The (position, sequence) of every banned sequence in ``full`` whose last id is at a position t >= start where
    the rule applies: t >= m, the sequence before it at least as long as the entry (L >= m)."""
    hits = []
    for s in banned:
        m = len(s)
        for t in range(max(start, m), len(full)):
            if tuple(full[t - m + 1:t + 1]) == tuple(s):
                hits.append((t, tuple(s)))
    return hits


def test_hand_cases():
    row = [[1.0, 2.0, -3.0, 0.5, 4.0, -0.0]]
    # a length-1 bias always applies; other ids keep their bits (-0.0 included)
    out = _ref(row, [[0, 1]], 6, {(3,): 1.5})[0]
    assert out.tolist() == [1.0, 2.0, -3.0, 2.0, 4.0, 0.0] and torch.signbit(out[5])
    # a multi-token entry that matches, one that does not, and one longer than the sequence (L < m)
    out = _ref(row, [[0, 4, 1]], 6, [[[4, 1, 2], 10.0], [[0, 1, 3], 10.0], [[5, 4, 1, 4], 10.0]])[0]
    assert out.tolist() == [1.0, 2.0, 7.0, 0.5, 4.0, -0.0]
    # L >= m is needed, not L >= m - 1: the sequence (4, 1) is the whole prefix of (4, 1, 0), but L = 2 < 3
    assert _ref(row, [[4, 1]], 6, [[[4, 1, 0], -1.0]])[0, 0].item() == 1.0
    assert _ref(row, [[5, 4, 1]], 6, [[[4, 1, 0], -1.0]])[0, 0].item() == 0.0
    # bias, then penalty: the penalty sees the biased value (-3 + 4 = 1 > 0, so it is divided)
    out = _ref(row, [[2]], 6, {(2,): 4.0}, penalty=2.0)[0]
    assert out[2].item() == 0.5
    # two entries with one target: the length-1 entry first, then the longer ones in the order given, in fp32
    big, small = 2.0 ** 24, 1.0
    out = _ref([[0.0, 0.0]], [[1, 1, 1]], 2, [[[1, 0], small], [[0], big], [[1, 1, 0], small]])[0]
    want = np.float32(np.float32(np.float32(big) + np.float32(small)) + np.float32(small))
    assert out[0].item() == float(want) == big                            # each add rounds: 2^24 + 1 -> 2^24
    out = _ref([[0.0, 0.0]], [[1, 1, 1]], 2, [[[1, 0], small], [[1, 1, 0], small], [[0], big]])[0]
    assert out[0].item() == big                                           # the length-1 entry first whatever the list
    out = _ref([[0.0, 0.0]], [[1, 1, 1]], 2, [[[1, 0], small], [[1, 1, 0], small], [[1], big]])[0]
    assert out[0].item() == 2.0 and out[1].item() == big                  # small + small first, then nothing else
    # a bad word equal to a stop id is dropped (a row can still stop); longer ones containing it are kept
    out = _ref(row, [[1, 0]], 6, bad_words_ids=[[5], [0, 4], [3]], stop_ids=[5])[0]
    assert out.tolist() == [1.0, 2.0, -3.0, -INF, -INF, -0.0]
    # a bad word crossing the prompt / reply boundary: prompt (7, 8), reply (9): bans 2 after (8, 9)
    out = _ref(torch.zeros(1, 10), [[7, 8, 9]], 10, bad_words_ids=[[8, 9, 2], [7, 9, 3]])[0]
    assert torch.isinf(out).nonzero().flatten().tolist() == [2]
    # a bad word on top of a bias and the penalty stays -inf; the n-gram ban on top of it too
    out = _ref(row, [[1, 1]], 6, {(1,): 3.0}, [[1, 1]], penalty=1.3, ngram=2)[0]
    assert out[1].item() == -INF


def test_reference_matches_huggingface_processors():
    lp = pytest.importorskip("transformers.generation.logits_process")
    g = np.random.default_rng(0)
    V = 60
    for trial in range(120):
        R, L = 5, int(g.integers(1, 14))
        ids = torch.from_numpy(g.integers(0, 6, (R, L)))                   # six ids: prefixes match often
        logits = torch.from_numpy((g.standard_normal((R, V)) * 4).astype(np.float32))
        logits[torch.from_numpy(g.random((R, V)) < 0.04)] = -INF
        logits[torch.from_numpy(g.random((R, V)) < 0.04)] = -0.0
        logits[torch.from_numpy(g.random((R, V)) < 0.04)] = 0.0
        sb = {}
        for _ in range(int(g.integers(1, 9))):
            m = int(g.integers(1, 5))
            s = tuple(int(x) for x in g.integers(0, 6, m))
            if g.random() < 0.6 and L >= m - 1 and m > 1:                  # plant a match of some row's tail
                r = int(g.integers(0, R))
                s = tuple(ids[r, L - (m - 1):].tolist()) + (int(g.integers(0, 8)),)
            sb[s] = float(g.standard_normal() * 3)
        bw = [[int(x) for x in g.integers(0, 6, int(g.integers(1, 4)))] for _ in range(int(g.integers(0, 4)))]
        p = [1.0, 1.3, 0.7][trial % 3]
        n = [0, 2, 3, 1][trial % 4]
        want = lp.SequenceBiasLogitsProcessor(sequence_bias=dict(sb))(ids, logits.clone())
        if p != 1.0:
            want = lp.RepetitionPenaltyLogitsProcessor(p)(ids, want)
        if n:
            want = lp.NoRepeatNGramLogitsProcessor(n)(ids, want)
        if bw:
            want = lp.NoBadWordsLogitsProcessor(bw, eos_token_id=None)(ids, want)
        got = _ref(logits, list(ids), V, sb, bw or None, penalty=p, ngram=n)
        assert torch.equal(_bits_pos_zero(got), _bits_pos_zero(want)), (trial, p, n)


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


def _options(free, prompt):
    """A bias and a ban list that act on ``free`` (the unbiased reply of ``prompt``): a bigram and a trigram of the
    reply banned, one id pushed down after its predecessor, one pushed up everywhere."""
    full = prompt + free
    P = len(prompt)
    bias = {(full[P + 1], full[P + 2]): -6.0, (full[P + 6],): 3.5, (full[P + 3], full[P + 4], full[P + 5]): -2.5}
    bad = [[full[P - 1], full[P]], full[P + 7:P + 10]]
    return bias, bad


def test_greedy_generate_matches_huggingface(tiny):
    _, hf = _hf_model(tiny)
    g = torch.Generator().manual_seed(7)
    n = 24
    for trial, (p, ng) in enumerate([(1.0, 0), (1.3, 0), (1.0, 2), (1.2, 3)]):
        prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 12), generator=g)
        free, _ = tiny.generate(prompt, max_new_tokens=n, temperature=0.0, repetition_penalty=p,
                                no_repeat_ngram_size=ng)
        bias, bad = _options(free[0].tolist(), prompt[0].tolist())
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), do_sample=False, max_new_tokens=n,
                               min_new_tokens=n, eos_token_id=None, pad_token_id=0, repetition_penalty=p,
                               no_repeat_ngram_size=ng, sequence_bias=bias, bad_words_ids=bad)[0, 12:]
        tokens, _ = tiny.generate(prompt, max_new_tokens=n, temperature=0.0, repetition_penalty=p,
                                  no_repeat_ngram_size=ng, sequence_bias=bias, bad_words_ids=bad)
        assert tokens[0].tolist() == want.tolist(), (trial, p, ng)
        assert tokens[0].tolist() != free[0].tolist(), trial                 # the options changed the reply


def test_beam_search_matches_huggingface_with_renormalised_bias(tiny):
    transformers, hf = _hf_model(tiny)

    class Renormalise(transformers.LogitsProcessor):
        """HF biases after its log-softmax; normalising again gives the renormalised bias of ops/repeats.py."""

        def __call__(self, input_ids, scores):
            return torch.log_softmax(scores, dim=-1)

    g = torch.Generator().manual_seed(11)
    n = 12
    for trial, (K, ng) in enumerate([(2, 0), (4, 2), (3, 0), (5, 3)]):
        prompt = torch.randint(0, tiny.cfg.vocab_size, (1, 12), generator=g)
        free, _, _ = tiny.beam_search(prompt, num_beams=K, max_new_tokens=n, length_penalty=0.0,
                                      no_repeat_ngram_size=ng)
        bias, bad = _options(free[0].tolist(), prompt[0].tolist())
        with torch.no_grad():
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), num_beams=K, do_sample=False,
                               length_penalty=0.0, max_new_tokens=n, min_new_tokens=n, eos_token_id=None,
                               pad_token_id=0, early_stopping=False, no_repeat_ngram_size=ng, sequence_bias=bias,
                               bad_words_ids=bad,
                               logits_processor=transformers.LogitsProcessorList([Renormalise()]))[0, 12:]
        tokens, _, _ = tiny.beam_search(prompt, num_beams=K, max_new_tokens=n, length_penalty=0.0,
                                        no_repeat_ngram_size=ng, sequence_bias=bias, bad_words_ids=bad)
        assert tokens[0].tolist() == want.tolist(), (trial, K, ng)


def _decoders(tiny, ids, lengths, **kw):
    """(name, tokens, n_new) of every decoder, each in several modes, with the same options ``kw``."""
    V = tiny.cfg.vocab_size
    out = []
    for seed in range(3):
        out.append(("generate", *tiny.generate(ids, lengths, max_new_tokens=12, temperature=1.0, top_p=1.0,
                                               seed=seed * 10, stop_ids=[V - 1], **kw)))
    out.append(("generate guided", *tiny.generate(ids, lengths, max_new_tokens=12, temperature=1.0, seed=3,
                                                  guidance_scale=1.5, **kw)))
    out.append(("beam", *tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=12, **kw)[:2]))
    out.append(("beam sampled", *tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=12, do_sample=True,
                                                  seed=5, **kw)[:2]))
    out.append(("beam groups", *tiny.beam_search(ids, lengths, num_beams=4, num_beam_groups=2,
                                                 diversity_penalty=0.5, max_new_tokens=12, **kw)[:2]))
    tok, nn, *_ = tiny.stochastic_beam_search(ids, lengths, num_beams=3, max_new_tokens=12, seed=2, **kw)
    out.append(("stochastic beam", tok.view(len(lengths), 3, -1)[:, 0], nn.view(len(lengths), 3)[:, 0]))
    out.append(("contrastive", *tiny.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.6, max_new_tokens=12,
                                                        **kw)))
    return out


def test_no_banned_sequence_in_any_decoder_output(tiny):
    g = torch.Generator().manual_seed(3)
    lengths = [14, 6, 10]
    ids = torch.randint(0, 40, (3, 14), generator=g)
    # the sequences the unbanned decoders produce (ending inside the reply): bigrams and trigrams, and their last ids
    free = _decoders(tiny, ids, lengths)
    seen = []
    for _, tokens, n_new in free:
        for b, x in enumerate(lengths):
            full = ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist()
            for m in (2, 3):
                for t in range(x, len(full)):
                    if t - m + 1 >= 0 and tuple(full[t - m + 1:t + 1]) not in seen:
                        seen.append(tuple(full[t - m + 1:t + 1]))
    banned = [list(s) for s in seen[:BIAS_MAX_ENTRIES - 8]]
    assert len(banned) > 50
    # ... a bias pushing some other replies up, so the ban is not the only control at work
    bias = {(int(ids[0, 3]),): 2.0, (int(ids[1, 2]), int(ids[1, 4])): 5.0}
    for name, tokens, n_new in _decoders(tiny, ids, lengths, bad_words_ids=banned, sequence_bias=bias):
        for b, x in enumerate(lengths):
            full = ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist()
            assert not occurrences(full, x, banned), (name, b, occurrences(full, x, banned))
    # without the ban the same prompts do produce them: the property is not vacuous for any decoder
    for name, tokens, n_new in free:
        assert any(occurrences(ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist(), x, banned)
                   for b, x in enumerate(lengths)), name


def test_defaults_run_nothing_new(tiny, monkeypatch):
    import adapcc_b200.models.gpt2 as gpt2
    import adapcc_b200.ops as ops

    def boom(*a, **k):
        raise AssertionError("sequence bias ran with its defaults")

    ids = torch.randint(0, tiny.cfg.vocab_size, (2, 9), generator=torch.Generator().manual_seed(0))
    want = tiny.generate(ids, max_new_tokens=6, temperature=0.0)
    want_beam = tiny.beam_search(ids, num_beams=3, max_new_tokens=6)
    want_cs = tiny.contrastive_search(ids, max_new_tokens=6)
    want_sbs = tiny.stochastic_beam_search(ids, num_beams=2, max_new_tokens=6)
    monkeypatch.setattr(gpt2, "penalize_repeats_reference", boom)
    monkeypatch.setattr(ops, "penalize_repeats_", boom)
    got = tiny.generate(ids, max_new_tokens=6, temperature=0.0, sequence_bias=None, bad_words_ids=None)
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    got = tiny.beam_search(ids, num_beams=3, max_new_tokens=6, sequence_bias=None, bad_words_ids=None)
    assert all(torch.equal(a, b) for a, b in zip(got, want_beam))
    got = tiny.contrastive_search(ids, max_new_tokens=6, sequence_bias=None, bad_words_ids=None)
    assert all(torch.equal(a, b) for a, b in zip(got, want_cs))
    got = tiny.stochastic_beam_search(ids, num_beams=2, max_new_tokens=6, sequence_bias={}, bad_words_ids=[])
    assert all(torch.equal(a, b) for a, b in zip(got, want_sbs))
    with pytest.raises(AssertionError):
        tiny.generate(ids, max_new_tokens=2, bad_words_ids=[[1]])


def test_argument_errors(tiny):
    V = tiny.cfg.vocab_size
    ids = torch.zeros(2, 5, dtype=torch.long)
    cases = [dict(sequence_bias={(V,): 1.0}), dict(sequence_bias={(-1,): 1.0}), dict(bad_words_ids=[[3, V]]),
             dict(bad_words_ids=[[-2]]), dict(sequence_bias={(): 1.0}), dict(bad_words_ids=[[]]),
             dict(sequence_bias=[[[1, 2], float("nan")]]), dict(sequence_bias={(1,): INF}),
             dict(sequence_bias={(1,): -INF}), dict(sequence_bias=[[[1, 2], 1.0], [[1, 2], 2.0]]),
             dict(bad_words_ids=[[i % V, i // V] for i in range(BIAS_MAX_ENTRIES + 1)]),
             dict(sequence_bias={(1,): 1.0}, bad_words_ids=[[2, i % V, i // V] for i in range(BIAS_MAX_ENTRIES)]),
             dict(bad_words_ids=[[1] * (BIAS_MAX_LEN + 1)]), dict(sequence_bias=[[[1.5], 1.0]]),
             dict(sequence_bias=[[[1], "x"]]), dict(bad_words_ids="abc"), dict(sequence_bias=[[1, 2, 3]])]
    for kw in cases:
        for call in (lambda: tiny.generate(ids, max_new_tokens=2, **kw),
                     lambda: tiny.beam_search(ids, num_beams=2, max_new_tokens=2, **kw),
                     lambda: tiny.stochastic_beam_search(ids, num_beams=2, max_new_tokens=2, **kw),
                     lambda: tiny.contrastive_search(ids, max_new_tokens=2, **kw)):
            with pytest.raises(ValueError, match="sequence_bias|bad_words_ids|BIAS_MAX"):
                call()
    # the limits themselves are fine
    check_sequence_bias_args("t", None, [[i % V, i // V] for i in range(BIAS_MAX_ENTRIES)], V)
    check_sequence_bias_args("t", {tuple(range(BIAS_MAX_LEN)): 1.0}, None, V)
    # with prompt lookup or an assistant
    for kw in (dict(sequence_bias={(1,): 1.0}), dict(bad_words_ids=[[1]])):
        with pytest.raises(ValueError, match="sequence_bias and bad_words_ids"):
            tiny.generate(ids, max_new_tokens=2, temperature=0.0, prompt_lookup_num_tokens=2, **kw)
        with pytest.raises(ValueError, match="sequence_bias and bad_words_ids"):
            tiny.generate(ids, max_new_tokens=2, assistant_model=tiny, **kw)
    # the op validates the table before it loads or launches anything
    from adapcc_b200.ops import penalize_repeats_

    R, T = 4, 16
    i32 = dict(dtype=torch.int32)
    good = dict(logits=torch.zeros(R, 10), vocab=10, seq=torch.zeros(R, T, **i32), prompt_len=torch.ones(R, **i32),
                lens=torch.ones(R, **i32), step=torch.zeros(1, **i32), ids=torch.zeros(R, dtype=torch.int64),
                parent=None, group=1, penalty=1.0, ngram=0)
    for bias in ({(1,): 1.0}, check_sequence_bias_args("t", {(11,): 1.0}, None, 12),
                 check_sequence_bias_args("t", None, [[3, 10]], 12)):
        with pytest.raises(ValueError, match="penalize_repeats_: .*bias"):
            penalize_repeats_(**good, bias=bias)


def test_table_layout():
    t = check_sequence_bias_args("t", [[[4, 1, 2], 0.5], [[2], 1.0], [[7, 3], -1.0]], [[5, 2], [2]], 10)
    assert t.targets.tolist() == [2, 3] and t.start.tolist() == [0, 4, 5]
    # target 2: its length-1 bias, the longer bias, then the bad words in order; target 3: its one entry
    assert t.bias.tolist() == [1.0, 0.5, -INF, -INF, -1.0] and t.pre_len.tolist() == [0, 2, 1, 0, 1]
    pre = [t.tab[o:o + n].tolist() for o, n in zip(t.pre_off, t.pre_len)]
    assert pre == [[], [4, 1], [5], [], [7]]
    assert t.max_id == 7 and t.num_entries == 5 and t.num_targets == 2
    assert check_sequence_bias_args("t", None, None, 10) is None
    assert check_sequence_bias_args("t", {}, [], 10) is None
    assert check_sequence_bias_args("t", None, [[3]], 10, stop_ids=[3]) is None


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
    for name in ("generate", "beam_search", "contrastive_search"):
        orig = getattr(tiny, name)

        def spy(*a, _orig=orig, _name=name, **k):
            seen.append((_name, k.get("sequence_bias"), k.get("bad_words_ids")))
            return _orig(*a, **k)
        monkeypatch.setattr(tiny, name, spy)
    dialogs = [([[1, 2]], [[3, 4, 5, 3, 4]]), ([[6]], [[7], [8, 9]])]
    sb, bw = {(3, 4): -2.0}, [[5], [7, 8]]
    kw = dict(max_length=6, sequence_bias=sb, bad_words_ids=bw)
    for extra in (dict(num_beams=0), dict(num_beams=2), dict(penalty_alpha=0.5, top_k=3)):
        assert len(convai.sample_replies(tiny, _Tok(), dialogs, no_sample=True, **kw, **extra)) == 2
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    # the sequential path has no sequence bias: with it on, f1 goes through the batched path
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", bad_words_ids=bw)
    assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", sequence_bias=sb)
    assert r["examples"] == 1
    assert seen == [("generate", sb, bw), ("beam_search", sb, bw), ("contrastive_search", sb, bw),
                    ("generate", None, bw), ("generate", sb, None)]
    with pytest.raises(ValueError, match="sequence_bias and bad_words_ids"):
        convai.sample_replies(tiny, _Tok(), dialogs, no_sample=True, prompt_lookup_num_tokens=2, **kw)
    # the example's --bad_words: each word with and without a leading space, each encoding once
    assert convai.bad_word_ids(_Tok(), ["ab", " c ", "", "ab"]) == [[97, 98], [32, 97, 98], [99], [32, 99]]
