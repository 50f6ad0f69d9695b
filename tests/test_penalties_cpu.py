"""Frequency / presence penalties and context n-gram blocking on the CPU: rules 2 and 4 of the definition
(ops/repeats.py) on hand cases, against a direct torch expression and against rule 3, greedy ``generate`` against an
uncached loop with the reference, the no-copied-prompt-n-gram and no-repeated-id properties of the decoders, the
defaults, argument errors and the ConvAI pass-through."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.repeats import (banned_ngram_ids, check_repeat_args, check_sequence_bias_args,  # noqa: E402
                                     penalize_repeats_reference)

INF = float("inf")
f32 = np.float32


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def _bits(t):
    return t.contiguous().view(torch.int32)


def _ref(row, prompt, reply, vocab, **kw):
    kw = dict(dict(penalty=1.0, ngram=0), **kw)
    p, n = kw.pop("penalty"), kw.pop("ngram")
    return penalize_repeats_reference(torch.tensor([row], dtype=torch.float32), [list(prompt) + list(reply)], vocab,
                                      p, n, prompt_lens=[len(prompt)], **kw)[0]


def test_frequency_and_presence_hand_cases():
    row = [1.0, 2.0, -3.0, 0.5, 4.0, -0.0, 7.0]
    # prompt ids do not count (5 and 1 only in the prompt); 2 seen 3x in the reply gets 3f, 3 seen once gets f
    out = _ref(row, [5, 1, 5, 2], [2, 2, 3, 2], 7, frequency=0.5)
    assert out.tolist() == [1.0, 2.0, -4.5, 0.0, 4.0, -0.0, 7.0]
    assert torch.signbit(out[5]) and not torch.signbit(out[3])
    # presence applies once per id however often it occurs
    out = _ref(row, [5], [2, 2, 2, 3], 7, presence=2.0)
    assert out.tolist() == [1.0, 2.0, -5.0, -1.5, 4.0, -0.0, 7.0]
    # frequency then presence, each rounded: fl32(fl32(l - fl32(c f)) - q)
    out = _ref([2.0 ** 24] * 3, [0], [1, 1, 1], 3, frequency=1.0 / 3, presence=1.0)
    want = f32(f32(f32(2.0 ** 24) - f32(3) * f32(1.0 / 3)) - f32(1.0))
    assert out[1].item() == float(want) and out[0].item() == 2.0 ** 24
    # negative values raise the logits
    out = _ref(row, [4], [0, 0, 6], 7, frequency=-1.0, presence=-0.25)
    assert out.tolist() == [3.25, 2.0, -3.0, 0.5, 4.0, -0.0, 8.25]
    # -inf stays -inf; with both off nothing is touched, so -0.0 keeps its bits
    out = _ref([-INF, 1.0, -0.0], [0], [0, 2, 0], 3, frequency=2.0, presence=1.0)
    assert out[0].item() == -INF and out[2].item() == -3.0
    out = _ref([-INF, 1.0, -0.0], [0], [0, 2, 2], 3)
    assert torch.equal(_bits(out), _bits(torch.tensor([-INF, 1.0, -0.0])))
    # ids at or past vocab (and negative ids) are ignored, without disturbing the others
    out = _ref(row, [0], [9, 9, 3, -1, 7], 7, frequency=1.0, presence=1.0)
    assert out.tolist() == [1.0, 2.0, -3.0, -1.5, 4.0, -0.0, 7.0]
    # the first token: an empty generated region changes nothing
    out = _ref(row, [2, 2, 3], [], 7, frequency=1.0, presence=1.0)
    assert out.tolist() == row


def _bans(out):
    return torch.isinf(out).nonzero().flatten().tolist()


def test_context_ngram_hand_cases():
    z = [0.0] * 10
    # m = 1: every prompt id, and no reply id
    assert _bans(_ref(z, [3, 1, 3], [4, 5], 10, context_ngram=1)) == [1, 3]
    # m = 3: rule 3 bans 4 (prompt) and 9 (reply); the context rule only the prompt's 4
    assert _bans(_ref(z, [2, 3, 4], [2, 3, 9, 2, 3], 10, ngram=3)) == [4, 9]
    assert _bans(_ref(z, [2, 3, 4], [2, 3, 9, 2, 3], 10, context_ngram=3)) == [4]
    # the tail (2, 3) crosses the prompt boundary: prompt (1, 2, 3, 4, 2), reply (3)
    assert _bans(_ref(z, [1, 2, 3, 4, 2], [3], 10, context_ngram=3)) == [4]
    # an m-gram ending on the prompt's last id counts, one ending on the first reply id does not
    assert _bans(_ref(z, [7, 8, 7], [8], 10, context_ngram=2)) == [7]
    assert _bans(_ref(z, [7, 8], [7, 8], 10, context_ngram=2)) == []
    assert _bans(_ref(z, [7, 8], [7, 8], 10, ngram=2)) == [7]
    assert _bans(_ref(z, [7, 8], [7, 6, 7], 10, context_ngram=2)) == [8]
    assert _bans(_ref(z, [7, 8], [7, 6, 7], 10, ngram=2)) == [6, 8]
    # the first token: the tail is the prompt's own end
    assert _bans(_ref(z, [2, 3, 4, 2, 3], [], 10, context_ngram=3)) == [4]
    # L < m: nothing; ids >= vocab are not banned
    assert _bans(_ref(z, [2, 3], [], 10, context_ngram=3)) == []
    assert _bans(_ref(z, [1, 12, 1], [], 10, context_ngram=2)) == []


def test_all_five_rules_in_order():
    """One row with every rule on: bias, penalty, frequency / presence, n-grams, context n-grams."""
    prompt, reply = [1, 2, 3], [4, 4, 1]
    row = [0.5, 3.0, -1.0, 2.0, 1.5, -0.0, 0.75, 8.0]
    table = check_sequence_bias_args("t", {(4,): 1.0, (1, 6): -0.5}, None, 8)
    out = _ref(row, prompt, reply, 8, penalty=2.0, ngram=2, bias=table, frequency=0.5, presence=0.25,
               context_ngram=1)
    want = np.array(row, dtype=np.float32)
    want[4] += f32(1.0)                                    # 0: (4,) always, (1, 6) after the tail 1
    want[6] += f32(-0.5)
    for i in (1, 2, 3, 4):                                 # 1: every distinct id of the sequence
        want[i] = want[i] * f32(2.0) if want[i] < 0 else want[i] / f32(2.0)
    want[4] = f32(f32(want[4] - f32(2) * f32(0.5)) - f32(0.25))  # 2: 4 twice, 1 once in the reply
    want[1] = f32(f32(want[1] - f32(1) * f32(0.5)) - f32(0.25))
    want[2] = -np.inf                                      # 3: the bigram (1, 2) after the tail 1
    want[[1, 2, 3]] = -np.inf                              # 4: m = 1, every prompt id
    assert torch.equal(_bits(out), _bits(torch.from_numpy(want)))
    assert out[4].item() == 0.0 and out[6].item() == 0.25 and torch.signbit(out[5])


def test_rule2_equals_torch_expression():
    g = np.random.default_rng(0)
    V = 97
    for trial in range(60):
        R = 6
        x = torch.from_numpy((g.standard_normal((R, V)) * 5).astype(np.float32))
        x[torch.from_numpy(g.random((R, V)) < 0.05)] = -INF
        x[torch.from_numpy(g.random((R, V)) < 0.05)] = -0.0
        f = float(g.choice([0.0, g.standard_normal(), 0.1, -2.5, 1e-3]))
        q = float(g.choice([0.0, g.standard_normal() * 3, 1.5, -0.7]))
        seqs, plens = [], []
        for _ in range(R):
            L = int(g.integers(1, 80))
            P = int(g.integers(0, L + 1))
            seqs.append(g.integers(0, [V, 12, V + 20][trial % 3], L))
            plens.append(P)
        got = penalize_repeats_reference(x, seqs, V, 1.0, 0, frequency=f, presence=q, prompt_lens=plens)
        want = x.clone()
        ft, qt = torch.tensor(f, dtype=torch.float32), torch.tensor(q, dtype=torch.float32)
        for r, (s, P) in enumerate(zip(seqs, plens)):
            gen = torch.from_numpy(s[P:])
            c = torch.bincount(gen[(gen >= 0) & (gen < V)], minlength=V)
            hit = c > 0
            v = want[r, hit]
            if f != 0:
                v = v - c[hit].to(torch.float32) * ft
            if q != 0:
                v = v - qt
            want[r, hit] = v
        assert torch.equal(_bits(got), _bits(want)), (trial, f, q)


def test_context_bans_are_rule3_bans_inside_the_prompt():
    g = np.random.default_rng(1)
    for trial in range(400):
        L = int(g.integers(1, 60))
        s = g.integers(0, [3, 6, 20][trial % 3], L)
        P = int(g.integers(0, L + 1))
        m = int(g.integers(1, 5))
        ctx = banned_ngram_ids(s, m, P)
        assert set(ctx.tolist()) <= set(banned_ngram_ids(s, m).tolist())
        # the definition, written out
        want = [int(s[j + m - 1]) for j in range(L) if L >= m and j + m - 1 < min(P, L)
                and s[j:j + m - 1].tolist() == s[L - m + 1:].tolist()]
        assert sorted(ctx.tolist()) == sorted(want), (trial, s.tolist(), P, m)
        # and through the reference: the rows' -inf sets nest the same way
        x = torch.zeros(1, 20)
        a = penalize_repeats_reference(x, [s], 20, 1.0, 0, context_ngram=m, prompt_lens=[P])
        b = penalize_repeats_reference(x, [s], 20, 1.0, m)
        assert set(_bans(a[0])) <= set(_bans(b[0]))


CONTROLS = [dict(frequency_penalty=0.6), dict(presence_penalty=1.5), dict(frequency_penalty=-0.3, presence_penalty=0.8),
            dict(context_no_repeat_ngram_size=1), dict(context_no_repeat_ngram_size=2),
            dict(frequency_penalty=0.5, presence_penalty=0.5, context_no_repeat_ngram_size=3, repetition_penalty=1.2,
                 no_repeat_ngram_size=4)]


def _ref_kw(kw):
    return dict(penalty=kw.get("repetition_penalty", 1.0), ngram=kw.get("no_repeat_ngram_size", 0),
                frequency=kw.get("frequency_penalty", 0.0), presence=kw.get("presence_penalty", 0.0),
                context_ngram=kw.get("context_no_repeat_ngram_size", 0))


def test_greedy_generate_equals_uncached_reference_loop(tiny):
    """Teacher-forced on ``generate``'s own tokens: at every step the arg-max of the uncached model's logits after
    the reference is the token ``generate`` chose (up to a near tie of the two paths' fp32 logits)."""
    g = torch.Generator().manual_seed(5)
    V, n = tiny.cfg.vocab_size, 16
    lengths = [12, 5, 9]
    ids = torch.randint(0, 60, (3, 12), generator=g)
    ids[0, 6:9] = ids[0, :3]                                   # a repeat inside a prompt
    # each prompt starts with its greedy reply's first id twice, so the context block has a pair to refuse
    ids[:, :2] = tiny.generate(ids, lengths, max_new_tokens=1, temperature=0.0)[0]
    for kw in CONTROLS:
        tokens, n_new = tiny.generate(ids, lengths, max_new_tokens=n, temperature=0.0, **kw)
        free, _ = tiny.generate(ids, lengths, max_new_tokens=n, temperature=0.0)
        assert n_new.tolist() == [n] * 3
        rk = _ref_kw(kw)
        p, ng = rk.pop("penalty"), rk.pop("ngram")
        for b, x in enumerate(lengths):
            seq = ids[b, :x].tolist()
            for i in range(n):
                with torch.no_grad():
                    h = tiny.hidden(torch.tensor([seq]), None)[0, -1]
                    logits = tiny.lm_logits(h)[None]
                lc = penalize_repeats_reference(logits, [seq], V, p, ng, prompt_lens=[x], **rk)[0]
                want, got = int(lc.argmax()), int(tokens[b, i])
                if want != got:
                    assert float(lc[want] - lc[got]) <= 1e-4, (kw, b, i, want, got)
                seq.append(got)
        assert not torch.equal(tokens, free), kw                 # every control changed some reply


def _decoders(tiny, ids, lengths, n=12, **kw):
    """(name, tokens [B, n], n_new [B]) of every decoder, each in several modes, with the same options ``kw``."""
    V = tiny.cfg.vocab_size
    out = []
    for seed in range(3):
        out.append(("generate", *tiny.generate(ids, lengths, max_new_tokens=n, temperature=1.0, top_p=1.0,
                                               seed=seed * 10, stop_ids=[V - 1], **kw)))
    out.append(("generate greedy", *tiny.generate(ids, lengths, max_new_tokens=n, temperature=0.0, **kw)))
    out.append(("generate guided", *tiny.generate(ids, lengths, max_new_tokens=n, temperature=1.0, seed=3,
                                                  guidance_scale=1.5, **kw)))
    out.append(("beam", *tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=n, **kw)[:2]))
    out.append(("beam sampled", *tiny.beam_search(ids, lengths, num_beams=3, max_new_tokens=n, do_sample=True,
                                                  seed=5, **kw)[:2]))
    out.append(("beam groups", *tiny.beam_search(ids, lengths, num_beams=4, num_beam_groups=2,
                                                 diversity_penalty=0.5, max_new_tokens=n, **kw)[:2]))
    tok, nn, *_ = tiny.stochastic_beam_search(ids, lengths, num_beams=3, max_new_tokens=n, seed=2, **kw)
    out.append(("stochastic beam", tok.view(len(lengths), 3, -1)[:, 0], nn.view(len(lengths), 3)[:, 0]))
    out.append(("contrastive", *tiny.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.6, max_new_tokens=n,
                                                        **kw)))
    return out


def copied_ngrams(full, P, m):
    """The positions t >= P (and t >= m, so a whole tail precedes) where ``full[t - m + 1:t + 1]`` is an m-gram of
    the prompt ``full[:P]``."""
    grams = {tuple(full[j:j + m]) for j in range(P - m + 1)}
    return [t for t in range(max(P, m), len(full)) if tuple(full[t - m + 1:t + 1]) in grams]


def test_no_decoder_completes_a_prompt_ngram(tiny):
    g = torch.Generator().manual_seed(3)
    lengths = [14, 6, 10]
    # prompts made of the ids the model likes to produce, so the unblocked replies do copy them
    seedp = torch.randint(0, tiny.cfg.vocab_size, (3, 14), generator=g)
    liked = torch.unique(torch.cat([t[:, :6].flatten() for _, t, _ in _decoders(tiny, seedp, lengths, n=6)]))
    liked = liked[liked >= 0]
    ids = liked[torch.randint(0, liked.numel(), (3, 14), generator=g)]
    for m in (1, 2, 3):
        hits_free = 0
        for _, tokens, n_new in _decoders(tiny, ids, lengths):
            for b, x in enumerate(lengths):
                hits_free += len(copied_ngrams(ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist(), x, m))
        for name, tokens, n_new in _decoders(tiny, ids, lengths, context_no_repeat_ngram_size=m):
            for b, x in enumerate(lengths):
                full = ids[b, :x].tolist() + tokens[b, :int(n_new[b])].tolist()
                assert not copied_ngrams(full, x, m), (m, name, b, full)
        if m < 3:
            assert hits_free > 0, m                              # without the block the replies do copy


def test_large_presence_penalty_never_repeats_a_reply_id(tiny):
    g = torch.Generator().manual_seed(8)
    lengths = [10, 4, 7]
    ids = torch.randint(0, tiny.cfg.vocab_size, (3, 10), generator=g)
    n = 20
    free, _ = tiny.generate(ids, lengths, max_new_tokens=n, temperature=0.0)
    assert any(len(set(r.tolist())) < n for r in free)           # greedy replies repeat themselves without it
    outs = [tiny.generate(ids, lengths, max_new_tokens=n, temperature=0.0, presence_penalty=1e4),
            tiny.contrastive_search(ids, lengths, top_k=4, penalty_alpha=0.6, max_new_tokens=n,
                                    presence_penalty=1e4)]
    for tokens, n_new in outs:
        for b in range(3):
            reply = tokens[b, :int(n_new[b])].tolist()
            assert len(reply) == n and len(set(reply)) == n, reply


def test_defaults_run_nothing_new(tiny, monkeypatch):
    import adapcc_b200.models.gpt2 as gpt2
    import adapcc_b200.ops as ops

    def boom(*a, **k):
        raise AssertionError("the penalties ran with their defaults")

    ids = torch.randint(0, tiny.cfg.vocab_size, (2, 9), generator=torch.Generator().manual_seed(0))
    off = dict(frequency_penalty=0.0, presence_penalty=0.0, context_no_repeat_ngram_size=0)
    want = tiny.generate(ids, max_new_tokens=6, temperature=0.0)
    want_beam = tiny.beam_search(ids, num_beams=3, max_new_tokens=6)
    want_cs = tiny.contrastive_search(ids, max_new_tokens=6)
    want_sbs = tiny.stochastic_beam_search(ids, num_beams=2, max_new_tokens=6)
    monkeypatch.setattr(gpt2, "penalize_repeats_reference", boom)
    monkeypatch.setattr(ops, "penalize_repeats_", boom)
    assert all(torch.equal(a, b) for a, b in zip(tiny.generate(ids, max_new_tokens=6, temperature=0.0, **off), want))
    assert all(torch.equal(a, b) for a, b in zip(tiny.beam_search(ids, num_beams=3, max_new_tokens=6, **off),
                                                 want_beam))
    assert all(torch.equal(a, b) for a, b in zip(tiny.contrastive_search(ids, max_new_tokens=6, **off), want_cs))
    assert all(torch.equal(a, b) for a, b in zip(tiny.stochastic_beam_search(ids, num_beams=2, max_new_tokens=6,
                                                                             **off), want_sbs))
    for kw in (dict(frequency_penalty=0.1), dict(presence_penalty=-0.1), dict(context_no_repeat_ngram_size=2)):
        with pytest.raises(AssertionError):
            tiny.generate(ids, max_new_tokens=2, **kw)


def test_argument_errors(tiny):
    ids = torch.zeros(2, 5, dtype=torch.long)
    cases = [(dict(frequency_penalty=float("nan")), "frequency_penalty"),
             (dict(frequency_penalty=INF), "frequency_penalty"), (dict(frequency_penalty=1e39), "frequency_penalty"),
             (dict(frequency_penalty="1"), "frequency_penalty"), (dict(presence_penalty=-INF), "presence_penalty"),
             (dict(presence_penalty=None), "presence_penalty"), (dict(presence_penalty=True), "presence_penalty"),
             (dict(context_no_repeat_ngram_size=-1), "context_no_repeat_ngram_size"),
             (dict(context_no_repeat_ngram_size=1.5), "context_no_repeat_ngram_size"),
             (dict(context_no_repeat_ngram_size="2"), "context_no_repeat_ngram_size")]
    for kw, name in cases:
        for call in (lambda: tiny.generate(ids, max_new_tokens=2, **kw),
                     lambda: tiny.beam_search(ids, num_beams=2, max_new_tokens=2, **kw),
                     lambda: tiny.stochastic_beam_search(ids, num_beams=2, max_new_tokens=2, **kw),
                     lambda: tiny.contrastive_search(ids, max_new_tokens=2, **kw)):
            with pytest.raises(ValueError, match=name):
                call()
    # any finite value of either sign is fine, and 0 and 1 are fine sizes
    check_repeat_args("t", 1.0, 0, -3e38, 3e38, 1)
    # with prompt lookup or an assistant
    for kw in (dict(frequency_penalty=0.5), dict(presence_penalty=0.5), dict(context_no_repeat_ngram_size=2)):
        with pytest.raises(ValueError, match="cannot be combined with prompt_lookup_num_tokens or assistant_model"):
            tiny.generate(ids, max_new_tokens=2, temperature=0.0, prompt_lookup_num_tokens=2, **kw)
        with pytest.raises(ValueError, match="cannot be combined with prompt_lookup_num_tokens or assistant_model"):
            tiny.generate(ids, max_new_tokens=2, assistant_model=tiny, **kw)
    # the reference needs the prompt lengths when a new rule is on
    with pytest.raises(ValueError, match="prompt_lens"):
        penalize_repeats_reference(torch.zeros(1, 4), [[1, 2]], 4, 1.0, 0, frequency=1.0)
    # the op validates before it loads or launches anything (CPU tensors would be refused after these checks)
    from adapcc_b200.ops import penalize_repeats_

    R, T = 4, 16
    i32 = dict(dtype=torch.int32)
    good = dict(logits=torch.zeros(R, 10), vocab=10, seq=torch.zeros(R, T, **i32), prompt_len=torch.ones(R, **i32),
                lens=torch.ones(R, **i32), step=torch.zeros(1, **i32), ids=torch.zeros(R, dtype=torch.int64),
                parent=None, group=1, penalty=1.0, ngram=0)
    for kw, name in ((dict(frequency=float("nan")), "frequency"), (dict(frequency=1e39), "frequency"),
                     (dict(presence=INF), "presence"), (dict(presence="x"), "presence"),
                     (dict(context_ngram=-1), "context_ngram"), (dict(context_ngram=2.5), "context_ngram")):
        with pytest.raises(ValueError, match=f"penalize_repeats_: {name}"):
            penalize_repeats_(**good, **kw)


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_convai_passes_the_options_through(tiny, monkeypatch):
    from adapcc_b200.eval import convai

    names = ("frequency_penalty", "presence_penalty", "context_no_repeat_ngram_size")
    seen = []
    for name in ("generate", "beam_search", "contrastive_search"):
        orig = getattr(tiny, name)

        def spy(*a, _orig=orig, _name=name, **k):
            seen.append((_name,) + tuple(k.get(x) for x in names))
            return _orig(*a, **k)
        monkeypatch.setattr(tiny, name, spy)
    dialogs = [([[1, 2]], [[3, 4, 5, 3, 4]]), ([[6]], [[7], [8, 9]])]
    kw = dict(max_length=6, frequency_penalty=0.4, presence_penalty=0.2, context_no_repeat_ngram_size=2)
    for extra in (dict(num_beams=0), dict(num_beams=2), dict(penalty_alpha=0.5, top_k=3)):
        assert len(convai.sample_replies(tiny, _Tok(), dialogs, no_sample=True, **kw, **extra)) == 2
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    # the sequential path has none of them: with any of them on, f1 goes through the batched path
    for one in (dict(frequency_penalty=0.3), dict(presence_penalty=-0.5), dict(context_no_repeat_ngram_size=3)):
        r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", **one)
        assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0
    assert seen == [("generate", 0.4, 0.2, 2), ("beam_search", 0.4, 0.2, 2), ("contrastive_search", 0.4, 0.2, 2),
                    ("generate", 0.3, 0.0, 0), ("generate", 0.0, -0.5, 0), ("generate", 0.0, 0.0, 3)]
    with pytest.raises(ValueError, match="cannot be combined"):
        convai.sample_replies(tiny, _Tok(), dialogs, no_sample=True, prompt_lookup_num_tokens=2, **kw)


def test_example_has_the_flags():
    src = open(os.path.join(ROOT, "examples", "eval_gpt2_convai.py")).read()
    for flag in ("--frequency_penalty", "--presence_penalty", "--context_no_repeat_ngram_size"):
        assert f'"{flag}"' in src
