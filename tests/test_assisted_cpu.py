"""Assisted generation on the CPU: ``GPT2DoubleHeads.generate(..., assistant_model=draft, num_assistant_tokens=k)``
against plain ``generate`` (greedy and sampled, with the target itself, an unrelated model and a cut-down model as the
draft), against HuggingFace's assisted greedy generation, hand cases of a round, argument errors, the ConvAI
pass-through, and the new kernels' build (nvcc only, no device)."""
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.assisted import assist_round, draw_slots  # noqa: E402
from adapcc_b200.ops.lookup import accept_row, lookup_accept, mean_tokens_per_step  # noqa: E402


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


@pytest.fixture(scope="module")
def other():
    torch.manual_seed(123)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


@pytest.fixture(scope="module")
def cut(tiny):
    """The target's first block with its embeddings and final LayerNorm."""
    cfg = GPT2Config.tiny()
    cfg.n_layer = 1
    m = GPT2DoubleHeads(cfg).eval()
    sd = {k: v for k, v in tiny.state_dict().items() if not k.startswith("h.") or k.startswith("h.0.")}
    m.load_state_dict(sd)
    return m


def _ragged(V, seed=1):
    g = torch.Generator().manual_seed(seed)
    lengths = [5, 30, 17, 30, 1]
    ids = torch.randint(0, 40, (5, 30), generator=g)
    tt = torch.randint(V - 5, V - 3, (5, 30), generator=g)
    return ids, lengths, tt


SAMPLED = [dict(temperature=0.0), dict(temperature=0.7, top_p=0.9, seed=3),
           dict(temperature=1.0, top_k=20, top_p=0.95, seed=11),
           dict(temperature=0.9, min_p=0.05, seed=torch.arange(5) * 7)]


@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("mode", range(len(SAMPLED)))
def test_assisted_generate_equals_plain_generate(tiny, other, k, mode):
    V = tiny.cfg.vocab_size
    ids, lengths, tt = _ragged(V)
    kw = dict(SAMPLED[mode], max_new_tokens=25)
    want, n_want = tiny.generate(ids, lengths, tt, **kw)
    for draft in (tiny, other):
        got, n_got = tiny.generate(ids, lengths, tt, assistant_model=draft, num_assistant_tokens=k, **kw)
        assert torch.equal(got, want) and torch.equal(n_got, n_want), (k, mode, draft is tiny)
        per_step = mean_tokens_per_step(tiny.assist_stats["emitted"], tiny.assist_stats["steps"])
        print(f"k = {k}, mode {mode}, draft {'self' if draft is tiny else 'other'}: {per_step:.2f} tokens per step")
        if draft is tiny:
            assert per_step > 0.8 * (k + 1) or k == 8            # the draft is the target: (nearly) all accepted
    # stop and suppressed ids, min_new_tokens
    stop = [int(want[0, 6]), int(want[1, 2]), int(want[3, 0])]
    kw.update(stop_ids=stop, suppress_ids=stop[2:], min_new_tokens=3)
    want, n_want = tiny.generate(ids, lengths, tt, **kw)
    got, n_got = tiny.generate(ids, lengths, tt, assistant_model=tiny, num_assistant_tokens=k, **kw)
    assert torch.equal(got, want) and torch.equal(n_got, n_want)
    assert n_want.min() < 25


def test_self_draft_accepts_everything_and_unrelated_draft_little(tiny, other, cut):
    V = tiny.cfg.vocab_size
    ids, lengths, tt = _ragged(V, seed=4)
    kw = dict(max_new_tokens=30, temperature=0.7, top_p=0.9, seed=5)
    want, _ = tiny.generate(ids, lengths, tt, **kw)
    rates = {}
    for name, draft in (("self", tiny), ("cut", cut), ("other", other)):
        got, _ = tiny.generate(ids, lengths, tt, assistant_model=draft, num_assistant_tokens=4, **kw)
        assert torch.equal(got, want), name
        rates[name] = mean_tokens_per_step(tiny.assist_stats["emitted"], tiny.assist_stats["steps"])
    print(rates)
    assert rates["self"] > 4.0 and rates["other"] < rates["self"] and rates["other"] >= 1.0


def test_greedy_assisted_equals_huggingface_assisted_generation(tiny, other):
    from test_lookup_cpu import _hf_model

    _, hf = _hf_model(tiny)
    _, hf_draft = _hf_model(other)
    g = torch.Generator().manual_seed(5)
    for k in (1, 3, 8):
        prompt = torch.randint(0, 100, (1, 12), generator=g)
        with torch.no_grad():
            hf_draft.generation_config.num_assistant_tokens = k
            hf_draft.generation_config.num_assistant_tokens_schedule = "constant"
            want = hf.generate(prompt, attention_mask=torch.ones_like(prompt), do_sample=False, max_new_tokens=30,
                               eos_token_id=tiny.cfg.vocab_size, pad_token_id=0, assistant_model=hf_draft)[0, 12:]
        tokens, _ = tiny.generate(prompt, max_new_tokens=30, temperature=0.0, assistant_model=other,
                                  num_assistant_tokens=k)
        assert tokens[0].tolist() == want.tolist(), k


# ---- hand cases of a round -----------------------------------------------------------------------------------------
def test_round_set_up():
    seq = torch.tensor([[4, 1, 2, 3, 0, 0], [5, 6, 7, 8, 9, 1], [1, 1, 0, 0, 0, 0]], dtype=torch.int32)
    ids, pos, nq, d_in, d_pos = assist_round(seq, torch.tensor([3, 5, 1]), torch.tensor([1, 8, 1]),
                                             torch.tensor([0, 0, 1]), 3, 10, 7)
    # row 0: r = min(3, 10 - 1 - 1) = 3; row 1: r = min(3, 10 - 8 - 1) = 1, at the cache's end; row 2: done
    assert ids.tolist() == [3, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0] and nq.tolist() == [4, 2, 0]
    assert pos.tolist() == [3, 4, 5, 5, 5, 5, 5, 5, 1, 2, 3, 4] and d_in.tolist() == [3, 1, 0]
    assert d_pos.tolist() == [[3, 5, 1], [4, 6, 2], [5, 6, 3], [6, 6, 4]]


def test_draft_and_verify_draws_use_the_slot_counters():
    from adapcc_b200.ops.sampling import reference_row

    g = torch.Generator().manual_seed(0)
    B, S, V = 3, 4, 50
    logits = torch.randn(B * S, V, generator=g) * 3
    lens, emitted = torch.tensor([7, 2, 9]), torch.tensor([1, 0, 4])
    done, nq = torch.tensor([0, 0, 1]), torch.tensor([4, 2, 0])
    seeds = [3, 4, 5]
    got = draw_slots(logits, V, 0.8, 0, 0.9, seeds, lens, emitted, done, nq, min_new=2, suppress_ids=[1, 2])
    for b in range(B):
        for j in range(S):
            if done[b] or j >= nq[b]:
                assert got[b, j] == -1
                continue
            want = reference_row(logits[b * S + j].numpy(), 0.8, 0, 0.9, seeds[b], int(lens[b]) + j + 1,
                                 int(emitted[b]) + j, 2, [1, 2])["token"]
            assert got[b, j] == want
    d = draw_slots(logits[::S].contiguous(), V, 0.8, 0, 0.9, seeds, lens, emitted, done, nq, slot0=1, draft=True)
    assert d[:, 0].tolist()[1:] == [-1, -1]                               # row 1: draft 2 >= nq; row 2: done
    assert d[0, 0] == reference_row(logits[0].numpy(), 0.8, 0, 0.9, 3, 9, 2)["token"]


def _accept(g, drafts, e=1, max_new=20, L=3, stop=(), done=0):
    seq = torch.zeros(1, 40, dtype=torch.int32)
    lens, emitted, dn = (torch.tensor([v], dtype=torch.int32) for v in (L, e, done))
    tokens = torch.full((1, max_new), -1, dtype=torch.int64)
    steps = torch.zeros(1, dtype=torch.int32)
    ids = torch.zeros(len(g), dtype=torch.int64)
    ids[1:1 + len(drafts)] = torch.tensor(drafts, dtype=torch.int64)
    lookup_accept(None, 10, ids, torch.tensor([len(g)], dtype=torch.int32), seq, lens, emitted, dn, tokens, steps,
                  stop_ids=stop, drawn=torch.tensor([g]))
    return tokens[0].tolist(), int(lens), int(emitted), int(dn), int(steps)


def test_drawn_acceptance_hand_cases():
    tok, L, e, done, steps = _accept([4, 5, 6, 7], [4, 5, 6])             # every draft accepted
    assert tok[1:5] == [4, 5, 6, 7] and (L, e, done, steps) == (7, 5, 0, 1)
    tok, L, e, done, _ = _accept([4, 5, 6, 7], [4, 5, 6], stop=[5])        # a stop id inside the accepted drafts
    assert tok[1:4] == [4, -1, -1] and done == 1 and (L, e) == (5, 3)
    tok, L, e, done, _ = _accept([4, 5, 6, 7], [4, 5, 6], e=2, max_new=4)  # the cap at max_new_tokens
    assert tok == [-1, -1, 4, 5] and done == 1 and (L, e) == (5, 4)
    tok, L, e, done, steps = _accept([4, 5], [4], done=1)                  # a done row
    assert tok == [-1] * 20 and (L, e, done, steps) == (3, 1, 1, 0)
    assert accept_row([4, 5], [3], 0, 20) == ([4], False)


@pytest.mark.parametrize("temperature", [0.0, 0.8])
def test_prompt_plus_max_new_reaching_n_positions(tiny, other, temperature):
    n_pos = tiny.cfg.n_positions
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(0, 100, (3, n_pos - 9), generator=g)
    lengths = [n_pos - 9, 4, n_pos - 20]
    kw = dict(max_new_tokens=9, temperature=temperature, seed=1)
    want, _ = tiny.generate(ids, lengths, **kw)
    for draft in (tiny, other):
        got, _ = tiny.generate(ids, lengths, assistant_model=draft, num_assistant_tokens=8, **kw)
        assert torch.equal(got, want)


# ---- arguments -----------------------------------------------------------------------------------------------------
def test_assisted_generate_rejects_bad_arguments(tiny, other, monkeypatch):
    from adapcc_b200.ops import LOOKUP_MAX_TOKENS

    ids = torch.zeros(2, 10, dtype=torch.long)
    wide = GPT2DoubleHeads(GPT2Config(vocab_size=520, n_positions=64, n_embd=64, n_layer=1, n_head=4)).eval()
    bad = [(dict(prompt_lookup_num_tokens=2, temperature=0.0), "prompt_lookup_num_tokens"),
           (dict(repetition_penalty=1.2), "repetition_penalty"),
           (dict(no_repeat_ngram_size=2), "no_repeat_ngram_size"),
           (dict(num_assistant_tokens=0), "num_assistant_tokens"),
           (dict(num_assistant_tokens=LOOKUP_MAX_TOKENS + 1), "num_assistant_tokens"),
           (dict(assistant_model=wide), "vocab_size"),
           (dict(assistant_model="draft"), "assistant_model"),
           (dict(max_new_tokens=0), "max_new_tokens")]
    calls = []
    monkeypatch.setattr(GPT2DoubleHeads, "hidden", lambda *a, **k: calls.append(1))
    for kw, name in bad:
        kw.setdefault("assistant_model", other)
        with pytest.raises(ValueError, match=name):
            tiny.generate(ids, **kw)
    assert not calls                                                      # raised before anything ran
    monkeypatch.undo()
    tiny.generate(ids, temperature=0.0, assistant_model=other, num_assistant_tokens=LOOKUP_MAX_TOKENS,
                  max_new_tokens=5)


def test_native_path_checks_the_draft_and_the_verify_rows(monkeypatch):
    """On the native path the draft must be bf16 on the model's device, and B·(k+1) is bounded by the 64-row LM head;
    both are checked before anything is launched, so a bf16 model that only claims to be on CUDA shows it."""
    from adapcc_b200.ops import LM_HEAD_MAX_ROWS

    model = GPT2DoubleHeads(GPT2Config.tiny()).to(torch.bfloat16).eval()
    fp32 = GPT2DoubleHeads(GPT2Config.tiny()).eval()
    bf16 = GPT2DoubleHeads(GPT2Config.tiny()).to(torch.bfloat16).eval()
    monkeypatch.setattr(type(model.wte.weight), "is_cuda", property(lambda self: True), raising=False)
    ids = torch.zeros(9, 4, dtype=torch.long)
    with pytest.raises(ValueError, match="assistant_model must have bf16 weights"):
        model.generate(ids[:2], assistant_model=fp32, num_assistant_tokens=2)
    assert 9 * 8 > LM_HEAD_MAX_ROWS >= 8 * 8
    with pytest.raises(ValueError, match=r"verify rows \(batch x \(num_assistant_tokens \+ 1\)\).*9 x 8"):
        model.generate(ids, assistant_model=bf16, num_assistant_tokens=7)


class _Tok:
    special_ids = (507, 508, 509, 510, 511)
    pad_id = 511

    def encode(self, s):
        return [ord(c) % 500 for c in s]

    def decode(self, ids):
        return " ".join(str(i % 7) for i in ids)


def test_sample_replies_with_an_assistant(tiny, other):
    from adapcc_b200.eval import convai

    dialogs = [([[1, 2, 3]], [[3, 4, 5, 1, 2]]), ([[6]], [[7], [8, 9, 7]])]
    for no_sample in (True, False):
        kw = dict(max_length=8, min_length=2, no_sample=no_sample, seeds=[4, 5])
        want = convai.sample_replies(tiny, _Tok(), dialogs, **kw)
        got = convai.sample_replies(tiny, _Tok(), dialogs, assistant_model=other, num_assistant_tokens=3, **kw)
        assert got == want and tiny.assist_stats["steps"].numel() == 2
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    r = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, no_sample=True, assistant_model=other,
                                num_assistant_tokens=2)
    w = convai.evaluate_dialogs(tiny, _Tok(), d, "f1", max_length=5, no_sample=True, batch_size=1)
    assert r == w


def test_assistant_is_rejected_where_it_cannot_draft(tiny, other):
    from adapcc_b200.eval import convai

    dialogs = [([[1, 2, 3]], [[3, 4, 5, 1, 2]])]
    for kw, name in ((dict(num_beams=2), "num_beams"), (dict(penalty_alpha=0.6, top_k=3), "penalty_alpha")):
        with pytest.raises(ValueError, match=name):
            convai.sample_replies(tiny, _Tok(), dialogs, max_length=4, assistant_model=other, **kw)
    logits = torch.zeros(6, 10)                                           # draft draws: one logits row per row
    with pytest.raises(ValueError, match="one logits row per row"):
        draw_slots(logits, 10, 0.7, 0, 0.9, [1, 2, 3], torch.tensor([3, 3, 3]), torch.zeros(3), torch.zeros(3),
                   torch.full((3,), 4), slot0=0, draft=True)


def test_build_log_shows_assisted_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    for src in ("ops_sample", "ops_lookup"):
        assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*%s\.cu" % src, log)
    for kernel in ("sample_slots_kernel", "sample_tokens_kernel", "lk_round_kernel", "lk_accept_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
