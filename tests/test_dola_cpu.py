"""DoLa layer-contrast decoding on the CPU: the candidate layers and their errors, the fp64 definition
(ops/dola.py) against an fp32 transcription of HuggingFace's selection and relative-top filter, its per-row choice,
hand-built cases, the tiny model's ``generate(dola_layers=)`` against an uncached loop that takes the hidden states
with forward hooks, the argument errors, the ConvAI pass-through and the kernels' build (nvcc only, no device)."""
import math
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.ops.dola import (LN_TENTH, check_dola_args, dola_candidate_layers, dola_js_reference,  # noqa: E402
                                  dola_scores_reference)
from adapcc_b200.ops.repeats import penalize_repeats_reference  # noqa: E402
from adapcc_b200.ops.sampling import sample_reference  # noqa: E402
from test_repeats_cpu import _Tok  # noqa: E402


@pytest.fixture(scope="module")
def tiny():
    torch.manual_seed(0)
    return GPT2DoubleHeads(GPT2Config.tiny()).eval()


def test_candidate_layers():
    assert dola_candidate_layers(12, "low") == [1, 3, 5]
    assert dola_candidate_layers(12, "high") == [6, 8, 10]
    assert dola_candidate_layers(2, "low") == [1] and dola_candidate_layers(2, "high") == [1]
    assert dola_candidate_layers(3, "low") == [1] and dola_candidate_layers(3, "high") == [1]
    assert dola_candidate_layers(40, "low") == list(range(1, 20, 2))
    assert dola_candidate_layers(40, "high") == list(range(20, 40, 2))
    assert dola_candidate_layers(48, "low") == list(range(1, 20, 2))
    assert dola_candidate_layers(48, "high") == list(range(28, 48, 2))
    assert dola_candidate_layers(12, [0, 5, 12, 40]) == [0, 5]
    assert dola_candidate_layers(12, (7, 3, 3)) == [7, 3, 3]               # the given order, duplicates kept
    assert dola_candidate_layers(2, [1, 0]) == [1, 0]
    assert dola_candidate_layers(48, list(range(16))) == list(range(16))
    assert dola_candidate_layers(12, [np.int64(4)]) == [4]
    for n_layer, spec in ((12, [-1, 3]), (12, [1.0]), (12, [True]), (12, ["1"]), (12, [12, 40]), (12, []),
                          (48, list(range(17))), (12, "middle"), (12, 5), (12, None)):
        with pytest.raises(ValueError, match="dola_layers"):
            dola_candidate_layers(n_layer, spec)
    assert check_dola_args("generate", None, 12) is None
    for kw in (dict(guidance_scale=1.5), dict(prompt_lookup_num_tokens=3), dict(assistant_model=object())):
        with pytest.raises(ValueError, match="generate: dola_layers"):
            check_dola_args("generate", "low", 12, **kw)
    with pytest.raises(ValueError, match="generate: dola_layers"):
        check_dola_args("generate", [20], 12)


def _hf_contrast(final, premature):
    """HuggingFace's ``_dola_select_contrast`` and ``_relative_top_filter`` (relative_top 0.1, min_tokens_to_keep 1) as
    fp32 torch, for one row batch, transcribed: the batch-mean JS over the stacked candidates, then final minus base
    over the ids the filter keeps. Returns (scores [B, V], chosen index)."""
    final = final.float()
    if premature.shape[0] == 1:
        chosen = 0
    else:
        sm = F.softmax(final, dim=-1)
        sp = F.softmax(premature, dim=-1)
        avg = 0.5 * (sm[None] + sp)
        kl1 = F.kl_div(F.log_softmax(final, dim=-1)[None], avg, reduction="none").mean(-1)
        kl2 = F.kl_div(F.log_softmax(premature, dim=-1), avg, reduction="none").mean(-1)
        js = (0.5 * (kl1 + kl2)).mean(-1)
        chosen = int(js.argmax())
    scores, base = final.log_softmax(-1), premature[chosen].log_softmax(-1)
    sorted_logits, _ = torch.sort(scores, descending=True)
    min_thresh = sorted_logits[..., 0]
    probs_thresh = torch.min(min_thresh, scores.max(-1).values + np.log(0.1)).unsqueeze(-1)
    mask = scores < probs_thresh
    base = base.masked_fill(mask, -1e-3)
    scores = scores.masked_fill(mask, float("-inf"))
    return scores - base, chosen


def _rows(g, B, V, C, scale=4.0):
    return torch.randn(B, V, generator=g) * scale, torch.randn(C, B, V, generator=g) * scale


@pytest.mark.parametrize("C", [1, 2, 3, 8])
def test_reference_matches_huggingface_transcription(C):
    g = torch.Generator().manual_seed(C)
    V = 1000
    for trial in range(6):
        f, q = _rows(g, 1, V, C, scale=[4.0, 1.0, 12.0][trial % 3])
        want, want_c = _hf_contrast(f, q)
        got, got_c = dola_scores_reference(f, q, V)
        assert int(got_c[0]) == want_c, trial
        lf = torch.log_softmax(f.double(), -1)
        margin = (lf - (lf.max() + LN_TENTH)).abs() < 1e-4                     # fp32 and fp64 at the threshold
        fin_w, fin_g = torch.isfinite(want), torch.isfinite(got)
        assert torch.equal(fin_w[~margin], fin_g[~margin]), trial
        both = fin_w & fin_g
        assert torch.allclose(got[both], want.double()[both], rtol=1e-5, atol=1e-4), trial


def test_rows_choose_their_own_layer():
    """Each row's scores and choice equal its B = 1 result; HuggingFace's batch mean would couple the rows."""
    g = torch.Generator().manual_seed(11)
    V, B, C = 300, 5, 4
    f, q = _rows(g, B, V, C)
    scores, chosen = dola_scores_reference(f, q, V)
    for b in range(B):
        s1, c1 = dola_scores_reference(f[b:b + 1], q[:, b:b + 1], V)
        assert torch.equal(s1[0], scores[b]) and int(c1[0]) == int(chosen[b]), b
    assert len(set(chosen.tolist())) > 1                                     # the rows do pick different layers


def test_hand_built_cases(monkeypatch):
    import adapcc_b200.ops.dola as dola

    g = torch.Generator().manual_seed(3)
    V = 200
    f, q = _rows(g, 2, V, 3)
    # a candidate identical to the final row has JS = 0, the least possible
    q[1] = f
    js = dola_js_reference(f, q, V)
    assert bool((js[1].abs() <= 1e-12).all()) and bool((js[[0, 2]] > 1e-3).all())
    assert dola_scores_reference(f, q, V)[1].tolist() != [1, 1]
    # tied candidates: the first one
    q[2] = q[0]
    _, chosen = dola_scores_reference(f, q, V)
    assert chosen.tolist() == [0, 0]
    q2 = torch.stack([q[1], q[0], q[0]])
    assert dola_scores_reference(f, q2, V)[1].tolist() == [1, 1]
    # one candidate: nothing is selected (no divergence computed)
    with monkeypatch.context() as mp:
        mp.setattr(dola, "_js", lambda *a: (_ for _ in ()).throw(AssertionError("JS computed for one candidate")))
        s, c = dola_scores_reference(f, q[2:3], V)
    assert c.tolist() == [0, 0]
    # the kept set is exactly lf >= thr, thr = fl32(max lf + fl32(ln 0.1)); the score there is lf - lq
    lf, lq = torch.log_softmax(f.double(), -1), torch.log_softmax(q[2].double(), -1)
    thr = torch.from_numpy(np.float32((lf.max(-1).values + LN_TENTH).numpy()).astype(np.float64))
    keep = lf >= thr[:, None]
    assert torch.equal(torch.isfinite(s), keep)
    assert torch.allclose(s[keep], (lf - lq)[keep], rtol=0, atol=1e-12)
    assert LN_TENTH == float(np.float32(math.log(0.1)))
    # an id exactly on the threshold is kept: row [a, a + d] with lf_1 - lf_0 = d; choose d so lf_1 lands on thr
    x = torch.tensor([[0.0, float(np.float32(math.log(0.1)))]])
    lfx = torch.log_softmax(x.double(), -1)
    s, _ = dola_scores_reference(x, torch.zeros(1, 1, 2), 2)
    assert bool(torch.isfinite(s[0, 0])) and bool(torch.isfinite(s[0, 1])) == bool(
        lfx[0, 1] >= float(np.float32(float(lfx[0, 0]) + LN_TENTH)))


def _uncached(model, ids, lengths, layers, n, temperature=0.0, top_k=0, top_p=1.0, seed=0, penalty=1.0, ngram=0):
    """``generate(dola_layers=layers)`` as a loop without a cache: every step a full forward over each row's whole
    sequence, with the streams entering the candidate blocks taken by forward pre-hooks on the blocks (the unfused
    block path, which calls them), then the fp64 contrast, the repetition reference and ``sample_reference``."""
    V = model.cfg.vocab_size
    head = model.wte.weight.float()
    seen = {}
    hooks = [blk.register_forward_pre_hook(lambda mod, args, i=i: seen.__setitem__(i, args[0][0, -1].clone()))
             for i, blk in enumerate(model.h)]
    fuse = model.fuse_add_ln
    model.fuse_add_ln = False
    out = torch.full((len(lengths), n), -1, dtype=torch.int64)
    try:
        for b, x in enumerate(lengths):
            seq = ids[b, :x].tolist()
            for i in range(n):
                with torch.no_grad():
                    h = model.hidden(torch.tensor([seq]), None)[:, -1]
                    taps = torch.stack([seen[c] for c in layers])[:, None]
                    scores, _ = dola_scores_reference(model.lm_logits(h, head), model.lm_logits(taps, head), V)
                scores = penalize_repeats_reference(scores.float(), [torch.tensor(seq)], V, penalty, ngram)
                nxt, tok, _ = sample_reference(scores, V, temperature, top_k, top_p, torch.tensor([seed + b]),
                                               torch.tensor([x + i]), i)
                out[b, i] = tok[0]
                seq.append(int(nxt[0]))
    finally:
        model.fuse_add_ln = fuse
        for hk in hooks:
            hk.remove()
    return out


@pytest.mark.parametrize("layers", ["low", [0], [1, 0]])
def test_tiny_generate_equals_uncached_loop(tiny, layers):
    g = torch.Generator().manual_seed(7)
    V, n = tiny.cfg.vocab_size, 10
    lengths = [12, 5, 9]
    ids = torch.randint(0, V, (3, 12), generator=g)
    C = dola_candidate_layers(tiny.cfg.n_layer, layers)
    for kw in (dict(temperature=0.0), dict(temperature=0.9, top_k=40, top_p=0.9, seed=21)):
        for rep in (dict(), dict(repetition_penalty=1.2, no_repeat_ngram_size=2)):
            got, n_new = tiny.generate(ids, lengths, max_new_tokens=n, dola_layers=layers, **kw, **rep)
            want = _uncached(tiny, ids, lengths, C, n, penalty=rep.get("repetition_penalty", 1.0),
                             ngram=rep.get("no_repeat_ngram_size", 0), **kw)
            assert torch.equal(got, want), (layers, kw, rep)
            assert n_new.tolist() == [n] * 3
    kw = dict(max_new_tokens=n, temperature=1.0, top_p=1.0, seed=3)
    assert not torch.equal(tiny.generate(ids, lengths, **kw)[0], tiny.generate(ids, lengths, dola_layers=layers, **kw)[0])


def test_tiny_generate_rows_alone_and_fp8_cache(tiny):
    g = torch.Generator().manual_seed(8)
    V = tiny.cfg.vocab_size
    lengths = [12, 5, 9]
    ids = torch.randint(0, V, (3, 12), generator=g)
    kw = dict(max_new_tokens=8, temperature=0.8, top_p=0.95, dola_layers="high", repetition_penalty=1.1)
    both, _ = tiny.generate(ids, lengths, seed=torch.tensor([4, 5, 6]), **kw)
    for b, x in enumerate(lengths):
        alone, _ = tiny.generate(ids[b:b + 1, :x], seed=torch.tensor([4 + b]), **kw)
        assert torch.equal(alone[0], both[b]), b
    tokens, n_new = tiny.generate(ids, lengths, kv_cache_dtype="fp8_e4m3", **dict(kw, seed=4))
    assert tokens.shape == (3, 8) and n_new.tolist() == [8] * 3


def test_argument_errors(tiny):
    ids = torch.zeros(2, 4, dtype=torch.long)
    for kw, match in [(dict(dola_layers="middle"), "dola_layers"), (dict(dola_layers=[-1]), "dola_layers"),
                      (dict(dola_layers=[2, 5]), "dola_layers"), (dict(dola_layers=[0] * 17), "dola_layers"),
                      (dict(dola_layers=[0.5]), "dola_layers"),
                      (dict(dola_layers="low", guidance_scale=2.0), "dola_layers"),
                      (dict(dola_layers="low", prompt_lookup_num_tokens=2, temperature=0.0), "dola_layers"),
                      (dict(dola_layers="low", assistant_model=tiny), "dola_layers")]:
        with pytest.raises(ValueError, match=match):
            tiny.generate(ids, max_new_tokens=3, **kw)


def test_dola_op_validates_before_launching():
    from adapcc_b200.ops import dola_contrast_

    good = dict(logits=torch.zeros(6, 10), vocab=10, B=2, n_cand=2, work=torch.zeros(64))
    for kw in (dict(n_cand=0), dict(n_cand=17), dict(B=0), dict(B=3), dict(vocab=11), dict(vocab=0),
               dict(logits=torch.zeros(6, 10, dtype=torch.float64)), dict(logits=torch.zeros(10, 6).t()), {}):
        with pytest.raises(ValueError, match="dola_contrast_"):
            dola_contrast_(**dict(good, **kw))                 # {} : CPU tensors are refused too


def test_convai_passes_dola_through(tiny, monkeypatch):
    from adapcc_b200.eval import convai

    tok = _Tok()
    seen = []
    orig = tiny.generate

    def spy(*a, **k):
        seen.append(k)
        return orig(*a, **k)
    monkeypatch.setattr(tiny, "generate", spy)
    dialogs = [([[1, 2], [3]], [[3, 4, 5, 3, 4]]), ([[6]], [[7], [8, 9]])]
    replies = convai.sample_replies(tiny, tok, dialogs, max_length=6, no_sample=True, dola_layers="low")
    assert len(replies) == 2 and seen[-1]["dola_layers"] == "low"
    convai.sample_replies(tiny, tok, dialogs, max_length=6, no_sample=True)
    assert "dola_layers" not in seen[-1]
    for kw in (dict(num_beams=2), dict(penalty_alpha=0.6), dict(guidance_scale=1.5)):
        with pytest.raises(ValueError, match="sample_replies: dola_layers"):
            convai.sample_replies(tiny, tok, dialogs, max_length=6, no_sample=True, dola_layers="low", **kw)
    d = [{"personality": ["i like tea"], "utterances": [{"history": ["hello there"], "candidates": ["x y", "1 2"]}]}]
    n_calls = len(seen)
    r = convai.evaluate_dialogs(tiny, tok, d, "f1", dola_layers=[1], max_length=6)
    assert r["examples"] == 1 and 0.0 <= r["f1"] <= 1.0
    assert len(seen) == n_calls + 1 and seen[-1]["dola_layers"] == [1]


def test_build_log_shows_dola_kernels_for_sm90a_without_spills():
    import __graft_entry__

    __graft_entry__.build()
    log = open(os.path.join(ROOT, "adapcc_b200", "_C", "build.log")).read()
    assert re.search(r"-gencode arch=compute_90a,code=sm_90a \S.*ops_dola\.cu", log)
    for kernel in ("dola_divergence_kernel", "dola_contrast_kernel"):
        hits = re.findall(r"Compiling entry function '(\w*%s\w*)' for 'sm_90a'" % kernel, log)
        assert hits, kernel
        for name in hits:
            props = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                              r"(\d+) bytes spill loads" % name, log)
            assert props and props.group(2) == "0" and props.group(3) == "0", (name, props and props.group(0))
