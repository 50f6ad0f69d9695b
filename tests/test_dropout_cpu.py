"""Training dropout on the CPU: the mask definition of ``ops/dropout.py`` against Philox known answers and binomial
bounds, the tiny GPT-2 model's behaviour with it (off at p = 0 and in ``eval()``, never in generation, repeatable from
``(seed, step)``), one training step against an fp64 reference that applies ``dropout_mask`` at the documented sites, and
what the checkpoints carry."""
import dataclasses
import math
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
from adapcc_b200.ops.dropout import (DropoutState, _philox_halves, dropout, dropout_mask, dropout_reference,
                                     site_attn, site_embed, site_mlp, site_summary, threshold)
from test_gpu_training_reference import (CPU_CFG, _ce, _rel_max, _vanishing, base_weights, build_model, leaves,
                                         make_batch, ref_step)

P3 = dict(embd_pdrop=0.1, resid_pdrop=0.1, summary_first_dropout=0.1)


# ---- the fp64 reference with masks ---------------------------------------------------------------------------------
def gpt2_ref_masked(p, batch, lm_coef, mc_coef, cfg, seed, step):
    """``gpt2_ref`` of tests/test_gpu_training_reference.py with ``dropout_mask`` applied where the model documents it:
    the embedding sum (site 0), block i's attention output (1 + 2i) and MLP output (2 + 2i) before they join the
    residual stream, the multiple-choice head's input (1 + 2 n_layer). ``step`` is the value the masks use (a model set
    to step s uses s + 1 in its next training forward). Probabilities come from ``cfg``."""
    B, C, T = batch["input_ids"].shape
    ids, tt = batch["input_ids"].reshape(B * C, T), batch["token_type_ids"].reshape(B * C, T)
    N, D, H = B * C, cfg.n_embd, cfg.n_head

    def drop(x, prob, site):
        cols = x.shape[-1]
        keep = torch.from_numpy(dropout_mask(x.numel() // cols, cols, prob, seed, step, site)).to(x.device)
        return x * keep.view(x.shape) * threshold(prob)[1]

    def ln(x, k):
        return F.layer_norm(x, (D,), p[k + ".weight"], p[k + ".bias"], cfg.layer_norm_epsilon)

    def lin(x, k):
        return F.linear(x, p[k + ".weight"], p[k + ".bias"])

    wte = p["wte.weight"]
    x = drop(wte[ids] + p["wpe.weight"][:T] + wte[tt], cfg.embd_pdrop, site_embed())
    for i in range(cfg.n_layer):
        b = f"h.{i}."
        q, k, v = (t.view(N, T, H, D // H).transpose(1, 2) for t in lin(ln(x, b + "ln_1"), b + "c_attn").split(D, -1))
        a = F.scaled_dot_product_attention(q, k, v, is_causal=True)
        x = x + drop(lin(a.transpose(1, 2).reshape(N, T, D), b + "c_proj"), cfg.resid_pdrop, site_attn(i))
        x = x + drop(lin(F.gelu(lin(ln(x, b + "ln_2"), b + "c_fc"), approximate="tanh"), b + "c_proj2"),
                     cfg.resid_pdrop, site_mlp(i))
    h = ln(x, "ln_f")
    logits = h[:, :-1] @ wte[:cfg.vocab_size].t()
    lm = _ce(logits.reshape(-1, cfg.vocab_size), batch["lm_labels"].reshape(N, T)[:, 1:].reshape(-1))
    cls = drop(h[torch.arange(N, device=h.device), batch["mc_token_ids"].reshape(-1)], cfg.summary_first_dropout,
               site_summary(cfg.n_layer))
    mc = _ce(F.linear(cls, p["mc_head.weight"], p["mc_head.bias"]).view(B, C), batch["mc_labels"])
    return lm_coef * lm + mc_coef * mc, lm, mc


def ref_step_masked(p, batch, lm_coef, mc_coef, cfg, seed, step):
    """-> (gradients by name, (loss, lm_loss, mc_loss) as floats) of ``gpt2_ref_masked``."""
    out = gpt2_ref_masked(p, batch, lm_coef, mc_coef, cfg, seed, step)
    grads = torch.autograd.grad(out[0], list(p.values()))
    return dict(zip(p, grads)), tuple(float(x.detach()) for x in out)


# ---- the definition ------------------------------------------------------------------------------------------------
def _halves(words):
    return [h for w in words for h in (w & 0xFFFF, w >> 16)]


def test_mask_known_answers():
    """Random123's philox4x32_10 vectors (tests/test_generate_cpu.py) through the counter and key layout: counter
    (row, vec, site, step), key (seed low, seed high); half 2j the low half of word j, half 2j + 1 the high half."""
    ones = 0xFFFFFFFF
    kat = [((0, 0, 0, 0), 0, (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((ones,) * 4, (ones << 32) | ones, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0x299f31d0 << 32) | 0xa4093822,
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for (row, vec, site, step), seed, words in kat:
        got = _philox_halves(np.array([row]), np.array([vec]), seed, step, site)
        assert got.shape == (1, 1, 8) and got[0, 0].tolist() == _halves(words)
    # the first vector is element (0, 0..7) of the mask of seed 0, step 0, site 0
    h = np.array(_halves(kat[0][2]))
    for p in (0.1, 0.5, 0.9):
        assert dropout_mask(1, 8, p, 0, 0, 0)[0].tolist() == (h >= threshold(p)[0]).tolist()
    # a signed 64-bit seed is the same key as its unsigned value, and columns past a multiple of 8 are a prefix
    assert np.array_equal(dropout_mask(3, 16, 0.5, -1, 2, 3), dropout_mask(3, 16, 0.5, 2 ** 64 - 1, 2, 3))
    assert np.array_equal(dropout_mask(3, 13, 0.5, 9, 2, 3), dropout_mask(3, 16, 0.5, 9, 2, 3)[:, :13])


def test_threshold_and_scale():
    assert threshold(0.0) == (0, 1.0)
    assert dropout_mask(64, 64, 0.0, 1, 2, 3).all()
    assert threshold(0.1) == (6554, float(np.float32(65536.0 / (65536 - 6554))))
    assert threshold(0.5) == (32768, 2.0)
    for p in (65535 / 65536, 1 - 2.0 ** -20, math.nextafter(1.0, 0.0)):          # clamped: one value of 65536 is kept
        assert threshold(p) == (65535, 65536.0)
    x = torch.randn(16, 24, dtype=torch.float64)
    assert torch.equal(dropout_reference(x, 0.0, 5, 6, 7), x)
    keep = torch.from_numpy(dropout_mask(16, 24, 0.25, 5, 6, 7))
    assert torch.equal(dropout_reference(x, 0.25, 5, 6, 7), x * keep * threshold(0.25)[1])


def test_mask_statistics():
    """2^20 elements. The keep count is Binomial(n, q) with q = 1 - thr / 65536; two masks that differ in site, step,
    seed, or that are adjacent rows of one mask, agree on a Binomial(n, q^2 + (1 - q)^2) count. Bounds: 5 sigma."""
    rows, cols = 2048, 512
    n = rows * cols
    for p in (0.1, 0.5):
        q = 1 - threshold(p)[0] / 65536
        m = dropout_mask(rows, cols, p, 1234, 5, 3)
        assert abs(m.sum() - n * q) <= 5 * math.sqrt(n * q * (1 - q)), (p, m.mean())
        a = q * q + (1 - q) ** 2
        others = {"site": dropout_mask(rows, cols, p, 1234, 5, 4), "step": dropout_mask(rows, cols, p, 1234, 6, 3),
                  "seed": dropout_mask(rows, cols, p, 1235, 5, 3),
                  "seed high word": dropout_mask(rows, cols, p, 1234 + (1 << 32), 5, 3)}
        for what, o in others.items():
            assert abs((m == o).sum() - n * a) <= 5 * math.sqrt(n * a * (1 - a)), (p, what, (m == o).mean())
        k = (rows - 1) * cols
        assert abs((m[1:] == m[:-1]).sum() - k * a) <= 5 * math.sqrt(k * a * (1 - a)), p
        # the eight halves of a call are used once each: every column class keeps about q
        for c in range(8):
            sub = m[:, c::8]
            assert abs(sub.sum() - sub.size * q) <= 5 * math.sqrt(sub.size * q * (1 - q)), (p, c)


def test_dropout_op_cpu():
    """The CPU op is the numpy definition in the tensor's precision; the backward applies the same mask."""
    st = DropoutState.create(seed=77, step=3)
    keep = torch.from_numpy(dropout_mask(6, 40, 0.3, 77, 3, 9))
    scale = threshold(0.3)[1]
    for dtype in (torch.float32, torch.bfloat16, torch.float64):
        x = torch.randn(2, 3, 40).to(dtype).requires_grad_(True)
        y = dropout(x, 0.3, st, 9)
        wide = x.detach() if dtype == torch.float64 else x.detach().float()
        assert torch.equal(y, (wide * scale * keep.view(2, 3, 40)).to(dtype))
        y.sum().backward()
        assert torch.equal(x.grad, (keep.view(2, 3, 40) * scale).to(dtype))
    st.advance()
    assert int(st.step) == 4


def test_argument_errors():
    st = DropoutState.create(1)
    x = torch.zeros(2, 8)
    for p in (-0.1, 1.0, 1.5, float("nan")):
        with pytest.raises(ValueError, match="probability"):
            dropout(x, p, st, 0)
        with pytest.raises(ValueError, match="probability"):
            threshold(p)
    with pytest.raises(ValueError, match="int64"):
        DropoutState(torch.zeros(1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32))
    with pytest.raises(ValueError, match="int32"):
        DropoutState(torch.zeros(1, dtype=torch.int64), torch.zeros(1, dtype=torch.int64))
    with pytest.raises(ValueError, match="DropoutState"):
        dropout(x, 0.1, (1, 2), 0)
    with pytest.raises(ValueError, match="probability"):
        GPT2DoubleHeads(dataclasses.replace(GPT2Config.tiny(), resid_pdrop=1.0))
    assert not hasattr(GPT2Config(), "attn_pdrop")


# ---- the tiny model ------------------------------------------------------------------------------------------------
def _tiny(**kw):
    torch.manual_seed(0)
    return GPT2DoubleHeads(dataclasses.replace(GPT2Config.tiny(), **kw))


def _step(model, batch):
    model.zero_grad()
    out = model(**batch)
    out[0].backward()
    return out[0].detach().clone(), {n: p.grad.clone() for n, p in model.named_parameters()}


def test_model_without_dropout_is_unchanged():
    """Probability 0 (given or defaulted) is the model without the fields: same loss and gradient bits, the counter
    untouched; eval() ignores p; state_dict() has the same keys either way."""
    batch = synthetic_batch(2, 2, 32, 512, seed=1)
    plain, zero, on = _tiny(), _tiny(embd_pdrop=0.0, resid_pdrop=0.0, summary_first_dropout=0.0), _tiny(**P3)
    assert not plain.has_dropout and not zero.has_dropout and on.has_dropout
    assert list(plain.state_dict()) == list(on.state_dict()) and "dropout_seed" not in plain.state_dict()
    zero.set_dropout(99, 7)
    l0, g0 = _step(plain, batch)
    l1, g1 = _step(zero, batch)
    assert torch.equal(l0, l1) and all(torch.equal(g0[n], g1[n]) for n in g0)
    assert int(zero.dropout_step) == 7 and int(plain.dropout_step) == 0
    on.set_dropout(99)
    with torch.no_grad():
        assert torch.equal(on.eval()(**batch)[0], plain.eval()(**batch)[0])
    assert int(on.dropout_step) == 0
    l2, _ = _step(on.train(), batch)
    assert not torch.equal(l2, l0) and int(on.dropout_step) == 1


def test_generation_never_drops():
    model = _tiny(**P3)
    model.set_dropout(3)
    ids = synthetic_batch(1, 2, 16, 512, seed=2)["input_ids"][0]
    kw = dict(max_new_tokens=6, temperature=0.0)
    want = model.eval().generate(ids, **kw)
    got = model.train().generate(ids, **kw)
    assert all(torch.equal(a, b) for a, b in zip(want, got)) and int(model.dropout_step) == 0
    cache = model.new_cache(2)
    with torch.no_grad():
        a = model.train().hidden(ids, None, cache)
        b = model.eval().hidden(ids, None, model.new_cache(2))
    assert torch.equal(a, b)
    with pytest.raises(ValueError, match="KV cache"):
        model.hidden(ids, None, cache, drop=model.dropout_state())


@pytest.mark.parametrize("fuse", [True, False])
def test_steps_repeat_from_seed_and_step(fuse):
    batch = synthetic_batch(2, 2, 32, 512, seed=3)
    a, b = _tiny(**P3), _tiny(**P3)
    a.fuse_add_ln = b.fuse_add_ln = fuse
    a.set_dropout(11, 4)
    b.set_dropout(11, 4)
    la, ga = _step(a, batch)
    lb, gb = _step(b, batch)
    assert torch.equal(la, lb) and all(torch.equal(ga[n], gb[n]) for n in ga)
    assert int(a.dropout_step) == 5                          # once per training forward
    l2, _ = _step(a, batch)                                   # the next step draws other masks
    assert int(a.dropout_step) == 6 and not torch.equal(l2, la)
    b.set_dropout(11, 5)
    assert torch.equal(_step(b, batch)[0], l2)               # ... which (seed, step) alone determine
    b.set_dropout(12, 4)
    assert not torch.equal(_step(b, batch)[0], la)


# ---- one training step against fp64 --------------------------------------------------------------------------------
def test_masked_reference_without_dropout_is_the_reference():
    """With every probability 0 the masked reference computes ``ref_step``'s bits, which pins it to the reference that
    is pinned to HuggingFace."""
    cfg = CPU_CFG
    w = base_weights(cfg, 3)
    batch = make_batch(cfg, 2, 2, 32, 4, "cpu")
    g0, l0 = ref_step(leaves(w, torch.float64), batch, 2.0, 0.5, cfg)
    g1, l1 = ref_step_masked(leaves(w, torch.float64), batch, 2.0, 0.5, cfg, seed=5, step=6)
    assert l0 == l1 and all(torch.equal(g0[n], g1[n]) for n in g0)


@pytest.mark.parametrize("fuse", [True, False])
@pytest.mark.parametrize("probs", [P3, dict(embd_pdrop=0.3), dict(resid_pdrop=0.2), dict(summary_first_dropout=0.5)])
def test_model_cpu_path_equals_masked_reference(fuse, probs):
    """The model's CPU path in fp64 against the masked reference (the tolerances of
    ``test_model_cpu_path_equals_reference``); each probability alone shows that its sites and no others are wired."""
    cfg = dataclasses.replace(CPU_CFG, **probs)
    lm_coef, mc_coef = 1.0, 1.0
    w = base_weights(cfg, 3)
    batch = make_batch(cfg, 2, 2, 32, 4, "cpu")
    g64, l64 = ref_step_masked(leaves(w, torch.float64), batch, lm_coef, mc_coef, cfg, seed=21, step=8)
    plain, _ = ref_step(leaves(w, torch.float64), batch, lm_coef, mc_coef, cfg)
    assert _rel_max(plain["h.0.c_fc.weight"], g64["h.0.c_fc.weight"]) > 1e-3        # the masks matter
    model = build_model(cfg, w, "cpu").double()
    model.fuse_add_ln = fuse
    model.set_dropout(21, 7)
    out = model(**batch, lm_coef=lm_coef, mc_coef=mc_coef)
    out[0].backward()
    for name, a, b in zip(("loss", "lm_loss", "mc_loss"), out, l64):
        assert abs(float(a) - b) <= 1e-6 * abs(b), (name, float(a), b)
    for n, p in model.named_parameters():
        err = _rel_max(p.grad, g64[n], _vanishing(n, lm_coef))
        assert err <= 1e-5, (n, err)


# ---- checkpoints ---------------------------------------------------------------------------------------------------
def test_engine_checkpoint_carries_the_dropout_state():
    from adapcc_b200.parallel.engine import FlatDataParallel

    plain = FlatDataParallel(_tiny(), None, world_size=1, param_dtype=torch.float32)
    assert "dropout" not in plain.state_dict()
    plain.close()
    a = FlatDataParallel(_tiny(**P3), None, world_size=1, param_dtype=torch.float32, dropout_seed=40)
    batch = synthetic_batch(2, 2, 32, 512, seed=5)
    with torch.no_grad():
        a.model(**batch)                                       # one training forward (the engine steps on a GPU only)
    sd = a.state_dict()
    assert sd["dropout"] == {"seed": 40, "step": 1}
    b = FlatDataParallel(_tiny(**P3), None, world_size=1, param_dtype=torch.float32, rank=0)
    b.load_state_dict(sd)
    assert int(b.model.dropout_seed) == 40 and int(b.model.dropout_step) == 1
    with torch.no_grad():                                     # the resumed run continues the mask sequence
        assert torch.equal(a.model(**batch)[0], b.model(**batch)[0])
    c = FlatDataParallel(_tiny(**P3), None, world_size=4, rank=3, param_dtype=torch.float32, dropout_seed=40,
                         comm_fn=lambda t: None)
    assert int(c.model.dropout_seed) == 43                    # ranks draw different masks
    assert c.state_dict(consolidate=False)["dropout"]["seed"] == 40      # the file holds the base seed ...
    c.load_state_dict(sd)
    assert int(c.model.dropout_seed) == 43 and int(c.model.dropout_step) == 1   # ... so rank r resumes seed + r
    with pytest.warns(UserWarning, match="no dropout state"):
        c.load_state_dict({k: v for k, v in sd.items() if k != "dropout"})
    with pytest.warns(UserWarning, match="same masks"):
        FlatDataParallel(_tiny(**P3), None, world_size=2, rank=1, param_dtype=torch.float32,
                         comm_fn=lambda t: None).close()
    for e in (a, b, c):
        e.close()


def test_dropout_state_is_not_a_buffer_and_follows_the_module():
    model = _tiny(**P3)
    assert not list(model.buffers()) and "dropout_seed" not in dict(model.named_buffers())
    model.set_dropout(9, 4)
    seed = model.dropout_seed
    model.double().bfloat16().to("cpu")
    assert model.dropout_seed.dtype == torch.int64 and model.dropout_step.dtype == torch.int32
    assert int(model.dropout_seed) == 9 and int(model.dropout_step) == 4 and model.dropout_seed.device == seed.device
    assert model.to("meta").dropout_seed.device.type == "meta"


def test_ddp_leaves_the_dropout_state_alone(tmp_path):
    """2 gloo ranks: DistributedDataParallel broadcasts rank 0's buffers at construction and before every forward. The
    dropout state is not a buffer, so after wrapping and after a forward every rank still holds seed + rank and its
    own step, and the wrapped model has no buffers to synchronise, with dropout on or off."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with socket.socket() as sock:
        sock.bind(("127.0.0.1", 0))
        port = sock.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "cpu_dropout_ddp_worker.py")]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, PYTHONPATH=root, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    rows = re.findall(r"\[rank (\d)\] p ([0-9.]+) sync_buffers (\w+) seed (\d+) step (\d+) (\w+)", r.stdout)
    assert len(rows) == 4, r.stdout
    for rank, p, sync, seed, step, verdict in rows:
        assert verdict == "ok" and sync == "False" and int(seed) == 100 + int(rank), rows
        assert int(step) == 5 * int(rank) + (1 if float(p) else 0), rows
