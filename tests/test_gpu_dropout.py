"""Training dropout on the GPU: the three kernels that draw masks (stand-alone, fused add-LayerNorm, fused embedding
sum) bit for bit against ``ops/dropout.py``'s numpy definition, a captured training step against eager steps, and the
GPT-2 small training step against the masked fp64 reference of tests/test_dropout_cpu.py."""
import dataclasses
from ctypes import c_void_p

import pytest
import torch

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
from adapcc_b200.ops.dropout import DropoutState, dropout, dropout_mask, threshold
from test_dropout_cpu import P3, ref_step_masked
from test_gpu_kernels_reference import (LN_WIDTHS, U16, _add_ln_fwd, _bits_equal, _nan16,  # noqa: F401
                                        _same_bits, _untouched, check_ln, check_ln_bwd, dev, embed_bwd_emulate)
from test_gpu_training_reference import base_weights, build_model, check_step, leaves, make_batch

pytestmark = pytest.mark.gpu
PROBS = [0.0, 0.1, 0.5, 65535 / 65536]


def _keep(rows, cols, p, seed, step, site, device):
    return torch.from_numpy(dropout_mask(rows, cols, p, seed, step, site)).to(device)


def _masked(x, keep, p):
    """fp32 ``mask * scale * x``: the product rounded to fp32 once, zero where dropped."""
    scale = torch.tensor(threshold(p)[1], dtype=torch.float32, device=x.device)
    return torch.where(keep, x.float() * scale, torch.zeros((), device=x.device))


# ---- the stand-alone kernel ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", LN_WIDTHS + [8, 40])
@pytest.mark.parametrize("p", PROBS)
def test_dropout_kernel_mask_bit_exact(dev, d, p):
    """x = 1 makes y the mask times the scale: equal to the definition for the first and last row, row counts around
    the 8 rows and 256 threads of a CTA, several sites, steps and seeds (a negative seed and one above 2^32), bf16 and
    fp32; then random x, forward and backward."""
    scale = threshold(p)[1]
    for rows, seed, step, site in ((1, 0, 0, 0), (7, 1234, 1, 1), (9, -5, 70000, 24), (1031, (1 << 40) + 3, 3, 25)):
        st = DropoutState.create(seed, step, dev)
        keep = _keep(rows, d, p, seed, step, site, dev)
        for dtype in (torch.bfloat16, torch.float32):
            y = dropout(torch.ones(rows, d, dtype=dtype, device=dev), p, st, site)
            assert torch.equal(y != 0, keep), (rows, dtype)
            assert torch.equal(y, (keep * torch.tensor(scale, device=dev)).to(dtype)), (rows, dtype)
            x = torch.randn(rows, d, device=dev).to(dtype).requires_grad_(True)
            y = dropout(x, p, st, site)
            assert torch.equal(y, _masked(x.detach(), keep, p).to(dtype))
            dy = torch.randn(rows, d, device=dev).to(dtype)
            y.backward(dy)
            assert torch.equal(x.grad, _masked(dy, keep, p).to(dtype))
        if p == 0.0:
            assert bool(keep.all())


def test_dropout_kernel_rejects_bad_arguments(dev):
    st = DropoutState.create(1, 0, dev)
    with pytest.raises(ValueError, match="multiple of 8"):
        dropout(torch.ones(4, 12, device=dev), 0.1, st, 0)
    with pytest.raises(ValueError, match="bf16 or fp32"):
        dropout(torch.ones(4, 16, device=dev, dtype=torch.float16), 0.1, st, 0)
    with pytest.raises(ValueError, match="is on"):
        dropout(torch.ones(4, 16, device=dev), 0.1, DropoutState.create(1), 0)


# ---- fused add-LayerNorm with dropout ------------------------------------------------------------------------------
def _drop_tail(p, st, site):
    from adapcc_b200.ops.dropout import drop_tail
    return drop_tail("test", p, st, site, st.seed.device)


def _add_ln_drop_fwd(x, res, gamma, beta, eps, tail):
    """adapcc_add_ln_drop_fwd into NaN-filled outputs with one guard row -> (sum_out, y, mean, rstd)."""
    from adapcc_b200.ops.layers import _lib, _p, _s
    from adapcc_b200.runtime.native import last_error

    rows, d = x.shape
    sum_out, y = _nan16(rows + 1, d, device=x.device), _nan16(rows + 1, d, device=x.device)
    mean = torch.full((rows,), float("nan"), dtype=torch.float32, device=x.device)
    rstd = torch.full((rows,), float("nan"), dtype=torch.float32, device=x.device)
    rc = _lib().adapcc_add_ln_drop_fwd(_p(x), _p(res), _p(gamma), _p(beta), _p(sum_out), _p(y), _p(mean), _p(rstd),
                                       rows, d, eps, *tail, _s())
    assert rc == 0, last_error()
    assert _untouched(sum_out[rows]) and _untouched(y[rows]), "add_ln_drop_fwd wrote past its last row"
    return sum_out[:rows], y[:rows], mean, rstd


def _add_ln_drop_bwd(dy, s, gamma, mean, rstd, dsum, tail):
    """adapcc_add_ln_drop_bwd into NaN-filled outputs with guard rows -> (dx, dres, dgamma, dbeta)."""
    from adapcc_b200.ops.layers import _lib, _p, _s
    from adapcc_b200.runtime.native import last_error

    lib = _lib()
    rows, d = s.shape
    dx, dres = _nan16(rows + 1, d, device=s.device), _nan16(rows + 1, d, device=s.device)
    dgamma, dbeta = _nan16(d, device=s.device), _nan16(d, device=s.device)
    part = torch.empty(2 * lib.adapcc_ln_partials(rows) * d, dtype=torch.float32, device=s.device)
    rc = lib.adapcc_add_ln_drop_bwd(_p(dy), _p(s), _p(gamma), _p(mean), _p(rstd),
                                    c_void_p(0) if dsum is None else _p(dsum), _p(dx), _p(dres), _p(dgamma),
                                    _p(dbeta), _p(part), rows, d, *tail, _s())
    assert rc == 0, last_error()
    assert _untouched(dx[rows]) and _untouched(dres[rows]), "add_ln_drop_bwd wrote past its last row"
    return dx[:rows], dres[:rows], dgamma, dbeta


@pytest.mark.parametrize("d", LN_WIDTHS)
@pytest.mark.parametrize("rows", [1, 7, 9, 4099])
@pytest.mark.parametrize("p", PROBS)
def test_add_layernorm_dropout_against_fp64(dev, d, rows, p):
    """Forward: ``sum_out`` is bf16(fp32(x) + mask scale fp32(res)) bit for bit (the product and the sum each one fp32
    operation, one rounding to bf16), and y, mean, rstd are the LayerNorm of that rounded sum within ``check_ln``'s
    bounds. Backward: dx, dgamma, dbeta within ``check_ln_bwd``'s bounds, as without dropout; dres is exactly zero
    where the mask drops and within one bf16 rounding of mask scale dx elsewhere (the kernel scales its fp32 dx, the
    test only sees the rounded one); a second launch repeats every bit. With p = 0 the forward returns the bits of
    ``adapcc_add_ln_fwd`` and the backward's dres is its dx bit for bit. (The backward with dropout is a separate
    instantiation whose fp32 multiply-adds the assembler may fuse differently, so its dx, dgamma and dbeta are held to
    the fp64 bounds, not to the other instantiation's last bit; a model at p = 0 never runs it.)"""
    g = torch.Generator().manual_seed(7 * d + rows)
    seed, step, site = 991 + rows, 3, 5
    st = DropoutState.create(seed, step, dev)
    tail = _drop_tail(p, st, site)
    x = (torch.randn(rows, d, generator=g) * 2 + 0.5).bfloat16().to(dev)
    res = (torch.randn(rows, d, generator=g) * 0.5).bfloat16().to(dev)
    gamma = (torch.randn(d, generator=g) * 0.5 + 1).bfloat16().to(dev)
    beta = (torch.randn(d, generator=g) * 0.1).bfloat16().to(dev)
    keep = _keep(rows, d, p, seed, step, site, dev)
    s, y, mean, rstd = _add_ln_drop_fwd(x, res, gamma, beta, 1e-5, tail)
    assert _same_bits(s, (x.float() + _masked(res, keep, p)).bfloat16())
    check_ln(y, mean, rstd, s, gamma, beta, 1e-5)
    dy = torch.randn(rows, d, generator=g).bfloat16().to(dev)
    scale = threshold(p)[1]
    for dsum in (None, torch.randn(rows, d, generator=g).bfloat16().to(dev)):
        dx, dres, dgamma, dbeta = _add_ln_drop_bwd(dy, s, gamma, mean, rstd, dsum, tail)
        check_ln_bwd(dx, dgamma, dbeta, dy, s, gamma, mean, rstd, dres=dsum)
        assert bool((dres[~keep] == 0).all())
        want = dx.double() * scale                        # dx is within U16 of the fp32 value the kernel scaled
        err = (dres.double() - want).abs()[keep]
        assert bool((err <= 2.5 * U16 * want.abs()[keep] + 1e-38).all()), float((err / want.abs()[keep]).max())
        again = _add_ln_drop_bwd(dy, s, gamma, mean, rstd, dsum, tail)
        assert all(_same_bits(a, b) for a, b in zip(again, (dx, dres, dgamma, dbeta)))
        if p == 0.0:
            assert _same_bits(dres, dx)
    if p == 0.0:
        plain = _add_ln_fwd(x, res, gamma, beta, 1e-5)
        assert _same_bits(s, plain[0]) and _same_bits(y, plain[1])
        assert torch.equal(mean, plain[2]) and torch.equal(rstd, plain[3])


def test_forward_add_with_dropout_autograd(dev):
    """``FusedLayerNorm.forward_add(drop=...)``: the fused kernels and the unfused fallback (a width the kernels do not
    take goes through ``dropout`` and ``F.layer_norm``) give x and res their own gradients, dres = mask scale dx."""
    from adapcc_b200.ops.layers import FusedLayerNorm

    for d in (768, 64):
        torch.manual_seed(d)
        ln = FusedLayerNorm(d).to(dev).bfloat16()
        st = DropoutState.create(17, 2, dev)
        x = torch.randn(5, 9, d, device=dev).bfloat16().requires_grad_(True)
        res = torch.randn(5, 9, d, device=dev).bfloat16().requires_grad_(True)
        s, y = ln.forward_add(x, res, (0.5, st, 4))
        keep = _keep(45, d, 0.5, 17, 2, 4, dev).view(5, 9, d)
        assert _same_bits(s, (x.detach().float() + _masked(res.detach(), keep, 0.5)).bfloat16())
        (s.float().sum() + (y.float() * torch.randn_like(y.float())).sum()).backward()
        assert bool((res.grad[~keep] == 0).all()) and bool((res.grad[keep] != 0).any())
        err = (res.grad.double() - 2.0 * x.grad.double()).abs()[keep]
        assert bool((err <= 2.5 * U16 * 2.0 * x.grad.double().abs()[keep]).all())


# ---- fused embedding sum with dropout ------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_embedding_dropout_bit_exact(dev, p):
    """wte[ids] + wpe[pos] + wte[tt] at D = 768 with repeated ids and the two token-type rows hit thousands of times.
    Forward: bf16(mask scale fp32 sum) bit for bit. Backward: the exact emulation of the fixed-point arithmetic applied
    to the masked, scaled dY (fp32); a second run gives the same bits."""
    from adapcc_b200.ops import fused_embedding_sum

    g = torch.Generator().manual_seed(int(p * 100))
    N, T, D, V, P = 4, 512, 768, 1000, 512
    n = N * T
    ids = torch.randint(0, V - 2, (N, T), generator=g)
    ids[:, :64] = 7                                            # one row hit 256 times
    tt = torch.randint(V - 2, V, (N, T), generator=g)          # two rows share all 2048 token-type lookups
    pos = torch.arange(T).repeat(N)
    seed, step, site = 2024, 6, 0
    st = DropoutState.create(seed, step, dev)
    keep = _keep(n, D, p, seed, step, site, dev)
    dy = (torch.randn(n, D, generator=g) * torch.logspace(-3, 1, n)[:, None]).bfloat16()
    tables = [(torch.randn(V, D, generator=g) * 0.02).bfloat16(), (torch.randn(P, D, generator=g) * 0.02).bfloat16()]
    idx = [ids.reshape(-1), pos, tt.reshape(-1)]
    # autograd receives fresh gradients here (no engine sink): the kernels accumulate into zeros
    want = embed_bwd_emulate([torch.zeros_like(t) for t in tables], (0, 1, 0), idx, _masked(dy.to(dev), keep, p).cpu())
    first = None
    for _ in range(2):
        wte, wpe = (t.to(dev).requires_grad_(True) for t in tables)
        y = fused_embedding_sum([wte, wpe], [(0, ids.to(dev)), (1, pos.to(dev)), (0, tt.to(dev))], (p, st, site))
        f = [t.detach().float() for t in (wte, wpe)]
        fsum = f[0][idx[0].to(dev)] + f[1][idx[1].to(dev)] + f[0][idx[2].to(dev)]
        assert _same_bits(y, _masked(fsum, keep, p).bfloat16())
        got = [t.cpu() for t in torch.autograd.grad(y, [wte, wpe], dy.to(dev))]
        for j in range(2):
            assert _bits_equal(got[j], want[j]), (j, int((got[j].float() != want[j].float()).sum()))
        assert first is None or all(_bits_equal(a, b) for a, b in zip(got, first))
        first = got


def test_embedding_dropout_unfused_path(dev):
    """fp32 tables take ``F.embedding`` sums and the stand-alone kernel: the same mask."""
    from adapcc_b200.ops import fused_embedding_sum

    torch.manual_seed(0)
    wte = torch.randn(50, 64, device=dev)
    ids = torch.randint(0, 50, (3, 10), device=dev)
    st = DropoutState.create(5, 1, dev)
    y = fused_embedding_sum([wte], [(0, ids)], (0.5, st, 0))
    keep = _keep(30, 64, 0.5, 5, 1, 0, dev)
    assert torch.equal(y, _masked(wte[ids.reshape(-1)], keep, 0.5))


# ---- the model -----------------------------------------------------------------------------------------------------
def _tiny_engine(dev, seed):
    from adapcc_b200.parallel.engine import FlatDataParallel

    torch.manual_seed(0)
    m = GPT2DoubleHeads(dataclasses.replace(GPT2Config.tiny(), **P3)).to(dev)
    return FlatDataParallel(m, None, world_size=1, lr=1e-3, dropout_seed=seed)


def test_graph_replay_equals_eager_and_draws_fresh_masks(dev):
    """One captured step of the tiny bf16 model at p = 0.1, replayed three times, against three eager steps from the
    same parameters, optimizer state, seed and step: losses and parameters bit for bit. The three replays use three
    masks (on one batch, at a learning rate too small to move the loss by itself, the losses differ), and the device
    counter reads start + 3."""
    batch = {k: v.to(dev) for k, v in synthetic_batch(2, 2, 32, 512, seed=9).items()}
    eager, graph = _tiny_engine(dev, 70), _tiny_engine(dev, 70)
    graph.capture(batch, warmup=2)
    for _ in range(2):
        eager.step(batch)
    assert torch.equal(eager.flat_param, graph.flat_param)
    start = 100
    for e in (eager, graph):
        e.model.set_dropout(70, start)
    losses = []
    for i in range(3):
        le, lg = eager.step(batch).clone(), graph.step_graph(batch).clone()
        assert torch.equal(le, lg), (i, float(le), float(lg))
        assert torch.equal(eager.flat_grad, graph.flat_grad), i
        losses.append(float(lg))
    for name in ("flat_param", "master", "exp_avg", "exp_avg_sq"):
        assert torch.equal(getattr(eager, name), getattr(graph, name)), name
    assert len(set(losses)) == 3, losses
    assert int(graph.model.dropout_step) == start + 3 == int(eager.model.dropout_step)
    # the same masks again give the same first loss only from the same parameters: rewind and check the mask alone
    frozen = _tiny_engine(dev, 70)
    frozen.set_lr(0.0)
    frozen.model.set_dropout(70, start)
    a = float(frozen.step(batch))
    b = float(frozen.step(batch))
    frozen.model.set_dropout(70, start)
    assert float(frozen.step(batch)) == a != b
    for e in (eager, graph, frozen):
        e.close()


def _native_step(cfg, w, batch, dev, monkeypatch, fused, seed, step):
    """One engine step at p > 0 -> (gradients by name, loss); ``fused``: the fused add-LayerNorm and embedding kernels,
    otherwise the stand-alone dropout kernel at every site."""
    from adapcc_b200.parallel.engine import FlatDataParallel

    monkeypatch.setenv("ADAPCC_FUSED_EMBED", "1" if fused else "0")
    monkeypatch.setenv("ADAPCC_FUSE_ADD_LN", "1" if fused else "0")
    m = build_model(cfg, w, dev)
    assert m.fuse_add_ln == fused and m.fused_embed == fused
    eng = FlatDataParallel(m, None, world_size=1, dropout_seed=seed)
    m.set_dropout(seed, step)
    loss = eng.step(dict(batch, lm_coef=1.0, mc_coef=1.0))
    names = {id(p): n for n, p in m.named_parameters()}
    grads = {names[id(p)]: eng.flat_grad[o:o + p.numel()].view(p.shape).clone() for p, o in zip(eng.params, eng._offsets)}
    eng.close()
    return grads, loss


def test_gpt2_small_training_step_with_dropout_against_fp64(dev, monkeypatch):
    """GPT-2 small (12 layers, D = 768, the full vocabulary) at B = 1, C = 2, T = 256, p = 0.1 at every site, through
    ``FlatDataParallel``: loss and every parameter gradient against the masked fp64 reference with the rule of
    tests/test_gpu_training_reference.py (the stock arm is the same masked reference in bf16), on the fused path and
    with ``ADAPCC_FUSE_ADD_LN=0 ADAPCC_FUSED_EMBED=0``. The two paths draw the same masks, so they are also held to
    each other: their losses differ by rounding only."""
    cfg = dataclasses.replace(GPT2Config(), **P3)
    w = base_weights(cfg, 41)
    batch = make_batch(cfg, 1, 2, 256, 42, dev)
    seed, step = 4321, 9
    ref = ref_step_masked(leaves(w, torch.float64, dev), batch, 1.0, 1.0, cfg, seed, step + 1)
    stock = ref_step_masked(leaves(w, torch.bfloat16, dev), batch, 1.0, 1.0, cfg, seed, step + 1)
    plain_loss = ref_step_masked(leaves(w, torch.float64, dev), batch, 1.0, 1.0, dataclasses.replace(cfg, embd_pdrop=0.0,
                                 resid_pdrop=0.0, summary_first_dropout=0.0), seed, step + 1)[1][0]
    assert abs(plain_loss - ref[1][0]) > 1e-3 * abs(plain_loss)             # the masks matter at this shape
    losses = {}
    for fused in (True, False):
        g, loss = _native_step(cfg, w, batch, dev, monkeypatch, fused, seed, step)
        ratio, where = check_step(g, (loss, None, None), ref, stock, cfg, batch, (1.0, 1.0), w, wpe_m_factor=3.0)
        print(f"[dropout] GPT-2 small, fused {fused}: largest e_nat / e_stock {ratio:.2f} at {where}")
        losses[fused] = float(loss)
    assert abs(losses[True] - losses[False]) <= 4 * U16 * abs(ref[1][0]), losses
