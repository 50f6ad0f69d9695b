"""The hand-written kernels against fp64 (or exact) references at the shapes and values where kernels go wrong.

Every checker compares one kernel output with a reference computed in fp64 from the same bf16 / fp32 inputs, per
element, against a bound derived next to it from the arithmetic the kernel does (output rounding, fp32 accumulation
depth, ``tanh.approx``). Each checker also has a CPU self-test that feeds it a slightly wrong copy of the reference and
expects a failure, so a subtly wrong kernel cannot pass. The fixed-point embedding backward is checked bit for bit
against an exact numpy emulation of its specified arithmetic; the emulation itself is checked on the CPU against fp64.

GPU tests are marked one by one: the emulator and self-tests run without a device.
"""
import math
import os

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

U32 = 2.0 ** -24          # unit roundoff of fp32 (round to nearest)
U16 = 2.0 ** -8           # unit roundoff of bf16 (8 significant bits)
# tanh.approx.f32: maximum relative error 2^-11 (PTX ISA); one bit of margin
TANH_REL = 2.0 ** -10


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)           # the in-tree .so must be the code under test
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


def assert_within(got, ref, bound, what):
    """|got - ref| <= bound element by element (NaN in got fails)."""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.flatten())[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound; first at flat index "
                             f"{i}: got {float(got.double().flatten()[i])!r} want {float(ref.flatten()[i])!r} "
                             f"bound {float(bound.flatten()[i]) if torch.is_tensor(bound) else bound!r}")


# ---- GEMM ----------------------------------------------------------------------------------------------------------
def _gemm_ref(x, w):
    """(fp64 A.W^T, accumulation bound). The products of bf16 operands are exact in fp32; fp32 accumulation of K of
    them in any order is off by at most K * 2^-23 * sum |a||w| (two units per add leaves room for a tensor core that
    truncates instead of rounding)."""
    x64, w64 = x.double(), w.double()
    k = x.shape[1]
    return x64 @ w64.t(), k * 2.0 ** -23 * (x64.abs() @ w64.abs().t())


def check_gemm_pre(pre, x, w, b):
    """pre = bf16(A.W^T + bias): accumulation bound, fp32 bias add (U32), then one bf16 rounding (U16)."""
    acc, accb = _gemm_ref(x, w)
    ref = acc + (b.double() if b is not None else 0.0)
    e = accb + U32 * ref.abs()
    assert_within(pre, ref, e + U16 * (ref.abs() + e), "gemm pre")


def _gelu_parts(a):
    k, c = math.sqrt(2.0 / math.pi), 0.044715
    u = k * (a + c * a ** 3)
    t = torch.tanh(u)
    # tanh.approx's own error plus the fp32 evaluation of its argument (3 roundings, |d tanh / du| <= 1)
    dt = TANH_REL * t.abs() + 3 * U32 * u.abs()
    return t, dt, k * (1 + 3 * c * a * a)


def check_gelu(out, pre):
    """out = bf16(gelu_tanh(pre)) with the kernel's own bf16 pre-activation as input: 0.5 a (1 + t) moves by 0.5 |a| dt
    for an error dt in t; fp32 products and the fma add 4 U32 relative; then one bf16 rounding."""
    a = pre.double()
    t, dt, _ = _gelu_parts(a)
    ref = 0.5 * a * (1 + t)
    e = 0.5 * a.abs() * dt + 4 * U32 * (0.5 * a.abs() * (1 + t.abs()))
    assert_within(out, ref, e + U16 * (ref.abs() + e), "gelu epilogue")


def check_dgelu(out, x, w, aux):
    """out = bf16((A.W^T) * gelu'(aux)), gelu'(a) = 0.5 (1 + t) + 0.5 a (1 - t^2) du: d gelu' / dt = 0.5 - a t du, so an
    error dt in t moves it by dt (0.5 + |a t| du); 8 fp32 roundings of the terms; accumulation error times |gelu'|."""
    acc, accb = _gemm_ref(x, w)
    a = aux.double()
    t, dt, du = _gelu_parts(a)
    d = 0.5 * (1 + t) + 0.5 * a * (1 - t * t) * du
    derr = dt * (0.5 + (a * t).abs() * du) + 8 * U32 * (1 + (a * du).abs())
    ref = acc * d
    e = d.abs() * accb + (acc.abs() + accb) * derr + 2 * U32 * ref.abs()
    assert_within(out, ref, e + U16 * (ref.abs() + e), "dgelu epilogue")


def check_residual(out, x, w, b, aux):
    """out = bf16(bf16(A.W^T + bias) + aux): accumulation + bias add, the projection's bf16 rounding, then the add's."""
    acc, accb = _gemm_ref(x, w)
    u = acc + b.double()
    e1 = accb + U32 * u.abs()
    e1 = e1 + U16 * (u.abs() + e1)
    ref = u + aux.double()
    assert_within(out, ref, e1 + U16 * (ref.abs() + e1), "residual epilogue")


def check_colsum(colsum, out):
    """fp32 column sums of the kernel's own bf16 output: any fp32 summation order of `rows` terms is off by at most
    (rows - 1) U32 sum |out|; +16 for the per-warp and per-tile partials."""
    o = out.double()
    rows = o.shape[0]
    assert_within(colsum, o.sum(0), (rows + 16) * U32 * o.abs().sum(0), "gemm colsum")


GEMM_M = [1, 8, 127, 129, 255, 257]
# Shapes where a persistent CTA (132 of them) or CTA pair (66) computes many tiles one after the other, so the stage
# ring's barrier parity, the epilogue staging ring and the aux prefetch all carry over from tile to tile:
GEMM_MANY_TILES = [
    (3072, 768, 8192),      # GPT-2's MLP up-projection: 384 pair tiles over 66 pairs, unevenly (5 or 6 each)
    (768, 3072, 8192),      # ... and its down-projection: 96 pair tiles, 48 K slabs = 16 trips round the 3-stage ring
    (3072, 768, 8193),      # odd number of row tiles: the last pair's second half is empty on all 12 column tiles
    (1024, 64, 40000),      # one K slab per tile, 9 or 10 tiles per pair: each stage of the ring serves a different
                            # tile on every use and its barrier parity goes 0, 1, 0 within one launch
    (384, 768, 20000),      # 128-wide tiles (variants 0 / 1): 471 tiles over the persistent CTAs
]
GEMM_CASES = [(n, k, m) for n, k in ((256, 192), (384, 768)) for m in GEMM_M] + GEMM_MANY_TILES


@gpu
@pytest.mark.parametrize("n,k,m", GEMM_CASES)
def test_gemm_against_fp64(dev, m, n, k):
    """Every variant at ragged M (one row, below one tile, one past a tile, odd numbers of row tiles for the CTA-pair
    variants), 256-wide (N % 256 == 0) and 128-wide tiles, with and without bias; `pre` against the fp64 GEMM and `out`
    against fp64 GELU of the kernel's own `pre`; the aux epilogues (dGELU, residual, column sums) at the same shapes,
    their aux holding values up to +-40 where gelu' has saturated to 1 or 0.
    Variants differ only in which CTA computes a tile: the K-slab order, the wgmma sequence and the swizzled smem layout
    (a multicast half lands exactly where a plain load would) are the same, so the bits must be identical. Variant 0
    launches one CTA per tile, so at the many-tile shapes this equality pins the persistent variants' tile-to-tile
    state exactly."""
    from adapcc_b200.ops.gemm import linear_act

    torch.manual_seed(1000 * m + n + k)
    x = torch.randn(m, k, device=dev).bfloat16()
    w = (torch.randn(n, k, device=dev) / k ** 0.5).bfloat16()
    b = torch.randn(n, device=dev).bfloat16()
    variants = [0, 1, 2, 3] if n % 256 == 0 else [0, 1]
    for act in ("none", "gelu"):
        for bias in (b, None):
            res = {v: linear_act(x, w, bias, act, save_pre=True, variant=v) for v in variants}
            out, pre = res[0]
            check_gemm_pre(pre, x, w, bias)
            if act == "none":
                assert torch.equal(out, pre)
            else:
                check_gelu(out, pre)
            for v in variants[1:]:
                assert torch.equal(res[v][0], out) and torch.equal(res[v][1], pre), (act, bias is None, v)
    del res
    aux = torch.randn(m, n, device=dev)
    at = torch.arange(0, m * n, 97, device=dev)                     # 97 is coprime to every N here: all columns are hit
    aux.view(-1)[at] = torch.tensor([3.0, -3.0, 6.0, -6.0, 12.0, -12.0, 40.0, -40.0], device=dev)[(at // 97) % 8]
    aux = aux.bfloat16()
    dg, _ = linear_act(x, w, None, "dgelu", aux=aux, variant=0)
    check_dgelu(dg, x, w, aux)
    rs, _ = linear_act(x, w, b, "residual", aux=aux, variant=0)
    check_residual(rs, x, w, b, aux)
    if n % 256 == 0:
        cs = torch.zeros(n, dtype=torch.float32, device=dev)
        dg3, _ = linear_act(x, w, None, "dgelu", aux=aux, colsum=cs, variant=3)
        assert torch.equal(dg3, dg)
        check_colsum(cs, dg3)


def test_gemm_checkers_reject_perturbed_reference():
    torch.manual_seed(0)
    m, n, k = 64, 128, 768
    x = torch.randn(m, k).bfloat16()
    w = (torch.randn(n, k) / k ** 0.5).bfloat16()
    b = torch.randn(n).bfloat16()
    x64, w64, b64 = x.double(), w.double(), b.double()
    exact = x64 @ w64.t() + b64
    check_gemm_pre(exact.bfloat16(), x, w, b)
    slab = x64[:, 64:128] @ w64[:, 64:128].t()                     # one K-slab of 64 dropped
    with pytest.raises(AssertionError):
        check_gemm_pre(exact - slab, x, w, b)
    pre = exact.bfloat16()
    a = pre.double()
    gelu = 0.5 * a * (1 + torch.tanh(math.sqrt(2 / math.pi) * (a + 0.044715 * a ** 3)))
    check_gelu(gelu.bfloat16(), pre)
    with pytest.raises(AssertionError):
        check_gelu(gelu * 1.01, pre)
    aux = torch.randn(m, n).bfloat16()
    t, _, du = _gelu_parts(aux.double())
    dref = (x64 @ w64.t()) * (0.5 * (1 + t) + 0.5 * aux.double() * (1 - t * t) * du)
    check_dgelu(dref.bfloat16(), x, w, aux)
    with pytest.raises(AssertionError):
        check_dgelu(dref * 1.01, x, w, aux)
    rref = exact.bfloat16().double() + aux.double()
    check_residual(rref.bfloat16(), x, w, b, aux)
    with pytest.raises(AssertionError):
        check_residual(rref - slab, x, w, b, aux)
    out = dref.bfloat16()
    check_colsum(out.double().sum(0), out)
    with pytest.raises(AssertionError):
        check_colsum(out.double()[1:].sum(0), out)                  # one row missing


# ---- fused cross-entropy -------------------------------------------------------------------------------------------
def check_ce(grad, row_loss, logits, labels, vocab, gs, exp_rounding):
    """grad = bf16((softmax - onehot) * gs) per element, row_loss = logsumexp - logit[label] per row (fp32).

    Relative to p * gs (p = fp64 softmax): the stored exponentials' bf16 rounding (`exp_rounding`: U16 for the
    shared-memory kernel, 0 for the one that recomputes them), __expf (2^-21 plus 2^-23 per unit of |x - max|), the
    fp32 sum of exponentials (per-thread run of stride / 512 terms, the warp and block trees, the online rescaling:
    (stride / 512 + 64) 2^-21); then the output rounding U16 of |grad|; 2^-120 absolute for results that underflow.
    The loss: log(sum) carries the sum's relative error plus __logf's 2^-21, and the fp32 adds 4 U32 of the terms."""
    x = logits.double()[:, :vocab]
    rows, stride = logits.shape
    valid = labels >= 0
    lab = labels.clamp(min=0)
    mx = x.max(1, keepdim=True).values
    lse = torch.logsumexp(x, 1, keepdim=True)
    p = torch.exp(x - lse)
    onehot = torch.zeros_like(p)
    onehot[torch.arange(rows, device=x.device), lab] = 1.0
    v = valid.double()[:, None]
    ref = (p - onehot) * gs * v
    eps_sum = (stride / 512 + 64) * 2.0 ** -21
    eps_exp = 2.0 ** -21 + (x - mx).abs() * 2.0 ** -23
    e = gs * p * (exp_rounding + eps_sum + eps_exp) * v + 2.0 ** -120 * gs
    want = torch.zeros(rows, stride, dtype=torch.float64, device=x.device)
    want[:, :vocab] = ref
    bound = torch.full_like(want, 2.0 ** -120 * gs)
    bound[:, :vocab] = e + U16 * (ref.abs() + e)
    assert_within(grad, want, bound, "fused_ce gradient")
    xl = x.gather(1, lab[:, None])
    loss_ref = ((lse - xl) * v)[:, 0]
    lb = (eps_sum + 2.0 ** -20 + 4 * U32 * ((lse - mx).abs() + mx.abs() + xl.abs()))[:, 0]
    assert_within(row_loss, loss_ref, lb, "fused_ce row loss")


def _ce_case(rows, vocab, stride, seed, dev):
    g = torch.Generator(device="cpu").manual_seed(seed)
    logits = (torch.randn(rows, stride, generator=g) * 3).bfloat16()
    labels = torch.randint(0, vocab, (rows,), generator=g)
    if rows >= 8:
        labels[0], labels[1] = 0, vocab - 1                        # first and last vocabulary entries
        labels[5::7] = -100
        logits[2, :] = torch.where(torch.rand(stride, generator=g) < 0.5, 60.0, -60.0).bfloat16()
        logits[3, :] = -60.0                                        # label certain: p ~ 1, loss ~ 0
        logits[3, labels[3]] = 60.0
        logits[4, :] = 60.0                                         # a flat row at the largest logit
    return logits.to(dev), labels.to(dev)


@gpu
@pytest.mark.parametrize("v1", [False, True])
@pytest.mark.parametrize("rows,vocab,stride,scaled", [
    (37, 50257, 50264, False),      # GPT-2's vocabulary: vocab % 8 == 1, 7 padding columns
    (16, 1001, 1016, True),         # 15 padding columns: a whole 16-byte vector of padding
    (64, 1000, 1000, True),         # no padding
    (8, 1000, 1000, False),         # every row ignored (set below)
    (4, 110000, 110000, False),     # a row too wide for shared memory: the recomputing kernel either way
])
def test_fused_ce_against_fp64(dev, monkeypatch, v1, rows, vocab, stride, scaled):
    from adapcc_b200.ops import fused_ce_

    monkeypatch.setenv("ADAPCC_CE_V1", "1" if v1 else "0")
    logits, labels = _ce_case(rows, vocab, stride, rows + vocab, dev)
    if rows == 8:
        labels[:] = -100
    gs = 0.125 if scaled else 1.0
    work = logits.clone()
    row_loss = fused_ce_(work, labels, vocab, grad_scale=torch.tensor([gs], device=dev) if scaled else None)
    smem = not v1 and stride * 2 <= 200 * 1024
    check_ce(work, row_loss, logits, labels, vocab, gs, U16 if smem else 0.0)
    if rows == 8:
        assert torch.all(work == 0) and torch.all(row_loss == 0)


def test_ce_checker_rejects_perturbed_reference():
    rows, vocab, stride = 16, 1001, 1016
    logits, labels = _ce_case(rows, vocab, stride, 3, "cpu")
    x = logits.double()[:, :vocab]
    p = torch.softmax(x, 1)
    onehot = torch.nn.functional.one_hot(labels.clamp(min=0), vocab).double()
    v = (labels >= 0).double()[:, None]
    grad = torch.zeros(rows, stride, dtype=torch.float64)
    grad[:, :vocab] = (p - onehot) * v * 0.5
    loss = ((torch.logsumexp(x, 1) - x.gather(1, labels.clamp(min=0)[:, None])[:, 0]) * v[:, 0])
    check_ce(grad.bfloat16(), loss.float(), logits, labels, vocab, 0.5, 0.0)
    with pytest.raises(AssertionError):
        check_ce(grad * 1.01, loss, logits, labels, vocab, 0.5, 0.0)
    swapped = loss.clone()
    swapped[[6, 7]] = loss[[7, 6]]
    with pytest.raises(AssertionError):
        check_ce(grad, swapped, logits, labels, vocab, 0.5, 0.0)


def test_fused_ce_rejects_bad_labels():
    """Checked before anything is launched: the kernel reads labels[row] as int64 for every row."""
    from adapcc_b200.ops import fused_ce_

    logits = torch.zeros(4, 16, dtype=torch.bfloat16)
    for labels in (torch.zeros(4, dtype=torch.int32), torch.zeros(8, dtype=torch.int64)[::2],
                   torch.zeros(3, dtype=torch.int64), torch.zeros(5, dtype=torch.int64)):
        with pytest.raises(ValueError):
            fused_ce_(logits, labels, 16)


# ---- LayerNorm statistics and column sums ---------------------------------------------------------------------------
def check_ln(y, mean, rstd, x, gamma, beta, eps):
    """One warp per row: each lane sums D / 32 values, then 5 shuffle levels: depth = D / 32 + 6 fp32 roundings of
    partial sums bounded by sum |x|. The variance is the two-pass sum of (x - mean_f)^2 = exact + D dmean^2, with the
    same depth plus 3 roundings per term; rsqrtf adds 2^-22 relative, half the variance's relative error carries over.
    y = (x - mean) rstd gamma + beta: the statistics' errors times |gamma|, 4 fp32 roundings, one bf16 rounding."""
    x64 = x.double()
    rows, d = x64.shape
    depth = d / 32 + 6
    mu = x64.mean(1)
    var = ((x64 - mu[:, None]) ** 2).mean(1)
    rs = 1.0 / torch.sqrt(var + eps)
    dmu = depth * U32 * x64.abs().mean(1) + U32 * mu.abs()
    assert_within(mean, mu, dmu, "layernorm mean")
    drs = rs * (0.5 * ((depth + 5) * U32 * var + dmu * dmu) / (var + eps) + 2 * U32 + 2.0 ** -22)
    assert_within(rstd, rs, drs, "layernorm rstd")
    g64, b64 = gamma.double(), beta.double()
    xc = x64 - mu[:, None]
    ref = xc * rs[:, None] * g64 + b64
    e = g64.abs() * (xc.abs() * drs[:, None] + dmu[:, None] * rs[:, None]) \
        + 4 * U32 * ((xc * rs[:, None] * g64).abs() + b64.abs())
    assert_within(y, ref, e + U16 * (ref.abs() + e), "layernorm y")


def _ln_fwd(x, gamma, beta, eps):
    from adapcc_b200.ops.layers import _lib, _p, _s

    rows, d = x.shape
    y = torch.empty_like(x)
    mean = torch.empty(rows, dtype=torch.float32, device=x.device)
    rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
    assert _lib().adapcc_ln_fwd(_p(x), _p(gamma), _p(beta), _p(y), _p(mean), _p(rstd), rows, d, eps, _s()) == 0
    return y, mean, rstd


def _ln_input(rows, d, kind, g):
    x = torch.randn(rows, d, generator=g) * 2 + 0.5
    if kind == "constant":
        x[::2] = 3.0                                  # every other row constant: variance exactly 0
    elif kind == "offset":
        x = 256.0 + torch.randn(rows, d, generator=g) * 4   # mean 64x the spread: one-pass E[x^2] - E[x]^2 fails
    return x.bfloat16()


@gpu
@pytest.mark.parametrize("d", [256, 512, 768, 1024])
@pytest.mark.parametrize("rows", [1, 7, 9, 4099])
@pytest.mark.parametrize("kind", ["normal", "constant", "offset"])
def test_layernorm_statistics_against_fp64(dev, d, rows, kind):
    g = torch.Generator().manual_seed(d + rows)
    x = _ln_input(rows, d, kind, g).to(dev)
    gamma = (torch.randn(d, generator=g) * 0.5 + 1).bfloat16().to(dev)
    beta = (torch.randn(d, generator=g) * 0.1).bfloat16().to(dev)
    y, mean, rstd = _ln_fwd(x, gamma, beta, 1e-5)
    check_ln(y, mean, rstd, x, gamma, beta, 1e-5)


def test_ln_checker_rejects_perturbed_reference():
    g = torch.Generator().manual_seed(0)
    x = _ln_input(9, 512, "normal", g)
    gamma = (torch.randn(512, generator=g) * 0.5 + 1).bfloat16()
    beta = (torch.randn(512, generator=g) * 0.1).bfloat16()
    x64 = x.double()
    mu = x64.mean(1)
    rs = 1.0 / torch.sqrt(((x64 - mu[:, None]) ** 2).mean(1) + 1e-5)
    y = ((x64 - mu[:, None]) * rs[:, None] * gamma.double() + beta.double())
    check_ln(y.bfloat16(), mu.float(), rs.float(), x, gamma, beta, 1e-5)
    with pytest.raises(AssertionError):
        check_ln(y, mu[[1, 0] + list(range(2, 9))], rs, x, gamma, beta, 1e-5)   # one row's statistics swapped
    with pytest.raises(AssertionError):
        check_ln(y, mu, rs[[1, 0] + list(range(2, 9))], x, gamma, beta, 1e-5)


# ---- fused add-LayerNorm forward -------------------------------------------------------------------------------------
LN_WIDTHS = [256, 512, 768, 1024]
# one row, one short of / exactly / one past a CTA's 8 rows, two unequal passes of the persistent grid at every
# width (4099), and about ten passes with idle CTAs and a 3-row group in the last one (20011)
LN_ROWS = [1, 7, 8, 9, 4099, 20011]
NAN16 = 0x7FC0            # the bf16 quiet NaN torch.full writes: the bit pattern of untouched output


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def _nan16(*shape, device):
    return torch.full(shape, float("nan"), dtype=torch.bfloat16, device=device)


def _untouched(t):
    return bool((t.view(torch.int16) == NAN16).all())


def _add_ln_fwd(x, res, gamma, beta, eps):
    """adapcc_add_ln_fwd into NaN-filled outputs with one guard row past `rows` -> (sum_out, y, mean, rstd)."""
    from adapcc_b200.ops.layers import _lib, _p, _s
    from adapcc_b200.runtime.native import last_error

    rows, d = x.shape
    sum_out, y = _nan16(rows + 1, d, device=x.device), _nan16(rows + 1, d, device=x.device)
    mean = torch.full((rows,), float("nan"), dtype=torch.float32, device=x.device)
    rstd = torch.full((rows,), float("nan"), dtype=torch.float32, device=x.device)
    rc = _lib().adapcc_add_ln_fwd(_p(x), _p(res), _p(gamma), _p(beta), _p(sum_out), _p(y), _p(mean), _p(rstd), rows, d,
                                  eps, _s())
    assert rc == 0, last_error()
    assert _untouched(sum_out[rows]) and _untouched(y[rows]), "add_ln_fwd wrote past its last row"
    return sum_out[:rows], y[:rows], mean, rstd


def _add_ln_input(rows, d, kind, g):
    """(x, res) whose sum is an `_ln_input` kind, nearly cancels, or is exactly constant on every other row."""
    if kind == "cancel":
        x = _ln_input(rows, d, "normal", g)
        return x, (-x.float() + torch.randn(rows, d, generator=g) * 0.01).bfloat16()   # sum ~ 0.01, spacing of x ~ 0.01
    if kind == "constsum":
        x = torch.randint(-32, 33, (rows, d), generator=g).float()                     # small integers: exact in bf16
        res = torch.randn(rows, d, generator=g)
        res[::2] = 3.0 - x[::2]                                                         # x + res = 3 exactly: variance 0
        return x.bfloat16(), res.bfloat16()
    return _ln_input(rows, d, kind, g), (torch.randn(rows, d, generator=g) * 0.5).bfloat16()


@gpu
@pytest.mark.parametrize("d", LN_WIDTHS)
@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("kind", ["normal", "offset", "cancel", "constsum"])
def test_add_layernorm_forward_against_fp64(dev, d, rows, kind):
    """The fused residual add: `sum_out` is the bf16 add bit for bit (one fp32 add, one rounding to nearest), and y,
    mean, rstd are the LayerNorm of that ROUNDED sum, held to the bounds of `check_ln`."""
    g = torch.Generator().manual_seed(3 * d + rows)
    x, res = (t.to(dev) for t in _add_ln_input(rows, d, kind, g))
    gamma = (torch.randn(d, generator=g) * 0.5 + 1).bfloat16().to(dev)
    beta = (torch.randn(d, generator=g) * 0.1).bfloat16().to(dev)
    s, y, mean, rstd = _add_ln_fwd(x, res, gamma, beta, 1e-5)
    assert _same_bits(s, x + res)
    if kind == "constsum":
        assert torch.all(s[::2] == 3.0)
    check_ln(y, mean, rstd, s, gamma, beta, 1e-5)


@gpu
def test_add_layernorm_forward_rejects_null_residual(dev):
    """Without `res` or `sum_out` the entry point reports an error and launches nothing."""
    from ctypes import c_void_p

    from adapcc_b200.ops.layers import _lib, _p, _s
    from adapcc_b200.runtime.native import last_error

    lib = _lib()
    rows, d = 9, 256
    x = torch.randn(rows, d, device=dev).bfloat16()
    gamma, beta = torch.ones(d, device=dev).bfloat16(), torch.zeros(d, device=dev).bfloat16()
    s, y = _nan16(rows, d, device=dev), _nan16(rows, d, device=dev)
    mean, rstd = torch.zeros(rows, device=dev), torch.zeros(rows, device=dev)
    before = lib.adapcc_launch_count()
    for res_p, sum_p in ((c_void_p(0), _p(s)), (_p(x), c_void_p(0))):
        assert lib.adapcc_add_ln_fwd(_p(x), res_p, _p(gamma), _p(beta), sum_p, _p(y), _p(mean), _p(rstd), rows, d, 1e-5,
                                     _s()) == -1
        assert "res and sum_out" in last_error()
    torch.cuda.synchronize()
    assert lib.adapcc_launch_count() == before
    assert _untouched(s) and _untouched(y)


# ---- LayerNorm backward --------------------------------------------------------------------------------------------
def _g(k):
    """k successive fp32 roundings move a value by at most k u / (1 - k u), relatively."""
    return k * U32 / (1 - k * U32)


def _ln_bwd_terms(dy, x, gamma, mean, rstd):
    """fp64 (xh, gy, c1, c2, rstd column) of the backward, from the fp32 statistics it is handed."""
    rs = rstd.double()[:, None]
    xh = (x.double() - mean.double()[:, None]) * rs
    gy = dy.double() * gamma.double()
    return xh, gy, gy.mean(1, keepdim=True), (gy * xh).mean(1, keepdim=True), rs


def check_ln_bwd(dx, dgamma, dbeta, dy, x, gamma, mean, rstd, dres=None):
    """dx = bf16(rstd (gy - c1 - xh c2) [+ dres]), dgamma = bf16(sum_rows dy xh), dbeta = bf16(sum_rows dy), with
    xh = (x - mean) rstd, gy = dy gamma, c1 = mean_D(gy), c2 = mean_D(gy xh).

    `mean` / `rstd` are the forward kernel's own fp32 outputs, taken as exact inputs here: `check_ln` bounds them
    against fp64, so the two checks compose into one of the whole LayerNorm.

    What the kernel rounds (fp32 unless said), each term of the bounds below in the same order:
      xh    two roundings (the subtraction, the product); gy = dy gamma is exact (8 x 8 significant bits).
      c1    a lane adds D / 32 values, 5 shuffle levels, the product with the rounded 1 / D: D / 32 + 6 roundings of
            partial sums bounded by sum |gy|.
      c2    the same tree over gy xh, whose terms carry xh's two roundings and the product's: D / 32 + 9, of
            sum |gy xh|.
      dx    gy and c1 go through gy - c1, the subtraction of xh c2 and the product with rstd (3 roundings); xh c2
            through xh's two, its product and the same last two (5). With dres one more rounding of the sum. Then ONE
            bf16 rounding. Everything is relative to rstd (|gy| + |c1| + |xh c2|), not to |dx|: the terms cancel.
      dgamma, dbeta   fp32 sums of `rows` terms in whatever order the per-lane, per-CTA and finalising passes take
            (rows + 64 roundings covers any order, as in `check_colsum_bf16`); a dgamma term also carries xh's two
            roundings and the product's; then one bf16 rounding."""
    xh, gy, c1, c2, rs = _ln_bwd_terms(dy, x, gamma, mean, rstd)
    rows, d = xh.shape
    depth = d / 32 + 6
    dc1 = _g(depth) * gy.abs().mean(1, keepdim=True)
    dc2 = _g(depth + 3) * (gy * xh).abs().mean(1, keepdim=True)
    ref = rs * (gy - c1 - xh * c2)
    e = rs * (dc1 + xh.abs() * dc2 + _g(3) * (gy.abs() + c1.abs() + dc1) + _g(5) * xh.abs() * (c2.abs() + dc2))
    if dres is not None:
        ref = ref + dres.double()
        e = e + U32 * (ref.abs() + e)
    assert_within(dx, ref, e + U16 * (ref.abs() + e), "layernorm dx")
    for got, term, per_term, what in ((dgamma, dy.double() * xh, 3, "dgamma"), (dbeta, dy.double(), 0, "dbeta")):
        want = term.sum(0)
        e = _g(rows + 64 + per_term) * term.abs().sum(0)
        assert_within(got, want, e + U16 * (want.abs() + e), f"layernorm {what}")


def _ln_bwd_grid(rows, d):
    """The backward's persistent grid (csrc/ops_norm.cu): 8 rows per CTA pass, at most 2 CTAs per SM (1 at D = 1024),
    shrunk until every CTA runs the same number of passes but the last."""
    groups = max(1, -(-rows // 8))
    cap = torch.cuda.get_device_properties(0).multi_processor_count * (2 if d <= 768 else 1)
    iters = -(-groups // cap)
    return -(-groups // iters)


def _sparse_rows(rows, grid):
    """Row 0, the last row, and a row of the last 8-row group that the middle CTA of `grid` runs."""
    groups, c = -(-rows // 8), grid // 2
    last_group = c + (groups - 1 - c) // grid * grid
    return sorted({0, rows - 1, min(last_group * 8 + 3, rows - 1)})


def _ln_bwd_case(rows, d, xkind, dykind, keep, g, device):
    """-> (x, dy, gamma). dykind "random": gamma has zeros and negative entries; "rowconst": dy constant along each row
    and gamma constant, so gy = c1 and dx cancels to the rounding of c2; "sparse": "random" with dy zero outside the
    rows `keep`, so every surviving term of dgamma / dbeta is visible at full precision."""
    x = _ln_input(rows, d, xkind, g)
    if dykind == "rowconst":
        gamma = torch.full((d,), 1.5)
        dy = (torch.randn(rows, 1, generator=g) * 2).expand(rows, d)
    else:
        gamma = torch.randn(d, generator=g) * 0.5 + 1
        gamma[::5] = 0.0
        gamma[1::7] *= -1.0
        dy = torch.randn(rows, d, generator=g)
        if dykind == "sparse":
            mask = torch.zeros(rows, 1)
            mask[keep] = 1.0
            dy = dy * mask
    return x.to(device), dy.bfloat16().contiguous().to(device), gamma.bfloat16().to(device)


def _ln_bwd(dy, x, gamma, mean, rstd, dres=None, add=False):
    """adapcc_ln_bwd (or adapcc_add_ln_bwd when `add`) into NaN-filled outputs -> (dx, dgamma, dbeta, part).

    `part` is handed over at exactly 2 * adapcc_ln_partials(rows) * d floats, NaN-filled, with NaN guards behind it;
    dx has one guard row. Neither guard may change."""
    from ctypes import c_void_p

    from adapcc_b200.ops.layers import _lib, _p, _s
    from adapcc_b200.runtime.native import last_error

    lib = _lib()
    rows, d = x.shape
    dx, dgamma, dbeta = _nan16(rows + 1, d, device=x.device), _nan16(d, device=x.device), _nan16(d, device=x.device)
    n = 2 * lib.adapcc_ln_partials(rows) * d
    scratch = torch.full((n + 1024,), float("nan"), dtype=torch.float32, device=x.device)
    if add:
        rc = lib.adapcc_add_ln_bwd(_p(dy), _p(x), _p(gamma), _p(mean), _p(rstd),
                                   c_void_p(0) if dres is None else _p(dres), _p(dx), _p(dgamma), _p(dbeta),
                                   _p(scratch), rows, d, _s())
    else:
        assert dres is None
        rc = lib.adapcc_ln_bwd(_p(dy), _p(x), _p(gamma), _p(mean), _p(rstd), _p(dx), _p(dgamma), _p(dbeta),
                               _p(scratch), rows, d, _s())
    assert rc == 0, last_error()
    assert _untouched(dx[rows]), "ln_bwd wrote past its last row"
    assert bool(torch.isnan(scratch[n:]).all()), "ln_bwd wrote past its scratch"
    return dx[:rows], dgamma, dbeta, scratch[:n]


@gpu
@pytest.mark.parametrize("d", LN_WIDTHS)
@pytest.mark.parametrize("rows", LN_ROWS)
@pytest.mark.parametrize("xkind", ["normal", "constant", "offset"])
def test_layernorm_backward_against_fp64(dev, d, rows, xkind):
    """Both entry points, with and without the residual-stream gradient, for every kind of dy. Constant rows of x have
    xh = 0 and rstd = 1 / sqrt(eps): dx is rstd (gy - c1) alone, 316 times the usual scale.

    Scratch layout: the dgamma partials are rows 0 .. grid - 1 of `part`, the dbeta partials start at grid * d (not
    at the half-way point), and nothing past 2 * grid * d is written; at d = 1024 the grid is smaller than
    adapcc_ln_partials(rows). The fp32 partials, summed in fp64, are held to dgamma's and dbeta's bounds WITHOUT the
    output rounding.

    Bits: the two entry points agree without dres; a second launch repeats dx, dgamma, dbeta; a row computed alone
    (rows = 1) equals that row of the batch."""
    from adapcc_b200.ops.layers import _lib

    grid, partials = _ln_bwd_grid(rows, d), _lib().adapcc_ln_partials(rows)
    assert grid == partials if d <= 768 else grid <= partials
    keep = _sparse_rows(rows, grid)
    g = torch.Generator().manual_seed(5 * d + rows)
    for dykind in ("random", "rowconst", "sparse"):
        x, dy, gamma = _ln_bwd_case(rows, d, xkind, dykind, keep, g, dev)
        _, mean, rstd = _ln_fwd(x, gamma, torch.zeros_like(gamma), 1e-5)
        dx, dgamma, dbeta, part = _ln_bwd(dy, x, gamma, mean, rstd)
        check_ln_bwd(dx, dgamma, dbeta, dy, x, gamma, mean, rstd)
        assert bool(torch.isfinite(part[:2 * grid * d]).all()), dykind
        assert bool(torch.isnan(part[2 * grid * d:]).all()), dykind
        xh, gy, c1, c2, rs = _ln_bwd_terms(dy, x, gamma, mean, rstd)
        for p, term, per_term in ((part[:grid * d], dy.double() * xh, 3), (part[grid * d:2 * grid * d], dy.double(), 0)):
            assert_within(p.view(grid, d).double().sum(0), term.sum(0), _g(rows + 64 + per_term) * term.abs().sum(0),
                          f"layernorm backward partials ({dykind})")
        again = _ln_bwd(dy, x, gamma, mean, rstd, add=True)
        assert all(_same_bits(a, b) for a, b in zip(again[:3], (dx, dgamma, dbeta))), dykind
        pre = rs * (gy - c1 - xh * c2)
        del xh, gy
        torch.manual_seed(rows + d)
        # a random gradient on the residual stream, and one that cancels dx to the rounding error of its fp32 value:
        # rounding before the add (bf16 twice) would then give exactly 0
        for name, dres in (("random", torch.randn(rows, d, device=dev).bfloat16()), ("cancel", (-pre).bfloat16())):
            dxr, dgr, dbr, _ = _ln_bwd(dy, x, gamma, mean, rstd, dres=dres, add=True)
            check_ln_bwd(dxr, dgr, dbr, dy, x, gamma, mean, rstd, dres=dres)
            assert _same_bits(dgr, dgamma) and _same_bits(dbr, dbeta), (dykind, name)
            again = _ln_bwd(dy, x, gamma, mean, rstd, dres=dres, add=True)
            assert all(_same_bits(a, b) for a, b in zip(again[:3], (dxr, dgr, dbr))), (dykind, name)
            for r in keep:
                alone = _ln_bwd(dy[r:r + 1], x[r:r + 1], gamma, mean[r:r + 1], rstd[r:r + 1], dres=dres[r:r + 1],
                                add=True)[0]
                assert _same_bits(alone[0], dxr[r]), (dykind, name, r)


def test_ln_bwd_checker_rejects_perturbed_reference():
    """The exact result passes; a backward without c1, without c2, with dres added after dx was rounded, with dgamma and
    dbeta swapped, or with one row missing from dgamma does not."""
    g = torch.Generator().manual_seed(0)
    rows, d = 4099, 512
    keep = _sparse_rows(rows, 257)

    def case(dykind):
        x, dy, gamma = _ln_bwd_case(rows, d, "normal", dykind, keep, g, "cpu")
        x64 = x.double()
        mu = x64.mean(1)
        mean, rstd = mu.float(), (1.0 / torch.sqrt(((x64 - mu[:, None]) ** 2).mean(1) + 1e-5)).float()
        return (dy, x, gamma, mean, rstd), _ln_bwd_terms(dy, x, gamma, mean, rstd)

    args, (xh, gy, c1, c2, rs) = case("random")
    pre = rs * (gy - c1 - xh * c2)
    dg, db = (args[0].double() * xh).sum(0).bfloat16(), args[0].double().sum(0).bfloat16()
    dres = (-pre).bfloat16()                                       # the sum is the rounding error of pre: a cancellation
    check_ln_bwd(pre.bfloat16(), dg, db, *args)
    check_ln_bwd((pre + dres.double()).bfloat16(), dg, db, *args, dres=dres)
    with pytest.raises(AssertionError, match="dx"):
        check_ln_bwd((rs * (gy - xh * c2)).bfloat16(), dg, db, *args)              # c1 dropped
    with pytest.raises(AssertionError, match="dx"):
        check_ln_bwd((rs * (gy - c1)).bfloat16(), dg, db, *args)                   # c2 dropped
    with pytest.raises(AssertionError, match="dx"):
        check_ln_bwd((pre.bfloat16().double() + dres.double()).bfloat16(), dg, db, *args, dres=dres)   # rounded twice
    with pytest.raises(AssertionError, match="dgamma"):
        check_ln_bwd(pre.bfloat16(), db, dg, *args)                                # swapped

    args, (xh, gy, c1, c2, rs) = case("sparse")
    pre = (rs * (gy - c1 - xh * c2)).bfloat16()
    term = args[0].double() * xh
    check_ln_bwd(pre, term.sum(0).bfloat16(), args[0].double().sum(0).bfloat16(), *args)
    for r in keep:
        with pytest.raises(AssertionError, match="dgamma"):
            check_ln_bwd(pre, (term.sum(0) - term[r]).bfloat16(), args[0].double().sum(0).bfloat16(), *args)


def check_colsum_bf16(out, a):
    """bf16 column sums of a bf16 matrix through fp32 partials: any order of `rows` fp32 adds (+64 for the split and
    finalise trees) is off by (rows + 64) U32 sum |a|, then one bf16 rounding."""
    a64 = a.double()
    ref = a64.sum(0)
    e = (a64.shape[0] + 64) * U32 * a64.abs().sum(0)
    assert_within(out, ref, e + U16 * (ref.abs() + e), "colsum")


@gpu
@pytest.mark.parametrize("rows", [1, 9, 63, 64, 200, 4099])
@pytest.mark.parametrize("cols", [8, 296, 2304])
def test_colsum_against_fp64(dev, rows, cols):
    """cols / 8 = 1, 37 (not a multiple of the 32 vectors a CTA covers) and 288; rows below one 64-row split."""
    from adapcc_b200.ops.layers import _lib, _p, _s

    torch.manual_seed(rows * cols)
    a = torch.randn(rows, cols, device=dev).bfloat16()
    lib = _lib()
    out = torch.empty(cols, dtype=torch.bfloat16, device=dev)
    part = torch.empty(lib.adapcc_colsum_splits(rows) * cols, dtype=torch.float32, device=dev)
    assert lib.adapcc_colsum(_p(a), rows, cols, _p(out), _p(part), _s()) == 0
    check_colsum_bf16(out, a)


def test_colsum_checker_rejects_perturbed_reference():
    a = torch.randn(200, 296).bfloat16()
    check_colsum_bf16(a.double().sum(0).bfloat16(), a)
    with pytest.raises(AssertionError):
        check_colsum_bf16(a.double()[1:].sum(0), a)


# ---- optimizers ----------------------------------------------------------------------------------------------------
def sumsq_bound(n, vec):
    """Relative bound of the deterministic sum of squares: a thread's run of ceil(n / (blocks 512 vec)) vectors (+ the
    tail in block 0), 5 + 4 levels of warp trees, the last block's sequential sum of `blocks` partials, the add into
    `out`, and the square's own rounding."""
    blocks = max(1, min(592, -(-(n // 8) // 512)))
    per_thread = -(-n // (blocks * 512 * vec)) * vec + vec
    return (per_thread + 9 + blocks + 2) * U32


def adamw_ref(w, grads, *, lr, betas, eps, wd, max_norm, gs, vec):
    """fp64 AdamW over the given gradient sequence -> (master, m, v, bound on |master_kernel - master|, bound on m, v).

    Error terms per step, carried over steps: the clip coefficient (half the sum of squares' relative bound, 4 U32 for
    sqrt / divide / products); m and v get 3 U32 of their two terms plus the coefficient's error; the update
    lr mhat / (sqrt(vhat) + eps) gets m's error, half of v's relative error and 4 U32; the weight 3 U32 of itself."""
    f32 = lambda x: float(np.float32(x))                           # the kernel receives fp32 hyperparameters
    b1, b2, lr, eps, wd, gs = f32(betas[0]), f32(betas[1]), f32(lr), f32(eps), f32(wd), f32(gs)
    w = w.double().clone()
    m = torch.zeros_like(w)
    v = torch.zeros_like(w)
    em = torch.zeros_like(w)
    ev = torch.zeros_like(w)
    ew = torch.zeros_like(w)
    n = w.numel()
    for t, g in enumerate(grads, 1):
        g = g.double()
        coef = gs
        crel = 0.0
        if max_norm > 0:
            norm = math.sqrt(float((g * g).sum())) * gs
            coef *= min(1.0, max_norm / (norm + 1e-6))
            crel = 0.5 * sumsq_bound(n, vec) + 4 * U32
        gg = g * coef
        em = b1 * em + 3 * U32 * (b1 * m.abs() + (1 - b1) * gg.abs()) + (1 - b1) * gg.abs() * (crel + U32)
        ev = b2 * ev + 3 * U32 * (b2 * v + (1 - b2) * gg * gg) + (1 - b2) * gg * gg * (2 * crel + 3 * U32)
        m = b1 * m + (1 - b1) * gg
        v = b2 * v + (1 - b2) * gg * gg
        bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
        mh, vh = m / bc1, v / bc2
        den = vh.sqrt() + eps
        evh = ev / bc2 + 4 * U32 * vh
        dsq = torch.minimum(evh / (2 * vh.sqrt()).clamp(min=1e-300), evh.sqrt())
        upd = mh / den
        eupd = (em / bc1 + 4 * U32 * mh.abs()) / den + mh.abs() / (den * den) * dsq + 4 * U32 * upd.abs()
        ew = ew * (1 - lr * wd) + 3 * U32 * w.abs() + lr * eupd
        w = w * (1 - lr * wd) - lr * upd
    return w, m, v, ew, em, ev


ADAMW_CONFIGS = [dict(lr=1e-2, betas=(0.9, 0.95), eps=1e-8, wd=0.1, max_norm=1.0, gs=0.5),
                 dict(lr=3e-3, betas=(0.8, 0.99), eps=1e-6, wd=0.0, max_norm=0.0, gs=2.0)]
OPT_SIZES = [1, 3, 5, 100_003, 3_000_007]
DTYPE_PAIRS = [(torch.bfloat16, torch.bfloat16), (torch.float32, torch.float32),
               (torch.bfloat16, torch.float32), (torch.float32, torch.bfloat16)]


def _check_master(master, m, v, ref, what):
    w64, m64, v64, ew, em, ev = ref
    assert_within(master, w64, 2 * ew + 1e-30, f"{what} master")
    assert_within(m, m64, 2 * em + 1e-30, f"{what} m")
    assert_within(v, v64, 2 * ev + 1e-30, f"{what} v")


@gpu
@pytest.mark.parametrize("n", OPT_SIZES)
@pytest.mark.parametrize("pdtype,gdtype", DTYPE_PAIRS)
def test_fused_adamw_against_fp64(dev, n, pdtype, gdtype):
    """Three steps of clip + AdamW in both configurations (clip with grad_scale; no clip, no weight decay); n = 3 000 007
    makes every grid-stride loop run more than once; master / m / v against fp64, params = round(master) exactly."""
    from adapcc_b200.ops import fused_adamw_, sumsq_

    for ci, c in enumerate(ADAMW_CONFIGS):
        torch.manual_seed(n + ci)
        w0 = torch.randn(n, device=dev)
        grads = [(torch.randn(n, device=dev) * 5).to(gdtype) for _ in range(3)]
        param, master = w0.to(pdtype).clone(), w0.clone()
        m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
        sumsq = torch.zeros(1, device=dev)
        for step, g in enumerate(grads, 1):
            sumsq.zero_()
            sumsq_(g, sumsq)
            fused_adamw_(param, g, master, m, v, lr=c["lr"], betas=c["betas"], eps=c["eps"], weight_decay=c["wd"],
                         step=step, max_norm=c["max_norm"], grad_scale=c["gs"], sumsq=sumsq)
        ref = adamw_ref(w0, grads, lr=c["lr"], betas=c["betas"], eps=c["eps"], wd=c["wd"], max_norm=c["max_norm"],
                        gs=c["gs"], vec=16 // grads[0].element_size())
        _check_master(master, m, v, ref, f"adamw {pdtype}/{gdtype} config {ci}")
        assert torch.equal(param, master.to(pdtype))


@gpu
@pytest.mark.parametrize("n", OPT_SIZES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_sumsq_against_fp64_and_repeatable(dev, n, dtype):
    from adapcc_b200.ops import sumsq_

    torch.manual_seed(n)
    g = (torch.randn(n, device=dev) * 3).to(dtype)
    out = torch.zeros(1, device=dev)
    sumsq_(g, out)
    ref = (g.double() ** 2).sum()
    assert_within(out[0], ref, sumsq_bound(n, 16 // g.element_size()) * ref, "sumsq")
    for _ in range(3):
        again = torch.zeros(1, device=dev)
        sumsq_(g, again)
        assert torch.equal(again, out)


@gpu
def test_sumsq_rejects_misaligned_pointer(dev):
    from adapcc_b200.ops import sumsq_
    from adapcc_b200.runtime.native import NativeError

    g = torch.randn(1001, device=dev)
    out = torch.zeros(1, device=dev)
    with pytest.raises(NativeError):
        sumsq_(g[1:], out)                                          # 4 bytes past a 16-byte boundary
    torch.cuda.synchronize()
    assert float(out) == 0.0


@gpu
@pytest.mark.parametrize("n", OPT_SIZES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_fused_sgd_against_fp64(dev, n, dtype):
    """master -= lr g grad_scale: lr g and its scaling round twice (2 U32 of |lr g gs|), the subtraction once."""
    from adapcc_b200.ops import fused_sgd_

    torch.manual_seed(n + 7)
    w0 = torch.randn(n, device=dev)
    param, master = w0.to(dtype).clone(), w0.clone()
    w64, e = w0.double(), torch.zeros(n, dtype=torch.float64, device=dev)
    for _ in range(2):
        g = torch.randn(n, device=dev).to(dtype)
        fused_sgd_(param, g, master, lr=0.05, grad_scale=0.25)
        step = float(np.float32(0.05)) * g.double() * 0.25
        e = e + 2 * U32 * step.abs() + U32 * (w64 - step).abs()
        w64 = w64 - step
    assert_within(master, w64, 2 * e + 1e-30, "sgd master")
    assert torch.equal(param, master.to(dtype))


@gpu
@pytest.mark.parametrize("n", [8, 4096, 3_000_008])
def test_zero_adamw_bcast_against_fp64(dev, n):
    """The ZeRO-1 shard step at world size 1 through the communicator's symmetric heap (multicast store when the heap
    has a multicast alias, else the peer-store path): master / m / v against fp64, and the heap's bf16 parameters
    equal round(master) exactly."""
    from adapcc_b200.ops import incr_, sumsq_, zero_adamw_bcast_
    from adapcc_b200.runtime.native import NativeComm

    comm = NativeComm(f"zero-{os.getpid()}-{n}", 0, 1, 0, staging_bytes=4 << 20, heap_bytes=16 << 20)
    try:
        c = ADAMW_CONFIGS[0]
        torch.manual_seed(n + 3)
        w0 = torch.randn(n, device=dev)
        param = comm.symm_empty(n, torch.bfloat16)
        param.copy_(w0.bfloat16())
        master = w0.clone()
        m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
        sumsq = torch.zeros(1, device=dev)
        step_t = torch.zeros(1, dtype=torch.int32, device=dev)
        grads = [(torch.randn(n, device=dev) * 5).bfloat16() for _ in range(3)]
        for g in grads:
            sumsq.zero_()
            sumsq_(g, sumsq)
            incr_(step_t)
            zero_adamw_bcast_(comm, param, g, master, m, v, lr=c["lr"], betas=c["betas"], eps=c["eps"],
                              weight_decay=c["wd"], max_norm=c["max_norm"], grad_scale=c["gs"], sumsq=sumsq,
                              step_tensor=step_t)
        comm.check()
        ref = adamw_ref(w0, grads, lr=c["lr"], betas=c["betas"], eps=c["eps"], wd=c["wd"], max_norm=c["max_norm"],
                        gs=c["gs"], vec=8)
        _check_master(master, m, v, ref, "zero_adamw")
        assert torch.equal(param, master.bfloat16())
    finally:
        comm.close()


def test_adamw_checker_rejects_perturbed_reference():
    torch.manual_seed(0)
    n = 4096
    w0 = torch.randn(n)
    grads = [(torch.randn(n) * 5).bfloat16() for _ in range(3)]
    for c in ADAMW_CONFIGS:
        kw = dict(betas=c["betas"], eps=c["eps"], wd=c["wd"], max_norm=c["max_norm"], gs=c["gs"], vec=8)
        ref = adamw_ref(w0, grads, lr=c["lr"], **kw)
        _check_master(ref[0].float(), ref[1].float(), ref[2].float(), ref, "self")
        bad = adamw_ref(w0, grads, lr=c["lr"] * 1.01, **kw)
        with pytest.raises(AssertionError):
            _check_master(bad[0], ref[1], ref[2], ref, "lr * 1.01")
        bad = adamw_ref(w0, [grads[0].double() * 1.01] + grads[1:], lr=c["lr"], **dict(kw, max_norm=0.0))
        ref0 = adamw_ref(w0, grads, lr=c["lr"], **dict(kw, max_norm=0.0))
        with pytest.raises(AssertionError):
            _check_master(ref0[0], bad[1], ref0[2], ref0, "gradient * 1.01")


# ---- fixed-point embedding backward --------------------------------------------------------------------------------
def embed_bwd_emulate(old_grads, spec, idx, dy):
    """Exact emulation of csrc/ops_embed.cu's backward -> new bf16 gradients (torch CPU tensors).

    old_grads: bf16 [rows_j, D] per distinct table; spec[k]: table of lookup k; idx[k]: int64 [n]; dy: bf16 [n, D].
    lookup_bits = ceil(log2(K n)); a table row's shift = 62 - lookup_bits - (e + 1) with e the exponent of the largest
    |dY| over every lookup hitting it (-126 for subnormals and zero); S = sum of rint(float32(dY 2^shift)), exact;
    new = bf16(float32(old) + float32(float64(S) 2^-shift)); rows whose dY held a non-finite value become NaN; rows no
    lookup hits keep their bits."""
    K, n = len(spec), int(idx[0].numel())
    total = K * n
    lookup_bits = 0
    while (1 << lookup_bits) < total:
        lookup_bits += 1
    dyf = dy.float().numpy()
    rowbits = np.abs(dyf).view(np.uint32).max(axis=1)                    # per token: bits of max |dY|
    out = []
    for j, old in enumerate(old_grads):
        ks = [k for k in range(K) if spec[k] == j]
        if not ks:
            out.append(old.clone())
            continue
        rows_j = old.shape[0]
        mb = np.zeros(rows_j, dtype=np.uint32)
        hit = np.zeros(rows_j, dtype=bool)
        for k in ks:
            ix = idx[k].numpy()
            np.maximum.at(mb, ix, rowbits)
            hit[ix] = True
        ex = ((mb >> 23) & 0xFF).astype(np.int64)
        e = np.where(ex == 0, -126, ex - 127)
        shift = 62 - lookup_bits - (e + 1)
        finite = mb < 0x7F800000
        S = np.zeros(old.shape, dtype=np.int64)
        for k in ks:
            ix = idx[k].numpy()
            sh = np.where(finite[ix], shift[ix], 0)[:, None].astype(np.int32)
            v = np.where(finite[ix][:, None], dyf, np.float32(0))
            q = np.rint(np.ldexp(v, sh).astype(np.float32)).astype(np.int64)
            np.add.at(S, ix, q)
        back = np.ldexp(S.astype(np.float64), -np.where(finite, shift, 0)[:, None]).astype(np.float32)
        new = (old.float().numpy() + back).astype(np.float32)
        new[~finite & hit] = np.nan
        new_bf = torch.from_numpy(new).bfloat16()
        keep = torch.from_numpy(~hit)
        new_bf[keep] = old[keep]
        out.append(new_bf)
    return out


def _bits_equal(a, b):
    an, bn = torch.isnan(a.float()), torch.isnan(b.float())
    return torch.equal(an, bn) and torch.equal(a.view(torch.int16)[~an], b.view(torch.int16)[~bn])


def _embed_case(name, g):
    """-> (table rows per distinct table, spec, idx list, dy, D)."""
    D = 64
    if name == "hot6":
        # one 64-lookup tile with 6 rows hit 8 times each; their first hits lie in both warps of the claiming threads
        # (3 before lookup 32, 3 after), so which 4 become hot depends on warp order; 16 single hits fill the tile
        n = 64
        ix = np.full(n, -1)
        ix[[0, 1, 2, 40, 41, 42]] = np.arange(10, 16)
        early = [r for r in (10, 11, 12) for _ in range(7)] + list(range(100, 116))      # fills lookups 3..39
        late = [r for r in (13, 14, 15) for _ in range(7)]                               # fills lookups 43..63
        ix[3:40] = np.array(early)[torch.randperm(len(early), generator=g).numpy()]
        ix[43:] = np.array(late)[torch.randperm(len(late), generator=g).numpy()]
        idx = [torch.from_numpy(ix.astype(np.int64))]
        dy = (torch.randn(n, D, generator=g) * torch.logspace(-3, 1, n)[:, None]).bfloat16()
        return [200], (0,), idx, dy, D
    if name == "cancel":
        # row 7 hit by lookups 0, 2, 4, 6 (the same thread group): +1, 2^-30, -1, 0 -> exact sum 2^-30
        n = 64
        ix = torch.arange(100, 100 + n)
        ix[[0, 2, 4, 6]] = 7
        dy = torch.zeros(n, D)
        dy[0, :], dy[2, :], dy[4, :] = 1.0, 2.0 ** -30, -1.0
        dy[8:] = torch.randn(n - 8, D, generator=g)
        return [200], (0,), [ix], dy.bfloat16(), D
    K, n = {"k1_pow2": (1, 1024), "k1_pow2p1": (1, 1025), "k4": (4, 256), "k4_odd": (4, 257)}[name]
    spec = (0, 1, 0, 2)[:K]
    sizes = [300, 64, 3][:max(spec) + 1]
    idx = []
    for k in range(K):
        rows = sizes[spec[k]]
        ix = torch.randint(0, rows, (n,), generator=g)
        if k == 0:
            ix[:40] = 5                                            # heavy duplication of one row
        idx.append(ix)
    dy = (torch.randn(n, D, generator=g) * torch.logspace(-4, 2, n)[:, None]).bfloat16()
    if name == "k4":
        dy[17, 3] = float("inf")                                   # rows hit by token 17 become NaN
    return sizes, spec, idx, dy, D


def _old_grads(name, sizes, D, g):
    """Pre-filled gradients (the tied LM head's dW is already in wte's gradient when the embedding backward runs); the
    cancellation row starts at zero so that its 2^-30 is the whole result."""
    old = [(torch.randn(r, D, generator=g) * 0.01).bfloat16() for r in sizes]
    if name == "cancel":
        old[0][7] = 0
    return old


EMBED_CASES = ["hot6", "cancel", "k1_pow2", "k1_pow2p1", "k4", "k4_odd"]


@gpu
@pytest.mark.parametrize("name", EMBED_CASES)
def test_embedding_backward_bit_exact(dev, name):
    """The three-launch backward through its C entry point, accumulating into pre-filled gradients (the tied LM head
    case), must equal the emulation bit for bit and leave its work buffers at INT_MAX / 0 / 0; repeated, the same."""
    from ctypes import c_int, c_void_p

    from adapcc_b200.ops import _lib, _ptr_array, _stream

    g = torch.Generator().manual_seed(EMBED_CASES.index(name))
    sizes, spec, idx, dy, D = _embed_case(name, g)
    old = _old_grads(name, sizes, D, g)
    want = embed_bwd_emulate(old, spec, idx, dy)
    K, n = len(spec), idx[0].numel()
    base = np.cumsum([0] + sizes[:-1]).tolist()
    n_owner = sum(sizes)
    owner = torch.empty(n_owner, dtype=torch.int32, device=dev)
    maxbits = torch.empty(n_owner, dtype=torch.int32, device=dev)
    scratch = torch.empty(K * n * D, dtype=torch.int64, device=dev)
    lib = _lib()
    assert lib.adapcc_embed_bwd_reset(c_void_p(owner.data_ptr()), c_void_p(maxbits.data_ptr()), n_owner,
                                      c_void_p(scratch.data_ptr()), scratch.numel(), _stream()) == 0
    idx_d = [i.to(dev) for i in idx]
    dy_d = dy.to(dev)
    first = None
    for _ in range(2):
        grads = [o.to(dev) for o in old]
        ob = (c_int * K)(*[base[j] for j in spec])
        assert lib.adapcc_embed_sum_bwd(c_void_p(dy_d.data_ptr()), _ptr_array(idx_d),
                                        _ptr_array([grads[j] for j in spec]), ob, K, n, D,
                                        c_void_p(owner.data_ptr()), c_void_p(maxbits.data_ptr()),
                                        c_void_p(scratch.data_ptr()), _stream()) == 0
        torch.cuda.synchronize()
        for j, (got, w) in enumerate(zip(grads, want)):
            assert _bits_equal(got.cpu(), w), (name, j, int((got.cpu().float() != w.float()).sum()))
        assert torch.all(owner == 2 ** 31 - 1) and torch.all(maxbits == 0) and torch.all(scratch == 0)
        if first is not None:
            assert all(_bits_equal(a, b) for a, b in zip(grads, first))
        first = grads


@gpu
def test_fused_embedding_sum_int32_indices_take_the_plain_path(dev):
    """The kernels read int64 indices: other index dtypes go through F.embedding (same values, autograd intact)."""
    from adapcc_b200.ops import fused_embedding_sum

    torch.manual_seed(0)
    wte = torch.randn(100, 64, device=dev).bfloat16().requires_grad_(True)
    ids = torch.randint(0, 100, (4, 16), device=dev)
    y64 = fused_embedding_sum([wte], [(0, ids)])
    y32 = fused_embedding_sum([wte], [(0, ids.int())])
    assert torch.equal(y64, y32)
    y32.float().sum().backward()
    assert wte.grad is not None and wte.grad.shape == wte.shape


def test_embedding_emulator_against_fp64():
    """The emulation against fp64 index_add_: the fixed-point rounding is at most half a unit of 2^-shift per lookup,
    the float32 conversions and add 2 U32, the bf16 result U16."""
    for ci, name in enumerate(EMBED_CASES):
        g = torch.Generator().manual_seed(ci)
        sizes, spec, idx, dy, D = _embed_case(name, g)
        old = _old_grads(name, sizes, D, g)
        got = embed_bwd_emulate(old, spec, idx, dy)
        K, n = len(spec), idx[0].numel()
        lookup_bits = max(0, math.ceil(math.log2(K * n)))
        for j, (o, gj) in enumerate(zip(old, got)):
            ref = o.double().clone()
            hits = torch.zeros(o.shape[0], dtype=torch.float64)
            mx = torch.zeros(o.shape[0], dtype=torch.float64)
            absum = o.double().abs().clone()
            for k in range(K):
                if spec[k] != j:
                    continue
                ref.index_add_(0, idx[k], dy.double())
                absum.index_add_(0, idx[k], dy.double().abs())
                hits.index_add_(0, idx[k], torch.ones(n, dtype=torch.float64))
                np.maximum.at(mx.numpy(), idx[k].numpy(), dy.double().abs().amax(1).numpy())   # in place
            nonfinite = ~torch.isfinite(ref).all(1)
            assert torch.isnan(gj[nonfinite].float()).all()
            e_row = torch.floor(torch.log2(mx.clamp(min=2.0 ** -126)))
            unit = 2.0 ** -(62 - lookup_bits - (e_row + 1))          # 2^-shift
            bound = 0.5 * hits[:, None] * unit[:, None] + 2 * U32 * absum
            bound = bound + U16 * (ref.abs() + bound)
            fin = ~nonfinite
            assert_within(gj[fin], ref[fin], bound[fin], f"emulator {name} table {j}")
            if name == "cancel":
                assert float(gj[7, 0]) == float((o[7, 0].double() + 2.0 ** -30).bfloat16())


# ---- MoE slot assignment -------------------------------------------------------------------------------------------
def stable_rank(expert, n_expert, capacity):
    """pos[i] = #{j < i : expert[j] == expert[i]}, -1 when >= capacity or the id is out of range; counts = bincount."""
    e = expert.long()
    valid = (e >= 0) & (e < n_expert)
    key = torch.where(valid, e, torch.full_like(e, n_expert))
    order = torch.argsort(key, stable=True)
    sk = key[order]
    start = torch.searchsorted(sk, torch.arange(n_expert + 1, device=e.device))
    rank = torch.empty_like(e)
    rank[order] = torch.arange(e.numel(), device=e.device) - start[sk]
    pos = torch.where(valid & (rank < capacity), rank, torch.full_like(rank, -1))
    return pos.int(), torch.bincount(e[valid], minlength=n_expert).int()


@gpu
def test_moe_assign_is_the_stable_rank(dev):
    from adapcc_b200.parallel.expert_parallel import ExpertExchange
    from adapcc_b200.runtime.native import NativeComm

    comm = NativeComm(f"moea-{os.getpid()}", 0, 1, 0, staging_bytes=4 << 20, heap_bytes=16 << 20)
    try:
        E, A, cap = 8, 65_536, 5000
        ex = ExpertExchange(comm, E, cap, 8)
        torch.manual_seed(4)
        expert = torch.randint(0, E, (A,), device=dev, dtype=torch.int32)
        expert[torch.randint(0, A, (500,), device=dev)] = -1         # ids out of range are dropped
        expert[torch.randint(0, A, (500,), device=dev)] = E
        expert[: A // 4] = 0                                        # expert 0 overflows its capacity
        pos, counts = ex.assign(expert)
        want_pos, want_counts = stable_rank(expert, E, cap)
        assert torch.equal(counts, want_counts)
        assert torch.equal(pos, want_pos), int((pos != want_pos).sum())
        with pytest.raises(TypeError):
            ex.assign(expert.long())
    finally:
        comm.close()
