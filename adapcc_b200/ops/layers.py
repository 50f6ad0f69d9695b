"""nn.Module wrappers around the fused transformer kernels (csrc/ops_norm.cu).

* ``FusedLayerNorm`` — single-pass bf16 LayerNorm forward/backward (row kept in registers, dgamma /
  dbeta reduced in the same pass). Falls back to ``F.layer_norm`` for CPU tensors, non-bf16 dtypes
  or widths other than 256/512/768/1024.
  ``forward_add(x, res)`` also fuses the preceding residual add (and, backward, the residual-stream
  gradient add); with ``drop`` the residual branch passes through dropout (ops/dropout.py) in the same kernels.
* ``FusedLinear`` — ``F.linear`` (cuBLASLt, bias epilogue) whose backward computes the bias gradient
  with the column-sum kernel instead of ATen's generic reduction.
"""
from __future__ import annotations

from ctypes import c_float, c_int, c_uint, c_void_p

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..runtime.native import NativeError, last_error, load_library

_bound = False
_LN_WIDTHS = (256, 512, 768, 1024)


def _lib():
    global _bound
    lib = load_library()
    if not _bound:
        lib.adapcc_ln_fwd.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                      c_float, c_void_p]
        lib.adapcc_ln_bwd.argtypes = [c_void_p] * 9 + [c_int, c_int, c_void_p]
        lib.adapcc_add_ln_fwd.argtypes = [c_void_p] * 8 + [c_int, c_int, c_float, c_void_p]
        lib.adapcc_add_ln_bwd.argtypes = [c_void_p] * 10 + [c_int, c_int, c_void_p]
        drop = [c_void_p, c_void_p, c_int, c_uint, c_float]            # seed, step, site, thr, scale
        lib.adapcc_add_ln_drop_fwd.argtypes = [c_void_p] * 8 + [c_int, c_int, c_float] + drop + [c_void_p]
        lib.adapcc_add_ln_drop_bwd.argtypes = [c_void_p] * 11 + [c_int, c_int] + drop + [c_void_p]
        lib.adapcc_ln_partials.argtypes = [c_int]
        lib.adapcc_colsum.argtypes = [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]
        lib.adapcc_colsum_splits.argtypes = [c_int]
        _bound = True
    return lib


def _s():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return c_void_p(t.data_ptr())


def _sink(p):
    """Direct-gradient protocol with the flat engine (parallel/engine.py): a parameter carrying a
    ``_adapcc_grad_sink`` has a preallocated ``.grad`` view inside the engine's flat gradient buffer,
    zeroed at the start of the step. The backward kernels then write that view directly and report
    ``done()`` — instead of returning a fresh tensor that autograd adds into ``.grad`` with one more
    elementwise kernel per parameter (148 launches and ~0.75 GB of traffic per GPT-2 step)."""
    if p is None or p.grad is None:
        return None
    return getattr(p, "_adapcc_grad_sink", None)


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        lib = _lib()
        d = x.shape[-1]
        x2 = x.reshape(-1, d).contiguous()
        rows = x2.shape[0]
        y = torch.empty_like(x2)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        if lib.adapcc_ln_fwd(_p(x2), _p(gamma), _p(beta), _p(y), _p(mean), _p(rstd), rows, d, eps, _s()) != 0:
            raise NativeError(f"ln_fwd failed: {last_error()}")
        ctx.save_for_backward(x2, gamma, mean, rstd)
        ctx.params = (gamma, beta)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        lib = _lib()
        x2, gamma, mean, rstd = ctx.saved_tensors
        rows, d = x2.shape
        dy2 = dy.reshape(rows, d).contiguous()
        dx = torch.empty_like(x2)
        dgamma, dbeta, finish = _ln_param_grads(ctx.params)
        part = torch.empty(2 * lib.adapcc_ln_partials(rows) * d, dtype=torch.float32, device=x2.device)
        if lib.adapcc_ln_bwd(_p(dy2), _p(x2), _p(gamma), _p(mean), _p(rstd), _p(dx), _p(dgamma), _p(dbeta), _p(part),
                             rows, d, _s()) != 0:
            raise NativeError(f"ln_bwd failed: {last_error()}")
        return (dx.view(dy.shape),) + finish() + (None,)


def _ln_param_grads(params):
    """-> (dgamma buffer, dbeta buffer, finish): the buffers are the parameters' own ``.grad`` views
    when the engine's direct-gradient protocol is on (finish() then reports them done and hands
    autograd ``None``), fresh tensors otherwise."""
    gamma, beta = params
    sg, sb = _sink(gamma), _sink(beta)
    dgamma = gamma.grad if sg is not None and sg.begin() else torch.empty_like(gamma)
    dbeta = beta.grad if sb is not None and sb.begin() else torch.empty_like(beta)

    def finish():
        if sg is not None:
            sg.done()
        if sb is not None:
            sb.done()
        return (None if sg is not None else dgamma, None if sb is not None else dbeta)
    return dgamma, dbeta, finish


class _AddLayerNormFn(torch.autograd.Function):
    """(x, res) -> (s = x + res, LayerNorm(s)) in one pass; the backward adds the gradient that
    arrives on ``s`` (the residual stream) to the LayerNorm input gradient in the same kernel."""

    @staticmethod
    def forward(ctx, x, res, gamma, beta, eps):
        lib = _lib()
        d = x.shape[-1]
        x2 = x.reshape(-1, d).contiguous()
        r2 = res.reshape(-1, d).contiguous()
        rows = x2.shape[0]
        ssum = torch.empty_like(x2)
        y = torch.empty_like(x2)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        if lib.adapcc_add_ln_fwd(_p(x2), _p(r2), _p(gamma), _p(beta), _p(ssum), _p(y), _p(mean), _p(rstd), rows, d,
                                 eps, _s()) != 0:
            raise NativeError(f"add_ln_fwd failed: {last_error()}")
        ctx.save_for_backward(ssum, gamma, mean, rstd)
        ctx.params = (gamma, beta)
        ctx.set_materialize_grads(False)              # an unused output's gradient arrives as None, not zeros
        return ssum.view(x.shape), y.view(x.shape)

    @staticmethod
    def backward(ctx, dsum, dy):
        lib = _lib()
        s2, gamma, mean, rstd = ctx.saved_tensors
        rows, d = s2.shape
        if dy is None:                                # only the sum was used downstream
            return dsum, dsum, None, None, None
        dy2 = dy.reshape(rows, d).contiguous()
        ds2 = None if dsum is None else dsum.reshape(rows, d).contiguous()   # keep alive past the launch
        dx = torch.empty_like(s2)
        dgamma, dbeta, finish = _ln_param_grads(ctx.params)
        part = torch.empty(2 * lib.adapcc_ln_partials(rows) * d, dtype=torch.float32, device=s2.device)
        if lib.adapcc_add_ln_bwd(_p(dy2), _p(s2), _p(gamma), _p(mean), _p(rstd), c_void_p(0) if ds2 is None else _p(ds2),
                                 _p(dx), _p(dgamma), _p(dbeta), _p(part), rows, d, _s()) != 0:
            raise NativeError(f"add_ln_bwd failed: {last_error()}")
        dx = dx.view(dy.shape)
        return (dx, dx) + finish() + (None,)


class _AddLayerNormDropFn(torch.autograd.Function):
    """(x, res) -> (s = x + drop(res), LayerNorm(s)) in one pass, the mask recomputed from ``(p, state, site)``
    (ops/dropout.py). The two inputs' gradients differ, so the backward kernel writes both: dx (LayerNorm input
    gradient plus the gradient arriving on ``s``) and dres = mask * scale * dx."""

    @staticmethod
    def forward(ctx, x, res, gamma, beta, eps, p, state, site):
        from .dropout import drop_tail

        lib = _lib()
        d = x.shape[-1]
        x2 = x.reshape(-1, d).contiguous()
        r2 = res.reshape(-1, d).contiguous()
        rows = x2.shape[0]
        ssum = torch.empty_like(x2)
        y = torch.empty_like(x2)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        ctx.drop = drop_tail("forward_add", p, state, site, x.device)
        if lib.adapcc_add_ln_drop_fwd(_p(x2), _p(r2), _p(gamma), _p(beta), _p(ssum), _p(y), _p(mean), _p(rstd), rows,
                                      d, eps, *ctx.drop, _s()) != 0:
            raise NativeError(f"add_ln_drop_fwd failed: {last_error()}")
        ctx.save_for_backward(ssum, gamma, mean, rstd)
        ctx.params = (gamma, beta)
        ctx.p, ctx.state = p, state                   # the state owns the tensors ctx.drop points at
        ctx.set_materialize_grads(False)
        return ssum.view(x.shape), y.view(x.shape)

    @staticmethod
    def backward(ctx, dsum, dy):
        lib = _lib()
        s2, gamma, mean, rstd = ctx.saved_tensors
        rows, d = s2.shape
        if dy is None:                                # only the sum was used downstream
            from .dropout import dropout
            return (dsum, dropout(dsum, ctx.p, ctx.state, ctx.drop[2])) + (None,) * 6
        dy2 = dy.reshape(rows, d).contiguous()
        ds2 = None if dsum is None else dsum.reshape(rows, d).contiguous()   # keep alive past the launch
        dx = torch.empty_like(s2)
        dres = torch.empty_like(s2)
        dgamma, dbeta, finish = _ln_param_grads(ctx.params)
        part = torch.empty(2 * lib.adapcc_ln_partials(rows) * d, dtype=torch.float32, device=s2.device)
        if lib.adapcc_add_ln_drop_bwd(_p(dy2), _p(s2), _p(gamma), _p(mean), _p(rstd),
                                      c_void_p(0) if ds2 is None else _p(ds2), _p(dx), _p(dres), _p(dgamma), _p(dbeta),
                                      _p(part), rows, d, *ctx.drop, _s()) != 0:
            raise NativeError(f"add_ln_drop_bwd failed: {last_error()}")
        return (dx.view(dy.shape), dres.view(dy.shape)) + finish() + (None,) * 4


class FusedLayerNorm(nn.LayerNorm):
    """``nn.LayerNorm`` whose bf16 CUDA forward / backward are single kernels (csrc/ops_norm.cu; optional residual add
    fused in: ``forward_add``); under the flat engine the backward writes d(gamma) / d(beta) straight into the flat
    gradient buffer (``_adapcc_grad_sink``)."""

    def _fusable(self, x):
        return (x.is_cuda and x.dtype == torch.bfloat16 and self.weight.dtype == torch.bfloat16
                and x.shape[-1] in _LN_WIDTHS and len(self.normalized_shape) == 1)

    def forward(self, x):
        if self._fusable(x):
            return _LayerNormFn.apply(x, self.weight, self.bias, self.eps)
        return F.layer_norm(x, self.normalized_shape, self.weight, self.bias, self.eps)

    def forward_add(self, x, res, drop=None):
        """-> (s, LayerNorm(s)) with s = x + res: the residual add of a pre-LN transformer block fused into
        the normalisation that follows it (one kernel forward, one backward). ``drop = (p, state, site)``: s = x +
        dropout(res) with the mask of ops/dropout.py, in the same kernels; None is the path without dropout."""
        fusable = self._fusable(x) and res.shape == x.shape and res.dtype == x.dtype
        if drop is not None:
            if fusable:
                return _AddLayerNormDropFn.apply(x, res, self.weight, self.bias, self.eps, *drop)
            from .dropout import dropout
            res = dropout(res, *drop)
        elif fusable:
            return _AddLayerNormFn.apply(x, res, self.weight, self.bias, self.eps)
        s = x + res
        return s, F.layer_norm(s, self.normalized_shape, self.weight, self.bias, self.eps)


class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        ctx.save_for_backward(x, w)
        ctx.params = (w, b)
        return F.linear(x, w, b)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        return linear_backward(ctx.params, x, w, dy, ctx.needs_input_grad[0])


def linear_backward(params, x, w, dy, needs_dx=True, db=None):
    """(dx, dw, db) of y = x @ w.T + b for bf16 CUDA tensors: two GEMMs + the column-sum kernel; dw / db
    go straight into the parameters' flat-buffer gradient views when the engine's sinks are attached.
    ``db``: the bias gradient if the caller already has it (fp32 [N], e.g. accumulated in a GEMM epilogue)."""
    lib = _lib()
    n = w.shape[0]
    dy2 = dy.reshape(-1, n)
    if not dy2.is_contiguous():
        dy2 = dy2.contiguous()
    x2 = x.reshape(-1, x.shape[-1])
    dx = (dy2 @ w).view(x.shape) if needs_dx else None
    pw, pb = params
    sw, sb = _sink(pw), _sink(pb)
    if sw is not None and sw.begin():                 # GEMM straight into the flat gradient buffer
        torch.mm(dy2.t(), x2, out=pw.grad)
        sw.done()
        dw = None
    else:
        dw = dy2.t() @ x2
    rows = dy2.shape[0]
    direct_b = sb is not None and pb.grad.dtype == dy2.dtype and sb.begin()
    if db is not None:                                # already reduced by the producer of dy
        if direct_b:
            pb.grad.copy_(db)
            sb.done()
            return dx, dw, None
        return dx, dw, db.to(dy2.dtype)
    db = pb.grad if direct_b else torch.empty(n, dtype=dy2.dtype, device=dy2.device)
    part = torch.empty(lib.adapcc_colsum_splits(rows) * n, dtype=torch.float32, device=dy2.device)
    if lib.adapcc_colsum(_p(dy2), rows, n, _p(db), _p(part), _s()) != 0:
        raise NativeError(f"colsum failed: {last_error()}")
    if direct_b:
        sb.done()
    return dx, dw, None if direct_b else db


class FusedLinear(nn.Linear):
    """``nn.Linear`` whose backward computes dW into the engine's flat gradient view (no accumulate kernel) and the
    bias gradient with the column-sum kernels of csrc/ops_norm.cu; the GEMMs themselves are cuBLAS."""

    def forward(self, x):
        if (x.is_cuda and x.dtype == torch.bfloat16 and self.bias is not None and self.weight.dtype == torch.bfloat16
                and self.out_features % 8 == 0 and torch.is_grad_enabled()):
            return _LinearFn.apply(x, self.weight, self.bias)
        return F.linear(x, self.weight, self.bias)
