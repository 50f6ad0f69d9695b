"""Hopper GEMMs with fused epilogues (csrc/gemm_wgmma.cu: TMA + mbarrier pipeline + wgmma, variants 0-3).

``linear_act(x, weight, bias, act)`` computes ``act(x @ weight.T + bias)`` for bf16 CUDA tensors with the
accumulator in registers and the activation applied in the epilogue; ``linear_gelu`` / ``mlp_gelu`` are the autograd
forms (the pre-activation is written by the same kernel; the backward GEMM applies gelu' and accumulates the bias
gradient in its epilogue). The GPT-2 MLP uses ``mlp_gelu`` by default (``ADAPCC_TCGEN05_MLP=0`` restores cuBLAS +
separate activation kernels; the variable keeps its original name so existing launch scripts still work).
"""
from __future__ import annotations

import os
from ctypes import c_int, c_void_p
from typing import Optional, Tuple

import torch

from ..runtime.native import NativeError, last_error, load_library

_bound = False
ACT = {"none": 0, "gelu": 1, "dgelu": 2, "residual": 3}


def _lib():
    global _bound
    lib = load_library()
    if not _bound:
        lib.adapcc_gemm_bias_act_v.argtypes = [c_void_p] * 5 + [c_int] * 5 + [c_void_p]
        lib.adapcc_gemm_pp.argtypes = [c_void_p] * 7 + [c_int] * 4 + [c_void_p]
        _bound = True
    return lib


def supported(x: torch.Tensor, weight: torch.Tensor) -> bool:
    return (x.is_cuda and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16
            and weight.shape[1] % 64 == 0 and weight.shape[0] % 128 == 0)


def default_variant() -> int:
    """0: one output tile per CTA. 1: persistent CTAs. 2: two-CTA clusters that share the W slab by TMA multicast,
    one 256 x 256 tile per cluster. 3 (default): persistent two-CTA clusters, the only variant with the column-sum
    output the MLP backward uses; shapes it does not cover (N % 256 != 0) go to variant 1. All four are checked element by
    element against fp64 references, and against each other bit for bit, by ``test_gemm_against_fp64``
    (tests/test_gpu_kernels_reference.py), at shapes where a persistent CTA runs many tiles included."""
    return int(os.environ.get("ADAPCC_TCGEN05_VARIANT", "3"))


def linear_act(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], act: str = "gelu",
               save_pre: bool = False, variant: Optional[int] = None,
               aux: Optional[torch.Tensor] = None,
               colsum: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """-> (result, pre-activation or None). x [..., K], weight [N, K], bias [N]; bf16.

    act "none" / "gelu": result = act(x @ weight.T + bias), optionally also the pre-activation.
    act "dgelu":    result = (x @ weight.T) * gelu'(aux)      — the MLP backward with the activation's derivative in
                    the epilogue (aux = the saved pre-activation, same shape as the result).
    act "residual": result = x @ weight.T + bias + aux        — projection with the residual add in the epilogue."""
    if not supported(x, weight):
        raise NativeError("linear_act: needs bf16 CUDA tensors with K % 64 == 0 and N % 128 == 0")
    n, k = weight.shape
    x2 = x.reshape(-1, k).contiguous()
    w = weight.contiguous()
    m = x2.shape[0]
    code = ACT[act]
    out = torch.empty(m, n, dtype=torch.bfloat16, device=x.device)
    v_req = default_variant() if variant is None else int(variant)
    if v_req == 3 and n % 256 == 0 and code <= 2:
        # variant 3: persistent two-CTA clusters; act "dgelu" can also accumulate the column sums of its result (the up-projection's bias gradient)
        if code == 2:
            if aux is None or aux.numel() != m * n or aux.dtype != torch.bfloat16:
                raise NativeError("linear_act(dgelu): aux must be a bf16 tensor with the result's shape")
            pre = aux.reshape(m, n).contiguous()
        else:
            pre = torch.empty_like(out) if save_pre else None
        if colsum is not None and (code != 2 or colsum.dtype != torch.float32 or colsum.numel() != n):
            raise NativeError("linear_act: colsum is an fp32 [N] accumulator of the dgelu mode")
        b = bias.contiguous() if bias is not None else None
        # per-row-tile column sums, added in a fixed order by the library: the same inputs give the same bits
        work = torch.empty((m + 127) // 128, n, dtype=torch.float32, device=x.device) if colsum is not None else None
        rc = _lib().adapcc_gemm_pp(c_void_p(x2.data_ptr()), c_void_p(w.data_ptr()),
                                   c_void_p(b.data_ptr() if b is not None else 0), c_void_p(out.data_ptr()),
                                   c_void_p(pre.data_ptr() if pre is not None else 0),
                                   c_void_p(colsum.data_ptr() if colsum is not None else 0),
                                   c_void_p(work.data_ptr() if work is not None else 0), m, n, k, code,
                                   c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc != 0:
            raise NativeError(f"gemm_pp failed: {last_error()}")
        shape = x.shape[:-1] + (n,)
        return out.view(shape), (pre.view(shape) if (pre is not None and code < 2) else None)
    if colsum is not None:
        raise NativeError("linear_act: colsum needs variant 3 (N % 256 == 0)")
    if v_req == 3:
        v_req = 1                                       # shapes variant 3 does not cover: persistent single CTAs
    if code >= 2:
        if aux is None or aux.numel() != m * n or aux.dtype != torch.bfloat16:
            raise NativeError(f"linear_act({act}): aux must be a bf16 tensor with the result's shape")
        pre = aux.reshape(m, n).contiguous()            # an INPUT in these modes
        v = 0                                           # only built for the per-tile variant
    else:
        pre = torch.empty_like(out) if save_pre else None
        v = v_req
    b = bias.contiguous() if bias is not None else None
    rc = _lib().adapcc_gemm_bias_act_v(c_void_p(x2.data_ptr()), c_void_p(w.data_ptr()),
                                       c_void_p(b.data_ptr() if b is not None else 0), c_void_p(out.data_ptr()),
                                       c_void_p(pre.data_ptr() if pre is not None else 0), m, n, k, code, v,
                                       c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc != 0:
        raise NativeError(f"gemm_bias_act failed: {last_error()}")
    shape = x.shape[:-1] + (n,)
    return out.view(shape), (pre.view(shape) if (pre is not None and code < 2) else None)


class _LinearGeluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        out, pre = linear_act(x, w, b, "gelu", save_pre=True)
        ctx.save_for_backward(x, w, pre)
        ctx.params = (w, b)
        return out

    @staticmethod
    def backward(ctx, dy):
        from .layers import linear_backward
        x, w, pre = ctx.saved_tensors
        du = torch.ops.aten.gelu_backward(dy.contiguous(), pre, approximate="tanh")
        return linear_backward(ctx.params, x, w, du, ctx.needs_input_grad[0])


def linear_gelu(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """gelu_tanh(x @ weight.T + bias) with the bias and activation in the GEMM's epilogue."""
    return _LinearGeluFn.apply(x, weight, bias)


class _MLPFn(torch.autograd.Function):
    """y = W2 gelu(W1 x + b1) + b2 with the GELU in the first GEMM's epilogue (forward) and its derivative in the
    epilogue of the backward GEMM dY.W2 — no stand-alone activation kernel in either direction."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2):
        h, pre = linear_act(x, w1, b1, "gelu", save_pre=True)
        y = torch.nn.functional.linear(h, w2, b2)
        ctx.save_for_backward(x, w1, w2, pre, h)
        ctx.params = ((w1, b1), (w2, b2))
        return y

    @staticmethod
    def backward(ctx, dy):
        from .layers import linear_backward
        x, w1, w2, pre, h = ctx.saved_tensors
        p1, p2 = ctx.params
        dy = dy.contiguous()
        _, dw2, db2 = linear_backward(p2, h, w2, dy, needs_dx=False)
        # dH = dY . W2 needs W2 as a K-major [N = d_hidden, K = d_model] operand: one 4.7 MB transpose per layer
        w2t = w2.t().contiguous()
        if default_variant() == 3 and w2t.shape[0] % 256 == 0:
            # ... and the up-projection's bias gradient (column sums of dH) falls out of the same epilogue
            db_acc = torch.zeros(w2t.shape[0], dtype=torch.float32, device=dy.device)
            du, _ = linear_act(dy, w2t, None, "dgelu", aux=pre, colsum=db_acc, variant=3)
            dx, dw1, db1 = linear_backward(p1, x, w1, du, ctx.needs_input_grad[0], db=db_acc)
        else:
            du, _ = linear_act(dy, w2t, None, "dgelu", aux=pre)
            dx, dw1, db1 = linear_backward(p1, x, w1, du, ctx.needs_input_grad[0])
        return dx, dw1, db1, dw2, db2


def mlp_gelu(x, w1, b1, w2, b2):
    """Transformer MLP ``linear(gelu(linear(x)))`` with both activation passes fused into GEMM epilogues."""
    return _MLPFn.apply(x, w1, b1, w2, b2)
