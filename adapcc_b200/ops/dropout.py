"""Training dropout whose masks are a pure function of ``(seed, step, site, row, column)`` (DESIGN.md §4a).

Nothing is stored for the backward (it evaluates the same function again), a step is repeatable bit for bit, and a
CUDA-graph replay draws fresh masks because seed and step live on the device (``DropoutState``).

The definition, which ``csrc/dropout.cuh`` equals bit for bit:

* One Philox4x32-10 call (``ops/sampling.py::philox4x32_10``) covers the 8 consecutive columns ``8v .. 8v + 7`` of one
  row: counter ``(row, v, site, step)``, key ``(seed & 0xffffffff, seed >> 32)`` of the seed taken as an unsigned 64-bit
  integer. The four output words give eight 16-bit halves: half ``2j`` is the LOW half of word ``j``, half ``2j + 1``
  its HIGH half. Column ``c`` uses half ``c & 7`` of the call ``v = c >> 3``.
* ``thr = round(p * 65536)`` clamped to ``[0, 65535]``; an element is kept iff its half ``>= thr``. The keep probability
  is exactly ``1 - thr / 65536`` and a kept element is multiplied by ``65536 / (65536 - thr)`` rounded to fp32, so the
  expectation is exact for the probability actually used. ``p = 0``: everything kept, scale exactly 1.
* Sites of GPT-2 (``site_*``): 0 the embedding sum, ``1 + 2i`` block i's attention output, ``2 + 2i`` block i's MLP
  output, ``1 + 2 n_layer`` the multiple-choice head's summary input. ``row`` is the row of the flattened ``[rows, D]``
  activation.
"""
from __future__ import annotations

from ctypes import c_float, c_int, c_uint, c_void_p
from typing import Optional, Tuple

import numpy as np
import torch

_MASK = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85


def site_embed() -> int:
    return 0


def site_attn(layer: int) -> int:
    return 1 + 2 * int(layer)


def site_mlp(layer: int) -> int:
    return 2 + 2 * int(layer)


def site_summary(n_layer: int) -> int:
    return 1 + 2 * int(n_layer)


def check_p(who: str, p: float) -> float:
    """``ValueError`` unless ``0 <= p < 1``."""
    p = float(p)
    if not 0.0 <= p < 1.0:
        raise ValueError(f"{who}: a dropout probability must be in [0, 1), got {p}")
    return p


def threshold(p: float) -> Tuple[int, float]:
    """-> (thr, scale) of probability ``p``: the 16-bit threshold and the fp32 scale of a kept element (as a float)."""
    thr = min(max(int(round(check_p("threshold", p) * 65536.0)), 0), 65535)
    return thr, float(np.float32(65536.0 / (65536.0 - thr)))


def _philox_halves(row_idx: np.ndarray, vec_idx: np.ndarray, seed: int, step: int, site: int) -> np.ndarray:
    """uint32 [len(row_idx), len(vec_idx), 8]: the eight 16-bit halves of Philox4x32-10 at counter (row, vec, site,
    step) for every pair of the two index arrays."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    rows, nvec = len(row_idx), len(vec_idx)
    c0 = np.broadcast_to(np.asarray(row_idx, dtype=np.uint64)[:, None], (rows, nvec)).copy()
    c1 = np.broadcast_to(np.asarray(vec_idx, dtype=np.uint64)[None, :], (rows, nvec)).copy()
    c2 = np.full((rows, nvec), int(site) & 0xFFFFFFFF, dtype=np.uint64)
    c3 = np.full((rows, nvec), int(step) & 0xFFFFFFFF, dtype=np.uint64)
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    s32 = np.uint64(32)
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ np.uint64(k0), p1 & _MASK, (p0 >> s32) ^ c3 ^ np.uint64(k1), p0 & _MASK
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    w = np.stack([c0, c1, c2, c3], axis=-1)                                    # [rows, nvec, 4]
    return np.stack([w & np.uint64(0xFFFF), w >> np.uint64(16)], axis=-1).reshape(rows, nvec, 8).astype(np.uint32)


def dropout_mask(rows: int, cols: int, p: float, seed: int, step: int, site: int) -> np.ndarray:
    """bool [rows, cols]: True where the element is kept."""
    thr, _ = threshold(p)
    nvec = (int(cols) + 7) // 8
    halves = _philox_halves(np.arange(int(rows)), np.arange(nvec), seed, step, site)
    return (halves >= thr).reshape(int(rows), nvec * 8)[:, :int(cols)]


def dropout_reference(x, p: float, seed: int, step: int, site: int) -> torch.Tensor:
    """``mask * scale * x`` in fp64 for ``x`` [..., cols], rows being the flattened leading dimensions; differentiable
    when ``x`` is an fp64 tensor that requires a gradient."""
    x = torch.as_tensor(x)
    x = x if x.dtype == torch.float64 else x.double()
    cols = x.shape[-1]
    mask = torch.from_numpy(dropout_mask(x.numel() // cols, cols, p, seed, step, site)).to(x.device).view(x.shape)
    return x * mask * threshold(p)[1]


class DropoutState:
    """The device-resident arguments of every mask of a model: ``seed`` int64 [1] and ``step`` int32 [1] (the training
    forwards run so far), both on the model's device, so kernels captured in a CUDA graph read the current values."""

    def __init__(self, seed: torch.Tensor, step: torch.Tensor):
        if seed.dtype != torch.int64 or seed.numel() != 1 or step.dtype != torch.int32 or step.numel() != 1:
            raise ValueError(f"DropoutState: seed must be a 1-element int64 tensor and step a 1-element int32 tensor, "
                             f"got {seed.dtype} {tuple(seed.shape)} and {step.dtype} {tuple(step.shape)}")
        if seed.device != step.device:
            raise ValueError(f"DropoutState: seed and step must be on one device, got {seed.device} and {step.device}")
        self.seed, self.step = seed, step

    @classmethod
    def create(cls, seed: int, step: int = 0, device="cpu") -> "DropoutState":
        s = int(seed) & 0xFFFFFFFFFFFFFFFF
        return cls(torch.tensor([s - (1 << 64) if s >= 1 << 63 else s], dtype=torch.int64, device=device),
                   torch.tensor([int(step)], dtype=torch.int32, device=device))

    def advance(self) -> None:
        """``step += 1`` on the device (one launch, capturable)."""
        if self.step.is_cuda:
            from . import incr_
            incr_(self.step)
        else:
            self.step += 1


_bound = False


def _lib():
    global _bound
    from ..runtime.native import load_library
    lib = load_library()
    if not _bound:
        lib.adapcc_dropout.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_uint,
                                       c_float, c_void_p]
        _bound = True
    return lib


def drop_tail(who: str, p: float, state: DropoutState, site: int, device) -> tuple:
    """The trailing ctypes arguments ``(seed, step, site, thr, scale)`` every dropout entry point takes, checked."""
    if not isinstance(state, DropoutState):
        raise ValueError(f"{who}: state must be a DropoutState, got {type(state).__name__}")
    if state.seed.device != device:
        raise ValueError(f"{who}: the dropout state is on {state.seed.device}, the activation on {device}")
    if int(site) < 0:
        raise ValueError(f"{who}: site must be >= 0, got {site}")
    thr, scale = threshold(check_p(who, p))
    return c_void_p(state.seed.data_ptr()), c_void_p(state.step.data_ptr()), int(site), thr, scale


def _native(x: torch.Tensor, p: float, state: DropoutState, site: int) -> torch.Tensor:
    from ..runtime.native import NativeError, last_error
    cols = x.shape[-1]
    x2 = x.reshape(-1, cols).contiguous()
    y = torch.empty_like(x2)
    rc = _lib().adapcc_dropout(c_void_p(x2.data_ptr()), c_void_p(y.data_ptr()), x2.shape[0], cols, x2.element_size(),
                               *drop_tail("dropout", p, state, site, x.device),
                               c_void_p(torch.cuda.current_stream().cuda_stream))
    if rc != 0:
        raise NativeError(f"dropout failed: {last_error()}")
    return y.view(x.shape)


def _numpy(x: torch.Tensor, p: float, state: DropoutState, site: int) -> torch.Tensor:
    cols = x.shape[-1]
    keep = dropout_mask(x.numel() // cols, cols, p, int(state.seed.item()), int(state.step.item()), site)
    scale = threshold(p)[1]
    wide = x if x.dtype == torch.float64 else x.float()             # the product in fp32 (fp64 for fp64), rounded once
    return torch.where(torch.from_numpy(keep).view(x.shape), wide * scale, torch.zeros_like(wide)).to(x.dtype)


class _DropoutFn(torch.autograd.Function):
    """y = mask * scale * x; the backward is the same function of dy (the mask is recomputed, not stored)."""

    @staticmethod
    def forward(ctx, x, p, state, site):
        ctx.args = (p, state, site)
        return _apply(x, p, state, site)

    @staticmethod
    def backward(ctx, dy):
        return _apply(dy, *ctx.args), None, None, None


def _apply(x, p, state, site):
    if x.is_cuda:
        if x.dtype not in (torch.bfloat16, torch.float32) or x.shape[-1] % 8 != 0:
            raise ValueError(f"dropout: a CUDA tensor must be bf16 or fp32 with a last dimension that is a multiple of "
                             f"8, got {x.dtype} {tuple(x.shape)}")
        return _native(x, p, state, site)
    return _numpy(x, p, state, site)


def dropout(x: torch.Tensor, p: float, state: DropoutState, site: int) -> torch.Tensor:
    """``mask * scale * x`` with the mask of ``(state.seed, state.step, site)`` over ``x`` flattened to
    ``[rows, x.shape[-1]]``. CUDA bf16 / fp32: the stand-alone kernel (``csrc/ops_dropout.cu``), forward and backward
    the same launch; CPU: the numpy definition. The step is read when the kernels run, so forward and backward agree as
    long as ``state.advance()`` is not called between them."""
    check_p("dropout", p)
    if not isinstance(state, DropoutState):
        raise ValueError(f"dropout: state must be a DropoutState, got {type(state).__name__}")
    if state.seed.device != x.device:
        raise ValueError(f"dropout: the dropout state is on {state.seed.device}, the activation on {x.device}")
    return _DropoutFn.apply(x, p, state, site)
