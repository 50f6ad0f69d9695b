"""Expert-parallel token exchange (dispatch / combine) on the native symmetric-memory kernels.

``ExpertExchange`` owns four [E_local, world, capacity, d] bf16 buffers inside the communicator's
symmetric heap (tokens in, expert outputs, and their two gradients) and exposes two autograd
functions:

* ``dispatch(rows, expert, pos)``  rows [A, d] -> local expert buffer [E_local, world*capacity, d]
  (forward: every rank PUSHES its rows into the owners' buffers; backward: pulls the rows' grads),
* ``combine(out_buffer, expert, pos)`` -> rows [A, d] (forward: every rank PULLS its rows' results;
  backward: pushes the rows' grads into the owners' grad buffers).

``A`` = tokens x top_k assignments. Slot assignment (``assign``) gives each assignment its stable rank
among the assignments to the same expert (token order) with a fixed per-(expert, source) capacity;
assignments past capacity are dropped (their rows come back as zeros), the same rule as
``MoEMLP._local``, and every shape stays static — the whole MoE layer is CUDA-graph capturable.
Replaces fastmoe's count/assign-pos + grouped ncclSend/ncclRecv exchange
(/root/reference/third-party/fastmoe/cuda/local_exchange.cuh, global_exchange.h).
"""
from __future__ import annotations

import ctypes
from ctypes import c_int, c_ulonglong, c_void_p
from typing import Optional, Sequence

import torch

from ..runtime.native import NativeError, last_error

_bound = False


def _bind(lib):
    global _bound
    if not _bound:
        ip = ctypes.POINTER(c_int)
        lib.adapcc_barrier.argtypes = [c_void_p, ip, c_int, c_void_p]
        lib.adapcc_moe_assign.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]
        lib.adapcc_moe_exchange.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_ulonglong,
                                            c_int, c_int, c_int, c_int, c_void_p]
        _bound = True


def _s():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


class ExpertExchange:
    """Token dispatch / combine for expert parallelism over peer memory: ``moe_push_kernel`` stores each token row
    directly into the symmetric window of the rank that owns its expert, ``moe_pull_kernel`` reads the expert
    outputs back (csrc/moe.cu) — the role of fastmoe's ``global_scatter / global_gather`` over grouped
    ``ncclSend/ncclRecv`` (third-party/fastmoe/cuda/global_exchange.h:11-55), without a collective library."""

    def __init__(self, comm, n_expert_local: int, capacity: int, d_model: int, active: Optional[Sequence[int]] = None):
        self.comm, self.e_local, self.capacity, self.d = comm, n_expert_local, capacity, d_model
        self.world, self.rank = comm.world, comm.rank
        self.active = list(range(comm.world)) if active is None else list(active)
        _bind(comm.lib)
        n = n_expert_local * self.world * capacity * d_model
        base = comm.lib.adapcc_ctx_heap_ptr(comm.handle)
        self.bufs, self.offs = {}, {}
        for name in ("x", "y", "gy", "gx"):
            t = comm.symm_empty(n, torch.bfloat16)
            t.zero_()
            self.bufs[name] = t.view(n_expert_local, self.world * capacity, d_model)
            self.offs[name] = t.data_ptr() - base
        self.n_expert = n_expert_local * self.world

    # -- raw ops -------------------------------------------------------------------------------
    def barrier(self):
        arr = (c_int * len(self.active))(*self.active)
        if self.comm.lib.adapcc_barrier(self.comm.handle, arr, len(self.active), _s()) != 0:
            raise NativeError(f"barrier failed: {last_error()}")

    def assign(self, expert: torch.Tensor):
        """expert: int32 [A] global expert ids -> (pos int32 [A], counts int32 [n_expert]).

        pos[i] = number of earlier assignments to the same expert, or -1 when that is >= capacity (dropped) or the id
        is out of range; counts = uncapped assignments per expert. Identical on every run."""
        if expert.dtype != torch.int32 or not expert.is_cuda or not expert.is_contiguous():
            raise TypeError(f"assign: expert ids must be a contiguous int32 CUDA tensor, got {expert.dtype}")
        counts = torch.zeros(self.n_expert, dtype=torch.int32, device=expert.device)
        pos = torch.empty_like(expert)
        if self.comm.lib.adapcc_moe_assign(c_void_p(expert.data_ptr()), expert.numel(), self.n_expert, self.capacity,
                                           c_void_p(counts.data_ptr()), c_void_p(pos.data_ptr()), _s()) != 0:
            raise NativeError(f"moe_assign failed: {last_error()}")
        return pos, counts

    def _exchange(self, direction: int, rows: torch.Tensor, expert, pos, which: str):
        assert rows.dtype == torch.bfloat16 and rows.is_contiguous() and rows.shape[1] == self.d
        rc = self.comm.lib.adapcc_moe_exchange(self.comm.handle, direction, c_void_p(rows.data_ptr()),
                                               c_void_p(expert.data_ptr()), c_void_p(pos.data_ptr()), None,
                                               self.offs[which], self.e_local, self.capacity, self.d, rows.shape[0],
                                               _s())
        if rc != 0:
            raise NativeError(f"moe_exchange failed: {last_error()}")

    # -- autograd ------------------------------------------------------------------------------
    def dispatch(self, rows, expert, pos):
        return _Dispatch.apply(rows, expert, pos, self)

    def combine(self, out_buf, expert, pos, n_rows):
        return _Combine.apply(out_buf, expert, pos, self, n_rows)


class _Dispatch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rows, expert, pos, ex: ExpertExchange):
        ctx.ex, ctx.n = ex, rows.shape[0]
        ctx.save_for_backward(expert, pos)
        ex.bufs["x"].zero_()
        ex.barrier()                                   # everyone's buffer is clean
        ex._exchange(0, rows.contiguous(), expert, pos, "x")
        ex.barrier()                                   # all rows have landed
        return ex.bufs["x"]

    @staticmethod
    def backward(ctx, g_buf):
        ex = ctx.ex
        expert, pos = ctx.saved_tensors
        ex.bufs["gx"].copy_(g_buf)                     # publish the grads of my experts' inputs
        ex.barrier()
        g_rows = torch.empty(ctx.n, ex.d, dtype=torch.bfloat16, device=g_buf.device)
        ex._exchange(1, g_rows, expert, pos, "gx")
        ex.barrier()                                   # peers are done reading before the next overwrite
        return g_rows, None, None, None


class _Combine(torch.autograd.Function):
    @staticmethod
    def forward(ctx, out_buf, expert, pos, ex: ExpertExchange, n_rows):
        ctx.ex = ex
        ctx.save_for_backward(expert, pos)
        ex.bufs["y"].copy_(out_buf)                    # publish my experts' outputs
        ex.barrier()
        rows = torch.empty(n_rows, ex.d, dtype=torch.bfloat16, device=out_buf.device)
        ex._exchange(1, rows, expert, pos, "y")
        ex.barrier()
        return rows

    @staticmethod
    def backward(ctx, g_rows):
        ex = ctx.ex
        expert, pos = ctx.saved_tensors
        ex.bufs["gy"].zero_()
        ex.barrier()
        ex._exchange(0, g_rows.contiguous(), expert, pos, "gy")
        ex.barrier()
        return ex.bufs["gy"].clone(), None, None, None, None
