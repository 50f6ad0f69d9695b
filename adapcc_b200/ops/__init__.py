"""Hand-written sm_90a ops used by the training engine and the workloads (bound through the same
in-tree ``libadapcc.so`` as the collectives). Every function launches on the current CUDA stream
and fails loudly if the native library is missing — there is no silent PyTorch fallback on a GPU.
"""
from __future__ import annotations

import ctypes
import math
from ctypes import c_float, c_int, c_longlong, c_uint, c_void_p
from typing import Optional

import torch

from ..constants import DTYPE_IDS
from ..runtime.native import NativeError, last_error, load_library

_bound = False


def _lib():
    global _bound
    lib = load_library()
    if not _bound:
        lib.adapcc_sumsq.argtypes = [c_void_p, c_longlong, c_int, c_void_p, c_void_p]
        lib.adapcc_grad_accum.argtypes = [c_void_p, c_void_p, c_longlong, c_int, c_int, c_void_p]
        lib.adapcc_grad_fold.argtypes = [c_void_p, c_void_p, c_longlong, c_int, c_float, c_void_p]
        lib.adapcc_fused_adamw.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int,
                                           c_float, c_float, c_float, c_float, c_float, c_int, c_float, c_float,
                                           c_void_p, c_void_p, c_void_p]
        lib.adapcc_fused_adamw_lr.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int,
                                              c_float, c_float, c_float, c_float, c_float, c_int, c_float, c_float,
                                              c_void_p, c_void_p, c_void_p, c_void_p]
        lib.adapcc_fused_sgd.argtypes = [c_void_p, c_void_p, c_void_p, c_longlong, c_int, c_int, c_float, c_float,
                                         c_void_p]
        lib.adapcc_incr_int.argtypes = [c_void_p, c_void_p]
        lib.adapcc_zero_adamw_bcast.argtypes = [c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p,
                                                c_void_p, c_longlong] + [c_float] * 7 + [c_void_p, c_void_p, c_void_p]
        lib.adapcc_fused_ce.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]
        lib.adapcc_fused_ce_scaled.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]
        lib.adapcc_embed_sum_fwd.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]
        lib.adapcc_embed_sum_bwd.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p,
                                             c_void_p, c_void_p, c_void_p]
        drop = [c_void_p, c_void_p, c_int, c_uint, c_float]            # seed, step, site, thr, scale
        lib.adapcc_embed_sum_drop_fwd.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p] + drop + [c_void_p]
        lib.adapcc_embed_sum_drop_bwd.argtypes = ([c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p,
                                                   c_void_p, c_void_p] + drop + [c_void_p])
        lib.adapcc_embed_bwd_reset.argtypes = [c_void_p, c_void_p, c_longlong, c_void_p, c_longlong, c_void_p]
        lib.adapcc_decode_attn.argtypes = [c_void_p] * 5 + [c_int] * 5 + [c_void_p] * 4
        lib.adapcc_kv_quantize.argtypes = [c_void_p] * 5 + [c_int] * 5 + [c_void_p]
        lib.adapcc_decode_attn_work.argtypes = [c_int] * 4
        lib.adapcc_decode_attn_work.restype = c_longlong
        lib.adapcc_lm_head_logits.argtypes = [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p]
        lib.adapcc_sample_tokens.argtypes = ([c_void_p, c_int, c_int, c_int, c_float, c_int, c_float]
                                             + [c_void_p] * 3 + [c_int, c_void_p, c_int, c_void_p, c_int]
                                             + [c_void_p] * 3 + [c_int, c_void_p])
        lib.adapcc_sample_tokens_filtered.argtypes = ([c_void_p, c_int, c_int, c_int, c_float, c_int]
                                                      + [c_float] * 5 + [c_void_p] * 3
                                                      + [c_int, c_void_p, c_int, c_void_p, c_int]
                                                      + [c_void_p] * 3 + [c_int, c_float, c_void_p])
        lib.adapcc_beam_step.argtypes = ([c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int]
                                         + [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int]
                                         + [c_void_p] * 11 + [c_float, c_void_p])
        lib.adapcc_beam_sample_step.argtypes = ([c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int]
                                                + [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int]
                                                + [c_void_p] * 11 + [c_float, c_int, c_float, c_void_p]
                                                + [c_float] * 5 + [c_void_p])
        lib.adapcc_beam_stochastic_step.argtypes = ([c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                                     c_int, c_void_p, c_int, c_void_p, c_int, c_int]
                                                    + [c_void_p] * 14 + [c_float, c_int, c_float, c_void_p]
                                                    + [c_float] * 5 + [c_void_p])
        lib.adapcc_kv_reorder.argtypes = [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p] * 3 + [c_int] + [c_void_p] * 4
        lib.adapcc_penalize_repeats.argtypes = ([c_void_p, c_int, c_int, c_int, c_void_p, c_int] + [c_void_p] * 5
                                                + [c_int, c_float, c_int, c_void_p, c_void_p, c_int, c_int]
                                                + [c_float, c_float, c_int, c_void_p])
        lib.adapcc_guidance_mix.argtypes = [c_void_p, c_int, c_int, c_int, c_float, c_void_p]
        lib.adapcc_cs_sim_numel.argtypes = [c_int] * 3
        lib.adapcc_cs_sim_numel.restype = c_longlong
        lib.adapcc_cand_attn.argtypes = [c_void_p] * 7 + [c_int] * 6 + [c_void_p, c_void_p]
        lib.adapcc_cs_select.argtypes = ([c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_int]
                                         + [c_void_p] * 5)
        lib.adapcc_cs_rerank.argtypes = ([c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p,
                                          c_void_p, c_int] + [c_void_p] * 4 + [c_int, c_void_p, c_void_p, c_int]
                                         + [c_void_p] * 5 + [c_int] * 3 + [c_void_p])
        lib.adapcc_cs_context_init.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                               c_void_p]
        lib.adapcc_verify_attn.argtypes = [c_void_p] * 6 + [c_int] * 6 + [c_void_p, c_void_p]
        lib.adapcc_lookup_argmax.argtypes = [c_void_p] + [c_int] * 6 + [c_void_p, c_int] + [c_void_p] * 5
        lib.adapcc_lookup_accept.argtypes = ([c_int] * 2 + [c_void_p, c_int] + [c_void_p] * 4 + [c_int]
                                             + [c_void_p] * 4 + [c_int, c_void_p, c_void_p, c_void_p])
        lib.adapcc_lookup_draft.argtypes = [c_void_p] + [c_int] * 5 + [c_void_p] * 7
        lib.adapcc_sample_slots.argtypes = ([c_void_p] + [c_int] * 6 + [c_float, c_int] + [c_float] * 5
                                            + [c_void_p] * 5 + [c_int, c_void_p, c_int] + [c_void_p] * 5
                                            + [c_float, c_void_p])
        lib.adapcc_spec_slots.argtypes = ([c_void_p] + [c_int] * 4 + [c_float, c_int] + [c_float] * 5
                                          + [c_void_p] * 5 + [c_int, c_void_p, c_int] + [c_void_p] * 6
                                          + [c_float, c_void_p])
        lib.adapcc_assist_round.argtypes = [c_void_p] + [c_int] * 5 + [c_void_p] * 10
        _bound = True
    return lib


def _stream() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def _dt(t: torch.Tensor) -> int:
    return DTYPE_IDS[str(t.dtype).replace("torch.", "")]


def _ck(rc: int, what: str) -> None:
    if rc != 0:
        raise NativeError(f"{what} failed: {last_error()}")


def _ptr(t: Optional[torch.Tensor]) -> c_void_p:
    """``t``'s data pointer; a null pointer for None."""
    return c_void_p(t.data_ptr() if t is not None else None)


def _id_list(who: str, name: str, t: Optional[torch.Tensor], cap: int):
    """(pointer, count) of an optional id list, which must be a contiguous 1-D int32 tensor of at most ``cap`` ids."""
    if t is not None and (t.dtype != torch.int32 or not t.is_contiguous() or t.dim() != 1 or t.numel() > cap):
        raise ValueError(f"{who}: {name} must be a contiguous 1-D int32 tensor of at most {cap} ids, got {t.dtype} "
                         f"{tuple(t.shape)}")
    return c_void_p(t.data_ptr() if t is not None and t.numel() else None), t.numel() if t is not None else 0


def _same_device(who: str, dev: torch.device, tensors) -> None:
    """``ValueError`` unless ``dev`` is a CUDA device and every tensor of ``tensors`` (None skipped) is on it."""
    tensors = [t for t in tensors if t is not None]
    if dev.type != "cuda" or any(t.device != dev for t in tensors):
        raise ValueError(f"{who}: all tensors must be on one CUDA device, got {dev} and "
                         f"{sorted(set(str(t.device) for t in tensors))}")


def sumsq_(grad: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out (1-element fp32, already zeroed) += sum(grad**2)."""
    _ck(_lib().adapcc_sumsq(c_void_p(grad.data_ptr()), grad.numel(), _dt(grad), c_void_p(out.data_ptr()), _stream()),
        "sumsq")
    return out


def _check_accum(who: str, grad: torch.Tensor, acc: torch.Tensor) -> None:
    if acc.dtype != torch.float32 or acc.numel() != grad.numel() or not (grad.is_contiguous() and acc.is_contiguous()):
        raise ValueError(f"{who}: acc must be a contiguous fp32 tensor of grad's {grad.numel()} elements, got {acc.dtype} "
                         f"{tuple(acc.shape)} (grad {grad.dtype} {tuple(grad.shape)})")


def grad_accum_(grad: torch.Tensor, acc: torch.Tensor, first: bool) -> torch.Tensor:
    """acc = f32(grad) when ``first``, else acc = f32(acc + f32(grad)): one micro-batch's (bf16 or fp32) gradient into
    the fp32 accumulator, each add rounded on its own. Both 16-byte aligned, numel a multiple of 8."""
    _check_accum("grad_accum", grad, acc)
    _ck(_lib().adapcc_grad_accum(c_void_p(grad.data_ptr()), c_void_p(acc.data_ptr()), grad.numel(), _dt(grad),
                                 int(bool(first)), _stream()), "grad_accum")
    return acc


def grad_fold_(grad: torch.Tensor, acc: torch.Tensor, scale: float) -> torch.Tensor:
    """In place: grad = round(f32(f32(acc + f32(grad)) * f32(scale))), the last micro-batch's gradient folded into the
    accumulator and scaled (by 1/M for the mean over M micro-batches), each add and multiply rounded on its own."""
    _check_accum("grad_fold", grad, acc)
    _ck(_lib().adapcc_grad_fold(c_void_p(grad.data_ptr()), c_void_p(acc.data_ptr()), grad.numel(), _dt(grad),
                                float(scale), _stream()), "grad_fold")
    return grad


def fused_adamw_(param: torch.Tensor, grad: torch.Tensor, master: torch.Tensor, m: torch.Tensor, v: torch.Tensor, *,
                 lr: float, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.01, step: int = 1,
                 max_norm: float = 0.0, grad_scale: float = 1.0, sumsq: Optional[torch.Tensor] = None,
                 step_tensor: Optional[torch.Tensor] = None, lr_tensor: Optional[torch.Tensor] = None) -> None:
    """One launch: clip (coefficient derived on the device from ``sumsq``), AdamW on the fp32
    master/m/v, write-back of the (bf16 or fp32) parameters. ``step_tensor`` (int32 on device) makes
    the bias correction replayable inside a CUDA graph; ``lr_tensor`` (fp32 on device) does the same for the learning
    rate, so a schedule only has to update that scalar between replays."""
    _ck(_lib().adapcc_fused_adamw_lr(c_void_p(param.data_ptr()), c_void_p(grad.data_ptr()), c_void_p(master.data_ptr()),
                                     c_void_p(m.data_ptr()), c_void_p(v.data_ptr()), param.numel(), _dt(param), _dt(grad),
                                     lr, betas[0], betas[1], eps, weight_decay, int(step), max_norm, grad_scale,
                                     c_void_p(sumsq.data_ptr() if sumsq is not None else None),
                                     c_void_p(step_tensor.data_ptr() if step_tensor is not None else None),
                                     c_void_p(lr_tensor.data_ptr() if lr_tensor is not None else None), _stream()),
        "fused_adamw")


def zero_adamw_bcast_(comm, param_shard: torch.Tensor, grad_shard: torch.Tensor, master: torch.Tensor,
                      m: torch.Tensor, v: torch.Tensor, *, lr: float, betas=(0.9, 0.999), eps: float = 1e-8,
                      weight_decay: float = 0.01, max_norm: float = 0.0, grad_scale: float = 1.0,
                      sumsq: Optional[torch.Tensor] = None, step_tensor: torch.Tensor = None) -> None:
    """ZeRO-1 step for one shard (csrc/zero.cu): AdamW on this rank's slice of the (symmetric-heap) parameter
    buffer; the updated bf16 parameters are written through the heap's multicast alias (``multimem.st``: the switch
    replicates them into every rank's copy) or, without multicast, stored into every peer's buffer. ``param_shard``
    must be a view inside ``comm``'s symmetric heap; master / m / v are the shard's fp32 state. The engine's default at
    N > 1 (``tests/gpu_zero1_worker.py``: parity with the replicated optimizer at 2 and 8 GPUs)."""
    n = param_shard.numel()
    if n == 0:
        return
    off = comm.heap_offset(param_shard)
    mc = comm.heap_mc_ptr()
    peers = None
    npeers = 0
    if not mc:
        ptrs = [comm.peer_heap_ptr(r) for r in range(comm.world)]
        peers = (c_void_p * len(ptrs))(*ptrs)
        npeers = len(ptrs)
    _ck(_lib().adapcc_zero_adamw_bcast(c_void_p(mc or None), peers, npeers, off, c_void_p(grad_shard.data_ptr()),
                                       c_void_p(master.data_ptr()), c_void_p(m.data_ptr()), c_void_p(v.data_ptr()), n,
                                       lr, betas[0], betas[1], eps, weight_decay, max_norm, grad_scale,
                                       c_void_p(sumsq.data_ptr() if sumsq is not None else None),
                                       c_void_p(step_tensor.data_ptr()), _stream()), "zero_adamw_bcast")


def fused_sgd_(param, grad, master, *, lr: float, grad_scale: float = 1.0) -> None:
    _ck(_lib().adapcc_fused_sgd(c_void_p(param.data_ptr()), c_void_p(grad.data_ptr()), c_void_p(master.data_ptr()),
                                param.numel(), _dt(param), _dt(grad), lr, grad_scale, _stream()), "fused_sgd")


def incr_(t: torch.Tensor) -> None:
    _ck(_lib().adapcc_incr_int(c_void_p(t.data_ptr()), _stream()), "incr")


def fused_ce_(logits: torch.Tensor, labels: torch.Tensor, vocab: int,
              grad_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """In place: bf16 ``logits`` [rows, stride] become d(sum of row losses)/d logits; returns the
    per-row losses (fp32). Rows whose label is negative are ignored (loss 0, zero gradient).
    ``grad_scale`` (1-element fp32 on the device): the gradient is multiplied by it inside the kernel (the row losses
    are not), so a mean loss's 1/n needs no extra pass over the gradient or over the GEMMs fed by it."""
    assert logits.dtype == torch.bfloat16 and logits.is_contiguous() and logits.dim() == 2
    rows, stride = logits.shape
    # the kernel reads labels[row] as int64 for every row: anything else would be read out of bounds
    if (labels.dtype != torch.int64 or not labels.is_contiguous() or labels.numel() != rows
            or labels.device != logits.device):
        raise ValueError(f"fused_ce_: labels must be a contiguous int64 tensor of {rows} elements on "
                         f"{logits.device}, got {labels.dtype} {tuple(labels.shape)} on {labels.device}")
    row_loss = torch.empty(rows, dtype=torch.float32, device=logits.device)
    gs = None
    if grad_scale is not None:
        assert grad_scale.dtype == torch.float32 and grad_scale.numel() == 1 and grad_scale.is_cuda
        gs = grad_scale.data_ptr()
    _ck(_lib().adapcc_fused_ce_scaled(c_void_p(logits.data_ptr()), c_void_p(labels.data_ptr()),
                                      c_void_p(row_loss.data_ptr()), rows, int(vocab), stride, c_void_p(gs), _stream()),
        "fused_ce")
    return row_loss


# ---- fused embedding sum (csrc/ops_embed.cu) ----------------------------------------------------------------------
_embed_work = {}


def _embed_buffers(device, n_owner: int, scratch_elems: int):
    """(owner int32 [n_owner] all INT_MAX, maxbits int32 [n_owner] all zero, scratch int64 fixed point [scratch_elems]
    all zero): the backward kernels leave all three in exactly that state again, so they are initialised once per
    (device, size)."""
    key = (device.index, n_owner, scratch_elems)
    buf = _embed_work.get(key)
    if buf is None:
        owner = torch.empty(n_owner, dtype=torch.int32, device=device)
        maxbits = torch.empty(n_owner, dtype=torch.int32, device=device)
        scratch = torch.empty(scratch_elems, dtype=torch.int64, device=device)
        _ck(_lib().adapcc_embed_bwd_reset(c_void_p(owner.data_ptr()), c_void_p(maxbits.data_ptr()), n_owner,
                                          c_void_p(scratch.data_ptr()), scratch_elems, _stream()), "embed_bwd_reset")
        buf = _embed_work[key] = (owner, maxbits, scratch)
    return buf


def _ptr_array(tensors):
    return (c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


class _EmbedSumFn(torch.autograd.Function):
    """y[t] = sum_k tables[spec[k]][idx_k[t]] (bf16, fp32 sum); args: spec, drop, K index tensors, then the tables.
    ``drop`` = (p, state, site) or None: y[t] = dropout(sum) with row t of the mask (ops/dropout.py), applied to the
    fp32 sum forward and to dY backward, recomputed both times."""

    @staticmethod
    def forward(ctx, spec, drop, *args):
        K = len(spec)
        idx, tables = args[:K], args[K:]
        n, D = idx[0].numel(), tables[0].shape[1]
        out = torch.empty(n, D, dtype=tables[0].dtype, device=tables[0].device)
        ctx.drop = None
        if drop is None:
            _ck(_lib().adapcc_embed_sum_fwd(_ptr_array([tables[j] for j in spec]), _ptr_array(idx), K, n, D,
                                            c_void_p(out.data_ptr()), _stream()), "embed_sum_fwd")
        else:
            from .dropout import drop_tail
            ctx.drop = drop_tail("fused_embedding_sum", *drop, out.device)
            ctx.state = drop[1]                            # owns the tensors ctx.drop points at
            _ck(_lib().adapcc_embed_sum_drop_fwd(_ptr_array([tables[j] for j in spec]), _ptr_array(idx), K, n, D,
                                                 c_void_p(out.data_ptr()), *ctx.drop, _stream()), "embed_sum_drop_fwd")
        ctx.spec, ctx.idx, ctx.tables, ctx.n, ctx.D = spec, idx, tables, n, D
        return out

    @staticmethod
    def backward(ctx, dy):
        from .layers import _sink

        spec, idx, tables, n, D = ctx.spec, ctx.idx, ctx.tables, ctx.n, ctx.D
        K = len(spec)
        dy = dy.contiguous()
        base, off = [], 0
        for t in tables:                                   # owner slots: one range per distinct table
            base.append(off)
            off += t.shape[0]
        owner, maxbits, scratch = _embed_buffers(dy.device, off, K * n * D)
        sinks = [_sink(t) for t in tables]
        grads, ret = [], []
        for t, s in zip(tables, sinks):
            if s is not None and s.begin():                # straight into the engine's flat gradient view (which may
                grads.append(t.grad)                       # already hold another contribution, e.g. a tied LM head)
                ret.append(None)
            else:
                g = torch.zeros_like(t)
                grads.append(g)
                ret.append(g)
        ob = (c_int * K)(*[base[j] for j in spec])
        work = (c_void_p(owner.data_ptr()), c_void_p(maxbits.data_ptr()), c_void_p(scratch.data_ptr()))
        if ctx.drop is None:
            _ck(_lib().adapcc_embed_sum_bwd(c_void_p(dy.data_ptr()), _ptr_array(idx),
                                            _ptr_array([grads[j] for j in spec]), ob, K, n, D, *work, _stream()),
                "embed_sum_bwd")
        else:
            _ck(_lib().adapcc_embed_sum_drop_bwd(c_void_p(dy.data_ptr()), _ptr_array(idx),
                                                 _ptr_array([grads[j] for j in spec]), ob, K, n, D, *work, *ctx.drop,
                                                 _stream()), "embed_sum_drop_bwd")
        for s in sinks:
            if s is not None:
                s.done()
        return (None, None) + (None,) * K + tuple(ret)


def fused_embedding_sum(tables, lookups, drop=None) -> torch.Tensor:
    """``sum_k tables[j_k][idx_k]`` for ``lookups = [(j_k, idx_k), ...]`` (idx_k: int64, all the same number of
    elements n) -> [n, D]. bf16 CUDA tables with int64 CUDA indices: one forward kernel and a sort-free three-launch
    backward that accumulates duplicate rows in 64-bit fixed point (csrc/ops_embed.cu). Anything else: plain
    ``F.embedding`` sums. ``drop = (p, state, site)``: dropout of the sum (``ops/dropout.py``), inside the same kernels
    on the fused path and through ``dropout`` otherwise."""
    t0 = tables[0]
    fused = (t0.is_cuda and all(t.dtype == torch.bfloat16 and t.is_contiguous() and t.shape[1] == t0.shape[1]
                                for t in tables) and t0.shape[1] % 8 == 0 and 1 <= len(lookups) <= 4
             and all(ix.dtype == torch.int64 and ix.device == t0.device for _, ix in lookups))
    if not fused:
        out = None
        for j, ix in lookups:
            e = torch.nn.functional.embedding(ix.reshape(-1), tables[j])
            out = e if out is None else out + e
        if drop is not None:
            from .dropout import dropout
            out = dropout(out, *drop)
        return out
    spec = tuple(int(j) for j, _ in lookups)
    idx = tuple(ix.reshape(-1).contiguous() for _, ix in lookups)
    return _EmbedSumFn.apply(spec, drop, *idx, *tables)


# ---- decode attention over a KV cache (csrc/ops_decode.cu) -------------------------------------------------------
def decode_attention_work_numel(batch: int, n_head: int, head_dim: int, t_max: int) -> int:
    """fp32 elements of the split-partials workspace ``decode_attention_`` needs for this cache shape."""
    return int(_lib().adapcc_decode_attn_work(batch, n_head, head_dim, t_max))


def _check_decode_attn(who: str, kq: int, qkv, k_cache, v_cache, lens, out, work, nq=None, side_k=None, side_v=None,
                       k_scale=None, v_scale=None):
    """``ValueError`` (prefixed ``who``) unless the tensors fit a decode-style attention of ``kq`` queries per cache row
    (``csrc/ops_decode.cu``); returns the cache shape (B, H, t_max, Dh). With ``k_scale`` / ``v_scale`` the caches are
    fp8 (uint8 bytes, ``ops/kvcache.py``)."""
    def bad(msg):
        raise ValueError(f"{who}: {msg}")

    fp8 = k_scale is not None or v_scale is not None
    rows = [(name, t) for name, t in (("out", out), ("side_k", side_k), ("side_v", side_v)) if t is not None]
    caches = [("k_cache", k_cache), ("v_cache", v_cache)]
    for name, t in [("qkv", qkv)] + ([] if fp8 else caches) + rows:
        if t.dtype != torch.bfloat16:
            bad(f"{name} must be bf16, got {t.dtype}")
    if fp8:
        if k_scale is None or v_scale is None:
            bad("an fp8 cache needs both k_scale and v_scale")
        for name, t in caches:
            if t.dtype != torch.uint8:
                bad(f"{name} must be uint8 (fp8 e4m3 bytes) with scales, got {t.dtype}")
    if k_cache.dim() != 4 or not k_cache.is_contiguous() or v_cache.shape != k_cache.shape or not v_cache.is_contiguous():
        bad(f"k_cache / v_cache must be contiguous [B, H, t_max, Dh] of one shape, got {tuple(k_cache.shape)} "
            f"and {tuple(v_cache.shape)}")
    B, H, t_max, Dh = k_cache.shape
    R = B * kq
    if qkv.dim() != 2 or qkv.shape != (R, 3 * H * Dh) or qkv.stride(1) != 1:
        bad(f"qkv must be [{R}, {3 * H * Dh}] with unit column stride, got {tuple(qkv.shape)} stride {qkv.stride()}")
    for name, t in rows:
        if t.shape != (R, H * Dh) or not t.is_contiguous():
            bad(f"{name} must be a contiguous [{R}, {H * Dh}] tensor, got {tuple(t.shape)}")
    for name, t in (("lens", lens), ("nq", nq)):
        if t is not None and (t.dtype != torch.int32 or not t.is_contiguous() or t.numel() != B):
            bad(f"{name} must be a contiguous int32 tensor of {B} elements, got {t.dtype} {tuple(t.shape)}")
    if work.dtype != torch.float32 or not work.is_contiguous():
        bad(f"work must be a contiguous fp32 tensor, got {work.dtype}")
    for name, t in (("k_scale", k_scale), ("v_scale", v_scale)):
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or t.shape != (B, H, t_max)):
            bad(f"{name} must be a contiguous fp32 [{B}, {H}, {t_max}] tensor, got {t.dtype} {tuple(t.shape)}")
    _same_device(who, k_cache.device, (qkv, v_cache, lens, nq, out, side_k, side_v, work, k_scale, v_scale))
    need = decode_attention_work_numel(R, H, Dh, t_max)
    if work.numel() < need:
        bad(f"work holds {work.numel()} elements, {need} needed")
    return B, H, t_max, Dh


def decode_attention_(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, lens: torch.Tensor,
                      out: torch.Tensor, work: torch.Tensor, *, k_scale: Optional[torch.Tensor] = None,
                      v_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Attention of one new token per row over a KV cache, in place. ``qkv`` bf16 [B, 3·H·Dh] (q | k | v of the new
    token; rows may be strided), ``k_cache`` / ``v_cache`` bf16 [B, H, t_max, Dh], ``lens`` int32 [B] (tokens already
    cached per row; read, never written). Stores the new k / v at position ``lens[b]`` and writes
    ``out[b] = softmax(q·K[0..lens[b]]ᵀ / √Dh)·V[0..lens[b]]`` (bf16 [B, H·Dh], fp32 softmax and accumulation). A row
    with ``lens[b]`` outside [0, t_max) is left alone and its output is zero. ``work``: fp32, at least
    ``decode_attention_work_numel`` elements. Repeatable bit for bit; no host sync, so it can be captured in a graph.

    With ``k_scale`` / ``v_scale`` (fp32 [B, H, t_max]) the caches are fp8: uint8 e4m3 bytes [B, H, t_max, Dh], read
    and stored as ``ops/kvcache.py`` defines. The new token attends to its own k / v unquantized and stores them
    quantized; the output has the bits of the bf16 op on a bf16 cache holding the dequantized values."""
    B, H, t_max, Dh = _check_decode_attn("decode_attention_", 1, qkv, k_cache, v_cache, lens, out, work,
                                         k_scale=k_scale, v_scale=v_scale)
    _ck(_lib().adapcc_decode_attn(_ptr(qkv), _ptr(k_cache), _ptr(v_cache), _ptr(lens), _ptr(out), B, H, Dh, t_max,
                                  qkv.stride(0), _ptr(work), _ptr(k_scale), _ptr(v_scale), _stream()), "decode_attn")
    return out


def kv_quantize_(kv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, k_scale: torch.Tensor,
                 v_scale: torch.Tensor) -> None:
    """The prefill of one layer's fp8 cache: quantizes positions [0, T) of every row in place, as ``ops/kvcache.py``
    defines. ``kv`` is the c_attn output, contiguous bf16 [B, T, 3·H·Dh] (q | k | v), read in place; ``k_cache`` /
    ``v_cache`` uint8 [B, H, t_max, Dh] and ``k_scale`` / ``v_scale`` fp32 [B, H, t_max]. Positions >= T are not
    touched. The grid depends on the shapes only; no host sync."""
    def bad(msg):
        raise ValueError(f"kv_quantize_: {msg}")

    if k_cache.dtype != torch.uint8 or v_cache.dtype != torch.uint8:
        bad(f"k_cache / v_cache must be uint8 (fp8 e4m3 bytes), got {k_cache.dtype}, {v_cache.dtype}")
    if k_cache.dim() != 4 or not k_cache.is_contiguous() or v_cache.shape != k_cache.shape or not v_cache.is_contiguous():
        bad(f"k_cache / v_cache must be contiguous [B, H, t_max, Dh] of one shape, got {tuple(k_cache.shape)} and "
            f"{tuple(v_cache.shape)}")
    B, H, t_max, Dh = k_cache.shape
    for name, t in (("k_scale", k_scale), ("v_scale", v_scale)):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.shape != (B, H, t_max):
            bad(f"{name} must be a contiguous fp32 [{B}, {H}, {t_max}] tensor, got {t.dtype} {tuple(t.shape)}")
    if kv.dtype != torch.bfloat16 or kv.dim() != 3 or not kv.is_contiguous() or kv.shape[0] != B or \
            kv.shape[2] != 3 * H * Dh or not 1 <= kv.shape[1] <= t_max:
        bad(f"kv must be a contiguous bf16 [{B}, T, {3 * H * Dh}] tensor with 1 <= T <= {t_max}, got {kv.dtype} "
            f"{tuple(kv.shape)}")
    _same_device("kv_quantize_", k_cache.device, (kv, v_cache, k_scale, v_scale))
    _ck(_lib().adapcc_kv_quantize(_ptr(kv), _ptr(k_cache), _ptr(v_cache), _ptr(k_scale), _ptr(v_scale), B,
                                  kv.shape[1], H, Dh, t_max, _stream()), "kv_quantize")


# ---- LM head and token sampling for generation (csrc/ops_sample.cu) ------------------------------------------------
LM_HEAD_MAX_ROWS = 64          # h rows the LM-head kernel takes per call (its h tile lives in shared memory)
SAMPLE_MAX_VOCAB = 56 * 1024   # vocabulary the sampler holds in shared memory per row
SAMPLE_MAX_IDS = 1024          # ids per suppress / stop list


def lm_head_logits_(h: torch.Tensor, weight: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """``out[b, i] = sum_d h[b, d] * weight[i, d]`` in place: ``h`` bf16 [B, D] with unit column stride (B <= 64),
    ``weight`` the contiguous bf16 [V, D] table, ``out`` contiguous fp32 [B, V]. fp32 accumulation in an order fixed by
    d alone, so a row's bits do not depend on B or the other rows; ``weight`` is read once per call. No host sync."""
    def bad(msg):
        raise ValueError(f"lm_head_logits_: {msg}")

    if h.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16 or out.dtype != torch.float32:
        bad(f"need bf16 h and weight and an fp32 out, got {h.dtype}, {weight.dtype}, {out.dtype}")
    if weight.dim() != 2 or not weight.is_contiguous():
        bad(f"weight must be a contiguous [V, D] tensor, got {tuple(weight.shape)} stride {weight.stride()}")
    V, D = weight.shape
    if h.dim() != 2 or h.shape[1] != D or h.stride(1) != 1 or not 1 <= h.shape[0] <= LM_HEAD_MAX_ROWS:
        bad(f"h must be [B, {D}] with unit column stride and 1 <= B <= {LM_HEAD_MAX_ROWS}, got {tuple(h.shape)} "
            f"stride {h.stride()}")
    B = h.shape[0]
    if out.shape != (B, V) or not out.is_contiguous():
        bad(f"out must be a contiguous [{B}, {V}] tensor, got {tuple(out.shape)}")
    if D % 8 != 0 or D > 1024 or h.stride(0) % 8 != 0:
        bad(f"D must be a multiple of 8 up to 1024 and h's row stride a multiple of 8, got D={D} stride {h.stride(0)}")
    dev = weight.device
    if dev.type != "cuda" or h.device != dev or out.device != dev:
        bad(f"all tensors must be on one CUDA device, got h {h.device}, weight {dev}, out {out.device}")
    _ck(_lib().adapcc_lm_head_logits(c_void_p(h.data_ptr()), h.stride(0), c_void_p(weight.data_ptr()), V, D,
                                     c_void_p(out.data_ptr()), B, _stream()), "lm_head_logits")
    return out


def sample_tokens_(logits: torch.Tensor, vocab: int, temperature: float, top_k: int, top_p: float,
                   seeds: torch.Tensor, pos: torch.Tensor, step: torch.Tensor, min_new: int,
                   suppress_ids: Optional[torch.Tensor], stop_ids: Optional[torch.Tensor], done: torch.Tensor,
                   next_ids: torch.Tensor, tokens: torch.Tensor, min_p: float = 0.0, typical_p: float = 1.0,
                   epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0, top_h: float = 0.0) -> None:
    """One seeded top-k / top-p draw per row, on the device (the definition in ``ops/sampling.py``, which computes the
    same in fp64). ``logits`` fp32 [B, ld] (the first ``vocab`` columns used), ``seeds`` int64 [B], ``pos`` int32 [B]
    (position of the drawn token: the Philox counter), ``step`` int32 [1] (tokens generated so far; incremented),
    ``suppress_ids`` / ``stop_ids`` int32 lists or None, ``done`` int32 [B]. Writes the token into ``next_ids`` int64
    [B] and column ``step`` of ``tokens`` int64 [B, max_new] (-1 for a stop id or a finished row) and sets ``done`` on
    a stop id. ``temperature == 0`` is greedy. No host sync, so it can be captured in a CUDA graph.

    ``min_p``, ``typical_p``, ``epsilon_cutoff`` and ``eta_cutoff`` (HuggingFace's truncation samplers; off at 0, 1,
    0 and 0) filter the ids that top-p kept, in that order, before the draw; ``top_h`` (HuggingFace's entropy-bounded
    top-h, in (0, 1]; 0: off) filters the row before top-k. None has an effect at temperature 0."""
    def bad(msg):
        raise ValueError(f"sample_tokens_: {msg}")

    if not temperature >= 0 or not top_k >= 0 or not 0 < top_p <= 1:
        bad(f"need temperature >= 0, top_k >= 0 and 0 < top_p <= 1, got {temperature}, {top_k}, {top_p}")
    from .sampling import check_filter_args

    check_filter_args("sample_tokens_", min_p, typical_p, epsilon_cutoff, eta_cutoff, top_h)
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1:
        bad(f"logits must be fp32 [B, ld] with unit column stride, got {logits.dtype} {tuple(logits.shape)}")
    B = logits.shape[0]
    if not 1 <= vocab <= min(logits.shape[1], SAMPLE_MAX_VOCAB):
        bad(f"vocab must be in [1, min(ld = {logits.shape[1]}, {SAMPLE_MAX_VOCAB})], got {vocab}")
    for name, t, dt in (("seeds", seeds, torch.int64), ("pos", pos, torch.int32), ("done", done, torch.int32),
                        ("next_ids", next_ids, torch.int64)):
        if t.dtype != dt or not t.is_contiguous() or t.numel() != B:
            bad(f"{name} must be a contiguous {dt} tensor of {B} elements, got {t.dtype} {tuple(t.shape)}")
    if step.dtype != torch.int32 or step.numel() != 1:
        bad(f"step must be a 1-element int32 tensor, got {step.dtype} {tuple(step.shape)}")
    if tokens.dtype != torch.int64 or tokens.dim() != 2 or tokens.shape[0] != B or not tokens.is_contiguous():
        bad(f"tokens must be a contiguous int64 [{B}, max_new] tensor, got {tokens.dtype} {tuple(tokens.shape)}")
    sup, n_sup = _id_list("sample_tokens_", "suppress_ids", suppress_ids, SAMPLE_MAX_IDS)
    stop, n_stop = _id_list("sample_tokens_", "stop_ids", stop_ids, SAMPLE_MAX_IDS)
    _same_device("sample_tokens_", logits.device, (seeds, pos, step, done, next_ids, tokens, suppress_ids, stop_ids))
    _ck(_lib().adapcc_sample_tokens_filtered(_ptr(logits), logits.stride(0), int(vocab), B, float(temperature),
                                             int(top_k), float(top_p), float(min_p), float(typical_p),
                                             float(epsilon_cutoff), float(eta_cutoff), _ptr(seeds), _ptr(pos),
                                             _ptr(step), int(min_new), sup, n_sup, stop, n_stop, _ptr(done),
                                             _ptr(next_ids), _ptr(tokens), tokens.shape[1], float(top_h), _stream()),
        "sample_tokens")


# ---- beam search selection and KV-cache reordering (csrc/ops_beam.cu) ----------------------------------------------
BEAM_MAX_BEAMS = 16            # beams per item
BEAM_MAX_STOP = 8              # stop ids (each row keeps its K + n_stop best candidates)
BEAM_MAX_SUPPRESS = 1024       # suppressed ids


class BeamState:
    """Device state of a batched beam search of ``batch`` items with ``num_beams`` beams each and up to ``max_new``
    tokens, as ``beam_step_`` reads and writes it. Rows are ``b * num_beams + k``.

    ``scores`` fp32 [B·K] running log-probability sums (beam 0 of each item at 0, the others dead at -inf);
    ``step`` int32 [1]; ``done`` int32 [B]; ``next_ids`` int64 [B·K] the new beams' tokens (the decode step's input);
    ``parent`` int32 [B·K] the row each new beam continues; ``hist_tok`` int64 / ``hist_back`` int32 [max_new, B·K]
    each step's tokens and parent beams (0..K-1); the finished sets ``fin_score`` fp32, ``fin_n`` and ``fin_src`` int32
    [B, K] (best first: normalised score, tokens without the stop token, and the beam whose history at step
    ``fin_n - 1`` holds them) with ``fin_count`` int32 [B]; ``pen`` fp32 [max_new + 1], ``pen[L] = L ** length_penalty``
    rounded to fp32 once on the host, so the kernel needs no ``powf``. With ``sample`` (beam sampling) the candidate
    scratch holds ``(BEAM_MAX_STOP + 1) · K`` keys per row, the most any sample draws, with ``cand_c`` fp32 beside it;
    a step with M = ``max(2, 1 + n_stop) · K`` uses the first ``B·K·M`` entries of each as [B·K, M].

    ``groups`` = G > 1 (diverse beam search, ``ops.beam.GroupBeamReference``; G divides K, not with ``sample``): group g
    owns beams ``g·K/G .. (g+1)·K/G - 1``, each group's beam 0 starts at 0, the finished arrays [B, K] are read as
    [B, G, K/G] (one set per group), ``fin_count`` and ``group_done`` are int32 [B·G], and ``done`` stays the item
    flag [B]: all of the item's groups are done.

    ``seeds`` (int64 [B], each item's Philox key; not with ``sample`` or ``groups``) makes the state stochastic beam
    search (``ops.beam.StochasticBeamReference``, rules R1-R8): ``scores`` are the live beams' log-probabilities φ,
    ``keys`` fp32 [B·K] their perturbed keys (beam 0 starts at the Gumbel of rule R1's start, rounded to fp32),
    ``fin_score`` holds the finished entries' keys and ``fin_phi`` fp32 [B, K] their log-probabilities, ``kappa`` fp32
    [B] the largest key pruned so far (-inf at the start), and ``cand_key`` / ``cand_phi`` fp32 [B·K, K + 1] the
    children each row offers, next to the first K + 1 entries of each ``cand`` row. ``length_penalty`` is unused."""

    def __init__(self, batch: int, num_beams: int, max_new: int, length_penalty: float, device, sample: bool = False,
                 groups: int = 1, seeds: Optional[torch.Tensor] = None):
        B, K, n, G = int(batch), int(num_beams), int(max_new), int(groups)
        if B < 1 or not 1 <= K <= BEAM_MAX_BEAMS or n < 1:
            raise ValueError(f"BeamState: need batch >= 1, 1 <= num_beams <= {BEAM_MAX_BEAMS} and max_new >= 1, got "
                             f"{batch}, {num_beams}, {max_new}")
        if not 1 <= G <= K or K % G != 0 or (G > 1 and sample):
            raise ValueError(f"BeamState: groups must divide num_beams = {K} and cannot be combined with sample, got "
                             f"{groups} (sample={sample})")
        if seeds is not None and (sample or G > 1 or seeds.dtype != torch.int64 or seeds.numel() != B):
            raise ValueError(f"BeamState: seeds (stochastic beam search) must be int64 with {B} elements and cannot "
                             f"be combined with sample or groups, got {seeds.dtype} {tuple(seeds.shape)} "
                             f"(sample={sample}, groups={groups})")
        self.batch, self.num_beams, self.max_new, self.length_penalty = B, K, n, float(length_penalty)
        self.groups = G
        i32, dev = dict(dtype=torch.int32, device=device), device
        self.scores = torch.full((B, K), float("-inf"), dtype=torch.float32, device=dev)
        self.scores[:, ::K // G] = 0.0
        self.scores = self.scores.reshape(B * K)
        self.step = torch.zeros(1, **i32)
        self.done = torch.zeros(B, **i32)
        self.next_ids = torch.zeros(B * K, dtype=torch.int64, device=dev)
        self.parent = torch.arange(B * K, **i32)
        self.hist_tok = torch.full((n, B * K), -1, dtype=torch.int64, device=dev)
        self.hist_back = torch.zeros(n, B * K, **i32)
        self.fin_score = torch.full((B, K), float("-inf"), dtype=torch.float32, device=dev)
        self.fin_n = torch.zeros(B, K, **i32)
        self.fin_src = torch.zeros(B, K, **i32)
        self.fin_count = torch.zeros(B * G, **i32)
        self.group_done = torch.zeros(B * G, **i32)
        self.pen = torch.tensor([float(L) ** self.length_penalty if L else 1.0 for L in range(n + 1)],
                                dtype=torch.float64).to(device=dev, dtype=torch.float32)
        self.sample = bool(sample)
        width = (BEAM_MAX_STOP + 1) * K if self.sample else K + BEAM_MAX_STOP
        self.cand = torch.empty(B * K, width, dtype=torch.int64, device=dev)
        self.cand_c = torch.empty(B * K, width, dtype=torch.float32, device=dev) if self.sample else None
        self.seeds = self.keys = self.fin_phi = self.kappa = self.cand_key = self.cand_phi = None
        if seeds is not None:
            from .beam import start_keys
            self.seeds = seeds.reshape(B).to(dev).contiguous()
            self.keys = torch.full((B, K), float("-inf"), dtype=torch.float32, device=dev)
            self.keys[:, 0] = torch.from_numpy(start_keys(self.seeds.cpu().tolist())).to(dev, torch.float32)
            self.keys = self.keys.reshape(B * K)
            self.fin_phi = torch.full((B, K), float("-inf"), dtype=torch.float32, device=dev)
            self.kappa = torch.full((B,), float("-inf"), dtype=torch.float32, device=dev)
            self.cand_key = torch.empty(B * K, K + 1, dtype=torch.float32, device=dev)
            self.cand_phi = torch.empty(B * K, K + 1, dtype=torch.float32, device=dev)

    def tensors(self):
        """Every device tensor of the state (what ``beam_step_`` checks for one device)."""
        return (self.scores, self.step, self.done, self.next_ids, self.parent, self.hist_tok, self.hist_back,
                self.fin_score, self.fin_n, self.fin_src, self.fin_count, self.group_done, self.pen, self.cand,
                self.cand_c, self.seeds, self.keys, self.fin_phi, self.kappa, self.cand_key, self.cand_phi)

    def finished(self):
        """The finished sets on the host: per item, per group, its ``(score, n, src)`` entries best first, with the
        log-probability φ as a fourth field in a stochastic state."""
        B, G, Kg = self.batch, self.groups, self.num_beams // self.groups
        count = self.fin_count.cpu().tolist()
        cols = [x.cpu().tolist() for x in (self.fin_score, self.fin_n, self.fin_src, self.fin_phi) if x is not None]
        return [[list(zip(*(c[b] for c in cols)))[g * Kg:g * Kg + count[b * G + g]] for g in range(G)]
                for b in range(B)]


def beam_step_(logits: torch.Tensor, vocab: int, state: BeamState, min_new: int = 0,
               suppress_ids: Optional[torch.Tensor] = None, stop_ids: Optional[torch.Tensor] = None,
               temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0,
               seeds: Optional[torch.Tensor] = None, diversity_penalty: float = 0.0, min_p: float = 0.0,
               typical_p: float = 1.0, epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0,
               top_h: float = 0.0) -> None:
    """One beam-search selection for every item, on the device (the definition in ``ops/beam.py``, which computes the
    same in fp64). ``logits`` fp32 [B·K, ld] (the first ``vocab`` columns used) are the beams' next-token logits;
    ``suppress_ids`` (removed while ``state.step < min_new``) and ``stop_ids`` (at most 8; they finish a hypothesis)
    are int32 lists or None. Updates ``state``: the new beams' tokens go into ``state.next_ids``, their parents into
    ``state.parent`` (for ``kv_reorder_``), and ``state.step`` is incremented. No host sync, so it can be captured in a
    CUDA graph.

    With ``seeds`` (int64 [B] on the device, each item's Philox key) the step is beam sampling
    (``BeamSampleReference``): a ``BeamState(..., sample=True)``, ``temperature > 0``, ``top_k`` (0: off) and
    ``top_p`` filter each beam's ids, and the candidates are drawn rather than ranked; vocab is at most
    ``SAMPLE_MAX_VOCAB``. Without ``seeds`` the sampling scalars are ignored. The truncation filters ``min_p``,
    ``typical_p``, ``epsilon_cutoff``, ``eta_cutoff`` and ``top_h`` (off at 0, 1, 0, 0 and 0) act in both sampled
    modes, as in ``sample_tokens_``; beam sampling keeps at least ``max(2, 1 + n_stop)`` ids in each.

    A state with ``groups`` > 1 is diverse beam search (``GroupBeamReference``): the groups select in order, a
    candidate's score lowered by ``diversity_penalty`` (finite, > 0; 0 for one group) per new beam of an earlier group
    of the item that took its token this step.

    A state with ``seeds`` is stochastic beam search (``StochasticBeamReference``): ``temperature > 0``, ``top_k`` and
    ``top_p`` filter each beam's ids as ``generate``'s sampler does, the state's own seeds drive the draws (``seeds``
    must be None) and vocab is at most ``SAMPLE_MAX_VOCAB``."""
    def bad(msg):
        raise ValueError(f"beam_step_: {msg}")

    if not isinstance(state, BeamState):
        bad(f"state must be a BeamState, got {type(state).__name__}")
    lam = float(diversity_penalty)
    if state.groups > 1 and not (math.isfinite(lam) and lam > 0):
        bad(f"a BeamState with {state.groups} groups needs a finite diversity_penalty > 0, got {diversity_penalty}")
    if state.groups == 1 and lam != 0:
        bad(f"diversity_penalty needs a BeamState with groups > 1, got {diversity_penalty}")
    if state.seeds is not None and seeds is not None:
        bad("a stochastic BeamState carries its items' seeds; pass seeds=None")
    if seeds is not None:
        if not state.sample:
            bad("sampling needs a BeamState(..., sample=True)")
        if seeds.dtype != torch.int64 or not seeds.is_contiguous() or seeds.numel() != state.batch:
            bad(f"seeds must be a contiguous int64 tensor of {state.batch} elements, got {seeds.dtype} "
                f"{tuple(seeds.shape)}")
    if state.seeds is not None or seeds is not None:
        mode = "stochastic beam search" if state.seeds is not None else "beam sampling"
        if not temperature > 0 or not int(top_k) >= 0 or not 0 < top_p <= 1:
            bad(f"need temperature > 0, top_k >= 0 and 0 < top_p <= 1, got {temperature}, {top_k}, {top_p}")
        from .sampling import check_filter_args

        check_filter_args("beam_step_", min_p, typical_p, epsilon_cutoff, eta_cutoff, top_h)
        if vocab > SAMPLE_MAX_VOCAB:
            bad(f"{mode} needs vocab <= {SAMPLE_MAX_VOCAB}, got {vocab}")
    B, K = state.batch, state.num_beams
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1 or logits.shape[0] != B * K:
        bad(f"logits must be fp32 [{B * K}, ld] with unit column stride, got {logits.dtype} {tuple(logits.shape)}")
    if not 1 <= vocab <= logits.shape[1] or K * vocab >= 1 << 32:
        bad(f"vocab must be in [1, ld = {logits.shape[1]}] with num_beams * vocab < 2^32, got {vocab}")
    if int(min_new) < 0:
        bad(f"min_new must be >= 0, got {min_new}")
    sup, n_sup = _id_list("beam_step_", "suppress_ids", suppress_ids, BEAM_MAX_SUPPRESS)
    stop, n_stop = _id_list("beam_step_", "stop_ids", stop_ids, BEAM_MAX_STOP)
    _same_device("beam_step_", logits.device, state.tensors() + (suppress_ids, stop_ids, seeds))
    filters = [float(v) for v in (min_p, typical_p, epsilon_cutoff, eta_cutoff, top_h)]
    if state.seeds is not None:
        _ck(_lib().adapcc_beam_stochastic_step(
            _ptr(logits), logits.stride(0), int(vocab), B, K, _ptr(state.scores), _ptr(state.keys), _ptr(state.step),
            int(min_new), sup, n_sup, stop, n_stop, state.max_new, _ptr(state.done), _ptr(state.cand),
            _ptr(state.cand_key), _ptr(state.cand_phi), _ptr(state.next_ids), _ptr(state.parent),
            _ptr(state.hist_tok), _ptr(state.hist_back), _ptr(state.fin_score), _ptr(state.fin_phi),
            _ptr(state.fin_n), _ptr(state.fin_src), _ptr(state.fin_count), _ptr(state.kappa), float(temperature),
            int(top_k), float(top_p), _ptr(state.seeds), *filters, _stream()), "beam_stochastic_step")
        return
    if seeds is not None:
        _ck(_lib().adapcc_beam_sample_step(
            _ptr(logits), logits.stride(0), int(vocab), B, K, _ptr(state.scores), _ptr(state.step), int(min_new), sup,
            n_sup, stop, n_stop, _ptr(state.pen), int(state.length_penalty > 0), state.max_new, _ptr(state.done),
            _ptr(state.cand), _ptr(state.cand_c), _ptr(state.next_ids), _ptr(state.parent), _ptr(state.hist_tok),
            _ptr(state.hist_back), _ptr(state.fin_score), _ptr(state.fin_n), _ptr(state.fin_src),
            _ptr(state.fin_count), float(temperature), int(top_k), float(top_p), _ptr(seeds), *filters, _stream()),
            "beam_sample_step")
        return
    _ck(_lib().adapcc_beam_step(
        _ptr(logits), logits.stride(0), int(vocab), B, K, state.groups, _ptr(state.scores), _ptr(state.step),
        int(min_new), sup, n_sup, stop, n_stop, _ptr(state.pen), int(state.length_penalty > 0), state.max_new,
        _ptr(state.done), _ptr(state.group_done), _ptr(state.cand), _ptr(state.next_ids), _ptr(state.parent),
        _ptr(state.hist_tok), _ptr(state.hist_back), _ptr(state.fin_score), _ptr(state.fin_n), _ptr(state.fin_src),
        _ptr(state.fin_count), lam, _stream()), "beam_step")


def kv_reorder_scratch_numel(k_cache: torch.Tensor, max_new: int, *, fp8: bool = False) -> int:
    """bf16 elements of the scratch ``kv_reorder_`` needs for caches shaped like ``k_cache`` [L, R, H, t_max, Dh];
    with ``fp8``, bytes (uint8) for an fp8 cache and its scales."""
    L, R, H, _, Dh = k_cache.shape
    return R * int(max_new) * L * 2 * H * (Dh + 4 if fp8 else Dh)


def kv_reorder_(k_cache: torch.Tensor, v_cache: torch.Tensor, parent: torch.Tensor, prompt_len: torch.Tensor,
                lens: torch.Tensor, max_new: int, scratch: torch.Tensor, *, k_scale: Optional[torch.Tensor] = None,
                v_scale: Optional[torch.Tensor] = None) -> None:
    """In place, for every layer l and row r with ``parent[r] != r``: ``k[l, r, :, pos] = k[l, parent[r], :, pos]`` and
    the same for ``v``, over the generated positions ``pos = prompt_len[r] + t``, ``0 <= t < max_new``, ``pos <
    lens[r]``. The caches are bf16 [L, R, H, t_max, Dh]; ``parent``, ``prompt_len`` and ``lens`` int32 [R]. Every
    source is read into ``scratch`` (bf16, ``kv_reorder_scratch_numel`` elements) before anything is written, so cycles
    and many-to-one maps come out right. The grid follows ``max_new``, not the lengths, so one capture serves every
    step. No host sync.

    With ``k_scale`` / ``v_scale`` (fp32 [L, R, H, t_max]) the caches are fp8 (uint8 bytes, ``ops/kvcache.py``; Dh a
    multiple of 16): the bytes and the scales move, and ``scratch`` is uint8 of ``kv_reorder_scratch_numel(...,
    fp8=True)`` bytes."""
    def bad(msg):
        raise ValueError(f"kv_reorder_: {msg}")

    fp8 = k_scale is not None or v_scale is not None
    dt = torch.uint8 if fp8 else torch.bfloat16
    if k_cache.dtype != dt or v_cache.dtype != dt or scratch.dtype != dt:
        bad(f"k_cache, v_cache and scratch must be {'uint8 with scales' if fp8 else 'bf16'}, got {k_cache.dtype}, "
            f"{v_cache.dtype}, {scratch.dtype}")
    if (k_cache.dim() != 5 or not k_cache.is_contiguous() or v_cache.shape != k_cache.shape
            or not v_cache.is_contiguous()):
        bad(f"k_cache / v_cache must be contiguous [L, R, H, t_max, Dh] of one shape, got {tuple(k_cache.shape)} and "
            f"{tuple(v_cache.shape)}")
    L, R, H, t_max, Dh = k_cache.shape
    if Dh % 8 != 0 or R > 65535 or int(max_new) < 1:
        bad(f"need Dh a multiple of 8, R <= 65535 and max_new >= 1, got Dh={Dh} R={R} max_new={max_new}")
    for name, t in (("parent", parent), ("prompt_len", prompt_len), ("lens", lens)):
        if t.dtype != torch.int32 or not t.is_contiguous() or t.numel() != R:
            bad(f"{name} must be a contiguous int32 tensor of {R} elements, got {t.dtype} {tuple(t.shape)}")
    if fp8:
        if Dh % 16 != 0:
            bad(f"an fp8 cache needs Dh a multiple of 16, got {Dh}")
        for name, t in (("k_scale", k_scale), ("v_scale", v_scale)):
            if t is None or t.dtype != torch.float32 or not t.is_contiguous() or t.shape != (L, R, H, t_max):
                bad(f"{name} must be a contiguous fp32 [{L}, {R}, {H}, {t_max}] tensor, got "
                    f"{None if t is None else (t.dtype, tuple(t.shape))}")
    need = kv_reorder_scratch_numel(k_cache, max_new, fp8=fp8)
    if not scratch.is_contiguous() or scratch.numel() < need:
        bad(f"scratch must be contiguous with at least {need} elements, got {scratch.numel()}")
    _same_device("kv_reorder_", k_cache.device, (v_cache, parent, prompt_len, lens, scratch, k_scale, v_scale))
    _ck(_lib().adapcc_kv_reorder(_ptr(k_cache), _ptr(v_cache), L, R, H, t_max, Dh, _ptr(parent), _ptr(prompt_len),
                                 _ptr(lens), int(max_new), _ptr(scratch), _ptr(k_scale), _ptr(v_scale), _stream()),
        "kv_reorder")


# ---- sequence bias, repetition / frequency / presence penalties, n-gram blocking (csrc/ops_repeats.cu) -------------
REPEATS_MAX_GROUP = 16         # rows per parent group (beams per item)
REPEATS_MAX_LEN = 1024         # sequence positions per row (GPT-2's n_positions)


def penalize_repeats_(logits: torch.Tensor, vocab: int, seq: torch.Tensor, prompt_len: torch.Tensor,
                      lens: torch.Tensor, step: torch.Tensor, ids: torch.Tensor, parent: Optional[torch.Tensor],
                      group: int, penalty: float, ngram: int, bias=None, frequency: float = 0.0,
                      presence: float = 0.0, context_ngram: int = 0) -> None:
    """The sequence bias, repetition penalty, frequency / presence penalties, no-repeat n-gram blocking and context
    n-gram blocking of every row, in place, on the device (the definition in ``ops/repeats.py``, which this kernel
    equals bit for bit). ``logits`` fp32 [R, ld] (the first ``vocab`` columns used); ``seq`` int32 [R, t_max] the rows'
    sequences, kept up to date here; ``prompt_len`` and ``lens`` int32 [R]; ``step`` int32 [1] (the counter of
    ``generate`` / ``BeamState``); ``ids`` int64 [R] the tokens the decode step just consumed; ``parent`` int32 [R] or
    None, each row's parent inside its group of ``group`` consecutive rows.

    With ``*step > 0`` the sequences first advance: a row with a parent takes the parent's generated region
    ``seq[parent[r], prompt_len[r]:lens[r] - 1]`` (cycles and many-to-one maps come out right), then
    ``seq[r, lens[r] - 1] = ids[r]``. With ``*step == 0`` the sequence is the prompt as stored. Row r's sequence is then
    ``seq[r, :lens[r]]``; ``bias`` (an ``ops.repeats.SequenceBias`` from ``check_sequence_bias_args``, None: off),
    ``penalty`` (1: off), ``frequency`` and ``presence`` (finite, rounded to fp32; 0: off), ``ngram`` (0: off) and
    ``context_ngram`` (0: off) are applied to it. ``frequency`` and ``presence`` count the generated region
    ``seq[r, prompt_len[r]:lens[r]]``; ``context_ngram`` bans only n-grams inside ``seq[r, :prompt_len[r]]``. The
    table goes to the device once per table and device and keeps its pointers, so a graph may capture it. The grid
    depends on R and ``group`` only and there is no host sync, so one capture serves every token."""
    from .repeats import SequenceBias, finite_fp32

    def bad(msg):
        raise ValueError(f"penalize_repeats_: {msg}")

    if not (math.isfinite(penalty) and penalty > 0) or int(ngram) < 0:
        bad(f"need a finite penalty > 0 and ngram >= 0, got {penalty}, {ngram}")
    for name, x in (("frequency", frequency), ("presence", presence)):
        if not finite_fp32(x):
            bad(f"{name} must be a number that is finite in fp32, got {x}")
    if isinstance(context_ngram, bool) or int(context_ngram) != context_ngram or int(context_ngram) < 0:
        bad(f"context_ngram must be an integer >= 0, got {context_ngram}")
    if bias is not None and not isinstance(bias, SequenceBias):
        bad(f"bias must be an ops.repeats.SequenceBias or None, got {type(bias).__name__}")
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1:
        bad(f"logits must be fp32 [R, ld] with unit column stride, got {logits.dtype} {tuple(logits.shape)}")
    R = logits.shape[0]
    if not 1 <= vocab <= logits.shape[1]:
        bad(f"vocab must be in [1, ld = {logits.shape[1]}], got {vocab}")
    if not 1 <= int(group) <= REPEATS_MAX_GROUP or R % int(group) != 0:
        bad(f"group must be in [1, {REPEATS_MAX_GROUP}] and divide R = {R}, got {group}")
    if (seq.dtype != torch.int32 or seq.dim() != 2 or seq.shape[0] != R or not seq.is_contiguous()
            or not 1 <= seq.shape[1] <= REPEATS_MAX_LEN):
        bad(f"seq must be a contiguous int32 [{R}, t_max] tensor with t_max <= {REPEATS_MAX_LEN}, got {seq.dtype} "
            f"{tuple(seq.shape)}")
    for name, t, dt, n in (("prompt_len", prompt_len, torch.int32, R), ("lens", lens, torch.int32, R),
                           ("step", step, torch.int32, 1), ("ids", ids, torch.int64, R),
                           ("parent", parent, torch.int32, R)):
        if t is not None and (t.dtype != dt or not t.is_contiguous() or t.numel() != n):
            bad(f"{name} must be a contiguous {dt} tensor of {n} elements, got {t.dtype} {tuple(t.shape)}")
    if bias is not None and bias.max_id >= vocab:
        bad(f"the bias table holds id {bias.max_id}, outside [0, vocab = {vocab})")
    _same_device("penalize_repeats_", logits.device, (seq, prompt_len, lens, step, ids, parent))
    tab, val = bias.device_tensors(logits.device) if bias is not None else (None, None)
    _ck(_lib().adapcc_penalize_repeats(_ptr(logits), logits.stride(0), int(vocab), R, _ptr(seq), seq.shape[1],
                                       _ptr(prompt_len), _ptr(lens), _ptr(step), _ptr(ids), _ptr(parent), int(group),
                                       float(penalty), int(ngram), _ptr(tab), _ptr(val),
                                       bias.num_targets if bias is not None else 0,
                                       bias.num_entries if bias is not None else 0, float(frequency), float(presence),
                                       int(context_ngram), _stream()), "penalize_repeats")


# ---- classifier-free guidance (csrc/ops_guidance.cu) ---------------------------------------------------------------
def guidance_mix_(logits: torch.Tensor, vocab: int, B: int, scale: float) -> torch.Tensor:
    """Classifier-free guidance in place, on the device (the definition in ``ops/guidance.py``, which computes the same
    in fp64): ``logits`` fp32 [2B, ld] hold the prompts' rows, then the negative prompts' rows. Row b's first ``vocab``
    columns become ``scale * (lc - lu) + lu``, ``lc`` / ``lu`` the log-softmaxes of rows b and B + b; the other
    columns and rows [B, 2B) are not written. fp32 sums in an order fixed by the thread layout, so a row's bits depend
    on its two input rows, ``vocab`` and ``scale`` only. No host sync."""
    def bad(msg):
        raise ValueError(f"guidance_mix_: {msg}")

    from .guidance import FP32_MAX

    if not (math.isfinite(scale) and abs(scale) <= FP32_MAX):
        bad(f"need a finite fp32 scale, got {scale}")
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1:
        bad(f"logits must be fp32 [2B, ld] with unit column stride, got {logits.dtype} {tuple(logits.shape)} stride "
            f"{logits.stride()}")
    if int(B) < 1 or logits.shape[0] != 2 * int(B):
        bad(f"logits must have 2B rows for B >= 1, got {logits.shape[0]} rows and B = {B}")
    if not 1 <= vocab <= logits.shape[1]:
        bad(f"vocab must be in [1, ld = {logits.shape[1]}], got {vocab}")
    _same_device("guidance_mix_", logits.device, ())
    _ck(_lib().adapcc_guidance_mix(_ptr(logits), logits.stride(0), int(vocab), int(B), float(scale), _stream()),
        "guidance_mix")
    return logits


# ---- contrastive search: candidate attention, selection, re-rank and commit (csrc/ops_contrastive.cu) ---------------
CONTRASTIVE_MAX_K = 16         # candidates per row
CONTRASTIVE_MAX_D = 1024       # hidden size the re-rank kernels hold per lane
CONTRASTIVE_MAX_IDS = 1024     # ids per suppress / stop list


def cand_attention_(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, lens: torch.Tensor, top_k: int,
                    out: torch.Tensor, side_k: torch.Tensor, side_v: torch.Tensor, work: torch.Tensor) -> torch.Tensor:
    """Decode attention of ``top_k`` candidate tokens per cache row. ``qkv`` bf16 [B·k, 3·H·Dh] (q | k | v of candidate
    j of row b in row ``b·k + j``; unit column stride), ``k_cache`` / ``v_cache`` bf16 [B, H, t_max, Dh], ``lens``
    int32 [B]. Candidate (b, j) attends over the row's cached positions ``0..lens[b]-1`` and its own new key and value at
    ``lens[b]``: ``out[b·k + j]`` (bf16 [B·k, H·Dh]) is bit-identical to ``decode_attention_`` on a row that holds that
    token. The cache is only read (each cached element once per CTA for all k queries); the new keys and values go to
    ``side_k`` / ``side_v`` (bf16 [B·k, H·Dh]). ``work``: fp32, ``decode_attention_work_numel(B·k, ...)`` elements.
    The grid depends on t_max, B and k only; no host sync."""
    K = int(top_k)
    if not 1 <= K <= CONTRASTIVE_MAX_K:
        raise ValueError(f"cand_attention_: top_k must be in [1, {CONTRASTIVE_MAX_K}], got {top_k}")
    B, H, t_max, Dh = _check_decode_attn("cand_attention_", K, qkv, k_cache, v_cache, lens, out, work, side_k=side_k,
                                         side_v=side_v)
    _ck(_lib().adapcc_cand_attn(_ptr(qkv), _ptr(k_cache), _ptr(v_cache), _ptr(lens), _ptr(out), _ptr(side_k),
                                _ptr(side_v), B, K, H, Dh, t_max, qkv.stride(0), _ptr(work), _stream()), "cand_attn")
    return out


class ContrastiveState:
    """Device state of a batched contrastive search of ``batch`` rows with ``top_k`` candidates each, up to ``max_new``
    tokens and a cache of ``t_max`` positions (``n_layer`` layers, ``n_head`` heads of ``head_dim``), as
    ``contrastive_select_`` and ``contrastive_rerank_`` read and write it. Candidate j of row b is row ``b·k + j``.

    ``step`` int32 [1] (tokens emitted); ``done`` int32 [B]; ``next_ids`` int64 [B·k] the candidates' ids (the candidate
    step's input; 0 in an invalid slot), ``cand_tok`` int32 [B·k] the same with -1 in an invalid slot, ``cand_p`` fp32
    [B·k] their probabilities; ``tokens`` int64 [B, max_new] the output (-1 after a stop); ``win_ids`` int64 [B] and
    ``win_h`` bf16 [B, D] each row's emitted candidate and its hidden state; ``ctx`` bf16 [B, t_max, D] and
    ``ctx_norm`` fp32 [B, t_max] the rows' context; ``side`` bf16 [n_layer, 2, B·k, D] the candidates' new keys and
    values; ``sim`` fp32 the re-rank scratch; ``work`` fp32 the candidate attention's split partials."""

    def __init__(self, batch: int, top_k: int, max_new: int, t_max: int, n_layer: int, n_head: int, head_dim: int,
                 device):
        B, K, n = int(batch), int(top_k), int(max_new)
        D = n_head * head_dim
        if B < 1 or not 1 <= K <= CONTRASTIVE_MAX_K or n < 1 or not 1 <= t_max or D > CONTRASTIVE_MAX_D:
            raise ValueError(f"ContrastiveState: need batch >= 1, 1 <= top_k <= {CONTRASTIVE_MAX_K}, max_new >= 1, "
                             f"t_max >= 1 and a hidden size <= {CONTRASTIVE_MAX_D}, got {batch}, {top_k}, {max_new}, "
                             f"{t_max}, {D}")
        self.batch, self.top_k, self.max_new, self.t_max = B, K, n, int(t_max)
        self.n_layer, self.n_head, self.head_dim = int(n_layer), int(n_head), int(head_dim)
        i32, dev = dict(dtype=torch.int32, device=device), device
        bf = dict(dtype=torch.bfloat16, device=dev)
        self.step = torch.zeros(1, **i32)
        self.done = torch.zeros(B, **i32)
        self.next_ids = torch.zeros(B * K, dtype=torch.int64, device=dev)
        self.cand_tok = torch.full((B * K,), -1, **i32)
        self.cand_p = torch.zeros(B * K, dtype=torch.float32, device=dev)
        self.tokens = torch.full((B, n), -1, dtype=torch.int64, device=dev)
        self.win_ids = torch.zeros(B, dtype=torch.int64, device=dev)
        self.win_h = torch.zeros(B, D, **bf)
        self.ctx = torch.zeros(B, self.t_max, D, **bf)
        self.ctx_norm = torch.zeros(B, self.t_max, dtype=torch.float32, device=dev)
        self.side = torch.zeros(self.n_layer, 2, B * K, D, **bf)
        self.sim = torch.empty(int(_lib().adapcc_cs_sim_numel(B, K, self.t_max)), dtype=torch.float32, device=dev)
        self.work = torch.empty(decode_attention_work_numel(B * K, n_head, head_dim, self.t_max), dtype=torch.float32,
                                device=dev)

    def tensors(self):
        """Every device tensor of the state (what the ops check for one device)."""
        return (self.step, self.done, self.next_ids, self.cand_tok, self.cand_p, self.tokens, self.win_ids, self.win_h,
                self.ctx, self.ctx_norm, self.side, self.sim, self.work)


def contrastive_select_(logits: torch.Tensor, vocab: int, state: ContrastiveState, min_new: int = 0,
                        suppress_ids: Optional[torch.Tensor] = None) -> None:
    """The candidates of every row, on the device (the definition in ``ops/contrastive.py``): the ``top_k`` ids with
    the largest logits of ``logits`` fp32 [B, ld] (the first ``vocab`` columns; ties to the lower id, -inf never),
    each with ``p = exp(l - m) / Z`` over the remaining ids; ``suppress_ids`` (int32 list or None) are removed while
    ``state.step < min_new``. A row that is done gets none. Writes ``state.next_ids``, ``cand_tok`` and ``cand_p``.
    No host sync."""
    def bad(msg):
        raise ValueError(f"contrastive_select_: {msg}")

    if not isinstance(state, ContrastiveState):
        bad(f"state must be a ContrastiveState, got {type(state).__name__}")
    B, K = state.batch, state.top_k
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1 or logits.shape[0] != B:
        bad(f"logits must be fp32 [{B}, ld] with unit column stride, got {logits.dtype} {tuple(logits.shape)}")
    if not 1 <= vocab <= logits.shape[1]:
        bad(f"vocab must be in [1, ld = {logits.shape[1]}], got {vocab}")
    if int(min_new) < 0:
        bad(f"min_new must be >= 0, got {min_new}")
    sup, n_sup = _id_list("contrastive_select_", "suppress_ids", suppress_ids, CONTRASTIVE_MAX_IDS)
    _same_device("contrastive_select_", logits.device, state.tensors() + (suppress_ids,))
    _ck(_lib().adapcc_cs_select(_ptr(logits), logits.stride(0), int(vocab), B, K, _ptr(state.step), int(min_new), sup,
                                n_sup, _ptr(state.done), _ptr(state.next_ids), _ptr(state.cand_tok), _ptr(state.cand_p),
                                _stream()), "cs_select")


def contrastive_rerank_(hc: torch.Tensor, state: ContrastiveState, alpha: float, k_cache: torch.Tensor,
                        v_cache: torch.Tensor, lens: torch.Tensor, stop_ids: Optional[torch.Tensor] = None) -> None:
    """Re-rank every row's candidates and commit the winner, on the device (the definition in ``ops/contrastive.py``).
    ``hc`` bf16 [B·k, D] (unit column stride) are the candidates' final hidden states; candidate j scores
    ``(1 - alpha) p_j - alpha max_c cos(h_j, c)`` over the row's context ``state.ctx[b, :lens[b]]`` (a zero norm gives
    cosine 0) and the best wins, ties to the lower rank; a row without a candidate emits id 0. Writes column
    ``state.step`` of ``state.tokens`` (-1 for a stop id, which also sets ``done``, or a row already done),
    ``state.win_ids`` and ``state.win_h``; appends the winner's hidden state and norm to the context at ``lens[b]``;
    copies its keys and values from ``state.side`` into ``k_cache`` / ``v_cache`` (bf16 [n_layer, B, H, t_max, Dh]) at
    ``lens[b]``; then advances ``lens`` (int32 [B]) and ``state.step``. No host sync."""
    def bad(msg):
        raise ValueError(f"contrastive_rerank_: {msg}")

    if not isinstance(state, ContrastiveState):
        bad(f"state must be a ContrastiveState, got {type(state).__name__}")
    if not 0.0 <= float(alpha) <= 1.0:
        bad(f"alpha must be in [0, 1], got {alpha}")
    B, K, t_max = state.batch, state.top_k, state.t_max
    Lyr, H, Dh = state.n_layer, state.n_head, state.head_dim
    D = H * Dh
    if hc.dtype != torch.bfloat16 or hc.dim() != 2 or hc.shape != (B * K, D) or hc.stride(1) != 1 or hc.stride(0) % 8:
        bad(f"hc must be bf16 [{B * K}, {D}] with unit column stride and a row stride that is a multiple of 8, got "
            f"{hc.dtype} {tuple(hc.shape)} stride {hc.stride()}")
    for name, t in (("k_cache", k_cache), ("v_cache", v_cache)):
        if t.dtype != torch.bfloat16 or t.shape != (Lyr, B, H, t_max, Dh) or not t.is_contiguous():
            bad(f"{name} must be a contiguous bf16 [{Lyr}, {B}, {H}, {t_max}, {Dh}] tensor, got {t.dtype} "
                f"{tuple(t.shape)}")
    if lens.dtype != torch.int32 or not lens.is_contiguous() or lens.numel() != B:
        bad(f"lens must be a contiguous int32 tensor of {B} elements, got {lens.dtype} {tuple(lens.shape)}")
    stop, n_stop = _id_list("contrastive_rerank_", "stop_ids", stop_ids, CONTRASTIVE_MAX_IDS)
    _same_device("contrastive_rerank_", hc.device, state.tensors() + (k_cache, v_cache, lens, stop_ids))
    _ck(_lib().adapcc_cs_rerank(_ptr(hc), hc.stride(0), B, K, D, _ptr(state.cand_tok), _ptr(state.cand_p),
                                float(alpha), _ptr(state.ctx), _ptr(state.ctx_norm), t_max, _ptr(state.sim),
                                _ptr(lens), _ptr(state.done), stop, n_stop, _ptr(state.step), _ptr(state.tokens),
                                state.max_new, _ptr(state.win_ids), _ptr(state.win_h), _ptr(state.side),
                                _ptr(k_cache), _ptr(v_cache), Lyr, H, Dh, _stream()), "cs_rerank")


def contrastive_context_init_(h: torch.Tensor, lens: torch.Tensor, state: ContrastiveState) -> None:
    """The rows' context from a prefill: ``state.ctx[b, p] = h[b, p]`` and its fp32 norm for ``p < lens[b]``, ``h`` the
    contiguous bf16 [B, T, D] final hidden states, ``lens`` int32 [B] the prompt lengths. No host sync."""
    def bad(msg):
        raise ValueError(f"contrastive_context_init_: {msg}")

    if not isinstance(state, ContrastiveState):
        bad(f"state must be a ContrastiveState, got {type(state).__name__}")
    B, D = state.batch, state.n_head * state.head_dim
    if h.dtype != torch.bfloat16 or h.dim() != 3 or h.shape[0] != B or h.shape[2] != D or not h.is_contiguous():
        bad(f"h must be a contiguous bf16 [{B}, T, {D}] tensor, got {h.dtype} {tuple(h.shape)}")
    if not 1 <= h.shape[1] <= state.t_max:
        bad(f"h holds {h.shape[1]} positions, the context at most {state.t_max}")
    if lens.dtype != torch.int32 or not lens.is_contiguous() or lens.numel() != B:
        bad(f"lens must be a contiguous int32 tensor of {B} elements, got {lens.dtype} {tuple(lens.shape)}")
    _same_device("contrastive_context_init_", h.device, [lens, state.ctx, state.ctx_norm])
    _ck(_lib().adapcc_cs_context_init(_ptr(h), B, h.shape[1], D, _ptr(lens), _ptr(state.ctx), _ptr(state.ctx_norm),
                                      state.t_max, _stream()), "cs_context_init")


# ---- speculative decoding: verify attention, arg-max, acceptance, prompt-lookup drafts (csrc/ops_lookup.cu) --------
LOOKUP_MAX_TOKENS = 15         # drafts per row: k + 1 <= 16 slots, each CTA of the verify attention runs them in turn
LOOKUP_MAX_NGRAM = 16          # max_matching_ngram_size
LOOKUP_MAX_IDS = 1024          # ids per suppress / stop list


def verify_attention_(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, lens: torch.Tensor,
                      nq: torch.Tensor, k: int, out: torch.Tensor, work: torch.Tensor) -> torch.Tensor:
    """Decode attention of ``k + 1`` slots per cache row. ``qkv`` bf16 [B·(k+1), 3·H·Dh] (q | k | v of slot j of row b
    in row ``b·(k+1) + j``; unit column stride), ``k_cache`` / ``v_cache`` bf16 [B, H, t_max, Dh], ``lens`` and ``nq``
    int32 [B] (read only). Row b's first ``nq[b]`` slots are real (at most k + 1 and the positions left in the cache);
    slot j sits at position ``lens[b] + j`` and attends over the cached keys ``0..lens[b]-1`` plus the new keys of the
    row's slots ``0..j``, read from ``qkv``. ``out[b·(k+1) + j]`` (bf16 [B·(k+1), H·Dh]) is bit-identical to
    ``decode_attention_`` with ``lens = lens[b] + j`` on a cache that already holds slots ``0..j-1``; a pad slot's
    output is zero. The real slots' keys and values are stored at ``lens[b] + j``; nothing else is written, and each
    cached element is read once per CTA for all of a row's slots. ``work``: fp32, ``decode_attention_work_numel(B·(k+1),
    ...)`` elements. The grid depends on t_max, B and k only; no host sync."""
    if not 0 <= int(k) <= LOOKUP_MAX_TOKENS:
        raise ValueError(f"verify_attention_: k must be in [0, {LOOKUP_MAX_TOKENS}], got {k}")
    S = int(k) + 1
    B, H, t_max, Dh = _check_decode_attn("verify_attention_", S, qkv, k_cache, v_cache, lens, out, work, nq=nq)
    _ck(_lib().adapcc_verify_attn(_ptr(qkv), _ptr(k_cache), _ptr(v_cache), _ptr(lens), _ptr(nq), _ptr(out), B, S, H,
                                  Dh, t_max, qkv.stride(0), _ptr(work), _stream()), "verify_attn")
    return out


class LookupState:
    """Device state of a batched prompt-lookup generation of ``batch`` rows with up to ``k`` drafts each, up to
    ``max_new`` tokens, a cache of ``t_max`` positions and n-grams of up to ``ngram`` tokens, as ``lookup_argmax_``,
    ``lookup_accept_`` and ``lookup_draft_`` read and write it. Slot j of row b is row ``b·(k+1) + j``.

    ``ids`` int64 [B·(k+1)] the verify step's input (slot 0 the row's last token, then its drafts, 0 in a pad slot),
    ``pos`` int64 [B·(k+1)] their positions, ``nq`` int32 [B] the real slots (1 at the start: the prefill's logits);
    ``seq`` int32 [B, t_max] each row's sequence (the caller stores the prompts); ``emitted`` int32 [B] the tokens
    emitted (a stop id included); ``done`` int32 [B]; ``tokens`` int64 [B, max_new] the output (-1 where nothing was
    emitted); ``steps`` int32 [B] verify steps per live row; ``g`` int32 [B·(k+1)] each real slot's token."""

    def __init__(self, batch: int, k: int, max_new: int, t_max: int, ngram: int, device):
        B, K, n = int(batch), int(k), int(max_new)
        if (B < 1 or not 1 <= K <= LOOKUP_MAX_TOKENS or n < 1 or int(t_max) < 1
                or not 1 <= int(ngram) <= LOOKUP_MAX_NGRAM):
            raise ValueError(f"LookupState: need batch >= 1, 1 <= k <= {LOOKUP_MAX_TOKENS}, max_new >= 1, t_max >= 1 "
                             f"and 1 <= ngram <= {LOOKUP_MAX_NGRAM}, got {batch}, {k}, {max_new}, {t_max}, {ngram}")
        self.batch, self.k, self.max_new, self.t_max, self.ngram = B, K, n, int(t_max), int(ngram)
        S = K + 1
        i32, i64 = dict(dtype=torch.int32, device=device), dict(dtype=torch.int64, device=device)
        self.ids = torch.zeros(B * S, **i64)
        self.pos = torch.zeros(B * S, **i64)
        self.nq = torch.ones(B, **i32)
        self.seq = torch.zeros(B, self.t_max, **i32)
        self.emitted = torch.zeros(B, **i32)
        self.done = torch.zeros(B, **i32)
        self.tokens = torch.full((B, n), -1, **i64)
        self.steps = torch.zeros(B, **i32)
        self.g = torch.zeros(B * S, **i32)

    def tensors(self):
        """Every device tensor of the state (what the ops check for one device)."""
        return (self.ids, self.pos, self.nq, self.seq, self.emitted, self.done, self.tokens, self.steps, self.g)


def lookup_argmax_(logits: torch.Tensor, vocab: int, state: LookupState, min_new: int = 0,
                   suppress_ids: Optional[torch.Tensor] = None) -> None:
    """Greedy verification of every row, on the device (step 2 of ``ops/lookup.py``). ``logits`` fp32 [B·ls, ld] (the
    first ``vocab`` columns used) holds ``ls`` slots per row: k + 1 after a verify step, 1 for the prefill's logits
    (with ``state.nq`` all 1). Each real slot's arg-max (ties to the lower id; ``suppress_ids`` removed while ``emitted
    + j < min_new``) goes to ``state.g[b·(k+1) + j]``, for ``lookup_accept_``. No host sync."""
    def bad(msg):
        raise ValueError(f"lookup_argmax_: {msg}")

    if not isinstance(state, LookupState):
        bad(f"state must be a LookupState, got {type(state).__name__}")
    B, S = state.batch, state.k + 1
    if (logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1
            or logits.shape[0] not in (B, B * S)):
        bad(f"logits must be fp32 [{B}, ld] or [{B * S}, ld] with unit column stride, got {logits.dtype} "
            f"{tuple(logits.shape)}")
    if not 1 <= vocab <= logits.shape[1]:
        bad(f"vocab must be in [1, ld = {logits.shape[1]}], got {vocab}")
    if int(min_new) < 0:
        bad(f"min_new must be >= 0, got {min_new}")
    sup, n_sup = _id_list("lookup_argmax_", "suppress_ids", suppress_ids, LOOKUP_MAX_IDS)
    _same_device("lookup_argmax_", logits.device, state.tensors() + (suppress_ids,))
    _ck(_lib().adapcc_lookup_argmax(_ptr(logits), logits.stride(0), int(vocab), B, S, logits.shape[0] // B,
                                    int(min_new), sup, n_sup, _ptr(state.g), _ptr(state.nq), _ptr(state.emitted),
                                    _ptr(state.done), _stream()), "lookup_argmax")


def lookup_accept_(state: LookupState, lens: torch.Tensor, stop_ids: Optional[torch.Tensor] = None,
                   count: bool = True, flagged: bool = False) -> None:
    """Acceptance of every row on the tokens ``state.g`` holds (``lookup_argmax_``'s arg-maxes, or the verify draws of
    ``sample_slots_``), on the device (step 3 of ``ops/lookup.py``): slot j's token is emitted while the next slot's
    draft in ``state.ids`` equals it; a stop id (not written) or ``state.max_new`` tokens end the row. ``flagged``
    (rejection sampling, after ``spec_slots_``): the row emits the drafts ``state.acc`` accepts, then ``state.last`` at
    the first slot whose draft is rejected (or the last real slot), with the same stop and length rules. Updates
    ``state.tokens``, ``seq``, ``emitted``, ``done`` and, with ``count``, ``steps``, and advances ``lens`` (int32 [B])
    by the number emitted. No host sync."""
    def bad(msg):
        raise ValueError(f"lookup_accept_: {msg}")

    if not isinstance(state, LookupState):
        bad(f"state must be a LookupState, got {type(state).__name__}")
    B, S = state.batch, state.k + 1
    if lens.dtype != torch.int32 or not lens.is_contiguous() or lens.numel() != B:
        bad(f"lens must be a contiguous int32 tensor of {B} elements, got {lens.dtype} {tuple(lens.shape)}")
    if flagged and getattr(state, "acc", None) is None:
        bad("flagged acceptance needs an AssistState made with a vocab")
    stop, n_stop = _id_list("lookup_accept_", "stop_ids", stop_ids, LOOKUP_MAX_IDS)
    _same_device("lookup_accept_", lens.device, state.tensors() + (stop_ids,))
    _ck(_lib().adapcc_lookup_accept(B, S, stop, n_stop, _ptr(state.last if flagged else state.g), _ptr(state.ids),
                                    _ptr(state.nq), _ptr(state.seq), state.t_max, _ptr(lens), _ptr(state.emitted),
                                    _ptr(state.done), _ptr(state.tokens), state.max_new,
                                    _ptr(state.steps if count else None), _ptr(state.acc if flagged else None),
                                    _stream()), "lookup_accept")


def lookup_draft_(state: LookupState, lens: torch.Tensor) -> None:
    """The next verify step's input for every row, on the device (the definition in ``ops/lookup.py``): a live row's
    drafts are the tokens after the earliest earlier occurrence of its sequence's last m tokens (m from
    ``state.ngram`` down to 1), at most ``min(k, max_new - emitted - 1)``. Writes ``state.ids`` (slot 0 the last token
    ``seq[b, lens[b]]``, then the drafts, 0 in a pad slot), ``state.pos`` (``lens[b] + j`` clamped to ``t_max - 1``)
    and ``state.nq`` (1 + drafts; 0 for a done row). No host sync."""
    def bad(msg):
        raise ValueError(f"lookup_draft_: {msg}")

    if not isinstance(state, LookupState):
        bad(f"state must be a LookupState, got {type(state).__name__}")
    B = state.batch
    if lens.dtype != torch.int32 or not lens.is_contiguous() or lens.numel() != B:
        bad(f"lens must be a contiguous int32 tensor of {B} elements, got {lens.dtype} {tuple(lens.shape)}")
    _same_device("lookup_draft_", lens.device, state.tensors())
    _ck(_lib().adapcc_lookup_draft(_ptr(state.seq), state.t_max, B, state.k + 1, state.ngram, state.max_new,
                                   _ptr(lens), _ptr(state.emitted), _ptr(state.done), _ptr(state.ids), _ptr(state.pos),
                                   _ptr(state.nq), _stream()), "lookup_draft")


# ---- assisted generation: per-slot draws (csrc/ops_sample.cu) and round set-up (ops_lookup.cu) ---------------------
class AssistState(LookupState):
    """A ``LookupState`` for assisted generation, where a draft model proposes the drafts (``ops/assisted.py``), plus
    the draft's input buffers: ``d_in`` int64 [B] the token the draft consumes next and ``d_pos`` int64 [k+1, B] its
    positions at each of its k + 1 steps of a round (``lens[b] + j`` clamped to the model's ``n_positions - 1``).

    ``vocab > 0`` adds the buffers of rejection-sampling verification: ``q`` fp32 [B, k, vocab] and ``zq`` fp32 [B, k]
    the draft's filtered weights at each draft step and their totals (``sample_slots_(..., weights=True)``), and
    ``acc`` int32 [B·(k+1)] the accepted flags and ``last`` int32 [B·(k+1)] the round's last token if it ends at slot
    j (``spec_slots_``). Otherwise they are None."""

    def __init__(self, batch: int, k: int, max_new: int, t_max: int, device, vocab: int = 0):
        super().__init__(batch, k, max_new, t_max, 1, device)
        self.d_in = torch.zeros(self.batch, dtype=torch.int64, device=device)
        self.d_pos = torch.zeros(self.k + 1, self.batch, dtype=torch.int64, device=device)
        self.q = self.zq = self.acc = self.last = None
        if int(vocab) > 0:
            B, K = self.batch, self.k
            self.q = torch.zeros(B, K, int(vocab), dtype=torch.float32, device=device)
            self.zq = torch.zeros(B, K, dtype=torch.float32, device=device)
            self.acc = torch.zeros(B * (K + 1), dtype=torch.int32, device=device)
            self.last = torch.zeros(B * (K + 1), dtype=torch.int32, device=device)

    def tensors(self):
        """Every device tensor of the state, the draft's and rejection sampling's buffers included."""
        return super().tensors() + tuple(t for t in (self.d_in, self.d_pos, self.q, self.zq, self.acc, self.last)
                                         if t is not None)


def sample_slots_(logits: torch.Tensor, vocab: int, temperature: float, top_k: int, top_p: float, seeds: torch.Tensor,
                  state: LookupState, lens: torch.Tensor, slot0: int = 0, min_new: int = 0,
                  suppress_ids: Optional[torch.Tensor] = None, draft: bool = False, min_p: float = 0.0,
                  typical_p: float = 1.0, epsilon_cutoff: float = 0.0, eta_cutoff: float = 0.0,
                  weights: bool = False, top_h: float = 0.0) -> None:
    """The draws of speculative decoding, one CTA per slot, on the device. ``logits`` fp32 [B·kq, ld] (the first
    ``vocab`` columns used) holds ``kq`` slots per row; its slot x of row b is slot ``j = slot0 + x``, drawn as
    ``sample_tokens_`` draws a row (the same bits) with the Philox counter ``lens[b] + j + 1`` (``lens`` int32 [B]) and
    step ``state.emitted[b] + j``; ``seeds`` int64 [B]. A done row (``state.done``) draws nothing.

    Verify draws (``draft=False``): slot j is real iff ``j < state.nq[b]`` and its token goes to ``state.g[b·(k+1) +
    j]``; pad slots are left alone. Draft draws (``draft=True``, an ``AssistState``, one logits row per row): the token
    is draft j + 1, real iff
    ``j + 1 < state.nq[b]``; it goes to ``state.ids[b·(k+1) + j + 1]`` and ``state.d_in[b]`` (0 for a pad draft or a
    done row). With ``weights`` (temperature > 0, an ``AssistState`` made with this ``vocab``), a real draft also
    writes the weights ``exp(x_i - m)`` of the ids its draw kept (0 elsewhere) to ``state.q[b, j]`` and their total Z'
    to ``state.zq[b, j]``; the tokens are the same bits either way. No host sync."""
    def bad(msg):
        raise ValueError(f"sample_slots_: {msg}")

    if not isinstance(state, LookupState) or (draft and not isinstance(state, AssistState)):
        bad(f"state must be a {'AssistState' if draft else 'LookupState'}, got {type(state).__name__}")
    if not temperature >= 0 or not top_k >= 0 or not 0 < top_p <= 1:
        bad(f"need temperature >= 0, top_k >= 0 and 0 < top_p <= 1, got {temperature}, {top_k}, {top_p}")
    from .sampling import check_filter_args

    check_filter_args("sample_slots_", min_p, typical_p, epsilon_cutoff, eta_cutoff, top_h)
    B, S = state.batch, state.k + 1
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1 or logits.shape[0] % B:
        bad(f"logits must be fp32 [{B}·kq, ld] with unit column stride, got {logits.dtype} {tuple(logits.shape)}")
    kq = logits.shape[0] // B
    if draft and kq != 1:
        bad(f"draft draws take one logits row per row (draft j + 1 depends on draft j), got {kq}")
    if not 0 <= int(slot0) or int(slot0) + kq + int(draft) > S:
        bad(f"slots {slot0}..{int(slot0) + kq - 1} do not fit {S} slots per row (draft: {draft})")
    _check_slot_inputs(bad, logits, vocab, seeds, lens, B, min_new)
    if weights and not (draft and temperature > 0 and state.q is not None and state.q.shape[2] == vocab):
        bad(f"weights need a draft draw at temperature > 0 and an AssistState made with vocab = {vocab}")
    sup, n_sup = _id_list("sample_slots_", "suppress_ids", suppress_ids, SAMPLE_MAX_IDS)
    _same_device("sample_slots_", logits.device, state.tensors() + (seeds, lens, suppress_ids))
    _ck(_lib().adapcc_sample_slots(_ptr(logits), logits.stride(0), int(vocab), B, kq, S, int(slot0),
                                   float(temperature), int(top_k), float(top_p), float(min_p), float(typical_p),
                                   float(epsilon_cutoff), float(eta_cutoff), _ptr(seeds), _ptr(lens),
                                   _ptr(state.emitted), _ptr(state.done), _ptr(state.nq), int(min_new), sup, n_sup,
                                   None if draft else _ptr(state.g), _ptr(state.ids) if draft else None,
                                   _ptr(state.d_in) if draft else None, _ptr(state.q if weights else None),
                                   _ptr(state.zq if weights else None), float(top_h), _stream()), "sample_slots")


def _check_slot_inputs(bad, logits: torch.Tensor, vocab: int, seeds: torch.Tensor, lens: torch.Tensor, B: int,
                       min_new: int) -> None:
    """The checks ``sample_slots_`` and ``spec_slots_`` share on their vocabulary, seeds, lengths and ``min_new``."""
    if not 1 <= vocab <= min(logits.shape[1], SAMPLE_MAX_VOCAB):
        bad(f"vocab must be in [1, min(ld = {logits.shape[1]}, {SAMPLE_MAX_VOCAB})], got {vocab}")
    for name, t, dt in (("seeds", seeds, torch.int64), ("lens", lens, torch.int32)):
        if t.dtype != dt or not t.is_contiguous() or t.numel() != B:
            bad(f"{name} must be a contiguous {dt} tensor of {B} elements, got {t.dtype} {tuple(t.shape)}")
    if int(min_new) < 0:
        bad(f"min_new must be >= 0, got {min_new}")


def spec_slots_(logits: torch.Tensor, vocab: int, temperature: float, top_k: int, top_p: float, seeds: torch.Tensor,
                state: AssistState, lens: torch.Tensor, min_new: int = 0, suppress_ids: Optional[torch.Tensor] = None,
                min_p: float = 0.0, typical_p: float = 1.0, epsilon_cutoff: float = 0.0,
                eta_cutoff: float = 0.0, top_h: float = 0.0) -> None:
    """Rejection-sampling verification of a round on the device (``ops/assisted.py``), one CTA per slot. ``logits``
    fp32 [B·(k+1), ld] holds the model's slots; ``state`` is an ``AssistState`` made with this ``vocab``, whose
    ``q`` / ``zq`` hold the round's draft weights (``sample_slots_(..., weights=True)``) and ``ids`` the drafts. For
    every real slot j of a live row it writes ``state.g[b·(k+1) + j]``, the draw ``sample_slots_`` makes (the same
    bits). For a slot with a real draft (``j + 1 < state.nq[b]``) it writes ``state.acc`` (draft j + 1 accepted: ``v
    Q_j(d) < P_j(d)``) and ``state.last`` the residual draw t_j; for the last real slot ``state.last`` is g_j. Then
    ``lookup_accept_(..., flagged=True)`` emits the round. Needs temperature > 0. No host sync."""
    def bad(msg):
        raise ValueError(f"spec_slots_: {msg}")

    if not isinstance(state, AssistState) or state.q is None:
        bad(f"state must be an AssistState made with a vocab, got {type(state).__name__}")
    if not temperature > 0 or not top_k >= 0 or not 0 < top_p <= 1:
        bad(f"need temperature > 0, top_k >= 0 and 0 < top_p <= 1, got {temperature}, {top_k}, {top_p}")
    from .sampling import check_filter_args

    check_filter_args("spec_slots_", min_p, typical_p, epsilon_cutoff, eta_cutoff, top_h)
    B, S = state.batch, state.k + 1
    if (logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1
            or logits.shape[0] != B * S):
        bad(f"logits must be fp32 [{B * S}, ld] with unit column stride, got {logits.dtype} {tuple(logits.shape)}")
    _check_slot_inputs(bad, logits, vocab, seeds, lens, B, min_new)
    if state.q.shape[2] != vocab:
        bad(f"the state's draft weights have {state.q.shape[2]} columns, not vocab = {vocab}")
    sup, n_sup = _id_list("spec_slots_", "suppress_ids", suppress_ids, SAMPLE_MAX_IDS)
    _same_device("spec_slots_", logits.device, state.tensors() + (seeds, lens, suppress_ids))
    _ck(_lib().adapcc_spec_slots(_ptr(logits), logits.stride(0), int(vocab), B, S, float(temperature), int(top_k),
                                 float(top_p), float(min_p), float(typical_p), float(epsilon_cutoff),
                                 float(eta_cutoff), _ptr(seeds), _ptr(lens), _ptr(state.emitted), _ptr(state.done),
                                 _ptr(state.nq), int(min_new), sup, n_sup, _ptr(state.ids), _ptr(state.q),
                                 _ptr(state.zq), _ptr(state.g), _ptr(state.acc), _ptr(state.last), float(top_h),
                                 _stream()),
        "spec_slots")


def assist_round_(state: AssistState, lens: torch.Tensor, d_lens: torch.Tensor, n_pos: int) -> None:
    """The start of a round of assisted generation, from the target's state alone (``ops/assisted.py``): writes
    ``state.ids`` (slot 0 the last token ``seq[b, lens[b]]``, 0 in the draft slots), ``state.pos`` (``lens[b] + j``
    clamped to ``t_max - 1``), ``state.nq`` (``1 + min(k, max_new - emitted - 1)``, 0 for a done row), ``state.d_in``
    (the last token), ``state.d_pos`` and the draft cache's lengths ``d_lens`` (int32 [B], set to ``lens``). No host
    sync."""
    def bad(msg):
        raise ValueError(f"assist_round_: {msg}")

    if not isinstance(state, AssistState):
        bad(f"state must be an AssistState, got {type(state).__name__}")
    B = state.batch
    for name, t in (("lens", lens), ("d_lens", d_lens)):
        if t.dtype != torch.int32 or not t.is_contiguous() or t.numel() != B:
            bad(f"{name} must be a contiguous int32 tensor of {B} elements, got {t.dtype} {tuple(t.shape)}")
    if int(n_pos) < 1:
        bad(f"n_pos must be >= 1, got {n_pos}")
    _same_device("assist_round_", lens.device, state.tensors() + (d_lens,))
    _ck(_lib().adapcc_assist_round(_ptr(state.seq), state.t_max, B, state.k + 1, state.max_new, int(n_pos),
                                   _ptr(lens), _ptr(state.emitted), _ptr(state.done), _ptr(state.ids), _ptr(state.pos),
                                   _ptr(state.nq), _ptr(state.d_in), _ptr(d_lens), _ptr(state.d_pos), _stream()),
        "assist_round")
