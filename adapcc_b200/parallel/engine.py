"""Flat-buffer data-parallel training engine (the native fast path next to the DDP hook).

The reference drives gradient communication through torch DDP buckets and a *blocking* hook
(/root/reference/train_ddp.py:35-41, /root/reference/commu.py:385-435). This engine keeps the same
semantics — synchronous data parallelism, bucketed gradient all-reduce overlapped with backward,
mean over the active ranks, clip + AdamW — but lays memory out for the hardware:

* all parameters are views into ONE flat bf16 buffer, all gradients views into ONE flat buffer that
  lives in the communicator's **symmetric heap**, so a bucket's all-reduce is zero-copy: peers read
  and write the gradient bucket directly over NVLink (two-shot) or the switch reduces it in flight
  (NVLS ``multimem.ld_reduce``), with the 1/N scale fused — no staging, no cast kernel, no NCCL;
* buckets are launched from ``post_accumulate_grad`` hooks onto a high-priority side stream as soon
  as their last gradient is produced (overlap with the rest of backward);
* the optimizer is two launches over the flat buffers (grad-norm reduction + fused clip/AdamW with
  fp32 master weights);
* the whole step — forward, backward, the collective kernels on the forked stream, optimizer — is
  captured once into a CUDA graph and replayed, which our kernels allow because their flag epochs
  live in device memory (nothing host-computed is baked into a launch).
"""
from __future__ import annotations

import os
import warnings
from collections.abc import Mapping
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence

import torch
import torch.nn as nn


@dataclass
class _Bucket:
    start: int          # element offsets into the flat buffers
    end: int
    n_params: int
    pending: int = 0


def shard_of(start: int, end: int, rank: int, world: int, elems_per_pack: int) -> tuple:
    """Element range [lo, hi) of ``rank``'s slice of the message [start, end) under the direct kernels' partition
    (csrc/kernels_direct.cuh::Partition): the message is cut into 16-byte packs, ``world`` contiguous slices of
    ceil(packs / world) packs each, slice r owned by rank r (trailing slices may be short or empty)."""
    packs = (end - start + elems_per_pack - 1) // elems_per_pack
    pps = (packs + world - 1) // world
    lo = min(packs, rank * pps) * elems_per_pack
    hi = min(packs, (rank + 1) * pps) * elems_per_pack
    return min(end, start + lo), min(end, start + hi)       # an empty trailing shard is (end, end), never lo > hi


class _GradSink:
    """Handed to the fused ops (ops/layers.py::_sink) through ``param._adapcc_grad_sink``: the op writes
    the parameter's gradient straight into its view of the flat buffer and reports it here."""
    __slots__ = ("engine", "index", "written")

    def __init__(self, engine: "FlatDataParallel", index: int):
        self.engine, self.index, self.written = engine, index, False

    def begin(self) -> bool:
        if self.written:
            raise RuntimeError("a parameter with direct gradient writes produced a second gradient in one step "
                               "(module applied twice / tied weights): build the engine with direct_grads=False")
        self.written = True
        return True

    def done(self) -> None:
        self.engine._grad_ready(self.index)


class FlatDataParallel:
    """Data-parallel training engine on flat buffers (see the module docstring): owns the parameters' and gradients'
    storage, launches bucket collectives from gradient-ready events, runs the (sharded) optimizer, captures the
    whole step in a CUDA graph, and checkpoints per parameter name."""

    def __init__(self, model: nn.Module, comm=None, *, world_size: int = 1, rank: int = 0,
                 bucket_mb: float = 32.0, lr: float = 6.25e-5, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.01, max_norm: float = 1.0, optimizer: str = "adamw",
                 param_dtype: torch.dtype = torch.bfloat16, algo: str = "auto", active: Optional[Sequence[int]] = None,
                 comm_fn: Optional[Callable] = None, direct_grads: Optional[bool] = None,
                 zero1: Optional[bool] = None, dropout_seed: Optional[int] = None,
                 gradient_accumulation_steps: int = 1):
        """``comm``: a :class:`~adapcc_b200.runtime.native.NativeComm` (or None for one GPU).
        ``comm_fn(flat_slice)``: alternative collective (e.g. an NCCL all-reduce) for baselines.
        ``direct_grads``: FusedLinear / FusedLayerNorm backward kernels write their parameter gradients
        straight into the flat buffer (no per-parameter accumulate kernel). Requires every such module to
        be applied once per step; default on (``ADAPCC_DIRECT_GRADS=0`` turns it off).
        ``zero1`` (default: on when eligible, see below): shard the optimizer over the ranks — buckets are
        reduce-SCATTERED during backward, every rank runs AdamW on its 1/N slices only and the updated parameters are
        broadcast by the same kernel through the NVSwitch multicast alias (csrc/zero.cu).
        ``dropout_seed``: ``model.set_dropout(dropout_seed + rank)``, so the ranks draw different masks (a model with
        dropout, see ``GPT2Config``); the captured step needs no new input, the state being on the device. Without it
        the model keeps the seed it has, and at world size > 1 a warning says that the ranks may share their masks.

        ``gradient_accumulation_steps`` M (default 1): one optimizer step runs M micro-batches in order, and ``step`` /
        ``step_graph`` / ``capture`` take a sequence of M batch dicts of equal shapes (a plain dict when M = 1). Each
        micro-batch runs as a step without accumulation does (``flat_grad`` zeroed, forward, backward with the fused ops'
        direct gradient writes; its loss is NOT scaled by 1/M) and leaves its bf16 gradient g_m. An fp32 buffer
        ``grad_acc`` of ``total`` elements, allocated only when M > 1, holds acc_1 = f32(g_1), acc_m = f32(acc_{m-1} +
        f32(g_m)); on the last micro-batch each bucket is folded, ``flat_grad = bf16(f32(f32(acc_{M-1} + f32(g_M)) *
        f32(1/M)))``, every add and multiply rounded on its own. Each bucket's accumulate (micro-batches 1..M-1) or fold
        (micro-batch M) runs on the collective stream as soon as the bucket's gradients are ready, overlapping the rest
        of the backward; after the fold the bucket's collective runs as it does without accumulation, so the gradient is
        sent once per step and not once per micro-batch. Everything after (ZeRO-1, the norm, clipping, AdamW / SGD) sees
        the folded ``flat_grad``. The loss returned is f32(sum_m loss_m) * f32(1/M), the mean of the micro-batch losses
        (HuggingFace's accumulation objective), which differs from the mean over the whole batch when the micro-batches
        score different numbers of labels. Each micro-batch's forward advances the dropout counter (M per step).
        ``steps_done``, ``step_t``, ``set_lr`` and checkpoints count optimizer steps; the accumulator is empty between
        steps, so a checkpoint does not depend on M. M = 1 is the engine without accumulation, launch for launch."""
        if (isinstance(gradient_accumulation_steps, bool) or not isinstance(gradient_accumulation_steps, int)
                or gradient_accumulation_steps < 1):
            raise ValueError(f"gradient_accumulation_steps must be an int >= 1, got {gradient_accumulation_steps!r}")
        self.grad_accum_steps = gradient_accumulation_steps
        self.model, self.comm, self.world_size, self.rank = model, comm, world_size, rank
        self.lr, self.betas, self.eps, self.weight_decay, self.max_norm = lr, betas, eps, weight_decay, max_norm
        self.optimizer, self.algo, self.comm_fn = optimizer, algo, comm_fn
        self.active = list(active) if active is not None else list(range(world_size))
        self.device = next(model.parameters()).device
        if dropout_seed is not None:
            model.set_dropout(int(dropout_seed) + rank)
        elif world_size > 1 and getattr(model, "has_dropout", False):
            warnings.warn("FlatDataParallel: the model has dropout and no dropout_seed was given: every rank keeps the "
                          "model's own seed, so ranks whose seeds are equal draw the same masks")
        params = [p for p in model.parameters() if p.requires_grad]
        self.params = params
        total = sum((p.numel() + 7) // 8 * 8 for p in params)       # every view 16-byte aligned
        self.total = total
        dev = self.device
        # ---- flat parameter / gradient / optimizer state ---------------------------------------
        esize = torch.empty((), dtype=param_dtype).element_size()
        # ZeRO-1 (sharded optimizer fused with its collectives) is the DEFAULT whenever it applies — N > 1, native
        # communicator, AdamW, bf16, all ranks active, heap large enough for parameters + gradients — since its parity
        # run (round 2: bit-identical losses to plain DP over 24 steps, eager and graph) and its measurement (2 GPUs:
        # 8.61 vs 9.06 ms per GPT-2 step). zero1=False / ADAPCC_ZERO1=0 keeps the replicated optimizer; zero1=True insists.
        eligible = bool(comm is not None and world_size > 1 and comm_fn is None and optimizer == "adamw"
                        and param_dtype == torch.bfloat16 and self.active == list(range(world_size))
                        and comm.heap_bytes >= 2 * (total * esize + 4096))
        if zero1 is None:
            self.zero1 = eligible and os.environ.get("ADAPCC_ZERO1", "1") != "0"
        else:
            self.zero1 = bool(zero1) and eligible
            if zero1 and world_size > 1 and not eligible:
                raise ValueError("zero1 needs a native communicator whose symmetric heap holds parameters AND gradients "
                                 f"({2 * total * esize >> 20} MB), bf16 parameters, AdamW and all ranks active")
        if self.zero1:
            self.flat_param = comm.symm_empty(total, param_dtype)   # peers write their updated slices into it
            self.flat_param.zero_()
        else:
            self.flat_param = torch.zeros(total, dtype=param_dtype, device=dev)
        self.zero_copy = False
        # ADAPCC_FORCE_HEAP=1: gradients in the symmetric heap at world size 1 too (diagnostic: isolates the cost of
        # producing gradients into peer-mapped / multicast-bound memory from the cost of the collectives themselves)
        force_heap = os.environ.get("ADAPCC_FORCE_HEAP", "0") == "1"
        if comm is not None and (world_size > 1 or force_heap) and comm.heap_bytes >= total * esize + 4096:
            self.flat_grad = comm.symm_empty(total, param_dtype)
            self.flat_grad.zero_()
            self.zero_copy = True
        else:
            self.flat_grad = torch.zeros(total, dtype=param_dtype, device=dev)
        # micro-batch gradient sums (gradient_accumulation_steps > 1): written before it is read in every step
        self.grad_acc = torch.empty(total, dtype=torch.float32, device=dev) if self.grad_accum_steps > 1 else None
        self._inv_m = torch.full((), 1.0 / self.grad_accum_steps, dtype=torch.float32, device=dev)
        self.master = torch.zeros(total, dtype=torch.float32, device=dev)
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=dev)
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self.step_t = torch.zeros(1, dtype=torch.int32, device=dev)
        self.lr_t = torch.full((1,), float(lr), dtype=torch.float32, device=dev)    # read by the optimizer kernel
        off = 0
        self._offsets: List[int] = []
        with torch.no_grad():
            for p in params:
                n = p.numel()
                self.master[off:off + n].copy_(p.detach().reshape(-1).float())
                view = self.flat_param[off:off + n].view_as(p)
                view.copy_(p.detach())
                p.data = view
                p.grad = self.flat_grad[off:off + n].view_as(p)
                self._offsets.append(off)
                off += (n + 7) // 8 * 8
        # ---- buckets: contiguous ranges, filled from the LAST parameter backwards (gradients are
        # produced roughly in reverse registration order) ------------------------------------------
        cap = max(1, int(bucket_mb * (1 << 20) / esize))
        self.buckets: List[_Bucket] = []
        self._bucket_of: Dict[int, int] = {}
        # Embedding tables (marked by the model) get a bucket of their own: their gradient is final only after the very
        # last op of the backward pass, so everything that shares their bucket would be reduced in the exposed tail too.
        def is_tail(j: int) -> bool:
            return bool(getattr(params[j], "_adapcc_embed_table", False))

        end, members = total, []
        for i in range(len(params) - 1, -1, -1):
            members.append(i)
            start = self._offsets[i]
            boundary = i > 0 and is_tail(i - 1) != is_tail(i)
            if end - start >= cap or i == 0 or boundary:
                if boundary and end - start < cap // 4 and self.buckets and not is_tail(i):
                    last = self.buckets[-1]                 # a small remainder in front of the tail: no bucket of its own
                    last.start, last.n_params = start, last.n_params + len(members)
                    for j in members:
                        self._bucket_of[j] = len(self.buckets) - 1
                else:
                    for j in members:
                        self._bucket_of[j] = len(self.buckets)
                    self.buckets.append(_Bucket(start, end, len(members)))
                end, members = start, []
        # ZeRO-1 slices: the direct kernels cut a message into world slices of ceil(packs / world) 16-byte
        # packs (csrc/kernels_direct.cuh::Partition); rank r owns slice r of every bucket
        self._my_slices: List[tuple] = []
        if self.zero1:
            self._my_slices = [shard_of(b.start, b.end, rank, world_size, 16 // esize) for b in self.buckets]
        self._hooks = [p.register_post_accumulate_grad_hook(self._make_hook(i)) for i, p in enumerate(params)]
        if direct_grads is None:
            direct_grads = os.environ.get("ADAPCC_DIRECT_GRADS", "1") != "0"
        self._sinks: List[_GradSink] = []
        if direct_grads and dev.type == "cuda":
            from ..ops.layers import FusedLayerNorm, FusedLinear
            index = {id(p): i for i, p in enumerate(params)}
            uses: Dict[int, int] = {}
            fused = [m for m in model.modules() if isinstance(m, (FusedLinear, FusedLayerNorm))]
            for m in fused:
                for p in (m.weight, m.bias):
                    if p is not None:
                        uses[id(p)] = uses.get(id(p), 0) + 1
            for m in fused:
                for p in (m.weight, m.bias):
                    if p is not None and id(p) in index and uses[id(p)] == 1 and p.dtype == param_dtype:
                        sink = _GradSink(self, index[id(p)])
                        p._adapcc_grad_sink = sink
                        self._sinks.append(sink)
            # embedding tables (models mark them `_adapcc_embed_table`): the fused embedding backward adds its rows
            # straight into the table's flat-buffer gradient view — which may already hold the tied LM head's dW,
            # written during the forward pass (models/gpt2.py::_ChunkedLMLoss) — and reports it done; it is the
            # last op of the backward pass, so the bucket launches right after it
            for p in params:
                if getattr(p, "_adapcc_embed_table", False) and p.dtype == param_dtype and id(p) not in uses:
                    sink = _GradSink(self, index[id(p)])
                    p._adapcc_grad_sink = sink
                    self._sinks.append(sink)
        self.direct_grads = bool(self._sinks)
        self._debug = os.environ.get("ADAPCC_ENGINE_DEBUG", "0") == "1"
        self._ready: List[bool] = [False] * len(params)
        self._micro = 1                                   # 1-based index of the micro-batch in flight
        self.comm_stream = torch.cuda.Stream(device=dev, priority=-1) if dev.type == "cuda" else None
        self._graph = None
        self._static_batches: List[Dict[str, torch.Tensor]] = []
        self._static_loss = None
        self.steps_done = 0
        self.native_launches_per_step = 0

    # -- gradient hooks ---------------------------------------------------------------------------
    def _grad_ready(self, i: int) -> None:
        """Parameter ``i``'s gradient is final in the flat buffer. Reported by the autograd post-accumulate hook or,
        for parameters whose fused op writes the gradient itself, by the op's sink. BOTH can fire for one parameter: the
        op returns ``None`` for it, and this torch still runs the parameter's AccumulateGrad node (and its hooks) with
        the undefined gradient right after the op's backward. Only the first report of a step counts — counting both
        launched every bucket after HALF of its gradients (found in round 2 with tools/engine_debug_worker.py: gradients
        produced after the early launch were never averaged)."""
        if self._ready[i]:
            return
        self._ready[i] = True
        b = self.buckets[self._bucket_of[i]]
        b.pending -= 1
        if self._debug and b.pending == 0:
            names = {id(p): n for n, p in self.model.named_parameters()}
            print(f"[engine] bucket {self._bucket_of[i]} ({b.n_params} params) launched by "
                  f"{names.get(id(self.params[i]), i)} after {sum(self._ready)} ready reports", flush=True)
        if b.pending == 0:
            self._launch_bucket(b)

    def _make_hook(self, i: int):
        def hook(_p):
            self._grad_ready(i)
        return hook

    def _launch_bucket(self, b: _Bucket) -> None:
        """Bucket ``b``'s gradients of the current micro-batch are final: on the collective stream, add them to the
        accumulator (micro-batches 1..M-1), or fold them into it (micro-batch M) and run the bucket's collective."""
        collective = self.world_size > 1 and (self.comm is not None or self.comm_fn is not None)
        M = self.grad_accum_steps
        if M == 1 and not collective:
            return
        cur = torch.cuda.current_stream(self.device)
        self.comm_stream.wait_stream(cur)
        self._forked = True
        with torch.cuda.stream(self.comm_stream):
            seg = self.flat_grad[b.start:b.end]
            if M > 1:
                from ..ops import grad_accum_, grad_fold_

                acc = self.grad_acc[b.start:b.end]
                if self._micro < M:
                    grad_accum_(seg, acc, first=self._micro == 1)
                    return
                grad_fold_(seg, acc, 1.0 / M)
                if not collective:
                    return
            if self.comm_fn is not None:
                self.comm_fn(seg)
            elif self.zero1:
                # reduce-scatter in place: the direct reduce kernel with root = self leaves the averaged
                # slice `rank` of the bucket in this rank's buffer and moves 1/2 of an all-reduce's bytes
                self.comm.reduce(seg, root=self.rank, op="avg", algo=self.algo, active=self.active)
            else:
                self.comm.all_reduce(seg, op="avg", algo=self.algo, active=self.active)

    # -- one training step -------------------------------------------------------------------------
    def _micro_step(self, batch: Dict[str, torch.Tensor]) -> torch.Tensor:
        """Forward and backward of one micro-batch into the zeroed ``flat_grad``; the buckets' accumulate / fold /
        collective launches happen from the gradient-ready events. Returns the (device) loss."""
        self.flat_grad.zero_()
        self._forked = False
        self._ready = [False] * len(self.params)
        for b in self.buckets:
            b.pending = b.n_params
        for sink in self._sinks:
            sink.written = False
        out = self.model(**batch)
        loss = out[0] if isinstance(out, (tuple, list)) else out
        loss.backward()
        for b in self.buckets:
            if b.pending > 0:                         # parameters that got no gradient this step (unused branch):
                b.pending = 0                         # their zeros still travel, or the bucket's other gradients
                self._launch_bucket(b)                # would stay un-averaged (same parameters on every rank, as in DDP)
        cur = torch.cuda.current_stream(self.device)
        if self._forked:                            # join the collective stream (also under capture); the next
            cur.wait_stream(self.comm_stream)       # micro-batch's zero_() must not overtake this one's accumulates
        return loss.detach()

    def _step_body(self, batches: List[Dict[str, torch.Tensor]]) -> torch.Tensor:
        from ..ops import fused_adamw_, fused_sgd_, incr_, sumsq_

        loss = None
        for m, batch in enumerate(batches, 1):
            self._micro = m
            lm = self._micro_step(batch)
            loss = lm if loss is None else loss + lm                  # fp32, in micro-batch order
        if len(batches) > 1:
            loss = loss.float() * self._inv_m
        incr_(self.step_t)
        if self.zero1:
            self._zero1_update()
        elif self.optimizer == "adamw":
            sumsq = None
            if self.max_norm and self.max_norm > 0:
                self.sumsq.zero_()
                sumsq_(self.flat_grad, self.sumsq)
                sumsq = self.sumsq
            fused_adamw_(self.flat_param, self.flat_grad, self.master, self.exp_avg, self.exp_avg_sq, lr=self.lr,
                         betas=self.betas, eps=self.eps, weight_decay=self.weight_decay, step=self.steps_done + 1,
                         max_norm=self.max_norm or 0.0, sumsq=sumsq, step_tensor=self.step_t, lr_tensor=self.lr_t)
        else:
            fused_sgd_(self.flat_param, self.flat_grad, self.master, lr=self.lr)
        return loss

    def set_lr(self, lr: float) -> None:
        """Change the learning rate (e.g. from a scheduler, once per step). The optimizer kernel reads it from a device
        scalar, so this also takes effect in an already captured CUDA graph."""
        self.lr = float(lr)
        self.lr_t.fill_(self.lr)

    def _zero1_update(self) -> None:
        """Sharded optimizer step: norm of my slices -> 4-byte all-reduce -> AdamW on my slices with the parameter
        broadcast fused into the kernel -> device barrier."""
        from ..ops import sumsq_, zero_adamw_bcast_

        clip = bool(self.max_norm and self.max_norm > 0)
        self.sumsq.zero_()
        if clip:
            for lo, hi in self._my_slices:
                if hi > lo:
                    sumsq_(self.flat_grad[lo:hi], self.sumsq)
        # also when not clipping: this all-reduce is the point after which no rank still reads the old parameters
        self.comm.all_reduce(self.sumsq, op="sum", active=self.active)
        for lo, hi in self._my_slices:
            if hi > lo:
                zero_adamw_bcast_(self.comm, self.flat_param[lo:hi], self.flat_grad[lo:hi], self.master[lo:hi],
                                  self.exp_avg[lo:hi], self.exp_avg_sq[lo:hi], lr=self.lr, betas=self.betas,
                                  eps=self.eps, weight_decay=self.weight_decay, max_norm=self.max_norm or 0.0,
                                  sumsq=self.sumsq if clip else None, step_tensor=self.step_t)
        self.comm.device_barrier(self.active)

    def _micro_batches(self, batches, who: str, like: Optional[List[Dict[str, torch.Tensor]]] = None):
        """``batches`` as a list of the step's M micro-batch dicts; ``ValueError`` unless it is a sequence of M dicts
        (or one dict when M = 1) whose keys and tensor shapes agree with each other and with ``like``'s."""
        M = self.grad_accum_steps
        if isinstance(batches, Mapping):
            if M != 1:
                raise ValueError(f"{who}: gradient_accumulation_steps = {M} takes a sequence of {M} micro-batch dicts, "
                                 "got one dict")
            batches = [batches]
        elif isinstance(batches, (list, tuple)):
            batches = list(batches)
        else:
            raise ValueError(f"{who}: expected a batch dict or a sequence of them, got {type(batches).__name__}")
        if len(batches) != M or not all(isinstance(b, Mapping) for b in batches):
            raise ValueError(f"{who}: gradient_accumulation_steps = {M} takes {M} micro-batch dicts, got "
                             f"{len(batches)} items")

        def shapes(b):
            return {k: tuple(v.shape) if torch.is_tensor(v) else None for k, v in b.items()}

        want = shapes(like[0] if like else batches[0])
        for m, b in enumerate(batches):
            if shapes(b) != want:
                raise ValueError(f"{who}: micro-batch {m} has shapes {shapes(b)}, "
                                 f"{'the captured step' if like else 'micro-batch 0'} has {want}")
        return batches

    def step(self, batch) -> torch.Tensor:
        """Eager optimizer step on device-resident inputs: one batch dict, or a sequence of
        ``gradient_accumulation_steps`` micro-batch dicts. Returns the (device) loss, the mean over the micro-batches."""
        loss = self._step_body(self._micro_batches(batch, "step"))
        self.steps_done += 1
        return loss

    # -- CUDA graph ---------------------------------------------------------------------------------
    def capture(self, example_batch, warmup: int = 2) -> None:
        """Capture one full optimizer step, all its micro-batches in one graph. ``example_batch`` (one batch dict, or the
        sequence of ``gradient_accumulation_steps`` micro-batch dicts ``step`` takes) fixes the shapes; later steps
        copy their inputs into the static buffers, one dict per micro-batch (``step_graph``)."""
        from ..runtime.native import load_library

        self._static_batches = [{k: v.clone() for k, v in b.items()} for b in self._micro_batches(example_batch, "capture")]
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(warmup):                       # allocator + cuBLAS workspaces settle
                self._step_body(self._static_batches)
                self.steps_done += 1
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        lib = load_library()
        c0 = lib.adapcc_launch_count() if hasattr(lib, "adapcc_launch_count") else 0
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            self._static_loss = self._step_body(self._static_batches)
        self.native_launches_per_step = (lib.adapcc_launch_count() - c0) if hasattr(lib, "adapcc_launch_count") else 0

    def step_graph(self, batch) -> torch.Tensor:
        """Copy ``batch`` (pinned host or device tensors; the form ``step`` takes) into the static inputs and
        replay. Every micro-batch dict must have the captured keys and shapes (``ValueError`` otherwise, also at M = 1:
        a key left out would replay the previous step's tensor)."""
        for static, batch in zip(self._static_batches, self._micro_batches(batch, "step_graph", self._static_batches)):
            for k, v in batch.items():
                static[k].copy_(v, non_blocking=True)
        self._graph.replay()
        self.steps_done += 1
        return self._static_loss

    # -- checkpoint / resume -------------------------------------------------------------------------
    def consolidate_optimizer_state(self) -> None:
        """ZeRO-1: every rank owns the fp32 master weights and AdamW moments of ITS slices only. Before a checkpoint
        (or before switching the sharding off) bring all slices to every rank: one broadcast per (bucket, owner) over
        ``torch.distributed`` — a checkpoint-time operation, not on the training path. Collective: call on every rank."""
        if not self.zero1:
            return
        import torch.distributed as dist

        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("consolidate_optimizer_state needs an initialised torch.distributed process group")
        esize = self.flat_param.element_size()
        for b in self.buckets:
            for r in range(self.world_size):
                lo, hi = shard_of(b.start, b.end, r, self.world_size, 16 // esize)
                if hi > lo:
                    for t in (self.master, self.exp_avg, self.exp_avg_sq):
                        dist.broadcast(t[lo:hi], src=r)

    def state_dict(self, consolidate: bool = True) -> Dict[str, object]:
        """Everything needed to resume: fp32 master weights and AdamW moments PER PARAMETER NAME (so a checkpoint
        survives a different bucket size, parameter order or world size), the step counter and the hyper-parameters.
        In ``zero1`` mode the state of slices owned by other ranks is first gathered (``consolidate_optimizer_state``,
        collective: call ``state_dict`` on every rank; ``consolidate=False`` skips it and returns this rank's view)."""
        if consolidate and self.zero1:
            self.consolidate_optimizer_state()
        names = {id(p): n for n, p in self.model.named_parameters()}
        per = {}
        for p, off in zip(self.params, self._offsets):
            n = p.numel()
            per[names[id(p)]] = {"master": self.master[off:off + n].detach().cpu().clone().view(p.shape),
                                 "exp_avg": self.exp_avg[off:off + n].detach().cpu().clone().view(p.shape),
                                 "exp_avg_sq": self.exp_avg_sq[off:off + n].detach().cpu().clone().view(p.shape)}
        sd = {"format": 1, "steps_done": int(self.steps_done), "step_t": int(self.step_t.item()),
              "hyper": {"lr": self.lr, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.weight_decay,
                        "max_norm": self.max_norm, "optimizer": self.optimizer}, "params": per}
        if getattr(self.model, "has_dropout", False):      # the mask sequence: a resumed run continues it. The seed is the
            # base seed (this rank's minus its rank), so that whichever rank writes the file, rank r resumes seed + r
            sd["dropout"] = {"seed": int(self.model.dropout_seed.item()) - self.rank,
                             "step": int(self.model.dropout_step.item())}
        return sd

    def load_state_dict(self, sd: Dict[str, object], strict: bool = True) -> None:
        """In place (buffer addresses — and therefore a captured CUDA graph — stay valid): fp32 state from the
        checkpoint, bf16 parameters re-derived from the master weights."""
        names = {id(p): n for n, p in self.model.named_parameters()}
        per = sd["params"]
        missing = [names[id(p)] for p in self.params if names[id(p)] not in per]
        if missing and strict:
            raise KeyError(f"checkpoint lacks optimizer state for {missing[:5]}{'...' if len(missing) > 5 else ''}")
        with torch.no_grad():
            for p, off in zip(self.params, self._offsets):
                e = per.get(names[id(p)])
                if e is None:
                    continue
                n = p.numel()
                if tuple(e["master"].shape) != tuple(p.shape):
                    raise ValueError(f"{names[id(p)]}: checkpoint shape {tuple(e['master'].shape)} != {tuple(p.shape)}")
                self.master[off:off + n].copy_(e["master"].reshape(-1))
                self.exp_avg[off:off + n].copy_(e["exp_avg"].reshape(-1))
                self.exp_avg_sq[off:off + n].copy_(e["exp_avg_sq"].reshape(-1))
                self.flat_param[off:off + n].copy_(self.master[off:off + n])          # fp32 -> param dtype
        self.steps_done = int(sd.get("steps_done", 0))
        self.step_t.fill_(int(sd.get("step_t", self.steps_done)))
        h = sd.get("hyper", {})
        self.set_lr(h.get("lr", self.lr))
        has = getattr(self.model, "has_dropout", False)
        if "dropout" in sd and has:
            self.model.set_dropout(sd["dropout"]["seed"] + self.rank, sd["dropout"]["step"])
        elif "dropout" in sd:
            warnings.warn("load_state_dict: the checkpoint carries a dropout state and the model has no dropout: ignored")
        elif has:
            warnings.warn("load_state_dict: the checkpoint carries no dropout state: the model keeps its seed and step, "
                          "so the mask sequence does not continue the checkpointed run's")

    def close(self) -> None:
        for h in self._hooks:
            h.remove()
        for sink in self._sinks:
            p = self.params[sink.index]
            if getattr(p, "_adapcc_grad_sink", None) is sink:
                del p._adapcc_grad_sink
        self._sinks = []
        self._graph = None
