"""torch DDP integration: the reference's usage (``ddp_model.register_comm_hook(state=None,
hook=AdapCC.communicator.cuda_allreduce_hook)``, /root/reference/train_ddp.py:35-41) plus an
optional zero-copy mode where DDP's gradient buckets are allocated from the communicator's
symmetric heap, so the hook's all-reduce touches them in place over NVLink."""
from __future__ import annotations

import contextlib
import torch


@contextlib.contextmanager
def symmetric_allocations(communicator):
    """Allocations made inside this context (on the communicator's device) come from the symmetric
    heap. ``wrap_ddp`` uses it around the ``DistributedDataParallel(...)`` construction and
    ``rebuild_buckets`` around DDP's one-off bucket rebuild; keep it narrow — everything allocated
    inside (activations included) would land in the heap."""
    native = communicator._ensure_native() if hasattr(communicator, "_ensure_native") else communicator
    if native is None or native.heap_bytes == 0:
        yield None
        return
    pool = native.mem_pool()
    with torch.cuda.use_mem_pool(pool, device=torch.device("cuda", native.device)):
        yield pool


def wrap_ddp(model: torch.nn.Module, communicator, local_rank: int, *, bucket_cap_mb: int = 25,
             zero_copy: bool = True, **ddp_kwargs):
    """DistributedDataParallel + AdapCC comm hook. Returns the DDP module."""
    from torch.nn.parallel import DistributedDataParallel as DDP

    ctx = symmetric_allocations(communicator) if (zero_copy and next(model.parameters()).is_cuda) else contextlib.nullcontext()
    with ctx:
        ddp = DDP(model, device_ids=[local_rank] if next(model.parameters()).is_cuda else None,
                  output_device=local_rank if next(model.parameters()).is_cuda else None,
                  bucket_cap_mb=bucket_cap_mb, gradient_as_bucket_view=True, **ddp_kwargs)
    ddp.register_comm_hook(state=None, hook=communicator.cuda_allreduce_hook)
    return ddp


def rebuild_buckets(ddp, communicator) -> bool:
    """DDP re-buckets its gradients once, after the first backward (order of gradient arrival). Call
    this right after iteration 0 so the NEW buckets are allocated from the symmetric heap too;
    otherwise the rebuild happens inside the next forward with ordinary memory and the hook falls back
    to the staged path. Returns True if a rebuild happened."""
    reducer = getattr(ddp, "reducer", None)
    if reducer is None:
        return False
    with symmetric_allocations(communicator):
        return bool(reducer._rebuild_buckets())


def ddp_accumulate(ddp, micro, **kwargs) -> torch.Tensor:
    """Forward and backward of one optimizer step's micro-batches (dicts of model inputs, ``kwargs`` added to each
    call) through DistributedDataParallel, or a bare module at world size 1, into the parameters' ``.grad``: ``no_sync``
    for all but the last, so the gradients are all-reduced once per step, and each loss (the model output's first
    element) times 1/M, so the gradient is that of the mean of the M micro-batch losses, the objective of
    ``FlatDataParallel(gradient_accumulation_steps=M)``. M = 1 is a plain forward and backward. -> that mean, detached."""
    M = len(micro)
    total = None
    for i, b in enumerate(micro):
        last = i == M - 1 or not hasattr(ddp, "no_sync")
        with contextlib.nullcontext() if last else ddp.no_sync():
            out = ddp(**b, **kwargs)
            loss = out[0] if isinstance(out, (tuple, list)) else out
            (loss * (1.0 / M) if M > 1 else loss).backward()
        total = loss.detach() if total is None else total + loss.detach()
    return total / M if M > 1 else total
