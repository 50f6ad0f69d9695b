"""Host → device input pipeline for static-shape batches.

The reference feeds the model with ``batch = tuple(t.to(device) for t in batch)`` from pageable memory inside the
step (/root/reference/models/gpt2/train_gpt2_ddp.py:173-174): a synchronous copy per tensor per step. Here every
batch is staged in a small ring of PINNED host slots,
copied with one async H2D per tensor on a side stream into a ring of preallocated DEVICE slots, and handed to the
training step as views of those fixed device buffers — so a CUDA-graph-captured step can read the same addresses every
replay (``static_out``) and the copy of batch *k+1* overlaps the compute of batch *k*.
"""
from __future__ import annotations

from typing import Dict, Iterable, Iterator, List, Optional

import torch


class PinnedPrefetcher:
    """Iterate over ``loader`` (dicts of equally-shaped CPU tensors), yielding dicts of device tensors.

    ``depth`` device slots rotate; a yielded batch stays valid until ``depth - 1`` further batches were requested.
    ``static_out``: a dict of device tensors (e.g. the example batch a CUDA graph was captured with) that receives
    every batch by a device-side copy on the consumer's stream — the yielded dict is then always ``static_out``."""

    def __init__(self, loader: Iterable[Dict[str, torch.Tensor]], device, depth: int = 2,
                 static_out: Optional[Dict[str, torch.Tensor]] = None):
        self.loader = loader
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        self.depth = max(2, int(depth))
        self.static_out = static_out
        self._host = [None] * self.depth
        self._dev = [None] * self.depth
        self._ready = [None] * self.depth
        self._stream = torch.cuda.Stream(self.device) if self.cuda else None
        self.bytes_per_batch = 0

    def _slots_for(self, batch: Dict[str, torch.Tensor], k: int):
        stale = self._host[k] is not None and any(tuple(self._host[k][n].shape) != tuple(t.shape) or self._host[k][n].dtype != t.dtype
                                                  for n, t in batch.items())
        if stale and self._ready[k] is not None:               # a ragged (last) batch: give the slot buffers of its shape
            self._ready[k].synchronize()
        if self._host[k] is None or stale:
            self._host[k] = {n: (torch.empty_like(t).pin_memory() if self.cuda else torch.empty_like(t))
                             for n, t in batch.items()}
            self._dev[k] = {n: torch.empty_like(t, device=self.device) for n, t in batch.items()}
            self.bytes_per_batch = sum(t.numel() * t.element_size() for t in batch.values())
        return self._host[k], self._dev[k]

    def _stage(self, batch: Dict[str, torch.Tensor], k: int) -> None:
        host, dev = self._slots_for(batch, k)
        if self.cuda:
            if self._ready[k] is not None:
                self._ready[k].synchronize()              # the slot's previous H2D must be done before the host side is reused
            for n, t in batch.items():
                host[n].copy_(t)
            self._stream.wait_stream(torch.cuda.current_stream(self.device))       # consumer done with this device slot
            with torch.cuda.stream(self._stream):
                for n in batch:
                    dev[n].copy_(host[n], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self._stream)
            self._ready[k] = ev
        else:
            for n, t in batch.items():
                dev[n].copy_(t)

    def __iter__(self) -> Iterator[Dict[str, torch.Tensor]]:
        it = iter(self.loader)
        k = 0
        try:
            nxt = next(it)
        except StopIteration:
            return
        self._stage(nxt, k)
        while True:
            cur = k
            try:
                nxt = next(it)
                k = (k + 1) % self.depth
                self._stage(nxt, k)                        # overlaps the consumer's work on `cur`
                more = True
            except StopIteration:
                more = False
            if self.cuda:
                torch.cuda.current_stream(self.device).wait_event(self._ready[cur])
            out = self._dev[cur]
            if self.static_out is not None:
                for n, t in out.items():
                    self.static_out[n].copy_(t, non_blocking=True)
                out = self.static_out
            yield out
            if not more:
                return


def micro_batch_groups(loader: Iterable[Dict[str, torch.Tensor]], device, M: int) -> Iterator[List[Dict[str, torch.Tensor]]]:
    """The loader's batches on ``device`` in groups of ``M`` consecutive ones, in order (an incomplete last group is
    dropped): the micro-batches of one optimizer step under gradient accumulation. The prefetcher ring holds M + 1
    slots, so every batch of a group is still the loader's batch when the group is yielded and until the next group is
    requested (with fewer slots the next batch's upload would already overwrite the first ones of the group)."""
    if int(M) < 1:
        raise ValueError(f"micro_batch_groups: M must be >= 1, got {M}")
    group: List[Dict[str, torch.Tensor]] = []
    for batch in PinnedPrefetcher(loader, device, depth=int(M) + 1):
        group.append(batch)
        if len(group) == M:
            yield group
            group = []
