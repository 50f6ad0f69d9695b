"""CPU reference executor: interprets the same tree roles / work items as the sm_90a tree kernel,
over ``torch.distributed`` point-to-point (gloo). It is (a) the oracle GPU tests compare against,
(b) the plumbing path for BASELINE config 1 (world_size=2, strategy/4.xml, no GPU), and (c) the
fallback data plane when a job runs with ``--backend gloo`` (the reference accepts that flag but
its native library is CUDA-only, /root/reference/train_ddp.py:62).
"""
from __future__ import annotations

from typing import Iterable, List, Optional

import torch
import torch.distributed as dist

from ..constants import (ALLREDUCE, BOARDCAST, REDUCE, RELAY_FORWARD, TR_HAS_LOCAL, TR_IN_BCAST, TR_IN_REDUCE,
                         TR_PUBLISH, TR_WANT_RESULT)
from .relay import tree_role
from .schedule import work_items
from .trees import Strategy


def _reduce_into(acc: Optional[torch.Tensor], x: torch.Tensor, op: str) -> torch.Tensor:
    if acc is None:
        return x.clone()
    if op == "max":
        return torch.maximum(acc, x)
    return acc.add_(x)


def tree_collective_cpu(prim: int, tensor: torch.Tensor, strategy: Strategy, rank: int, world: int,
                        active: Optional[Iterable[int]] = None, op: str = "sum",
                        chunk_bytes: int = 4 << 20, relay_mode: int = RELAY_FORWARD,
                        wire_dtype: Optional[torch.dtype] = None, group=None) -> torch.Tensor:
    """In-place tree allreduce / reduce / broadcast of a 1-D contiguous CPU tensor."""
    if prim not in (ALLREDUCE, REDUCE, BOARDCAST):
        raise ValueError(f"primitive {prim} has no tree schedule")
    act = sorted(set(range(world) if active is None else active))
    wire_dtype = wire_dtype or tensor.dtype
    acc_dtype = torch.float32 if tensor.dtype.is_floating_point else tensor.dtype
    flat = tensor.view(-1)
    roles = [tree_role(t, rank, act, prim, relay_mode) for t in strategy.trees]
    n_contrib = len(act)
    scale = 1.0 / n_contrib if (op == "avg" and n_contrib) else 1.0
    tag = 0
    for it in work_items(flat.numel(), len(strategy.trees), chunk_bytes, torch.empty((), dtype=wire_dtype).element_size()):
        role = roles[it.tree]
        tag += 1
        if not role.any():
            continue
        seg = flat[it.start:it.start + it.length]
        is_root = role.parent < 0
        publish: Optional[torch.Tensor] = None
        # ------------------------------- reduce phase ----------------------------------
        if prim != BOARDCAST and role.has(TR_IN_REDUCE):
            bufs = [torch.empty(it.length, dtype=wire_dtype) for _ in role.children]
            reqs = [dist.irecv(b, src=c, group=group, tag=tag) for b, c in zip(bufs, role.children)]
            acc = seg.to(acc_dtype).clone() if role.has(TR_HAS_LOCAL) else None
            for r, b in zip(reqs, bufs):
                r.wait()
                acc = _reduce_into(acc, b.to(acc_dtype), op)
            if acc is None:
                acc = torch.zeros(it.length, dtype=acc_dtype)
            if is_root:
                acc = acc * scale if scale != 1.0 else acc
                if role.has(TR_WANT_RESULT):
                    seg.copy_(acc.to(tensor.dtype))
                publish = acc.to(wire_dtype)
            else:
                dist.send(acc.to(wire_dtype), dst=role.parent, group=group, tag=tag)
        elif prim == BOARDCAST and is_root:
            publish = seg.to(wire_dtype)
        # ------------------------------ broadcast phase --------------------------------
        if prim != REDUCE:
            if not is_root and role.has(TR_IN_BCAST):
                publish = torch.empty(it.length, dtype=wire_dtype)
                dist.recv(publish, src=role.parent, group=group, tag=tag + (1 << 20))
                if role.has(TR_WANT_RESULT):
                    seg.copy_(publish.to(tensor.dtype))
            if role.has(TR_PUBLISH) and publish is not None:
                kids = _bcast_children(strategy, it.tree, rank, act, prim, relay_mode)
                reqs = [dist.isend(publish, dst=c, group=group, tag=tag + (1 << 20)) for c in kids]
                for r in reqs:
                    r.wait()
    return tensor


def _bcast_children(strategy: Strategy, t: int, rank: int, act: List[int], prim: int, relay_mode: int) -> List[int]:
    """Ranks that pull from ``rank`` in the broadcast phase: those whose effective parent is me."""
    tree = strategy.trees[t]
    out = []
    for r in tree.nodes:
        if r == rank:
            continue
        role = tree_role(tree, r, act, prim, relay_mode)
        if role.has(TR_IN_BCAST) and role.parent == rank:
            out.append(r)
    return out


def all_reduce_cpu(tensor, strategy, rank, world, **kw):
    return tree_collective_cpu(ALLREDUCE, tensor, strategy, rank, world, **kw)


def reduce_cpu(tensor, strategy, rank, world, **kw):
    return tree_collective_cpu(REDUCE, tensor, strategy, rank, world, **kw)


def boardcast_cpu(tensor, strategy, rank, world, **kw):
    return tree_collective_cpu(BOARDCAST, tensor, strategy, rank, world, **kw)
