"""Tree micro-benchmarks — what the authors explored in nccl-perf/tree/*.cu
(/root/reference/nccl-perf/tree/{tree,tree_chunk,send_recv,all_reduce}.cu; report_tree_chunk128.txt:
a hand-built 4-GPU ncclSend/ncclRecv reduction tree with a separate 2-input reduceKernel took
1.6-2.1 s per rank at 128-byte chunks, 196 608 kernel launches). Here the same comparison on H100:

  * ``nccl_sendrecv_tree``: the reference-style tree built from batched isend/irecv + an add per hop,
  * ``adapcc_tree``      : our single-kernel strategy tree (reduce CTAs + broadcast CTAs),
  * ``nccl_allreduce``   : the library collective,

for a chain and a binary tree over all ranks, several chunk sizes, device-timed, max over ranks.

    torchrun --nproc-per-node 4 -m adapcc_b200.bench.tree_bench --mb 64
"""
import argparse
import os

import torch
import torch.distributed as dist

from ..constants import ALLREDUCE
from ..runtime.native import NativeComm
from ..runtime.rendezvous import unique_name
from ..strategy import make_strategy


def sendrecv_tree_allreduce(x, tmp, tree, rank, chunk_elems):
    """Reduce up / broadcast down the tree with NCCL point-to-point, chunk by chunk."""
    kids, parent = tree.kids(rank), tree.parent.get(rank)
    for s in range(0, x.numel(), chunk_elems):
        seg, t = x[s:s + chunk_elems], tmp[s:s + chunk_elems]
        for c in kids:
            dist.recv(t, src=c)
            seg.add_(t)
        if parent is not None:
            dist.send(seg, dst=parent)
    for s in range(0, x.numel(), chunk_elems):
        seg = x[s:s + chunk_elems]
        if parent is not None:
            dist.recv(seg, src=parent)
        for c in kids:
            dist.send(seg, dst=c)


def timed(fn, iters, dev):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    t = torch.tensor([a.elapsed_time(b) / iters], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=64.0)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    n = int(a.mb * (1 << 20)) // 4
    x, tmp = torch.randn(n, device=dev), torch.empty(n, device=dev)
    comm = NativeComm(unique_name("treebench"), rank, world, local, staging_bytes=max(n * 4, 1 << 20))
    f = 2 * (world - 1) / world
    if rank == 0:
        print(f"# {a.mb} MiB fp32, world {world}; ms per all-reduce (bus GB/s)")
    t = timed(lambda: dist.all_reduce(x), a.iters, dev)
    if rank == 0:
        print(f"nccl_allreduce            {t:9.3f} ms ({n * 4 * f / t / 1e6:7.1f})")
    for shape in ("chain", "binary"):
        s = make_strategy(world, 1, shape)
        comm.load_strategy(s.to_xml())
        for chunk in (1 << 16, 1 << 20, 4 << 20):
            ce = chunk // 4
            if n // ce <= 4096:
                t = timed(lambda: sendrecv_tree_allreduce(x, tmp, s.trees[0], rank, ce), max(1, a.iters // 2), dev)
                if rank == 0:
                    print(f"nccl_sendrecv_tree {shape:6s} chunk {chunk >> 10:5d}K {t:9.3f} ms ({n * 4 * f / t / 1e6:7.1f})")
            t = timed(lambda: comm.tree_collective(ALLREDUCE, x, chunk_bytes=chunk), a.iters, dev)
            comm.check()
            if rank == 0:
                print(f"adapcc_tree        {shape:6s} chunk {chunk >> 10:5d}K {t:9.3f} ms ({n * 4 * f / t / 1e6:7.1f})")
    dist.barrier()
    comm.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
