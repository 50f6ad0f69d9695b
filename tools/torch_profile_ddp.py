#!/usr/bin/env python
"""In-situ per-rank kernel timeline of the data-parallel GPT-2 step (graph engine, N GPUs) from torch.profiler/CUPTI.

    torchrun --nproc-per-node N tools/torch_profile_ddp.py --out gpurun_out/ddp_timeline_N.md [--zero1] [--impl nccl]

For every profiled step of rank 0 it lists each gradient-bucket collective (start relative to the step's first kernel,
duration, whether it overlapped compute), the end of the last backward compute kernel, the start of the optimizer
(`sumsq_kernel`) — the gap between the two is the EXPOSED communication tail — and the step length; plus the same step's
compute-kernel time so SM contention shows up as inflation against the 1-GPU table of
tools/torch_profile_step.py. Times are device timestamps (CUPTI), not wall clock.
"""
from __future__ import annotations

import argparse
import os
import re
import sys
from types import SimpleNamespace

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

COMM_PAT = re.compile(r"allreduce_direct_kernel|allreduce_pipelined|tree_collective|broadcast_direct|ncclDevKernel|"
                      r"ncclKernel|allreduce_ll_kernel|zero_adamw|barrier_kernel|skip_op")


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/ddp_timeline.md")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--impl", default="adapcc", choices=["adapcc", "nccl"])
    ap.add_argument("--zero1", action="store_true", help="(the default at N > 1)")
    ap.add_argument("--no_zero1", action="store_true", help="replicated optimizer + all-reduce")
    ap.add_argument("--bucket_mb", type=float, default=32.0)
    a = ap.parse_args()

    import torch
    import torch.distributed as dist
    from torch.profiler import ProfilerActivity, profile

    from adapcc_b200 import ALLREDUCE
    from adapcc_b200.adapcc import AdapCC
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
    from adapcc_b200.parallel.engine import FlatDataParallel

    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    cfg = GPT2Config()
    torch.manual_seed(1234)
    model = GPT2DoubleHeads(cfg).to(dev)
    n_params = model.num_parameters()
    work = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "gpurun_out", "bench_work")
    os.makedirs(os.path.join(work, "strategy"), exist_ok=True)
    comm, comm_fn = None, None
    if a.impl == "adapcc" and world > 1:
        args = SimpleNamespace(port=5100, strategy_file=os.path.join(work, "strategy", f"prof_{world}.xml"),
                               logical_graph=os.path.join(work, "topology", f"logical_graph_{world}.xml"),
                               entry_point=-1, parallel_degree=min(4, world), profile_freq=500, work_dir=work,
                               relay_control=False, algo="auto", heap_mb=((1 if a.no_zero1 else 2) * n_params * 2 >> 20) + 64,
                               staging_mb=64, backend="nccl")
        AdapCC.init(args, local, rank, world)
        AdapCC.setup(ALLREDUCE)
        comm = AdapCC.communicator.native
    elif world > 1:
        def comm_fn(seg):
            dist.all_reduce(seg, op=dist.ReduceOp.AVG)
    eng = FlatDataParallel(model, comm, world_size=world, rank=rank, bucket_mb=a.bucket_mb, lr=6.25e-5, max_norm=1.0,
                           comm_fn=comm_fn, zero1=False if a.no_zero1 else None)
    batch = synthetic_batch(4, 2, 1024, cfg.vocab_size, device=dev, seed=rank)
    eng.capture(batch, warmup=2)
    for _ in range(5):
        eng._graph.replay()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps + 1):          # the first profiled step absorbs CUPTI's start-up skew between the ranks
            eng._graph.replay()
        torch.cuda.synchronize()
    ks = []
    for ev in prof.events():
        if ev.device_type is not None and str(ev.device_type).endswith("CUDA") and ev.device_time_total > 0:
            ks.append((ev.time_range.start, ev.time_range.end, ev.name))
    ks.sort()
    # one `incr_int_kernel` per step marks the start of the optimizer; the optimizer's own kernels follow it
    OPT_PAT = re.compile(r"sumsq_kernel|adamw|barrier|allreduce_direct_kernel|allreduce_ll_kernel|skip_op|ncclDevKernel")

    def in_optimizer(k):            # tiny fills / memsets (sumsq.zero_()) belong to it; the 249 MB gradient clear does not
        return bool(OPT_PAT.search(k[2])) or ((k[1] - k[0]) < 5.0 and re.search(r"Fill|Memset|elementwise", k[2]) is not None)
    starts = [i for i, k in enumerate(ks) if "incr_int_kernel" in k[2]]
    lines = []
    bucket_elems = [b.end - b.start for b in eng.buckets]
    lines.append(f"# DDP step timeline, rank {rank} of {world}, impl={a.impl}, zero1={bool(getattr(eng, 'zero1', False))}, "
                 f"{len(eng.buckets)} buckets (MB: {[round(e * 2 / 2**20, 1) for e in bucket_elems]}, launch order = list order)\n")
    step_begin = 0
    summary = []
    for si, opt_i in enumerate(starts):
        skip_first = si == 0 and len(starts) > 1
        last = opt_i
        while last + 1 < len(ks) and in_optimizer(ks[last + 1]):
            last += 1
        seg = ks[step_begin:last + 1]
        step_begin = last + 1
        if skip_first:
            continue
        t0 = seg[0][0]
        comm_k = [k for k in seg if COMM_PAT.search(k[2]) and "adamw" not in k[2] and k[0] < ks[opt_i][0]]
        comp_k = [k for k in seg if not COMM_PAT.search(k[2])]
        sumsq_start = ks[opt_i][0]
        opt_len = (seg[-1][1] - sumsq_start) / 1e3
        bwd_end = max((k[1] for k in comp_k if k[1] <= sumsq_start), default=sumsq_start)
        comp_time = sum(k[1] - k[0] for k in comp_k)
        lines.append(f"## step {si}: length {(seg[-1][1] - t0) / 1e3:.3f} ms, compute-kernel time {comp_time / 1e3:.3f} ms, "
                     f"last backward kernel ends at {(bwd_end - t0) / 1e3:.3f} ms, optimizer starts at {(sumsq_start - t0) / 1e3:.3f} ms "
                     f"-> exposed tail {(sumsq_start - bwd_end) / 1e3:.3f} ms; optimizer section {opt_len:.3f} ms\n")
        lines.append("| collective kernel | start ms | duration us | overlaps compute |\n|---|---|---|---|\n")
        for k in comm_k:
            ov = any(c[0] < k[1] and c[1] > k[0] for c in comp_k)
            nm = re.sub(r"^void\s+|adapcc::", "", k[2])[:70]
            lines.append(f"| {nm} | {(k[0] - t0) / 1e3:.3f} | {(k[1] - k[0]):.1f} | {'yes' if ov else 'NO (exposed)'} |\n")
        lines.append("\n")
        if si == len(starts) - 1:
            # the last 24 kernels before the optimizer (what the step's tail is made of) ...
            before = [k for k in seg if k[0] < sumsq_start][-24:]
            lines.append("last kernels before the optimizer (start ms, us, name):\n\n```\n")
            for k in before:
                lines.append(f"{(k[0] - t0) / 1e3:8.3f} {(k[1] - k[0]):8.1f}  {re.sub(r'^void |adapcc::', '', k[2])[:100]}\n")
            lines.append("```\n\n")
            # ... and the step's compute kernels by name, to diff against another world size
            by = {}
            for k in comp_k:
                nm = re.sub(r"<.*", "", re.sub(r"^void\s+", "", k[2])).replace("at::native::", "native::")[:80]
                c, t = by.get(nm, (0, 0.0))
                by[nm] = (c + 1, t + (k[1] - k[0]))
            lines.append("| compute kernel (this step) | launches | us |\n|---|---|---|\n")
            for nm, (c, t) in sorted(by.items(), key=lambda kv: -kv[1][1])[:40]:
                lines.append(f"| {nm} | {c} | {t:.1f} |\n")
            lines.append("\n")
        summary.append(((seg[-1][1] - t0) / 1e3, comp_time / 1e3, (sumsq_start - bwd_end) / 1e3,
                        sum(k[1] - k[0] for k in comm_k) / 1e3))
    if summary:
        n = len(summary)
        lines.insert(1, "mean over %d steps: step %.3f ms, compute kernels %.3f ms, exposed tail %.3f ms, collective kernel "
                        "time %.3f ms\n\n" % (n, *(sum(s[i] for s in summary) / n for i in range(4))))
    out = a.out if rank == 0 else a.out.replace(".md", f"_rank{rank}.md")
    if rank in (0, world - 1):
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        with open(out, "w") as f:
            f.writelines(lines)
    if rank == 0:
        print("".join(lines)[:2500])
    if comm is not None:
        AdapCC.communicator.synchronize()
        AdapCC.clear(ALLREDUCE)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
