#!/usr/bin/env python
"""What gradient accumulation costs on the GPU this runs on (it fails without one): the captured GPT-2 small training
step of ``FlatDataParallel`` at micro-batch B = 4, C = 2, T = 1024 (``bench.py``'s shape) with
``gradient_accumulation_steps`` M = 1, 2 and 4, and the accumulate and fold kernels alone over the whole flat buffer.

    python tools/grad_accum_bench.py [--steps 20] [--rounds 3] [--iters 50]

The three engines are built and captured first; then each round replays every engine ``--steps`` optimizer steps in
turn, so the variants alternate inside one process and the spread across rounds is visible. A reading is CUDA events
around the replays: milliseconds per optimizer step and per micro-batch, and the per-micro-batch overhead against
M = 1 of the same round. The kernels are timed over ``--iters`` back-to-back launches on buffers of the engine's
``total`` elements (far past the 50 MB L2); their bytes come from the shapes (bf16 gradient read, fp32 accumulator
read and / or written, bf16 gradient written by the fold), and the share is those bytes per second over the H100 SXM
data sheet's 3.35 TB/s. The card's name and power limit are printed first: they are part of every number.
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

HBM = 3.35e12
B, C, T = 4, 2, 1024
MS = (1, 2, 4)


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_steps(dev, steps, rounds):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
    from adapcc_b200.parallel.engine import FlatDataParallel

    cfg = GPT2Config()
    batches = [{k: v.to(dev) for k, v in synthetic_batch(B, C, T, cfg.vocab_size, seed=i).items()} for i in range(max(MS))]
    engines = {}
    for M in MS:
        torch.manual_seed(1234)
        eng = FlatDataParallel(GPT2DoubleHeads(cfg).to(dev), None, world_size=1, lr=6.25e-5, max_norm=1.0,
                               gradient_accumulation_steps=M)
        inputs = batches[:M] if M > 1 else batches[0]
        eng.capture(inputs, warmup=2)
        engines[M] = (eng, inputs)
        print(f"M = {M}: {len(eng.buckets)} buckets, {eng.native_launches_per_step} native launches per step, "
              f"accumulator {0 if eng.grad_acc is None else eng.grad_acc.numel() * 4 / 2**20:.0f} MiB", flush=True)
    total = engines[1][0].total
    for eng, inputs in engines.values():
        timed(lambda: eng.step_graph(inputs), 3)
    print(f"captured GPT-2 small step, micro-batch B = {B}, C = {C}, T = {T} ({B * C * T} tokens), {steps} steps "
          f"per reading:")
    for r in range(rounds):
        ms = {M: timed(lambda: eng.step_graph(inputs), steps) for M, (eng, inputs) in engines.items()}
        cells = [f"M = {M}: {ms[M]:7.2f} ms/step {ms[M] / M:6.2f} ms/micro-batch "
                 f"(+{ms[M] / M - ms[1]:.3f} ms over M = 1)" for M in MS]
        print(f"  round {r}: " + " | ".join(cells), flush=True)
    for eng, _ in engines.values():
        eng.close()
    return total


def bench_kernels(dev, total, iters, rounds):
    from adapcc_b200.ops import grad_accum_, grad_fold_

    g = torch.randn(total, device=dev).bfloat16()
    acc = torch.randn(total, device=dev)
    variants = {"accumulate (first)": (lambda: grad_accum_(g, acc, True), total * (2 + 4)),
                "accumulate": (lambda: grad_accum_(g, acc, False), total * (2 + 4 + 4)),
                "fold": (lambda: grad_fold_(g, acc, 0.25), total * (2 + 4 + 2))}
    for fn, _ in variants.values():
        timed(fn, 3)
    print(f"kernels over the flat buffer ({total} elements, bf16 gradient), {iters} launches per reading:")
    for r in range(rounds):
        cells = []
        for name, (fn, nbytes) in variants.items():
            ms = timed(fn, iters)
            cells.append(f"{name} {ms * 1e3:6.1f} us {nbytes / 1e9:5.2f} GB "
                         f"{nbytes / (ms * 1e-3) / HBM * 100:4.1f} % of 3.35 TB/s")
        print(f"  round {r}: " + " | ".join(cells), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grad_accum_bench.py needs a GPU: a CPU run says nothing about these kernels")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print(f"GPU: {torch.cuda.get_device_name(0)}; name, power limit, max SM clock: {q.stdout.strip() or 'nvidia-smi unavailable'}")
    total = bench_steps(dev, a.steps, a.rounds)
    bench_kernels(dev, total, a.iters, a.rounds)


if __name__ == "__main__":
    main()
