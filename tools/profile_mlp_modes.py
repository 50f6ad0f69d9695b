#!/usr/bin/env python
"""Per-kernel time of one eager GPT-2 training step with the MLP on our fused wgmma GEMM (``ADAPCC_TCGEN05_MLP=2``)
and on cuBLAS + separate activation kernels (``=0``), side by side, from torch.profiler (CUPTI) kernel durations:

    python tools/profile_mlp_modes.py OUT_DIR [--steps 3]

Writes OUT_DIR/mlp_modes.md (kernels grouped by shortened name, us per step in each mode and the difference) and
OUT_DIR/mlp_modes.json. The eager engine is used so that every kernel is attributed; its host overhead does not enter
the kernel times.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

from torch_profile_step import short  # noqa: E402


def profile_mode(mode: str, steps: int, batch: int, candidates: int, seq: int) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile

    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
    from adapcc_b200.parallel.engine import FlatDataParallel

    os.environ["ADAPCC_TCGEN05_MLP"] = mode         # read when the blocks are built
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    cfg = GPT2Config()
    model = GPT2DoubleHeads(cfg).to(dev)
    data = synthetic_batch(batch, candidates, seq, cfg.vocab_size, device=dev)
    eng = FlatDataParallel(model, None, world_size=1, lr=1e-4, max_norm=1.0)
    for _ in range(3):
        eng.step(data)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            eng.step(data)
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type is not None and str(ev.device_type).endswith("CUDA") and ev.device_time_total > 0:
            k = short(ev.name)
            n, t = rows.get(k, (0, 0.0))
            rows[k] = (n + 1, t + ev.device_time_total)
    del eng, model
    torch.cuda.empty_cache()
    return {k: {"launches": n / steps, "us": t / steps} for k, (n, t) in rows.items()}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--candidates", type=int, default=2)
    ap.add_argument("--seq", type=int, default=1024)
    a = ap.parse_args()
    import torch

    modes = {m: profile_mode(m, a.steps, a.batch, a.candidates, a.seq) for m in ("2", "0")}
    os.makedirs(a.out_dir, exist_ok=True)
    names = sorted(set(modes["2"]) | set(modes["0"]),
                   key=lambda k: -max(modes["2"].get(k, {}).get("us", 0), modes["0"].get(k, {}).get("us", 0)))
    tot = {m: sum(r["us"] for r in modes[m].values()) for m in modes}
    lines = [f"# GPT-2 small eager step, B={a.batch} C={a.candidates} T={a.seq}, torch.profiler kernel durations, "
             f"{torch.cuda.get_device_name(0)}, {a.steps} steps\n",
             f"kernel time per step: MLP=2 {tot['2'] / 1e3:.3f} ms, MLP=0 {tot['0'] / 1e3:.3f} ms\n",
             "| kernel | MLP=2 launches | MLP=2 us/step | MLP=0 launches | MLP=0 us/step | 2 - 0 us |",
             "|---|---|---|---|---|---|"]
    for k in names:
        r2, r0 = modes["2"].get(k, {"launches": 0, "us": 0.0}), modes["0"].get(k, {"launches": 0, "us": 0.0})
        lines.append(f"| {k} | {r2['launches']:.0f} | {r2['us']:.1f} | {r0['launches']:.0f} | {r0['us']:.1f} | "
                     f"{r2['us'] - r0['us']:+.1f} |")
    text = "\n".join(lines) + "\n"
    with open(os.path.join(a.out_dir, "mlp_modes.md"), "w") as f:
        f.write(text)
    with open(os.path.join(a.out_dir, "mlp_modes.json"), "w") as f:
        json.dump({"device": torch.cuda.get_device_name(0), "steps": a.steps, "modes": modes}, f, indent=1)
    print(text[:6000])
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
