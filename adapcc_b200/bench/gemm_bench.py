"""wgmma GEMM (+bias+GELU / dGELU epilogues) vs cuBLAS(+separate activation kernels), device-timed.

    python -m adapcc_b200.bench.gemm_bench [--m 8192 --n 3072 --ks 768,1536,3072] [--iters 50] [--json out.json]

Each arm is captured once as a CUDA graph of ``iters`` back-to-back calls, replayed 5 times after 3 warm-up replays
between two CUDA events; the median replay is reported per call. The graph takes the host out of the number: an eager
call of ``linear_act`` costs a Python call, a ``torch.empty``, two tensor-map encodings and a ctypes call, which is
comparable to the kernel itself at these shapes. No explicit L2 flush: at the default shape one call streams 70-120 MB
(A 12.6 MB, W 4.7 MB, one or two 50 MB outputs), more than the H100's 50 MB L2, so the outputs of one call evict the
operands of the next.

The K sweep separates the mainloop from the per-tile fixed cost: time(K) ~ intercept + slope K, where the slope is the
wgmma mainloop's rate and the intercept the epilogue + pipeline refill. Each row also reports the least time the
hardware could take, max(FLOPs / 989 TFLOP/s, bytes / 3.35 TB/s) (H100 SXM dense BF16 and HBM3 data-sheet figures),
which of the two bounds it, and the achieved share of it.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess

import torch
import torch.nn.functional as F

PEAK_FLOPS = 989e12
PEAK_BYTES = 3.35e12


def card() -> dict:
    """Name, power limit and max SM clock of cuda:0, read in the same process as the measurement."""
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock_max"] = [x.strip() for x in q.split(",")][:2]
    except (OSError, ValueError, subprocess.TimeoutExpired):
        info["power_limit"] = info["sm_clock_max"] = "unknown"
    return info


def _time(fn, iters: int, replays: int = 5) -> float:
    """Median ms per call over `replays` replays of a graph of `iters` captured calls."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):                          # eager warm-up: module load, cuBLAS heuristics, launch setup
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    out = []
    for _ in range(replays):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / iters)
    del g
    return statistics.median(out)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=8192)
    ap.add_argument("--n", type=int, default=3072)
    ap.add_argument("--ks", default="768", help="comma list of K values (a sweep fits time = intercept + slope K)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--variants", default="3", help="comma list of GEMM kernel variants (0-3) to time")
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    from adapcc_b200.ops.gemm import linear_act

    dev = torch.device("cuda:0")
    info = card()
    print(f"# {info['name']}, power limit {info['power_limit']}, max SM clock {info['sm_clock_max']}", flush=True)
    rows = []
    m, n = a.m, a.n
    for k in (int(t) for t in a.ks.split(",") if t.strip()):
        torch.manual_seed(0)
        x = torch.randn(m, k, device=dev).bfloat16()
        w = (torch.randn(n, k, device=dev) / k ** 0.5).bfloat16()
        b = torch.randn(n, device=dev).bfloat16()
        flops = 2.0 * m * n * k
        ab = 2.0 * (m * k + n * k)                  # operand bytes; one bf16 [M, N] tensor is 2 M N
        mn = 2.0 * m * n
        print(f"## M={m} N={n} K={k}", flush=True)

        def add(name, fn, nbytes, check=None):
            ms = _time(fn, a.iters)
            t_min = max(flops / PEAK_FLOPS, nbytes / PEAK_BYTES)
            bound = "compute" if flops / PEAK_FLOPS >= nbytes / PEAK_BYTES else "memory"
            rows.append({"arm": name, "k": k, "us": ms * 1e3, "tflops": flops / (ms * 1e-3) / 1e12,
                         "gbytes_per_s": nbytes / (ms * 1e-3) / 1e9, "bound": bound,
                         "share_of_bound": t_min / (ms * 1e-3), "max_abs_err": check})
            r = rows[-1]
            print(f"{name:46s} {r['us']:8.1f} us  {r['tflops']:6.1f} TFLOP/s ({100 * r['tflops'] * 1e12 / PEAK_FLOPS:4.1f} % "
                  f"of 989)  {r['gbytes_per_s']:6.0f} GB/s  {bound}-bound, {100 * r['share_of_bound']:4.1f} % of that bound"
                  + (f"  max|err| {check:.3g}" if check is not None else ""), flush=True)

        ref_pre = F.linear(x, w, b)
        ref = F.gelu(ref_pre, approximate="tanh")
        aux = ref_pre
        cs = torch.zeros(n, dtype=torch.float32, device=dev)
        work = 2.0 * 4 * ((m + 127) // 128) * n     # the [tiles_m, N] fp32 column-sum rows, written and read back
        add("cuBLAS linear (bias epilogue)", lambda: F.linear(x, w, b), ab + mn)
        add("cuBLAS linear + torch gelu kernel", lambda: F.gelu(F.linear(x, w, b), approximate="tanh"), ab + mn)
        add("cuBLAS matmul + gelu_backward + colsum", lambda: torch.ops.aten.gelu_backward(
            x @ w.t(), aux, approximate="tanh").float().sum(0), ab + 2 * mn)
        for v in (int(t) for t in a.variants.split(",") if t.strip()):
            out, _ = linear_act(x, w, b, "gelu", save_pre=True, variant=v)
            torch.cuda.synchronize()
            err = float((out.float() - ref.float()).abs().max())
            add(f"wgmma v{v}: gelu(xW^T+b), no pre", lambda v=v: linear_act(x, w, b, "gelu", variant=v), ab + mn, err)
            add(f"wgmma v{v}: gelu(xW^T+b) + pre", lambda v=v: linear_act(x, w, b, "gelu", save_pre=True, variant=v),
                ab + 2 * mn)
            if v == 3 and n % 256 == 0:
                # the MLP backward: dH = (dY . W2) * gelu'(pre) + the up-projection's bias gradient (column sums of dH)
                add("wgmma v3: dgelu + bias-grad column sums",
                    lambda: linear_act(x, w, None, "dgelu", aux=aux, colsum=cs, variant=3), ab + 2 * mn + work)
            elif v == 0:
                add("wgmma v0: dgelu", lambda: linear_act(x, w, None, "dgelu", aux=aux, variant=0), ab + 2 * mn)
        del x, w, b, ref_pre, ref, aux
    res = {"shape": [m, n], "dtype": "bf16", "iters": a.iters, "card": info, "timing": "CUDA graph of iters calls",
           "l2": "working set per call (inputs + 1-2 outputs, 70-120 MB at K=768) streams through L2", "rows": rows}
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
