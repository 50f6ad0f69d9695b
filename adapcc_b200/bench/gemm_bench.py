"""wgmma GEMM (+bias+GELU epilogue) vs cuBLAS(+separate GELU kernel), device-timed.

    python -m adapcc_b200.bench.gemm_bench [--m 8192 --n 3072 --k 768] [--iters 50] [--json out.json]

Each arm: 5 warm-up calls, then 5 batches of ``iters`` back-to-back launches between two CUDA events on the
launching stream; the median batch is reported as TFLOP/s = 2 M N K / t. No explicit L2 flush: at the default shape
one call streams 70-120 MB (A 12.6 MB, W 4.7 MB, one or two 50 MB outputs), more than the H100's 50 MB L2, so the
outputs of one call evict the operands of the next; the JSON records this.
"""
from __future__ import annotations

import argparse
import json
import statistics

import torch
import torch.nn.functional as F


def _time(fn, iters: int, batches: int = 5) -> float:
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(batches):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / iters)
    return statistics.median(out)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=8192)
    ap.add_argument("--n", type=int, default=3072)
    ap.add_argument("--k", type=int, default=768)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--variants", default="0", help="comma list of GEMM kernel variants (0-3) to time")
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    from adapcc_b200.ops.gemm import linear_act

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    x = torch.randn(a.m, a.k, device=dev).bfloat16()
    w = (torch.randn(a.n, a.k, device=dev) / a.k ** 0.5).bfloat16()
    b = torch.randn(a.n, device=dev).bfloat16()
    flops = 2.0 * a.m * a.n * a.k
    rows = []

    def add(name, fn, check=None):
        ms = _time(fn, a.iters)
        rows.append({"arm": name, "ms": ms, "tflops": flops / (ms * 1e-3) / 1e12, "max_abs_err": check})
        print(f"{name:44s} {ms * 1e3:9.1f} us  {rows[-1]['tflops']:8.1f} TFLOP/s" +
              (f"  max|err| {check:.3g}" if check is not None else ""), flush=True)

    ref_pre = F.linear(x, w, b)
    ref = F.gelu(ref_pre, approximate="tanh")
    add("cuBLAS linear (bias epilogue)", lambda: F.linear(x, w, b))
    add("cuBLAS linear + torch gelu kernel", lambda: F.gelu(F.linear(x, w, b), approximate="tanh"))
    for v in (int(t) for t in a.variants.split(",") if t != ""):
        out, pre = linear_act(x, w, b, "gelu", save_pre=True, variant=v)
        torch.cuda.synchronize()
        err = float((out.float() - ref.float()).abs().max())
        add(f"wgmma variant {v}: gelu(xW^T+b), no pre", lambda v=v: linear_act(x, w, b, "gelu", variant=v), err)
        add(f"wgmma variant {v}: gelu(xW^T+b) + pre", lambda v=v: linear_act(x, w, b, "gelu", save_pre=True, variant=v))
        if v == 3 and a.n % 256 == 0:
            # the MLP backward: dH = (dY . W2) * gelu'(pre) (+ the up-projection's bias gradient = column sums of dH)
            aux = ref_pre
            cs = torch.zeros(a.n, dtype=torch.float32, device=dev)
            add("cuBLAS matmul + torch gelu_backward kernel",
                lambda: torch.ops.aten.gelu_backward(x @ w.t(), aux, approximate="tanh"))
            add("cuBLAS matmul + gelu_backward + colsum kernels",
                lambda: torch.ops.aten.gelu_backward(x @ w.t(), aux, approximate="tanh").float().sum(0))
            add("wgmma variant 3: (xW^T) * gelu'(aux)", lambda: linear_act(x, w, None, "dgelu", aux=aux, variant=3))
            add("wgmma variant 3: dgelu + bias-grad column sums",
                lambda: linear_act(x, w, None, "dgelu", aux=aux, colsum=cs, variant=3))
    res = {"shape": [a.m, a.n, a.k], "dtype": "bf16", "iters": a.iters,
           "l2": "working set per call (inputs + 1-2 outputs, 70-120 MB at the default shape) streams through L2",
           "rows": rows}
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
