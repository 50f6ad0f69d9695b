"""Single-GPU driver for ncu captures of our hot kernels (run under ``ncu -k regex:<name>``):
the collective kernels run with world size 1 and ``force_kernel`` (all phases execute: stage-in
cast, flag barrier, reduce/multimem phase, stage-out), plus the fused optimizer / CE / LayerNorm
kernels at GPT-2 shapes. ncu replays kernels, so this must never be a multi-rank command."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from adapcc_b200.ops import fused_adamw_, fused_ce_, sumsq_  # noqa: E402
from adapcc_b200.ops.layers import FusedLayerNorm  # noqa: E402
from adapcc_b200.runtime.native import NativeComm  # noqa: E402


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    if which in ("all", "comm"):
        comm = NativeComm("ncu-%d" % os.getpid(), 0, 1, 0, staging_bytes=256 << 20, heap_bytes=300 << 20)
        comm.set_tunable("force_kernel", 1)
        x = torch.randn(64 << 20, device=dev)                       # 256 MB fp32, staged
        g = comm.symm_empty(124_000_000, torch.bfloat16)            # a gradient-sized bf16 buffer, zero-copy
        g.normal_()
        for _ in range(3):
            comm.all_reduce(x, op="avg", algo="two_shot")
            comm.all_reduce(x, op="avg", algo="two_shot", wire="bfloat16")
            comm.all_reduce(g, op="avg", algo="two_shot")
            if comm.multicast:
                comm.all_reduce(g, op="avg", algo="nvls")
            comm.all_reduce(x[: 1 << 14], algo="one_shot")
        comm.check()
        comm.close()
    if which in ("all", "ops"):
        n = 124_476_673 // 8 * 8
        p = torch.randn(n, device=dev).bfloat16()
        gr = torch.randn(n, device=dev).bfloat16()
        master, m, v = p.float(), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
        ss = torch.zeros(1, device=dev)
        for i in range(3):
            ss.zero_()
            sumsq_(gr, ss)
            fused_adamw_(p, gr, master, m, v, lr=1e-4, step=i + 1, max_norm=1.0, sumsq=ss)
        logits = torch.randn(2048, 50304, device=dev).bfloat16()
        labels = torch.randint(0, 50262, (2048,), device=dev)
        for _ in range(3):
            fused_ce_(logits.clone(), labels, 50262)
        ln = FusedLayerNorm(768).to(dev).bfloat16()
        xx = torch.randn(8192, 768, device=dev).bfloat16().requires_grad_(True)
        for _ in range(3):
            ln(xx).backward(torch.randn(8192, 768, device=dev).bfloat16())
    if which in ("all", "gemm"):
        # the wgmma GEMM at the GPT-2 MLP up-projection shape, both variants
        # (ncu -k regex:gemm_bias_act_wgmma --set full ... python tools/ncu_targets.py gemm [variants, e.g. 0,1])
        from adapcc_b200.ops.gemm import linear_act
        variants = [int(t) for t in (sys.argv[2] if len(sys.argv) > 2 else "0").split(",")]
        a = torch.randn(8192, 768, device=dev).bfloat16()
        w = (torch.randn(3072, 768, device=dev) / 28).bfloat16()
        b = torch.randn(3072, device=dev).bfloat16()
        for v in variants:
            for _ in range(3):
                linear_act(a, w, b, "gelu", save_pre=True, variant=v)
        for _ in range(3):                                           # the cuBLAS kernels it competes with
            torch.nn.functional.gelu(torch.nn.functional.linear(a, w, b), approximate="tanh")
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
