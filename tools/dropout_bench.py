#!/usr/bin/env python
"""What training dropout costs on the GPU this runs on (it fails without one): the fused add-LayerNorm and embedding
kernels with and without their masks, and the captured GPT-2 small training step at p = 0, at p = 0.1, and with
``F.dropout`` at the same sites for comparison.

    python tools/dropout_bench.py [--iters 4000] [--steps 30] [--rounds 3]

Every shape is warmed first; the variants of a comparison alternate inside one process, ``--rounds`` times, and each
round is printed so the spread is visible. Kernel times are CUDA events around ``--iters`` back-to-back launches (about
0.1 s per reading at the default). The add-LayerNorm launches rotate over ``SETS`` sets of input and output buffers,
200 MB in all, so that a launch finds none of its 50 MB in the 50 MB L2 left by the previous one. The bytes a variant
moves are computed from its shapes (every tensor read or written once), and the share is those bytes per second over
the H100 SXM data sheet's 3.35 TB/s. The ``F.dropout`` arm of the step comparison also runs the residual adds
unfused from the LayerNorms and leaves out the summary site: it is an upper bound for stock dropout, not an isolated
dropout cost. The card's name and power limit are printed first: they are part of every number.
"""
import argparse
import dataclasses
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

HBM = 3.35e12
ROWS, D = 8192, 768                          # bench.py's activation: 4 dialogues x 2 candidates x 1024 tokens
SETS = 4                                     # buffer sets the add-LayerNorm launches rotate over


def timed(fn, iters):
    """Milliseconds per call over ``iters`` launches (CUDA events); ``fn``: a callable, or a list of them taken in turn."""
    fns = fn if isinstance(fn, list) else [fn]
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        fns[i % len(fns)]()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def report(title, variants, iters, rounds):
    """variants: {name: (fn, bytes moved)}; warm each, then alternate them ``rounds`` times."""
    for fn, _ in variants.values():
        timed(fn, 16)
    torch.cuda.synchronize()
    print(title)
    for r in range(rounds):
        cells = []
        for name, (fn, nbytes) in variants.items():
            ms = timed(fn, iters)
            cells.append(f"{name} {ms * 1e3:7.1f} us  {nbytes / 1e6:6.1f} MB  {nbytes / (ms * 1e-3) / HBM * 100:4.1f} % of 3.35 TB/s")
        print(f"  round {r}: " + " | ".join(cells))


def bench_add_ln(dev, iters, rounds):
    from adapcc_b200.ops.dropout import DropoutState, drop_tail
    from adapcc_b200.ops.layers import _lib, _p, _s

    lib = _lib()
    bf = dict(dtype=torch.bfloat16, device=dev)
    gamma, beta = torch.ones(D, **bf), torch.zeros(D, **bf)
    dg, db = torch.empty(D, **bf), torch.empty(D, **bf)
    mean, rstd = (torch.empty(ROWS, dtype=torch.float32, device=dev) for _ in range(2))
    part = torch.empty(2 * lib.adapcc_ln_partials(ROWS) * D, dtype=torch.float32, device=dev)
    st = DropoutState.create(1, 1, dev)
    tail = drop_tail("bench", 0.1, st, 3, dev)
    t = ROWS * D * 2                                    # one bf16 activation
    fwd, fwd_drop, bwd, bwd_drop = [], [], [], []
    for _ in range(SETS):
        x, res, dy, dsum = (torch.randn(ROWS, D, **bf) for _ in range(4))
        s, y, dx, dres = (torch.empty(ROWS, D, **bf) for _ in range(4))
        lib.adapcc_add_ln_fwd(_p(x), _p(res), _p(gamma), _p(beta), _p(s), _p(y), _p(mean), _p(rstd), ROWS, D, 1e-5, _s())
        fwd.append(lambda x=x, res=res, s=s, y=y: lib.adapcc_add_ln_fwd(
            _p(x), _p(res), _p(gamma), _p(beta), _p(s), _p(y), _p(mean), _p(rstd), ROWS, D, 1e-5, _s()))
        fwd_drop.append(lambda x=x, res=res, s=s, y=y: lib.adapcc_add_ln_drop_fwd(
            _p(x), _p(res), _p(gamma), _p(beta), _p(s), _p(y), _p(mean), _p(rstd), ROWS, D, 1e-5, *tail, _s()))
        bwd.append(lambda dy=dy, s=s, dsum=dsum, dx=dx: lib.adapcc_add_ln_bwd(
            _p(dy), _p(s), _p(gamma), _p(mean), _p(rstd), _p(dsum), _p(dx), _p(dg), _p(db), _p(part), ROWS, D, _s()))
        bwd_drop.append(lambda dy=dy, s=s, dsum=dsum, dx=dx, dres=dres: lib.adapcc_add_ln_drop_bwd(
            _p(dy), _p(s), _p(gamma), _p(mean), _p(rstd), _p(dsum), _p(dx), _p(dres), _p(dg), _p(db), _p(part), ROWS,
            D, *tail, _s()))
    report(f"add-LayerNorm forward {ROWS} x {D} (x, res -> sum, y), {SETS} buffer sets in rotation",
           {"plain  ": (fwd, 4 * t), "dropout": (fwd_drop, 4 * t)}, iters, rounds)
    report(f"add-LayerNorm backward {ROWS} x {D} (dy, sum, dsum -> dx [, dres]; + column-sum finalise), {SETS} buffer "
           f"sets in rotation", {"plain  ": (bwd, 4 * t), "dropout": (bwd_drop, 5 * t)}, iters, rounds)


def bench_embed(dev, iters, rounds):
    from adapcc_b200.ops import fused_embedding_sum
    from adapcc_b200.ops.dropout import DropoutState

    V, T = 50304, 1024
    g = torch.Generator().manual_seed(0)
    wte = torch.randn(V, D, generator=g).bfloat16().to(dev).requires_grad_(True)
    wpe = torch.randn(T, D, generator=g).bfloat16().to(dev).requires_grad_(True)
    ids = torch.randint(0, 50257, (ROWS,), generator=g).to(dev)
    tt = torch.randint(50257, 50259, (ROWS,), generator=g).to(dev)
    pos = torch.arange(T).repeat(ROWS // T).to(dev)
    dy = torch.randn(ROWS, D, generator=g).bfloat16().to(dev)
    st = DropoutState.create(1, 1, dev)
    lookups = [(0, ids), (1, pos), (0, tt)]
    t = ROWS * D * 2

    def fwd(drop):
        with torch.no_grad():
            fused_embedding_sum([wte, wpe], lookups, drop)

    def both(drop):
        torch.autograd.grad(fused_embedding_sum([wte, wpe], lookups, drop), [wte, wpe], dy)

    # the gathered rows come from a 77 MB table and the output is a fresh allocation each call; the positional rows
    # (1.5 MB) and the two token-type rows do stay in L2, as they do in training
    report(f"embedding forward {ROWS} x {D}, 3 lookups (3 gathered rows read, 1 written)",
           {"plain  ": (lambda: fwd(None), 4 * t), "dropout": (lambda: fwd((0.1, st, 0)), 4 * t)}, iters // 4, rounds)
    # backward: claim and scatter each read dY once per lookup; the int64 scratch and the two zero-filled gradient
    # tables autograd allocates here are the same for both variants and are not counted
    report(f"embedding forward + backward {ROWS} x {D} (dY read 6 times on top of the forward)",
           {"plain  ": (lambda: both(None), 10 * t), "dropout": (lambda: both((0.1, st, 0)), 10 * t)}, max(iters // 8, 10),
           rounds)


def _f_dropout_model(cfg, p):
    """GPT2DoubleHeads with ``F.dropout`` on the embedding sum and on every block's attention and MLP output (the 25
    activation-sized sites; the [8, 768] summary input is left out): PyTorch's generator and kernels, one stand-alone
    pass per site forward and backward, and the residual adds unfused from the LayerNorms (the comparison arm only)."""
    from adapcc_b200.models.gpt2 import GPT2DoubleHeads

    class M(GPT2DoubleHeads):
        def _blocks(self, x, cache, drop=None):
            x = F.dropout(x, p, True)
            for i, blk in enumerate(self.h):
                x = x + F.dropout(blk._attn(blk.ln_1(x), cache, i), p, True)
                x = x + F.dropout(blk._mlp(blk.ln_2(x)), p, True)
            return self.ln_f(x)

    return M(cfg)


def bench_step(dev, steps, rounds):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch
    from adapcc_b200.parallel.engine import FlatDataParallel

    batch = {k: v.to(dev) for k, v in synthetic_batch(4, 2, 1024, GPT2Config().vocab_size, seed=1000).items()}
    engines = {}
    for name, p, build in (("p = 0      ", 0.0, GPT2DoubleHeads), ("p = 0.1    ", 0.1, GPT2DoubleHeads),
                           ("F.dropout, unfused adds", 0.1, None)):
        torch.manual_seed(1234)
        cfg = dataclasses.replace(GPT2Config(), embd_pdrop=p, resid_pdrop=p, summary_first_dropout=p)
        model = (build(cfg) if build else _f_dropout_model(GPT2Config(), p)).to(dev)
        eng = FlatDataParallel(model, None, world_size=1, lr=6.25e-5, dropout_seed=7 if build and p else None)
        eng.capture(batch, warmup=3)
        engines[name] = eng
    print("captured FlatDataParallel GPT-2 small step, B = 4, C = 2, T = 1024 (bench.py's shape), ms per step")
    for eng in engines.values():
        for _ in range(5):
            eng.step_graph(batch)
    for r in range(rounds):
        cells = [f"{name} {timed(lambda e=eng: e.step_graph(batch), steps):7.3f}" for name, eng in engines.items()]
        print(f"  round {r}: " + " | ".join(cells))
    for eng in engines.values():
        eng.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=4000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dropout_bench.py needs a GPU: a CPU run says nothing about these kernels")
    dev = torch.device("cuda", 0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print(f"GPU: {torch.cuda.get_device_name(0)}; name, power limit, max SM clock: {q.stdout.strip() or 'nvidia-smi unavailable'}")
    bench_add_ln(dev, a.iters, a.rounds)
    bench_embed(dev, a.iters, a.rounds)
    bench_step(dev, a.steps, a.rounds)


if __name__ == "__main__":
    main()
