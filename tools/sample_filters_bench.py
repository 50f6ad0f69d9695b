#!/usr/bin/env python
"""The cost of the sampler's truncation filters (min-p, typical, epsilon, eta, top-h) on GPT-2's vocabulary.

Prints one JSON line. Needs a CUDA device (there is no CPU fallback) and writes nothing into the repository.

* ``kernels``: ``sample_tokens_`` alone at B = 1 / 8 / 64 and vocab 50262, temperature 0.7, ``top_p = 0.9``, on
  ``randn * 3`` logits, with every filter off and with each filter on (and min-p to eta together). 50 launches are
  captured in a CUDA graph and timed with CUDA events over ``--launches`` launches; the configurations are alternated
  and each figure is the median over ``--rounds`` rounds. ``--baseline-lib`` times another build of ``libadapcc.so``
  (for example the one before the filters existed) through its ``adapcc_sample_tokens`` in the same rounds, so the
  filters-off figure can be compared with it.
* ``generate``: ms per generated token of ``GPT2DoubleHeads.generate`` (GPT-2 small, bf16, seeded random weights,
  B = 8, prompts of 512 tokens, 64 new tokens, temperature 0.7, ``top_p = 0.9``), prefill and graph capture included,
  with and without ``typical_p = 0.9``, alternated call by call; the median of ``--reps`` calls after a warm-up each.

Usage: ``python tools/sample_filters_bench.py [--launches 1000] [--rounds 5] [--reps 7] [--baseline-lib PATH]``
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

VOCAB = 50262
GRAPH_LAUNCHES = 50
NEW_TOKENS = 64
FILTERS = [("off", {}), ("min_p=0.05", dict(min_p=0.05)), ("typical_p=0.9", dict(typical_p=0.9)),
           ("epsilon_cutoff=3e-4", dict(epsilon_cutoff=3e-4)), ("eta_cutoff=3e-4", dict(eta_cutoff=3e-4)),
           ("all four", dict(min_p=0.05, typical_p=0.9, epsilon_cutoff=3e-4, eta_cutoff=3e-4)),
           ("top_h=0.9", dict(top_h=0.9))]


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    fields = (r.stdout.strip().split(", ") + ["?"] * 3)[:3] if r.returncode == 0 else ["?"] * 3
    return {"device": torch.cuda.get_device_name(), "nvidia_smi_name": fields[0], "power_limit": fields[1],
            "max_sm_clock": fields[2]}


class _Graph:
    """``GRAPH_LAUNCHES`` calls of ``fn`` captured once; ``us(launches)`` is the time per call from CUDA events."""

    def __init__(self, fn):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn()
        torch.cuda.current_stream().wait_stream(s)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            for _ in range(GRAPH_LAUNCHES):
                fn()
        self.graph.replay()

    def us(self, launches):
        reps = max(1, launches // GRAPH_LAUNCHES)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            self.graph.replay()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / (reps * GRAPH_LAUNCHES)


def _baseline(path):
    # deep binding: the other build resolves its own kernels and CUDA runtime, not this build's same-named symbols
    lib = ctypes.CDLL(os.path.abspath(path), mode=os.RTLD_LOCAL | os.RTLD_DEEPBIND)
    p, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    lib.adapcc_sample_tokens.argtypes = [p, i, i, i, f, i, f] + [p] * 3 + [i, p, i, p, i] + [p] * 3 + [i, p]
    return lib


def bench_kernels(launches, rounds, baseline):
    from adapcc_b200.ops import sample_tokens_

    out = []
    for B in (1, 8, 64):
        g = torch.Generator(device="cuda").manual_seed(B)
        logits = torch.randn(B, VOCAB, device="cuda", generator=g) * 3
        seeds = torch.arange(B, dtype=torch.int64, device="cuda")
        pos = torch.zeros(B, dtype=torch.int32, device="cuda")
        step = torch.zeros(1, dtype=torch.int32, device="cuda")
        done = torch.zeros(B, dtype=torch.int32, device="cuda")
        nxt = torch.zeros(B, dtype=torch.int64, device="cuda")
        toks = torch.zeros(B, 1, dtype=torch.int64, device="cuda")     # step runs past max_new: nothing is written
        graphs = {}
        for name, f in FILTERS:
            graphs[name] = _Graph(lambda f=f: sample_tokens_(logits, VOCAB, 0.7, 0, 0.9, seeds, pos, step, 0, None,
                                                             None, done, nxt, toks, **f))
        if baseline is not None:
            ptr = [ctypes.c_void_p(t.data_ptr()) for t in (logits, seeds, pos, step, done, nxt, toks)]

            def old():
                rc = baseline.adapcc_sample_tokens(ptr[0], VOCAB, VOCAB, B, 0.7, 0, 0.9, ptr[1], ptr[2], ptr[3], 0,
                                                   None, 0, None, 0, ptr[4], ptr[5], ptr[6], 1,
                                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
                assert rc == 0, "baseline adapcc_sample_tokens failed"

            graphs["off, baseline library"] = _Graph(old)
        times = {name: [] for name in graphs}
        for _ in range(rounds):
            for name, gr in graphs.items():
                times[name].append(gr.us(launches))
        out.append({"batch": B, "us": {k: round(statistics.median(v), 2) for k, v in times.items()},
                    "spread_us": {k: round(max(v) - min(v), 2) for k, v in times.items()}})
    return out


def bench_generate(reps):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    g = torch.Generator(device="cuda").manual_seed(0)
    prompt = torch.randint(0, model.cfg.vocab_size, (8, 512), device="cuda", generator=g)
    kw = dict(max_new_tokens=NEW_TOKENS, temperature=0.7, top_k=0, top_p=0.9, seed=1)
    runs = {"top_p=0.9": {}, "top_p=0.9, typical_p=0.9": dict(typical_p=0.9)}
    times = {k: [] for k in runs}
    for f in runs.values():
        model.generate(prompt, **kw, **f)                           # warm-up
    for _ in range(reps):
        for name, f in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.generate(prompt, **kw, **f)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / NEW_TOKENS)
    return {"batch": 8, "prompt": 512, "new_tokens": NEW_TOKENS,
            "ms_per_token": {k: round(statistics.median(v), 3) for k, v in times.items()},
            "range_ms_per_token": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--launches", type=int, default=1000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--baseline-lib", default=None, help="another libadapcc.so whose adapcc_sample_tokens is timed too")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sample_filters_bench: needs a CUDA device")
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    baseline = _baseline(args.baseline_lib) if args.baseline_lib else None
    result = dict(_gpu_info(), vocab=VOCAB, kernels=bench_kernels(args.launches, args.rounds, baseline),
                  generate=bench_generate(args.reps))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
