#!/usr/bin/env python
"""GPT-2 small DoLa layer contrast: ``generate(dola_layers=...)`` against plain ``generate``, and the two DoLa kernels
on their own.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository.

* ``generate``: ms per generated token, prefill and graph capture included (64 new tokens, bf16, seeded random weights,
  128-token prompts, temperature 0.7, top-p 0.9, no stop ids, so every call runs all 64 tokens), with DoLa off,
  ``"low"`` and ``"high"`` (three candidate layers each) at B = 1 / 8 / 16 / 64. DoLa runs the LM head on 4B rows
  instead of B, in launches of at most 64 rows. Medians of ``--reps`` runs after one warm-up run, the three calls
  alternated run by run.
* ``kernel``: ``dola_contrast_`` (vocab 50257; the divergence and the contrast kernel) at the same B with 1 and 3
  candidates, 50 launches captured in a CUDA graph and timed with CUDA events over ``--launches`` launches, next to
  ``lm_head_logits_`` on 64 rows. GB/s counts the least traffic the two kernels need: every one of the (1 + C)·B rows
  read once and the B final rows written once.

Usage: ``python tools/dola_bench.py [--reps 3] [--launches 1000]``
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

NEW_TOKENS = 64
PROMPT = 128
GRAPH_LAUNCHES = 50
BATCHES = (1, 8, 16, 64)


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return {"device": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power}


def _time_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def bench_generate(model, reps):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    kw = dict(max_new_tokens=NEW_TOKENS, temperature=0.7, top_p=0.9)
    for B in BATCHES:
        prompt = torch.randint(0, model.cfg.vocab_size, (B, PROMPT), device="cuda", generator=g)
        calls = {"off": lambda: model.generate(prompt, **kw),
                 "low": lambda: model.generate(prompt, dola_layers="low", **kw),
                 "high": lambda: model.generate(prompt, dola_layers="high", **kw)}
        times = {k: [] for k in calls}
        for fn in calls.values():                                  # warm-up of each shape
            fn()
        for _ in range(reps):
            for k, fn in calls.items():
                times[k].append(_time_ms(fn))
        ms = {k: statistics.median(v) / NEW_TOKENS for k, v in times.items()}
        rows.append({"batch": B, **{f"{k}_ms_per_token": round(v, 3) for k, v in ms.items()},
                     "spread_ms_per_token": round(max(max(v) - min(v) for v in times.values()) / NEW_TOKENS, 3)})
    return rows


def _graph_us(fn, launches):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(GRAPH_LAUNCHES):
            fn()
    graph.replay()
    reps = max(1, launches // GRAPH_LAUNCHES)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * GRAPH_LAUNCHES)


def bench_kernel(model, launches):
    from adapcc_b200.ops import dola_contrast_, dola_work_numel, lm_head_logits_

    cfg, W = model.cfg, model.wte.weight
    V = cfg.vocab_size
    g = torch.Generator(device="cuda").manual_seed(1)
    h = torch.randn(64, cfg.n_embd, device="cuda", generator=g).to(torch.bfloat16)
    head_out = torch.empty(64, W.shape[0], dtype=torch.float32, device="cuda")
    out = [{"lm_head_64_rows_us": round(_graph_us(lambda: lm_head_logits_(h, W, head_out), launches), 2)}]
    for B in BATCHES:
        for C in (1, 3):
            logits = torch.randn((1 + C) * B, W.shape[0], device="cuda", generator=g) * 3
            work = torch.empty(dola_work_numel(B, C), dtype=torch.float32, device="cuda")
            # repeated launches rewrite the final rows with scores and -inf: the passes still read every id, the
            # work stays the same in each launch
            us = _graph_us(lambda: dola_contrast_(logits, V, B, C, work), launches)
            moved = ((1 + C) * B + B) * V * 4
            out.append({"batch": B, "candidates": C, "dola_us": round(us, 2),
                        "GBps_min_traffic": round(moved / (us * 1e-6) / 1e9, 1)})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dola_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, new_tokens=NEW_TOKENS, prompt=PROMPT, kernel=bench_kernel(model, args.launches),
                  generate=bench_generate(model, args.reps))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
