#!/usr/bin/env python
"""Sampled GPT-2 small generation: the sequential sampling loop against ``GPT2DoubleHeads.generate``, and the LM-head
and sampling kernels on their own.

Prints one JSON line. Needs a CUDA device (there is no CPU fallback) and writes nothing into the repository.

* ``generate``: ms per generated token, prefill included (64 new tokens, bf16, seeded random weights), for
  (a) ``loop``: the body of ``sample_sequence`` at batch B (``DecodeGraph``, the fp32 copy of the tied head, torch
  top-k / sort-based top-p / multinomial), (b) ``generate``: one graph of decode step, bf16 LM head and sampler.
  Both build their graph inside the timed call, as a user's call does. B = 1 / 8 / 32, prompts of 128 / 512 tokens,
  ``top_p = 0.9`` and ``top_k = 20``. Each figure is the median of ``--reps`` timed runs after one warm-up run.
* ``kernels``: ``lm_head_logits_`` (GB/s over the bytes of W, and that over the H100 SXM's 3.35 TB/s) and
  ``sample_tokens_`` (top-p 0.9, vocab 50262) at B = 1 / 8 / 64, each captured 50 to a CUDA graph and timed with CUDA
  events over ``--launches`` launches.

Usage: ``python tools/generate_bench.py [--reps 5] [--launches 1000]``
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
GRAPH_LAUNCHES = 50
HBM_TBPS = 3.35


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return {"device": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power}


def _median_ms(fn, reps):
    fn()                                                           # warm-up of this shape
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def bench_generate(model, reps):
    from adapcc_b200.models.gpt2 import sample_sequence

    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8, 32):
        for T in (128, 512):
            prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
            for name, k, p in (("top_p=0.9", 0, 0.9), ("top_k=20", 20, 1.0)):
                kw = dict(max_new_tokens=NEW_TOKENS, temperature=0.7, top_k=k, top_p=p)
                gen = torch.Generator(device="cuda").manual_seed(1)
                loop = _median_ms(lambda: sample_sequence(model, prompt, None, generator=gen, **kw), reps)
                new = _median_ms(lambda: model.generate(prompt, seed=1, **kw), reps)
                rows.append({"batch": B, "prompt": T, "filter": name,
                             "loop_ms_per_token": round(loop / NEW_TOKENS, 3),
                             "generate_ms_per_token": round(new / NEW_TOKENS, 3),
                             "speedup": round(loop / new, 2)})
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


def bench_kernels(model, launches):
    from adapcc_b200.ops import lm_head_logits_, sample_tokens_

    W = model.wte.weight
    V, D = W.shape
    vocab = model.cfg.vocab_size
    rows = []
    for B in (1, 8, 64):
        g = torch.Generator(device="cuda").manual_seed(B)
        h = torch.randn(B, D, device="cuda", generator=g).to(torch.bfloat16)
        logits = torch.empty(B, V, dtype=torch.float32, device="cuda")
        us = _graph_us(lambda: lm_head_logits_(h, W, logits), launches)
        gbps = V * D * 2 / (us * 1e-6) / 1e9
        lm = {"us": round(us, 2), "GBps": round(gbps, 1), "share_of_3.35TBps": round(gbps / (HBM_TBPS * 1e3), 3)}
        logits.copy_(torch.randn(B, V, device="cuda", generator=g) * 3)
        seeds = torch.arange(B, dtype=torch.int64, device="cuda")
        pos = torch.zeros(B, dtype=torch.int32, device="cuda")
        step = torch.zeros(1, dtype=torch.int32, device="cuda")
        done = torch.zeros(B, dtype=torch.int32, device="cuda")
        nxt = torch.zeros(B, dtype=torch.int64, device="cuda")
        toks = torch.zeros(B, 1, dtype=torch.int64, device="cuda")     # step runs past max_new: nothing is written
        sus = {}
        for name, k, p in (("top_p=0.9", 0, 0.9), ("top_k=20", 20, 1.0)):
            sus[name] = round(_graph_us(lambda: sample_tokens_(logits, vocab, 0.7, k, p, seeds, pos, step, 0, None,
                                                               None, done, nxt, toks), launches), 2)
        rows.append({"batch": B, "lm_head": lm, "sample_us": sus})
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("generate_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, new_tokens=NEW_TOKENS, kernels=bench_kernels(model, args.launches),
                  generate=bench_generate(model, args.reps))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
