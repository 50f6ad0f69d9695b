#!/usr/bin/env python
"""GPT-2 small classifier-free guidance: ``generate(guidance_scale=1.5)`` against plain ``generate`` at B and at 2B rows,
and the guidance mix kernel on its own.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository.

* ``generate``: ms per generated token, prefill and graph capture included (64 new tokens, bf16, seeded random weights,
  temperature 0.7, top-p 0.9, no stop ids, so every call runs all 64 tokens), for B = 1 / 8 / 32 and prompts of 128 /
  512 tokens. The guided call's negative prompts are other prompts of the same length, so its 2B cache rows hold as
  many tokens as plain ``generate`` at 2B rows, which does the same decode-step and LM-head work; the difference is
  what guidance adds (the mix kernel and the id copy). Medians of ``--reps`` runs after one warm-up run, the three
  calls alternated run by run.
* ``kernel``: ``guidance_mix_`` (vocab 50257) at B = 1 / 8 / 32 row pairs, 50 launches captured in a CUDA graph and
  timed with CUDA events over ``--launches`` launches, next to ``lm_head_logits_`` at the same 2B rows. GB/s counts
  the least traffic the mix needs: both rows read once and the prompt row written once (the kernel reads both rows
  three times; the second and third reads mostly hit L2).

Usage: ``python tools/guidance_bench.py [--reps 3] [--launches 1000]``
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
SCALE = 1.5


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
    for B in (1, 8, 32):
        for T in (128, 512):
            prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
            neg = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
            calls = {"guided": lambda: model.generate(prompt, guidance_scale=SCALE, negative_prompt_ids=neg, **kw),
                     "plain_B": lambda: model.generate(prompt, **kw),
                     "plain_2B": lambda: model.generate(torch.cat([prompt, neg]), **kw)}
            times = {k: [] for k in calls}
            for k, fn in calls.items():                            # warm-up of each shape
                fn()
            for _ in range(reps):
                for k, fn in calls.items():
                    times[k].append(_time_ms(fn))
            ms = {k: statistics.median(v) / NEW_TOKENS for k, v in times.items()}
            rows.append({"batch": B, "prompt": T,
                         "guided_ms_per_token": round(ms["guided"], 3),
                         "plain_B_ms_per_token": round(ms["plain_B"], 3),
                         "plain_2B_ms_per_token": round(ms["plain_2B"], 3),
                         "guidance_cost_ms_per_token": round(ms["guided"] - ms["plain_2B"], 3)})
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
    from adapcc_b200.ops import guidance_mix_, lm_head_logits_

    cfg, W = model.cfg, model.wte.weight
    V = cfg.vocab_size
    g = torch.Generator(device="cuda").manual_seed(1)
    out = []
    for B in (1, 8, 32):
        h = torch.randn(2 * B, cfg.n_embd, device="cuda", generator=g).to(torch.bfloat16)
        logits = torch.empty(2 * B, W.shape[0], dtype=torch.float32, device="cuda")
        lm_us = _graph_us(lambda: lm_head_logits_(h, W, logits), launches)
        # repeated mixes rewrite the prompt rows with scores of the same range: every launch does the same work
        logits.copy_(torch.randn(2 * B, W.shape[0], device="cuda", generator=g) * 3)
        mix_us = _graph_us(lambda: guidance_mix_(logits, V, B, SCALE), launches)
        moved = 3 * B * V * 4
        out.append({"batch": B, "rows": 2 * B, "mix_us": round(mix_us, 2), "lm_head_us": round(lm_us, 2),
                    "mix_GBps_min_traffic": round(moved / (mix_us * 1e-6) / 1e9, 1)})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("guidance_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, new_tokens=NEW_TOKENS, scale=SCALE, kernel=bench_kernel(model, args.launches),
                  generate=bench_generate(model, args.reps))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
