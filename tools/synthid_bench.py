#!/usr/bin/env python
"""GPT-2 SynthID Text watermarking: the sampler step with and without the tournament, ``generate`` with and without
it, the detector kernel, and the scores of watermarked replies.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository.

* ``sampler``: one ``sample_tokens_`` call (vocab 50257, fp32 logits, temperature 1, generated step 64 of a
  1024-column reply buffer) at B = 1 / 8 / 64 rows, with top-k 50 and with every id kept (top-k 0, top-p 1), SynthID
  off and on at m = 9 and m = 30 layers (n = 5). Each call is preceded by a one-thread reset of the step counter (the
  same in every variant); CUDA events over ``--launches`` calls, after warm-up, report µs per call.
* ``generate``: ms per generated token (64 new tokens, 128-token prompts, bf16, seeded random weights, temperature
  0.7, top-p 0.9, no stop ids), prefill and graph capture included, for B = 8 / 64, SynthID off and on (m = 9, n =
  5). Medians of ``--reps`` runs after one warm-up run, the calls alternated run by run.
* ``count``: ``synthid_count_`` on 64 rows of 1024 ids (m = 9 and 30, H = 1024), µs per call.
* ``scores``: the mean score, mean weighted score and mean z of 64 sampled replies of 64 tokens (temperature 1, top-p
  1, m = 9 and 30), scored on their own, and the same without the watermark.

Usage: ``python tools/synthid_bench.py [--reps 3] [--launches 200]``
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

V, LD = 50257, 50304
NEW_TOKENS = 64
KEYS30 = [int(k) for k in np.random.default_rng(0).integers(-2 ** 63, 2 ** 63, 30)]
CONFIGS = {"m9": dict(ngram_len=5, keys=KEYS30[:9]), "m30": dict(ngram_len=5, keys=KEYS30)}


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return {"device": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power}


def _events_us(fn, launches):
    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches


def bench_sampler(dev, launches):
    from adapcc_b200.ops import sample_tokens_

    out = {}
    g = torch.Generator(device=dev).manual_seed(0)
    for B in (1, 8, 64):
        logits = torch.randn(B, LD, device=dev, generator=g) * 2
        tokens = torch.randint(0, V, (B, 1024), device=dev, generator=g)
        seeds = torch.arange(B, dtype=torch.int64, device=dev)
        pos = torch.full((B,), 100, dtype=torch.int32, device=dev)
        step = torch.zeros(1, dtype=torch.int32, device=dev)
        done = torch.zeros(B, dtype=torch.int32, device=dev)
        nxt = torch.zeros(B, dtype=torch.int64, device=dev)
        for filt, (k, p) in (("top_k50", (50, 1.0)), ("all_kept", (0, 1.0))):
            for name, cfg in (("off", None),) + tuple(CONFIGS.items()):
                def call(cfg=cfg, k=k, p=p):
                    step.fill_(NEW_TOKENS)
                    sample_tokens_(logits, V, 1.0, k, p, seeds, pos, step, 0, None, None, done, nxt, tokens,
                                   synthid=cfg)
                out[f"B{B}_{filt}_{name}_us"] = round(_events_us(call, launches), 2)
    return out


def bench_generate(model, dev, reps):
    out = {}
    for B in (8, 64):
        g = torch.Generator(device=dev).manual_seed(B)
        ids = torch.randint(0, 300, (B, 128), device=dev, generator=g)
        kw = dict(max_new_tokens=NEW_TOKENS, temperature=0.7, top_p=0.9, seed=1)
        runs = {"off": [], "on": []}
        for name, cfg in (("off", None), ("on", CONFIGS["m9"])):
            model.generate(ids, **kw, watermarking_config=cfg)          # warm-up
        for _ in range(reps):
            for name, cfg in (("off", None), ("on", CONFIGS["m9"])):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model.generate(ids, **kw, watermarking_config=cfg)
                torch.cuda.synchronize()
                runs[name].append((time.perf_counter() - t0) * 1e3 / NEW_TOKENS)
        for name, v in runs.items():
            out[f"B{B}_{name}_ms_per_token"] = round(statistics.median(v), 4)
            out[f"B{B}_{name}_runs"] = [round(x, 4) for x in v]
    return out


def bench_count(dev, launches):
    from adapcc_b200.ops import synthid_count_

    out = {}
    g = torch.Generator(device=dev).manual_seed(3)
    B, T = 64, 1024
    ids = torch.randint(0, V, (B, T), device=dev, generator=g, dtype=torch.int32)
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    start = torch.zeros(B, dtype=torch.int32, device=dev)
    for name, cfg in CONFIGS.items():
        o = torch.empty(B, 1 + len(cfg["keys"]), dtype=torch.int32, device=dev)
        out[f"{name}_us"] = round(_events_us(lambda cfg=cfg, o=o: synthid_count_(ids, lens, start, cfg, out=o),
                                             launches), 2)
    return out


def bench_scores(model, dev):
    from adapcc_b200.ops.synthid import detect_synthid

    out = {}
    g = torch.Generator(device=dev).manual_seed(9)
    ids = torch.randint(0, 300, (64, 16), device=dev, generator=g)
    kw = dict(max_new_tokens=NEW_TOKENS, temperature=1.0, top_p=1.0, seed=5)
    for name, cfg in CONFIGS.items():
        for mark in ("on", "off"):
            tokens, _ = model.generate(ids, **kw, watermarking_config=cfg if mark == "on" else None)
            det = detect_synthid(tokens, cfg, z_threshold=4.0)
            out[f"{name}_{mark}"] = {"mean_score": round(float(np.nanmean(det.mean_score)), 4),
                                     "weighted_mean_score": round(float(np.nanmean(det.weighted_mean_score)), 4),
                                     "mean_z": round(float(np.nanmean(det.z_score)), 2),
                                     "flagged_z4": int(det.prediction.sum())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("synthid_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device=dev, dtype=torch.bfloat16).eval()
    res = {"gpu": _gpu_info(), "sampler": bench_sampler(dev, args.launches),
           "count": bench_count(dev, args.launches), "generate": bench_generate(model, dev, args.reps),
           "scores": bench_scores(model, dev)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
