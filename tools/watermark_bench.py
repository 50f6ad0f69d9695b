#!/usr/bin/env python
"""GPT-2 green-list watermarking: the bias kernel, the detector kernel, ``generate`` with and without the watermark,
and the mean z-score the watermark gives.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository.

* ``kernel``: ``watermark_`` (vocab 50257, every row's sequence 512 ids long) at R = 1 / 8 / 32 / 64 rows, for
  lefthash w = 1 and selfhash w = 4, 50 launches captured in a CUDA graph and timed with CUDA events over
  ``--launches`` launches, next to ``lm_head_logits_`` at the same rows. ``bound_us`` is R·V·8 bytes (every logit read
  and written once) over the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s, and ``share_of_bound`` that bound over
  the kernel time. The kernel reads and writes only the green logits, so it can beat the bound when it is not
  compute-bound.
* ``count``: ``watermark_count_`` on 64 rows of 1024 ids, both schemes, with and without ``ignore_repeated_ngrams``.
* ``generate``: ms per generated token (64 new tokens, 128-token prompts, bf16, seeded random weights, temperature
  0.7, top-p 0.9, no stop ids), prefill and graph capture included, for B = 1 / 8 / 64, watermark off and on
  (lefthash w = 1, δ = 2). Medians of ``--reps`` runs after one warm-up run, the calls alternated run by run.
* ``z``: the mean z-score of 64 sampled replies of 64 tokens (their prompts as context, not scored) for δ = 1, 2, 4,
  γ = 0.25, temperature 1, with ``no_repeat_ngram_size=1`` (seeded random GPT-2 small otherwise repeats the ids
  already in its context).

Usage: ``python tools/watermark_bench.py [--reps 3] [--launches 1000]``
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
HBM_BYTES_PER_S = 3.35e12
SCHEMES = {"lefthash_w1": dict(seeding_scheme="lefthash", context_width=1),
           "selfhash_w4": dict(seeding_scheme="selfhash", context_width=4)}


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
    from adapcc_b200.ops import lm_head_logits_, watermark_

    cfg, W = model.cfg, model.wte.weight
    V = cfg.vocab_size
    g = torch.Generator(device="cuda").manual_seed(1)
    out = []
    for R in (1, 8, 32, 64):
        h = torch.randn(R, cfg.n_embd, device="cuda", generator=g).to(torch.bfloat16)
        logits = torch.empty(R, W.shape[0], dtype=torch.float32, device="cuda")
        lm_us = _graph_us(lambda: lm_head_logits_(h, W, logits), launches)
        seq = torch.randint(0, V, (R, 1024), dtype=torch.int32, device="cuda", generator=g)
        lens = torch.full((R,), 512, dtype=torch.int32, device="cuda")
        bound_us = R * V * 8 / HBM_BYTES_PER_S * 1e6
        row = {"rows": R, "lm_head_us": round(lm_us, 2), "bound_us": round(bound_us, 2)}
        for name, scheme in SCHEMES.items():
            wm = dict(scheme, bias=2.0)
            us = _graph_us(lambda: watermark_(logits, V, seq, lens, wm), launches)
            row[name] = {"us": round(us, 2), "share_of_bound": round(bound_us / us, 3)}
        out.append(row)
    return out


def bench_count(launches):
    from adapcc_b200.ops import watermark_count_

    g = torch.Generator(device="cuda").manual_seed(2)
    B, T = 64, 1024
    ids = torch.randint(0, 50257, (B, T), dtype=torch.int32, device="cuda", generator=g)
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    start = torch.zeros(B, dtype=torch.int32, device="cuda")
    counts = torch.empty(B, 2, dtype=torch.int32, device="cuda")
    out = {"rows": B, "ids_per_row": T}
    for name, scheme in SCHEMES.items():
        for ignore in (False, True):
            us = _graph_us(lambda: watermark_count_(ids, lens, start, scheme, ignore, out=counts), launches)
            out[f"{name}{'_ignore_repeated' if ignore else ''}_us"] = round(us, 2)
    return out


def bench_generate(model, reps):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    kw = dict(max_new_tokens=NEW_TOKENS, temperature=0.7, top_p=0.9)
    wm = dict(bias=2.0)
    for B in (1, 8, 64):
        prompt = torch.randint(0, model.cfg.vocab_size, (B, 128), device="cuda", generator=g)
        calls = {"off": lambda: model.generate(prompt, **kw),
                 "on": lambda: model.generate(prompt, watermarking_config=wm, **kw)}
        times = {k: [] for k in calls}
        for fn in calls.values():                                  # warm-up of each shape
            fn()
        for _ in range(reps):
            for k, fn in calls.items():
                times[k].append(_time_ms(fn))
        ms = {k: statistics.median(v) / NEW_TOKENS for k, v in times.items()}
        rows.append({"batch": B, "off_ms_per_token": round(ms["off"], 4), "on_ms_per_token": round(ms["on"], 4),
                     "cost_ms_per_token": round(ms["on"] - ms["off"], 4)})
    return rows


def bench_z(model):
    from adapcc_b200.ops.watermark import detect_watermark

    g = torch.Generator(device="cuda").manual_seed(3)
    B, T = 64, 32
    prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
    out = []
    for delta in (1.0, 2.0, 4.0):
        wm = dict(bias=delta, greenlist_ratio=0.25)
        tokens, n_new = model.generate(prompt, max_new_tokens=NEW_TOKENS, temperature=1.0, top_p=1.0, seed=5,
                                       no_repeat_ngram_size=1, watermarking_config=wm)
        ids = torch.cat([prompt, tokens.clamp(min=0)], 1)
        det = detect_watermark(ids, wm, lengths=(T + n_new).tolist(), scored_from=T)
        out.append({"delta": delta, "mean_z": round(float(det.z_score.mean()), 3),
                    "min_z": round(float(det.z_score.min()), 3), "detected": float(det.prediction.mean())})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("watermark_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, kernel=bench_kernel(model, args.launches), count=bench_count(args.launches),
                  generate=bench_generate(model, args.reps), z=bench_z(model))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
