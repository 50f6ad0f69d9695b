#!/usr/bin/env python
"""GPT-2 small repetition controls: the ``penalize_repeats_`` kernel on its own, and ``generate`` / ``beam_search`` per
token with and without ``repetition_penalty`` and ``no_repeat_ngram_size``.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository.

* ``kernel``: ``penalize_repeats_`` (vocab 50257, ld 50304, n = 3, p = 1.2) at R = 1 / 8 / 64 rows and sequences of
  128 / 512 / 1024 ids, with a step counter > 0, so every launch also appends a token; ``reorder`` adds a parent map
  that moves every row's 64 generated ids within groups of min(R, 8) rows (the beam-search case). 50 launches captured
  in a CUDA graph, timed with CUDA events over ``--launches`` launches. Next to it, the LM head and ``beam_step_`` at
  64 rows, the two launches the kernel sits between.
* ``decode``: ms per generated token, prefill and graph capture included (GPT-2 small, bf16, seeded random weights,
  prompt 512, 64 new tokens, no stop ids, so every call runs all 64 tokens), for ``generate`` (top_p 0.9) and
  ``beam_search`` (4 beams) at 8 and 64 rows, with both controls off and on (p = 1.2, n = 3), the two alternated in one
  process. Medians of ``--reps`` runs after one warm-up run of each.

Usage: ``python tools/repeats_bench.py [--reps 5] [--launches 1000]``
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
PROMPT = 512
GRAPH_LAUNCHES = 50
P, N = 1.2, 3


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return {"device": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power}


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
    from adapcc_b200.ops import BeamState, beam_step_, lm_head_logits_, penalize_repeats_

    V, W = model.cfg.vocab_size, model.wte.weight
    g = torch.Generator(device="cuda").manual_seed(1)
    i32 = dict(dtype=torch.int32, device="cuda")
    rows = []
    for R in (1, 8, 64):
        logits = torch.randn(R, W.shape[0], device="cuda", generator=g) * 3
        ids = torch.randint(0, V, (R,), device="cuda", generator=g)
        step = torch.ones(1, **i32)
        for L in (128, 512, 1024):
            seq = torch.randint(0, 2000, (R, 1024), device="cuda", generator=g).to(torch.int32)
            lens = torch.full((R,), L, **i32)
            prompt_len = lens - 64
            K = min(R, 8)
            parent = (torch.arange(R, **i32).view(-1, K).roll(1, 1) if K > 1 else torch.arange(R, **i32)).flatten()
            entry = {"rows": R, "seq_len": L}
            for name, par, grp in (("plain", None, 1), ("reorder", parent.contiguous(), K)):
                us = _graph_us(lambda: penalize_repeats_(logits, V, seq, prompt_len, lens, step, ids, par, grp, P, N),
                               launches)
                entry[f"{name}_us"] = round(us, 2)
            rows.append(entry)
    h = torch.randn(64, model.cfg.n_embd, device="cuda", generator=g).to(torch.bfloat16)
    logits = torch.empty(64, W.shape[0], dtype=torch.float32, device="cuda")
    lm_us = _graph_us(lambda: lm_head_logits_(h, W, logits), launches)
    logits.copy_(torch.randn(64, W.shape[0], device="cuda", generator=g) * 3)
    st = BeamState(8, 8, launches + 4 * GRAPH_LAUNCHES, 1.0, "cuda")
    st.scores.zero_()
    step_us = _graph_us(lambda: beam_step_(logits, V, st), launches)
    return {"p": P, "n": N, "per_config": rows, "lm_head_64_rows_us": round(lm_us, 2),
            "beam_step_64_rows_us": round(step_us, 2)}


def _ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def bench_decode(model, reps):
    V = model.cfg.vocab_size
    g = torch.Generator(device="cuda").manual_seed(0)
    out = []
    for mode, rows in (("generate", 8), ("generate", 64), ("beam_search", 8), ("beam_search", 64)):
        B = rows if mode == "generate" else rows // 4
        prompt = torch.randint(0, V, (B, PROMPT), device="cuda", generator=g)

        def run(on):
            kw = dict(repetition_penalty=P, no_repeat_ngram_size=N) if on else {}
            if mode == "generate":
                return lambda: model.generate(prompt, max_new_tokens=NEW_TOKENS, seed=3, **kw)
            return lambda: model.beam_search(prompt, num_beams=4, max_new_tokens=NEW_TOKENS, **kw)

        off_fn, on_fn = run(False), run(True)
        off_fn()
        on_fn()
        times = {False: [], True: []}
        for _ in range(reps):                                       # alternated, so drift hits both alike
            times[False].append(_ms(off_fn))
            times[True].append(_ms(on_fn))
        off, on = statistics.median(times[False]), statistics.median(times[True])
        out.append({"mode": mode, "rows": rows, "off_ms_per_token": round(off / NEW_TOKENS, 3),
                    "on_ms_per_token": round(on / NEW_TOKENS, 3),
                    "cost_ms_per_token": round((on - off) / NEW_TOKENS, 3),
                    "off_range_ms_per_token": [round(min(times[False]) / NEW_TOKENS, 3),
                                               round(max(times[False]) / NEW_TOKENS, 3)],
                    "on_range_ms_per_token": [round(min(times[True]) / NEW_TOKENS, 3),
                                              round(max(times[True]) / NEW_TOKENS, 3)]})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("repeats_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, new_tokens=NEW_TOKENS, prompt=PROMPT, kernel=bench_kernel(model, args.launches),
                  decode=bench_decode(model, args.reps))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
