#!/usr/bin/env python
"""GPT-2 small assisted generation: ``generate(assistant_model=draft, num_assistant_tokens=k)`` against plain
``generate`` with the same arguments (bf16, no stop ids), with the mean tokens per verify step of each assisted call.

Two times per configuration, in ms per generated token: ``e2e`` for a call of 64 new tokens (prefill and graph capture
included), and ``steady`` = (time of a 192-token call - time of a 64-token call) / 128, where the prefill and the
capture cancel, so it is the cost of the replays alone (every row runs to the end: there are no stop ids).

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device and writes nothing
into the repository. The weights are seeded random ones, so the acceptance seen here says nothing about trained models;
the drafts bound it instead:

* ``self``: the target itself, the acceptance ceiling;
* ``cut``: the target's first two blocks with its wte / wpe / ln_f;
* ``other``: an independently seeded two-block model, whose acceptance is about zero: the pure overhead.

B = 1 / 8 rows, prompts of 128 / 512 random tokens, k = 2 / 4 / 7, greedy (temperature 0) and sampled (temperature 0.7,
top-p 0.9). Plain and assisted calls are alternated in one process; medians of ``--reps`` calls after one warm-up call
per configuration and length.

Usage: ``python tools/assist_bench.py [--reps 3]``
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
LONG_TOKENS = 192
KS = (2, 4, 7)
MODES = {"greedy": dict(temperature=0.0), "sampled": dict(temperature=0.7, top_p=0.9)}


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return {"device": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power}


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def _drafts(target):
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads

    cut = GPT2DoubleHeads(GPT2Config(n_layer=2)).to(device="cuda", dtype=torch.bfloat16).eval()
    cut.load_state_dict({k: v for k, v in target.state_dict().items()
                         if not k.startswith("h.") or k.split(".")[1] in ("0", "1")})
    torch.manual_seed(77)
    other = GPT2DoubleHeads(GPT2Config(n_layer=2)).to(device="cuda", dtype=torch.bfloat16).eval()
    return {"self": target, "cut": cut, "other": other}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    drafts = _drafts(model)
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for B in (1, 8):
        for T in (128, 512):
            prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
            for mode, kw in MODES.items():
                cfgs = [None] + [(name, k) for name in drafts for k in KS]
                times = {(c, m): [] for c in cfgs for m in (NEW_TOKENS, LONG_TOKENS)}
                per_step = {c: [] for c in cfgs}
                for rep in range(args.reps + 1):                 # rep 0 warms every configuration up
                    for c in cfgs:
                        extra = {} if c is None else dict(assistant_model=drafts[c[0]], num_assistant_tokens=c[1])
                        for m in (NEW_TOKENS, LONG_TOKENS):
                            ms = _timed(lambda: model.generate(prompt, max_new_tokens=m, seed=1, **kw, **extra))
                            if rep:
                                times[(c, m)].append(ms)
                            if rep and c is not None and m == LONG_TOKENS:
                                st = model.assist_stats
                                per_step[c].append(float((st["emitted"] - 1).sum()) / max(1, int(st["steps"].sum())))

                def cost(c):
                    short, long_ = statistics.median(times[(c, NEW_TOKENS)]), statistics.median(times[(c, LONG_TOKENS)])
                    return short / NEW_TOKENS, (long_ - short) / (LONG_TOKENS - NEW_TOKENS)

                plain_e2e, plain_steady = cost(None)
                for c in cfgs[1:]:
                    e2e, steady = cost(c)
                    rows.append({"B": B, "T": T, "mode": mode, "draft": c[0], "k": c[1],
                                 "plain_e2e_ms_per_token": round(plain_e2e, 4), "e2e_ms_per_token": round(e2e, 4),
                                 "plain_steady_ms_per_token": round(plain_steady, 4),
                                 "steady_ms_per_token": round(steady, 4),
                                 "steady_speedup": round(plain_steady / steady, 3),
                                 "tokens_per_step": round(statistics.median(per_step[c]), 3)})
                    print(json.dumps(rows[-1]), file=sys.stderr)
    print(json.dumps({"gpu": _gpu_info(), "new_tokens": [NEW_TOKENS, LONG_TOKENS], "reps": args.reps,
                      "generate": rows}))


if __name__ == "__main__":
    main()
