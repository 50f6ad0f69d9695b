#!/usr/bin/env python
"""GPT-2 small sequence bias and bad words: rule 0 of the ``penalize_repeats_`` kernel on its own, and ``generate`` /
``beam_search`` per token with and without a bad-word list.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository.

* ``kernel``: ``penalize_repeats_`` with only the sequence bias on (vocab 50257, ld 50304, sequences of 512 ids, a
  step counter > 0, so every launch also appends a token) at R = 1 / 8 / 64 rows, with 0, 64 and 1024 entries of 1
  to 4 ids (a quarter of them bad words, targets spread over the vocabulary). 0 entries is the launch with every
  rule off. 50 launches captured in a CUDA graph, timed with CUDA events over ``--launches`` launches.
* ``decode``: ms per generated token, prefill and graph capture included (GPT-2 small, bf16, seeded random weights,
  prompt 512, 64 new tokens, no stop ids, so every call runs all 64 tokens), for ``generate`` (top_p 0.9) at 8 rows
  and ``beam_search`` (4 beams) at 8 items, with no bad words and with 256 bad words of 1 to 3 ids, the two
  alternated in one process. Medians of ``--reps`` runs after one warm-up run of each.

Usage: ``python tools/sequence_bias_bench.py [--reps 5] [--launches 1000]``
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.dont_write_bytecode = True                          # the tree may be read-only: no __pycache__ for repeats_bench

import numpy as np  # noqa: E402
import torch  # noqa: E402
from repeats_bench import NEW_TOKENS, PROMPT, _gpu_info, _graph_us, _ms  # noqa: E402

SEQ_LEN = 512


def _entries(rng, n, V):
    """``n`` distinct entries of 1 to 4 ids: ``(sequence_bias dict, bad_words_ids)``, a quarter of them bad words."""
    sb, bad, seen = {}, [], set()
    while len(sb) + len(bad) < n:
        s = tuple(int(x) for x in rng.integers(0, V, int(rng.integers(1, 5))))
        if s in seen:
            continue
        seen.add(s)
        if len(bad) < n // 4:
            bad.append(list(s))
        else:
            sb[s] = float(rng.standard_normal())
    return sb, bad


def bench_kernel(V, LD, launches):
    from adapcc_b200.ops import penalize_repeats_
    from adapcc_b200.ops.repeats import check_sequence_bias_args

    g = torch.Generator(device="cuda").manual_seed(1)
    rng = np.random.default_rng(1)
    i32 = dict(dtype=torch.int32, device="cuda")
    rows = []
    for R in (1, 8, 64):
        logits = torch.randn(R, LD, device="cuda", generator=g) * 3
        ids = torch.randint(0, V, (R,), device="cuda", generator=g)
        step = torch.ones(1, **i32)
        seq = torch.randint(0, V, (R, 1024), device="cuda", generator=g).to(torch.int32)
        lens = torch.full((R,), SEQ_LEN, **i32)
        prompt_len = lens - 64
        entry = {"rows": R}
        for n in (0, 64, 1024):
            table = check_sequence_bias_args("bench", *_entries(rng, n, V), V) if n else None
            us = _graph_us(lambda: penalize_repeats_(logits, V, seq, prompt_len, lens, step, ids, None, 1, 1.0, 0,
                                                     table), launches)
            entry[f"entries_{n}_us"] = round(us, 2)
        rows.append(entry)
    return {"seq_len": SEQ_LEN, "per_config": rows}


def bench_decode(model, reps):
    V = model.cfg.vocab_size
    g = torch.Generator(device="cuda").manual_seed(0)
    _, bad = _entries(np.random.default_rng(2), 1024, V)
    bad = [w[:3] for w in bad[:256]]
    out = []
    for mode, rows in (("generate", 8), ("beam_search", 32)):
        B = rows if mode == "generate" else rows // 4
        prompt = torch.randint(0, V, (B, PROMPT), device="cuda", generator=g)

        def run(on):
            kw = dict(bad_words_ids=bad) if on else {}
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
        out.append({"mode": mode, "rows": rows, "bad_words": len(bad),
                    "off_ms_per_token": round(off / NEW_TOKENS, 3), "on_ms_per_token": round(on / NEW_TOKENS, 3),
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
        sys.exit("sequence_bias_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, new_tokens=NEW_TOKENS, prompt=PROMPT,
                  kernel=bench_kernel(model.cfg.vocab_size, model.wte.weight.shape[0], args.launches),
                  decode=bench_decode(model, args.reps))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
