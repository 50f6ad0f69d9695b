#!/usr/bin/env python
"""GPT-2 small prompt-lookup decoding: ``generate(temperature=0, prompt_lookup_num_tokens=k)`` against plain greedy
``generate``, one verify step against one decode step, and the lookup kernels alone.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository. The weights are seeded random ones, so the acceptance seen here says
nothing about trained GPT-2; the step costs give the speed-up for any acceptance.

* ``generate``: ms per generated token, prefill and graph capture included (64 new tokens, bf16, no stop ids), for
  B = 1 / 8 rows, prompts of 128 / 512 random tokens, and k off / 2 / 4 / 7, the modes alternated call by call in one
  process. Medians of ``--reps`` calls after one warm-up call per mode. With each lookup result: the mean tokens per
  verify step and the replays issued after the last row finished (the early-stop poll's overshoot) at that median
  call, and the same two numbers for poll periods 2, 4 and 8 at B = 8, T = 128.
* ``steps``: one verify step (the model on B·(k+1) slots and the LM head on them) against one decode step (the model
  on B rows and the LM head), both replayed from CUDA graphs of 50 steps at 128 / 512 cached tokens.
* ``kernels`` (one layer of GPT-2 small, 12 heads of 64, 8 rows, 128 / 512 cached tokens): ``verify_attention_``
  against k + 1 sequential ``decode_attention_`` launches, and ``lookup_argmax_`` + ``lookup_accept_`` +
  ``lookup_draft_`` after a verify step (each launch also restores 8 lengths). 50 launches captured in a CUDA graph,
  timed with CUDA events over ``--launches`` launches.

Usage: ``python tools/lookup_bench.py [--reps 5] [--launches 1000]``
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
KS = (2, 4, 7)


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return {"device": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power}


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def _stats(model):
    st = model.lookup_stats
    steps = st["steps"]
    return {"tokens_per_step": round(float((st["emitted"] - 1).sum()) / max(1, int(steps.sum())), 3),
            "replays_after_last_row": int(st["replays"]) - int(steps.max())}


def bench_generate(model, reps):
    import adapcc_b200.models.gpt2 as gpt2

    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8):
        for T in (128, 512):
            prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
            modes = (0,) + KS
            times = {k: [] for k in modes}
            stats = {k: [] for k in modes}
            for rep in range(reps + 1):                             # rep 0 warms every mode up
                for k in modes:
                    ms, _ = _timed(lambda: model.generate(prompt, max_new_tokens=NEW_TOKENS, temperature=0.0,
                                                          prompt_lookup_num_tokens=k))
                    if rep:
                        times[k].append(ms)
                        stats[k].append(_stats(model) if k else {})
            greedy = statistics.median(times[0]) / NEW_TOKENS
            for k in KS:
                med = sorted(range(reps), key=lambda i: times[k][i])[reps // 2]
                rows.append(dict({"batch": B, "prompt": T, "k": k,
                                  "lookup_ms_per_token": round(times[k][med] / NEW_TOKENS, 4),
                                  "greedy_ms_per_token": round(greedy, 4)}, **stats[k][med]))
    # the early-stop poll period of the lookup path
    prompt = torch.randint(0, model.cfg.vocab_size, (8, 128), device="cuda", generator=g)
    periods = []
    default = gpt2.LOOKUP_POLL_PERIOD
    try:
        for period in (2, 4, 8):
            gpt2.LOOKUP_POLL_PERIOD = period
            for k in KS:
                model.generate(prompt, max_new_tokens=NEW_TOKENS, temperature=0.0, prompt_lookup_num_tokens=k)
                ts = []
                for _ in range(reps):
                    ms, _ = _timed(lambda: model.generate(prompt, max_new_tokens=NEW_TOKENS, temperature=0.0,
                                                          prompt_lookup_num_tokens=k))
                    ts.append(ms)
                periods.append(dict({"period": period, "k": k,
                                     "ms_per_token": round(statistics.median(ts) / NEW_TOKENS, 4)}, **_stats(model)))
    finally:
        gpt2.LOOKUP_POLL_PERIOD = default
    return rows, periods


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


@torch.no_grad()
def bench_steps(model, launches):
    from adapcc_b200.models.gpt2 import VerifyKV
    from adapcc_b200.ops import decode_attention_work_numel, lm_head_logits_

    cfg, W = model.cfg, model.wte.weight
    H, Dh = cfg.n_head, cfg.n_embd // cfg.n_head
    out = []
    for B in (1, 8):
        for T in (128, 512):
            t_max = T + NEW_TOKENS
            cache = model.new_cache(B, t_max)
            model.hidden(torch.randint(0, cfg.vocab_size, (B, T), device="cuda"), None, cache=cache)
            lens0 = cache.lens.clone()
            ids = torch.randint(0, cfg.vocab_size, (B,), device="cuda")
            logits = torch.empty(B * (max(KS) + 1), W.shape[0], dtype=torch.float32, device="cuda")

            def decode():
                cache.lens.copy_(lens0)
                h = model._blocks(model._embed(ids, None, cache.lens.long()), cache)
                lm_head_logits_(h, W, logits[:B])

            row = {"batch": B, "cached": T, "decode_step_us": round(_graph_us(decode, launches), 1)}
            for k in KS:
                S = k + 1
                work = torch.empty(decode_attention_work_numel(B * S, H, Dh, t_max), dtype=torch.float32,
                                   device="cuda")
                nq = torch.full((B,), S, dtype=torch.int32, device="cuda")
                vids = torch.randint(0, cfg.vocab_size, (B * S,), device="cuda")
                pos = (lens0.long()[:, None] + torch.arange(S, device="cuda")).view(-1)
                verify = VerifyKV(cache, S, nq, work)

                def step():
                    h = model._verify_hidden(vids, pos, None, verify)
                    lm_head_logits_(h, W, logits[:B * S])

                row[f"verify_step_us_k{k}"] = round(_graph_us(step, launches), 1)
            out.append(row)
            del cache
    return out


def bench_kernels(model, launches):
    from adapcc_b200.ops import (LookupState, decode_attention_, decode_attention_work_numel, lookup_accept_,
                                 lookup_argmax_, lookup_draft_, verify_attention_)

    cfg = model.cfg
    B, H, Dh, D, V = 8, cfg.n_head, cfg.n_embd // cfg.n_head, cfg.n_embd, cfg.vocab_size
    g = torch.Generator(device="cuda").manual_seed(1)
    out = []
    for T in (128, 512):
        t_max = T + NEW_TOKENS
        kc = torch.randn(B, H, t_max, Dh, device="cuda", generator=g).to(torch.bfloat16)
        vc = torch.randn_like(kc.float()).to(torch.bfloat16)
        lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
        for k in KS:
            S = k + 1
            qkv = torch.randn(B * S, 3 * D, device="cuda", generator=g).to(torch.bfloat16)
            o = torch.empty(B * S, D, dtype=torch.bfloat16, device="cuda")
            nq = torch.full((B,), S, dtype=torch.int32, device="cuda")
            work = torch.empty(decode_attention_work_numel(B * S, H, Dh, t_max), dtype=torch.float32, device="cuda")
            ver_us = _graph_us(lambda: verify_attention_(qkv, kc, vc, lens, nq, k, o, work), launches)
            lj = [(lens + j).contiguous() for j in range(S)]
            oj = torch.empty(B, D, dtype=torch.bfloat16, device="cuda")
            q3 = qkv.view(B, S, 3 * D)

            def sequential():
                for j in range(S):
                    decode_attention_(q3[:, j], kc, vc, lj[j], oj, work)

            seq_us = _graph_us(sequential, launches)
            # acceptance and drafts after a verify step of B·(k+1) slots (never done: max_new beyond every launch)
            st = LookupState(B, k, 200000, t_max, 2, "cuda")
            st.seq.random_(0, 50, generator=g)
            st.nq.fill_(S)
            logits = torch.randn(B * S, (V + 63) // 64 * 64, device="cuda", generator=g)
            rl = lens.clone()

            def accept_draft():
                rl.copy_(lens)
                lookup_argmax_(logits, V, st)
                lookup_accept_(st, rl)
                lookup_draft_(st, rl)

            acc_us = _graph_us(accept_draft, launches)
            out.append({"rows": B, "k": k, "cached": T, "verify_attention_us": round(ver_us, 2),
                        "sequential_decode_attention_us": round(seq_us, 2), "accept_draft_us": round(acc_us, 2)})
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lookup_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    kernels = bench_kernels(model, args.launches)
    steps = bench_steps(model, args.launches)
    gen, periods = bench_generate(model, args.reps)
    print(json.dumps(dict(info, new_tokens=NEW_TOKENS, kernels=kernels, steps=steps, generate=gen,
                          poll_period=periods)))


if __name__ == "__main__":
    main()
