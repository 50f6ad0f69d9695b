#!/usr/bin/env python
"""Greedy GPT-2 small generation with and without the KV cache, and the decode-attention kernel on its own.

Prints one JSON line. Needs a CUDA device (there is no CPU fallback) and writes nothing into the repository.

* ``generate``: ms per generated token (prefill included, 64 new tokens, greedy, bf16, seeded random weights) for
  (a) ``uncached``: the loop as it was before the cache — the whole prefix through the model and an fp32 copy of the
  tied LM head per token, (b) ``eager``: prefill once, then ``decode_step`` per token, (c) ``graph``: the same with the
  decode step replayed from a CUDA graph (captured once per cache, outside the timed window; ``capture_ms``). Prompt
  lengths 128 / 512 / 896, batch 1 and 8. Each figure is the median of ``--reps`` timed runs.
* ``kernel``: split + combine launches of ``decode_attention_``, captured 100 to a CUDA graph and timed with CUDA
  events over ``--launches`` launches,
  H = 12, Dh = 64, t_max = 1024, every row at ``lens``; GB/s over the K / V bytes read, 2 (lens + 1) H Dh 2 per row,
  and that rate over the H100 SXM's 3.35 TB/s.

Usage: ``python tools/decode_bench.py [--reps 3] [--launches 2000]``
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
GRAPH_LAUNCHES = 100
HBM_TBPS = 3.35


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


def uncached(model, prompt):
    ids = prompt
    vocab = model.cfg.vocab_size
    for _ in range(NEW_TOKENS):
        h = model.hidden(ids, None)
        nxt = (h[:, -1].float() @ model.wte.weight.float().t())[:, :vocab].argmax(-1, keepdim=True)
        ids = torch.cat([ids, nxt], 1)
    return ids[:, prompt.shape[1]:]


def cached(model, prompt, cache, step, head):
    vocab = model.cfg.vocab_size
    h = model.hidden(prompt, None, cache=cache)[:, -1]
    out = []
    for i in range(NEW_TOKENS):
        nxt = (h.float() @ head.t())[:, :vocab].argmax(-1)
        out.append(nxt)
        if i + 1 < NEW_TOKENS:
            h = step(nxt)
    return torch.stack(out, 1)


def bench_generate(model, reps):
    from adapcc_b200.models.gpt2 import DecodeGraph

    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8):
        cache_e, cache_g = model.new_cache(B), model.new_cache(B)
        for T in (128, 512, 896):
            prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
            with torch.no_grad():
                model.hidden(prompt, None, cache=cache_g)
                c_ms, graph = _timed(lambda: DecodeGraph(model, cache_g, token_types=False))
                res = {"batch": B, "prompt": T, "capture_ms": round(c_ms, 2)}
                runs = {
                    "uncached": lambda: uncached(model, prompt),
                    "eager": lambda: cached(model, prompt, cache_e, lambda t: model.decode_step(t, None, cache_e),
                                            model.wte.weight.float()),
                    "graph": lambda: cached(model, prompt, cache_g, lambda t: graph(t), model.wte.weight.float()),
                }
                toks = {}
                for name, fn in runs.items():
                    fn()                                                   # warm-up of this shape
                    times = []
                    for _ in range(reps):
                        ms, toks[name] = _timed(fn)
                        times.append(ms)
                    res[f"{name}_ms_per_token"] = round(statistics.median(times) / NEW_TOKENS, 3)
                res["speedup_graph_vs_uncached"] = round(res["uncached_ms_per_token"] / res["graph_ms_per_token"], 2)
                res["graph_equals_eager"] = bool(torch.equal(toks["graph"], toks["eager"]))
                res["tokens_equal_uncached"] = int((toks["graph"] == toks["uncached"]).all(0).long().cumprod(0).sum())
            rows.append(res)
            del graph
    return rows


def bench_kernel(launches):
    from adapcc_b200.ops import decode_attention_, decode_attention_work_numel

    H, Dh, t_max = 12, 64, 1024
    rows = []
    for B in (1, 8):
        g = torch.Generator(device="cuda").manual_seed(1)
        qkv = torch.randn(B, 3 * H * Dh, device="cuda", generator=g).to(torch.bfloat16)
        kc = torch.randn(B, H, t_max, Dh, device="cuda", generator=g).to(torch.bfloat16)
        vc = torch.randn_like(kc)
        out = torch.empty(B, H * Dh, dtype=torch.bfloat16, device="cuda")
        work = torch.empty(decode_attention_work_numel(B, H, Dh, t_max), dtype=torch.float32, device="cuda")
        for L in (128, 512, 1023):
            lens = torch.full((B,), L, dtype=torch.int32, device="cuda")
            # launches replayed from a graph, so the host's per-launch cost stays out of the device time
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                decode_attention_(qkv, kc, vc, lens, out, work)
            torch.cuda.current_stream().wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(GRAPH_LAUNCHES):
                    decode_attention_(qkv, kc, vc, lens, out, work)
            graph.replay()
            reps = max(1, launches // GRAPH_LAUNCHES)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / (reps * GRAPH_LAUNCHES)
            gbps = B * 2 * (L + 1) * H * Dh * 2 / (us * 1e-6) / 1e9
            rows.append({"BH": B * H, "lens": L, "us": round(us, 2), "GBps": round(gbps, 1),
                         "share_of_3.35TBps": round(gbps / (HBM_TBPS * 1e3), 3)})
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=2000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("decode_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, new_tokens=NEW_TOKENS, kernel=bench_kernel(args.launches),
                  generate=bench_generate(model, args.reps))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
