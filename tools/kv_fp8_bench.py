#!/usr/bin/env python
"""The fp8 (e4m3) KV cache against the bf16 one on GPT-2 small (seeded random weights, H = 12, Dh = 64).

Prints one JSON line with the card's name and power limit, read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository. bf16 and fp8 alternate call by call; every figure is a median.

* ``kernel``: split + combine launches of ``decode_attention_``, 100 captured in a CUDA graph, timed with CUDA events,
  t_max = 1024, every row at ``lens``, B in {1, 8, 64}. GB/s over the bytes read: per row and head, L cached keys and
  values (bf16: 2 Dh bytes each; fp8: Dh bytes and a 4-byte scale) and the new key and value from qkv (2 Dh bytes).
* ``reorder``: ``kv_reorder_`` at 64 rows (8 items of 8 beams, a cyclic parent map), 12 layers, t_max = 1024, with 16
  and 64 generated positions.
* ``generate`` / ``beam_search``: steady-state ms per token at 512-token prompts, as (192-token call - 64-token call)
  / 128 (greedy ``generate`` at 64 rows; ``beam_search`` at B = 8, K = 8), so the prefill cancels.
* ``accuracy``: teacher-forced logits of 64 tokens after 256-token prompts (8 rows) through each cache, against the
  fp32 model without a cache: max |error| and the share of positions whose arg-max agrees. Reported, not gated.

Usage: ``python tools/kv_fp8_bench.py [--reps 5] [--launches 2000]``
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

GRAPH_LAUNCHES = 100
H, DH, T_MAX = 12, 64, 1024
FP8 = "fp8_e4m3"


def _gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2] if r.returncode == 0 else ("?", "?")
    return {"device": torch.cuda.get_device_name(), "nvidia_smi_name": name, "power_limit": power}


def _graph(fn):
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
    return graph


def _us(graph, launches):
    reps = max(1, launches // GRAPH_LAUNCHES)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * GRAPH_LAUNCHES)


def _alternate(graphs, launches, reps):
    """Median µs per launch of each graph, timed in turn ``reps`` times."""
    times = {k: [] for k in graphs}
    for _ in range(reps):
        for k, g in graphs.items():
            times[k].append(_us(g, launches))
    return {k: statistics.median(v) for k, v in times.items()}


def bench_kernel(launches, reps):
    from adapcc_b200.ops import decode_attention_, decode_attention_work_numel
    from adapcc_b200.ops.kvcache import quantize

    rows = []
    for B in (1, 8, 64):
        g = torch.Generator(device="cuda").manual_seed(1)
        qkv = torch.randn(B, 3 * H * DH, device="cuda", generator=g).to(torch.bfloat16)
        kc = torch.randn(B, H, T_MAX, DH, device="cuda", generator=g).to(torch.bfloat16)
        vc = torch.randn_like(kc)
        (kq, ks), (vq, vs) = quantize(kc), quantize(vc)
        out = torch.empty(B, H * DH, dtype=torch.bfloat16, device="cuda")
        work = torch.empty(decode_attention_work_numel(B, H, DH, T_MAX), dtype=torch.float32, device="cuda")
        for L in (128, 512, 1023):
            lens = torch.full((B,), L, dtype=torch.int32, device="cuda")
            graphs = {"bf16": _graph(lambda: decode_attention_(qkv, kc, vc, lens, out, work)),
                      "fp8": _graph(lambda: decode_attention_(qkv, kq, vq, lens, out, work, k_scale=ks, v_scale=vs))}
            us = _alternate(graphs, launches, reps)
            nbytes = {"bf16": B * H * 2 * (L + 1) * DH * 2, "fp8": B * H * 2 * (L * (DH + 4) + 2 * DH)}
            row = {"B": B, "lens": L}
            for k in graphs:
                row[f"{k}_us"] = round(us[k], 2)
                row[f"{k}_GBps"] = round(nbytes[k] / (us[k] * 1e-6) / 1e9, 1)
            row["fp8_over_bf16"] = round(us["fp8"] / us["bf16"], 3)
            rows.append(row)
            del graphs
    return rows


def bench_reorder(launches, reps):
    from adapcc_b200.ops import kv_reorder_, kv_reorder_scratch_numel

    L, R, K = 12, 64, 8
    parent = torch.tensor([(r // K) * K + (r + 1) % K for r in range(R)], dtype=torch.int32, device="cuda")
    prompt_len = torch.full((R,), 512, dtype=torch.int32, device="cuda")
    kb = torch.zeros(L, R, H, T_MAX, DH, dtype=torch.bfloat16, device="cuda")
    vb = torch.zeros_like(kb)
    kq = torch.zeros(L, R, H, T_MAX, DH, dtype=torch.uint8, device="cuda")
    vq = torch.zeros_like(kq)
    ks = torch.zeros(L, R, H, T_MAX, device="cuda")
    vs = torch.zeros_like(ks)
    rows = []
    for n in (16, 64):
        lens = prompt_len + n
        sb = torch.empty(kv_reorder_scratch_numel(kb, n), dtype=torch.bfloat16, device="cuda")
        s8 = torch.empty(kv_reorder_scratch_numel(kq, n, fp8=True), dtype=torch.uint8, device="cuda")
        graphs = {"bf16": _graph(lambda: kv_reorder_(kb, vb, parent, prompt_len, lens, n, sb)),
                  "fp8": _graph(lambda: kv_reorder_(kq, vq, parent, prompt_len, lens, n, s8, k_scale=ks,
                                                    v_scale=vs))}
        us = _alternate(graphs, launches // 10, reps)
        rows.append({"rows": R, "new_positions": n, "bf16_us": round(us["bf16"], 1), "fp8_us": round(us["fp8"], 1),
                     "fp8_over_bf16": round(us["fp8"] / us["bf16"], 3)})
        del graphs, sb, s8
    return rows


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def bench_decoders(model, reps):
    g = torch.Generator(device="cuda").manual_seed(2)
    V = model.cfg.vocab_size
    cases = {"generate": (torch.randint(0, V, (64, 512), device="cuda", generator=g),
                          lambda ids, n, dt: model.generate(ids, max_new_tokens=n, temperature=0.0, kv_cache_dtype=dt)),
             "beam_search": (torch.randint(0, V, (8, 512), device="cuda", generator=g),
                             lambda ids, n, dt: model.beam_search(ids, num_beams=8, max_new_tokens=n,
                                                                  kv_cache_dtype=dt))}
    res = {}
    for name, (ids, run) in cases.items():
        for dt in (None, FP8):                                   # warm-up of every shape
            for n in (64, 192):
                run(ids, n, dt)
        times = {(dt, n): [] for dt in (None, FP8) for n in (64, 192)}
        for _ in range(reps):
            for n in (64, 192):
                for dt in (None, FP8):
                    times[(dt, n)].append(_timed(lambda: run(ids, n, dt)))
        med = {k: statistics.median(v) for k, v in times.items()}
        per = {("fp8" if dt else "bf16"): (med[(dt, 192)] - med[(dt, 64)]) / 128 for dt in (None, FP8)}
        res[name] = {"rows": int(ids.shape[0]) * (8 if name == "beam_search" else 1), "prompt": 512,
                     "bf16_ms_per_token": round(per["bf16"], 3), "fp8_ms_per_token": round(per["fp8"], 3),
                     "fp8_over_bf16": round(per["fp8"] / per["bf16"], 3)}
    return res


def accuracy(model):
    import copy

    g = torch.Generator(device="cuda").manual_seed(3)
    B, P, n = 8, 256, 64
    ids = torch.randint(0, model.cfg.vocab_size, (B, P + n), device="cuda", generator=g)
    ref_model = copy.deepcopy(model).float()
    with torch.no_grad():
        ref = ref_model.lm_logits(ref_model.hidden(ids, None))[:, P - 1:P + n - 1]       # [B, n, V]
        del ref_model
        head = model.wte.weight.float()
        res = {}
        for name, dt in (("bf16", None), ("fp8", FP8)):
            cache = model.new_cache(B, P + n, dt)
            h = model.hidden(ids[:, :P], None, cache=cache)[:, -1]
            out = []
            for i in range(n):
                out.append(model.lm_logits(h, head))
                if i + 1 < n:
                    h = model.decode_step(ids[:, P + i], None, cache)
            got = torch.stack(out, 1)
            res[name] = {"max_abs_err": round(float((got - ref).abs().max()), 4),
                         "argmax_agree": round(float((got.argmax(-1) == ref.argmax(-1)).float().mean()), 4)}
    return dict(rows=B, prompt=P, tokens=n, **res)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=2000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("kv_fp8_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, kernel=bench_kernel(args.launches, args.reps), reorder=bench_reorder(args.launches, args.reps),
                  decoders=bench_decoders(model, max(3, args.reps // 2)), accuracy=accuracy(model))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
