#!/usr/bin/env python
"""GPT-2 small contrastive search: ``GPT2DoubleHeads.contrastive_search`` against greedy ``generate`` at the same rows,
the candidate attention kernel against ``decode_attention_`` over a k-fold copied cache, and the re-rank kernel alone.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository.

* ``search``: ms per generated token, prefill and graph capture included (64 new tokens, bf16, seeded random weights,
  no stop ids), for B = 1 / 8 rows, k = 4 / 8 candidates and prompts of 128 / 512 tokens, next to
  ``generate(temperature=0)`` at the same B rows. Medians of ``--reps`` runs after one warm-up run.
* ``kernels`` (one layer of GPT-2 small, 12 heads of 64, at 8 rows with 128 / 512 cached tokens and k = 4 / 8):
  ``cand_attention_`` against ``decode_attention_`` on a k-fold copy of the cache (the copy itself timed apart), and
  ``contrastive_rerank_`` (similarities against the context, score, commit of 12 layers' keys and values). 50 launches
  captured in a CUDA graph, timed with CUDA events over ``--launches`` launches.

Usage: ``python tools/contrastive_bench.py [--reps 3] [--launches 1000]``
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


def bench_search(model, reps):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8):
        for T in (128, 512):
            prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
            greedy = _median_ms(lambda: model.generate(prompt, max_new_tokens=NEW_TOKENS, temperature=0.0), reps)
            for K in (4, 8):
                cs = _median_ms(lambda: model.contrastive_search(prompt, top_k=K, penalty_alpha=0.6,
                                                                 max_new_tokens=NEW_TOKENS), reps)
                rows.append({"batch": B, "top_k": K, "prompt": T,
                             "contrastive_ms_per_token": round(cs / NEW_TOKENS, 3),
                             "greedy_ms_per_token": round(greedy / NEW_TOKENS, 3)})
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
    from adapcc_b200.ops import (ContrastiveState, cand_attention_, contrastive_rerank_, decode_attention_,
                                 decode_attention_work_numel)

    cfg = model.cfg
    B, H, Dh, L, D = 8, cfg.n_head, cfg.n_embd // cfg.n_head, cfg.n_layer, cfg.n_embd
    g = torch.Generator(device="cuda").manual_seed(1)
    out = []
    for T in (128, 512):
        t_max = T + NEW_TOKENS
        kc = torch.randn(B, H, t_max, Dh, device="cuda", generator=g).to(torch.bfloat16)
        vc = torch.randn_like(kc.float()).to(torch.bfloat16)
        lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
        for K in (4, 8):
            qkv = torch.randn(B * K, 3 * D, device="cuda", generator=g).to(torch.bfloat16)
            o = torch.empty(B * K, D, dtype=torch.bfloat16, device="cuda")
            sk, sv = torch.empty_like(o), torch.empty_like(o)
            work = torch.empty(decode_attention_work_numel(B * K, H, Dh, t_max), dtype=torch.float32, device="cuda")
            cand_us = _graph_us(lambda: cand_attention_(qkv, kc, vc, lens, K, o, sk, sv, work), launches)
            kx, vx = kc.repeat_interleave(K, 0).contiguous(), vc.repeat_interleave(K, 0).contiguous()
            lx = lens.repeat_interleave(K).contiguous()
            copy_us = _graph_us(lambda: (kx.copy_(kc.repeat_interleave(K, 0)), vx.copy_(vc.repeat_interleave(K, 0))),
                                launches)
            dec_us = _graph_us(lambda: decode_attention_(qkv, kx, vx, lx, o, work), launches)
            # re-rank and commit: a context of T positions, every layer's cache
            st = ContrastiveState(B, K, 1, t_max, L, H, Dh, "cuda")   # step runs past max_new: no token writes
            st.ctx.normal_(generator=g)
            st.ctx_norm.copy_(st.ctx.float().norm(dim=-1))
            st.cand_tok.copy_(torch.arange(B * K, dtype=torch.int32))
            st.cand_p.fill_(0.1)
            hc = torch.randn(B * K, D, device="cuda", generator=g).to(torch.bfloat16)
            ck = torch.zeros(L, B, H, t_max, Dh, dtype=torch.bfloat16, device="cuda")
            cv = torch.zeros_like(ck)
            rl = lens.clone()

            def rerank():
                rl.copy_(lens)                                    # every launch at the same context length
                contrastive_rerank_(hc, st, 0.6, ck, cv, rl)

            rr_us = _graph_us(rerank, launches)
            out.append({"rows": B, "top_k": K, "cached": T, "cand_attention_us": round(cand_us, 2),
                        "decode_attention_on_copy_us": round(dec_us, 2), "kfold_copy_us": round(copy_us, 2),
                        "rerank_commit_us": round(rr_us, 2)})
            del ck, cv, st
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("contrastive_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    result = dict(info, new_tokens=NEW_TOKENS, kernels=bench_kernels(model, args.launches),
                  search=bench_search(model, args.reps))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
