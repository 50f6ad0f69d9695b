#!/usr/bin/env python
"""GPT-2 small beam search: ``GPT2DoubleHeads.beam_search`` against greedy ``generate`` at the same number of rows,
beam sampling against beam search, diverse beam search by group count, and the selection and cache-reordering
kernels on their own.

Prints one JSON line with the device name and power limit read in the same run. Needs a CUDA device (there is no CPU
fallback) and writes nothing into the repository.

* ``search``: ms per generated token, prefill and graph capture included (64 new tokens, bf16, seeded random weights,
  no stop ids, so every call runs all 64 tokens), for B = 1 / 8 items, K = 4 / 8 beams and prompts of 128 / 512 tokens.
  Next to each, ``generate(temperature=0)`` at B·K rows does the same decode-step and LM-head work, so the difference
  is what beam search adds (selection, cache reordering, the B·K-row cache copy). Medians of ``--reps`` runs after one
  warm-up run.
* ``kernels``: ``beam_step_`` (vocab 50257) and ``kv_reorder_`` (12 layers, 12 heads, Dh 64, every row taking another
  row's cache) at 64 rows (8 items x 8 beams) with 16 and 64 generated positions, 50 launches captured in a CUDA graph
  and timed with CUDA events over ``--launches`` launches. GB/s for the reorder counts the generated region read and
  written twice (into the scratch and back). Also the sampled ``beam_step_`` (temperature 1, no top-k, every id kept)
  with top-p 1 and 0.9.
* ``sampled``: ``beam_search(do_sample=True, top_k=50)`` against ``do_sample=False``, ms per generated token as in
  ``search``, the two alternated run by run in this process (medians of ``--reps`` pairs after one warm-up each).
* ``groups``: diverse beam search, ``beam_search(num_beam_groups=G, diversity_penalty=0.5)`` for B = 8 items, K = 8
  beams, G = 1 / 2 / 4 / 8 and 128-token prompts, ms per generated token as in ``search`` (no stop ids, so every call
  runs all 64 tokens), the four alternated run by run; and ``beam_step_`` alone at 64 rows (vocab 50257) with G = 1
  against G = 8, timed as in ``kernels``.
* ``stochastic``: ``stochastic_beam_search(top_k=50)`` against ``beam_search(do_sample=True, top_k=50)`` for B = 8
  items, K = 8 beams and 128-token prompts, ms per generated token as in ``sampled`` (no stop ids, 64 new tokens),
  the two alternated run by run; and the stochastic ``beam_step_`` (its rows and select kernels, temperature 1, no
  top-k) alone at 64 rows (vocab 50257), timed as in ``kernels``.
* ``filters``: the sampled ``beam_step_`` of beam sampling and of stochastic beam search (temperature 0.7, no top-k,
  top-p 1, two stop ids, so beam sampling keeps 3 ids in every filter) at 64 rows (vocab 50257), timed as in
  ``kernels``, with the truncation filters off and with each one on: top-h, min-p, typical, epsilon and eta.

Usage: ``python tools/beam_bench.py [--reps 3] [--launches 1000] [--sections kernels,filters,...]``
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
        for K in (4, 8):
            for T in (128, 512):
                prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
                wide = prompt.repeat_interleave(K, dim=0)
                beam = _median_ms(lambda: model.beam_search(prompt, num_beams=K, max_new_tokens=NEW_TOKENS), reps)
                greedy = _median_ms(lambda: model.generate(wide, max_new_tokens=NEW_TOKENS, temperature=0.0), reps)
                rows.append({"batch": B, "beams": K, "prompt": T,
                             "beam_search_ms_per_token": round(beam / NEW_TOKENS, 3),
                             "generate_rows_ms_per_token": round(greedy / NEW_TOKENS, 3),
                             "beam_cost_ms_per_token": round((beam - greedy) / NEW_TOKENS, 3)})
    return rows


def bench_sampled(model, reps):
    rows = []
    g = torch.Generator(device="cuda").manual_seed(2)
    for B in (1, 8):
        for K in (4, 8):
            for T in (128, 512):
                prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
                runs = {False: lambda: model.beam_search(prompt, num_beams=K, max_new_tokens=NEW_TOKENS),
                        True: lambda: model.beam_search(prompt, num_beams=K, max_new_tokens=NEW_TOKENS,
                                                        do_sample=True, temperature=1.0, top_k=50, seed=3)}
                times = {False: [], True: []}
                for sample in (False, True):
                    runs[sample]()                                 # warm-up of this shape
                for _ in range(reps):
                    for sample in (False, True):
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        runs[sample]()
                        torch.cuda.synchronize()
                        times[sample].append((time.perf_counter() - t0) * 1e3)
                greedy, sampled = (statistics.median(times[x]) for x in (False, True))
                rows.append({"batch": B, "beams": K, "prompt": T,
                             "beam_search_ms_per_token": round(greedy / NEW_TOKENS, 3),
                             "beam_sample_ms_per_token": round(sampled / NEW_TOKENS, 3),
                             "sample_cost_ms_per_token": round((sampled - greedy) / NEW_TOKENS, 3)})
    return rows


def bench_groups(model, reps, launches):
    from adapcc_b200.ops import BeamState, beam_step_

    B, K, lam = 8, 8, 0.5
    g = torch.Generator(device="cuda").manual_seed(5)
    prompt = torch.randint(0, model.cfg.vocab_size, (B, 128), device="cuda", generator=g)
    groups = (1, 2, 4, 8)

    def run(G):
        return model.beam_search(prompt, num_beams=K, max_new_tokens=NEW_TOKENS, num_beam_groups=G,
                                 diversity_penalty=lam if G > 1 else 0.0)

    times = {G: [] for G in groups}
    for G in groups:
        run(G)                                                     # warm-up of this shape
    for _ in range(reps):
        for G in groups:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(G)
            torch.cuda.synchronize()
            times[G].append((time.perf_counter() - t0) * 1e3)
    out = {"batch": B, "beams": K, "prompt": 128, "diversity_penalty": lam,
           "ms_per_token": {str(G): round(statistics.median(times[G]) / NEW_TOKENS, 3) for G in groups}}
    logits = torch.randn(B * K, model.wte.weight.shape[0], device="cuda", generator=g) * 3
    max_new = launches + 4 * GRAPH_LAUNCHES
    for G in (1, 8):
        st = BeamState(B, K, max_new, 1.0, "cuda", groups=G)
        st.scores.zero_()
        kw = dict(diversity_penalty=lam) if G > 1 else {}
        out[f"beam_step_G{G}_us"] = round(_graph_us(lambda: beam_step_(logits, model.cfg.vocab_size, st, **kw),
                                                    launches), 2)
    return out


def bench_stochastic(model, reps, launches):
    from adapcc_b200.ops import BeamState, beam_step_

    B, K, T = 8, 8, 128
    g = torch.Generator(device="cuda").manual_seed(7)
    prompt = torch.randint(0, model.cfg.vocab_size, (B, T), device="cuda", generator=g)
    runs = {"stochastic": lambda: model.stochastic_beam_search(prompt, num_beams=K, max_new_tokens=NEW_TOKENS,
                                                                top_k=50, seed=3),
            "beam_sample": lambda: model.beam_search(prompt, num_beams=K, max_new_tokens=NEW_TOKENS, do_sample=True,
                                                     temperature=1.0, top_k=50, seed=3)}
    times = {k: [] for k in runs}
    for fn in runs.values():
        fn()                                                       # warm-up of this shape
    for _ in range(reps):
        for k, fn in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    out = {"batch": B, "beams": K, "prompt": T, "top_k": 50,
           "ms_per_token": {k: round(statistics.median(v) / NEW_TOKENS, 3) for k, v in times.items()}}
    V = 50257
    logits = torch.randn(B * K, model.wte.weight.shape[0], device="cuda", generator=g) * 3
    st = BeamState(B, K, launches + 4 * GRAPH_LAUNCHES, 1.0, "cuda", seeds=torch.arange(B, dtype=torch.int64))
    st.scores.zero_()                                              # every beam live, so no item finishes
    st.keys.zero_()
    out["stochastic_step_us"] = round(_graph_us(lambda: beam_step_(logits, V, st), launches), 2)
    return out


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
    from adapcc_b200.ops import BeamState, beam_step_, kv_reorder_, kv_reorder_scratch_numel, lm_head_logits_

    B, K = 8, 8
    cfg = model.cfg
    W = model.wte.weight
    g = torch.Generator(device="cuda").manual_seed(1)
    h = torch.randn(B * K, cfg.n_embd, device="cuda", generator=g).to(torch.bfloat16)
    logits = torch.empty(B * K, W.shape[0], dtype=torch.float32, device="cuda")
    lm_us = _graph_us(lambda: lm_head_logits_(h, W, logits), launches)
    logits.copy_(torch.randn(B * K, W.shape[0], device="cuda", generator=g) * 3)
    # room for every launch: the step never reaches max_new and, without stop ids, no item finishes
    max_new = launches + 4 * GRAPH_LAUNCHES
    st = BeamState(B, K, max_new, 1.0, "cuda")
    st.scores.zero_()
    step_us = _graph_us(lambda: beam_step_(logits, cfg.vocab_size, st), launches)
    out = {"rows": B * K, "lm_head_us": round(lm_us, 2), "beam_step_us": round(step_us, 2), "kv_reorder": []}
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")
    for top_p in (1.0, 0.9):
        st = BeamState(B, K, max_new, 1.0, "cuda", sample=True)
        st.scores.zero_()
        us = _graph_us(lambda: beam_step_(logits, cfg.vocab_size, st, top_p=top_p, seeds=seeds), launches)
        out[f"beam_sample_step_top_p_{top_p}_us"] = round(us, 2)
    L, H, Dh, T = cfg.n_layer, cfg.n_head, cfg.n_embd // cfg.n_head, 512
    for gen in (16, 64):
        cache = model.new_cache(B * K, T + 64)
        cache.k.normal_(generator=g)
        cache.v.normal_(generator=g)
        prompt_len = torch.full((B * K,), T, dtype=torch.int32, device="cuda")
        lens = prompt_len + gen
        parent = torch.arange(B * K, dtype=torch.int32, device="cuda").roll(1)
        scratch = torch.empty(kv_reorder_scratch_numel(cache.k, 64), dtype=torch.bfloat16, device="cuda")
        us = _graph_us(lambda: kv_reorder_(cache.k, cache.v, parent, prompt_len, lens, 64, scratch), launches)
        moved = B * K * gen * L * 2 * H * Dh * 2                       # bytes of the generated region, k and v
        out["kv_reorder"].append({"generated": gen, "us": round(us, 2), "MB_moved": round(moved / 1e6, 1),
                                  "GBps": round(4 * moved / (us * 1e-6) / 1e9, 1)})
        del cache, scratch
    return out


FILTERS = [("off", {}), ("top_h=0.9", dict(top_h=0.9)), ("min_p=0.05", dict(min_p=0.05)),
           ("typical_p=0.9", dict(typical_p=0.9)), ("epsilon_cutoff=3e-4", dict(epsilon_cutoff=3e-4)),
           ("eta_cutoff=3e-4", dict(eta_cutoff=3e-4))]


def bench_filters(model, launches):
    from adapcc_b200.ops import BeamState, beam_step_

    B, K, V = 8, 8, 50257
    g = torch.Generator(device="cuda").manual_seed(9)
    logits = torch.randn(B * K, model.wte.weight.shape[0], device="cuda", generator=g) * 3
    stop = torch.tensor([11, 13], dtype=torch.int32, device="cuda")
    seeds = torch.arange(B, dtype=torch.int64, device="cuda")
    max_new = launches + 4 * GRAPH_LAUNCHES
    out = {"rows": B * K, "temperature": 0.7, "beam_sample_step_us": {}, "stochastic_step_us": {}}
    for name, f in FILTERS:
        st = BeamState(B, K, max_new, 1.0, "cuda", sample=True)
        st.scores.zero_()
        us = _graph_us(lambda: beam_step_(logits, V, st, 0, None, stop, temperature=0.7, seeds=seeds, **f), launches)
        out["beam_sample_step_us"][name] = round(us, 2)
        st = BeamState(B, K, max_new, 1.0, "cuda", seeds=seeds.cpu())
        st.scores.zero_()
        st.keys.zero_()
        us = _graph_us(lambda: beam_step_(logits, V, st, 0, None, stop, temperature=0.7, **f), launches)
        out["stochastic_step_us"][name] = round(us, 2)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=1000)
    ap.add_argument("--sections", default="kernels,search,sampled,groups,stochastic,filters",
                    help="comma-separated sections to run (default: all)")
    args = ap.parse_args()
    sections = set(args.sections.split(","))
    if not torch.cuda.is_available():
        sys.exit("beam_bench: needs a CUDA device")
    from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads
    from adapcc_b200.runtime.native import load_library

    load_library(build_if_missing=False)
    torch.cuda.set_device(0)
    info = _gpu_info()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config()).to(device="cuda", dtype=torch.bfloat16).eval()
    runs = dict(kernels=lambda: bench_kernels(model, args.launches), search=lambda: bench_search(model, args.reps),
                sampled=lambda: bench_sampled(model, args.reps),
                groups=lambda: bench_groups(model, args.reps, args.launches),
                stochastic=lambda: bench_stochastic(model, args.reps, args.launches),
                filters=lambda: bench_filters(model, args.launches))
    result = dict(info, new_tokens=NEW_TOKENS, **{k: fn() for k, fn in runs.items() if k in sections})
    print(json.dumps(result))


if __name__ == "__main__":
    main()
