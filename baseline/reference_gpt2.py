#!/usr/bin/env python
"""The reference's GPT-2 arm, run through its own stock code path (no repo model, kernel or engine).

What the reference's flagship script does (/root/reference/models/gpt2/train_gpt2_ddp.py):

* ``GPT2DoubleHeadsModel(GPT2Config())`` — GPT-2 small, random init (:157-159) — plus the five PersonaChat special
  tokens via ``resize_token_embeddings`` (:28-30, 54-59);
* ``AdamW(model.parameters(), lr=args.lr, correct_bias=True)`` (:163) — HuggingFace's AdamW, ``weight_decay=0``;
* ``DDP(model, device_ids=[LOCAL_RANK], output_device=LOCAL_RANK)`` over NCCL (:145, 166) — also at world size 1;
* the step body ``update`` (:172-198): ``model.train()``, the batch ``.to(LOCAL_RANK)``, forward with
  ``token_type_ids / mc_token_ids / mc_labels / labels``, ``loss = lm_loss * lm_coef + mc_loss * mc_coef``,
  ``backward``, ``clip_grad_norm_(max_norm)``, ``optimizer.step()``, ``optimizer.zero_grad()``, ``loss.item()``.

The script itself cannot be launched here: it imports ``ignite`` (not in the image) and ``transformers.AdamW``
(removed in transformers 5), reads ``OMPI_COMM_WORLD_*`` and downloads the tokenizer and PersonaChat. This file
therefore executes THAT step body with THOSE classes — HuggingFace's model, torch's DDP/NCCL, ``torch.optim.AdamW``
with the HF defaults — and takes the hyper-parameters (special tokens, lr, max_norm, loss coefficients, batch size,
candidates) from the unmodified source under ``baseline/_ref`` when it is present (``ast``-parsed, not imported).
Replaced, and said so in the JSON line (``reference_class``): the ignite ``Engine`` loop (a plain ``for``), the
dataset (synthetic PersonaChat-shaped ``[B, C, T]`` batches) and the compute precision (bf16 autocast by default, the
dtype the comparison is quoted in; ``--ref_precision fp32`` is the script's literal fp32).

Nothing from ``adapcc_b200`` is imported and ``libadapcc.so`` is never mapped in this process.
"""
from __future__ import annotations

import ast
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SCRIPT = os.path.join(ROOT, "baseline", "_ref", "models", "gpt2", "train_gpt2_ddp.py")

# the reference script's literals (used when baseline/_ref is absent; identical values)
DEFAULTS = {"SPECIAL_TOKENS": ["<bos>", "<eos>", "<speaker1>", "<speaker2>", "<pad>"], "lr": 6.25e-5, "max_norm": 1.0,
            "lm_coef": 1.0, "mc_coef": 1.0, "train_batch_size": 4, "num_candidates": 2}


def reference_hyperparameters(path: str = REF_SCRIPT) -> dict:
    """SPECIAL_TOKENS and the argparse defaults, read from the unmodified reference source without importing it."""
    out = dict(DEFAULTS)
    out["source"] = "built-in copy of the reference's literals (baseline/_ref absent)"
    try:
        tree = ast.parse(open(path).read())
    except (OSError, SyntaxError):
        return out
    for node in ast.walk(tree):
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and getattr(node.targets[0], "id", "") == "SPECIAL_TOKENS":
            out["SPECIAL_TOKENS"] = ast.literal_eval(node.value)
        if isinstance(node, ast.Call) and getattr(node.func, "attr", "") == "add_argument" and node.args:
            try:
                name = ast.literal_eval(node.args[0]).lstrip("-")
            except (ValueError, SyntaxError):
                continue
            if name in DEFAULTS:
                for kw in node.keywords:
                    if kw.arg == "default":
                        try:
                            out[name] = ast.literal_eval(kw.value)
                        except (ValueError, SyntaxError):
                            pass
    out["source"] = os.path.relpath(path, ROOT)
    return out


def synthetic_personachat(batch: int, candidates: int, seq_len: int, vocab: int, seed: int, pin: bool):
    """[B, C, T] ids / token types / labels, [B, C] mc_token_ids, [B] mc_labels in the reference's MODEL_INPUTS order
    semantics (train_gpt2_ddp.py:31, 62-74): history carries -100 labels, only the last candidate's reply is scored,
    the classification token is the last one."""
    import torch

    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, vocab, (batch, candidates, seq_len), generator=g)
    tt = torch.randint(vocab - 3, vocab - 1, (batch, candidates, seq_len), generator=g)       # <speaker1>/<speaker2>
    labels = torch.full((batch, candidates, seq_len), -100, dtype=torch.long)
    reply = max(1, seq_len // 4)
    labels[:, -1, -reply:] = ids[:, -1, -reply:]
    mc_token_ids = torch.full((batch, candidates), seq_len - 1, dtype=torch.long)
    mc_labels = torch.full((batch,), candidates - 1, dtype=torch.long)
    b = (ids, mc_token_ids, labels, mc_labels, tt)                                           # MODEL_INPUTS order
    if pin and torch.cuda.is_available():
        b = tuple(t.pin_memory() for t in b)
    return b


def run(a, ClockSampler=None) -> int:
    """``a``: bench.py's argparse namespace (gpus, steps, warmup, batch, candidates, seq, tiny, ref_precision)."""
    import torch
    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP
    from transformers import GPT2Config, GPT2DoubleHeadsModel

    hp = reference_hyperparameters()
    rank = int(os.environ.get("RANK", os.environ.get("OMPI_COMM_WORLD_RANK", 0)))
    world = int(os.environ.get("WORLD_SIZE", os.environ.get("OMPI_COMM_WORLD_SIZE", 1)))
    local = int(os.environ.get("LOCAL_RANK", os.environ.get("OMPI_COMM_WORLD_LOCAL_RANK", 0)))
    cuda = torch.cuda.is_available()
    if not cuda and not getattr(a, "allow_cpu", False):
        if rank == 0:
            print(json.dumps({"impl": "reference", "unavailable": "no CUDA device in this container (the reference arm "
                              "is HF GPT2DoubleHeadsModel + torch DDP over NCCL: it runs on the GPU box)"}), flush=True)
        return 0
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29534")
    if cuda:
        torch.cuda.set_device(local)
        dev = torch.device("cuda", local)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:                                                   # CPU plumbing test only (tests/test_bench_contract.py)
        dev = torch.device("cpu")
        dist.init_process_group("gloo", rank=rank, world_size=world)
    sampler = ClockSampler(local) if (ClockSampler is not None and cuda) else None
    if sampler is not None and rank == 0:
        sampler.start()

    precision = getattr(a, "ref_precision", "bf16")
    if precision == "tf32":
        torch.backends.cuda.matmul.allow_tf32 = True
        torch.backends.cudnn.allow_tf32 = True
    configuration = GPT2Config(n_layer=2, n_embd=64, n_head=4, vocab_size=512, n_positions=64) if a.tiny else GPT2Config()
    seq = min(a.seq, configuration.n_positions)
    torch.manual_seed(1234)
    model = GPT2DoubleHeadsModel(configuration).to(dev)
    vocab = configuration.vocab_size + len(hp["SPECIAL_TOKENS"])                 # add_special_tokens_ (:54-59)
    model.resize_token_embeddings(new_num_tokens=vocab)
    n_params = sum(p.numel() for p in model.parameters())
    # transformers.AdamW(lr, correct_bias=True): betas (0.9, 0.999), eps 1e-6, weight_decay 0.0
    optimizer = torch.optim.AdamW(model.parameters(), lr=hp["lr"], betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0)
    model = DDP(model, device_ids=[local], output_device=local) if cuda else DDP(model)

    host = [synthetic_personachat(a.batch, a.candidates, seq, vocab, seed=1000 * rank + i, pin=True) for i in range(4)]
    dev_batch = tuple(t.to(dev) for t in host[0])
    h2d = sum(t.numel() * t.element_size() for t in host[0])
    autocast = (lambda: torch.autocast(dev.type, dtype=torch.bfloat16)) if precision == "bf16" else (lambda: torch.autocast(dev.type, enabled=False))

    def update(batch, read_loss: bool):
        """train_gpt2_ddp.py:172-198 (the ignite ``update`` closure), statement for statement."""
        model.train()
        batch = tuple(input_tensor.to(dev, non_blocking=True) for input_tensor in batch)
        input_ids, mc_token_ids, lm_labels, mc_labels, token_type_ids = batch
        with autocast():
            output = model(input_ids, token_type_ids=token_type_ids, mc_token_ids=mc_token_ids,
                           mc_labels=mc_labels, labels=lm_labels)
        lm_loss = output.loss
        mc_loss = output.mc_loss
        loss = (lm_loss * hp["lm_coef"] + mc_loss * hp["mc_coef"])
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), hp["max_norm"])
        optimizer.step()
        optimizer.zero_grad()
        return loss.item() if read_loss else loss.detach()

    def barrier():
        dist.barrier()
        if cuda:
            torch.cuda.synchronize()

    def max_over_ranks(x: float) -> float:
        t = torch.tensor([x], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    W, K = max(3, a.warmup), a.steps
    if sampler is not None:
        sampler.mark_begin()
    # (1) device-timed, inputs resident, no loss read-back (the most favourable timing of the reference)
    for _ in range(W):
        update(dev_batch, False)
    barrier()
    if cuda:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    t0 = time.perf_counter()
    for _ in range(K):
        update(dev_batch, False)
    if cuda:
        e1.record()
    barrier()
    wall = (time.perf_counter() - t0) * 1e3
    ms_dev = max_over_ranks((e0.elapsed_time(e1) if cuda else wall) / K)
    # (2) end to end = the script's literal step: host batch -> .to(device) every step, loss.item() every step
    for i in range(W):
        update(host[i % len(host)], True)
    barrier()
    if cuda:
        e0.record()
    t0 = time.perf_counter()
    last = 0.0
    for i in range(K):
        last = update(host[i % len(host)], True)
    if cuda:
        e1.record()
    barrier()
    wall = (time.perf_counter() - t0) * 1e3
    ms_e2e = max_over_ranks(max(e0.elapsed_time(e1) if cuda else 0.0, wall) / K)
    clocks = sampler.stop() if (sampler is not None and rank == 0) else {}
    mapped = [ln.split()[-1] for ln in open("/proc/self/maps") if "libadapcc" in ln] if os.path.exists("/proc/self/maps") else []

    if rank == 0:
        tokens = a.batch * a.candidates * seq * world
        print(json.dumps({
            "metric": "gpt2_small_ddp_train_tokens_per_sec", "value": tokens / (ms_dev * 1e-3), "unit": "tokens/s",
            "n_gpus": world, "steps": K, "warmup": W, "ms_per_step": ms_dev, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": {"bf16": "bf16", "tf32": "tf32", "fp32": "fp32"}[precision],
            "data": "synthetic", "impl": "reference",
            "reference_class": ("transformers.GPT2DoubleHeadsModel(GPT2Config()) + 5 special tokens, torch DDP over NCCL, "
                                "AdamW (HF defaults) + clip_grad_norm_, step body of models/gpt2/train_gpt2_ddp.py:172-198; "
                                "replaced: ignite Engine loop -> for loop, PersonaChat -> synthetic [B,C,T] batches, "
                                "fp32 -> bf16 autocast" if precision == "bf16" else
                                "transformers.GPT2DoubleHeadsModel(GPT2Config()) + 5 special tokens, torch DDP over NCCL, "
                                "AdamW (HF defaults) + clip_grad_norm_, step body of models/gpt2/train_gpt2_ddp.py:172-198; "
                                "replaced: ignite Engine loop -> for loop, PersonaChat -> synthetic [B,C,T] batches"),
            "hyperparameters_from": hp["source"], "repo_code_on_path": bool(mapped or any(m.startswith("adapcc_b200") for m in sys.modules)),
            "config": {"model": "gpt2-small-double-heads (HF GPT2DoubleHeadsModel, vocab %d, %d params)" % (vocab, n_params),
                       "global_batch": a.batch * world, "per_gpu_batch": a.batch, "candidates": a.candidates,
                       "seq_len": seq, "parallelism": f"dp{world}", "engine": "torch DDP (stock, bucket_cap_mb=25)",
                       "optimizer": "torch.optim.AdamW(lr=%g, eps=1e-6, wd=0) + clip %.1f" % (hp["lr"], hp["max_norm"]),
                       "precision": precision, "attn_implementation": getattr(model.module.config, "_attn_implementation", None),
                       "l2": "working set (params+grads+optimizer state ~2 GB/step) exceeds the 50 MB L2; no flush needed"},
            "e2e": {"value": tokens / (ms_e2e * 1e-3), "unit": "tokens/s", "ms_per_step": ms_e2e,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4, "last_loss": last},
            "gpu_launches": 0, "clocks": clocks}), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    return 0
