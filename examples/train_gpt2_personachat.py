"""GPT-2 double-heads fine-tuning on PersonaChat-format dialogues, end to end: tokenizer → dataset → distributed
loaders → training (LM + multiple-choice loss, AdamW, clip, linear lr decay) → per-epoch validation (hits@1 / NLL /
perplexity) → checkpoint. The full data path of the reference's workload
(/root/reference/models/gpt2/train_gpt2_ddp.py:120-214: tokenizer, ``get_data_loaders``, ignite trainer + evaluator +
``PiecewiseLinear`` + ``ModelCheckpoint``), where ``examples/train_gpt2_ddp.py`` / ``bench.py`` only time the step on
synthetic tensors.

    torchrun --nproc-per-node 8 examples/train_gpt2_personachat.py --dataset_path personachat_self_original.json --graph
    torchrun --nproc-per-node 2 examples/train_gpt2_personachat.py --backend gloo --tiny --n_epochs 2     # CPU

No file given → template dialogues in the same schema are generated (no network here). CUDA: the flat engine
(zero-copy buckets, ZeRO-1, fused optimizer, optional whole-step CUDA graph) fed by a pinned-memory prefetcher;
``--backend gloo``: torch DDP + the communicator's hook on the CPU executor.
"""
import argparse
import math
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from adapcc_b200 import ALLREDUCE  # noqa: E402
from adapcc_b200.adapcc import AdapCC  # noqa: E402
from adapcc_b200.data import (DialogTokenizer, corpus_of, get_data_loaders, micro_batch_groups,  # noqa: E402
                              synthetic_personachat)
from adapcc_b200.eval import evaluate_tensors, pack_checkpoint  # noqa: E402
from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads  # noqa: E402
from adapcc_b200.parallel.ddp import ddp_accumulate  # noqa: E402


def build_tokenizer(a, cfg, rank):
    """Load the tokenizer file, or (rank 0) build it — from the published GPT-2 vocabulary if a directory is given,
    else by training byte-level BPE on the corpus — then everybody loads the same file."""
    if not os.path.exists(a.tokenizer):
        if rank == 0:
            if a.gpt2_vocab_dir:
                tok = DialogTokenizer.from_gpt2_files(a.gpt2_vocab_dir, cfg.vocab_size)
            else:
                import json

                raw = json.load(open(a.dataset_path, encoding="utf-8")) if a.dataset_path else synthetic_personachat(**a.synthetic)
                tok = DialogTokenizer.train(corpus_of(raw), vocab_size=min(a.bpe_vocab, cfg.vocab_size - 5),
                                            model_vocab=cfg.vocab_size)
            tok.save(a.tokenizer)
        if dist.is_initialized():
            dist.barrier()
    return DialogTokenizer.load(a.tokenizer)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--dataset_path", default="", help="PersonaChat-schema JSON; empty: synthetic dialogues")
    p.add_argument("--dataset_cache", default="", help="prefix of the tokenized-dataset cache file")
    p.add_argument("--tokenizer", default="./dialog_tokenizer.json")
    p.add_argument("--gpt2_vocab_dir", default="", help="directory with GPT-2's vocab.json + merges.txt (optional)")
    p.add_argument("--bpe_vocab", type=int, default=8192)
    p.add_argument("--synthetic_dialogs", type=int, default=256)
    p.add_argument("--num_candidates", type=int, default=2)
    p.add_argument("--max_history", type=int, default=2)
    p.add_argument("--personality_permutations", type=int, default=1)
    p.add_argument("--train_batch_size", type=int, default=4)
    p.add_argument("--valid_batch_size", type=int, default=4)
    p.add_argument("--seq_len", type=int, default=0, help="0: longest input rounded up to 64")
    p.add_argument("--n_epochs", type=int, default=3)
    p.add_argument("--max_steps", type=int, default=0)
    p.add_argument("--lr", type=float, default=6.25e-5)
    p.add_argument("--lm_coef", type=float, default=1.0)
    p.add_argument("--mc_coef", type=float, default=1.0)
    p.add_argument("--max_norm", type=float, default=1.0)
    p.add_argument("--eval_before_start", action="store_true")
    p.add_argument("--graph", action="store_true", help="CUDA: capture the whole step once and replay it")
    p.add_argument("--checkpoint", default="", help="written after every epoch (rank 0), resumed from if present")
    p.add_argument("--tiny", action="store_true")
    p.add_argument("--backend", default="nccl", choices=["nccl", "gloo"])
    p.add_argument("--port", default="5000")
    p.add_argument("--strategy_file", default="./strategy/gpt2.xml")
    p.add_argument("--logical_graph", default="./topology/logical_graph.xml")
    p.add_argument("--entry_point", type=int, default=-1)
    p.add_argument("--parallel_degree", type=int, default=4)
    p.add_argument("--profile_freq", type=int, default=0)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--dropout", type=float, default=0.0,
                   help="embedding, residual and summary dropout probability (HF GPT-2's default is 0.1); 0: off")
    p.add_argument("--dropout_seed", type=int, default=0, help="seed of the dropout masks (rank r uses seed + r)")
    p.add_argument("--gradient_accumulation_steps", type=int, default=1,
                   help="micro-batches (of --train_batch_size each) per optimizer step; steps count optimizer steps")
    a = p.parse_args()
    M = a.gradient_accumulation_steps
    if M < 1:
        raise SystemExit("--gradient_accumulation_steps must be >= 1")
    a.synthetic = dict(n_train=a.synthetic_dialogs, n_valid=max(8, a.synthetic_dialogs // 8), n_candidates=4, seed=a.seed)

    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    cuda = a.backend == "nccl" and torch.cuda.is_available()
    dev = torch.device("cuda", local) if cuda else torch.device("cpu")
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "1234")
    if cuda:
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        a.backend = "gloo"
        dist.init_process_group("gloo", rank=rank, world_size=world)

    cfg = GPT2Config.tiny() if a.tiny else GPT2Config()
    cfg.embd_pdrop = cfg.resid_pdrop = cfg.summary_first_dropout = a.dropout
    if a.tiny:
        cfg.n_positions = 128
    tok = build_tokenizer(a, cfg, rank)
    train_loader, valid_loader, train_sampler, _ = get_data_loaders(a, tok, distributed=world > 1, rank=rank, world_size=world,
                                                                   seq_len=min(a.seq_len, cfg.n_positions) or None)
    T = train_loader.dataset.tensors["input_ids"].shape[-1]
    if T > cfg.n_positions:
        raise SystemExit(f"inputs are {T} tokens long, the model has {cfg.n_positions} positions: pass --seq_len")
    steps_per_epoch = len(train_loader) // M                      # optimizer steps; a partial last group is skipped
    if steps_per_epoch == 0:
        raise SystemExit(f"{len(train_loader)} batches per epoch are fewer than --gradient_accumulation_steps {M}")
    total_steps = a.n_epochs * steps_per_epoch if not a.max_steps else min(a.max_steps, a.n_epochs * steps_per_epoch)
    if rank == 0:
        print(f"train {tuple(train_loader.dataset.tensors['input_ids'].shape)} valid "
              f"{tuple(valid_loader.dataset.tensors['input_ids'].shape)} (N, candidates, T); {steps_per_epoch} steps/epoch/rank of {M} micro-batch(es); "
              f"vocab {tok.base_vocab} + 5 special of {cfg.vocab_size}", flush=True)

    torch.manual_seed(a.seed)
    model = GPT2DoubleHeads(cfg).to(dev)
    a.relay_control = not cuda and world > 1
    a.heap_mb = ((model.num_parameters() * 4 >> 20) + 64) if cuda else 0
    AdapCC.init(a, local, rank, world)
    AdapCC.setup(ALLREDUCE)
    comm = AdapCC.communicator
    eng = ddp = opt = None
    start_epoch = 0
    if cuda:
        from adapcc_b200.parallel.engine import FlatDataParallel

        eng = FlatDataParallel(model, comm.native if world > 1 else None, world_size=world, rank=rank, lr=a.lr,
                               max_norm=a.max_norm, weight_decay=0.0, dropout_seed=a.dropout_seed,
                               gradient_accumulation_steps=M)
        if a.checkpoint and os.path.exists(a.checkpoint):
            ck = torch.load(a.checkpoint, map_location="cpu", weights_only=False)
            eng.load_state_dict(ck["engine"])
            start_epoch = int(ck.get("epoch", -1)) + 1
    else:
        from adapcc_b200.parallel.ddp import wrap_ddp

        model.set_dropout(a.dropout_seed + rank)
        ddp = wrap_ddp(model, comm, local, zero_copy=False) if world > 1 else model
        opt = torch.optim.AdamW(model.parameters(), lr=a.lr, weight_decay=0.0)
        if a.checkpoint and os.path.exists(a.checkpoint):
            ck = torch.load(a.checkpoint, map_location="cpu", weights_only=False)
            model.load_state_dict(ck["model"])
            if "dropout" in ck:                           # continue the mask sequence (the flat engine does it itself)
                model.set_dropout(ck["dropout"]["seed"] + rank, ck["dropout"]["step"])
            start_epoch = int(ck.get("epoch", -1)) + 1

    def validate(tag):
        model.eval()
        m = evaluate_tensors(model, valid_loader, device=dev)
        model.train()
        if world > 1:                                   # every rank scored its shard of the validation set
            t = torch.tensor([m["hits"], m["examples"], m["nll_sum"], m["tokens"]], dtype=torch.float64, device=dev)
            dist.all_reduce(t)
            hits, n, nll_sum, ntok = t.tolist()
            nll = nll_sum / max(1.0, ntok)
            m = {"hits@1": hits / max(1.0, n), "nll": nll, "ppl": math.exp(min(nll, 50.0)), "examples": int(n), "tokens": int(ntok)}
        if rank == 0:
            print(f"validation {tag}: accuracy(hits@1) {m['hits@1']:.4f} nll {m['nll']:.4f} average_ppl {m['ppl']:.2f} "
                  f"({m['examples']} examples, {m['tokens']} reply tokens)", flush=True)
        return m

    if a.eval_before_start:
        validate("before training")
    step = start_epoch * steps_per_epoch
    captured = False
    for epoch in range(start_epoch, a.n_epochs):
        if train_sampler is not None:
            train_sampler.set_epoch(epoch)
        t0, seen, run_loss = time.time(), 0, None
        for micro in micro_batch_groups(train_loader, dev, M):
            if step >= total_steps:
                break
            lr = a.lr * max(0.0, 1.0 - step / max(1, total_steps))            # PiecewiseLinear(lr -> 0)
            if eng is not None:
                eng.set_lr(lr)
                inputs = micro if M > 1 else micro[0]
                if a.graph and not captured:
                    eng.capture(inputs)
                    captured = True
                loss = eng.step_graph(inputs) if a.graph else eng.step(inputs)
            else:
                for g in opt.param_groups:
                    g["lr"] = lr
                comm.update_relay(step)
                opt.zero_grad(set_to_none=False)
                loss = ddp_accumulate(ddp, micro, lm_coef=a.lm_coef, mc_coef=a.mc_coef)
                torch.nn.utils.clip_grad_norm_(model.parameters(), a.max_norm)
                opt.step()
            step += 1
            seen += sum(b["input_ids"].numel() for b in micro)
            if step % 10 == 0 or step == total_steps:
                v = float(loss)                                                # one device→host read per 10 steps
                run_loss = v if run_loss is None else 0.98 * run_loss + 0.02 * v
                if rank == 0:
                    print(f"epoch {epoch} step {step}/{total_steps} loss {v:.4f} (running {run_loss:.4f}) lr {lr:.3e}", flush=True)
        if cuda:
            torch.cuda.synchronize()
        dt = time.time() - t0
        if rank == 0 and seen:
            print(f"epoch {epoch}: {seen * world / dt:,.0f} tokens/s ({dt:.1f} s)", flush=True)
        validate(f"epoch {epoch}")
        if a.checkpoint:
            extra = {"epoch": epoch}
            if eng is None and model.has_dropout:         # rank 0's seed is the base seed; every rank has run as many steps
                extra["dropout"] = {"seed": int(model.dropout_seed) - rank, "step": int(model.dropout_step)}
            ck = pack_checkpoint(model, os.path.abspath(a.tokenizer), eng, extra)   # collective under ZeRO-1
            if rank == 0:
                torch.save(ck, a.checkpoint + ".tmp")
                os.replace(a.checkpoint + ".tmp", a.checkpoint)
        if step >= total_steps:
            break
    comm.synchronize()
    AdapCC.clear(ALLREDUCE)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
