"""GPT-2 small (double heads) data-parallel training — the reference's flagship workload
(/root/reference/models/gpt2/train_gpt2_ddp.py) on this library, with synthetic PersonaChat-shaped
batches (no network). Two engines:

  --engine flat  (default)  adapcc_b200.parallel.FlatDataParallel: flat bf16 grads in the symmetric
                            heap, zero-copy bucket all-reduce on a side stream, fused clip+AdamW,
                            optional --graph capture of the whole step;
  --engine ddp              torch DistributedDataParallel + AdapCC.communicator.cuda_allreduce_hook
                            (the reference's integration), AdamW lr 6.25e-5, clip 1.0.

    torchrun --nproc-per-node 8 examples/train_gpt2_ddp.py --steps 50 --entry_point 7
"""
import argparse
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from adapcc_b200 import ALLREDUCE  # noqa: E402
from adapcc_b200.adapcc import AdapCC  # noqa: E402
from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, lm_rows_needed, synthetic_batch  # noqa: E402
from adapcc_b200.parallel.ddp import ddp_accumulate, rebuild_buckets, wrap_ddp  # noqa: E402
from adapcc_b200.parallel.engine import FlatDataParallel  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--port", default="5000")
    p.add_argument("--strategy_file", default="./strategy/gpt2.xml")
    p.add_argument("--logical_graph", default="./topology/logical_graph.xml")
    p.add_argument("--entry_point", type=int, default=-1)
    p.add_argument("--parallel_degree", type=int, default=4)
    p.add_argument("--profile_freq", type=int, default=500)
    p.add_argument("--engine", default="flat", choices=["flat", "ddp"])
    p.add_argument("--graph", action="store_true")
    p.add_argument("--train_batch_size", type=int, default=4)
    p.add_argument("--num_candidates", type=int, default=2)
    p.add_argument("--seq_len", type=int, default=1024)
    p.add_argument("--lr", type=float, default=6.25e-5)
    p.add_argument("--max_norm", type=float, default=1.0)
    p.add_argument("--lm_coef", type=float, default=1.0)
    p.add_argument("--mc_coef", type=float, default=1.0)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--tiny", action="store_true")
    p.add_argument("--linear_decay", action="store_true",
                   help="flat engine: lr decays linearly to 0 over --steps (the schedule of the conversational-AI script the "
                        "reference's GPT-2 workload derives from; it imports ignite's PiecewiseLinear, "
                        "train_gpt2_ddp.py:21). Works under --graph: the kernel reads lr from a device scalar")
    p.add_argument("--checkpoint", default="", help="flat engine: resume from this file if it exists, write it at the end")
    p.add_argument("--fuse_add_ln", action="store_true", help="residual adds fused into the following LayerNorm")
    p.add_argument("--lm_rows", default="all", choices=["all", "scored"],
                   help="scored: LM head only on rows with a label (same loss/gradients, ~1/8 of the rows)")
    p.add_argument("--dropout", type=float, default=0.0,
                   help="embedding, residual and summary dropout probability (HF GPT-2's default is 0.1); 0: off")
    p.add_argument("--dropout_seed", type=int, default=0, help="seed of the dropout masks (rank r uses seed + r)")
    p.add_argument("--gradient_accumulation_steps", type=int, default=1,
                   help="micro-batches (of --train_batch_size each) per optimizer step; --steps counts optimizer steps")
    a = p.parse_args()
    M = a.gradient_accumulation_steps
    if M < 1:
        raise SystemExit("--gradient_accumulation_steps must be >= 1")

    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "1234")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    cfg = GPT2Config.tiny() if a.tiny else GPT2Config()
    cfg.embd_pdrop = cfg.resid_pdrop = cfg.summary_first_dropout = a.dropout
    torch.manual_seed(0)
    model = GPT2DoubleHeads(cfg).to(dev)
    a.heap_mb = (model.num_parameters() * 2 >> 20) + 64
    a.relay_control = a.engine == "ddp"
    AdapCC.init(a, local, rank, world)
    AdapCC.setup(ALLREDUCE)
    comm = AdapCC.communicator
    seq = min(a.seq_len, cfg.n_positions)
    batches = [synthetic_batch(a.train_batch_size, a.num_candidates, seq, cfg.vocab_size, device=dev, seed=rank * 100 + i)
               for i in range(4)]
    model.fuse_add_ln = a.fuse_add_ln or model.fuse_add_ln
    if a.lm_rows == "scored":                      # capacity from the host side of the loader, never a device sync
        model.lm_row_capacity = max(lm_rows_needed(b["lm_labels"].cpu()) for b in batches)
    if a.engine == "flat":
        eng = FlatDataParallel(model, comm.native if world > 1 else None, world_size=world, rank=rank, lr=a.lr,
                               max_norm=a.max_norm, dropout_seed=a.dropout_seed, gradient_accumulation_steps=M)
        if a.checkpoint and os.path.exists(a.checkpoint):            # before capture: the lr is baked into the graph
            eng.load_state_dict(torch.load(a.checkpoint, map_location="cpu", weights_only=False))
            if rank == 0:
                print("resumed from %s at step %d" % (a.checkpoint, eng.steps_done), flush=True)
        if a.graph:
            eng.capture([batches[j % len(batches)] for j in range(M)] if M > 1 else batches[0])
        step = (lambda b: eng.step_graph(b)) if a.graph else (lambda b: eng.step(b))
    else:
        model = model.bfloat16()
        model.set_dropout(a.dropout_seed + rank)
        ddp = wrap_ddp(model, comm, local, bucket_cap_mb=25)
        opt = torch.optim.AdamW(ddp.parameters(), lr=a.lr, fused=True)

        def step(micro, _i=[0]):
            comm.update_relay(step=_i[0])
            opt.zero_grad(set_to_none=False)
            loss = ddp_accumulate(ddp, micro if M > 1 else [micro], lm_coef=a.lm_coef, mc_coef=a.mc_coef)
            torch.nn.utils.clip_grad_norm_(ddp.parameters(), a.max_norm)
            opt.step()
            if _i[0] == 0:
                rebuild_buckets(ddp, comm)
            _i[0] += 1
            return loss

    for i in range(a.steps):
        if i and AdapCC.profile_freq and i % AdapCC.profile_freq == 0 and a.engine == "ddp":
            AdapCC.reconstruct_topology(a, ALLREDUCE)
        t0 = time.time()
        if a.linear_decay and a.engine == "flat":
            eng.set_lr(a.lr * max(0.0, 1.0 - i / max(1, a.steps)))
        loss = step([batches[(i * M + j) % len(batches)] for j in range(M)] if M > 1 else batches[i % len(batches)])
        torch.cuda.synchronize()
        if rank == 0:
            print("step %d loss %.4f computation time: %.3f" % (i, loss.item(), time.time() - t0), flush=True)
    comm.synchronize()
    if a.checkpoint and a.engine == "flat" and rank == 0:            # replicas are identical: one writer
        torch.save(eng.state_dict(), a.checkpoint + ".tmp")
        os.replace(a.checkpoint + ".tmp", a.checkpoint)
    AdapCC.clear(ALLREDUCE)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
