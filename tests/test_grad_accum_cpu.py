"""Gradient accumulation without a GPU: ``FlatDataParallel``'s argument and input checks, ``micro_batch_groups``
handing out the loader's batches in order, the PersonaChat example with ``--gradient_accumulation_steps 2`` on 2 gloo
ranks, and ``ddp_accumulate`` (``no_sync`` for all but the last micro-batch, each loss times 1/M) on
DistributedDataParallel against autograd over the mean of the micro-batch losses.

This file is also the worker of the last test:

    torchrun --nproc-per-node 2 tests/test_grad_accum_cpu.py
"""
import os
import socket
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch  # noqa: E402


def _engine(M, **kw):
    from adapcc_b200.parallel.engine import FlatDataParallel

    torch.manual_seed(0)
    return FlatDataParallel(GPT2DoubleHeads(GPT2Config.tiny()), None, world_size=1, gradient_accumulation_steps=M, **kw)


def test_argument_errors():
    for bad in (0, -1, 1.5, True, "2", None):
        with pytest.raises(ValueError, match="gradient_accumulation_steps must be an int >= 1"):
            _engine(bad)
    assert _engine(1).grad_acc is None
    eng = _engine(2)
    assert eng.grad_acc.dtype == torch.float32 and eng.grad_acc.numel() == eng.total
    b = synthetic_batch(2, 2, 32, 512, seed=1)
    short = synthetic_batch(2, 2, 16, 512, seed=2)
    for method in (eng.step, eng.capture):
        with pytest.raises(ValueError, match="got one dict"):
            method(b)
        for wrong in ([b], [b, b, b], []):
            with pytest.raises(ValueError, match=f"takes 2 micro-batch dicts, got {len(wrong)} items"):
                method(wrong)
        with pytest.raises(ValueError, match="micro-batch 1 has shapes"):
            method([b, short])
        with pytest.raises(ValueError, match="micro-batch 1 has shapes"):
            method([b, {k: v for k, v in b.items() if k != "mc_labels"}])
        with pytest.raises(ValueError, match="expected a batch dict or a sequence"):
            method("batch")
    with pytest.raises(ValueError, match="the captured step has"):
        eng._micro_batches([short, short], "step_graph", [b, b])
    assert len(eng._micro_batches((b, b), "step")) == 2
    assert eng.steps_done == 0


def test_micro_batch_groups_are_the_loaders_batches_in_order():
    """Each group holds M consecutive batches of the loader, checked when the group is handed out (when a step uses
    it), for group sizes past the prefetcher's default ring of two slots; an incomplete last group is dropped. A group
    collected from the default two-slot prefetcher instead would hold batch k + 2 where batch k belongs."""
    from adapcc_b200.data import PinnedPrefetcher, micro_batch_groups

    loader = [{"x": torch.full((3, 5), float(i)), "y": torch.arange(4) + 10 * i} for i in range(11)]
    for M in (1, 2, 3, 4, 5):
        seen = []
        for group in micro_batch_groups(loader, "cpu", M):
            assert len(group) == M
            k = len(seen)
            for j, b in enumerate(group):
                assert torch.equal(b["x"], loader[k + j]["x"]) and torch.equal(b["y"], loader[k + j]["y"]), (M, k, j)
            seen.extend(int(b["x"][0, 0]) for b in group)
        assert seen == list(range(11 // M * M)), (M, seen)
    kept = []                                          # what collecting from the default ring would hand a step
    for b in PinnedPrefetcher(loader[:3], "cpu"):
        kept.append(b)
    assert [int(b["x"][0, 0]) for b in kept] == [2, 1, 2]
    with pytest.raises(ValueError, match="M must be >= 1"):
        next(micro_batch_groups(loader, "cpu", 0))


def _port():
    with socket.socket() as sock:
        sock.bind(("127.0.0.1", 0))
        return sock.getsockname()[1]


def test_personachat_example_with_accumulation(tmp_path):
    """``--tiny --backend gloo --gradient_accumulation_steps 2 --max_steps 2`` on 2 ranks completes both optimizer
    steps (four micro-batches per rank) and validates."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2", ADAPCC_COORD_PORT=str(_port()))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(_port()), os.path.join(ROOT, "examples", "train_gpt2_personachat.py"),
           "--backend", "gloo", "--tiny", "--synthetic_dialogs", "24", "--n_epochs", "1", "--max_steps", "2",
           "--gradient_accumulation_steps", "2", "--port", str(_port())]
    r = subprocess.run(cmd, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    assert "of 2 micro-batch(es)" in r.stdout, r.stdout[-1500:]
    assert "step 2/2 loss" in r.stdout, r.stdout[-1500:]
    assert "validation epoch 0" in r.stdout, r.stdout[-1500:]


def test_no_sync_branch_gradient_matches_autograd(tmp_path):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(_port()), os.path.abspath(__file__)]
    r = subprocess.run(cmd, cwd=tmp_path, capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2"))
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    assert r.stdout.count(" OK\n") == 2, r.stdout[-3000:]


def _worker():
    """Each rank: two micro-batches of its own through ``ddp_accumulate`` (what both GPT-2 examples' DDP branches call)
    on DistributedDataParallel (gloo), against autograd of the mean of the same two losses on a copy of the model,
    averaged over the ranks."""
    import copy

    import torch.distributed as dist
    from torch.nn.parallel import DistributedDataParallel as DDP

    from adapcc_b200.parallel.ddp import ddp_accumulate

    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    torch.manual_seed(0)
    model = GPT2DoubleHeads(GPT2Config.tiny())
    ref = copy.deepcopy(model)
    ddp = DDP(model)
    micro = [synthetic_batch(2, 2, 32, 512, seed=10 * rank + j) for j in range(2)]
    loss = ddp_accumulate(ddp, micro, lm_coef=2.0, mc_coef=0.5)
    losses = [ref(**b, lm_coef=2.0, mc_coef=0.5)[0] for b in micro]
    mean = (losses[0] + losses[1]) / 2
    want = torch.autograd.grad(mean, list(ref.parameters()))
    mean = mean.detach()
    ok = abs(float(loss) - float(mean)) <= 1e-6 * abs(float(mean))
    worst = 0.0
    for p, g in zip(model.parameters(), want):
        g = g.clone()
        dist.all_reduce(g)
        g /= world
        err = float((p.grad - g).abs().max()) / max(float(g.abs().max()), 1e-30)
        worst = max(worst, err)
    ok &= worst <= 1e-4
    # the ranks' gradients are all-reduced once: every rank holds the same
    flat = torch.cat([p.grad.flatten() for p in model.parameters()])
    other = flat.clone()
    dist.broadcast(other, src=0)
    ok &= bool(torch.equal(flat, other))
    print(f"[rank {rank}] loss {float(loss):.6f} (autograd {float(mean):.6f}), largest relative gradient error "
          f"{worst:.2e} {'OK' if ok else 'FAIL'}", flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    _worker()
