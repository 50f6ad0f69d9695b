"""Worker of tests/test_dropout_cpu.py::test_ddp_leaves_the_dropout_state_alone (gloo ranks under torch.distributed.run):
the model's dropout state under DistributedDataParallel, plain and through ``wrap_ddp``'s stock path."""
import dataclasses
import os

import torch
import torch.distributed as dist
from torch.nn.parallel import DistributedDataParallel as DDP

from adapcc_b200.models.gpt2 import GPT2Config, GPT2DoubleHeads, synthetic_batch


def main():
    rank = int(os.environ["RANK"])
    dist.init_process_group("gloo")
    batch = synthetic_batch(1, 2, 16, 512, seed=rank)
    for p in (0.0, 0.1):
        torch.manual_seed(0)
        cfg = dataclasses.replace(GPT2Config.tiny(), embd_pdrop=p, resid_pdrop=p, summary_first_dropout=p)
        model = GPT2DoubleHeads(cfg)
        assert not list(model.buffers()), [n for n, _ in model.named_buffers()]
        model.set_dropout(100 + rank, 5 * rank)
        ddp = DDP(model)
        sync = ddp.will_sync_module_buffers()
        seed_wrapped = int(model.dropout_seed)
        ddp(**batch)[0].backward()
        steps = 5 * rank + (1 if p else 0)
        ok = (not sync and seed_wrapped == 100 + rank and int(model.dropout_seed) == 100 + rank
              and int(model.dropout_step) == steps)
        print(f"[rank {rank}] p {p} sync_buffers {sync} seed {int(model.dropout_seed)} step {int(model.dropout_step)} "
              f"{'ok' if ok else 'WRONG'}", flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
