"""One rank per GPU, world 2: a torch LambdaLR with multipliers 1, 0, 1, 0, ... on the Trainer's captured DDP step
(tests/test_lr_schedule.py runs it).  The ranks' bf16 weights are bitwise equal after every step, the zero-lr steps
leave them bitwise unchanged and the others move them.  Exits non-zero on any mismatch.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29593 \
        tests/ddp_lr_schedule_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist
from torch.optim.lr_scheduler import LambdaLR

from parity import b2, bert_ref, state_from_hf_init, tiny_config

STEPS = 6


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = tiny_config()
    model = b2.BertForSequenceClassification(cfg)
    model.load_state_dict(state_from_hf_init(cfg, seed=123))
    model.cuda()
    net = b2.DistributedDataParallel(model, device_ids=[local])
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank = local, world, rank
    opt = b2.build_optimizer(net, args)
    sched = LambdaLR(opt, lambda s: float(s % 2 == 0))
    tr = b2.Trainer(args, cfg, net, torch.nn.CrossEntropyLoss(), opt, scheduler=sched)
    for s in range(STEPS):
        before = model._engine.shadow.clone()
        tr.train_step(bert_ref.synthetic_batch(cfg, 4, 128, 9300 + 10 * s + rank, padded=True))
        torch.cuda.synchronize()
        sh = model._engine.shadow
        shs = [torch.zeros_like(sh.view(torch.int16)) for _ in range(world)]
        dist.all_gather(shs, sh.view(torch.int16))
        assert all(torch.equal(x, shs[0]) for x in shs), "step %d: ranks hold different bf16 weights" % s
        if s % 2 == 1:
            assert torch.equal(sh, before), "step %d has lr 0 but the weights moved" % s
        else:
            assert not torch.equal(sh, before), "step %d did not move the weights" % s
    assert sched.last_epoch == STEPS
    torch.cuda.synchronize()
    dist.barrier()
    net.close()
    if rank == 0:
        print("ddp_lr_schedule_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
