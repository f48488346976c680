"""One rank per GPU, world 2: Trainer(pack=True) under the peer-HBM DDP path on 512-padded long-text batches.  Each
rank packs its own batch into bins of the length it needs (128 to 512 tokens); the loss trajectory must follow the
oracle's DDP restatement (oracle/ddp_ref.py) on the PADDED batches, and the ranks must hold the same weights.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29605 \
        tests/ddp_pack_long_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist

from parity import TOL_TRAJ, b2, make_model, state_from_hf_init
from test_packing_long import LONG_TEXT, long_batch, long_config

STEPS = 4


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from oracle import ddp_ref
    cfg = long_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    batches = [[long_batch(cfg, 8, 1000 + 10 * s + r, **LONG_TEXT[(s + 2 * r) % 5]) for r in range(world)]
               for s in range(STEPS)]
    hist = ddp_ref.train({k: v.clone() for k, v in state.items()}, cfg, batches)
    model = make_model(cfg, state, dev)
    net = b2.DistributedDataParallel(model, device_ids=[local])
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank, args.pack = local, world, rank, True
    opt = b2.build_optimizer(net, args)
    tr = b2.Trainer(args, cfg, net, torch.nn.CrossEntropyLoss(), opt)
    worst = 0.0
    for s in range(STEPS):
        mean = float(tr.train_step(batches[s][rank]))
        worst = max(worst, abs(mean - float(hist[s]["loss_mean"])))
    lens = sorted({key[2] for key in tr._packed})
    sh = model._engine.shadow.view(torch.int16).to(torch.int64)
    sig = torch.stack([sh.sum(), (sh * (torch.arange(sh.numel(), device=dev) % 8191 + 1)).sum()])
    sigs = [torch.zeros_like(sig) for _ in range(world)]
    dist.all_gather(sigs, sig)
    stats = torch.tensor([worst], dtype=torch.float64, device=dev)
    dist.all_reduce(stats, op=dist.ReduceOp.MAX)
    worst = float(stats[0])
    if rank == 0:
        print("ddp_pack_long_worker: worst |dloss_mean| %.2e (tol %.0e), bin lengths on rank 0: %s"
              % (worst, TOL_TRAJ, lens), flush=True)
    assert all(torch.equal(x, sigs[0]) for x in sigs), "ranks hold different weights"
    assert worst <= TOL_TRAJ
    torch.cuda.synchronize()
    dist.barrier()
    net.close()
    if rank == 0:
        print("ddp_pack_long_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
