"""One rank per GPU, world 2, under torch.use_deterministic_algorithms(True): two runs of the same Trainer program
(same weights, dropout 0.1 from the same RNG state, same batches per rank) must leave every rank with bitwise the same
losses, bf16 gradients, fp32 masters and optimizer state in both gradient-exchange forms (B2_DDP_DMA = 0 and 1).
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29611 \
        tests/ddp_determinism_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist

from parity import b2, make_model, state_from_hf_init, tiny_config
from test_determinism import _snapshot, assert_bitwise_equal
from test_packing import short_batch

STEPS = 3


def run(cfg, state, batches, dev, local, world, rank, dma):
    os.environ["B2_DDP_DMA"] = dma
    model = make_model(cfg, state, dev)
    model.set_dropout_rng_state([91 + rank, 0])
    net = b2.DistributedDataParallel(model, device_ids=[local])
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank, args.full_determinism = local, world, rank, True
    opt = b2.build_optimizer(net, args)
    tr = b2.Trainer(args, cfg, net, torch.nn.CrossEntropyLoss(), opt)
    losses = [tr.train_step(b).clone() for b in batches]
    snap = _snapshot(model, opt, losses)
    torch.cuda.synchronize()
    dist.barrier()
    net.close()
    return snap


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = [short_batch(cfg, 8, 2000 + 10 * s + rank) for s in range(STEPS)]
    for dma in ("0", "1"):
        a = run(cfg, state, batches, dev, local, world, rank, dma)
        b = run(cfg, state, batches, dev, local, world, rank, dma)
        assert_bitwise_equal(a, b)
        if rank == 0:
            print("ddp_determinism_worker: B2_DDP_DMA=%s: two runs bitwise equal" % dma, flush=True)
    torch.use_deterministic_algorithms(False)
    dist.barrier()
    if rank == 0:
        print("ddp_determinism_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
