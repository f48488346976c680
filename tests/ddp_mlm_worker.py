"""One rank per GPU: BertForMaskedLM under the peer-HBM DistributedDataParallel wrapper, through the Trainer's eager,
captured (fused) and packed paths.  Each path's rank-mean loss trajectory must follow the masked-LM oracle's DDP
restatement (tests/mlm_oracle.py: per-rank HF loss, gradients averaged over the ranks, torch AdamW with HF AdamW's
eps and no weight decay), and the ranks must hold the same weights -- the tied word-embedding gradient, whose decoder
part lands on rows no rank's batch touches, is exchanged in the embeddings bucket.  dev() must equal a host
recomputation over every rank's labelled tokens.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29627 \
        tests/ddp_mlm_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist
import torch.nn.functional as F

import mlm_oracle as mlm
from parity import TOL_TRAJ, b2, tiny_config

STEPS = 4
LR = 1e-3
PATHS = {"eager": dict(fused=False), "fused": dict(fused=True), "packed": dict(fused=True, pack=True)}


def oracle_losses(state, cfg, batches, world):
    ref = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    opt = torch.optim.AdamW(list(ref.values()), lr=LR, eps=1e-6, weight_decay=0.0)
    out = []
    for per_rank in batches:
        opt.zero_grad()
        total = 0.0
        for bt in per_rank:
            loss, _ = mlm.forward(ref, cfg, bt["input_ids"], None, bt["attention_mask"], bt["label"])
            (loss / world).backward()
            total += float(loss) / world
        opt.step()
        out.append(total)
    return out


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = tiny_config(vocab_size=1000, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = mlm.mlm_state_from_hf_init(cfg)
    batches = [[b2.synthetic_mlm_batch(cfg, 4, 128, 2000 + 10 * s + r, padded=True) for r in range(world)]
               for s in range(STEPS)]
    want = oracle_losses(state, cfg, batches, world)
    for path, extra in PATHS.items():
        model = b2.BertForMaskedLM(cfg)
        model.load_state_dict(state, strict=True)
        model.to(dev)
        net = b2.DistributedDataParallel(model, device_ids=[local])
        args = b2.Args()
        args.local_rank, args.local_world_size, args.rank, args.learning_rate = local, world, rank, LR
        args.weight_decay = 0.0
        for k, v in extra.items():
            setattr(args, k, v)
        opt = b2.build_optimizer(net, args)
        tr = b2.Trainer(args, cfg, net, None, opt)
        worst = 0.0
        for s in range(STEPS):
            mean = float(tr.train_step(batches[s][rank]))
            worst = max(worst, abs(mean - want[s]))
        torch.cuda.synchronize()
        sh = model._engine.shadow.view(torch.int16).to(torch.int64)
        sig = torch.stack([sh.sum(), (sh * (torch.arange(sh.numel(), device=dev) % 8191 + 1)).sum()])
        sigs = [torch.zeros_like(sig) for _ in range(world)]
        dist.all_gather(sigs, sig)
        stats = torch.tensor([worst], dtype=torch.float64, device=dev)
        dist.all_reduce(stats, op=dist.ReduceOp.MAX)
        worst = float(stats[0])
        assert all(torch.equal(x, sigs[0]) for x in sigs), "%s: ranks hold different weights" % path
        assert worst <= TOL_TRAJ, (path, worst)
        loader = [b2.synthetic_mlm_batch(cfg, 4, 128, 3000 + 10 * i + rank, padded=True) for i in range(2)]
        loss, acc = tr.dev(loader)
        model.eval()
        want_loss, counts = 0.0, torch.zeros(2, dtype=torch.float64, device=dev)
        with torch.no_grad():
            for bt in loader:
                z = model(input_ids=bt["input_ids"].to(dev), attention_mask=bt["attention_mask"].to(dev)).logits
                y = bt["label"].to(dev).reshape(-1)
                l = F.cross_entropy(z.reshape(-1, cfg.vocab_size).double(), y).reshape(1)
                dist.all_reduce(l)
                want_loss += float(l) / world
                keep = y != -100
                pred = z.reshape(-1, cfg.vocab_size).argmax(-1)
                counts += torch.tensor([float((pred[keep] == y[keep]).sum()), float(keep.sum())],
                                       dtype=torch.float64, device=dev)
        dist.all_reduce(counts)
        assert abs(float(loss) - want_loss) <= 1e-3 * max(1.0, want_loss), (path, float(loss), want_loss)
        assert abs(acc - float(counts[0] / counts[1])) <= 2.0 / float(counts[1]), (path, acc, counts)
        if rank == 0:
            print("ddp_mlm_worker: %s worst |dloss_mean| %.2e (tol %.0e), dev acc %.4f" % (path, worst, TOL_TRAJ, acc),
                  flush=True)
        torch.cuda.synchronize()
        dist.barrier()
        net.close()
    if rank == 0:
        print("ddp_mlm_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
