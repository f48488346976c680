"""One rank per GPU: BertForMultipleChoice under the peer-HBM DistributedDataParallel wrapper, through the Trainer's
eager, captured (fused) and packed paths, in the kernel and the copy-engine exchange form.  The rank-mean loss
trajectory must follow the oracle's DDP restatement (tests/mc_oracle.py: per-rank HF loss, gradients averaged over the
ranks).  The ranks must hold the same weights, and dev() must equal a host
recomputation over every rank's examples (loss_reduce of the loss, all_gather_rows of the [B, N] logits and the
labels).
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29643 \
        tests/ddp_mc_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist

import mc_oracle as mc
from parity import TOL_TRAJ, adamw_ref, b2, tiny_config

STEPS = 4
LR = 1e-3
PATHS = {"eager": dict(fused=False), "fused": dict(fused=True), "packed": dict(fused=True, pack=True)}


def ddp_ref(state, cfg, batches):
    ref = {k: v.clone() for k, v in state.items()}
    opt = adamw_ref.HFAdamW(ref, lr=LR, weight_decay=0.01)
    means = []
    for rank_batches in batches:
        out = [mc.loss_and_grads(ref, cfg, b) for b in rank_batches]
        means.append(float(torch.stack([o[0] for o in out]).mean()))
        opt.step({k: sum(o[2][k] for o in out) / len(out) for k in ref})
    return means


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = mc.mc_state_from_hf_init(cfg)
    batches = [[b2.synthetic_mc_batch(cfg, 4, 4, 128, 2000 + 10 * s + r, padded=True) for r in range(world)]
               for s in range(STEPS)]
    hist = ddp_ref(state, cfg, batches)
    for dma in ("0", "1"):
        os.environ["B2_DDP_DMA"] = dma
        for path, extra in PATHS.items():
            model = b2.BertForMultipleChoice(cfg)
            model.load_state_dict(state, strict=True)
            model.to(dev)
            net = b2.DistributedDataParallel(model, device_ids=[local])
            args = b2.Args()
            args.local_rank, args.local_world_size, args.rank, args.learning_rate = local, world, rank, LR
            for k, v in extra.items():
                setattr(args, k, v)
            opt = b2.build_optimizer(net, args)
            tr = b2.Trainer(args, cfg, net, None, opt)
            worst = 0.0
            for s in range(STEPS):
                worst = max(worst, abs(float(tr.train_step(batches[s][rank])) - hist[s]))
            torch.cuda.synchronize()
            sh = model._engine.shadow.view(torch.int16).to(torch.int64)
            sig = torch.stack([sh.sum(), (sh * (torch.arange(sh.numel(), device=dev) % 8191 + 1)).sum()])
            sigs = [torch.zeros_like(sig) for _ in range(world)]
            dist.all_gather(sigs, sig)
            stats = torch.tensor([worst], dtype=torch.float64, device=dev)
            dist.all_reduce(stats, op=dist.ReduceOp.MAX)
            worst = float(stats[0])
            assert all(torch.equal(x, sigs[0]) for x in sigs), "%s: ranks hold different weights" % path
            assert worst <= TOL_TRAJ, (dma, path, worst)
            loader = [b2.synthetic_mc_batch(cfg, 4, 4, 128, 3000 + 10 * i + rank, padded=True) for i in range(2)]
            loss, acc = tr.dev(loader)
            want_loss, counts = 0.0, torch.zeros(2, dtype=torch.float64, device=dev)
            model.eval()
            for bt in loader:
                d = {k: v.to(dev) for k, v in bt.items()}
                with torch.no_grad():
                    o = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                              attention_mask=d["attention_mask"], labels=d["label"])
                l = o.loss.reshape(1).clone()
                dist.all_reduce(l)
                want_loss += float(l) / world
                hit = o.logits.argmax(1) == d["label"]
                counts += torch.tensor([float(hit.sum()), float(hit.numel())], dtype=torch.float64, device=dev)
            dist.all_reduce(counts)
            assert abs(float(loss) - want_loss) <= 1e-5 * max(1.0, want_loss), (path, float(loss), want_loss)
            assert abs(acc - float(counts[0] / counts[1])) <= 1e-12, (path, acc, counts)
            if rank == 0:
                print("ddp_mc_worker: dma=%s %s worst |dloss_mean| %.2e (tol %.0e), dev accuracy %.4f"
                      % (dma, path, worst, TOL_TRAJ, acc), flush=True)
            torch.cuda.synchronize()
            dist.barrier()
            net.close()
    if rank == 0:
        print("ddp_mc_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
