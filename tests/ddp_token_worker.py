"""One rank per GPU: BertForTokenClassification under the peer-HBM DistributedDataParallel wrapper, through the
Trainer's eager, captured (fused) and packed paths.  Each path's rank-mean loss trajectory and its AdamW first moments
must follow the token oracle's DDP restatement (tests/token_oracle.py: per-rank HF loss, gradients averaged over the
ranks), the ranks must hold the same weights, and dev() / test() must equal a host recomputation over every rank's
tokens (loss_reduce of the scalar loss, all_gather_rows of [B, S, C] logits and [B, S] labels).
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29617 \
        tests/ddp_token_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist
import torch.nn.functional as F

import token_oracle as tok
from parity import TOL_GRAD_REL_QK, TOL_TRAJ, assert_grads_within_tolerance, b2, tiny_config

STEPS = 4
LR = 1e-3
PATHS = {"eager": dict(fused=False), "fused": dict(fused=True), "packed": dict(fused=True, pack=True)}


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = tiny_config(num_labels=9, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = tok.token_state_from_hf_init(cfg)
    batches = [[tok.token_batch(cfg, 4, 128, 2000 + 10 * s + r) for r in range(world)] for s in range(STEPS)]
    ref = {k: v.clone() for k, v in state.items()}
    hist, ref_opt = tok.ddp_train(ref, cfg, batches, lr=LR)
    ref_m = {n: ref_opt.state[n]["exp_avg"] for n in ref}
    for path, extra in PATHS.items():
        model = b2.BertForTokenClassification(cfg)
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
            mean = float(tr.train_step(batches[s][rank]))
            worst = max(worst, abs(mean - float(hist[s]["loss_mean"])))
        torch.cuda.synchronize()
        moments = {n: ea.detach().cpu() for n, (ea, _v) in opt.moments().items()}
        qk, other = assert_grads_within_tolerance(moments, ref_m, qk_tol=TOL_GRAD_REL_QK)
        sh = model._engine.shadow.view(torch.int16).to(torch.int64)
        sig = torch.stack([sh.sum(), (sh * (torch.arange(sh.numel(), device=dev) % 8191 + 1)).sum()])
        sigs = [torch.zeros_like(sig) for _ in range(world)]
        dist.all_gather(sigs, sig)
        stats = torch.tensor([worst], dtype=torch.float64, device=dev)
        dist.all_reduce(stats, op=dist.ReduceOp.MAX)
        worst = float(stats[0])
        assert all(torch.equal(x, sigs[0]) for x in sigs), "%s: ranks hold different weights" % path
        assert worst <= TOL_TRAJ, (path, worst)
        # dev() / test() over the gathered tokens: each rank evaluates its own batches
        loader = [tok.token_batch(cfg, 4, 128, 3000 + 10 * i + rank) for i in range(2)]
        loss, acc = tr.dev(loader)
        want_loss, counts = 0.0, torch.zeros(2, dtype=torch.float64, device=dev)
        for bt in loader:
            z, y = tr.eval_step(bt)
            z, y = z.detach(), y.to(dev)
            l = F.cross_entropy(z.reshape(-1, 9), y.reshape(-1)).reshape(1)
            dist.all_reduce(l)
            want_loss += float(l) / world
            keep = y.reshape(-1) != -100
            pred = z.reshape(-1, 9).argmax(-1)
            counts += torch.tensor([float((pred[keep] == y.reshape(-1)[keep]).sum()), float(keep.sum())],
                                   dtype=torch.float64, device=dev)
        dist.all_reduce(counts)
        assert abs(float(loss) - want_loss) <= 1e-5 * max(1.0, want_loss), (path, float(loss), want_loss)
        assert abs(acc - float(counts[0] / counts[1])) <= 1e-12, (path, acc, counts)
        report = tr.test(net, loader, ["t%d" % i for i in range(9)])
        assert "t8" in report
        if rank == 0:
            print("ddp_token_worker: %s worst |dloss_mean| %.2e (tol %.0e), moments rel-L2 q/k %.2e others %.2e, "
                  "dev acc %.4f" % (path, worst, TOL_TRAJ, qk, other, acc), flush=True)
        torch.cuda.synchronize()
        dist.barrier()
        net.close()
    if rank == 0:
        print("ddp_token_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
