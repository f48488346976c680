"""One rank per GPU, world 2: gradient accumulation under the peer-HBM DDP path.  Trainer with
gradient_accumulation_steps = 2 on the CUDA-graph step, where rank r's micro-batch i of step s is the batch of rank 2r + i
in the world-4 fixture (tests/golden/config_a_ddp.pt): the 2 x 2 micro-batches of a step are then exactly the fixture's
world-4 step.  Tolerances of bench.py's parity block.  Exits non-zero on any mismatch.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29583 \
        tests/ddp_accum_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch
import torch.distributed as dist

import pytorch_distributed_nlp_b200 as b2

K, LR = 2, 3e-5


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "config_a_ddp.pt"))
    fw, steps = fx["worlds"][world * K], int(fx["steps"])
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg)
    model.cuda()
    net = b2.DistributedDataParallel(model, device_ids=[local])
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank = local, world, rank
    args.gradient_accumulation_steps = K
    opt = b2.build_optimizer(net, args)
    tr = b2.Trainer(args, cfg, net, torch.nn.CrossEntropyLoss(), opt)
    d_local, d_mean = 0.0, 0.0
    for s in range(steps):
        means = []
        for i in range(K):
            fr = K * rank + i
            batch = b2.synthetic_batch(cfg, 32, 128, 5000 + 100 * s + fr, padded=(s % 2 == 1))
            mean = tr.train_step(batch)               # rank mean of this micro-batch's loss
            d_local = max(d_local, abs(float(tr._fused.loss_out) - float(fw["loss"][s][fr])))
            means.append(float(mean))
        d_mean = max(d_mean, abs(sum(means) / K - float(fw["loss"][s].mean())))
    assert int(opt._state()["step"]) == steps
    sd = net.state_dict()
    d_w, d_norm = 0.0, 0.0
    norm_floor = 1e-3 * max(fw["final_norms"].values())
    for k, ref in fw["final_samples"].items():
        f = sd["module." + k].detach().flatten()
        if f.numel() > ref.numel():
            f = f[(torch.arange(ref.numel(), dtype=torch.int64) * (f.numel() - 1) // (ref.numel() - 1)).to(f.device)]
        d_w = max(d_w, float((f.cpu() - ref).abs().max()))
        d_norm = max(d_norm, abs(float(sd["module." + k].double().norm()) - fw["final_norms"][k]) /
                     max(fw["final_norms"][k], norm_floor))
    sh = model._engine.shadow.view(torch.int16).to(torch.int64)
    sig = torch.stack([sh.sum(), (sh * (torch.arange(sh.numel(), device=dev) % 8191 + 1)).sum()])
    sigs = [torch.zeros_like(sig) for _ in range(world)]
    dist.all_gather(sigs, sig)
    stats = torch.tensor([d_local, d_mean, d_w, d_norm], dtype=torch.float64, device=dev)
    dist.all_reduce(stats, op=dist.ReduceOp.MAX)
    d_local, d_mean, d_w, d_norm = (float(v) for v in stats)
    tol_w = 2 * LR * steps + 2e-5
    if rank == 0:
        print("ddp_accum_worker: dloss %.2e dloss_mean %.2e dweight %.2e (tol %.2e) dnorm_rel %.2e"
              % (d_local, d_mean, d_w, tol_w, d_norm), flush=True)
    assert all(torch.equal(x, sigs[0]) for x in sigs), "ranks hold different weights"
    assert d_local <= 1e-2 and d_mean <= 1e-2 and d_w <= tol_w and d_norm <= 1e-3
    torch.cuda.synchronize()
    dist.barrier()
    net.close()
    if rank == 0:
        print("ddp_accum_worker: OK (world %d x %d micro-batches)" % (world, K), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
