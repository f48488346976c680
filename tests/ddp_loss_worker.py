"""One rank per GPU, world 2: multi-label BCEWithLogitsLoss(pos_weight) on the Trainer's captured DDP step
(tests/test_losses.py runs it).  The rank-mean loss and the fp32 masters follow the oracle's DDP mean (each rank's
mean-loss gradient, averaged over the ranks), and dev() computes the subset accuracy of the gathered float labels.
Exits non-zero on any mismatch.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29597 \
        tests/ddp_loss_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist

from loss_ref import labelled_batch, loss_and_grads
from parity import TOL_TRAJ, adamw_ref, b2, state_from_hf_init, tiny_config

STEPS, LR, C = 3, 3e-5, 4
POS_WEIGHT = [0.5, 2.0, 1.0, 3.0]


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = tiny_config(num_labels=C, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg, seed=123)
    batches = [[labelled_batch(cfg, 4, 128, 9700 + 10 * s + r, "multi") for r in range(world)] for s in range(STEPS)]
    # the oracle's DDP step: the mean over ranks of each rank's mean-loss gradient
    crit_ref = torch.nn.BCEWithLogitsLoss(pos_weight=torch.tensor(POS_WEIGHT))
    ref = {k: v.clone() for k, v in state.items()}
    ref_opt = adamw_ref.HFAdamW(ref, lr=LR, weight_decay=0.01)
    ref_losses = []
    for s in range(STEPS):
        outs = [loss_and_grads(ref, cfg, batches[s][r], crit_ref) for r in range(world)]
        ref_losses.append(sum(float(o[0]) for o in outs) / world)
        ref_opt.step({k: sum(o[2][k] for o in outs) / world for k in ref})

    model = b2.BertForSequenceClassification(cfg)
    model.load_state_dict(state)
    model.cuda()
    net = b2.DistributedDataParallel(model, device_ids=[local])
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank = local, world, rank
    args.learning_rate, args.weight_decay = LR, 0.01
    opt = b2.build_optimizer(net, args)
    crit = torch.nn.BCEWithLogitsLoss(pos_weight=torch.tensor(POS_WEIGHT, device=dev))
    tr = b2.Trainer(args, cfg, net, crit, opt)
    for s in range(STEPS):
        loss = float(tr.train_step(batches[s][rank]))
        assert abs(loss - ref_losses[s]) <= TOL_TRAJ, (s, loss, ref_losses[s])
    torch.cuda.synchronize()
    w = {n: v.detach().cpu() for n, v in net.state_dict().items()}
    for n, v in ref.items():
        assert float((w[n] - v).abs().max()) <= 2 * LR * STEPS + 2e-5, n

    # dev(): subset accuracy over both ranks' rows, against the gathered eager logits
    loader = [labelled_batch(cfg, 4, 128, 9800 + 10 * i + rank, "multi") for i in range(2)]
    _loss, acc = tr.dev(loader)
    model.eval()
    hits, rows = 0, 0
    with torch.no_grad():
        for b in loader:
            d = {k: v.to(dev) for k, v in b.items()}
            z = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                      attention_mask=d["attention_mask"]).logits
            pair = ((z > 0) == (d["label"] >= 0.5)).all(dim=-1).float()
            got = [torch.zeros_like(pair) for _ in range(world)]
            dist.all_gather(got, pair)
            hits += float(sum(g.sum() for g in got))
            rows += sum(g.numel() for g in got)
    assert abs(float(acc) - hits / rows) <= 1e-12, (acc, hits / rows)
    torch.cuda.synchronize()
    dist.barrier()
    net.close()
    if rank == 0:
        print("ddp_loss_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
