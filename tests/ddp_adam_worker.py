"""One rank per GPU, world 2: torch's AdamW (the package's TorchAdamW, amsgrad on) with gradient clipping under the
peer-HBM DDP path (tests/test_torch_adam.py runs it with B2_DDP_DMA=0 and =1).  The eager loop (backward,
clip_grad_norm_, step) and the Trainer's CUDA-graph step with max_grad_norm, against the oracle: fp32 clip_grad_norm_ on
the mean of the ranks' oracle gradients, then torch.optim.AdamW.  The weights stay within the bound of the update size
and the first moments of this rank's slices within the parity tolerance; every rank holds the same bf16 weights.  Exits
non-zero on any mismatch.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29598 \
        tests/ddp_adam_worker.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist
import torch.nn.functional as F

from parity import TOL_GRAD_REL_QK, b2, bert_ref, rel_l2, state_from_hf_init, tiny_config

LR, WD, STEPS = 1e-3, 0.01, 3


def groups(named):
    named = list(named)
    nd = lambda n: "bias" in n or "LayerNorm.weight" in n
    return [{"params": [p for n, p in named if not nd(n)], "weight_decay": WD},
            {"params": [p for n, p in named if nd(n)], "weight_decay": 0.0}]


def oracle(cfg, state, batches, world):
    ref = {k: torch.nn.Parameter(v.clone()) for k, v in state.items()}
    opt = torch.optim.AdamW(groups(ref.items()), lr=LR, amsgrad=True, foreach=False)
    max_norm = None
    for s in range(STEPS):
        mean = None
        for r in range(world):
            _l, _z, g = bert_ref.loss_and_grads({k: p.detach() for k, p in ref.items()}, cfg, batches[s][r])
            mean = {k: x / world for k, x in g.items()} if mean is None else {k: mean[k] + x / world
                                                                               for k, x in g.items()}
        for k, p in ref.items():
            p.grad = mean[k].clone()
        if max_norm is None:
            max_norm = 0.25 * float(torch.nn.utils.get_total_norm([p.grad for p in ref.values()]))
        torch.nn.utils.clip_grad_norm_(list(ref.values()), max_norm)
        opt.step()
    return max_norm, {k: p.detach().clone() for k, p in ref.items()}, {k: opt.state[p]["exp_avg"] for k, p in ref.items()}


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg, seed=123)
    batches = [[bert_ref.synthetic_batch(cfg, 4, 128, 9300 + 10 * s + r, padded=(s % 2 == 1)) for r in range(world)]
               for s in range(STEPS)]
    max_norm, rw, rm = oracle(cfg, state, batches, world)
    for mode in ("eager", "fused"):
        model = b2.BertForSequenceClassification(cfg)
        model.load_state_dict(state)
        model.cuda()
        net = b2.DistributedDataParallel(model, device_ids=[local])
        args = b2.Args()
        args.local_rank, args.local_world_size, args.rank = local, world, rank
        args.max_grad_norm = max_norm
        opt = b2.TorchAdamW(groups(net.module.named_parameters()), lr=LR, amsgrad=True)
        tr = b2.Trainer(args, cfg, net, torch.nn.CrossEntropyLoss(), opt)
        for s in range(STEPS):
            if mode == "eager":
                d = {k: v.to(dev) for k, v in batches[s][rank].items()}
                out = net(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                          attention_mask=d["attention_mask"], labels=d["label"])
                F.cross_entropy(out[1], d["label"]).backward()
                b2.clip_grad_norm_(net.parameters(), max_norm)
                opt.step()
            else:
                tr.train_step(batches[s][rank])
        torch.cuda.synchronize()
        sh = model._engine.shadow.view(torch.int16)
        shs = [torch.zeros_like(sh) for _ in range(world)]
        dist.all_gather(shs, sh)
        assert all(torch.equal(x, shs[0]) for x in shs), "%s: ranks hold different bf16 weights" % mode
        sd = net.state_dict()
        for k, v in rw.items():
            err = float((sd["module." + k].cpu() - v).abs().max())
            assert err <= 2 * LR * STEPS + 2e-5, (mode, k, err)
            assert not torch.equal(sd["module." + k].cpu(), state[k]), (mode, k, "did not move")
        # this rank's slices of the first moment, against the oracle's laid out in the flat space
        lay = model._layout
        flat = torch.zeros(lay.total)
        for k, m in rm.items():
            off, _shape = lay.entries[k]
            flat[off:off + m.numel()] = m.flatten()
        ours = opt._state()["exp_avg"].cpu()
        idx = torch.cat([torch.arange(b, e) for (b, e) in model._ddp._slices])
        err = rel_l2(ours[idx], flat[idx])
        assert err <= TOL_GRAD_REL_QK, (mode, err)
        if rank == 0:
            print("ddp_adam_worker: mode %s dma %s exp_avg rel-L2 %.2e" % (mode, os.environ.get("B2_DDP_DMA", "0"), err),
                  flush=True)
        torch.cuda.synchronize()
        dist.barrier()
        net.close()
    if rank == 0:
        print("ddp_adam_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
