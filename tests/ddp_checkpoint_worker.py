"""One rank per GPU, world 2: checkpoints under the peer-HBM DDP path (tests/test_checkpoint.py runs it).
  * train() with save_steps = 2 (fused path, dropout on, TorchAdamW with amsgrad, a linear schedule);
  * rank 0 alone calls optimizer.state_dict() and model.state_dict() after more captured replays than the last gather
    saw: the gathered state and masters equal every rank's own slices, which each rank dumps;
  * a world-2 resume from checkpoint-2 follows the uninterrupted world-2 run within TOL_TRAJ;
  * the world-2 optimizer file loads on one GPU with equal moments and step;
  * close() leaves the optimizer usable, with gathered private state.
Exits non-zero on any mismatch.
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29601 \
        tests/ddp_checkpoint_worker.py
"""
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist
import torch.nn.functional as F

from parity import TOL_TRAJ, b2, bert_ref, state_from_hf_init, tiny_config

LR, WD, BATCHES, EXTRA = 2e-4, 0.01, 6, 2


def groups(named):
    named = list(named)
    nd = lambda n: "bias" in n or "LayerNorm.weight" in n
    return [{"params": [p for n, p in named if not nd(n)], "weight_decay": WD},
            {"params": [p for n, p in named if nd(n)], "weight_decay": 0.0}]


def run(cfg, state, batches, local, world, rank, out, resume=None):
    model = b2.BertForSequenceClassification(cfg)
    model.load_state_dict(state)
    model.cuda()
    net = b2.DistributedDataParallel(model, device_ids=[local])
    opt = b2.TorchAdamW(groups(net.module.named_parameters()), lr=LR, amsgrad=True)
    a = b2.Args()
    a.local_rank, a.local_world_size, a.rank = local, world, rank
    a.epochs, a.dev, a.log_every = 1, False, 1000
    a.lr_scheduler_type = "linear"
    a.output_dir, a.save_steps = out, 2
    a.ckpt_path = os.path.join(out, "final-%d.pt" % rank)
    tr = b2.Trainer(a, cfg, net, torch.nn.CrossEntropyLoss(), opt)
    losses = []
    step = tr.train_step
    tr.train_step = lambda bt: losses.append(float(step(bt))) or losses[-1]
    tr.train(batches, resume_from_checkpoint=resume)
    torch.cuda.synchronize()
    return net, model, opt, losses, tr


def flat_of(sd, model, key):
    """the per-parameter `key` tensors of an optimizer state_dict laid out in the model's flat space"""
    lay = model._layout
    flat = torch.zeros(lay.total)
    names = [p._b2_name for g in model._optimizer.param_groups for p in g["params"]]
    for i, entry in sd["state"].items():
        off, _shape = lay.entries[names[i]]
        flat[off:off + entry[key].numel()] = entry[key].flatten().cpu()
    return flat


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = tiny_config()
    state = state_from_hf_init(cfg, seed=123)
    batches = [bert_ref.synthetic_batch(cfg, 4, 128, 9700 + 10 * s + rank, padded=True) for s in range(BATCHES)]
    box = [tempfile.mkdtemp(prefix="b2ckpt-") if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    root = box[0]
    keys = ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")

    # 1. the uninterrupted run (its last checkpoint and the final ckpt_path save gathered the masters on rank 0), then
    # EXTRA more captured replays, which run no Python; rank 0 alone gathers the optimizer state and the masters again,
    # every rank dumps its own slices
    net, model, opt, losses, tr = run(cfg, state, batches, local, world, rank, os.path.join(root, "full"))
    w_full = net.state_dict()
    for s in range(EXTRA):
        tr.train_step(batches[s])
    torch.cuda.synchronize()
    st = opt._state()
    torch.save({"slices": model._ddp._slices, "master": model._flat.cpu(), **{k: st[k].cpu() for k in keys}},
               os.path.join(root, "own-%d.pt" % rank))
    dist.barrier()
    if rank == 0:
        sd = opt.state_dict()
        msd = model.state_dict()
        torch.save(sd, os.path.join(root, "opt.pt"))
        lay = model._layout
        master = torch.zeros(lay.total)
        for name, (off, shape) in lay.entries.items():
            master[off:off + msd[name].numel()] = msd[name].flatten().cpu()
        for r in range(world):
            own = torch.load(os.path.join(root, "own-%d.pt" % r))
            idx = torch.cat([torch.arange(b, e) for (b, e) in own["slices"]])
            for k in keys:
                assert torch.equal(flat_of(sd, model, k)[idx], own[k][idx]), ("gathered != rank %d's own" % r, k)
            assert torch.equal(master[idx], own["master"][idx]), "gathered masters != rank %d's own" % r
        print("ddp_checkpoint_worker: the gathered state and masters equal every rank's slices", flush=True)
    dist.barrier()

    # 2. close() leaves the optimizer usable, with gathered private state
    before = {k: v.clone() for k, v in opt._state().items() if k in keys}
    peer_ptrs = {k: opt._state()[k].data_ptr() for k in keys}
    net.close()
    after = opt._state()
    for k in keys:
        assert after[k].data_ptr() != peer_ptrs[k], k
    if rank == 0:
        for k in keys:
            assert torch.equal(after[k], before[k]), k      # rank 0 had gathered them already
    sd_closed = opt.state_dict()
    for k in keys:
        assert torch.equal(flat_of(sd_closed, model, k), flat_of(torch.load(os.path.join(root, "opt.pt")), model, k)), k
    d = {k: v.to(dev) for k, v in batches[0].items()}
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    opt.step()
    torch.cuda.synchronize()
    assert int(opt._state()["step"]) == BATCHES + EXTRA + 1
    del net, model, opt, tr
    dist.barrier()

    # 3. a world-2 resume from checkpoint-2 follows the uninterrupted run
    ck = os.path.join(root, "full", "checkpoint-2")
    net, model, opt, resumed, _tr = run(cfg, state_from_hf_init(cfg, seed=9), batches, local, world, rank,
                                   os.path.join(root, "res"), resume=ck)
    assert len(resumed) == BATCHES - 2, resumed
    dl = max(abs(x - y) for x, y in zip(losses[2:], resumed))
    w_res = net.state_dict()
    dw = max(float((w_res[k] - w_full[k]).abs().max()) for k in w_full)
    assert dl <= TOL_TRAJ and dw <= TOL_TRAJ, (rank, losses[2:], resumed, dw)
    if rank == 0:
        print("ddp_checkpoint_worker: world-2 resume |dloss| %.2e |dw| %.2e" % (dl, dw), flush=True)
    torch.cuda.synchronize()
    dist.barrier()
    net.close()
    del net, model, opt
    dist.barrier()

    # 4. the world-2 optimizer file on one GPU
    if rank == 0:
        one = b2.BertForSequenceClassification(cfg).cuda()
        o1 = b2.TorchAdamW(groups(one.named_parameters()), lr=LR, amsgrad=True)
        sd = torch.load(os.path.join(root, "opt.pt"))
        o1.load_state_dict(sd)
        m = o1.moments()
        names = [p._b2_name for g in o1.param_groups for p in g["params"]]
        for i, entry in sd["state"].items():
            ea, eas = m[names[i]]
            assert torch.equal(ea.cpu(), entry["exp_avg"]) and torch.equal(eas.cpu(), entry["exp_avg_sq"]), names[i]
        assert int(o1._state()["step"]) == BATCHES + EXTRA
        print("ddp_checkpoint_worker: the world-2 state loads on one GPU", flush=True)
    dist.barrier()
    if rank == 0:
        import shutil
        shutil.rmtree(root, ignore_errors=True)
        print("ddp_checkpoint_worker: OK (world %d)" % world, flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
