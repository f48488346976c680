"""Checkpoint and resume: the fused optimizers' state_dict / load_state_dict in torch's format, the model's dropout
stream and save_pretrained, and Trainer save_checkpoint / train(resume_from_checkpoint=...).

Two runs of the same step are not bitwise equal (the bias gradients are summed by float atomics), so the bitwise checks
are made on the state and on updates from one shared gradient buffer, and trajectories are checked to TOL_TRAJ."""
import copy
import functools
import io
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from parity import TOL_TRAJ, b2, bert_ref, make_model, state_from_hf_init, tiny_config, to_dev
from pytorch_distributed_nlp_b200.trainer import latest_checkpoint, rotate_checkpoints, sorted_checkpoints

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def _no_decay(n):
    return "bias" in n or "LayerNorm.weight" in n


def _groups(named, wd=0.01):
    """the reference's two groups (multi-gpu-distributed-cls.py:100-111)"""
    named = list(named)
    return [{"params": [p for n, p in named if not _no_decay(n)], "weight_decay": wd},
            {"params": [p for n, p in named if _no_decay(n)], "weight_decay": 0.0}]


def _hf_model(cfg):
    from oracle import cpu_step
    return cpu_step.build_hf_model(cfg)


# (name, package class + kwargs on the reference's groups, the stock torch class it restates or None)
OPTS = {
    "hf_adamw": (lambda g: b2.AdamW(g, lr=1e-3), None),
    "torch_adamw": (lambda g: b2.TorchAdamW(g, lr=1e-3), lambda g: torch.optim.AdamW(g, lr=1e-3)),
    "torch_adamw_amsgrad": (lambda g: b2.TorchAdamW(g, lr=1e-3, amsgrad=True),
                            lambda g: torch.optim.AdamW(g, lr=1e-3, amsgrad=True)),
    "adam_coupled": (lambda g: b2.Adam(g, lr=1e-3), lambda g: torch.optim.Adam(g, lr=1e-3)),
    "sgd_nesterov": (lambda g: b2.SGD(g, lr=0.05, momentum=0.9, nesterov=True),
                     lambda g: torch.optim.SGD(g, lr=0.05, momentum=0.9, nesterov=True)),
    "sgd_plain": (lambda g: b2.SGD(g, lr=0.05), lambda g: torch.optim.SGD(g, lr=0.05)),
}


# ---- CPU: the format before the first step, the load errors, save_pretrained, checkpoint directories -----------------
def test_named_parameters_order_is_hfs():
    cfg = tiny_config()
    assert [n for n, _p in b2.BertForSequenceClassification(cfg).named_parameters()] == \
        [n for n, _p in _hf_model(cfg).named_parameters()]


@pytest.mark.parametrize("name", list(OPTS))
def test_state_dict_before_the_first_step_is_torchs(name):
    cfg = tiny_config()
    ours, theirs = OPTS[name]
    sd = ours(_groups(b2.BertForSequenceClassification(cfg).named_parameters())).state_dict()
    assert sd["state"] == {}
    assert [g["params"] for g in sd["param_groups"]] == [list(range(0, 17)), list(range(17, 41))]
    if theirs is None:       # transformers 4.28.1 AdamW's group keys
        assert all(set(g) == {"lr", "betas", "eps", "weight_decay", "correct_bias", "params"} for g in sd["param_groups"])
        return
    ref = theirs(_groups(_hf_model(cfg).named_parameters())).state_dict()
    assert sd == ref


def _stepped_torch_state(cfg, make, steps=2):
    """the stock optimizer's state_dict after `steps` steps on random gradients of an HF model (CPU)"""
    hf = _hf_model(cfg)
    opt = make(_groups(hf.named_parameters()))
    gen = torch.Generator().manual_seed(7)
    for _ in range(steps):
        for p in hf.parameters():
            p.grad = torch.randn(p.shape, generator=gen) * 1e-2
        opt.step()
    return opt.state_dict()


def test_load_errors_are_torchs():
    cfg = tiny_config()
    model = b2.BertForSequenceClassification(cfg)
    opt = b2.TorchAdamW(_groups(model.named_parameters()), lr=1e-3)
    good = opt.state_dict()
    ref = torch.optim.AdamW(_groups(_hf_model(cfg).named_parameters()), lr=1e-3)
    one_group = copy.deepcopy(good)
    one_group["param_groups"] = one_group["param_groups"][:1]
    short = copy.deepcopy(good)
    short["param_groups"][1]["params"] = short["param_groups"][1]["params"][:-1]
    for bad in (one_group, short):
        with pytest.raises(ValueError) as t:
            ref.load_state_dict(bad)
        with pytest.raises(ValueError) as o:
            opt.load_state_dict(bad)
        assert str(o.value) == str(t.value)
    # the constructor's group rules, which leave the optimizer as it was
    for field, value, match in (("betas", (0.8, 0.999), "differ only in weight_decay"),
                                ("weight_decay", 0.02, "one non-zero weight_decay")):
        bad = copy.deepcopy(good)
        bad["param_groups"][1][field] = value
        with pytest.raises(ValueError, match=match):
            opt.load_state_dict(bad)
        assert opt.state_dict() == good


def test_load_errors_of_the_per_parameter_state():
    cfg = tiny_config()
    sd = _stepped_torch_state(cfg, lambda g: torch.optim.AdamW(g, lr=1e-3))
    opt = b2.TorchAdamW(_groups(b2.BertForSequenceClassification(cfg).named_parameters()), lr=1e-3)
    partial = copy.deepcopy(sd)
    del partial["state"][3]
    with pytest.raises(ValueError, match="covers 40 of 41"):
        opt.load_state_dict(partial)
    for bad_step in (torch.tensor(3.0), 3, 3.0):
        disagree = copy.deepcopy(sd)
        disagree["state"][5]["step"] = bad_step
        with pytest.raises(ValueError, match="disagree on step"):
            opt.load_state_dict(disagree)
    ams = b2.TorchAdamW(_groups(b2.BertForSequenceClassification(cfg).named_parameters()), lr=1e-3, amsgrad=True)
    bad = copy.deepcopy(sd)
    for g in bad["param_groups"]:
        g["amsgrad"] = True
    with pytest.raises(ValueError, match="no max_exp_avg_sq after 2 steps"):
        ams.load_state_dict(bad)
    # a state with steps needs the model on the GPU
    with pytest.raises(RuntimeError, match="model.cuda"):
        opt.load_state_dict(sd)


def test_save_pretrained_round_trip(tmp_path):
    cfg = tiny_config(problem_type="multi_label_classification", hidden_dropout_prob=0.05)
    model = b2.BertForSequenceClassification(cfg)
    with torch.no_grad():
        model._flat.add_(torch.randn_like(model._flat) * 1e-3)
    model.save_pretrained(str(tmp_path))
    assert sorted(os.listdir(tmp_path)) == ["config.json", "pytorch_model.bin"]
    back = b2.BertForSequenceClassification.from_pretrained(str(tmp_path))
    assert vars(back.config) == vars(cfg)
    ours, theirs = model.state_dict(), back.state_dict()
    assert list(ours) == list(theirs)
    for k in ours:
        assert torch.equal(ours[k], theirs[k]), k
    saved = torch.load(os.path.join(tmp_path, "pytorch_model.bin"))
    assert set(saved) == set(ours) and not any(k.startswith("module.") for k in saved)


def test_checkpoint_directories(tmp_path):
    assert sorted_checkpoints(str(tmp_path / "missing")) == [] and latest_checkpoint(None) is None
    for n in (10, 2, 40, 9):
        (tmp_path / ("checkpoint-%d" % n)).mkdir()
    (tmp_path / "checkpoint-x").mkdir()
    (tmp_path / "checkpoint-7").write_text("a file, not a checkpoint")
    (tmp_path / "other").mkdir()
    names = lambda: [os.path.basename(p) for p in sorted_checkpoints(str(tmp_path))]
    assert names() == ["checkpoint-2", "checkpoint-9", "checkpoint-10", "checkpoint-40"]
    assert os.path.basename(latest_checkpoint(str(tmp_path))) == "checkpoint-40"
    rotate_checkpoints(str(tmp_path), None)
    rotate_checkpoints(str(tmp_path), 0)
    assert len(names()) == 4
    rotate_checkpoints(str(tmp_path), 2)
    assert names() == ["checkpoint-10", "checkpoint-40"]
    assert (tmp_path / "checkpoint-x").is_dir() and (tmp_path / "other").is_dir()
    a = b2.Args()
    assert (a.output_dir, a.save_steps, a.save_total_limit) == (None, None, None)


def test_save_steps_without_output_dir_raises():
    model = b2.BertForSequenceClassification(tiny_config())
    a = b2.Args()
    a.save_steps = 1
    tr = b2.Trainer(a, model.config, model, None, b2.AdamW(model.parameters()))
    tr.global_step = 1
    with pytest.raises(ValueError, match="output_dir"):
        tr._maybe_save()


# ---- GPU: one H100 -------------------------------------------------------------------------------------------------
def _batch(cfg, seed, bsz=4):
    return bert_ref.synthetic_batch(cfg, bsz, 128, seed, padded=True)


def _loop_step(model, opt, d):
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    opt.step()


def _through_bytes(obj):
    buf = io.BytesIO()
    torch.save(obj, buf)
    buf.seek(0)
    return torch.load(buf, map_location="cpu")


def _snapshot(model, opt):
    return _through_bytes({"model": model.state_dict(), "opt": opt.state_dict(), "rng": model.dropout_rng_state()})


def _restore(model, opt, snap):
    model.load_state_dict(snap["model"])
    opt.load_state_dict(snap["opt"])
    model.set_dropout_rng_state(snap["rng"])


def _same_state_dict(a, b):
    assert a["param_groups"] == b["param_groups"]
    assert list(a["state"]) == list(b["state"])
    for i in a["state"]:
        assert list(a["state"][i]) == list(b["state"][i]), i
        for k, v in a["state"][i].items():
            w = b["state"][i][k]
            if isinstance(v, torch.Tensor):
                assert v.dtype == w.dtype and v.shape == w.shape and torch.equal(v.cpu(), w.cpu()), (i, k)
            else:
                assert v == w, (i, k)


def _same_device_state(oa, ob):
    sa, sb = oa._state(), ob._state()
    for k in oa._flat_keys:
        assert (sa.get(k) is None) == (sb.get(k) is None), k
        if sa.get(k) is not None:
            assert torch.equal(sa[k], sb[k]), k
    assert torch.equal(sa["decay"], sb["decay"])


@gpu
@pytest.mark.parametrize("name", list(OPTS))
def test_round_trip_is_bitwise(cuda_dev, name):
    """3 eager steps with dropout on, then model + optimizer + dropout state through torch.save / torch.load into fresh
    objects: everything bitwise equal; then one shared gradient stepped by both keeps them bitwise equal"""
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    make = OPTS[name][0]
    a = make_model(cfg, state, cuda_dev).train()
    oa = make(_groups(a.named_parameters()))
    a._engine.seed_dropout(1234, 0)
    for i in range(3):
        _loop_step(a, oa, to_dev(_batch(cfg, 8400 + i), cuda_dev))
    snap = _snapshot(a, oa)
    b = make_model(cfg, state_from_hf_init(cfg, seed=5), cuda_dev).train()
    ob = make(_groups(b.named_parameters()))
    _restore(b, ob, snap)
    torch.cuda.synchronize()
    assert torch.equal(a._flat, b._flat) and torch.equal(a._engine.shadow, b._engine.shadow)
    assert torch.equal(a.dropout_rng_state(), b.dropout_rng_state())
    assert a.dropout_rng_state()[1].item() == 3
    _same_state_dict(oa.state_dict(), ob.state_dict())
    _same_device_state(oa, ob)
    if name != "sgd_plain":
        assert oa.state_dict()["state"], "no state after 3 steps"
    if not name.startswith("sgd"):
        assert int(oa._state()["step"]) == int(ob._state()["step"]) == 3
    # one backward on a; its gradients stepped by both
    d = to_dev(_batch(cfg, 8500), cuda_dev)
    out = a(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
            labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    b._engine.grads.copy_(a._engine.grads)
    oa.step()
    ob.step()
    torch.cuda.synchronize()
    assert torch.equal(a._flat, b._flat) and torch.equal(a._engine.shadow, b._engine.shadow)
    _same_state_dict(oa.state_dict(), ob.state_dict())
    _same_device_state(oa, ob)


@gpu
def test_sgd_without_a_loaded_buffer_initialises_it_from_the_gradient(cuda_dev):
    """momentum SGD loaded with an empty state (torch's momentum 0 dict) after steps: the next update starts the buffer
    from the gradient, as torch's `momentum_buffer is None` does -- the same update a fresh optimizer makes"""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    a = make_model(cfg, state, cuda_dev).train()
    oa = b2.SGD(a.parameters(), lr=0.05, momentum=0.9)
    for i in range(2):
        _loop_step(a, oa, to_dev(_batch(cfg, 8600 + i), cuda_dev))
    oa.load_state_dict(b2.SGD(b2.BertForSequenceClassification(cfg).parameters(), lr=0.05, momentum=0.9).state_dict())
    assert oa.state_dict()["state"] == {}
    b = make_model(cfg, state, cuda_dev).train()
    b.load_state_dict(a.state_dict())
    ob = b2.SGD(b.parameters(), lr=0.05, momentum=0.9)
    d = to_dev(_batch(cfg, 8700), cuda_dev)
    out = a(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
            labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    b._engine.grads.copy_(a._engine.grads)
    oa.step()
    ob.step()
    torch.cuda.synchronize()
    assert torch.equal(a._flat, b._flat)
    _same_state_dict(oa.state_dict(), ob.state_dict())


def _max_diff(xs, ys):
    return max(abs(float(x) - float(y)) for x, y in zip(xs, ys))


@gpu
@pytest.mark.parametrize("kind,name", [("fused", "hf_adamw"), ("fused", "torch_adamw_amsgrad"),
                                       ("packed", "hf_adamw"), ("packed", "sgd_nesterov")])
def test_load_in_place_under_capture(cuda_dev, kind, name):
    """a captured train step keeps replaying, without recapture, on a state loaded into the same objects: 2 steps,
    snapshot, 3 more; load the snapshot and replay those 3 again"""
    cfg = tiny_config()
    model = make_model(cfg, state_from_hf_init(cfg), cuda_dev).train()
    opt = OPTS[name][0](_groups(model.named_parameters()))
    bt = _batch(cfg, 8800)
    if kind == "fused":
        st = b2.FusedTrainStep(model, opt, 4, 128)
        run = lambda: float(st(bt))
    else:
        packed = b2.pack_batch(bt["input_ids"], bt["token_type_ids"], bt["attention_mask"])
        st = b2.PackedTrainStep(model, opt, packed["bins"], 4)
        run = lambda: float(st(packed, bt["label"]))
    for _ in range(2):
        run()
    snap = _snapshot(model, opt)
    first = [run() for _ in range(3)]
    graph = st.graph
    assert graph is not None
    w_first = model._flat.detach().clone()
    dev_state = opt._state()
    ptrs = {k: v.data_ptr() for k, v in dev_state.items() if isinstance(v, torch.Tensor)}
    assert int(dev_state["step"]) == 5
    _restore(model, opt, snap)
    # the same buffers the graph reads, holding the snapshot's step (SGD's device step only says "the buffer exists")
    loaded = 1 if name.startswith("sgd") else 2
    assert opt._state() is dev_state and int(dev_state["step"]) == loaded
    assert {k: v.data_ptr() for k, v in dev_state.items() if isinstance(v, torch.Tensor)} == ptrs
    again = [run() for _ in range(3)]
    torch.cuda.synchronize()
    assert st.graph is graph and len(st._graphs) == 1
    assert int(dev_state["step"]) == loaded + 3
    assert _max_diff(first, again) <= TOL_TRAJ, (first, again)
    assert float((model._flat - w_first).abs().max()) <= TOL_TRAJ


@gpu
def test_interop_with_stock_torch(cuda_dev):
    """a package TorchAdamW / SGD dict loads into the stock class on an HF CPU model with equal tensors; a stock
    torch.optim.AdamW(fused=True) / SGD state of the same grouping loads into the package class exactly"""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    for ours_make, theirs_make in (
            (lambda g: b2.TorchAdamW(g, lr=1e-3, amsgrad=True), lambda g: torch.optim.AdamW(g, lr=1e-3, amsgrad=True)),
            (lambda g: b2.SGD(g, lr=0.05, momentum=0.9), lambda g: torch.optim.SGD(g, lr=0.05, momentum=0.9))):
        model = make_model(cfg, state, cuda_dev).train()
        opt = ours_make(_groups(model.named_parameters()))
        for i in range(2):
            _loop_step(model, opt, to_dev(_batch(cfg, 8900 + i), cuda_dev))
        sd = _through_bytes(opt.state_dict())
        hf = _hf_model(cfg)
        ref = theirs_make(_groups(hf.named_parameters()))
        ref.load_state_dict(sd)
        params = [p for g in ref.param_groups for p in g["params"]]
        assert len(ref.state) == len(params)
        mine = opt.state_dict()
        for i, p in enumerate(params):
            for k, v in mine["state"][i].items():
                w = ref.state[p][k]
                assert torch.equal(torch.as_tensor(v).cpu(), w.cpu()), (i, k)
    # the other way: stock fused AdamW on a CUDA HF model
    hf = _hf_model(cfg).to(cuda_dev)
    ref = torch.optim.AdamW(_groups(hf.named_parameters()), lr=1e-3, fused=True)
    gen = torch.Generator(device=cuda_dev).manual_seed(3)
    for _ in range(2):
        for p in hf.parameters():
            p.grad = torch.randn(p.shape, device=cuda_dev, generator=gen) * 1e-2
        ref.step()
    model = make_model(cfg, state, cuda_dev)
    opt = b2.TorchAdamW(_groups(model.named_parameters()), lr=1e-3)
    opt.load_state_dict(ref.state_dict())
    names = {id(p): n for n, p in hf.named_parameters()}
    moments = opt.moments()
    for p, s in ref.state.items():
        m, v = moments[names[id(p)]]
        assert torch.equal(m, s["exp_avg"]) and torch.equal(v, s["exp_avg_sq"]), names[id(p)]
    assert int(opt._state()["step"]) == 2
    _same_state_dict(opt.state_dict(), ref.state_dict())
    # torch SGD -> package SGD
    hf = _hf_model(cfg)
    names = {id(p): n for n, p in hf.named_parameters()}
    ref = torch.optim.SGD(_groups(hf.named_parameters()), lr=0.05, momentum=0.9)
    for _ in range(2):
        for p in hf.parameters():
            p.grad = torch.randn(p.shape) * 1e-2
        ref.step()
    opt = b2.SGD(_groups(model.named_parameters()), lr=0.05, momentum=0.9)
    opt.load_state_dict(ref.state_dict())
    bufs = opt.momentum_buffers()
    for p, s in ref.state.items():
        assert torch.equal(bufs[names[id(p)]].cpu(), s["momentum_buffer"])


def _trainer_run(cuda_dev, cfg, state, batches, tmp, mode, resume=None, restore_dropout=True, epochs=1, save_steps=2,
                 seen=None, loaded=None):
    """train() of a fresh model, HF AdamW and Trainer; returns (losses, final masters, trainer).  seen: a list that
    receives every batch trained; loaded: a dict that receives the optimizer / scaler state right after the resume's
    load_checkpoint"""
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.AdamW(_groups(model.named_parameters()), lr=2e-4)
    a = b2.Args()
    a.local_rank, a.epochs, a.dev = 0, epochs, False
    a.fused, a.use_amp = mode == "fused", mode == "amp"
    a.gradient_accumulation_steps = 2
    a.max_grad_norm = 1.0
    a.lr_scheduler_type = "linear"
    a.output_dir, a.save_steps = str(tmp), save_steps
    a.ckpt_path = os.path.join(str(tmp), "final.pt")
    a.log_every = 1000
    tr = b2.Trainer(a, cfg, model, torch.nn.CrossEntropyLoss(), opt)
    losses = []
    step = tr.train_step
    if seen is None:
        seen = []
    tr.train_step = lambda bt: seen.append(bt) or losses.append(float(step(bt))) or losses[-1]
    load = functools.partial(tr.load_checkpoint, restore_dropout=restore_dropout)

    def load_and_probe(path):
        out = load(path)
        if loaded is not None:
            loaded["opt"] = _through_bytes(opt.state_dict())
            loaded["step"] = int(opt._state()["step"])
            loaded["scaler"] = None if tr._scaler is None else tr._scaler.state_dict()
        return out
    tr.load_checkpoint = load_and_probe
    tr.train(batches, resume_from_checkpoint=resume)
    torch.cuda.synchronize()
    return losses, model._flat.detach().clone(), tr


@gpu
@pytest.mark.parametrize("mode", ["fused", "amp"])
def test_trainer_resume_follows_the_uninterrupted_run(cuda_dev, tmp_path, mode):
    """train() over 8 batches (dropout on, k = 2, max_grad_norm, a linear schedule, save_steps = 2), then a fresh model,
    optimizer and Trainer resumed from checkpoint-2: the losses and weights of the rest of the run match the uninterrupted
    run.  Control: the same resume without the dropout state is off by clearly more."""
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = [_batch(cfg, 9000 + i) for i in range(8)]
    full_dir = tmp_path / "full"
    losses, w_full, tr = _trainer_run(cuda_dev, cfg, state, batches, full_dir, mode)
    assert tr.global_step == 4 and tr.lr_scheduler.last_epoch == 4
    ckpts = [os.path.basename(p) for p in sorted_checkpoints(str(full_dir))]
    assert ckpts == ["checkpoint-2", "checkpoint-4"]
    ck = str(full_dir / "checkpoint-2")
    files = set(os.listdir(ck))
    assert {"pytorch_model.bin", "config.json", "optimizer.pt", "scheduler.pt", "rng_state_0.pth",
            "trainer_state.json"} <= files and (("scaler.pt" in files) == (mode == "amp"))
    import json
    with open(os.path.join(ck, "trainer_state.json")) as f:
        progress = json.load(f)
    assert progress == {"batches": 4, "epoch": 1, "batches_in_epoch": 4, "best_acc": 0.0, "global_step": 2}
    back = b2.BertForSequenceClassification.from_pretrained(ck)
    saved = torch.load(os.path.join(ck, "pytorch_model.bin"))
    for k, v in back.state_dict().items():
        assert torch.equal(v, saved[k]), k
    loaded = {}
    resumed, w_res, tr2 = _trainer_run(cuda_dev, cfg, state_from_hf_init(cfg, seed=9), batches, tmp_path / "res", mode,
                                       resume=ck, loaded=loaded)
    assert len(resumed) == 4 and tr2.global_step == 4 and tr2.lr_scheduler.last_epoch == 4
    # right after the load the optimizer (and the GradScaler) hold exactly the uninterrupted run's state at step 2: the
    # few-1e-4 moves of the rest of the run could not tell a missing optimizer restore apart on their own
    assert loaded["step"] == 2
    _same_state_dict(loaded["opt"], torch.load(os.path.join(ck, "optimizer.pt")))
    if mode == "amp":
        assert loaded["scaler"] == torch.load(os.path.join(ck, "scaler.pt"))
    else:
        assert loaded["scaler"] is None
    d_ok = max(_max_diff(losses[4:], resumed), float((w_res - w_full).abs().max()))
    assert d_ok <= TOL_TRAJ, (losses[4:], resumed, d_ok)
    ctrl, w_ctrl, _ = _trainer_run(cuda_dev, cfg, state, batches, tmp_path / "ctrl", mode, resume=ck,
                                   restore_dropout=False)
    d_ctrl = _max_diff(losses[4:], ctrl)
    print("resume %s: |dloss| restored %.2e, without the dropout state %.2e" % (mode, d_ok, d_ctrl))
    assert d_ctrl > 5 * d_ok and d_ctrl > 1e-3, (d_ok, d_ctrl)


@gpu
def test_resume_with_a_shuffling_dataloader_sees_the_uninterrupted_batches(cuda_dev, tmp_path):
    """DataLoader(shuffle=True) draws its order from the CPU RNG when an epoch's iterator starts.  Two epochs of 8
    batches, k = 2, a checkpoint every optimizer step; resumed from checkpoint-3 (6 batches into epoch 1), the run trains
    exactly the batches the uninterrupted run trained after it, in the same order, through the second epoch."""
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    big = _batch(cfg, 9200, bsz=32)
    data = [{k: big[k][i] for k in ("input_ids", "token_type_ids", "attention_mask", "label")} for i in range(32)]
    loader = torch.utils.data.DataLoader(data, batch_size=4, shuffle=True)
    full, res = [], []
    torch.manual_seed(11)
    _trainer_run(cuda_dev, cfg, state, loader, tmp_path / "full", "fused", epochs=2, save_steps=1, seen=full)
    assert len(full) == 16 and not torch.equal(full[0]["input_ids"], full[8]["input_ids"])
    torch.manual_seed(12)        # whatever the CPU RNG is now, the resume takes the checkpoint's
    _trainer_run(cuda_dev, cfg, state, loader, tmp_path / "res", "fused", epochs=2, save_steps=1, seen=res,
                 resume=str(tmp_path / "full" / "checkpoint-3"))
    assert len(res) == 10
    for i, (a, b) in enumerate(zip(full[6:], res)):
        for k in a:
            assert torch.equal(a[k], b[k]), (i, k)


@gpu
def test_resume_true_takes_the_latest_checkpoint(cuda_dev, tmp_path):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = [_batch(cfg, 9100 + i) for i in range(8)]
    losses, w_full, _tr = _trainer_run(cuda_dev, cfg, state, batches, tmp_path, "fused")
    resumed, w_res, tr = _trainer_run(cuda_dev, cfg, state, batches, tmp_path, "fused", resume=True)
    assert resumed == [] and tr.global_step == 4 and torch.equal(w_res, w_full)


# ---- GPU: DDP world 2 ---------------------------------------------------------------------------------------------
@gpu
def test_ddp_world2_checkpoint():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29601", os.path.join(ROOT, "tests", "ddp_checkpoint_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_checkpoint_worker: OK" in r.stdout, r.stdout[-3000:]
