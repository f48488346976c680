"""Learning-rate schedules: the package's HF schedules, Trainer scheduler= / lr_scheduler_type, the device lr
(b2_adamw_hparams_t.lr_dev) of the AdamW kernels, and the captured steps reading the lr at every replay.

The zero-lr checks are exact: an AdamW step with lr 0 leaves the fp32 master weights bitwise unchanged (the weight
decay term is lr x wd x w = 0 too), so a schedule that the step ignores shows up as weights that moved."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F
from torch.optim.lr_scheduler import LambdaLR

from parity import (TOL_GRAD_REL_QK, adamw_ref, assert_grads_within_tolerance, b2, bert_ref, full_config, make_model,
                    state_from_hf_init, tiny_config, to_dev)
from pytorch_distributed_nlp_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LR = 3e-5
bf = torch.bfloat16
gpu = pytest.mark.gpu
ZERO_ONE = lambda s: float(s % 2 == 0)       # noqa: E731  multipliers 1, 0, 1, 0, ...


# ---- CPU: schedules, warmup, step count, errors ----------------------------------------------------------------------
def _lrs(sched, n):
    out = []
    for _ in range(n):
        out.append(sched.get_last_lr()[0])
        sched.optimizer.step()
        sched.step()
    return out


def _sgd():
    return torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=LR)


@pytest.mark.parametrize("name", ["linear", "cosine", "constant", "constant_with_warmup"])
@pytest.mark.parametrize("warmup,total", [(0, 10), (3, 10), (10, 10), (0, 1), (1, 1), (4, 7)])
def test_schedules_match_transformers(name, warmup, total):
    """the lr sequence, including steps past `total`, is float-equal to transformers.get_scheduler's"""
    transformers = pytest.importorskip("transformers")
    ours = b2.get_scheduler(name, _sgd(), num_warmup_steps=warmup, num_training_steps=total)
    theirs = transformers.get_scheduler(name, _sgd(), num_warmup_steps=warmup, num_training_steps=total)
    assert _lrs(ours, total + 5) == _lrs(theirs, total + 5)


def test_unknown_schedule_type_raises():
    with pytest.raises(ValueError, match="constant_with_warmup"):
        b2.get_scheduler("polynomial", _sgd(), 0, 10)


def _args(**kw):
    a = b2.Args()
    a.local_rank, a.epochs = None, 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_warmup_ratio_is_ceiled_and_warmup_steps_wins():
    for kw, want in [({"warmup_ratio": 0.25}, 3), ({"warmup_ratio": 0.2}, 2), ({"warmup_ratio": 0.25, "warmup_steps": 5}, 5),
                     ({}, 0)]:
        opt = _sgd()
        tr = b2.Trainer(_args(lr_scheduler_type="linear", **kw), None, None, None, opt)
        sched = tr.create_scheduler(10)
        assert sched is tr.lr_scheduler and sched.lr_lambdas[0].keywords["num_warmup_steps"] == want, (kw, want)
    tr = b2.Trainer(_args(), None, None, None, _sgd())
    assert tr.create_scheduler(10) is None           # lr_scheduler_type None: a constant lr


@pytest.mark.parametrize("epochs,batches,k,want", [(1, 7, 1, 7), (2, 7, 3, 6), (3, 8, 4, 6), (1, 1, 4, 1)])
def test_trainer_total_steps(epochs, batches, k, want):
    """train() builds the schedule over epochs x ceil(batches / k) optimizer steps (the partial window steps too)"""
    tr = b2.Trainer(_args(lr_scheduler_type="linear", epochs=epochs, gradient_accumulation_steps=k), None, None, None,
                    _sgd())
    assert tr.num_training_steps(range(batches)) == want
    tr.train_step = lambda batch: torch.zeros(())
    tr.train(list(range(batches)))
    assert tr.lr_scheduler.lr_lambdas[0].keywords["num_training_steps"] == want


def test_explicit_scheduler_wins_over_args():
    opt = _sgd()
    mine = LambdaLR(opt, ZERO_ONE)
    tr = b2.Trainer(_args(lr_scheduler_type="linear"), None, None, None, opt, scheduler=mine)
    assert tr.create_scheduler(10) is mine


def test_scheduler_errors():
    with pytest.raises(ValueError, match="belong"):
        b2.Trainer(_args(), None, None, None, _sgd(), scheduler=LambdaLR(_sgd(), ZERO_ONE))
    tr = b2.Trainer(_args(lr_scheduler_type="cosine"), None, None, None, _sgd())
    with pytest.raises(RuntimeError, match="create_scheduler"):
        tr.train_step({})


def test_unequal_group_lrs_raise_at_step():
    model = b2.BertForSequenceClassification(tiny_config())
    opt = b2.build_optimizer(model, _args(weight_decay=0.01, learning_rate=LR))
    opt.param_groups[1]["lr"] = 2 * LR
    with pytest.raises(ValueError, match="different learning rates"):
        opt.step()


# ---- GPU, kernel level: the device lr is the by-value lr, bit for bit -------------------------------------------------
def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    itype = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}[got.dtype]
    assert torch.equal(got.view(itype), want.view(itype))


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _kernel_run(cuda_dev, kernel, lr, lr_dev, steps=2):
    """`steps` updates of one slice; lr_dev: the lr comes from a device fp64 scalar (hp.lr is then a decoy)"""
    world = 2 if kernel == "reduce2" else 1
    n = 8 * 20000
    b, e = 8 * 37, n - 8 * 101
    gen = torch.Generator(device=cuda_dev).manual_seed(3)
    decay = (torch.rand(n // 8, device=cuda_dev, generator=gen) < 0.5).to(torch.uint8)
    master = torch.randn(n, device=cuda_dev, generator=gen)
    master0 = master.clone()
    m, v = torch.zeros(n, device=cuda_dev), torch.zeros(n, device=cuda_dev)
    shadow = [torch.zeros(n, dtype=bf, device=cuda_dev) for _ in range(world)]
    step = torch.zeros(1, dtype=torch.int64, device=cuda_dev)
    ss = torch.zeros(1, device=cuda_dev)
    lr_t = torch.tensor([lr], dtype=torch.float64, device=cuda_dev)
    hp = L.AdamWHParams()
    hp.lr, hp.beta1, hp.beta2, hp.eps, hp.weight_decay, hp.correct_bias = lr, 0.9, 0.999, 1e-6, 0.01, 1
    if lr_dev:
        hp.lr, hp.lr_dev = 0.37, lr_t.data_ptr()
    for _ in range(steps):
        grads = [(torch.randn(n, device=cuda_dev, generator=gen) * 1e-2).to(bf) for _ in range(world)]
        if kernel == "slim":
            L.call("b2_adamw_prepare", hp, step.data_ptr(), ss.data_ptr(), _stream())
            L.call("b2_adamw_background", grads[0].data_ptr(), shadow[0].data_ptr(), master.data_ptr(), m.data_ptr(),
                   v.data_ptr(), decay.data_ptr(), b, e, hp, ss.data_ptr(), _stream())
        else:
            L.call("b2_bucket_reduce_adamw", L.ptr_array([g.data_ptr() for g in grads]),
                   L.ptr_array([s.data_ptr() for s in shadow]), world, 0, master.data_ptr(), m.data_ptr(),
                   v.data_ptr(), decay.data_ptr(), b, e, hp, step.data_ptr(), _stream())
        L.call("b2_step_advance", step.data_ptr(), None, None, _stream())
    torch.cuda.synchronize()
    return [master, m, v] + shadow, master0


@gpu
@pytest.mark.parametrize("lr", [3e-5, 1.7e-4, 0.0])
@pytest.mark.parametrize("kernel", ["reduce1", "reduce2", "slim"])
def test_device_lr_is_the_by_value_lr(cuda_dev, kernel, lr):
    """master, moments and shadow with lr_dev holding x are bitwise those with x passed by value"""
    for got, want in zip(_kernel_run(cuda_dev, kernel, lr, True)[0], _kernel_run(cuda_dev, kernel, lr, False)[0]):
        _same(got, want)


@gpu
@pytest.mark.parametrize("kernel", ["reduce1", "reduce2", "slim"])
def test_device_lr_zero_leaves_the_master(cuda_dev, kernel):
    """lr 0 from the device: the fp32 master is bitwise its initial value, the moments those of an lr 1e-3 run"""
    zero, master0 = _kernel_run(cuda_dev, kernel, 0.0, True)
    moved, _ = _kernel_run(cuda_dev, kernel, 1e-3, True)
    _same(zero[0], master0)
    assert not torch.equal(moved[0], master0)
    _same(zero[1], moved[1])
    _same(zero[2], moved[2])


# ---- GPU, end to end: a [1, 0, 1, 0, ...] schedule is exact on every path --------------------------------------------
def _tiny(**kw):
    cfg = tiny_config(**kw)
    return cfg, state_from_hf_init(cfg)


def _batch(cfg, seed=8100, bsz=4):
    return bert_ref.synthetic_batch(cfg, bsz, 128, seed, padded=True)


def _check_zero_one(model, run_step, steps, sched):
    """run_step(i) takes optimizer step i; sched multiplies by 1, 0, 1, 0, ...: the master moves exactly on the 1s"""
    for i in range(steps):
        before = model._flat.detach().clone()
        assert sched.get_last_lr()[0] == LR * ZERO_ONE(i)
        run_step(i)
        torch.cuda.synchronize()
        if ZERO_ONE(i) == 0.0:
            assert torch.equal(model._flat, before), "step %d has lr 0 but the master weights moved" % i
        else:
            assert not torch.equal(model._flat, before), "step %d did not move the master weights" % i


def _opt(model):
    return b2.build_optimizer(model, _args(weight_decay=0.01, learning_rate=LR))


@gpu
@pytest.mark.parametrize("kind", ["fused", "packed"])
def test_zero_lr_steps_on_the_captured_steps(cuda_dev, kind):
    """FusedTrainStep / PackedTrainStep driven directly, a torch LambdaLR on the optimizer: two eager warm-up
    steps, then capture and replays"""
    cfg, state = _tiny()
    model = make_model(cfg, state, cuda_dev).train()
    opt = _opt(model)
    sched = LambdaLR(opt, ZERO_ONE)
    bt = _batch(cfg)
    if kind == "fused":
        st = b2.FusedTrainStep(model, opt, 4, 128)
        call = lambda: st(bt)      # noqa: E731
    else:
        packed = b2.pack_batch(bt["input_ids"], bt["token_type_ids"], bt["attention_mask"])
        st = b2.PackedTrainStep(model, opt, packed["bins"], 4)
        call = lambda: st(packed, bt["label"])      # noqa: E731

    def run(i):
        call()
        sched.step()
    _check_zero_one(model, run, 7, sched)
    assert st.graph is not None


@gpu
@pytest.mark.parametrize("mode,k,clip", [("fused", 1, None), ("packed", 1, None), ("eager", 1, None),
                                         ("fused", 2, None), ("eager", 2, None), ("fused", 1, 1.0),
                                         ("packed", 1, 1.0), ("eager", 1, 1.0)])
def test_zero_lr_steps_through_the_trainer(cuda_dev, mode, k, clip):
    """Trainer(scheduler=...): stepped once per optimizer step (per window with k = 2), with and without clipping"""
    cfg, state = _tiny()
    model = make_model(cfg, state, cuda_dev).train()
    opt = _opt(model)
    sched = LambdaLR(opt, ZERO_ONE)
    args = _args(fused=mode != "eager", pack=mode == "packed", gradient_accumulation_steps=k, max_grad_norm=clip)
    args.local_rank = 0
    tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt, scheduler=sched)

    def run(i):
        for j in range(k):
            before = model._flat.detach().clone()
            tr.train_step(_batch(cfg, 8100 + 10 * i + j))
            if j < k - 1:
                torch.cuda.synchronize()
                assert torch.equal(model._flat, before), "a micro-batch moved the weights"
                assert sched.last_epoch == i, "the scheduler stepped on a micro-batch"
    _check_zero_one(model, run, 6, sched)
    assert sched.last_epoch == 6


@gpu
def test_zero_lr_steps_in_an_eager_loop_after_the_captured_step(cuda_dev):
    """once a FusedTrainStep has armed the optimizer, an eager backward launches the per-bucket background update: its
    step size is prepared from the lr current at that backward, not at the previous step()"""
    cfg, state = _tiny()
    model = make_model(cfg, state, cuda_dev).train()
    opt = _opt(model)
    bt = _batch(cfg)
    st = b2.FusedTrainStep(model, opt, 4, 128)
    st(bt)
    torch.cuda.synchronize()
    assert opt._armed
    sched = LambdaLR(opt, ZERO_ONE)
    d = to_dev(bt, cuda_dev)

    def run(i):
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                    labels=d["label"])
        F.cross_entropy(out[1], d["label"]).backward()
        opt.step()
        sched.step()
    _check_zero_one(model, run, 6, sched)


# ---- GPU, against the oracle: Trainer lr_scheduler_type="linear" with warmup -------------------------------------------
STEPS, WARMUP = 4, 1
_CACHE = {}


def _oracle_setup(size):
    if size not in _CACHE:
        transformers = pytest.importorskip("transformers")
        if size == "tiny":
            cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
            state = state_from_hf_init(cfg)
            bsz, odev = 4, "cpu"
        else:
            cfg = full_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
            b2.set_seed(123)
            m = b2.BertForSequenceClassification(cfg)
            state = {k: v.detach().clone() for k, v in m.state_dict().items() if k in m._params_by_name}
            del m
            bsz, odev = 8, "cuda"
        batches = [bert_ref.synthetic_batch(cfg, bsz, 128, 8500 + s, padded=True) for s in range(STEPS)]
        ref = {k: v.to(odev).clone() for k, v in state.items()}
        opt = adamw_ref.HFAdamW(ref, lr=LR, weight_decay=0.01)
        up = transformers.get_scheduler("linear", _sgd(), num_warmup_steps=WARMUP, num_training_steps=STEPS)
        for bt in batches:
            opt.lr = up.get_last_lr()[0]
            _l, _z, g = bert_ref.loss_and_grads(ref, cfg, to_dev(bt, odev))
            opt.step(g)
            up.optimizer.step()
            up.step()
        _CACHE[size] = (cfg, state, batches, {k: v.cpu() for k, v in ref.items()},
                        {k: opt.state[k]["exp_avg"].cpu() for k in ref})
    return _CACHE[size]


@gpu
@pytest.mark.parametrize("mode", ["loop", "eager", "fused", "packed"])
@pytest.mark.parametrize("size", ["tiny", "configA"])
def test_linear_warmup_schedule_matches_oracle(cuda_dev, size, mode):
    """4 steps, warmup 1, dropout off: weights and first moments against HF AdamW with the upstream schedule's lr;
    the first step has lr 0 and leaves the master bitwise unchanged.  `loop` attaches transformers' own scheduler to
    the package AdamW in a hand-written loop."""
    cfg, state, batches, rw, rm = _oracle_setup(size)
    model = make_model(cfg, state, cuda_dev).train()
    if mode == "loop":
        import transformers
        opt = _opt(model)
        sched = transformers.get_scheduler("linear", opt, num_warmup_steps=WARMUP, num_training_steps=STEPS)

        def step(bt):
            d = to_dev(bt, cuda_dev)
            out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                        attention_mask=d["attention_mask"], labels=d["label"])
            F.cross_entropy(out[1], d["label"]).backward()
            opt.step()
            sched.step()
    else:
        args = _args(fused=mode != "eager", pack=mode == "packed", lr_scheduler_type="linear", warmup_steps=WARMUP,
                     weight_decay=0.01, learning_rate=LR)
        args.local_rank = 0
        opt = b2.build_optimizer(model, args)
        tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)
        tr.create_scheduler(STEPS)
        step = tr.train_step
    for i, bt in enumerate(batches):
        before = model._flat.detach().clone()
        step(bt)
        if i == 0:
            torch.cuda.synchronize()
            assert torch.equal(model._flat, before), "warmup step 0 has lr 0"
    torch.cuda.synchronize()
    w = {n: v.detach().cpu() for n, v in model.state_dict().items()}
    m = {n: ea.detach().cpu() for n, (ea, _v) in opt.moments().items()}
    for n, v in rw.items():
        assert float((w[n] - v).abs().max()) <= 2 * LR * STEPS + 2e-5, n
    assert_grads_within_tolerance(m, rm, qk_tol=TOL_GRAD_REL_QK)
    torch.cuda.empty_cache()


# ---- GPU: GradScaler skip, guard, groups ------------------------------------------------------------------------------
class _PoisonedLoss(torch.nn.CrossEntropyLoss):
    """the loss of call `bad` is inf: every gradient of that step is non-finite and GradScaler skips it"""

    def __init__(self, bad):
        super().__init__()
        self.calls, self.bad = 0, bad

    def forward(self, logits, label):
        loss = super().forward(logits, label)
        self.calls += 1
        return loss * float("inf") if self.calls - 1 == self.bad else loss


@gpu
def test_gradscaler_skip_does_not_step_the_schedule(cuda_dev):
    """Trainer use_amp: a skipped step leaves the weights, the AdamW step count and get_last_lr() as they were, and
    the next step runs at the lr the skipped one would have used (it lands where the run without that batch lands)"""
    cfg, state = _tiny(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)   # the skip still bumps the RNG
    lr, mult = 1e-3, [1.0, 0.5, 0.25, 0.125]
    batches = [_batch(cfg, 8700 + s) for s in range(3)]
    runs = []
    for bad in (None, 1):
        model = make_model(cfg, state, cuda_dev).train()
        opt = b2.build_optimizer(model, _args(weight_decay=0.01, learning_rate=lr))
        sched = LambdaLR(opt, lambda s: mult[s])
        args = _args(fused=False, use_amp=True)
        args.local_rank = 0
        tr = b2.Trainer(args, cfg, model, _PoisonedLoss(-1 if bad is None else bad), opt, scheduler=sched)
        seq = [batches[0], batches[1], batches[2]] if bad is not None else [batches[0], batches[2]]
        for i, bt in enumerate(seq):
            before = (model._flat.detach().clone(), int(opt._state()["step"]), sched.get_last_lr())
            tr.train_step(bt)
            torch.cuda.synchronize()
            if i == bad:
                assert torch.equal(model._flat, before[0])
                assert int(opt._state()["step"]) == before[1] and sched.get_last_lr() == before[2]
        assert sched.get_last_lr()[0] == lr * mult[2]
        runs.append(model._flat.detach().clone())
    assert float((runs[0] - runs[1]).abs().max()) <= 1e-6


@gpu
@pytest.mark.parametrize("field,value", [("betas", (0.8, 0.999)), ("weight_decay", 0.02), ("eps", 1e-8),
                                         ("correct_bias", False)])
def test_captured_step_rejects_changed_hyperparameters(cuda_dev, field, value):
    cfg, state = _tiny()
    model = make_model(cfg, state, cuda_dev).train()
    opt = _opt(model)
    bt = _batch(cfg)
    st = b2.FusedTrainStep(model, opt, 4, 128)
    for _ in range(4):
        st(bt)
    assert st.graph is not None
    opt.param_groups[0][field] = value
    with pytest.raises(RuntimeError, match=field):
        st(bt)


@gpu
def test_unequal_group_lrs_raise_on_the_gpu_paths(cuda_dev):
    cfg, state = _tiny()
    model = make_model(cfg, state, cuda_dev).train()
    opt = _opt(model)
    bt = _batch(cfg)
    LambdaLR(opt, [lambda s: 1.0, lambda s: 0.5])      # one lambda per group: group 1 runs at half the lr
    d = to_dev(bt, cuda_dev)
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    with pytest.raises(ValueError, match="different learning rates"):
        opt.step()
    with pytest.raises(ValueError, match="different learning rates"):
        b2.FusedTrainStep(model, opt, 4, 128)
    assert not opt._armed
    opt.param_groups[1]["lr"] = opt.param_groups[0]["lr"]
    st = b2.FusedTrainStep(model, opt, 4, 128)
    opt.param_groups[1]["lr"] = 0.5 * opt.param_groups[0]["lr"]
    with pytest.raises(ValueError, match="different learning rates"):
        st(bt)


# ---- GPU: DDP world 2 --------------------------------------------------------------------------------------------------
@gpu
def test_ddp_world2_schedule():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29593", os.path.join(ROOT, "tests", "ddp_lr_schedule_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_lr_schedule_worker: OK" in r.stdout, r.stdout[-3000:]
