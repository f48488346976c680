"""SGD with momentum: the package's torch.optim.SGD on the fused update (b2_bucket_reduce_sgd / b2_sgd_background).

Kernel level the update is bitwise torch.optim.SGD(foreach=False) on the GPU over the same fp32 gradient.  Model level
it is the oracle (bert_ref.loss_and_grads) plus torch SGD on the fp32 oracle parameters, to the rel-L2 tolerances of
tests/parity.py, on every training path."""
import itertools
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F
from torch.optim.lr_scheduler import CosineAnnealingLR, LambdaLR

from parity import (TOL_GRAD_REL_QK, assert_grads_within_tolerance, b2, bert_ref, full_config, make_model,
                    state_from_hf_init, tiny_config, to_dev)
from pytorch_distributed_nlp_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
bf = torch.bfloat16
gpu = pytest.mark.gpu


def _args(**kw):
    a = b2.Args()
    a.local_rank, a.epochs = None, 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


# ---- CPU: constructor, groups, build_optimizer, ABI ------------------------------------------------------------------
def _tiny_model():
    return b2.BertForSequenceClassification(tiny_config())


@pytest.mark.parametrize("kw", [dict(lr=-1e-3), dict(momentum=-0.1), dict(weight_decay=-0.01),
                                dict(nesterov=True), dict(nesterov=True, momentum=0.9, dampening=0.1)])
def test_constructor_validation_matches_torch(kw):
    with pytest.raises(ValueError) as theirs:
        torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], **kw)
    with pytest.raises(ValueError) as ours:
        b2.SGD(_tiny_model().parameters(), **kw)
    assert str(ours.value) == str(theirs.value)


def test_defaults_and_ignored_flags():
    model = _tiny_model()
    opt = b2.SGD(model.parameters(), foreach=True, fused=False, differentiable=False)
    g = opt.param_groups[0]
    assert (g["lr"], g["momentum"], g["dampening"], g["weight_decay"], g["nesterov"], g["maximize"]) == \
        (1e-3, 0, 0, 0, False, False)
    assert model._optimizer is opt
    with pytest.raises(ValueError, match="differentiable"):
        b2.SGD(model.parameters(), differentiable=True)


def test_foreign_and_partial_parameters_are_rejected():
    with pytest.raises(TypeError, match="ONE b200"):
        b2.SGD([torch.nn.Parameter(torch.zeros(8))], lr=0.1)
    a, b = _tiny_model(), _tiny_model()
    with pytest.raises(TypeError, match="ONE b200"):
        b2.SGD(list(a.parameters()) + list(b.parameters()), lr=0.1)
    with pytest.raises(ValueError, match="every parameter"):
        b2.SGD(list(a.parameters())[:-1], lr=0.1)


def test_group_rules():
    model = _tiny_model()
    named = list(model.named_parameters())
    dec = [p for n, p in named if "bias" not in n]
    nod = [p for n, p in named if "bias" in n]
    opt = b2.SGD([{"params": dec, "weight_decay": 0.01}, {"params": nod, "weight_decay": 0.0}], lr=0.1, momentum=0.9)
    assert opt._wd == 0.01
    for kw in (dict(momentum=0.5), dict(dampening=0.1), dict(maximize=True), dict(lr=0.2)):
        with pytest.raises(ValueError, match="differ only in weight_decay"):
            b2.SGD([{"params": dec}, dict(params=nod, **kw)], lr=0.1, momentum=0.9)
    with pytest.raises(ValueError, match="one non-zero weight_decay"):
        b2.SGD([{"params": dec, "weight_decay": 0.01}, {"params": nod, "weight_decay": 0.02}], lr=0.1)
    opt.param_groups[1]["lr"] = 0.05
    with pytest.raises(ValueError, match="different learning rates"):
        opt.step()


def test_build_optimizer_optim_sgd_is_fabrics_call():
    model = _tiny_model()
    opt = b2.build_optimizer(model, _args(optim="sgd", learning_rate=0.02, weight_decay=0.01))
    assert type(opt) is b2.SGD and len(opt.param_groups) == 1
    g = opt.param_groups[0]
    assert (g["lr"], g["momentum"], g["dampening"], g["weight_decay"], g["nesterov"], g["maximize"]) == \
        (0.02, 0, 0, 0, False, False)
    assert len(g["params"]) == len(list(model.parameters()))
    with pytest.raises(ValueError, match="optim"):
        b2.build_optimizer(_tiny_model(), _args(optim="adam"))
    assert b2.Args.optim == "adamw"
    opt = b2.build_optimizer(_tiny_model(), _args(weight_decay=0.01))
    assert type(opt) is b2.AdamW and [g["weight_decay"] for g in opt.param_groups] == [0.01, 0.0]


def test_signatures_carry_the_sgd_entry_points():
    assert "b2_bucket_reduce_sgd" in L._SIGNATURES and "b2_sgd_background" in L._SIGNATURES
    assert {"b2_bucket_reduce_sgd", "b2_sgd_background"} <= set(L.EXPORTED_SYMBOLS)
    assert [f for f, _t in L.SGDHParams._fields_] == ["lr", "momentum", "dampening", "weight_decay", "nesterov",
                                                     "maximize", "grad_scale", "found_inf", "clip_coef", "grad_f32",
                                                     "lr_dev"]


def test_slim_sgd_kernel_fits_beside_the_gemm():
    """ptxas: the background form at <= 32 registers with no spills"""
    import re
    import tempfile
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc"
    src = os.path.join(ROOT, "pytorch-distributed-nlp_b200", "csrc", "optim.cu")
    with tempfile.TemporaryDirectory() as tmp:
        try:
            r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-Xptxas", "-v",
                                "-c", src, "-o", os.path.join(tmp, "optim.o")], capture_output=True, text=True)
        except FileNotFoundError:
            pytest.skip("nvcc not found")
    assert r.returncode == 0, r.stderr[-2000:]
    text = r.stderr
    blocks = text.split("Compiling entry function")
    slim = [b for b in blocks if "slim_update_kernel" in b and "SgdRule" in b]
    assert len(slim) == 1, text[-2000:]
    regs = int(re.search(r"Used (\d+) registers", slim[0]).group(1))
    assert regs <= 32 and "0 bytes spill stores, 0 bytes spill loads" in slim[0], slim[0]


# ---- GPU, kernel level: bitwise torch.optim.SGD(foreach=False) ---------------------------------------------------------
def _same(got, want, what=""):
    assert got.dtype == want.dtype and got.shape == want.shape, what
    itype = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}[got.dtype]
    bad = int((got.view(itype) != want.view(itype)).sum())
    assert bad == 0, "%s: %d elements differ" % (what, bad)


def _stream():
    return torch.cuda.current_stream().cuda_stream


N = 8 * 20000
B0, E0 = 8 * 37, N - 8 * 101       # the slice the kernels update; everything outside it must stay put


class _Run:
    """One flat state (master, decay flags, optional momentum buffer, shadows, step count) stepped by one kernel form:
    'reduce1' / 'reduce2' (world 2: two gradient buffers on this device) / 'slim'."""

    def __init__(self, dev, kernel, lr=0.05, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False,
                 maximize=False, seed=5):
        self.dev, self.kernel = dev, kernel
        self.world = 2 if kernel == "reduce2" else 1
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.decay = (torch.rand(N // 8, device=dev, generator=gen) < 0.5).to(torch.uint8)
        self.master = torch.randn(N, device=dev, generator=gen)
        self.master0 = self.master.clone()
        self.buf = torch.full((N,), float("nan"), device=dev) if momentum != 0 else None   # never read before set
        self.shadow = [torch.zeros(N, dtype=bf, device=dev) for _ in range(self.world)]
        self.step = torch.zeros(1, dtype=torch.int64, device=dev)
        self.hp = L.SGDHParams()
        self.hp.lr, self.hp.momentum, self.hp.dampening, self.hp.weight_decay = lr, momentum, dampening, weight_decay
        self.hp.nesterov, self.hp.maximize = int(nesterov), int(maximize)
        self.cfg = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov,
                        maximize=maximize)
        self.gen = gen

    def grads(self, scale=1.0):
        return [(torch.randn(N, device=self.dev, generator=self.gen) * 1e-1 * scale).to(bf) for _ in range(self.world)]

    def step_once(self, grads, **fields):
        """one update + b2_step_advance; fields: optional b2_sgd_hparams_t pointers for this step only"""
        for k, v in fields.items():
            setattr(self.hp, k, v)
        if self.kernel == "slim":
            L.call("b2_sgd_background", grads[0].data_ptr(), self.shadow[0].data_ptr(), self.master.data_ptr(),
                   L.ptr(self.buf), self.decay.data_ptr(), B0, E0, self.hp, self.step.data_ptr(), _stream())
        else:
            L.call("b2_bucket_reduce_sgd", L.ptr_array([g.data_ptr() for g in grads]),
                   L.ptr_array([s.data_ptr() for s in self.shadow]), self.world, 0, self.master.data_ptr(),
                   L.ptr(self.buf), self.decay.data_ptr(), B0, E0, self.hp, self.step.data_ptr(), _stream())
        L.call("b2_step_advance", self.step.data_ptr(), None, fields.get("found_inf"), _stream())
        for k in fields:
            setattr(self.hp, k, None)

    def state(self):
        torch.cuda.synchronize()
        out = [self.master.clone()] + [s.clone() for s in self.shadow]
        return out + ([self.buf.clone()] if self.buf is not None else [])


def _fp32_grad(grads):
    """the gradient the kernels form: rank-order fp32 sum from +0, times 1/world"""
    g = torch.zeros(N, device=grads[0].device)
    for x in grads:
        g = g + x.float()
    return g * (1.0 / len(grads))


class _Torch:
    """torch.optim.SGD(foreach=False) on the same slice: group 0 the decayed elements, group 1 the rest"""

    def __init__(self, run):
        self.mask = run.decay.repeat_interleave(8)[B0:E0].bool()
        w = run.master0[B0:E0]
        self.p = [torch.nn.Parameter(w[self.mask].clone()), torch.nn.Parameter(w[~self.mask].clone())]
        c = dict(run.cfg)
        wd = c.pop("weight_decay")
        self.opt = torch.optim.SGD([{"params": [self.p[0]], "weight_decay": wd},
                                    {"params": [self.p[1]], "weight_decay": 0.0}], foreach=False, **c)

    def step(self, g):
        g = g[B0:E0]
        self.p[0].grad, self.p[1].grad = g[self.mask].clone(), g[~self.mask].clone()
        self.opt.step()

    def flat(self, parts):
        out = torch.empty(E0 - B0, device=parts[0].device)
        out[self.mask], out[~self.mask] = parts[0], parts[1]
        return out


def _check_against_torch(run, ref):
    st = run.state()
    master = st[0]
    _same(master[B0:E0], ref.flat([p.detach() for p in ref.p]), "master")
    _same(master[:B0], run.master0[:B0], "master before the slice")
    _same(master[E0:], run.master0[E0:], "master after the slice")
    for s in st[1:1 + run.world]:
        _same(s[B0:E0], master[B0:E0].to(bf), "shadow")
    if run.buf is not None:
        _same(st[-1][B0:E0], ref.flat([ref.opt.state[p]["momentum_buffer"] for p in ref.p]), "momentum buffer")
    else:
        assert all("momentum_buffer" not in ref.opt.state[p] or ref.opt.state[p]["momentum_buffer"] is None
                   for p in ref.p)


def _combos():
    for mom, damp, nest, wd, mx in itertools.product([0.0, 0.9], [0.0, 0.1], [False, True], [0.0, 1e-2],
                                                     [False, True]):
        if nest and (mom <= 0 or damp != 0):
            continue        # torch rejects it
        yield dict(momentum=mom, dampening=damp, nesterov=nest, weight_decay=wd, maximize=mx)


COMBOS = list(_combos())
KERNELS = ["reduce1", "reduce2", "slim"]


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cfg", COMBOS, ids=lambda c: "m%g-d%g-n%d-wd%g-max%d" % (
    c["momentum"], c["dampening"], c["nesterov"], c["weight_decay"], c["maximize"]))
def test_kernel_is_torch_sgd_bitwise(cuda_dev, kernel, cfg):
    """4 steps on a random flat state with random decay flags: master, buffer and shadow bitwise torch's"""
    run = _Run(cuda_dev, kernel, **cfg)
    ref = _Torch(run)
    for _ in range(4):
        grads = run.grads()
        run.step_once(grads)
        ref.step(_fp32_grad(grads))
    _check_against_torch(run, ref)


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
def test_first_step_buffer_is_the_gradient(cuda_dev, kernel):
    run = _Run(cuda_dev, kernel, momentum=0.9, dampening=0.1)
    grads = run.grads()
    run.step_once(grads)
    _same(run.state()[-1][B0:E0], _fp32_grad(grads)[B0:E0], "buffer after the first step")
    assert int(run.step) == 1


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("lr", [0.05, 1.7e-4, 0.0])
def test_device_lr_is_the_by_value_lr(cuda_dev, kernel, lr):
    """lr_dev holding x gives bitwise the run with x by value (hp.lr is a decoy then)"""
    cfg = dict(momentum=0.9, weight_decay=1e-2, nesterov=True)
    a, b = _Run(cuda_dev, kernel, lr=lr, **cfg), _Run(cuda_dev, kernel, lr=0.37, **cfg)
    lr_t = torch.tensor([lr], dtype=torch.float64, device=cuda_dev)
    for _ in range(3):
        a.step_once(a.grads())
        b.step_once(b.grads(), lr_dev=lr_t.data_ptr())
    for x, y in zip(a.state(), b.state()):
        _same(y, x, "lr_dev")


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
def test_zero_lr_leaves_the_master_and_moves_the_buffer(cuda_dev, kernel):
    run = _Run(cuda_dev, kernel, lr=0.0, momentum=0.9, weight_decay=1e-2)
    bufs = []
    for _ in range(2):
        run.step_once(run.grads())
        bufs.append(run.state()[-1])
    _same(run.master, run.master0, "master at lr 0")
    assert not torch.equal(bufs[0][B0:E0], bufs[1][B0:E0])


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
def test_clip_coef_is_torch_on_the_clipped_gradient(cuda_dev, kernel):
    run = _Run(cuda_dev, kernel, momentum=0.9, weight_decay=1e-2)
    ref = _Torch(run)
    coef = torch.tensor(0.3, device=cuda_dev)
    for _ in range(3):
        grads = run.grads()
        run.step_once(grads, clip_coef=coef.data_ptr())
        ref.step(_fp32_grad(grads) * coef)
    _check_against_torch(run, ref)


@gpu
@pytest.mark.parametrize("world", [1, 2])
def test_grad_f32_equals_the_peer_read(cuda_dev, world):
    kernel = "reduce%d" % world
    cfg = dict(momentum=0.9, dampening=0.1, weight_decay=1e-2)
    a, b = _Run(cuda_dev, kernel, **cfg), _Run(cuda_dev, kernel, **cfg)
    for _ in range(3):
        ga, gb = a.grads(), b.grads()
        a.step_once(ga)
        stash = _fp32_grad(gb)[B0:E0].contiguous()
        b.step_once(gb, grad_f32=stash.data_ptr())
    for x, y in zip(a.state(), b.state()):
        _same(y, x, "grad_f32")


@gpu
@pytest.mark.parametrize("world", [1, 2])
def test_grad_scale_unscales(cuda_dev, world):
    kernel = "reduce%d" % world
    cfg = dict(momentum=0.9, weight_decay=1e-2)
    a, b = _Run(cuda_dev, kernel, **cfg), _Run(cuda_dev, kernel, **cfg)
    scale = torch.tensor(1024.0, device=cuda_dev)
    for _ in range(3):
        ga, gb = a.grads(), b.grads(scale=1024.0)      # a power of two: bf16(1024 x) = 1024 bf16(x)
        a.step_once(ga)
        b.step_once(gb, grad_scale=scale.data_ptr())
    for x, y in zip(a.state(), b.state()):
        _same(y, x, "grad_scale")


@gpu
@pytest.mark.parametrize("world", [1, 2])
def test_found_inf_skips_everything_and_the_next_step_initialises_the_buffer(cuda_dev, world):
    kernel = "reduce%d" % world
    cfg = dict(momentum=0.9, dampening=0.1, weight_decay=1e-2)
    run = _Run(cuda_dev, kernel, **cfg)
    before = run.state()
    inf = torch.tensor(1.0, device=cuda_dev)
    run.step_once(run.grads(), found_inf=inf.data_ptr())
    for x, y in zip(run.state(), before):
        _same(x, y, "skipped step")
    assert int(run.step) == 0
    # the next applied step is torch's first one
    ref = _Torch(run)
    for _ in range(2):
        grads = run.grads()
        run.step_once(grads)
        ref.step(_fp32_grad(grads))
    _check_against_torch(run, ref)
    assert int(run.step) == 2


@gpu
def test_buffer_pointer_matches_momentum(cuda_dev):
    """momentum 0 never touches a buffer (NULL is passed); a buffer with momentum 0, or none with momentum, raises"""
    run = _Run(cuda_dev, "reduce1", momentum=0.0)
    g = run.grads()
    run.buf = torch.zeros(N, device=cuda_dev)
    with pytest.raises(RuntimeError, match="momentum_buffer"):
        run.step_once(g)
    run = _Run(cuda_dev, "slim", momentum=0.9)
    run.buf = None
    with pytest.raises(RuntimeError, match="momentum_buffer"):
        run.step_once(g)


# ---- GPU, model level: the oracle + torch SGD ---------------------------------------------------------------------------
STEPS, LR, MOM, WD = 4, 0.01, 0.9, 0.01     # lr: deltas far above the fp32 rounding of w, a short trajectory
_CACHE = {}


def _base(size):
    if size == "tiny":
        cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
        return cfg, state_from_hf_init(cfg), 4, "cpu"
    cfg = full_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    b2.set_seed(123)
    m = b2.BertForSequenceClassification(cfg)
    state = {k: v.detach().clone() for k, v in m.state_dict().items() if k in m._params_by_name}
    del m
    return cfg, state, 8, "cuda"


def _oracle(size, k, clip):
    """STEPS torch SGD(momentum, weight_decay) + CosineAnnealingLR steps on the fp32 oracle; a step's gradient is the
    mean over its k micro-batches, clipped (torch.nn.utils.clip_grad_norm_) to a quarter of the first step's norm"""
    key = (size, k, clip)
    if key not in _CACHE:
        if size not in _CACHE:
            _CACHE[size] = _base(size)
        cfg, state, bsz, odev = _CACHE[size]
        batches = [[bert_ref.synthetic_batch(cfg, bsz, 128, 8800 + 10 * s + j, padded=True) for j in range(k)]
                   for s in range(STEPS)]
        ref = {n: torch.nn.Parameter(v.to(odev).clone()) for n, v in state.items()}
        opt = torch.optim.SGD(list(ref.values()), lr=LR, momentum=MOM, weight_decay=WD, foreach=False)
        sched = CosineAnnealingLR(opt, T_max=STEPS)
        max_norm = None
        for s in range(STEPS):
            g = None
            for bt in batches[s]:
                _l, _z, gi = bert_ref.loss_and_grads({n: p.detach() for n, p in ref.items()}, cfg, to_dev(bt, odev))
                g = {n: x / k for n, x in gi.items()} if g is None else {n: g[n] + x / k for n, x in gi.items()}
            for n, p in ref.items():
                p.grad = g[n].clone()
            if clip:
                if max_norm is None:
                    max_norm = 0.25 * float(torch.nn.utils.get_total_norm([p.grad for p in ref.values()]))
                torch.nn.utils.clip_grad_norm_(list(ref.values()), max_norm)
            opt.step()
            sched.step()
        deltas = {n: (p.detach().cpu() - state[n]) for n, p in ref.items()}
        bufs = {n: opt.state[p]["momentum_buffer"].cpu() for n, p in ref.items()}
        _CACHE[key] = (cfg, state, batches, max_norm, deltas, bufs)
    return _CACHE[key]


def _loop_step(model, opt, d, max_norm):
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    if max_norm is not None:
        b2.clip_grad_norm_(model.parameters(), max_norm)
    opt.step()


MODES = ["loop", "eager", "fused", "packed", "amp", "k2"]


@gpu
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("size", ["tiny", "configA"])
def test_sgd_matches_oracle(cuda_dev, size, mode, clip):
    """4 steps of SGD(momentum=0.9, weight_decay=0.01) with CosineAnnealingLR, dropout off: the weight deltas and the
    momentum buffers per tensor against torch SGD on the oracle"""
    k = 2 if mode == "k2" else 1
    cfg, state, batches, max_norm, rdelta, rbuf = _oracle(size, k, clip)
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.SGD(model.parameters(), lr=LR, momentum=MOM, weight_decay=WD)
    sched = CosineAnnealingLR(opt, T_max=STEPS)
    if mode == "loop":
        for s in range(STEPS):
            _loop_step(model, opt, to_dev(batches[s][0], cuda_dev), max_norm)
            sched.step()
    else:
        args = _args(fused=mode in ("fused", "packed", "k2"), pack=mode == "packed", use_amp=mode == "amp",
                     gradient_accumulation_steps=k, max_grad_norm=max_norm)
        args.local_rank = 0
        tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt, scheduler=sched)
        for s in range(STEPS):
            for bt in batches[s]:
                tr.train_step(bt)
    torch.cuda.synchronize()
    assert sched.last_epoch == STEPS
    w = {n: v.detach().cpu() for n, v in model.state_dict().items()}
    delta = {n: w[n] - state[n] for n in rdelta}
    assert_grads_within_tolerance(delta, rdelta, qk_tol=TOL_GRAD_REL_QK)
    bufs = {n: v.detach().cpu() for n, v in opt.momentum_buffers().items()}
    assert_grads_within_tolerance(bufs, rbuf, qk_tol=TOL_GRAD_REL_QK)
    torch.cuda.empty_cache()


def _tiny_run():
    cfg = tiny_config()
    return cfg, state_from_hf_init(cfg)


def _batch(cfg, seed=8100, bsz=4):
    return bert_ref.synthetic_batch(cfg, bsz, 128, seed, padded=True)


@gpu
@pytest.mark.parametrize("kind", ["fused", "packed", "eager"])
def test_zero_lr_leaves_the_master_on_every_path(cuda_dev, kind):
    """lr 0 (weight decay 0.01 too): the fp32 master is bitwise unchanged through capture and replays, while the
    momentum buffer keeps moving"""
    cfg, state = _tiny_run()
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.SGD(model.parameters(), lr=0.0, momentum=MOM, weight_decay=WD)
    args = _args(fused=kind != "eager", pack=kind == "packed")
    args.local_rank = 0
    tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)
    master0 = model._flat.detach().clone()
    prev = None
    bt = _batch(cfg)        # one batch: one packed shape, so the packed step is captured too
    for i in range(5):
        tr.train_step(bt)
        torch.cuda.synchronize()
        buf = opt._state()["momentum_buffer"].clone()
        assert torch.equal(model._flat, master0), "step %d moved the master at lr 0" % i
        assert prev is None or not torch.equal(buf, prev), "step %d left the momentum buffer" % i
        prev = buf
    if kind != "eager":
        held = tr._packed if kind == "packed" else {None: tr._fused}
        assert any(st.graph is not None for st in held.values())


@gpu
def test_fabric_call_trains_every_tensor(cuda_dev):
    """build_optimizer(optim="sgd") = fabric-cls.py's SGD(model.parameters(), lr): one default Trainer step moves every
    parameter's master"""
    cfg, state = _tiny_run()
    model = make_model(cfg, state, cuda_dev).train()
    args = _args(optim="sgd", learning_rate=0.05)
    args.local_rank = 0
    opt = b2.build_optimizer(model, args)
    tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)
    names = list(model._params_by_name)
    before = {n: v.detach().cpu().clone() for n, v in model.state_dict().items() if n in names}
    for i in range(3):
        tr.train_step(_batch(cfg, 8200 + i))
    torch.cuda.synchronize()
    after = {n: v.detach().cpu() for n, v in model.state_dict().items() if n in names}
    assert len(before) == len(names)
    still = [n for n in before if torch.equal(before[n], after[n])]
    assert not still, still
    assert opt.momentum_buffers() == {}


@gpu
@pytest.mark.parametrize("field,value", [("momentum", 0.8), ("dampening", 0.1), ("weight_decay", 0.02),
                                         ("nesterov", True), ("maximize", True)])
def test_captured_step_rejects_changed_hyperparameters(cuda_dev, field, value):
    cfg, state = _tiny_run()
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.SGD(model.parameters(), lr=1e-3, momentum=MOM, weight_decay=WD)
    bt = _batch(cfg)
    st = b2.FusedTrainStep(model, opt, 4, 128)
    for _ in range(4):
        st(bt)
    assert st.graph is not None
    opt.param_groups[0][field] = value
    with pytest.raises(RuntimeError, match=field):
        st(bt)


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
def test_gradscaler_skip_skips_the_update_and_the_schedule(cuda_dev):
    """Trainer use_amp: the poisoned step leaves master, buffer, step count and get_last_lr() as they were; the run
    lands where the run without that batch lands, with the same momentum buffer"""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    mult = [1.0, 0.5, 0.25, 0.125]
    batches = [_batch(cfg, 8700 + s) for s in range(3)]
    runs = []
    for bad in (None, 0, 1):
        model = make_model(cfg, state, cuda_dev).train()
        opt = b2.SGD(model.parameters(), lr=0.05, momentum=MOM, dampening=0.1, weight_decay=WD)
        sched = LambdaLR(opt, lambda s: mult[s])
        args = _args(fused=False, use_amp=True)
        args.local_rank = 0
        tr = b2.Trainer(args, cfg, model, _PoisonedLoss(-1 if bad is None else bad), opt, scheduler=sched)
        seq = [batches[0], batches[2]]
        if bad is not None:
            seq.insert(bad, batches[1])
        for i, bt in enumerate(seq):
            st = opt._state()
            before = (model._flat.detach().clone(), int(st["step"]), sched.get_last_lr(),
                      None if st["momentum_buffer"] is None else st["momentum_buffer"].clone())
            tr.train_step(bt)
            torch.cuda.synchronize()
            if i == bad:
                assert torch.equal(model._flat, before[0])
                assert int(opt._state()["step"]) == before[1] and sched.get_last_lr() == before[2]
                if before[3] is not None:
                    assert torch.equal(opt._state()["momentum_buffer"], before[3])
        runs.append((model._flat.detach().clone(), opt._state()["momentum_buffer"].clone()))
    for w, b in runs[1:]:
        assert float((w - runs[0][0]).abs().max()) <= 1e-6
        assert float((b - runs[0][1]).abs().max()) <= 1e-6


# ---- GPU: DDP world 2 -------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dma", ["0", "1"])
def test_ddp_world2_sgd(dma):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29597", os.path.join(ROOT, "tests", "ddp_sgd_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, B2_DDP_DMA=dma))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_sgd_worker: OK" in r.stdout, r.stdout[-3000:]
