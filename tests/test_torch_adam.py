"""torch's Adam and AdamW: the package's Adam / TorchAdamW on the fused update (b2_bucket_reduce_adam /
b2_adam_background).

Kernel level the update is bitwise torch.optim.Adam / AdamW(fused=True) on the GPU over the same fp32 gradient.  Model
level it is the oracle (bert_ref.loss_and_grads) plus torch.optim.AdamW on the fp32 oracle parameters, on every training
path: the weights within the bound of the update size and the first moments to the rel-L2 tolerances of
tests/parity.py, as for the package AdamW."""
import itertools
import os
import re
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.nn.functional as F
from torch.optim.lr_scheduler import LambdaLR

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


PAIRS = [(b2.Adam, torch.optim.Adam), (b2.TorchAdamW, torch.optim.AdamW)]
BAD = [dict(lr=-1e-3), dict(lr=float("nan")), dict(eps=-1e-8), dict(betas=(1.0, 0.999)), dict(betas=(-0.1, 0.999)),
       dict(betas=(0.9, 1.0)), dict(betas=(0.9, 0)), dict(betas=(1, 0.999)), dict(weight_decay=-0.01),
       dict(lr=torch.tensor([1e-3, 1e-3])), dict(lr=torch.tensor(1e-3), foreach=True), dict(fused=True, foreach=True),
       dict(fused=True, differentiable=True)]


@pytest.mark.parametrize("ours,theirs", PAIRS, ids=["Adam", "AdamW"])
@pytest.mark.parametrize("kw", BAD, ids=[str(i) for i in range(len(BAD))])
def test_constructor_errors_match_torch(ours, theirs, kw):
    with pytest.raises(Exception) as t:
        theirs([torch.nn.Parameter(torch.zeros(1))], **kw)
    with pytest.raises(Exception) as o:
        ours(_tiny_model().parameters(), **kw)
    assert type(o.value) is type(t.value) and str(o.value) == str(t.value)


@pytest.mark.parametrize("ours,theirs", PAIRS, ids=["Adam", "AdamW"])
def test_defaults_equal_torch(ours, theirs):
    t = theirs([torch.nn.Parameter(torch.zeros(1))]).defaults
    o = ours(_tiny_model().parameters()).defaults
    assert o == t
    assert ours(_tiny_model().parameters(), betas=(0.8, 0.99)).defaults["betas"] == (0.8, 0.99)


def test_signature_is_torch():
    import inspect
    for ours, theirs in PAIRS:
        a, b = inspect.signature(ours).parameters, inspect.signature(theirs).parameters
        assert [(p.name, p.default, p.kind) for p in a.values()] == [(p.name, p.default, p.kind) for p in b.values()]


def test_ignored_flags_tensor_lr_and_differentiable():
    model = _tiny_model()
    opt = b2.TorchAdamW(model.parameters(), foreach=True, capturable=True, fused=False)
    assert model._optimizer is opt and opt.param_groups[0]["decoupled_weight_decay"] is True
    opt = b2.Adam(_tiny_model().parameters(), fused=True, capturable=False)
    assert opt.param_groups[0]["decoupled_weight_decay"] is False
    opt = b2.TorchAdamW(_tiny_model().parameters(), lr=torch.tensor(2e-3))
    assert opt.current_lr() == pytest.approx(2e-3) and opt._hparams().lr == pytest.approx(2e-3)
    for cls in (b2.Adam, b2.TorchAdamW):
        with pytest.raises(ValueError, match="differentiable"):
            cls(_tiny_model().parameters(), differentiable=True)
        with pytest.raises(ValueError, match="Tensor betas"):
            cls(_tiny_model().parameters(), betas=(torch.tensor(0.9), torch.tensor(0.999)))
    assert b2.AdamW is not b2.TorchAdamW and not issubclass(b2.TorchAdamW, b2.AdamW)


def test_foreign_and_partial_parameters_are_rejected():
    for cls in (b2.Adam, b2.TorchAdamW):
        with pytest.raises(TypeError, match="ONE b200"):
            cls([torch.nn.Parameter(torch.zeros(8))], lr=0.1)
        a, b = _tiny_model(), _tiny_model()
        with pytest.raises(TypeError, match="ONE b200"):
            cls(list(a.parameters()) + list(b.parameters()), lr=0.1)
        with pytest.raises(ValueError, match="every parameter"):
            cls(list(a.parameters())[:-1], lr=0.1)


def test_group_rules():
    model = _tiny_model()
    named = list(model.named_parameters())
    dec = [p for n, p in named if "bias" not in n]
    nod = [p for n, p in named if "bias" in n]
    opt = b2.TorchAdamW([{"params": dec, "weight_decay": 0.01}, {"params": nod, "weight_decay": 0.0}], lr=0.1)
    assert opt._wd == 0.01 and opt._hparams().decoupled == 1 and opt._hparams().weight_decay == 0.01
    for kw in (dict(betas=(0.8, 0.999)), dict(eps=1e-6), dict(amsgrad=True), dict(maximize=True),
               dict(decoupled_weight_decay=False), dict(lr=0.2)):
        with pytest.raises(ValueError, match="differ only in weight_decay"):
            b2.TorchAdamW([{"params": dec}, dict(params=nod, **kw)], lr=0.1)
    with pytest.raises(ValueError, match="one non-zero weight_decay"):
        b2.Adam([{"params": dec, "weight_decay": 0.01}, {"params": nod, "weight_decay": 0.02}], lr=0.1)
    opt.param_groups[1]["lr"] = 0.05
    with pytest.raises(ValueError, match="different learning rates"):
        opt.step()


def test_captured_hparams_fields():
    opt = b2.Adam(_tiny_model().parameters(), betas=(0.8, 0.99), eps=1e-7, weight_decay=0.01, amsgrad=True,
                  maximize=True)
    assert opt.captured_hparams() == {"betas": ((0.8, 0.99),), "eps": (1e-7,), "weight_decay": (0.01,),
                                      "amsgrad": (True,), "maximize": (True,), "decoupled_weight_decay": (False,)}


def test_build_optimizer_adamw_torch():
    for name in ("adamw_torch", "adamw_torch_fused"):
        model = _tiny_model()
        opt = b2.build_optimizer(model, _args(optim=name, learning_rate=2e-5, weight_decay=0.01))
        assert type(opt) is b2.TorchAdamW
        assert [g["weight_decay"] for g in opt.param_groups] == [0.01, 0.0]
        names = {id(p): n for n, p in model.named_parameters()}
        nod = [names[id(p)] for p in opt.param_groups[1]["params"]]
        assert nod and all("bias" in n or "LayerNorm.weight" in n for n in nod)
        assert not any("bias" in names[id(p)] or "LayerNorm.weight" in names[id(p)]
                       for p in opt.param_groups[0]["params"])
        g = opt.param_groups[0]
        assert (g["lr"], g["betas"], g["eps"], g["amsgrad"], g["maximize"], g["decoupled_weight_decay"]) == \
            (2e-5, (0.9, 0.999), 1e-8, False, False, True)
    assert b2.Args.optim == "adamw"
    assert type(b2.build_optimizer(_tiny_model(), _args())) is b2.AdamW
    with pytest.raises(ValueError, match="optim"):
        b2.build_optimizer(_tiny_model(), _args(optim="adam"))


def test_abi():
    assert L.ABI_VERSION == 23 and L.load().b2_abi_version() == 23
    names = {"b2_bucket_reduce_adam", "b2_adam_prepare", "b2_adam_background"}
    assert names <= set(L._SIGNATURES) and names <= set(L.EXPORTED_SYMBOLS)
    assert [f for f, _t in L.AdamHParams._fields_] == ["lr", "beta1", "beta2", "eps", "weight_decay", "amsgrad",
                                                       "maximize", "decoupled", "grad_scale", "found_inf",
                                                       "clip_coef", "grad_f32", "lr_dev"]


def test_slim_adam_kernels_fit_beside_the_gemm():
    """ptxas: both slim TorchAdamRule instantiations (with and without amsgrad) at <= 32 registers with no spills, so
    the amsgrad update also takes the background form"""
    nvcc = "/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else "nvcc"
    src = os.path.join(ROOT, "pytorch-distributed-nlp_b200", "csrc", "optim.cu")
    with tempfile.TemporaryDirectory() as tmp:
        try:
            r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-Xptxas", "-v",
                                "-c", src, "-o", os.path.join(tmp, "optim.o")], capture_output=True, text=True)
        except FileNotFoundError:
            pytest.skip("nvcc not found")
    assert r.returncode == 0, r.stderr[-2000:]
    blocks = r.stderr.split("Compiling entry function")
    slim = [b for b in blocks if "slim_update_kernel" in b and "TorchAdamRule" in b]
    assert len(slim) == 2 and any("ILb1E" in b for b in slim), r.stderr[-2000:]
    for b in slim:
        regs = int(re.search(r"Used (\d+) registers", b).group(1))
        assert regs <= 32 and "0 bytes spill stores, 0 bytes spill loads" in b, b


# ---- GPU, kernel level: bitwise torch.optim.Adam / AdamW(fused=True) --------------------------------------------------
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
    """One flat state (master, decay flags, moments, amsgrad buffer, shadows, step count) stepped by one kernel form:
    'reduce1' / 'reduce2' (world 2: two gradient buffers on this device) / 'slim'."""

    def __init__(self, dev, kernel, lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False,
                 maximize=False, decoupled=True, seed=5):
        self.dev, self.kernel = dev, kernel
        self.world = 2 if kernel == "reduce2" else 1
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.decay = (torch.rand(N // 8, device=dev, generator=gen) < 0.5).to(torch.uint8)
        self.master = torch.randn(N, device=dev, generator=gen)
        self.master0 = self.master.clone()
        self.m, self.v = torch.zeros(N, device=dev), torch.zeros(N, device=dev)
        self.vmax = torch.zeros(N, device=dev) if amsgrad else None
        self.prepared = torch.zeros(2, device=dev)
        self.shadow = [torch.zeros(N, dtype=bf, device=dev) for _ in range(self.world)]
        self.step = torch.zeros(1, dtype=torch.int64, device=dev)
        self.hp = L.AdamHParams()
        self.hp.lr, self.hp.beta1, self.hp.beta2, self.hp.eps = lr, betas[0], betas[1], eps
        self.hp.weight_decay, self.hp.amsgrad, self.hp.maximize = weight_decay, int(amsgrad), int(maximize)
        self.hp.decoupled = int(decoupled)
        self.cfg = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad, maximize=maximize,
                        decoupled_weight_decay=decoupled)
        self.gen = gen

    def grads(self, scale=1.0):
        return [(torch.randn(N, device=self.dev, generator=self.gen) * 1e-1 * scale).to(bf) for _ in range(self.world)]

    def step_once(self, grads, **fields):
        """one update + b2_step_advance; fields: optional b2_adam_hparams_t pointers for this step only"""
        for k, v in fields.items():
            setattr(self.hp, k, v)
        if self.kernel == "slim":
            L.call("b2_adam_prepare", self.hp, self.step.data_ptr(), self.prepared.data_ptr(), _stream())
            L.call("b2_adam_background", grads[0].data_ptr(), self.shadow[0].data_ptr(), self.master.data_ptr(),
                   self.m.data_ptr(), self.v.data_ptr(), L.ptr(self.vmax), self.decay.data_ptr(), B0, E0, self.hp,
                   self.prepared.data_ptr(), _stream())
        else:
            L.call("b2_bucket_reduce_adam", L.ptr_array([g.data_ptr() for g in grads]),
                   L.ptr_array([s.data_ptr() for s in self.shadow]), self.world, 0, self.master.data_ptr(),
                   self.m.data_ptr(), self.v.data_ptr(), L.ptr(self.vmax), self.decay.data_ptr(), B0, E0, self.hp,
                   self.step.data_ptr(), _stream())
        L.call("b2_step_advance", self.step.data_ptr(), None, fields.get("found_inf"), _stream())
        for k in fields:
            setattr(self.hp, k, None)

    def state(self):
        torch.cuda.synchronize()
        out = [self.master.clone(), self.m.clone(), self.v.clone()] + [s.clone() for s in self.shadow]
        return out + ([self.vmax.clone()] if self.vmax is not None else [])


def _fp32_grad(grads):
    """the gradient the kernels form: rank-order fp32 sum from +0, times 1/world"""
    g = torch.zeros(N, device=grads[0].device)
    for x in grads:
        g = g + x.float()
    return g * (1.0 / len(grads))


class _Torch:
    """torch.optim.Adam on the same slice (`form`: fused=True, foreach=True or the for-loop): group 0 the decayed
    elements, group 1 the rest.  `tensors`: (flat begin, size) of decayed tensors torch steps as tensors of their own
    (sizes that are not multiples of 4 take torch's unaligned loop); the padding up to 8 after each is not compared."""

    def __init__(self, run, form="fused", tensors=()):
        own = torch.zeros(E0 - B0, dtype=torch.bool, device=run.dev)
        self.tensors = [(b - B0, n) for (b, n) in tensors]
        for b, n in self.tensors:
            own[b:b + (n + 7) // 8 * 8] = True
        dec = run.decay.repeat_interleave(8)[B0:E0] != 0
        self.mask, self.rest = dec & ~own, ~dec & ~own
        self.covered = ~own
        for b, n in self.tensors:
            self.covered[b:b + n] = True
        w = run.master0[B0:E0]
        self.p = [torch.nn.Parameter(w[self.mask].clone())] + \
            [torch.nn.Parameter(w[b:b + n].clone()) for b, n in self.tensors] + [torch.nn.Parameter(w[self.rest].clone())]
        c = dict(run.cfg)
        wd = c.pop("weight_decay")
        kw = {"fused": dict(fused=True), "foreach": dict(foreach=True), "single": dict(foreach=False)}[form]
        self.opt = torch.optim.Adam([{"params": self.p[:-1], "weight_decay": wd},
                                     {"params": self.p[-1:], "weight_decay": 0.0}], **kw, **c)

    def step(self, g):
        g = g[B0:E0]
        self.p[0].grad, self.p[-1].grad = g[self.mask].clone(), g[self.rest].clone()
        for (b, n), q in zip(self.tensors, self.p[1:-1]):
            q.grad = g[b:b + n].clone()
        self.opt.step()

    def flat(self, parts):
        out = torch.full((E0 - B0,), float("nan"), device=parts[0].device)
        out[self.mask], out[self.rest] = parts[0], parts[-1]
        for (b, n), x in zip(self.tensors, parts[1:-1]):
            out[b:b + n] = x
        return out

    def master(self):
        return self.flat([p.detach() for p in self.p])

    def buf(self, key):
        return self.flat([self.opt.state[p][key] for p in self.p])


def _check_against_torch(run, ref):
    st = run.state()
    master = st[0]
    c = ref.covered
    _same(master[B0:E0][c], ref.master()[c], "master")
    _same(master[:B0], run.master0[:B0], "master before the slice")
    _same(master[E0:], run.master0[E0:], "master after the slice")
    _same(st[1][B0:E0][c], ref.buf("exp_avg")[c], "exp_avg")
    _same(st[2][B0:E0][c], ref.buf("exp_avg_sq")[c], "exp_avg_sq")
    for s in st[3:3 + run.world]:
        _same(s[B0:E0], master[B0:E0].to(bf), "shadow")
    if run.vmax is not None:
        _same(st[-1][B0:E0][c], ref.buf("max_exp_avg_sq")[c], "max_exp_avg_sq")
    steps = {float(ref.opt.state[p]["step"]) for p in ref.p}
    assert steps == {float(run.step)}, (steps, int(run.step))


def _combos():
    for ams, mx, dec, wd, (betas, eps) in itertools.product(
            [False, True], [False, True], [True, False], [0.0, 1e-2], [((0.9, 0.999), 1e-8), ((0.8, 0.95), 1e-6)]):
        yield dict(amsgrad=ams, maximize=mx, decoupled=dec, weight_decay=wd, betas=betas, eps=eps)


COMBOS = list(_combos())
KERNELS = ["reduce1", "reduce2", "slim"]
STEPS_K = 6


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("cfg", COMBOS, ids=lambda c: "ams%d-max%d-dec%d-wd%g-b%g-%g-eps%g" % (
    c["amsgrad"], c["maximize"], c["decoupled"], c["weight_decay"], c["betas"][0], c["betas"][1], c["eps"]))
def test_kernel_is_torch_fused_adam_bitwise(cuda_dev, kernel, cfg):
    """6 steps (the bias correction moves) on a random flat state with random decay flags: master, moments, amsgrad
    buffer, shadow and step count bitwise torch's fused Adam / AdamW"""
    run = _Run(cuda_dev, kernel, **cfg)
    ref = _Torch(run)
    for _ in range(STEPS_K):
        grads = run.grads()
        run.step_once(grads)
        ref.step(_fp32_grad(grads))
    _check_against_torch(run, ref)


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("maximize", [False, True])
@pytest.mark.parametrize("decoupled", [True, False])
@pytest.mark.parametrize("amsgrad", [False, True])
def test_within_torchs_own_spread_of_foreach_and_for_loop(cuda_dev, kernel, amsgrad, decoupled, maximize):
    """against torch's foreach and for-loop forms the difference per element is at most twice what those forms show
    against torch's fused form on the same inputs"""
    cfg = dict(amsgrad=amsgrad, weight_decay=1e-2, decoupled=decoupled, maximize=maximize)
    run = _Run(cuda_dev, kernel, **cfg)
    refs = {f: _Torch(run, f) for f in ("fused", "foreach", "single")}
    for _ in range(STEPS_K):
        grads = run.grads()
        run.step_once(grads)
        g = _fp32_grad(grads)
        for r in refs.values():
            r.step(g)
    ours = run.state()[0][B0:E0]
    fused = refs["fused"].master()
    for form in ("foreach", "single"):
        theirs = refs[form].master()
        assert float((ours - theirs).abs().max()) <= 2 * float((theirs - fused).abs().max()), form


# tensors torch steps through its unaligned loop: sizes that are not multiples of 4, one past 1024 elements so that
# it spans three of that loop's lanes (element j is in lane (j % 2048) / 512)
UNALIGNED = [(8 * 61, 6), (8 * 200, 1030)]


def _mark_unaligned(run, tensors):
    """the decay flags optim.Adam gives these tensors' vectors (decayed)"""
    for b, n in tensors:
        j = torch.arange(0, n, 8, device=run.dev)
        run.decay[b // 8:b // 8 + len(j)] = (1 + L.ADAM_DECAY_UNALIGNED + L.ADAM_DECAY_LANE0 * ((j % 2048) < 512)).to(
            torch.uint8)


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("maximize", [False, True])
@pytest.mark.parametrize("amsgrad", [False, True])
def test_unaligned_tensors_are_torch_fused_bitwise(cuda_dev, kernel, amsgrad, maximize):
    """Adam's L2 term in tensors whose size is not a multiple of 4, beside the aligned ones"""
    run = _Run(cuda_dev, kernel, weight_decay=1e-2, decoupled=False, amsgrad=amsgrad, maximize=maximize)
    _mark_unaligned(run, UNALIGNED)
    ref = _Torch(run, tensors=UNALIGNED)
    for _ in range(STEPS_K):
        grads = run.grads()
        run.step_once(grads)
        ref.step(_fp32_grad(grads))
    _check_against_torch(run, ref)


@gpu
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("cfg", [dict(decoupled=False), dict(decoupled=False, maximize=True),
                                 dict(decoupled=False, amsgrad=True), dict(decoupled=True)],
                         ids=["adam", "adam-max", "adam-ams", "adamw"])
def test_grad_scale_is_torch_fused_with_a_grad_scaler_bitwise(cuda_dev, world, cfg):
    """a GradScaler scale against torch's fused Adam handed the same grad_scale (its kernel unscales, and forms the L2
    term as one fma then)"""
    run = _Run(cuda_dev, "reduce%d" % world, weight_decay=1e-2, **cfg)
    _mark_unaligned(run, UNALIGNED)
    ref = _Torch(run, tensors=UNALIGNED)
    scale = torch.tensor(1024.0, device=cuda_dev)
    ref.opt.grad_scale, ref.opt.found_inf = scale, torch.zeros((), device=cuda_dev)
    for _ in range(STEPS_K):
        grads = run.grads(scale=1024.0)       # a power of two: exact in bf16 and in the unscale
        run.step_once(grads, grad_scale=scale.data_ptr())
        ref.step(_fp32_grad(grads))
    _check_against_torch(run, ref)


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("lr", [1e-2, 1.7e-4, 0.0])
def test_device_lr_is_the_by_value_lr(cuda_dev, kernel, lr):
    """lr_dev holding x gives bitwise the run with x by value (hp.lr is a decoy then)"""
    cfg = dict(weight_decay=1e-2, amsgrad=True)
    a, b = _Run(cuda_dev, kernel, lr=lr, **cfg), _Run(cuda_dev, kernel, lr=0.37, **cfg)
    lr_t = torch.tensor([lr], dtype=torch.float64, device=cuda_dev)
    for _ in range(3):
        a.step_once(a.grads())
        b.step_once(b.grads(), lr_dev=lr_t.data_ptr())
    for x, y in zip(a.state(), b.state()):
        _same(y, x, "lr_dev")
    if lr == 0.0:
        _same(a.master, a.master0, "master at lr 0")


@gpu
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("decoupled", [True, False])
def test_clip_coef_is_torch_on_the_clipped_gradient(cuda_dev, kernel, decoupled):
    run = _Run(cuda_dev, kernel, weight_decay=1e-2, amsgrad=True, decoupled=decoupled)
    ref = _Torch(run)
    coef = torch.tensor(0.3, device=cuda_dev)
    for _ in range(5):
        grads = run.grads()
        run.step_once(grads, clip_coef=coef.data_ptr())
        ref.step(_fp32_grad(grads) * coef)
    _check_against_torch(run, ref)


@gpu
@pytest.mark.parametrize("world", [1, 2])
def test_grad_f32_equals_the_peer_read(cuda_dev, world):
    kernel = "reduce%d" % world
    cfg = dict(weight_decay=1e-2, amsgrad=True)
    a, b = _Run(cuda_dev, kernel, **cfg), _Run(cuda_dev, kernel, **cfg)
    coef = torch.tensor(0.3, device=cuda_dev)
    for _ in range(3):
        ga, gb = a.grads(), b.grads()
        a.step_once(ga, clip_coef=coef.data_ptr())
        stash = _fp32_grad(gb)[B0:E0].contiguous()
        b.step_once(gb, grad_f32=stash.data_ptr(), clip_coef=coef.data_ptr())
    for x, y in zip(a.state(), b.state()):
        _same(y, x, "grad_f32")


@gpu
@pytest.mark.parametrize("world", [1, 2])
def test_grad_scale_unscales(cuda_dev, world):
    kernel = "reduce%d" % world
    cfg = dict(weight_decay=1e-2)
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
def test_found_inf_skips_everything(cuda_dev, world):
    """a skipped step leaves master, moments, amsgrad buffer, shadow and the step count; the run then goes on as
    torch's from the state it had"""
    kernel = "reduce%d" % world
    run = _Run(cuda_dev, kernel, weight_decay=1e-2, amsgrad=True)
    ref = _Torch(run)
    for _ in range(2):
        grads = run.grads()
        run.step_once(grads)
        ref.step(_fp32_grad(grads))
    before = run.state()
    inf = torch.tensor(1.0, device=cuda_dev)
    run.step_once(run.grads(), found_inf=inf.data_ptr())
    for x, y in zip(run.state(), before):
        _same(x, y, "skipped step")
    assert int(run.step) == 2
    for _ in range(3):
        grads = run.grads()
        run.step_once(grads)
        ref.step(_fp32_grad(grads))
    _check_against_torch(run, ref)


@gpu
def test_amsgrad_buffer_pointer_matches_the_flag(cuda_dev):
    run = _Run(cuda_dev, "reduce1", amsgrad=False)
    g = run.grads()
    run.vmax = torch.zeros(N, device=cuda_dev)
    with pytest.raises(RuntimeError, match="max_exp_avg_sq"):
        run.step_once(g)
    run = _Run(cuda_dev, "slim", amsgrad=True)
    run.vmax = None
    with pytest.raises(RuntimeError, match="max_exp_avg_sq"):
        run.step_once(g)


# ---- GPU, model level: the oracle + torch AdamW ---------------------------------------------------------------------
STEPS, LR, WD = 4, 3e-5, 0.01
_CACHE = {}


def _warmup(s):
    return (s + 1) / STEPS          # linear warmup over the run


# How far STEPS Adam steps can move a weight: each step moves it by at most lr * |m_hat| / sqrt(v_hat) (+ lr * wd * |w|
# for AdamW), and by Cauchy-Schwarz |m_hat| / sqrt(v_hat) <= sqrt(sum_i a_i^2 / c_i) with a_i, c_i the bias-corrected
# EMA weights of the two moments: 1.007 at t = 4 for betas (0.9, 0.999).  So |delta| <= 1.03 x the summed lr here.
SUM_LR = LR * sum(_warmup(s) for s in range(STEPS))
MAX_MOVE = 1.03 * SUM_LR + 1e-6


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


def _no_decay(n):
    return "bias" in n or "LayerNorm.weight" in n


def _groups(named, wd=WD):
    named = list(named)
    return [{"params": [p for n, p in named if not _no_decay(n)], "weight_decay": wd},
            {"params": [p for n, p in named if _no_decay(n)], "weight_decay": 0.0}]


def _oracle(size, k, clip, variant="adamw"):
    """STEPS torch AdamW (or `variant`) steps with the linear warmup on the fp32 oracle, the reference's two groups; a
    step's gradient is the mean over its k micro-batches, clipped (torch.nn.utils.clip_grad_norm_) to a quarter of the
    first step's norm"""
    key = (size, k, clip, variant)
    if key not in _CACHE:
        if size not in _CACHE:
            _CACHE[size] = _base(size)
        cfg, state, bsz, odev = _CACHE[size]
        batches = [[bert_ref.synthetic_batch(cfg, bsz, 128, 8900 + 10 * s + j, padded=True) for j in range(k)]
                   for s in range(STEPS)]
        ref = {n: torch.nn.Parameter(v.to(odev).clone()) for n, v in state.items()}
        opt = _VARIANTS[variant][0](_groups(ref.items()), lr=LR, foreach=False)
        sched = LambdaLR(opt, _warmup)
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
        w = {n: p.detach().cpu() for n, p in ref.items()}
        m = {n: opt.state[p]["exp_avg"].cpu() for n, p in ref.items()}
        _CACHE[key] = (cfg, state, batches, max_norm, w, m)
    return _CACHE[key]


_VARIANTS = {
    "adamw": (torch.optim.AdamW, b2.TorchAdamW),
    "adam_coupled": (lambda groups, **kw: torch.optim.Adam(groups, **kw), b2.Adam),
    "adamw_amsgrad": (lambda groups, **kw: torch.optim.AdamW(groups, amsgrad=True, **kw),
                      lambda groups, **kw: b2.TorchAdamW(groups, amsgrad=True, **kw)),
}


def _loop_step(model, opt, d, max_norm):
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    if max_norm is not None:
        b2.clip_grad_norm_(model.parameters(), max_norm)
    opt.step()


def _train(cuda_dev, size, mode, clip, variant="adamw"):
    k = 2 if mode == "k2" else 1
    cfg, state, batches, max_norm, rw, rm = _oracle(size, k, clip, variant)
    model = make_model(cfg, state, cuda_dev).train()
    opt = _VARIANTS[variant][1](_groups(model.named_parameters()), lr=LR)
    sched = LambdaLR(opt, _warmup)
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
    for n, v in rw.items():
        assert float((w[n] - state[n]).abs().max()) <= MAX_MOVE, n          # a step-size error shows here
        assert float((w[n] - v).abs().max()) <= 2 * MAX_MOVE, n
    m = {n: ea.detach().cpu() for n, (ea, _v) in opt.moments().items()}
    assert_grads_within_tolerance(m, rm, qk_tol=TOL_GRAD_REL_QK)
    moved = [n for n in rw if not torch.equal(w[n], state[n])]
    assert len(moved) == len(rw)
    return opt


MODES = ["loop", "eager", "fused", "packed", "amp", "k2"]


@gpu
@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("size", ["tiny", "configA"])
def test_torch_adamw_matches_oracle(cuda_dev, size, mode, clip):
    """4 steps of TorchAdamW on the reference's groups with a linear warmup, dropout off: weights and first moments
    against torch AdamW on the oracle"""
    _train(cuda_dev, size, mode, clip)
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("variant", ["adam_coupled", "adamw_amsgrad"])
def test_adam_variants_match_oracle(cuda_dev, variant):
    """Adam(weight_decay=0.01) (coupled) and TorchAdamW(amsgrad=True) on the captured step"""
    opt = _train(cuda_dev, "tiny", "fused", False, variant)
    assert (opt.max_exp_avg_sqs() != {}) == (variant == "adamw_amsgrad")


def _tiny_run():
    cfg = tiny_config()
    return cfg, state_from_hf_init(cfg)


def _batch(cfg, seed=8100, bsz=4):
    return bert_ref.synthetic_batch(cfg, bsz, 128, seed, padded=True)


@gpu
@pytest.mark.parametrize("amsgrad", [False, True])
@pytest.mark.parametrize("kind", ["fused", "packed", "eager", "amp", "k2"])
def test_zero_lr_leaves_the_master_on_every_path(cuda_dev, kind, amsgrad):
    """lr 0 (weight decay 0.01 too): the fp32 master is bitwise unchanged through capture and replays, while the
    moments keep moving"""
    cfg, state = _tiny_run()
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.TorchAdamW(_groups(model.named_parameters()), lr=0.0, amsgrad=amsgrad)
    k = 2 if kind == "k2" else 1
    args = _args(fused=kind in ("fused", "packed", "k2"), pack=kind == "packed", use_amp=kind == "amp",
                 gradient_accumulation_steps=k)
    args.local_rank = 0
    tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)
    master0 = model._flat.detach().clone()
    prev = None
    bt = _batch(cfg)        # one batch: one packed shape, so the packed step is captured too
    for i in range(5 * k):
        tr.train_step(bt)
        torch.cuda.synchronize()
        assert torch.equal(model._flat, master0), "step %d moved the master at lr 0" % i
        m = opt._state()["exp_avg"].clone()
        if (i + 1) % k == 0:
            assert prev is None or not torch.equal(m, prev), "step %d left the moments" % i
            prev = m
    if kind in ("fused", "packed"):
        held = tr._packed if kind == "packed" else {None: tr._fused}
        assert any(st.graph is not None for st in held.values())


@gpu
@pytest.mark.parametrize("field,value", [("betas", (0.8, 0.999)), ("eps", 1e-6), ("weight_decay", 0.02),
                                         ("amsgrad", True), ("maximize", True), ("decoupled_weight_decay", False)])
def test_captured_step_rejects_changed_hyperparameters(cuda_dev, field, value):
    cfg, state = _tiny_run()
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.TorchAdamW(model.parameters(), lr=1e-3)
    bt = _batch(cfg)
    st = b2.FusedTrainStep(model, opt, 4, 128)
    for _ in range(4):
        st(bt)
    assert st.graph is not None
    opt.param_groups[0][field] = value
    with pytest.raises(RuntimeError, match=field):
        st(bt)


@gpu
def test_amsgrad_turned_on_before_the_first_update_is_torchs(cuda_dev):
    """amsgrad set after the state exists (moments() read) but before any update: the buffer comes with that update,
    and the run equals one built with amsgrad=True"""
    cfg, state = _tiny_run()
    runs = []
    for late in (False, True):
        model = make_model(cfg, state, cuda_dev).train()
        opt = b2.TorchAdamW(model.parameters(), lr=1e-3, amsgrad=not late)
        opt.moments()
        if late:
            assert opt.max_exp_avg_sqs() == {}
            opt.param_groups[0]["amsgrad"] = True
        for i in range(2):
            _loop_step(model, opt, to_dev(_batch(cfg, 8300 + i), cuda_dev), None)
        torch.cuda.synchronize()
        runs.append((model._flat.detach().clone(), opt._state()["max_exp_avg_sq"].clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


@gpu
def test_amsgrad_turned_on_after_the_first_step_raises(cuda_dev):
    cfg, state = _tiny_run()
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.TorchAdamW(model.parameters(), lr=1e-3)
    d = to_dev(_batch(cfg), cuda_dev)
    _loop_step(model, opt, d, None)
    assert opt.max_exp_avg_sqs() == {}
    opt.param_groups[0]["amsgrad"] = True
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    w0 = model._flat.detach().clone()
    with pytest.raises(ValueError, match="amsgrad"):
        opt.step()
    torch.cuda.synchronize()
    assert torch.equal(model._flat, w0)


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
    """Trainer use_amp: the poisoned step leaves master, moments, amsgrad buffer, step count and get_last_lr() as they
    were; the run lands where the run without that batch lands"""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    mult = [1.0, 0.5, 0.25, 0.125]
    batches = [_batch(cfg, 8700 + s) for s in range(3)]
    runs = []
    for bad in (None, 0, 1):
        model = make_model(cfg, state, cuda_dev).train()
        opt = b2.TorchAdamW(_groups(model.named_parameters()), lr=1e-3, amsgrad=True)
        sched = LambdaLR(opt, lambda s: mult[s])
        args = _args(fused=False, use_amp=True)
        args.local_rank = 0
        tr = b2.Trainer(args, cfg, model, _PoisonedLoss(-1 if bad is None else bad), opt, scheduler=sched)
        seq = [batches[0], batches[2]]
        if bad is not None:
            seq.insert(bad, batches[1])
        for i, bt in enumerate(seq):
            st = opt._state()
            before = (model._flat.detach().clone(), int(st["step"]), sched.get_last_lr(), st["exp_avg"].clone(),
                      st["exp_avg_sq"].clone(), st["max_exp_avg_sq"].clone())
            tr.train_step(bt)
            torch.cuda.synchronize()
            if i == bad:
                st = opt._state()
                assert torch.equal(model._flat, before[0])
                assert int(st["step"]) == before[1] and sched.get_last_lr() == before[2]
                for key, was in zip(("exp_avg", "exp_avg_sq", "max_exp_avg_sq"), before[3:]):
                    assert torch.equal(st[key], was), key
        st = opt._state()
        runs.append((model._flat.detach().clone(), st["exp_avg"].clone()))
    for w, m in runs[1:]:
        assert float((w - runs[0][0]).abs().max()) <= 1e-6
        assert float((m - runs[0][1]).abs().max()) <= 1e-6


# ---- GPU: DDP world 2 -------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dma", ["0", "1"])
def test_ddp_world2_torch_adamw(dma):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29598", os.path.join(ROOT, "tests", "ddp_adam_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, B2_DDP_DMA=dma))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_adam_worker: OK" in r.stdout, r.stdout[-3000:]
