"""Losses: HF's three problem types (regression, single- and multi-label classification) and torch's weighted and
label-smoothed cross-entropy, on the device loss kernel (b2_loss_fwd_bwd) and on every training path.

CPU: the reference losses against the installed HF model, the problem-type rule, label checks, the criterion mapping
of the captured steps and the loss kernel's register use.  GPU: the kernel against torch in float64, its degenerate
batches and graph replays, the default path bit for bit, and 4 optimizer steps of each loss against the oracle on the
eager, captured, packed, accumulating and clipped paths."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from loss_ref import criterion_loss, hf_loss, labelled_batch, loss_and_grads
from parity import (TOL_GRAD_REL_QK, TOL_TRAJ, adamw_ref, assert_grads_within_tolerance, b2, make_model,
                    state_from_hf_init, tiny_config, to_dev)
from oracle import cpu_step
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.losses import criterion_key
from pytorch_distributed_nlp_b200.trainer import step_loss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu
LR = 3e-5
NO_DROP = dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


# ---- CPU: the reference losses against HF ------------------------------------------------------------------------------
@pytest.mark.parametrize("problem_type,C,kind", [(None, 1, "regression"), ("regression", 3, "regression"),
                                                 (None, 4, "multi"), (None, 6, "single")])
def test_reference_losses_equal_hf(problem_type, C, kind):
    """the oracle's logits under loss_ref.hf_loss == HF BertForSequenceClassification(problem_type) (eager attention):
    loss, logits and every parameter gradient"""
    pytest.importorskip("transformers")
    cfg = tiny_config(num_labels=C, **NO_DROP)
    hf = cpu_step.build_hf_model(cfg, seed=123)
    hf.config.problem_type = problem_type
    state = {k: v.detach().clone() for k, v in hf.named_parameters()}
    b = labelled_batch(cfg, 4, 128, 1100, kind)
    out = hf(input_ids=b["input_ids"], token_type_ids=b["token_type_ids"], attention_mask=b["attention_mask"],
             labels=b["label"])
    out.loss.backward()
    pt = hf.config.problem_type
    assert pt == (problem_type or b2.infer_problem_type(C, b["label"]))
    loss, logits, grads = loss_and_grads(state, cfg, b, lambda z, y: hf_loss(z, y, pt, C))
    assert abs(float(out.loss.detach()) - float(loss)) < 1e-6
    assert float((out.logits.detach() - logits).abs().max()) < 1e-6
    for k, p in hf.named_parameters():
        assert float((grads[k] - p.grad).abs().max()) < 1e-6 + 1e-5 * float(p.grad.abs().max()), k


# ---- CPU: host logic ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,dtype,want", [
    (1, torch.float32, "regression"), (1, torch.int64, "regression"), (6, torch.int64, "single_label_classification"),
    (6, torch.int32, "single_label_classification"), (6, torch.float32, "multi_label_classification"),
    (6, torch.float64, "multi_label_classification"), (2, torch.int16, "multi_label_classification")])
def test_problem_type_inference(C, dtype, want):
    assert b2.infer_problem_type(C, torch.zeros(3, dtype=dtype)) == want


def test_config_problem_type():
    assert b2.BertConfig(num_labels=3).problem_type is None
    assert b2.BertConfig(num_labels=3, problem_type="regression").problem_type == "regression"
    with pytest.raises(ValueError, match="problem_type"):
        b2.BertConfig(problem_type="ordinal")


def test_step_loss_follows_the_problem_type():
    """with no criterion the captured steps use the config's problem type; unset, one label is regression and more
    are single-label (int64 labels, as before)"""
    for C, pt, mode in [(1, None, L.LOSS_MSE), (6, None, L.LOSS_CE), (3, "regression", L.LOSS_MSE),
                        (4, "multi_label_classification", L.LOSS_BCE)]:
        model = b2.BertForSequenceClassification(tiny_config(num_labels=C, problem_type=pt))
        fn = step_loss(model, None)
        assert fn.mode == mode
        assert fn.plain_ce == (mode == L.LOSS_CE)


def test_label_checks():
    ce, mse1, mse3, bce = (b2.Loss(L.LOSS_CE, 6), b2.Loss(L.LOSS_MSE, 1), b2.Loss(L.LOSS_MSE, 3),
                           b2.Loss(L.LOSS_BCE, 3))
    ce.check_labels(torch.zeros(4, dtype=torch.int64), 4)
    with pytest.raises(TypeError, match="int64"):
        ce.check_labels(torch.zeros(4), 4)
    with pytest.raises(TypeError, match="int64"):
        ce.check_labels(torch.zeros(4, dtype=torch.int32), 4)
    with pytest.raises(ValueError, match=r"\[batch\]"):
        ce.check_labels(torch.zeros(5, dtype=torch.int64), 4)
    for shape in [(4,), (4, 1)]:
        mse1.check_labels(torch.zeros(shape), 4)
    mse1.check_labels(torch.zeros(()), 1)
    mse1.check_labels(torch.zeros(1, dtype=torch.float64), 1)
    for bad in [(4, 2), (5,), (1, 4)]:
        with pytest.raises(ValueError):
            mse1.check_labels(torch.zeros(bad), 4)
    with pytest.raises(TypeError, match="floating"):
        mse1.check_labels(torch.zeros(4, dtype=torch.int64), 4)
    for fn in (mse3, bce):
        fn.check_labels(torch.zeros(4, 3), 4)
        for bad in [(4,), (4, 1), (3, 4), (4, 3, 1)]:
            with pytest.raises(ValueError):
                fn.check_labels(torch.zeros(bad), 4)
        with pytest.raises(TypeError, match="floating"):
            fn.check_labels(torch.zeros(4, 3, dtype=torch.int64), 4)
    assert mse1.label_shape(4) == (4,) and mse3.label_shape(4) == (4, 3) and ce.label_shape(4) == (4,)
    assert bce.device_labels(torch.ones(2, 3, dtype=torch.float64), 2).dtype == torch.float32


class _MyCE(nn.CrossEntropyLoss):
    pass


W6 = torch.tensor([0.2, 1.0, 3.0, 0.5, 2.0, 1.0])


@pytest.mark.parametrize("make,mode,plain,opts", [
    (lambda: nn.CrossEntropyLoss(), L.LOSS_CE, True, dict(ignore_index=-100, label_smoothing=0.0)),
    (lambda: nn.CrossEntropyLoss(weight=W6), L.LOSS_CE, False, dict(weight=W6)),
    (lambda: nn.CrossEntropyLoss(ignore_index=3), L.LOSS_CE, False, dict(ignore_index=3)),
    (lambda: nn.CrossEntropyLoss(label_smoothing=0.1), L.LOSS_CE, False, dict(label_smoothing=0.1)),
    (lambda: nn.CrossEntropyLoss(weight=W6, ignore_index=0, label_smoothing=0.2), L.LOSS_CE, False,
     dict(weight=W6, ignore_index=0, label_smoothing=0.2)),
    (lambda: nn.MSELoss(), L.LOSS_MSE, False, {}),
    (lambda: nn.BCEWithLogitsLoss(), L.LOSS_BCE, False, dict(pos_weight=None)),
    (lambda: nn.BCEWithLogitsLoss(pos_weight=W6), L.LOSS_BCE, False, dict(pos_weight=W6)),
])
def test_criterion_mapping_accepts(make, mode, plain, opts):
    fn = b2.loss_from_criterion(make(), 6, "cpu")
    assert fn.mode == mode and fn.plain_ce == plain
    for k, v in opts.items():
        got = getattr(fn, k)
        if isinstance(v, torch.Tensor):
            assert torch.equal(got, v) and got is not v     # copied once, at build
        else:
            assert got == pytest.approx(v) if isinstance(v, float) else got == v


@pytest.mark.parametrize("make", [
    lambda: _MyCE(), lambda: nn.CrossEntropyLoss(reduction="sum"), lambda: nn.CrossEntropyLoss(reduction="none"),
    lambda: nn.MSELoss(reduction="sum"), lambda: nn.BCEWithLogitsLoss(weight=W6),
    lambda: nn.BCEWithLogitsLoss(reduction="sum"), lambda: nn.NLLLoss(), lambda: nn.L1Loss(),
    lambda: (lambda logits, label: F.cross_entropy(logits, label)),
])
def test_criterion_mapping_rejects(make):
    with pytest.raises(ValueError, match=r"args\.fused = False") as e:
        b2.loss_from_criterion(make(), 6, "cpu")
    assert "CrossEntropyLoss" in str(e.value) and "BCEWithLogitsLoss" in str(e.value)


def test_criterion_weight_shapes_and_key():
    with pytest.raises(ValueError, match="shape"):
        b2.loss_from_criterion(nn.CrossEntropyLoss(weight=torch.ones(5)), 6, "cpu")
    with pytest.raises(ValueError, match="shape"):
        b2.loss_from_criterion(nn.BCEWithLogitsLoss(pos_weight=torch.ones(1)), 6, "cpu")
    c = nn.CrossEntropyLoss(weight=W6.clone())
    k0 = criterion_key(c)
    assert criterion_key(c) == k0
    c.weight.mul_(2.0)                       # in place: the cached captured step must rebuild
    assert criterion_key(c) != k0
    k1 = criterion_key(c)
    c.label_smoothing = 0.1
    assert criterion_key(c) != k1


def test_loss_kernel_does_not_spill():
    """every instantiation of the loss kernel fits its registers (ptxas -v: 0 spill bytes)"""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) and shutil.which(nvcc) is None:
        pytest.skip("no nvcc")
    src = os.path.join(ROOT, "pytorch-distributed-nlp_b200", "csrc", "head.cu")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-Xptxas", "-v",
                            "-c", src, "-o", os.path.join(d, "head.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    found = re.findall(r"Function properties for (\S*loss_fwd_bwd_kernel\S*)\n\s*(.*)", r.stderr)
    assert len(found) == 4, r.stderr[-3000:]
    for name, props in found:
        assert "0 bytes spill stores, 0 bytes spill loads" in props, (name, props)


# ---- GPU: the kernel against torch in float64 ---------------------------------------------------------------------------
_KERNEL_CASES = ["ce", "ce_w", "ce_ls", "ce_w_ls", "ce_ignore", "mse", "bce", "bce_pw"]


def _kernel_case(case, B, C, dev, seed=0):
    """(losses.Loss, torch float64 reference loss function, logits fp32, labels)"""
    g = torch.Generator().manual_seed(seed + 1000 * B + C)
    logits = (3 * torch.randn(B, C, generator=g)).to(dev)
    w = (0.1 + 2.9 * torch.rand(C, generator=g)).to(dev)
    if case.startswith("ce"):
        y = torch.randint(0, C, (B,), generator=g)
        kw = {}
        if "_w" in case or case == "ce_ignore":
            kw["weight"] = w
        if "ls" in case or case == "ce_ignore":
            kw["label_smoothing"] = 0.1 if case != "ce_ignore" else 0.2
        if case == "ce_ignore":
            kw["ignore_index"] = 1
            y[1::3] = 1
        y = y.to(dev)
        fn = b2.Loss(L.LOSS_CE, C, dev, **kw)
        ref = lambda z: F.cross_entropy(z, y, **{k: (v.double() if torch.is_tensor(v) else v)  # noqa: E731
                                                 for k, v in kw.items()})
        return fn, ref, logits, y
    if case == "mse":
        y = torch.randn((B,) if C == 1 else (B, C), generator=g).to(dev)
        ref = lambda z: F.mse_loss(z.reshape(y.shape), y.double())  # noqa: E731
        return b2.Loss(L.LOSS_MSE, C, dev), ref, logits, y
    y = (torch.rand(B, C, generator=g) < 0.3).float().to(dev)
    pw = w if case == "bce_pw" else None
    ref = lambda z: F.binary_cross_entropy_with_logits(  # noqa: E731
        z, y.double(), pos_weight=None if pw is None else pw.double())
    return b2.Loss(L.LOSS_BCE, C, dev, pos_weight=pw), ref, logits, y


def _launch(fn, logits, labels, loss, dl):
    B = logits.shape[0]
    fn.launch(logits.data_ptr(), fn.device_labels(labels, B), B, loss.data_ptr(), None if dl is None else dl.data_ptr(),
              torch.cuda.current_stream().cuda_stream)


@gpu
@pytest.mark.parametrize("C", [1, 2, 6, 35])
@pytest.mark.parametrize("B", [1, 7, 32, 300])
@pytest.mark.parametrize("case", _KERNEL_CASES)
def test_loss_kernel_matches_torch_float64(cuda_dev, case, B, C):
    fn, ref, logits, y = _kernel_case(case, B, C, cuda_dev)
    loss = torch.empty((), device=cuda_dev)
    dl = torch.full_like(logits, float("nan"))
    _launch(fn, logits, y, loss, dl)
    z = logits.double().requires_grad_(True)
    r = ref(z)
    r.backward()
    torch.cuda.synchronize()
    rl, rg = float(r), z.grad
    if not np.isfinite(rl):          # every row ignored: nan, as torch (B = 1 and the row is label 1)
        assert torch.isnan(loss) and torch.equal(dl, torch.zeros_like(dl))
        return
    assert abs(float(loss) - rl) <= 5e-5 * abs(rl) + 1e-6, (float(loss), rl)
    err = (dl.double() - rg).abs()
    bound = 1e-4 * rg.abs() + 1e-6 * float(rg.abs().max()) + 1e-12
    assert bool((err <= bound).all()), float((err / bound).max())
    # a forward without dlogits gives the same loss bits
    loss2 = torch.empty((), device=cuda_dev)
    _launch(fn, logits, y, loss2, None)
    assert torch.equal(loss, loss2)


@gpu
def test_degenerate_batches_give_nan_and_zero(cuda_dev):
    """CE with every row ignored, or a zero total weight over the counted rows: loss nan (as torch), dlogits 0"""
    B, C = 9, 5
    logits = torch.randn(B, C, device=cuda_dev)
    cases = [(dict(label_smoothing=0.1), torch.full((B,), -100)),
             (dict(weight=torch.ones(C), ignore_index=4), torch.full((B,), 4)),
             (dict(weight=torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0])), torch.tensor([0, 1] * 4 + [0])),
             (dict(weight=torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0]), label_smoothing=0.3), torch.tensor([0, 1] * 4 + [1]))]
    for kw, y in cases:
        y = y.to(cuda_dev)
        fn = b2.Loss(L.LOSS_CE, C, cuda_dev, **kw)
        loss, dl = torch.empty((), device=cuda_dev), torch.full_like(logits, 7.0)
        _launch(fn, logits, y, loss, dl)
        torch.cuda.synchronize()
        ref = F.cross_entropy(logits, y, **{k: (v.to(cuda_dev) if torch.is_tensor(v) else v) for k, v in kw.items()})
        assert torch.isnan(ref) and torch.isnan(loss), kw
        assert torch.equal(dl, torch.zeros_like(dl)), kw


@gpu
@pytest.mark.parametrize("case", _KERNEL_CASES)
def test_graph_replays_are_bitwise_equal(cuda_dev, case):
    fn, _ref, logits, y = _kernel_case(case, 300, 35, cuda_dev, seed=5)
    lab = fn.device_labels(y, 300)
    loss, dl = torch.empty((), device=cuda_dev), torch.empty_like(logits)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _launch(fn, logits, lab.view(y.shape), loss, dl)       # eager, then captured
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    eager = (loss.clone(), dl.clone())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn.launch(logits.data_ptr(), lab, 300, loss.data_ptr(), dl.data_ptr(), torch.cuda.current_stream().cuda_stream)
    outs = []
    for _ in range(2):
        loss.zero_()
        dl.zero_()
        g.replay()
        torch.cuda.synchronize()
        outs.append((loss.clone(), dl.clone()))
    for a, b in (outs[0], outs[1]), (outs[0], eager):
        assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))
        assert torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


# ---- GPU: the default path, bit for bit ---------------------------------------------------------------------------------
class _RawCE:
    """the captured step's loss as the parent ran it: b2_ce_fwd_bwd, called directly"""
    float_labels, plain_ce = False, True

    def __init__(self, C):
        self.C = C

    def label_shape(self, rows):
        return (rows,)

    def device_labels(self, labels, batch):
        return labels.contiguous().view(-1)

    def launch(self, logits, labels, batch, loss, dlogits, stream):
        L.call("b2_ce_fwd_bwd", logits, labels.data_ptr(), batch, self.C, loss, dlogits, stream)


@gpu
def test_default_loss_path_is_bitwise_unchanged(cuda_dev):
    """criterion None and CrossEntropyLoss(): at each of 3 captured steps (dropout on) the step's loss and
    d(loss)/d(logits) are bitwise what b2_ce_fwd_bwd gives on that step's logits and labels.  The fp32 masters follow a
    step that calls b2_ce_fwd_bwd itself to within the backward's run-to-run noise: its bias / LayerNorm gradients are
    fp32 reductions at L2 whose order is not fixed, so two runs of the same step are not bitwise equal either."""
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = [labelled_batch(cfg, 4, 128, 4400 + i, "single") for i in range(3)]
    masters = {}
    for variant in ("raw", "none", "ce"):
        model = make_model(tiny_config(), state, cuda_dev).train()
        opt = b2.build_optimizer(model, b2.Args())
        st = b2.FusedTrainStep(model, opt, 4, 128, criterion=nn.CrossEntropyLoss() if variant == "ce" else None)
        if variant == "raw":
            st.loss_fn = _RawCE(cfg.num_labels)
        assert variant == "raw" or st.loss_fn.plain_ce
        ws = model._engine.workspace(4, 128, 4)
        for b in batches:
            loss = st(b).clone()
            torch.cuda.synchronize()
            got_dl = ws["dloss_logits"].clone()
            want_loss, want_dl = torch.empty((), device=cuda_dev), torch.empty_like(got_dl)
            L.call("b2_ce_fwd_bwd", ws["logits"].data_ptr(), st.d_lab.data_ptr(), 4, cfg.num_labels,
                   want_loss.data_ptr(), want_dl.data_ptr(), torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            assert torch.equal(loss, want_loss) and torch.equal(got_dl, want_dl), variant
        masters[variant] = model._flat.detach().clone()
    for v in ("none", "ce"):
        assert float((masters[v] - masters["raw"]).abs().max()) <= 2 * 3e-5 * len(batches), v


# ---- GPU: 4 optimizer steps against the oracle on every path ------------------------------------------------------------
STEPS = 4
_CASES = {
    # name: (num_labels, config problem_type, label kind, criterion factory (None: the model's own loss))
    "regression1": (1, None, "regression", None),
    "regression3": (3, "regression", "regression", lambda: nn.MSELoss()),
    "multilabel_pos_weight": (4, None, "multi", lambda: nn.BCEWithLogitsLoss(pos_weight=torch.tensor([0.5, 2., 1., 3.]))),
    "ce_weight_smoothing": (6, None, "single",
                            lambda: nn.CrossEntropyLoss(weight=W6.clone(), label_smoothing=0.1)),
}
_REF = {}


def _reference(case, size, k=1, clip=None):
    """oracle trajectory: (config kwargs, initial state, batches, final weights, first moments, micro-batch losses)"""
    key = (case, size, k, clip)
    if key in _REF:
        return _REF[key]
    C, pt, kind, make = _CASES[case]
    kw = dict(num_labels=C, problem_type=pt, **NO_DROP)
    if size == "tiny":
        cfg = tiny_config(**kw)
        state = state_from_hf_init(cfg)
        bsz, odev = 4, "cpu"
    else:
        cfg = b2.chinese_bert_wwm_ext_config(**kw)
        b2.set_seed(123)
        m = b2.BertForSequenceClassification(cfg)
        state = {n: v.detach().clone() for n, v in m.state_dict().items() if n in m._params_by_name}
        del m
        bsz, odev = 8, "cuda"
    crit = None if make is None else make().to(odev)
    if crit is None:
        loss_fn = lambda z, y: hf_loss(z, y, "regression", C)  # noqa: E731
    else:
        loss_fn = lambda z, y: criterion_loss(crit, z, y)  # noqa: E731
    batches = [labelled_batch(cfg, bsz, 128, 8700 + i, kind) for i in range(STEPS * k)]
    ref = {n: v.to(odev).clone() for n, v in state.items()}
    opt = adamw_ref.HFAdamW(ref, lr=LR, weight_decay=0.01)
    losses = []
    for s in range(STEPS):
        gsum = None
        for j in range(k):
            l, _z, g = loss_and_grads(ref, cfg, to_dev(batches[s * k + j], odev), loss_fn)
            losses.append(float(l))
            g = {n: v / k for n, v in g.items()}
            gsum = g if gsum is None else {n: gsum[n] + g[n] for n in g}
        if clip is not None:
            norm = float(torch.sqrt(sum((v.double() ** 2).sum() for v in gsum.values())))
            coef = min(1.0, clip / (norm + 1e-6))
            gsum = {n: v * coef for n, v in gsum.items()}
        opt.step(gsum)
    out = (kw, state, batches, {n: v.cpu() for n, v in ref.items()},
           {n: opt.state[n]["exp_avg"].cpu() for n in ref}, losses)
    _REF[key] = out
    return out


def _args(**kw):
    a = b2.Args()
    a.local_rank, a.epochs, a.weight_decay, a.learning_rate = 0, 1, 0.01, LR
    for k, v in kw.items():
        setattr(a, k, v)
    return a


_PATHS = {"loop": {}, "eager": dict(fused=False), "fused": dict(fused=True), "packed": dict(fused=True, pack=True),
          "fused_accum2": dict(fused=True, gradient_accumulation_steps=2),
          "fused_clip": dict(fused=True, max_grad_norm=1.0)}


def _train_and_check(cuda_dev, case, size, path):
    extra = _PATHS[path]
    k = extra.get("gradient_accumulation_steps", 1)
    clip = extra.get("max_grad_norm")
    kw, state, batches, rw, rm, rlosses = _reference(case, size, k, clip)
    cfg = (tiny_config if size == "tiny" else b2.chinese_bert_wwm_ext_config)(**kw)
    model = make_model(cfg, state, cuda_dev).train()
    make = _CASES[case][3]
    crit = None if make is None else make().to(cuda_dev)
    losses = []
    if path == "loop":
        opt = b2.build_optimizer(model, _args())
        for bt in batches:
            d = to_dev(bt, cuda_dev)
            out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                        attention_mask=d["attention_mask"], labels=d["label"])
            loss = out.loss if crit is None else criterion_loss(crit, out.logits, d["label"])
            loss.backward()
            opt.step()
            losses.append(float(loss))
    else:
        args = _args(**extra)
        opt = b2.build_optimizer(model, args)
        tr = b2.Trainer(args, cfg, model, crit, opt)
        for bt in batches:
            losses.append(float(tr.train_step(bt)))
    torch.cuda.synchronize()
    if _CASES[case][1] is None:
        assert cfg.problem_type == b2.infer_problem_type(cfg.num_labels, batches[0]["label"])
    assert max(abs(a - b) for a, b in zip(losses, rlosses)) <= TOL_TRAJ, (losses, rlosses)
    w = {n: v.detach().cpu() for n, v in model.state_dict().items()}
    m = {n: ea.detach().cpu() for n, (ea, _v) in opt.moments().items()}
    for n, v in rw.items():
        assert float((w[n] - v).abs().max()) <= 2 * LR * STEPS + 2e-5, n
    assert_grads_within_tolerance(m, rm, qk_tol=TOL_GRAD_REL_QK)


@gpu
@pytest.mark.parametrize("path", sorted(_PATHS))
@pytest.mark.parametrize("case", sorted(_CASES))
def test_losses_match_oracle_on_every_path(cuda_dev, case, path):
    _train_and_check(cuda_dev, case, "tiny", path)


@gpu
@pytest.mark.parametrize("case", sorted(_CASES))
def test_losses_match_oracle_config_a(cuda_dev, case):
    _train_and_check(cuda_dev, case, "configA", "fused")
    torch.cuda.empty_cache()


# ---- GPU: HF's problem-type rule in the model -------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("problem_type,C,kind", [(None, 1, "regression"), ("regression", 3, "regression"),
                                                 (None, 4, "multi"), (None, 6, "single")])
def test_in_model_loss_is_hfs(cuda_dev, problem_type, C, kind):
    cfg = tiny_config(num_labels=C, problem_type=problem_type, **NO_DROP)
    model = make_model(cfg, state_from_hf_init(cfg), cuda_dev).eval()
    d = to_dev(labelled_batch(cfg, 5, 128, 5100, kind), cuda_dev)
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    assert cfg.problem_type == (problem_type or b2.infer_problem_type(C, d["label"]))
    ref = float(hf_loss(out.logits.double(), d["label"].double() if kind != "single" else d["label"],
                        cfg.problem_type, C))
    assert abs(float(out.loss) - ref) <= 1e-5 * abs(ref) + 1e-6
    if kind != "single":
        with pytest.raises(TypeError, match="floating"):
            model(input_ids=d["input_ids"], labels=d["label"].long())
        with pytest.raises(ValueError):
            model(input_ids=d["input_ids"], labels=d["label"].reshape(-1)[:3])
    else:
        with pytest.raises(TypeError, match="int64"):
            model(input_ids=d["input_ids"], labels=d["label"].float())


@gpu
def test_one_label_trains_regression(cuda_dev):
    """num_labels = 1 is HF's regression: without weight decay the masters move at every step (with cross-entropy over
    one class the gradient was 0 and only weight decay moved them)"""
    for fused in (True, False):
        cfg = tiny_config(num_labels=1, **NO_DROP)
        model = make_model(cfg, state_from_hf_init(cfg), cuda_dev).train()
        args = _args(fused=fused, weight_decay=0.0)
        tr = b2.Trainer(args, cfg, model, None, b2.build_optimizer(model, args))
        for i in range(3):
            before = model._flat.detach().clone()
            loss = tr.train_step(labelled_batch(cfg, 4, 128, 6100 + i, "regression"))
            torch.cuda.synchronize()
            assert float(loss) > 0 and not torch.equal(model._flat, before), (fused, i)
        assert cfg.problem_type == "regression"


@gpu
def test_captured_step_rejects_what_it_cannot_reproduce(cuda_dev):
    cfg = tiny_config(**NO_DROP)
    model = make_model(cfg, state_from_hf_init(cfg), cuda_dev).train()
    args = _args(fused=True)
    tr = b2.Trainer(args, cfg, model, _MyCE(), b2.build_optimizer(model, args))
    with pytest.raises(ValueError, match=r"args\.fused = False"):
        tr.train_step(labelled_batch(cfg, 4, 128, 1, "single"))
    st = b2.FusedTrainStep(model, tr.optimizer, 4, 128)
    with pytest.raises(TypeError, match="int64"):
        st(labelled_batch(tiny_config(num_labels=6), 4, 128, 1, "multi"))


@gpu
def test_trainer_rebuilds_the_step_when_the_criterion_changes(cuda_dev):
    cfg = tiny_config(**NO_DROP)
    model = make_model(cfg, state_from_hf_init(cfg), cuda_dev).train()
    args = _args(fused=True)
    crit = nn.CrossEntropyLoss(weight=W6.clone().to(cuda_dev))
    tr = b2.Trainer(args, cfg, model, crit, b2.build_optimizer(model, args))
    bt = labelled_batch(cfg, 4, 128, 2, "single")
    tr.train_step(bt)
    first = tr._fused
    tr.train_step(bt)
    assert tr._fused is first
    crit.weight.mul_(0.5)
    tr.train_step(bt)
    assert tr._fused is not first and torch.equal(tr._fused.loss_fn.weight, crit.weight)


# ---- GPU: dev() / test() ----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("kind", ["multi", "regression"])
def test_dev_and_test_metrics(cuda_dev, kind, fused):
    from sklearn.metrics import classification_report
    C = 4 if kind == "multi" else 1
    cfg = tiny_config(num_labels=C, **NO_DROP)
    model = make_model(cfg, state_from_hf_init(cfg), cuda_dev)
    args = _args(fused=fused)
    tr = b2.Trainer(args, cfg, model, None, b2.build_optimizer(model, args))
    loader = [labelled_batch(cfg, 8, 128, 9900 + i, kind) for i in range(3)]
    loss_total, metric = tr.dev(loader)
    model.eval()
    with torch.no_grad():
        logits = torch.cat([model(**{k: v for k, v in to_dev(b, cuda_dev).items() if k != "label"}).logits.cpu()
                            for b in loader])
    labels = torch.cat([b["label"] for b in loader])
    ref_loss = sum(float(hf_loss(logits[8 * i:8 * i + 8].double(), b["label"].double(), cfg.problem_type, C))
                   for i, b in enumerate(loader))
    assert abs(float(loss_total) - ref_loss) <= 1e-5 * abs(ref_loss) + 1e-5
    if kind == "multi":
        want = float(((logits > 0) == (labels >= 0.5)).all(dim=1).double().mean())
        assert float(metric) == pytest.approx(want, abs=1e-12)
        names = ["a", "b", "c", "d"]
        report = tr.test(model, loader, names)
        assert report == classification_report((labels >= 0.5).numpy().astype(int), (logits > 0).numpy().astype(int),
                                                target_names=names)
    else:
        want = float(np.corrcoef(logits.reshape(-1).numpy(), labels.numpy())[0, 1])
        assert abs(metric - want) <= 1e-6
        with pytest.raises(ValueError, match="regression"):
            tr.test(model, loader, ["y"])


# ---- two GPUs --------------------------------------------------------------------------------------------------------------
@gpu
def test_ddp_multilabel_world2():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29597", os.path.join(ROOT, "tests", "ddp_loss_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_loss_worker: OK" in r.stdout, r.stdout[-3000:]
