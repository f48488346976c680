"""Gradient-norm clipping: clip_grad_norm_, Args.max_grad_norm, and the kernels under them (b2_grad_reduce_sumsq,
b2_grad_norm_finalize, the clip coefficient and fp32 source of the update kernels).

The oracle is live: bert_ref.loss_and_grads -> fp32 torch.nn.utils.clip_grad_norm_ on the oracle gradients (on the DDP
mean for world > 1) -> adamw_ref.HFAdamW.  The argument checks at the top run without a GPU."""
import contextlib
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from parity import (TOL_GRAD_REL_QK, adamw_ref, assert_grads_within_tolerance, b2, bert_ref, full_config, make_model,
                    state_from_hf_init, tiny_config, to_dev)
from pytorch_distributed_nlp_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LR = 3e-5
bf = torch.bfloat16
gpu = pytest.mark.gpu


# ---- argument validation (CPU) ------------------------------------------------------------------------------------------
def _cpu_model():
    return b2.BertForSequenceClassification(tiny_config())


def test_clip_rejects_other_norm_types():
    m = _cpu_model()
    for nt in (1.0, float("inf"), 3):
        with pytest.raises(ValueError, match="norm_type"):
            b2.clip_grad_norm_(m.parameters(), 1.0, norm_type=nt)


def test_clip_rejects_foreign_and_partial_parameter_lists():
    m, other = _cpu_model(), _cpu_model()
    with pytest.raises(TypeError, match="ONE b200"):
        b2.clip_grad_norm_(torch.nn.Linear(4, 4).parameters(), 1.0)
    with pytest.raises(TypeError, match="ONE b200"):
        b2.clip_grad_norm_(list(m.parameters()) + list(other.parameters()), 1.0)
    with pytest.raises(TypeError, match="ONE b200"):
        b2.clip_grad_norm_([], 1.0)
    with pytest.raises(ValueError, match="every parameter"):
        b2.clip_grad_norm_(list(m.parameters())[:-1], 1.0)
    with pytest.raises(ValueError, match="every parameter"):
        b2.clip_grad_norm_(m.classifier.weight, 1.0)


def test_clip_has_no_cpu_path():
    m = _cpu_model()
    with pytest.raises(RuntimeError, match="not on CUDA"):
        b2.clip_grad_norm_(m.parameters(), 1.0)


# ---- helpers ------------------------------------------------------------------------------------------------------------
def _same(got, want):
    """bitwise equal, NaN wherever the other is NaN"""
    assert got.dtype == want.dtype and got.shape == want.shape
    if not want.is_floating_point():
        assert torch.equal(got, want)
        return
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    itype = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}[got.dtype]
    assert torch.equal(got.view(itype)[~nan], want.view(itype)[~nan])


def _ranges():
    lay = b2.modeling._Layout(tiny_config())
    n = lay.total
    return n, [(0, n), (8, n - 8), (24, 24 + 8 * 777), (lay.buckets[1][0], lay.buckets[2][1]), (40, 40)]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _reduce(peers, b, e, stash=None, partials=None):
    ns = L.sumsq_slots(e - b)
    partials = torch.full((ns + 4,), 7.0, dtype=torch.float64, device=peers[0].device) if partials is None else partials
    L.call("b2_grad_reduce_sumsq", L.ptr_array([p.data_ptr() for p in peers]), len(peers), L.ptr(stash), b, e,
           partials.data_ptr(), _stream())
    return partials, ns


def _finalize(partials, ns, max_norm, scale=None, found_inf=None):
    dev = partials.device
    out = [torch.full((), 5.0, device=dev) for _ in range(3)]
    L.call("b2_grad_norm_finalize", partials.data_ptr(), ns, None, None, 1, 0, 0, None, max_norm, L.ptr(scale),
           L.ptr(found_inf), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), _stream())
    torch.cuda.synchronize()
    return out


def _torch_coef(norm, max_norm):
    """torch 2.11 clip_grads_with_norm_ on an fp32 norm"""
    return torch.clamp(torch.tensor(max_norm, dtype=torch.float32) / (norm.cpu() + 1e-6), max=1.0)


# ---- 1. reduce + sum of squares -----------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("world", [1, 2, 4])
def test_reduce_sumsq_kernel(cuda_dev, world):
    """the stash is the rank-order fp32 sum x 1/world bitwise, the norm is float64's within 1e-6, two launches agree
    bitwise, nothing outside the slice (or past the slots) is written, and the coefficient is torch's formula"""
    n, ranges = _ranges()
    gen = torch.Generator().manual_seed(11 + world)
    peers0 = [(torch.randn(n, generator=gen) * 1e-2 * (1 + r)).to(bf) for r in range(world)]
    peers = [p.to(cuda_dev) for p in peers0]
    for (b, e) in ranges:
        stash = torch.full((e - b + 16,), 7.0, device=cuda_dev) if world > 1 else None
        partials, ns = _reduce(peers, b, e, stash)
        torch.cuda.synchronize()
        if world > 1:
            acc = torch.zeros(e - b)
            for p in peers0:
                acc = acc + p[b:e].float()
            want = acc * (1.0 / world)
            _same(stash[:e - b].cpu(), want)
            assert bool((stash[e - b:] == 7.0).all())
        else:
            want = peers0[0][b:e].float()
        for p, p0 in zip(peers, peers0):
            _same(p.cpu(), p0)
        assert bool((partials[ns:] == 7.0).all())
        if e == b:
            continue
        ref = math.sqrt(float(np.sum(want.numpy().astype(np.float64) ** 2)))
        norm, coef, skip = _finalize(partials, ns, 0.5 * ref)
        assert abs(float(norm) - ref) <= 1e-6 * ref, (float(norm), ref)
        _same(coef.cpu(), _torch_coef(norm, 0.5 * ref))
        assert float(skip) == 0.0
        again, _ = _reduce(peers, b, e, stash)
        torch.cuda.synchronize()
        _same(again, partials)
        # GradScaler: the norm of the unscaled gradients
        scale = torch.tensor(1024.0, device=cuda_dev)
        snorm, scoef, _ = _finalize(partials, ns, 0.5 * ref / 1024, scale=scale)
        assert float(snorm) == float(norm) / 1024
        _same(scoef.cpu(), _torch_coef(snorm, 0.5 * ref / 1024))


@gpu
@pytest.mark.parametrize("bad", ["inf", "nan"])
def test_reduce_sumsq_nonfinite(cuda_dev, bad):
    """inf / nan reach the norm; torch's coefficient follows (0 for inf, NaN for NaN); under a GradScaler the step is
    flagged for skipping"""
    n = 8 * 5000
    g = (torch.randn(n, device=cuda_dev) * 1e-2).to(bf)
    g[4321] = float(bad)
    for world in (1, 2):
        peers = [g] * world
        stash = torch.empty(n, device=cuda_dev) if world > 1 else None
        partials, ns = _reduce(peers, 0, n, stash)
        norm, coef, skip = _finalize(partials, ns, 1.0)
        assert (math.isinf(float(norm)) and float(coef) == 0.0) if bad == "inf" else \
            (math.isnan(float(norm)) and math.isnan(float(coef)))
        assert float(skip) == 0.0       # no scaler: a non-finite norm propagates as in torch
        _n, _c, skip = _finalize(partials, ns, 1.0, scale=torch.tensor(2.0, device=cuda_dev))
        assert float(skip) == 1.0
    fi = torch.tensor(1.0, device=cuda_dev)
    ok = (torch.randn(n, device=cuda_dev) * 1e-2).to(bf)
    partials, ns = _reduce([ok], 0, n)
    assert float(_finalize(partials, ns, 1.0, scale=torch.tensor(2.0, device=cuda_dev), found_inf=fi)[2]) == 1.0


@gpu
def test_reduce_sumsq_rejects_bad_arguments(cuda_dev):
    g = torch.zeros(64, dtype=bf, device=cuda_dev)
    st = torch.zeros(64, device=cuda_dev)
    part = torch.zeros(8, dtype=torch.float64, device=cuda_dev)
    with pytest.raises(RuntimeError, match="8-element"):
        L.call("b2_grad_reduce_sumsq", L.ptr_array([g.data_ptr()]), 1, None, 4, 64, part.data_ptr(), _stream())
    with pytest.raises(RuntimeError, match="stash"):
        L.call("b2_grad_reduce_sumsq", L.ptr_array([g.data_ptr()] * 2), 2, None, 0, 64, part.data_ptr(), _stream())
    with pytest.raises(RuntimeError, match="stash"):
        L.call("b2_grad_reduce_sumsq", L.ptr_array([g.data_ptr()]), 1, st.data_ptr(), 0, 64, part.data_ptr(),
               _stream())


# ---- 2. coefficient 1 is today's update ---------------------------------------------------------------------------------
def _hp(coef=None, grad_f32=None):
    hp = L.AdamWHParams()
    hp.lr, hp.beta1, hp.beta2, hp.eps, hp.weight_decay, hp.correct_bias = 1e-2, 0.9, 0.999, 1e-6, 0.01, 1
    hp.clip_coef, hp.grad_f32 = L.ptr(coef), grad_f32
    return hp


@gpu
@pytest.mark.parametrize("kernel", ["reduce1", "reduce2", "slim"])
def test_clip_coefficient_one_is_todays_update(cuda_dev, kernel):
    """max_norm = inf: coefficient exactly 1, and master, moments and shadow are bitwise the unclipped update (two
    steps, so the moments are non-trivial).  reduce2: a simulated world 2 whose clipped update reads the stash."""
    world = 2 if kernel == "reduce2" else 1
    n = 8 * 20000
    b, e = 8 * 37, n - 8 * 101
    gen = torch.Generator(device=cuda_dev).manual_seed(3)
    decay = (torch.rand(n // 8, device=cuda_dev, generator=gen) < 0.5).to(torch.uint8)
    master0 = torch.randn(n, device=cuda_dev, generator=gen)
    runs = []
    for clip in (False, True):
        gen.manual_seed(4)
        master, m, v = master0.clone(), torch.zeros(n, device=cuda_dev), torch.zeros(n, device=cuda_dev)
        shadow = [torch.zeros(n, dtype=bf, device=cuda_dev) for _ in range(world)]
        step = torch.zeros(1, dtype=torch.int64, device=cuda_dev)
        ss = torch.zeros(1, device=cuda_dev)
        for _ in range(2):
            grads = [(torch.randn(n, device=cuda_dev, generator=gen) * 1e-2).to(bf) for _ in range(world)]
            coef, stash = None, None
            if clip:
                stash = torch.empty(e - b, device=cuda_dev) if world > 1 else None
                partials, ns = _reduce(grads, b, e, stash)
                _norm, coef, _skip = _finalize(partials, ns, float("inf"))
                assert float(coef) == 1.0
            hp = _hp(coef, L.ptr(stash))
            if kernel == "slim":
                L.call("b2_adamw_prepare", hp, step.data_ptr(), ss.data_ptr(), _stream())
                L.call("b2_adamw_background", grads[0].data_ptr(), shadow[0].data_ptr(), master.data_ptr(),
                       m.data_ptr(), v.data_ptr(), decay.data_ptr(), b, e, hp, ss.data_ptr(), _stream())
            else:
                L.call("b2_bucket_reduce_adamw", L.ptr_array([g.data_ptr() for g in grads]),
                       L.ptr_array([s.data_ptr() for s in shadow]), world, 0, master.data_ptr(), m.data_ptr(),
                       v.data_ptr(), decay.data_ptr(), b, e, hp, step.data_ptr(), _stream())
            L.call("b2_step_advance", step.data_ptr(), None, None, _stream())
        torch.cuda.synchronize()
        runs.append([master, m, v] + shadow)
    for got, want in zip(runs[1], runs[0]):
        _same(got, want)


@gpu
def test_clip_coefficient_scales_the_gradient(cuda_dev):
    """a coefficient c < 1 gives the update of the gradient c * g (the 256-thread kernel on the fp32 stash, and the
    background kernel on bf16 gradients where c * g is exact: c a power of two)"""
    n = 8 * 4096
    gen = torch.Generator(device=cuda_dev).manual_seed(8)
    g = (torch.randn(n, device=cuda_dev, generator=gen) * 1e-2).to(bf)
    decay = torch.ones(n // 8, dtype=torch.uint8, device=cuda_dev)
    c = torch.tensor(0.25, device=cuda_dev)
    out = []
    for clipped in (True, False):
        master, m, v = torch.ones(n, device=cuda_dev), torch.zeros(n, device=cuda_dev), torch.zeros(n, device=cuda_dev)
        sh = torch.zeros(n, dtype=bf, device=cuda_dev)
        step, ss = torch.zeros(1, dtype=torch.int64, device=cuda_dev), torch.zeros(1, device=cuda_dev)
        gg = g if clipped else (g.float() * 0.25).to(bf)
        hp = _hp(c if clipped else None)
        L.call("b2_adamw_prepare", hp, step.data_ptr(), ss.data_ptr(), _stream())
        L.call("b2_adamw_background", gg.data_ptr(), sh.data_ptr(), master.data_ptr(), m.data_ptr(), v.data_ptr(),
               decay.data_ptr(), 0, n, hp, ss.data_ptr(), _stream())
        torch.cuda.synchronize()
        out.append((master, m, v))
    for a, b_ in zip(*out):
        _same(a, b_)


# ---- 3-5. end to end, world 1 -------------------------------------------------------------------------------------------
def _oracle_clip(grads, max_norm):
    ps = {}
    for k, g in grads.items():
        p = torch.zeros_like(g, requires_grad=True)
        p.grad = g.clone()
        ps[k] = p
    norm = torch.nn.utils.clip_grad_norm_(list(ps.values()), max_norm)
    return float(norm), {k: p.grad for k, p in ps.items()}


def _oracle(cfg, state, windows, factor=0.25, dev="cpu"):
    """windows: list of lists of batches (one optimizer step each, loss / k).  Returns (max_norm, norms, weights,
    exp_avg) of HF AdamW on the clipped window means; max_norm = factor x the step-0 norm"""
    ref = {k: v.to(dev).clone() for k, v in state.items()}
    opt = adamw_ref.HFAdamW(ref, lr=LR, weight_decay=0.01)
    max_norm, norms = None, []
    for win in windows:
        acc = None
        for bt in win:
            _l, _z, g = bert_ref.loss_and_grads(ref, cfg, to_dev(bt, dev))
            acc = {k: x / len(win) for k, x in g.items()} if acc is None else \
                {k: acc[k] + x / len(win) for k, x in g.items()}
        if max_norm is None:
            max_norm = factor * math.sqrt(sum(float(x.double().pow(2).sum()) for x in acc.values()))
        norm, clipped = _oracle_clip(acc, max_norm)
        norms.append(norm)
        opt.step(clipped)
    return max_norm, norms, {k: v.cpu() for k, v in ref.items()}, \
        {k: opt.state[k]["exp_avg"].cpu() for k in ref}


def _eager_step(model, opt, win, dev, max_norm, flush=False):
    k = len(win)
    for i, bt in enumerate(win):
        d = to_dev(bt, dev)
        inside = i < k - 1 or flush
        with (model.no_sync() if inside else contextlib.nullcontext()):
            out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                        attention_mask=d["attention_mask"], labels=d["label"])
            (F.cross_entropy(out[1], d["label"]) / k).backward()
    norm = b2.clip_grad_norm_(model.parameters(), max_norm) if max_norm is not None else None
    opt.step()
    return norm


def _trainer(cfg, state, dev, mode, max_norm, k=1, **kw):
    model = make_model(cfg, state, dev)
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank = 0, 1, 0
    args.fused, args.pack, args.max_grad_norm = mode != "eager", mode == "packed", max_norm
    args.gradient_accumulation_steps = k
    for key, v in kw.items():
        setattr(args, key, v)
    opt = b2.build_optimizer(model, args)
    return model, opt, b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)


def _run(mode, cfg, state, windows, dev, max_norm, **kw):
    """-> (norms, weights, exp_avg) after one optimizer step per window"""
    k = len(windows[0])
    if mode == "loop":
        model = make_model(cfg, state, dev).train()
        opt = b2.build_optimizer(model, type("A", (), {"weight_decay": 0.01, "learning_rate": LR}))
        norms = [_eager_step(model, opt, w, dev, max_norm) for w in windows]
    else:
        model, opt, tr = _trainer(cfg, state, dev, mode, max_norm, k=k, **kw)
        norms = []
        for w in windows:
            for bt in w:
                tr.train_step(bt)
            norms.append(tr.last_grad_norm)
    norms = [None if x is None else float(x) for x in norms]
    torch.cuda.synchronize()
    w = {n: v.detach().cpu().clone() for n, v in model.state_dict().items()}
    m = {n: ea.detach().cpu().clone() for n, (ea, _v) in opt.moments().items()}
    return norms, w, m


def _check(got, oracle, steps):
    norms, w, m = got
    _mx, rnorms, rw, rm = oracle
    for a, r in zip(norms, rnorms):
        assert abs(a - r) <= 1e-2 * r, (norms, rnorms)
    for n, v in rw.items():
        assert float((w[n] - v).abs().max()) <= 2 * LR * steps + 2e-5, n
    # the first moment is the clipped gradient's running mean: clipping left out would be off by 1 / coefficient
    assert_grads_within_tolerance(m, rm, qk_tol=TOL_GRAD_REL_QK)


_CACHE = {}


def _setup(size):
    if size not in _CACHE:
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
            bsz, odev = 8, "cuda"     # the fp32 oracle of BERT-base runs on the device (same torch code)
        windows = [[bert_ref.synthetic_batch(cfg, bsz, 128, 8100 + s, padded=True)] for s in range(3)]
        _CACHE[size] = (cfg, state, windows, _oracle(cfg, state, windows, dev=odev))
    return _CACHE[size]


@gpu
@pytest.mark.parametrize("mode", ["loop", "eager", "fused", "packed"])
@pytest.mark.parametrize("size", ["tiny", "configA"])
def test_clipped_training_matches_oracle(cuda_dev, size, mode):
    """3 steps, dropout off, max_norm = 0.25 x the oracle's step-0 norm (the clip bites at every step): the returned
    norm / Trainer.last_grad_norm, the weights and the first moments against the oracle"""
    cfg, state, windows, oracle = _setup(size)
    got = _run(mode, cfg, state, windows, cuda_dev, oracle[0])
    _check(got, oracle, len(windows))
    torch.cuda.empty_cache()


@gpu
def test_clip_far_above_the_norm_is_bitwise_unclipped(cuda_dev):
    """max_norm far above the norm, on the same gradients and optimizer state: master, moments and bf16 weights after
    clip_grad_norm_ + step() are bitwise those of step() alone"""
    cfg, state, windows, _oracle_run = _setup("tiny")
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.build_optimizer(model, type("A", (), {"weight_decay": 0.01, "learning_rate": LR}))
    eng = model._engine
    _eager_step(model, opt, windows[0], cuda_dev, None)             # non-trivial moments
    d = to_dev(windows[1][0], cuda_dev)
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    st = opt._state()
    keep = [model._flat, eng.shadow, eng.grads, st["exp_avg"], st["exp_avg_sq"], st["step"], st["step_size"]]
    saved = [t.clone() for t in keep]
    opt.step()
    plain = [t.clone() for t in keep]
    for t, v in zip(keep, saved):
        t.copy_(v)
    norm = b2.clip_grad_norm_(model.parameters(), 1e9)
    assert float(opt._clip_buf["coef"]) == 1.0 and 0 < float(norm) < 1e9
    opt.step()
    torch.cuda.synchronize()
    for t, v in zip(keep, plain):
        _same(t, v)


@gpu
@pytest.mark.parametrize("mode", ["fused", "packed"])
def test_clip_far_above_the_norm_on_the_captured_steps(cuda_dev, mode):
    """the captured steps with max_norm far above the norm: coefficient exactly 1 at every step, and the weights of
    the unclipped run.  Not bitwise across the two runs: the bias gradients are summed by float atomics, so two runs of
    the same step can differ in their last bits whether or not they clip"""
    cfg, state, windows, _oracle_run = _setup("tiny")
    _n, w0, m0 = _run(mode, cfg, state, windows, cuda_dev, None)
    norms, w1, m1 = _run(mode, cfg, state, windows, cuda_dev, 1e9)
    assert all(x is not None and 0 < x < 1e9 for x in norms)
    for n in m0:
        assert float((w1[n] - w0[n]).abs().max()) <= 2 * LR * len(windows), n
        assert float((m1[n] - m0[n]).abs().max()) <= 1e-3 * max(float(m0[n].abs().max()), 1e-12), n


# ---- 4. accumulation ---------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("k,close", [(2, "final"), (3, "final"), (2, "flush"), (3, "flush"), (2, "fused")])
def test_clipped_accumulation_window_matches_oracle(cuda_dev, k, close):
    """the norm is that of the window mean: closed by a final backward, by a flush (every pass inside no_sync()), or
    on the captured step with gradient_accumulation_steps = k"""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    windows = [[bert_ref.synthetic_batch(cfg, 4, 128, 8300 + 10 * s + i, padded=(i % 2 == 1)) for i in range(k)]
               for s in range(2)]
    oracle = _oracle(cfg, state, windows)
    if close == "fused":
        got = _run("fused", cfg, state, windows, cuda_dev, oracle[0])
    else:
        model = make_model(cfg, state, cuda_dev).train()
        opt = b2.build_optimizer(model, type("A", (), {"weight_decay": 0.01, "learning_rate": LR}))
        norms = [float(_eager_step(model, opt, w, cuda_dev, oracle[0], flush=(close == "flush"))) for w in windows]
        got = (norms, {n: v.detach().cpu() for n, v in model.state_dict().items()},
               {n: ea.detach().cpu() for n, (ea, _v) in opt.moments().items()})
    _check(got, oracle, len(windows))


# ---- 5. GradScaler ------------------------------------------------------------------------------------------------------
@gpu
def test_clip_under_gradscaler(cuda_dev):
    """Trainer use_amp + max_grad_norm lands where the unscaled loop lands, with the norm of the unscaled gradients;
    an inf written into the gradients after backward makes the step skip (weights and step count unchanged)"""
    cfg, state, windows, oracle = _setup("tiny")
    n0, w0, _m0 = _run("eager", cfg, state, windows, cuda_dev, oracle[0])
    n1, w1, _m1 = _run("eager", cfg, state, windows, cuda_dev, oracle[0], use_amp=True)
    for a, c in zip(n0, n1):
        assert abs(a - c) <= 1e-3 * c, (n0, n1)
    for n in w0:
        assert float((w0[n].double() - w1[n].double()).abs().max()) <= 2e-5, n
    model, opt, tr = _trainer(cfg, state, cuda_dev, "eager", oracle[0], use_amp=True)
    tr.train_step(windows[0][0])
    scaler = tr._scaler
    before = {n: v.detach().clone() for n, v in model.state_dict().items()}
    d = to_dev(windows[1][0], cuda_dev)
    with torch.autocast("cuda"):
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                    labels=d["label"])
        loss = F.cross_entropy(out[1], d["label"])
    scaler.scale(loss).backward()
    model._engine.grads[model._layout.off("bert.encoder.layer.0.output.dense.weight") + 5] = float("inf")
    norm = b2.clip_grad_norm_(model.parameters(), oracle[0])
    scaler.step(opt)
    scaler.update()
    torch.cuda.synchronize()
    assert math.isinf(float(norm)) and int(opt._state()["step"]) == 1
    after = model.state_dict()
    for n in before:
        assert torch.equal(before[n], after[n]), n


# ---- 6. errors ----------------------------------------------------------------------------------------------------------
@gpu
def test_clip_errors(cuda_dev):
    cfg, state, windows, oracle = _setup("tiny")
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.build_optimizer(model, type("A", (), {"weight_decay": 0.01, "learning_rate": LR}))
    with pytest.raises(RuntimeError, match="optimizer"):
        b2.clip_grad_norm_(make_model(cfg, state, cuda_dev).parameters(), 1.0)
    d = to_dev(windows[0][0], cuda_dev)

    def backward():
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                    labels=d["label"])
        F.cross_entropy(out[1], d["label"]).backward()

    backward()
    norm = b2.clip_grad_norm_(model.parameters(), 1.0)
    assert norm.is_cuda and norm.dtype == torch.float32 and norm.dim() == 0
    with pytest.raises(RuntimeError, match="twice"):
        b2.clip_grad_norm_(model.parameters(), 1.0)
    opt.step()
    backward()
    before = {n: v.detach().clone() for n, v in model.state_dict().items()}
    model._engine.grads[3] = float("inf")
    with pytest.raises(RuntimeError, match="non-finite"):
        b2.clip_grad_norm_(model.parameters(), 1.0, error_if_nonfinite=True)
    after = model.state_dict()
    for n in before:
        assert torch.equal(before[n], after[n]), n
    assert opt._clip is None and int(opt._state()["step"]) == 1


# ---- 7. DDP world 2 -----------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dma", ["0", "1"])
def test_ddp_world2_clip(dma):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29591", os.path.join(ROOT, "tests", "ddp_clip_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, B2_DDP_DMA=dma))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_clip_worker: OK" in r.stdout, r.stdout[-3000:]
