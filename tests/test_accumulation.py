"""GPU: gradient accumulation -- no_sync() micro-batches, Trainer gradient_accumulation_steps, and the fp32 accumulator
kernel (b2_grad_accumulate) under them.

The headline check: on one GPU, k micro-batches with loss / k make the same update as a world-k DDP step, so the
committed world-2/4/8 fixture (tests/golden/config_a_ddp.pt) is reproduced by one rank."""
import contextlib
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from parity import (TOL_GRAD_REL, TOL_LOSS, adamw_ref, b2, bert_ref, full_config, grad_report, make_model,
                    oracle_masks, state_from_hf_init, tiny_config, to_dev)
from pytorch_distributed_nlp_b200 import _lib as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
LR = 3e-5


class A:
    weight_decay, learning_rate = 0.01, LR


def _same(got, want):
    """bitwise equal, NaN wherever the other is NaN (the device and torch may pick different NaN payloads)"""
    assert got.dtype == want.dtype and got.shape == want.shape
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    itype = torch.int16 if got.dtype == torch.bfloat16 else torch.int32
    assert torch.equal(got.view(itype)[~nan], want.view(itype)[~nan])


# ---- 1. the kernel ------------------------------------------------------------------------------------------------------
def _ranges():
    lay = b2.modeling._Layout(tiny_config())
    n = lay.total
    return n, [(0, n), (8, n - 8), (24, 24 + 8 * 777), (lay.buckets[1][0], lay.buckets[2][1]), (40, 40)]


@pytest.mark.parametrize("mode", ["store", "add", "fold", "flush"])
def test_grad_accumulate_kernel_matches_torch(cuda_dev, mode):
    """each mode against torch over several slices: 8-element (16-byte bf16) starts that are not 16-element aligned, a
    slice of whole buckets, an empty one; inf / nan in both operands pass through; nothing outside the slice moves"""
    op = {"store": L.ACCUM_STORE, "add": L.ACCUM_ADD, "fold": L.ACCUM_FOLD, "flush": L.ACCUM_FLUSH}[mode]
    n, ranges = _ranges()
    gen = torch.Generator().manual_seed(5)
    g0 = (torch.randn(n, generator=gen) * 1e-3).to(torch.bfloat16)
    a0 = torch.randn(n, generator=gen) * 1e-3
    for t in (g0, a0):
        t[100], t[101], t[102] = float("inf"), float("-inf"), float("nan")
    a0[203], g0[204] = float("nan"), float("inf")
    a0[3000] = 3.0e38                       # fp32 sum overflows, then rounds to bf16 inf
    g0[3000] = 3.0e38
    s = torch.cuda.current_stream(cuda_dev).cuda_stream
    for (b, e) in ranges:
        g, a = g0.to(cuda_dev), a0.to(cuda_dev)
        L.call("b2_grad_accumulate", g.data_ptr(), a.data_ptr(), b, e, op, s)
        torch.cuda.synchronize()
        wg, wa = g0.clone(), a0.clone()
        if mode == "store":
            wa[b:e] = g0[b:e].float()
        elif mode == "add":
            wa[b:e] = a0[b:e] + g0[b:e].float()
        elif mode == "fold":
            wg[b:e] = (a0[b:e] + g0[b:e].float()).to(torch.bfloat16)
        else:
            wg[b:e] = a0[b:e].to(torch.bfloat16)
        _same(g.cpu(), wg)
        _same(a.cpu(), wa)
    g, a = g0.to(cuda_dev), a0.to(cuda_dev)
    with pytest.raises(RuntimeError, match="8-element"):
        L.call("b2_grad_accumulate", g.data_ptr(), a.data_ptr(), 4, 64, op, s)
    with pytest.raises(RuntimeError, match="mode"):
        L.call("b2_grad_accumulate", g.data_ptr(), a.data_ptr(), 0, 64, 7, s)


# ---- 2. eager no_sync() against the oracle --------------------------------------------------------------------------------
def _eager_pass(model, b, dev, k, inside):
    d = to_dev(b, dev)
    with (model.no_sync() if inside else contextlib.nullcontext()):
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                    labels=d["label"])
        loss = F.cross_entropy(out[1], d["label"])
        (loss / k).backward()
    torch.cuda.synchronize()
    return float(loss.detach())


@pytest.mark.parametrize("k,last", [(2, "final"), (3, "final"), (2, "flush"), (3, "flush")])
@pytest.mark.parametrize("dropout", [False, True])
def test_eager_no_sync_window_matches_oracle(cuda_dev, k, last, dropout):
    """k micro-batches, loss / k, the first k - 1 (last="flush": all k) inside no_sync(): every micro-batch's loss,
    grad_dict() along the window (the running oracle sum, then the mean) and the weights after step() against the
    oracle.  With dropout, micro-batch i draws the masks of rng step (step + i): the stream moves once per pass."""
    cfg = tiny_config() if dropout else tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.build_optimizer(model, A)
    seed, step0 = 99, 7
    model._engine.seed_dropout(seed, step0)
    batches = [bert_ref.synthetic_batch(cfg, 4, 128, 4000 + i, padded=(i % 2 == 1)) for i in range(k)]
    want = None
    for i, b in enumerate(batches):
        loss = _eager_pass(model, b, cuda_dev, k, inside=(i < k - 1 or last == "flush"))
        masks = oracle_masks(cfg, 4, 128, seed, step0 + i) if dropout else None
        rl, _rz, rg = bert_ref.loss_and_grads(state, cfg, b, masks=masks)
        assert abs(loss - float(rl)) <= TOL_LOSS, (i, loss, float(rl))
        want = {n: g / k for n, g in rg.items()} if want is None else {n: want[n] + g / k for n, g in rg.items()}
        worst, rows = grad_report(model.grad_dict(), want)
        assert worst <= TOL_GRAD_REL, (i, sorted(rows, key=lambda r: -r[1])[:5])
    assert model._engine.accum_live == (last == "flush")
    opt.step()
    assert not model._engine.accum_live and int(opt._state()["step"]) == 1
    ref = {n: v.clone() for n, v in state.items()}
    adamw_ref.HFAdamW(ref, lr=LR, weight_decay=0.01).step(want)
    sd = model.state_dict()
    for n, v in ref.items():    # one AdamW step moves a weight by ~lr; sign flips of near-zero gradients bound the error
        assert float((sd[n].cpu() - v).abs().max()) <= 2 * LR + 1e-6, n
    # the next window starts afresh (STORE): one plain step equals the oracle's on the updated weights.  The stream
    # has moved once per accumulating pass and once in step()
    b = bert_ref.synthetic_batch(cfg, 4, 128, 4100)
    loss = _eager_pass(model, b, cuda_dev, 1, inside=False)
    masks = oracle_masks(cfg, 4, 128, seed, step0 + k + (last == "flush")) if dropout else None
    rl, _rz, rg = bert_ref.loss_and_grads({n: v.cpu() for n, v in sd.items() if n in state}, cfg, b, masks=masks)
    assert abs(loss - float(rl)) <= TOL_LOSS
    worst, rows = grad_report(model.grad_dict(), rg)
    assert worst <= TOL_GRAD_REL, sorted(rows, key=lambda r: -r[1])[:5]
    opt.step()


def test_no_sync_errors_and_no_accumulator_without_accumulation(cuda_dev):
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.build_optimizer(model, A)
    b = bert_ref.synthetic_batch(cfg, 4, 128, 3)
    # accumulation never asked for: no accumulator, eager or captured
    _eager_pass(model, b, cuda_dev, 1, inside=False)
    opt.step()
    step = b2.FusedTrainStep(model, opt, 4, 128)
    for _ in range(4):
        step(b)
    torch.cuda.synchronize()
    assert model._engine.accum is None and not model._engine.accum_in_use and step.graph is not None
    # a backward inside no_sync() right after an un-stepped plain one would drop the plain one's gradients
    _eager_pass(model, b, cuda_dev, 1, inside=False)
    with pytest.raises(RuntimeError, match="no_sync"):
        _eager_pass(model, b, cuda_dev, 1, inside=True)
    opt.step()
    # repeated backwards inside no_sync() accumulate
    for _ in range(3):
        _eager_pass(model, b, cuda_dev, 3, inside=True)
    assert model._engine.accum is not None and model._engine.accum.numel() == model._layout.total
    opt.step()


# ---- 3. one GPU, k micro-batches == the world-k DDP fixture -------------------------------------------------------------
def _fixture_run(k, fused, dev):
    """bench.py's `parity` block with world k replaced by k micro-batches on this GPU; returns the deviations"""
    fx = torch.load(os.path.join(GOLD, "config_a_ddp.pt"))
    fw, steps = fx["worlds"][k], int(fx["steps"])
    cfg = full_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg)
    chk = float(sum(p.detach().double().sum() for p in model.parameters()))
    assert abs(chk - fx["init_checksum"]) <= 1e-6 * max(1.0, abs(fx["init_checksum"])), "initialiser drifted"
    model.to(dev)
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank = 0, 1, 0
    args.gradient_accumulation_steps, args.fused = k, fused
    opt = b2.build_optimizer(model, args)
    tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)
    d_local, d_mean = 0.0, 0.0
    for s in range(steps):
        losses = []
        for r in range(k):
            batch = b2.synthetic_batch(cfg, 32, 128, 5000 + 100 * s + r, padded=(s % 2 == 1))
            losses.append(float(tr.train_step(batch)))
            d_local = max(d_local, abs(losses[-1] - float(fw["loss"][s][r])))
        d_mean = max(d_mean, abs(sum(losses) / k - float(fw["loss"][s].mean())))
    assert int(opt._state()["step"]) == steps
    sd = model.state_dict()
    d_w, d_norm = 0.0, 0.0
    norm_floor = 1e-3 * max(fw["final_norms"].values())
    for n, ref in fw["final_samples"].items():
        f = sd[n].detach().flatten()
        if f.numel() > ref.numel():
            f = f[(torch.arange(ref.numel(), dtype=torch.int64) * (f.numel() - 1) // (ref.numel() - 1)).to(f.device)]
        d_w = max(d_w, float((f.cpu() - ref).abs().max()))
        d_norm = max(d_norm, abs(float(sd[n].double().norm()) - fw["final_norms"][n]) / max(fw["final_norms"][n],
                                                                                               norm_floor))
    del tr, opt, model
    torch.cuda.empty_cache()
    return d_local, d_mean, d_w, d_norm, 2 * LR * steps + 2e-5


@pytest.mark.parametrize("k,fused", [(2, True), (4, True), (8, True), (2, False)])
def test_one_gpu_accumulation_reproduces_world_k_fixture(cuda_dev, k, fused):
    """config A full size, dropout off, set_seed(123) weights: Trainer with gradient_accumulation_steps = k, micro-batch
    r of step s = fixture rank r's batch.  Tolerances of bench.py's parity block."""
    d_local, d_mean, d_w, d_norm, tol_w = _fixture_run(k, fused, cuda_dev)
    print("k=%d fused=%s: dloss %.2e, dloss_mean %.2e, dweight %.2e (tol %.2e), dnorm_rel %.2e"
          % (k, fused, d_local, d_mean, d_w, tol_w, d_norm))
    assert d_local <= 1e-2 and d_mean <= 1e-2, (d_local, d_mean)
    assert d_w <= tol_w, (d_w, tol_w)
    assert d_norm <= 1e-3, d_norm


# ---- 4-7. the Trainer paths agree ------------------------------------------------------------------------------------
def _trainer(cfg, state, dev, k, **kw):
    model = make_model(cfg, state, dev)
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank = 0, 1, 0
    args.gradient_accumulation_steps = k
    for key, v in kw.items():
        setattr(args, key, v)
    opt = b2.build_optimizer(model, args)
    return model, opt, b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)


def _train(tr, model, batches, seed=None):
    if seed is not None:
        model._engine.seed_dropout(seed, 0)
    losses = [float(tr.train_step(b)) for b in batches]
    return losses, {n: v.detach().clone() for n, v in model.state_dict().items()}


def test_eager_and_fused_accumulation_agree_with_dropout(cuda_dev):
    """tiny config, dropout ON, k = 2 over 3 windows: the eager Trainer loop (no_sync + loss / k) and the captured steps
    (one graph per role) draw the same masks and land on the same weights"""
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = [bert_ref.synthetic_batch(cfg, 4, 128, 2200 + i, padded=(i % 2 == 1)) for i in range(6)]
    m0, o0, t0 = _trainer(cfg, state, cuda_dev, 2, fused=False)
    l0, w0 = _train(t0, m0, batches, seed=17)
    m1, o1, t1 = _trainer(cfg, state, cuda_dev, 2, fused=True)
    l1, w1 = _train(t1, m1, batches, seed=17)
    assert int(o0._state()["step"]) == int(o1._state()["step"]) == 3
    assert len(t1._fused._graphs) == 2 and t1._fused.graph is not None
    for a, c in zip(l0, l1):
        assert abs(a - c) <= 5e-4, (l0, l1)
    for n in w0:
        assert float((w0[n].double() - w1[n].double()).abs().max()) <= 2e-5, n


def test_packed_accumulation_agrees_with_padded(cuda_dev):
    from test_packing import short_batch
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    batches = [short_batch(cfg, 16, 500 + i, hi=(30 if i % 2 else 90)) for i in range(4)]
    m0, o0, t0 = _trainer(cfg, state, cuda_dev, 2, pack=False)
    l0, w0 = _train(t0, m0, batches)
    m1, o1, t1 = _trainer(cfg, state, cuda_dev, 2, pack=True)
    l1, w1 = _train(t1, m1, batches)
    assert int(o1._state()["step"]) == 2 and len(t1._packed) >= 2
    for a, c in zip(l0, l1):
        assert abs(a - c) <= TOL_LOSS, (l0, l1)
    for n in w0:
        assert float((w0[n].cpu() - w1[n].cpu()).abs().max()) <= 2e-4, n


def test_gradscaler_accumulation(cuda_dev):
    """use_amp with k = 2 lands where the plain eager loop lands; an inf loss in one micro-batch skips the whole
    window (weights and step count unchanged, scale halved) and the next window trains normally"""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    batches = [bert_ref.synthetic_batch(cfg, 4, 128, 2300 + i, padded=(i % 2 == 1)) for i in range(4)]
    m0, o0, t0 = _trainer(cfg, state, cuda_dev, 2, fused=False)
    l0, w0 = _train(t0, m0, batches)
    m1, o1, t1 = _trainer(cfg, state, cuda_dev, 2, fused=False, use_amp=True)
    l1, w1 = _train(t1, m1, batches)
    for a, c in zip(l0, l1):
        assert abs(a - c) <= 5e-4, (l0, l1)
    for n in w0:
        assert float((w0[n].double() - w1[n].double()).abs().max()) <= 2e-5, n
    scaler = t1._scaler
    assert float(scaler.get_scale()) == 65536.0
    t_before = int(o1._state()["step"])

    def micro(b, inside, poison):
        d = to_dev(b, cuda_dev)
        with (m1.no_sync() if inside else contextlib.nullcontext()):
            with torch.autocast("cuda"):
                out = m1(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                         attention_mask=d["attention_mask"], labels=d["label"])
                loss = F.cross_entropy(out[1], d["label"]) * (float("inf") if poison else 1.0)
            scaler.scale(loss / 2).backward()

    micro(batches[0], True, True)
    micro(batches[1], False, False)
    scaler.step(o1)
    scaler.update()
    assert float(scaler.get_scale()) == 32768.0 and int(o1._state()["step"]) == t_before
    after = m1.state_dict()
    for n in w1:
        assert torch.equal(w1[n], after[n]), n
    micro(batches[2], True, False)
    micro(batches[3], False, False)
    scaler.step(o1)
    scaler.update()
    assert int(o1._state()["step"]) == t_before + 1
    sd = m1.state_dict()
    assert all(bool(torch.isfinite(v).all()) for v in sd.values())
    assert float((sd["classifier.weight"] - w1["classifier.weight"]).abs().max()) > 0


@pytest.mark.parametrize("fused", [True, False])
def test_trainer_train_closes_the_partial_window(cuda_dev, tmp_path, fused):
    """5 batches with k = 2: two full windows, and the epoch's last batch is applied by the closing step"""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    model, opt, tr = _trainer(cfg, state, cuda_dev, 2, fused=fused)
    tr.args.ckpt_path = str(tmp_path / "ckpt.pt")
    batches = [bert_ref.synthetic_batch(cfg, 4, 128, 2400 + i, padded=(i % 2 == 1)) for i in range(5)]
    tr.train(batches)
    assert int(opt._state()["step"]) == 3 and tr._micro == 0 and not model._engine.accum_live
    # the oracle: mean of (b0, b1), mean of (b2, b3), then b4 alone scaled by 1/2
    ref = {n: v.clone() for n, v in state.items()}
    ropt = adamw_ref.HFAdamW(ref, lr=LR, weight_decay=0.01)
    for win in ([0, 1], [2, 3], [4]):
        acc = None
        for i in win:
            _l, _z, g = bert_ref.loss_and_grads(ref, cfg, batches[i])
            acc = {n: x / 2 for n, x in g.items()} if acc is None else {n: acc[n] + x / 2 for n, x in g.items()}
        ropt.step(acc)
    sd = model.state_dict()
    for n, v in ref.items():
        assert float((sd[n].cpu() - v).abs().max()) <= 2e-4, n


# ---- 8. DDP: world 2 x k = 2 == the world-4 fixture ------------------------------------------------------------------
def test_ddp_world2_accumulation_reproduces_world4_fixture():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29583", os.path.join(ROOT, "tests", "ddp_accum_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_accum_worker: OK" in r.stdout, r.stdout[-3000:]
