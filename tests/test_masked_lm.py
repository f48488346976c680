"""GPU: BertForMaskedLM -- the masked-LM head kernels (csrc/mlm_head.cu) against float64, the model against the
masked-LM oracle (tests/mlm_oracle.py), the eager full-logit path against the labelled-rows path, the tied
word-embedding gradient, the vocabulary padding under every optimizer, determinism, checkpoints and the Trainer.

Kernel bounds.  fp32 unit roundoff u = 2^-24, bf16 2^-8 relative.  The cross-entropy kernel's log-sum-exp over V
columns adds V terms of at most 1 (each exp within a few u of exact), so lse is off by at most (V + 8) u relative to
the sum, i.e. (V + 8) u absolute in the log; a row loss lse - x_y is then off by that plus u |lse|.  d_logits is one
bf16 rounding (2^-8 |ref|) of a value whose fp32 error is a few u times the scale.
"""
import numpy as np
import pytest
import torch
import torch.nn as nn

import mlm_oracle as mlm
from parity import TOL_GRAD_REL_QK, TOL_LOSS, assert_grads_within_tolerance, b2, tiny_config
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import vocab_pad

gpu = pytest.mark.gpu
U32 = 2.0 ** -24
NO_DROP = dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
DEV = "cuda"


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cfg(**kw):
    d = dict(vocab_size=1000)
    d.update(kw)
    return tiny_config(**d)


def _model(cfg, seed=9):
    state = mlm.mlm_state_from_hf_init(cfg, seed)
    m = b2.BertForMaskedLM(cfg)
    m.load_state_dict(state, strict=True)
    return m.to(DEV), state


def _to_dev(batch):
    return {k: v.to(DEV) for k, v in batch.items()}


def _ce(logits, labels, rows, V, n_rows, d_loss=None, with_dl=True):
    Vp = logits.shape[1]
    dev = logits.device
    lab = torch.tensor(labels, dtype=torch.int32, device=dev)
    n_rows_t = torch.tensor([n_rows], dtype=torch.int32, device=dev)
    n_lab = torch.tensor([int(((lab >= 0) & (torch.arange(rows, device=dev) < n_rows)).sum())], dtype=torch.int32,
                         device=dev)
    row_loss = torch.full((rows,), float("nan"), device=dev)
    pred = torch.full((rows,), -7, dtype=torch.int32, device=dev)
    dl = torch.full((rows, Vp), float("nan"), dtype=torch.bfloat16, device=dev) if with_dl else None
    loss = torch.full((), float("nan"), device=dev)
    L.call("b2_mlm_ce", logits.data_ptr(), rows, V, Vp, lab.data_ptr(), n_rows_t.data_ptr(), n_lab.data_ptr(),
           L.ptr(d_loss), None, 0, row_loss.data_ptr(), pred.data_ptr(), L.ptr(dl), loss.data_ptr(), _stream())
    torch.cuda.synchronize()
    return row_loss, pred, dl, loss, int(n_lab)


@gpu
@pytest.mark.parametrize("V", [64, 21128, 30522])
def test_ce_kernel_against_float64(V):
    torch.manual_seed(V)
    rows, n_rows = 300, 261            # 300 is no multiple of any block size; rows past 261 are capacity padding
    Vp = vocab_pad(V)
    x = torch.randn(rows, Vp, dtype=torch.float64) * 3
    x[:, V:] = 1e4                     # the padded columns must not be read into the softmax
    labels = torch.randint(0, V, (rows,))
    labels[::7] = -1                   # ignored rows
    lx = x.float().to(DEV)
    d_loss = torch.tensor(1.7, device=DEV)
    row_loss, pred, dl, loss, n = _ce(lx, labels.tolist(), rows, V, n_rows, d_loss)
    xr = lx.double().cpu()[:, :V]
    lse = torch.logsumexp(xr, 1)
    live = (labels >= 0) & (torch.arange(rows) < n_rows)
    ref_row = torch.where(live, lse - xr.gather(1, labels.clamp(min=0)[:, None])[:, 0], torch.zeros(rows,
                                                                                                   dtype=torch.float64))
    bound = ((V + 8) * U32 + U32 * lse.abs()) * 2
    assert torch.all((row_loss.double().cpu() - ref_row).abs() <= torch.where(live, bound, torch.zeros_like(bound)))
    ref_loss = ref_row.sum() / n
    assert abs(float(loss) - float(ref_loss)) <= float(bound.max()) + rows * U32 * float(ref_row.abs().max())
    ref_pred = torch.where(live, xr.argmax(1), torch.full((rows,), -1))
    assert torch.equal(pred.long().cpu(), ref_pred)
    sm = torch.softmax(xr, 1)
    onehot = torch.zeros_like(sm)
    onehot[torch.arange(rows), labels.clamp(min=0)] = 1
    ref_dl = torch.where(live[:, None], (sm - onehot) * 1.7 / n, torch.zeros_like(sm))
    got = dl.double().cpu()
    assert torch.all(got[:, V:] == 0)
    err = (got[:, :V] - ref_dl).abs()
    assert torch.all(err <= 2.0 ** -8 * ref_dl.abs() + 16 * U32 * 1.7 / n), float(err.max())
    assert torch.all(got[~live] == 0)


@gpu
def test_ce_kernel_all_ignored_is_nan_with_zero_gradient():
    V, rows = 21128, 128
    lx = torch.randn(rows, vocab_pad(V), device=DEV)
    row_loss, pred, dl, loss, n = _ce(lx, [-1] * rows, rows, V, 100)
    assert n == 0 and torch.isnan(loss)
    assert torch.all(dl.float() == 0) and torch.all(pred == -1) and torch.all(row_loss == 0)


@gpu
def test_compaction_exact():
    torch.manual_seed(1)
    M, V, cap = 4096, 21128, 768
    lab = torch.full((M,), -100, dtype=torch.int64)
    pick = torch.rand(M) < 0.15
    lab[pick] = torch.randint(0, V, (int(pick.sum()),))
    n = int(pick.sum())
    assert n <= cap
    d = lab.to(DEV)
    rows = torch.full((cap,), -7, dtype=torch.int32, device=DEV)
    slot = torch.full((M,), -7, dtype=torch.int32, device=DEV)
    slab = torch.full((cap,), -7, dtype=torch.int32, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    L.call("b2_mlm_compact", d.data_ptr(), M, -100, V, cap, rows.data_ptr(), slot.data_ptr(), slab.data_ptr(),
           cnt.data_ptr(), _stream())
    torch.cuda.synchronize()
    idx = torch.nonzero(pick)[:, 0]
    assert int(cnt) == n
    assert torch.equal(rows[:n].long().cpu(), idx) and torch.all(rows[n:] == 0)
    assert torch.equal(slab[:n].long().cpu(), lab[idx]) and torch.all(slab[n:] == -1)
    ref_slot = torch.full((M,), -1, dtype=torch.int64)
    ref_slot[idx] = torch.arange(n)
    assert torch.equal(slot.long().cpu(), ref_slot)
    # gather and scatter around the compaction
    H = 256
    x = torch.randn(M, H, device=DEV).to(torch.bfloat16)
    g = torch.full((cap, H), float("nan"), dtype=torch.bfloat16, device=DEV)
    L.call("b2_mlm_gather_rows", x.data_ptr(), rows.data_ptr(), cnt.data_ptr(), cap, H, g.data_ptr(), _stream())
    src = torch.randn(cap, H, device=DEV)
    dx = torch.full((M, H), float("nan"), device=DEV)
    L.call("b2_mlm_scatter_rows", src.data_ptr(), slot.data_ptr(), M, H, dx.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert torch.equal(g[:n], x[idx.to(DEV)]) and torch.all(g[n:] == 0)
    ref = torch.zeros(M, H, device=DEV)
    ref[idx.to(DEV)] = src[:n]
    assert torch.equal(dx, ref)


def _grads_vs_oracle(cfg, B, S, seed):
    m, state = _model(cfg)
    batch = b2.synthetic_mlm_batch(cfg, B, S, seed, padded=True)
    d = _to_dev(batch)
    out = m(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
            labels=d["label"])
    out.loss.backward()
    got = m.grad_dict()
    loss_ref, logits_ref, ref = mlm.loss_and_grads(state, cfg, batch)
    return m, out, got, loss_ref, logits_ref, ref, batch


@gpu
@pytest.mark.parametrize("shape", ["tiny", "config_a"])
def test_model_against_oracle(shape):
    if shape == "tiny":
        cfg, B, S = _cfg(**NO_DROP), 4, 128
    else:
        cfg, B, S = b2.chinese_bert_wwm_ext_config(**NO_DROP), 8, 128
    m, out, got, loss_ref, logits_ref, ref, batch = _grads_vs_oracle(cfg, B, S, 3)
    assert abs(float(out.loss) - float(loss_ref)) < TOL_LOSS * max(1.0, float(loss_ref))
    assert out.logits.shape == (B, S, cfg.vocab_size) and out.logits.dtype == torch.float32
    mask = batch["attention_mask"].bool()
    assert float((out.logits.cpu()[mask] - logits_ref[mask]).abs().max()) < 5e-2
    assert_grads_within_tolerance(got, ref, qk_tol=TOL_GRAD_REL_QK)
    # the tied table's pad row: the decoder part alone reaches it
    pr, pg = ref["bert.embeddings.word_embeddings.weight"][0], got["bert.embeddings.word_embeddings.weight"][0].cpu()
    assert float(pr.norm()) > 0
    assert float((pg - pr).norm() / pr.norm()) < 2e-2


@gpu
def test_eager_dense_path_agrees_with_labelled_rows():
    cfg = _cfg(**NO_DROP)
    batch = _to_dev(b2.synthetic_mlm_batch(cfg, 4, 128, 5, padded=True))
    m, _ = _model(cfg)
    out = m(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], labels=batch["label"])
    out.loss.backward()
    g_rows = m.grad_dict()
    # a loss-only backward allocates no dense gradient over every row
    full = [hb for (M, rows, f), hb in m._engine._mlm_ws.items() if f]
    assert full and all(hb["dlog"] is None for hb in full)
    m2, _ = _model(cfg)
    out2 = m2(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"])
    loss2 = nn.CrossEntropyLoss()(out2.logits.reshape(-1, cfg.vocab_size), batch["label"].reshape(-1))
    loss2.backward()
    g_dense = m2.grad_dict()
    assert abs(float(loss2) - float(out.loss)) < 1e-4 * float(out.loss)
    # per tensor within the oracle tolerances (tensors whose norm is negligible, such as the key bias, whose exact
    # gradient is zero, are skipped by the helper's floor)
    assert_grads_within_tolerance({k: v.cpu() for k, v in g_rows.items()}, {k: v.cpu() for k, v in g_dense.items()},
                                  qk_tol=TOL_GRAD_REL_QK)


@gpu
@pytest.mark.parametrize("opt", ["adamw", "adam", "sgd", "adamw_torch"])
def test_vocab_padding_stays_zero(opt):
    cfg = _cfg(**NO_DROP)
    m, _ = _model(cfg)
    params = list(m.parameters())
    o = {"adamw": lambda: b2.AdamW(params, lr=1e-3, weight_decay=0.1),
         "adam": lambda: b2.Adam(params, lr=1e-3, weight_decay=0.1),
         "sgd": lambda: b2.SGD(params, lr=1e-2, momentum=0.9, weight_decay=0.1),
         "adamw_torch": lambda: b2.TorchAdamW(params, lr=1e-3, weight_decay=0.1)}[opt]()
    lay, H, V = m._layout, cfg.hidden_size, cfg.vocab_size
    Vp = lay.vocab_pad
    ow, ob = lay.off("bert.embeddings.word_embeddings.weight"), lay.off("cls.predictions.bias")
    for step in range(5):
        batch = _to_dev(b2.synthetic_mlm_batch(cfg, 2, 128, 20 + step))
        out = m(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], labels=batch["label"])
        out.loss.backward()
        g = m._engine.grads
        assert torch.all(g[ow + V * H:ow + Vp * H] == 0) and torch.all(g[ob + V:ob + Vp] == 0)
        o.step()
        o.zero_grad()
    torch.cuda.synchronize()
    for buf in (m._flat, m._engine.shadow.float()):
        assert torch.all(buf[ow + V * H:ow + Vp * H] == 0) and torch.all(buf[ob + V:ob + Vp] == 0)


def _run_steps(cfg, n=3, seed=9):
    m, _ = _model(cfg, seed)
    o = b2.AdamW(list(m.parameters()), lr=1e-3, weight_decay=0.01)
    m.set_dropout_rng_state(torch.tensor([1234, 0]))
    losses = []
    for step in range(n):
        batch = _to_dev(b2.synthetic_mlm_batch(cfg, 4, 128, 40 + step, padded=True))
        out = m(input_ids=batch["input_ids"], attention_mask=batch["attention_mask"], labels=batch["label"])
        out.loss.backward()
        losses.append(out.loss.detach().clone())
        o.step()
    torch.cuda.synchronize()
    return torch.stack(losses).cpu(), m._flat.clone(), m._engine.grads.clone()


@gpu
def test_determinism_bitwise():
    cfg = _cfg()
    torch.use_deterministic_algorithms(True)
    try:
        a = _run_steps(cfg)
        b = _run_steps(cfg)
    finally:
        torch.use_deterministic_algorithms(False)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@gpu
def test_trajectory_against_oracle():
    """5 eager AdamW steps (dropout off): the losses against the oracle's, with the oracle stepping torch AdamW"""
    cfg = _cfg(**NO_DROP)
    m, state = _model(cfg)
    o = b2.TorchAdamW(list(m.parameters()), lr=1e-4, weight_decay=0.0)
    ref = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    ro = torch.optim.AdamW(list(ref.values()), lr=1e-4, weight_decay=0.0)
    for step in range(5):
        batch = b2.synthetic_mlm_batch(cfg, 4, 128, 60 + step, padded=True)
        d = _to_dev(batch)
        out = m(input_ids=d["input_ids"], attention_mask=d["attention_mask"], labels=d["label"])
        out.loss.backward()
        o.step()
        ro.zero_grad()
        rl, _ = mlm.forward(ref, cfg, batch["input_ids"], None, batch["attention_mask"], batch["label"])
        rl.backward()
        ro.step()
        assert abs(float(out.loss) - float(rl)) < 1e-2 * max(1.0, float(rl)), step


@gpu
def test_trainer_eager_paths_dev_and_test():
    cfg = _cfg()
    for amp, accum, clip, optim in ((False, 1, None, "adamw"), (True, 2, 1.0, "adamw_torch"), (False, 2, 0.5, "sgd")):
        m, _ = _model(cfg)
        args = b2.Args()
        args.fused, args.use_amp, args.gradient_accumulation_steps, args.max_grad_norm = False, amp, accum, clip
        args.optim, args.learning_rate, args.local_rank = optim, 1e-3, 0
        opt = b2.build_optimizer(m, args)
        tr = b2.Trainer(args, cfg, m, None, opt)
        for step in range(4):
            loss = tr.train_step(b2.synthetic_mlm_batch(cfg, 4, 128, 80 + step, padded=True))
            assert torch.isfinite(loss)
        assert tr.global_step == 4 // accum
        assert tr.problem_type(None) == "masked_lm"
    dev = [b2.synthetic_mlm_batch(cfg, 4, 128, 90 + i, padded=True) for i in range(2)]
    loss, acc = tr.dev(dev)
    m.eval()
    ref_loss, correct, total = 0.0, 0, 0
    with torch.no_grad():
        for b in dev:
            d = _to_dev(b)
            out = m(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"])
            lg = out.logits.reshape(-1, cfg.vocab_size).double().cpu()
            lab = b["label"].reshape(-1)
            ref_loss += float(nn.functional.cross_entropy(lg, lab))
            keep = lab != -100
            correct += int((lg.argmax(1)[keep] == lab[keep]).sum())
            total += int(keep.sum())
    assert abs(float(loss) - ref_loss) < 1e-3 * ref_loss
    assert acc == pytest.approx(correct / total, abs=2.0 / total)
    with pytest.raises(ValueError):
        tr.test(m, dev, None)
    args.fused = True
    assert torch.isfinite(b2.Trainer(args, cfg, m, None, opt).train_step(dev[0]))


@gpu
def test_checkpoint_roundtrip(tmp_path):
    cfg = _cfg()
    m, _ = _model(cfg)
    o = b2.AdamW(list(m.parameters()), lr=1e-3)
    batch = _to_dev(b2.synthetic_mlm_batch(cfg, 2, 128, 7))
    m(input_ids=batch["input_ids"], labels=batch["label"]).loss.backward()
    o.step()
    m.save_pretrained(str(tmp_path))
    fresh = b2.BertForMaskedLM.from_pretrained(str(tmp_path), config=cfg).to(DEV)
    for (n, p), (n2, p2) in zip(m.named_parameters(), fresh.named_parameters()):
        assert n == n2 and torch.equal(p, p2), n
    m.eval()
    fresh.eval()
    with torch.no_grad():
        a = m(input_ids=batch["input_ids"], labels=batch["label"])
        b = fresh(input_ids=batch["input_ids"], labels=batch["label"])
    assert torch.equal(a.logits, b.logits) and torch.equal(a.loss, b.loss)


@gpu
def test_labels_must_be_int64_and_present():
    cfg = _cfg(**NO_DROP)
    m, _ = _model(cfg)
    b = _to_dev(b2.synthetic_mlm_batch(cfg, 2, 128, 1))
    for bad in (b["label"].int(), b["label"].to(torch.uint8), b["label"][:, :64]):
        with pytest.raises(TypeError):
            m(input_ids=b["input_ids"], labels=bad)
        with pytest.raises(TypeError):
            m.masked_lm_eval(b["input_ids"], labels=bad)
    with pytest.raises(ValueError, match="labels"):
        m.masked_lm_eval(b["input_ids"])
    with pytest.raises(TypeError):
        m._engine.forward(b["input_ids"], None, None, b["label"].int(), training=False, need_backward=False)
    big = b["label"].clone()
    big[0, 3] = cfg.vocab_size
    with pytest.raises(ValueError):
        m(input_ids=b["input_ids"], labels=big)


@gpu
def test_tied_add_kernel_against_float64():
    """grad = bf16(grad + dec): one fp32 add and one rounding, the pad row and untouched (zero) rows included"""
    torch.manual_seed(2)
    V, H = 1000, 256
    scatter = torch.randn(V, H, device=DEV).to(torch.bfloat16)
    scatter[0] = 0                    # the pad row: no scatter part
    scatter[500:] = 0                 # rows the batch never touched
    dec = torch.randn(V, H, device=DEV) * 1e-2
    g = scatter.clone()
    L.call("b2_mlm_tied_add", dec.data_ptr(), g.data_ptr(), V * H, _stream())
    torch.cuda.synchronize()
    assert torch.equal(g, (scatter.float() + dec).to(torch.bfloat16))
    exact = scatter.double() + dec.double()
    assert torch.all((g.double() - exact).abs() <= 2.0 ** -8 * exact.abs() + 1e-30)
    assert torch.equal(g[0], dec[0].to(torch.bfloat16))


def _trainer(cfg, fused, pack=False, seed=9, **kw):
    m, _ = _model(cfg, seed)
    m.set_dropout_rng_state(torch.tensor([77, 0]))
    args = b2.Args()
    args.fused, args.pack, args.local_rank, args.learning_rate = fused, pack, 0, 1e-4
    for k, v in kw.items():
        setattr(args, k, v)
    return b2.Trainer(args, cfg, m, None, b2.build_optimizer(m, args)), m


def _losses(tr, batches):
    return torch.tensor([float(tr.train_step(b)) for b in batches])


@gpu
@pytest.mark.parametrize("path", ["captured", "packed128", "packed512"])
def test_captured_paths_match_eager(path):
    """5 steps with dropout off on the captured / packed steps against the eager path: losses at every step, and
    AdamW's first moments and the weights at the end"""
    S = 512 if path == "packed512" else 128
    cfg = _cfg(max_position_embeddings=512, **NO_DROP)
    bts = [b2.synthetic_mlm_batch(cfg, 4, S, 100 + i, padded=True) for i in range(5)]
    ref_tr, ref_m = _trainer(cfg, False)
    tr, m = _trainer(cfg, True, pack=path != "captured")
    la, lb = _losses(ref_tr, bts), _losses(tr, bts)
    assert torch.all((la - lb).abs() < 2e-3 * la.abs()), (la, lb)
    if path != "captured":
        assert tr._packed and tr._fused is None
    else:
        assert tr._fused is not None and tr._fused.mlm
    ma, mb = ref_tr.optimizer._state()["exp_avg"], tr.optimizer._state()["exp_avg"]
    assert float((ma - mb).norm() / ma.norm()) < 3e-2
    assert float((ref_m._flat - m._flat).norm() / ref_m._flat.norm()) < 1e-4


@gpu
def test_captured_against_oracle_and_capacity_cache():
    cfg = _cfg(**NO_DROP)
    tr, m = _trainer(cfg, True)
    state = mlm.mlm_state_from_hf_init(cfg, 9)
    ref = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    bts = [b2.synthetic_mlm_batch(cfg, 4, 128, 130 + i, padded=True) for i in range(3)]
    first = tr.train_step(bts[0])
    rl, _ = mlm.forward(ref, cfg, bts[0]["input_ids"], None, bts[0]["attention_mask"], bts[0]["label"])
    assert abs(float(first) - float(rl)) < TOL_LOSS * max(1.0, float(rl))
    # a batch with many more labelled tokens takes a larger capacity: one more graph, no new step object
    dense = dict(bts[1])
    dense["label"] = torch.where(dense["attention_mask"] == 1, dense["input_ids"], torch.full_like(dense["input_ids"],
                                                                                                   -100))
    step = tr._fused
    tr.train_step(bts[1])
    tr.train_step(dense)
    tr.train_step(bts[2])
    assert tr._fused is step
    caps = {role[2] for role in set(step._warm) | set(step._graphs)}   # a role's first two passes run eagerly
    assert len(caps) >= 2 and max(caps) <= 4 * 128 and all(c % 128 == 0 for c in caps)


@gpu
def test_captured_criterion_rules():
    cfg = _cfg()
    m, _ = _model(cfg)
    opt = b2.AdamW(list(m.parameters()), lr=1e-4)
    for bad in (nn.CrossEntropyLoss(label_smoothing=0.1), nn.CrossEntropyLoss(weight=torch.ones(cfg.vocab_size)),
                nn.CrossEntropyLoss(reduction="sum")):
        with pytest.raises(ValueError, match="fused = False"):
            b2.FusedTrainStep(m, opt, 2, 128, criterion=bad)
    for bad in (nn.MSELoss(), nn.BCEWithLogitsLoss()):
        with pytest.raises(ValueError):
            b2.FusedTrainStep(m, opt, 2, 128, criterion=bad)
    st = b2.FusedTrainStep(m, opt, 2, 128, criterion=nn.CrossEntropyLoss(ignore_index=-1))
    b = b2.synthetic_mlm_batch(cfg, 2, 128, 4)
    b["label"][b["label"] == -100] = -1
    assert torch.isfinite(st(b))
    b["label"][0, 5] = cfg.vocab_size
    with pytest.raises(ValueError):
        st(b)


@gpu
@pytest.mark.parametrize("fused", [False, True])
def test_trainer_switches(fused, tmp_path):
    """accumulation, clipping, a linear schedule and each optimizer; full_determinism: two runs bitwise equal"""
    cfg = _cfg()
    bts = [b2.synthetic_mlm_batch(cfg, 4, 128, 150 + i, padded=True) for i in range(4)]
    for optim in ("adamw", "adamw_torch", "sgd"):
        tr, m = _trainer(cfg, fused, optim=optim, gradient_accumulation_steps=2, max_grad_norm=0.5,
                         lr_scheduler_type="linear")
        tr.create_scheduler(4)
        losses = _losses(tr, bts)
        assert torch.all(torch.isfinite(losses)) and tr.global_step == 2
        assert tr.last_grad_norm is not None and float(tr.last_grad_norm) > 0
        assert tr.optimizer.param_groups[0]["lr"] < 1e-4
    runs = []
    for _ in range(2):
        tr, m = _trainer(cfg, fused, full_determinism=True)
        try:
            runs.append((_losses(tr, bts), m._flat.clone()))
        finally:
            torch.use_deterministic_algorithms(False)
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


@gpu
@pytest.mark.parametrize("fused", [False, True])
def test_trainer_save_and_resume(fused, tmp_path):
    """2 steps, checkpoint, 2 steps; a fresh model from a different init resumed from the checkpoint repeats the last
    2 steps bitwise (dropout on)"""
    cfg = _cfg()
    bts = [b2.synthetic_mlm_batch(cfg, 4, 128, 170 + i, padded=True) for i in range(4)]
    tr, m = _trainer(cfg, fused)
    _losses(tr, bts[:2])
    tr.save_checkpoint(str(tmp_path / "ck"))
    tail = _losses(tr, bts[2:])
    tr2, m2 = _trainer(cfg, fused, seed=31)
    tr2.load_checkpoint(str(tmp_path / "ck"))
    tail2 = _losses(tr2, bts[2:])
    assert torch.equal(tail, tail2)
    assert torch.equal(m._flat, m2._flat)


@gpu
def test_dev_fused_equals_eager():
    cfg = _cfg()
    dev = [b2.synthetic_mlm_batch(cfg, 4, 128, 190 + i, padded=True) for i in range(2)]
    tr_f, m = _trainer(cfg, True)
    lf, af = tr_f.dev(dev)
    assert tr_f._fused_eval
    tr_f.args.fused = False
    le, ae = tr_f.dev(dev)
    assert abs(float(lf) - float(le)) < 1e-6 * abs(float(le)) and af == ae
    tr_f.criterion = nn.CrossEntropyLoss(label_smoothing=0.1)
    with pytest.raises(ValueError):
        tr_f.dev(dev)


@gpu
@pytest.mark.parametrize("world", [1, 2])
def test_ddp_mlm_worker(world):
    """tests/ddp_mlm_worker.py on `world` ranks: eager, captured and packed against the oracle's DDP mean"""
    import os
    import subprocess
    import sys
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", str(29627 + world),
           os.path.join(root, "tests", "ddp_mlm_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_mlm_worker: OK (world %d)" % world in r.stdout
