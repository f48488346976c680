"""GPU: BertForMultipleChoice -- the model against the multiple-choice oracle (tests/mc_oracle.py) padded and packed,
its bitwise identity with a one-label sequence model on the flattened rows, the captured step's launch count, every
training path through the Trainer, fixed-order determinism, checkpoints, dev() / test(), and the model in a loopback
DistributedDataParallel group.  The head is the sequence head's kernels with one label and the loss the existing
cross-entropy over [B, N], so the model is held to the sequence model's tolerances (tests/parity.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

import loopback as lb
import mc_oracle as mc
from parity import (TOL_LOGITS, TOL_LOSS, TOL_TRAJ, adamw_ref, assert_grads_within_tolerance, b2, oracle_masks,
                    tiny_config)
from pytorch_distributed_nlp_b200 import _lib as L
from test_checkpoint import _groups

gpu = pytest.mark.gpu
NO_DROP = dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
LR = 1e-4
# The choice loss's d_logits sum to zero over each example's N choices, so the gradient it sends into the encoder -- a
# sum over rows of terms that nearly cancel between the choices of an example, which at HF's init differ little -- is
# about 1/1000 of the same sum taken without the cancellation (tiny config, CPU oracle), while bf16 rounding acts on
# the summands.  With dropout off, the per-tensor relative error of that gradient measures the cancellation, not the
# kernels (0.1 to 0.9 on an H100).  The gradients are therefore held to the sequence model's tolerances where the
# cancellation does not dominate: with dropout on (the masks differ between choices), and for an objective that adds
# a non-cancelling function of the logits to the loss.  With dropout off, the multiple-choice gradients are bit for
# bit the one-label sequence model's on the flattened rows (test_logits_and_gradients_equal_...).


def _user(loss, logits):
    """the loss plus a function of the logits whose gradient does not cancel between an example's choices: positive
    weights, each example's summing to N / B"""
    w = torch.linspace(0.5, 1.5, logits.shape[1], device=logits.device)
    return loss + (logits * w).sum() / logits.shape[0]


def _model(cfg, state, dev, cls=None):
    m = (cls or b2.BertForMultipleChoice)(cfg)
    m.load_state_dict(state, strict=True)
    return m.to(dev)


def _dev_batch(b, dev):
    return {k: v.to(dev) for k, v in b.items()}


def _call(model, d, labels=True):
    return model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                 labels=d["label"] if labels else None)


def _packed_call(model, p, labels, dev):
    dv = lambda k: p[k].to(dev)
    return model(input_ids=dv("input_ids"), token_type_ids=dv("token_type_ids"), position_ids=dv("position_ids"),
                 segments=dv("segments"), cls_index=dv("cls_index"), labels=None if labels is None else labels.to(dev))


# ---- the model against the oracle ---------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dropout", [False, True])
@pytest.mark.parametrize("size", ["tiny", "configA"])
def test_model_matches_oracle(cuda_dev, size, dropout):
    """B = 8 examples of N = 4 choices: config A's 32 rows of 128 tokens"""
    mk = tiny_config if size == "tiny" else b2.chinese_bert_wwm_ext_config
    cfg = mk(num_labels=6, **({} if dropout else NO_DROP))
    B, N, S = 8, 4, 128
    state = mc.mc_state_from_hf_init(cfg)
    model = _model(cfg, state, cuda_dev).train()
    seed = 4242
    model._engine.seed_dropout(seed, 0)
    b = b2.synthetic_mc_batch(cfg, B, N, S, 1000, padded=True)
    b["label"][3] = -100
    out = _call(model, _dev_batch(b, cuda_dev))
    assert out.logits.shape == (B, N) and out.logits.dtype == torch.float32 and len(out) == 2
    out.loss.backward()
    torch.cuda.synchronize()
    masks = oracle_masks(cfg, B * N, S, seed, 0) if dropout else None
    rl, rlog, rg = mc.loss_and_grads(state, cfg, b, masks=masks)
    assert abs(float(out.loss.detach()) - float(rl)) <= TOL_LOSS
    assert float((out.logits.detach().cpu() - rlog).abs().max()) <= TOL_LOGITS
    if dropout:        # (dropout off: see the note on the choice loss's cancellation above)
        assert_grads_within_tolerance(model.grad_dict(), rg)
    own = nn.CrossEntropyLoss()(out.logits.detach().cpu(), b["label"])
    assert abs(float(own) - float(out.loss)) <= 1e-5


@gpu
@pytest.mark.parametrize("which", ["logits", "loss_and_logits"])
def test_backward_from_the_logits(cuda_dev, which):
    cfg = tiny_config(**NO_DROP)
    state = mc.mc_state_from_hf_init(cfg)
    model = _model(cfg, state, cuda_dev).train()
    b = b2.synthetic_mc_batch(cfg, 8, 4, 128, 17, padded=True)
    w_host = torch.linspace(-1, 1, 4)
    user = lambda loss, logits: (logits * w_host.to(logits.device)).square().mean() + (loss if which != "logits" else 0)
    out = _call(model, _dev_batch(b, cuda_dev))
    user(out.loss, out.logits).backward()
    torch.cuda.synchronize()
    leaf = {k: v.detach().clone().requires_grad_(True) for k, v in state.items()}
    rl, rlog = mc.forward(leaf, cfg, b["input_ids"], b["token_type_ids"], b["attention_mask"], b["label"])
    user(rl, rlog).backward()
    assert_grads_within_tolerance(model.grad_dict(), {k: v.grad for k, v in leaf.items()})


@gpu
def test_eval_forward_and_argument_errors(cuda_dev):
    cfg = tiny_config(**NO_DROP)
    model = b2.BertForMultipleChoice.from_config(cfg, seed=2).to(cuda_dev)
    d = _dev_batch(b2.synthetic_mc_batch(cfg, 2, 3, 128, 1), cuda_dev)
    with pytest.raises(ValueError, match=r"\[batch, num_choices, seq\]"):
        model(input_ids=d["input_ids"][:, 0])
    with pytest.raises(ValueError, match=r"must be \[2\]"):
        model(input_ids=d["input_ids"], labels=d["label"][:, None])
    model.eval()
    with torch.no_grad():
        out = model(input_ids=d["input_ids"], attention_mask=d["attention_mask"])
        assert len(out) == 1 and out.loss is None and out.logits.shape == (2, 3)
        out = _call(model, d)
    assert out.loss.dim() == 0 and len(out) == 2
    assert getattr(cfg, "problem_type", None) is None


@gpu
@pytest.mark.parametrize("packed", [False, True])
def test_logits_and_gradients_equal_a_one_label_sequence_model_bitwise(cuda_dev, packed):
    """dropout off, the same weights: the multiple-choice logits on [B, N, S] are bit for bit a num_labels = 1
    sequence model's on the flattened [B·N, S], and (fixed-order backward) so are the gradients of the same function
    of those logits"""
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=1, **NO_DROP)
    state = mc.mc_state_from_hf_init(cfg)
    b = b2.synthetic_mc_batch(cfg, 8, 4, 128, 5, padded=True)
    flat = {k: v.reshape(32, 128) for k, v in b.items() if k != "label"}
    w = torch.linspace(-1, 1, 32, device=cuda_dev)
    got = {}
    torch.use_deterministic_algorithms(True)      # the bias-gradient accumulators are atomic otherwise
    try:
        for kind, cls, batch in (("mc", b2.BertForMultipleChoice, b), ("seq", b2.BertForSequenceClassification,
                                                                        flat)):
            model = _model(cfg, state, cuda_dev, cls).train()
            if packed:
                p = b2.pack_batch(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"], 128)
                logits = _packed_call(model, p, None, cuda_dev).logits
            else:
                logits = _call(model, _dev_batch(batch, cuda_dev), labels=False).logits
            (logits.reshape(-1) * w).square().sum().backward()
            torch.cuda.synchronize()
            got[kind] = (logits.detach().reshape(-1).clone(), model._engine.grads.view(torch.int16).clone())
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(got["mc"][0].view(torch.int32), got["seq"][0].view(torch.int32))
    assert torch.equal(got["mc"][1], got["seq"][1])


@gpu
@pytest.mark.parametrize("seq", [128, 256])
def test_packed_model_matches_oracle_and_padded(cuda_dev, seq):
    """packed forward and backward (of the loss plus a non-cancelling function of the logits) against the oracle,
    and the packed logits against the padded ones"""
    cfg = tiny_config(max_position_embeddings=512, **NO_DROP)
    state = mc.mc_state_from_hf_init(cfg)
    b = b2.synthetic_mc_batch(cfg, 6, 4, seq, 21, padded=True)
    p = b2.pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], seq, labels=b["label"])
    assert p["cls_index"].shape == (6, 4) and p["bins"] < 24
    model = _model(cfg, state, cuda_dev).train()
    pk = _packed_call(model, p, p["labels"], cuda_dev)
    assert pk.logits.shape == (6, 4)
    _user(pk.loss, pk.logits).backward()
    torch.cuda.synchronize()
    leaf = {k: v.detach().clone().requires_grad_(True) for k, v in state.items()}
    rl, rlog = mc.forward(leaf, cfg, b["input_ids"], b["token_type_ids"], b["attention_mask"], b["label"])
    _user(rl, rlog).backward()
    assert abs(float(pk.loss.detach()) - float(rl)) <= TOL_LOSS
    assert float((pk.logits.detach().cpu() - rlog.detach()).abs().max()) <= TOL_LOGITS
    assert_grads_within_tolerance(model.grad_dict(), {k: v.grad for k, v in leaf.items()})
    padded = _model(cfg, state, cuda_dev).eval()
    with torch.no_grad():
        pd = _call(padded, _dev_batch(b, cuda_dev))
    assert float((pk.logits.detach() - pd.logits).abs().max()) <= TOL_LOGITS
    assert abs(float(pk.loss) - float(pd.loss)) <= TOL_LOSS


@gpu
def test_captured_step_launches_as_many_kernels_as_the_sequence_step(cuda_dev):
    """the captured multiple-choice step at B = 8, N = 4 issues exactly the library launches of the captured sequence
    step on the flattened 32 rows (both run their bodies without a graph here, so every launch is counted)"""
    cfg = tiny_config(num_labels=4, **NO_DROP)
    counts = {}
    b = b2.synthetic_mc_batch(cfg, 8, 4, 128, 9, padded=True)
    flat = {k: v.reshape(32, 128) for k, v in b.items() if k != "label"}
    flat["label"] = torch.randint(0, 4, (32,))
    for kind in ("mc", "seq"):
        cls = b2.BertForMultipleChoice if kind == "mc" else b2.BertForSequenceClassification
        model = cls.from_config(cfg, seed=3).to(cuda_dev).train()
        opt = b2.build_optimizer(model, type("A", (), {"weight_decay": 0.01, "learning_rate": LR}))
        if kind == "mc":
            step = b2.FusedTrainStep(model, opt, 8, 128, use_graph=False, choices=4)
            batch = b
        else:
            step = b2.FusedTrainStep(model, opt, 32, 128, use_graph=False)
            batch = flat
        step(batch)
        torch.cuda.synchronize()
        before = L.launch_count()
        step(batch)
        torch.cuda.synchronize()
        counts[kind] = L.launch_count() - before
    assert counts["mc"] == counts["seq"] and counts["mc"] > 0, counts


@gpu
def test_captured_steps_reject_batches_that_do_not_fit(cuda_dev):
    cfg = tiny_config(**NO_DROP)
    model = b2.BertForMultipleChoice.from_config(cfg, seed=3).to(cuda_dev).train()
    opt = b2.build_optimizer(model, type("A", (), {"weight_decay": 0.01, "learning_rate": LR}))
    with pytest.raises(ValueError, match="choices=N"):
        b2.FusedTrainStep(model, opt, 8, 128)
    step = b2.FusedTrainStep(model, opt, 2, 128, choices=4)
    with pytest.raises(ValueError, match="2x4x128"):
        step(b2.synthetic_mc_batch(cfg, 2, 3, 128, 1))
    bad = b2.synthetic_mc_batch(cfg, 2, 4, 128, 1)
    bad["label"][0] = 4
    with pytest.raises(ValueError, match="choice label 4 is outside"):
        step(bad)
    with pytest.raises(ValueError, match="MSELoss does not apply"):
        b2.FusedTrainStep(model, opt, 2, 128, choices=4, criterion=nn.MSELoss())
    b = b2.synthetic_mc_batch(cfg, 2, 4, 128, 1, padded=True)
    p = b2.pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], 128)
    pstep = b2.PackedTrainStep(model, opt, p["bins"], 2, choices=4)
    with pytest.raises(ValueError, match="PackedTrainStep was built for"):
        pstep(p, torch.zeros(3, dtype=torch.int64))


# ---- training paths: 5-step trajectories against the oracle ----------------------------------------------------------------
STEPS = 5
_REF = {}


def _ref_trajectory(criterion_name):
    if criterion_name in _REF:
        return _REF[criterion_name]
    cfg = tiny_config(**NO_DROP)
    state = mc.mc_state_from_hf_init(cfg)
    batches = [b2.synthetic_mc_batch(cfg, 4, 4, 128, 500 + i, padded=True) for i in range(STEPS)]
    batches[1]["label"][2] = -100
    crit = _CRITERIA[criterion_name]()
    ref = {n: v.clone() for n, v in state.items()}
    opt = adamw_ref.HFAdamW(ref, lr=LR, weight_decay=0.01)
    losses = []
    for bt in batches:
        l, _lg, gr = mc.loss_and_grads(ref, cfg, bt, criterion=crit)
        losses.append(float(l))
        opt.step(gr)
    _REF[criterion_name] = (cfg, state, batches, losses)
    return _REF[criterion_name]


def _args(**kw):
    a = b2.Args()
    a.local_rank, a.epochs, a.weight_decay, a.learning_rate = 0, 1, 0.01, LR
    for k_, v in kw.items():
        setattr(a, k_, v)
    return a


_PATHS = {"eager": dict(fused=False), "amp": dict(fused=False, use_amp=True), "fused": dict(fused=True),
          "packed": dict(fused=True, pack=True)}
_CRITERIA = {"none": lambda: None,
             "ce_options": lambda: nn.CrossEntropyLoss(weight=torch.tensor([0.5, 1.0, 1.5, 2.0]), label_smoothing=0.1)}


@gpu
@pytest.mark.parametrize("criterion", sorted(_CRITERIA))
@pytest.mark.parametrize("path", sorted(_PATHS))
def test_trajectories_match_oracle(cuda_dev, path, criterion):
    cfg, state, batches, rlosses = _ref_trajectory(criterion)
    model = _model(cfg, state, cuda_dev).train()
    args = _args(**_PATHS[path])
    opt = b2.build_optimizer(model, args)
    crit = _CRITERIA[criterion]()
    tr = b2.Trainer(args, cfg, model, None if crit is None else crit.to(cuda_dev), opt)
    losses = [float(tr.train_step(bt)) for bt in batches]
    torch.cuda.synchronize()
    assert max(abs(a - b_) for a, b_ in zip(losses, rlosses)) <= TOL_TRAJ, (losses, rlosses)
    if path == "packed":
        assert len(tr._packed) > 0 and all(k[-1] == 4 for k in tr._packed)
    if path == "fused":
        assert tr._fused.batch_shape == (4, 4, 128)


@gpu
@pytest.mark.parametrize("path", ["eager", "fused", "packed"])
def test_accumulation_of_two_matches_one_batch_of_twice_the_size(cuda_dev, path):
    """k = 2 over two batches of 4 examples against one step on their 8 examples (each half's loss is a mean over
    the same number of labelled examples, so the mean of the two means is the mean over all 8)"""
    cfg = tiny_config(**NO_DROP)
    state = mc.mc_state_from_hf_init(cfg)
    halves = [b2.synthetic_mc_batch(cfg, 4, 4, 128, 60 + i, padded=True) for i in range(2)]
    whole = {k: torch.cat([h[k] for h in halves]) for k in halves[0]}
    weights = []
    for k, batches in ((2, halves), (1, [whole])):
        model = _model(cfg, state, cuda_dev).train()
        args = _args(fused=path != "eager", pack=path == "packed", gradient_accumulation_steps=k)
        tr = b2.Trainer(args, cfg, model, None, b2.build_optimizer(model, args))
        for bt in batches:
            tr.train_step(bt)
        torch.cuda.synchronize()
        assert tr.global_step == 1
        weights.append(model._flat.detach().clone())
    assert float((weights[0] - weights[1]).abs().max()) <= 2e-5


@gpu
@pytest.mark.parametrize("optim", ["adamw", "sgd", "adamw_torch", "adamw_torch_fused"])
def test_trainer_switches_agree_with_eager(cuda_dev, optim):
    """accumulation (k = 2), clipping and a linear schedule on every optimizer: the captured and packed paths against
    eager, in the losses, the pre-clip gradient norms and the weights"""
    cfg = tiny_config(**NO_DROP)
    state = mc.mc_state_from_hf_init(cfg)
    batches = [b2.synthetic_mc_batch(cfg, 4, 4, 128, 300 + i, padded=True) for i in range(6)]
    runs = {}
    for path in ("eager", "fused", "packed"):
        model = _model(cfg, state, cuda_dev).train()
        args = _args(fused=path != "eager", pack=path == "packed", gradient_accumulation_steps=2, max_grad_norm=0.5,
                     lr_scheduler_type="linear", optim=optim, learning_rate=1e-3 if optim == "sgd" else LR)
        opt = b2.build_optimizer(model, args)
        tr = b2.Trainer(args, cfg, model, None, opt)
        tr.create_scheduler(3)
        losses, norms = [], []
        for bt in batches:
            losses.append(float(tr.train_step(bt)))
            if tr._micro == 0:
                norms.append(float(tr.last_grad_norm))
        torch.cuda.synchronize()
        runs[path] = (losses, norms, model._flat.detach().clone())
    el, en, ew = runs["eager"]
    for path in ("fused", "packed"):
        l, n, w = runs[path]
        assert max(abs(a - b_) for a, b_ in zip(l, el)) <= TOL_TRAJ, (path, l, el)
        assert all(abs(a - b_) <= 2e-2 * b_ for a, b_ in zip(n, en)), (path, n, en)
        assert len(n) == 3 and all(np.isfinite(n))
        assert float((w - ew).abs().max()) <= 5e-3, path


@gpu
@pytest.mark.parametrize("sched", ["cosine", "constant", "constant_with_warmup"])
def test_lr_schedules_on_the_captured_step(cuda_dev, sched):
    """every lr_scheduler_type: the captured step follows eager"""
    cfg = tiny_config(**NO_DROP)
    state = mc.mc_state_from_hf_init(cfg)
    batches = [b2.synthetic_mc_batch(cfg, 4, 4, 128, 800 + i, padded=True) for i in range(4)]
    ws = []
    for fused in (False, True):
        model = _model(cfg, state, cuda_dev).train()
        args = _args(fused=fused, lr_scheduler_type=sched, warmup_steps=1, learning_rate=1e-3)
        tr = b2.Trainer(args, cfg, model, None, b2.build_optimizer(model, args))
        tr.create_scheduler(4)
        for bt in batches:
            tr.train_step(bt)
        torch.cuda.synchronize()
        ws.append(model._flat.detach().clone())
    assert float((ws[0] - ws[1]).abs().max()) <= 5e-3


def _det_run(cfg, state, batches, pack, cuda_dev):
    model = _model(cfg, state, cuda_dev).train()
    model._engine.seed_dropout(77, 0)
    args = _args(fused=True, pack=pack, full_determinism=True)
    opt = b2.build_optimizer(model, args)
    tr = b2.Trainer(args, cfg, model, None, opt)
    losses = [tr.train_step(bt).clone() for bt in batches]
    torch.cuda.synchronize()
    return torch.stack(losses), model._engine.grads.clone(), model._flat.detach().clone()


@gpu
@pytest.mark.parametrize("pack", [False, True])
def test_two_deterministic_runs_are_bitwise_identical(cuda_dev, pack):
    cfg = tiny_config()   # dropout on
    state = mc.mc_state_from_hf_init(cfg)
    batches = [b2.synthetic_mc_batch(cfg, 4, 4, 128, 40 + i, padded=True) for i in range(3)]
    try:
        a = _det_run(cfg, state, batches, pack, cuda_dev)
        b_ = _det_run(cfg, state, batches, pack, cuda_dev)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(a[0], b_[0]) and torch.equal(a[1].view(torch.int16), b_[1].view(torch.int16))
    assert torch.equal(a[2], b_[2])


# ---- checkpoints ------------------------------------------------------------------------------------------------------------
def _ckpt_run(cuda_dev, cfg, state, batches, tmp, resume=None):
    """deterministic, dropout on, the captured step, k = 2, max_grad_norm, a linear schedule, save_steps = 2"""
    model = _model(cfg, state, cuda_dev).train()
    model.set_dropout_rng_state(torch.tensor([5, 0]))
    opt = b2.AdamW(_groups(model.named_parameters()), lr=2e-4)
    a = _args(fused=True, gradient_accumulation_steps=2, max_grad_norm=1.0, lr_scheduler_type="linear",
              output_dir=str(tmp), save_steps=2, log_every=1000, dev=False, full_determinism=True,
              ckpt_path=os.path.join(str(tmp), "final.pt"))
    tr = b2.Trainer(a, cfg, model, None, opt)
    losses = []
    step = tr.train_step
    tr.train_step = lambda bt: losses.append(step(bt).clone()) or losses[-1]
    tr.train(batches, resume_from_checkpoint=resume)
    torch.cuda.synchronize()
    return losses, model._flat.detach().clone(), tr


@gpu
def test_checkpoint_resume_equals_the_uninterrupted_run_bitwise(cuda_dev, tmp_path):
    cfg = tiny_config()
    state = mc.mc_state_from_hf_init(cfg)
    batches = [b2.synthetic_mc_batch(cfg, 4, 4, 128, 9000 + i, padded=True) for i in range(8)]
    try:
        losses, w_full, tr = _ckpt_run(cuda_dev, cfg, state, batches, tmp_path / "full")
        assert tr.global_step == 4
        ck = str(tmp_path / "full" / "checkpoint-2")
        back = b2.BertForMultipleChoice.from_pretrained(ck)
        saved = torch.load(os.path.join(ck, "pytorch_model.bin"))
        for k, v in back.state_dict().items():
            assert torch.equal(v, saved[k]), k
        resumed, w_res, tr2 = _ckpt_run(cuda_dev, cfg, mc.mc_state_from_hf_init(cfg, seed=9), batches,
                                        tmp_path / "res", resume=ck)
    finally:
        torch.use_deterministic_algorithms(False)
    assert len(resumed) == 4 and tr2.global_step == 4
    assert torch.equal(torch.stack(losses[4:]), torch.stack(resumed))
    assert torch.equal(w_full, w_res)


# ---- dev() / test() ---------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("fused", [False, True])
def test_dev_and_test_on_a_known_batch(cuda_dev, fused):
    """the choice accuracy over the labels that are not ignored, and the classification report over the choice
    index, against a host recomputation from the model's own logits"""
    from sklearn.metrics import classification_report
    cfg = tiny_config(**NO_DROP)
    model = b2.BertForMultipleChoice.from_config(cfg, seed=8).to(cuda_dev)
    args = _args(fused=fused)
    tr = b2.Trainer(args, cfg, model, None, b2.build_optimizer(model, args))
    loader = [b2.synthetic_mc_batch(cfg, 6, 4, 128, 70 + i, padded=True) for i in range(3)]
    loader[1]["label"][0] = -100
    model.eval()
    logits, labels, want_loss = [], [], 0.0
    for bt in loader:
        with torch.no_grad():
            o = _call(model, _dev_batch(bt, cuda_dev))
        logits.append(o.logits.cpu())
        labels.append(bt["label"])
        want_loss += float(o.loss)
    pred, lab = torch.cat(logits).argmax(1), torch.cat(labels)
    keep = lab != -100
    want_acc = float((pred[keep] == lab[keep]).double().mean())
    loss, acc = tr.dev(loader)
    assert abs(float(loss) - want_loss) <= 1e-5 * max(1.0, want_loss)
    assert acc == pytest.approx(want_acc, abs=1e-12)
    names = ["A", "B", "C", "D"]
    got = tr.test(model, loader, names)
    assert got == classification_report(lab[keep].tolist(), pred[keep].tolist(), target_names=names)


# ---- DistributedDataParallel: a loopback group on one GPU, and the real worker ------------------------------------------
@pytest.fixture
def deterministic():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(prev)


@gpu
@pytest.mark.parametrize("dma", ["0", "1"])
def test_loopback_ddp_world2_matches_the_one_gpu_mean(cuda_dev, monkeypatch, deterministic, dma):
    """two loopback replicas (tests/loopback.py) with different batches, dropout off, in the kernel and the
    copy-engine exchange form: loss_reduce is the rank mean, and the final masters are within 2e-4 of one GPU stepping
    on the mean of the two ranks' gradients (the oracle's HF AdamW).  (output_reduce's gather of the [B, N] logits runs
    in tests/ddp_mc_worker.py: the loopback has no eval gathers.)"""
    monkeypatch.setenv("B2_DDP_DMA", dma)
    cfg = tiny_config(**NO_DROP)
    state = mc.mc_state_from_hf_init(cfg)
    world, steps = 2, 3
    batches = [[b2.synthetic_mc_batch(cfg, 4, 4, 128, 7000 + 10 * s + r, padded=True) for r in range(world)]
               for s in range(steps)]
    ref = {k: v.clone() for k, v in state.items()}
    opt_ref = adamw_ref.HFAdamW(ref, lr=3e-5, weight_decay=0.01)
    ref_means = []
    for rank_batches in batches:
        out = [mc.loss_and_grads(ref, cfg, bt) for bt in rank_batches]
        ref_means.append(float(torch.stack([o[0] for o in out]).mean()))
        opt_ref.step({k: sum(o[2][k] for o in out) / world for k in ref})
    build = lambda m: b2.build_optimizer(m, type("A", (), {"weight_decay": 0.01, "learning_rate": 3e-5}))
    dev = torch.device("cuda", 0)
    with lb.Group(world) as g:
        models = [_model(cfg, state, dev).train() for _ in range(world)]
        wrappers, opts = g.wrap(models, build)
        for s in range(steps):
            losses = []
            for r in range(world):
                g.fake.local.rank = g.driving = r
                out = _call(wrappers[r], _dev_batch(batches[s][r], dev))
                out.loss.backward()
                losses.append(out.loss.detach())
            torch.cuda.synchronize()
            mean = g.run(lambda r: wrappers[r].loss_reduce(losses[r]).cpu())
            want = lb.rank_mean([x.cpu() for x in losses])
            assert all(float(v) == float(want) for v in mean)
            assert abs(float(want) - ref_means[s]) <= TOL_TRAJ
            g.step(opts)
        sd = {k: v.clone() for k, v in models[0].state_dict().items()}
        g.close()
    for k, v in ref.items():
        assert float((sd[k].cpu() - v).abs().max()) <= 2e-4, k


@gpu
def test_ddp_mc_worker_world2():
    """tests/ddp_mc_worker.py on two ranks: eager, captured and packed, in both exchange forms, against the oracle's
    DDP mean"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29643", os.path.join(root, "tests", "ddp_mc_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_mc_worker: OK (world 2)" in r.stdout
