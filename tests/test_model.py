"""Whole-step parity of the CUDA path (through the reference-facing Python surface) against the fp32 oracle (GPU)."""
import os

import pytest
import torch
import torch.nn.functional as F

from parity import (TOL_GRAD_REL, TOL_GRAD_REL_QK, TOL_LOGITS, TOL_LOSS, TOL_TRAJ, adamw_ref, assert_grads_within_tolerance, b2, bert_ref,
                    full_config, grad_report, grad_tol, make_model, oracle_masks, report, state_from_hf_init,
                    tiny_config, to_dev)

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _fwd_bwd(model, batch, dev):
    d = to_dev(batch, dev)
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    loss = F.cross_entropy(out[1], d["label"])      # the reference's criterion(logits, label) [:169]
    loss.backward()
    torch.cuda.synchronize()
    return out, loss


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("dropout", [False, True])
def test_tiny_step_matches_oracle(cuda_dev, padded, dropout):
    cfg = tiny_config() if dropout else tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev).train()
    model._engine.seed_dropout(99, 7)
    batch = bert_ref.synthetic_batch(cfg, 4, 128, 1000, padded=padded)
    out, loss = _fwd_bwd(model, batch, cuda_dev)
    masks = oracle_masks(cfg, 4, 128, 99, 7) if dropout else None
    rl, rz, rg = bert_ref.loss_and_grads(state, cfg, batch, masks=masks)
    assert abs(float(loss) - float(rl)) <= TOL_LOSS
    assert abs(float(out[0]) - float(rl)) <= TOL_LOSS            # HF's in-model loss == criterion loss
    assert float((out[1].detach().cpu() - rz).abs().max()) <= TOL_LOGITS
    worst, rows = grad_report(model.grad_dict(), rg)
    assert worst <= TOL_GRAD_REL, sorted(rows, key=lambda r: -r[1])[:5]


@pytest.mark.parametrize("dropout", [False, True])
def test_tiny_step_with_all_padding_sample_matches_oracle(cuda_dev, dropout):
    """one sample of the padded batch is all padding (attention_mask all zeros): HF gives its query rows a uniform
    softmax over the keys, so its value / query / key gradients are not zero and must reach the weights"""
    cfg = tiny_config() if dropout else tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev).train()
    model._engine.seed_dropout(99, 7)
    batch = bert_ref.synthetic_batch(cfg, 4, 128, 1000, padded=True)
    batch["input_ids"][2] = 0
    batch["attention_mask"][2] = 0
    out, loss = _fwd_bwd(model, batch, cuda_dev)
    masks = oracle_masks(cfg, 4, 128, 99, 7) if dropout else None
    rl, rz, rg = bert_ref.loss_and_grads(state, cfg, batch, masks=masks)
    assert abs(float(loss) - float(rl)) <= TOL_LOSS
    assert float((out[1].detach().cpu() - rz).abs().max()) <= TOL_LOGITS
    worst, rows = grad_report(model.grad_dict(), rg)
    assert worst <= TOL_GRAD_REL, sorted(rows, key=lambda r: -r[1])[:5]


@pytest.mark.parametrize("name,cfg_kw,batch,seq", [
    # BASELINE.json config B (bert-base, seq 512): the multi-block attention paths (online softmax rescale forward,
    # dQ accumulation across key blocks backward) and the padded tail blocks, at 2 layers
    ("config-B-shape", dict(vocab_size=2000, hidden_size=768, num_hidden_layers=2, num_attention_heads=12,
                            intermediate_size=3072, max_position_embeddings=512), 2, 512),
    # BASELINE.json config C (bert-large widths: H 1024, 16 heads, I 4096), at 2 layers
    ("config-C-shape", dict(vocab_size=2000, hidden_size=1024, num_hidden_layers=2, num_attention_heads=16,
                            intermediate_size=4096, max_position_embeddings=512), 4, 128),
    ("seq-256", dict(max_position_embeddings=256), 3, 256),
])
@pytest.mark.parametrize("dropout", [False, True])
def test_other_baseline_shapes_match_oracle(cuda_dev, name, cfg_kw, batch, seq, dropout):
    kw = dict(cfg_kw)
    if not dropout:
        kw.update(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    cfg = tiny_config(**kw)
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev).train()
    model._engine.seed_dropout(31, 2)
    b = bert_ref.synthetic_batch(cfg, batch, seq, 4242, padded=True)
    out, loss = _fwd_bwd(model, b, cuda_dev)
    masks = oracle_masks(cfg, batch, seq, 31, 2) if dropout else None
    rl, rz, rg = bert_ref.loss_and_grads(state, cfg, b, masks=masks)
    assert abs(float(loss) - float(rl)) <= TOL_LOSS
    assert float((out[1].detach().cpu() - rz).abs().max()) <= TOL_LOGITS
    # 2e-2; query / key projections of the long-sequence / wide parity shapes 4e-2 (parity.TOL_GRAD_REL_QK)
    qk, other = assert_grads_within_tolerance(model.grad_dict(), rg, qk_tol=TOL_GRAD_REL_QK)
    report("shape_grads", {"name": name, "dropout": dropout, "worst_qk": qk, "worst_other": other})


def test_eval_forward_and_output_surface(cuda_dev):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev).eval()
    batch = bert_ref.synthetic_batch(cfg, 4, 128, 5, padded=True)
    d = to_dev(batch, cuda_dev)
    with torch.no_grad():
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                    labels=d["label"])
        out2 = model(input_ids=d["input_ids"], attention_mask=d["attention_mask"])
    rl, rz = bert_ref.forward(state, cfg, batch["input_ids"], batch["token_type_ids"], batch["attention_mask"],
                              batch["label"])
    assert len(out) == 2 and out[1] is out.logits and out[0] is out.loss
    assert len(out2) == 1 and out2[0] is out2.logits
    assert float((out.logits.cpu() - rz).abs().max()) <= TOL_LOGITS
    assert abs(float(out.loss) - float(rl)) <= TOL_LOSS
    assert float((out2.logits - out.logits).abs().max()) == 0.0   # token_type_ids=None == zeros
    with pytest.raises(ValueError, match="multiples of 128"):
        model(input_ids=d["input_ids"][:, :100])
    with pytest.raises(TypeError, match="int64"):
        model(input_ids=d["input_ids"].int())


def test_tiny_trajectory_eager_and_fused(cuda_dev):
    """5 optimizer steps (dropout off): reference-style eager loop, the fused CUDA-graph step, and the oracle agree."""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    batches = [bert_ref.synthetic_batch(cfg, 4, 128, 2000 + i, padded=(i % 2 == 1)) for i in range(5)]

    class A:
        weight_decay, learning_rate = 0.01, 3e-5

    ref_params = {k: v.clone() for k, v in state.items()}
    hist = __import__("oracle.ddp_ref", fromlist=["train"]).train(ref_params, cfg, [[b] for b in batches])

    # eager, reference-shaped loop
    model = make_model(cfg, state, cuda_dev).train()
    opt = b2.build_optimizer(model, A)
    losses = []
    for b in batches:
        d = to_dev(b, cuda_dev)
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                    attention_mask=d["attention_mask"], labels=d["label"])
        loss = F.cross_entropy(out[1], d["label"])
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    for i, h in enumerate(hist):
        assert abs(losses[i] - float(h["loss_mean"])) <= TOL_TRAJ, (i, losses[i], float(h["loss_mean"]))
    sd = model.state_dict()
    for k, v in ref_params.items():
        assert float((sd[k].cpu() - v).abs().max()) <= 2e-4, k      # lr 3e-5 * 5 steps bounds any drift

    # fused CUDA-graph step
    model2 = make_model(cfg, state, cuda_dev).train()
    opt2 = b2.build_optimizer(model2, A)
    step = b2.FusedTrainStep(model2, opt2, 4, 128)
    losses2 = []
    for b in batches:
        step(b)
        losses2.append(step.loss_to_host())
    assert step.graph is not None
    for a, c in zip(losses, losses2):   # ulp-level dlogits differences (torch CE vs our CE kernel) grow over the steps
        assert abs(a - c) <= 5e-4, (losses, losses2)
    sd2 = model2.state_dict()
    # same kernels, same order; d(loss)/d(logits) comes from torch in one case and from our CE kernel in the other, and
    # the fused bias-gradient sums use fp32 atomics (order not fixed): ulp-level differences, amplified over 5 steps
    for k in sd:
        assert float((sd[k].double() - sd2[k].double()).abs().max()) <= 2e-5, k


def test_amp_script_loop_with_gradscaler(cuda_dev):
    """The -amp scripts' loop (multi-gpu-distributed-mp-amp-cls.py:166-171: autocast, scaler.scale(loss).backward(),
    scaler.step(optimizer), scaler.update(), and no zero_grad) runs unchanged and lands where the plain loop lands:
    the loss scale (2^16) is divided out inside the fused AdamW; a poisoned step is skipped like GradScaler skips it."""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    batches = [bert_ref.synthetic_batch(cfg, 4, 128, 2100 + i, padded=(i % 2 == 1)) for i in range(4)]

    class A:
        weight_decay, learning_rate = 0.01, 3e-5

    def fwd(model, b):
        d = to_dev(b, cuda_dev)
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                    attention_mask=d["attention_mask"], labels=d["label"])
        return F.cross_entropy(out[1], d["label"])

    plain = make_model(cfg, state, cuda_dev).train()
    opt = b2.build_optimizer(plain, A)
    ref_losses = []
    for b in batches:
        loss = fwd(plain, b)
        opt.zero_grad()
        loss.backward()
        opt.step()
        ref_losses.append(float(loss))

    amp = make_model(cfg, state, cuda_dev).train()
    opt2 = b2.build_optimizer(amp, A)
    scaler = torch.amp.GradScaler("cuda")
    for i, b in enumerate(batches):
        with torch.autocast("cuda"):
            loss = fwd(amp, b)
        scaler.scale(loss).backward()
        scaler.step(opt2)
        scaler.update()
        assert abs(float(loss) - ref_losses[i]) <= 5e-4, (i, float(loss), ref_losses[i])
    assert float(scaler.get_scale()) == 65536.0
    sd, sd2 = plain.state_dict(), amp.state_dict()
    for k in sd:
        assert float((sd[k].double() - sd2[k].double()).abs().max()) <= 2e-5, k
    # a non-finite loss: GradScaler's inf check sees it through the classifier.bias probe, the update and the AdamW
    # step count are skipped on the device, the scale backs off
    before = {k: v.clone() for k, v in amp.state_dict().items()}
    t_before = int(opt2._state()["step"])
    with torch.autocast("cuda"):
        loss = fwd(amp, batches[0]) * float("inf")
    scaler.scale(loss).backward()
    scaler.step(opt2)
    scaler.update()
    assert float(scaler.get_scale()) == 32768.0
    assert int(opt2._state()["step"]) == t_before
    after = amp.state_dict()
    for k in before:
        assert torch.equal(before[k], after[k]), k


def test_second_backward_without_step_raises(cuda_dev):
    """gradients live in the bf16 bucket space and are OVERWRITTEN by every backward (zero_grad is a no-op): with an
    optimizer attached, a second backward before optimizer.step() must raise instead of silently dropping the first
    one's gradients (torch would have accumulated them)"""
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    model = make_model(cfg, state_from_hf_init(cfg), cuda_dev).train()

    class A:
        weight_decay, learning_rate = 0.01, 3e-5

    opt = b2.build_optimizer(model, A)
    b = bert_ref.synthetic_batch(cfg, 4, 128, 3)
    _fwd_bwd(model, b, cuda_dev)
    with pytest.raises(RuntimeError, match="accumulation"):
        _fwd_bwd(model, b, cuda_dev)
    opt.step()
    _fwd_bwd(model, b, cuda_dev)          # fine again after the step
    opt.step()


def test_state_dict_round_trip_and_hf_loadable(cuda_dev):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev)
    sd = model.state_dict()
    assert "bert.embeddings.position_ids" in sd
    for k, v in state.items():
        assert torch.equal(sd[k].cpu(), v)
    from oracle import cpu_step
    hf = cpu_step.build_hf_model(cfg, seed=1)
    res = hf.load_state_dict({k: v.cpu() for k, v in sd.items()}, strict=False)
    assert not res.missing_keys
    wrapped = {"module." + k: v for k, v in sd.items()}          # what the reference's DDP checkpoints look like
    stripped = {k[len("module."):]: v for k, v in wrapped.items()}
    model.load_state_dict(stripped)


def test_full_config_step_matches_golden(cuda_dev):
    """BASELINE config A (chinese-bert-wwm-ext, B=32, S=128), dropout off: loss / logits / per-tensor gradient norms
    against the fixture produced by tests/golden/make_golden.py from HF transformers on CPU."""
    path = os.path.join(GOLD, "config_a_step0.pt")
    gold = torch.load(path)
    cfg = full_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    chk = float(sum(v.double().sum() for v in state.values()))
    assert abs(chk - gold["init_checksum"]) <= 1e-6 * max(1.0, abs(gold["init_checksum"])), \
        "HF init under seed 123 differs from the fixture's"
    model = make_model(cfg, state, cuda_dev).train()
    batch = bert_ref.synthetic_batch(cfg, 32, 128, 1000, padded=True)
    assert torch.equal(batch["input_ids"], gold["input_ids"])
    out, loss = _fwd_bwd(model, batch, cuda_dev)
    assert abs(float(loss) - gold["loss"]) <= TOL_LOSS
    assert float((out[1].detach().cpu() - gold["logits"]).abs().max()) <= TOL_LOGITS
    g = model.grad_dict()
    scale = max(gold["grad_norms"].values())
    for k, n in gold["grad_norms"].items():
        got = float(g[k].double().norm())
        assert abs(got - n) <= TOL_GRAD_REL * max(n, 1e-3 * scale), (k, got, n)
    # 64-value samples are noisier than whole-tensor norms (bf16 rounding noise does not average out over 64 values):
    # they guard against layout / indexing mistakes, at 3x the whole-tensor tolerance
    for k, ref in gold["grad_samples"].items():
        got = g[k].flatten()[: ref.numel()].cpu()
        assert float((got - ref).norm()) <= 3 * TOL_GRAD_REL * max(float(ref.norm()), 1e-3 * scale), k


def test_dropout_statistics_and_determinism(cuda_dev):
    """p=0.1 training forward: keep-rate 0.9 +- 0.002 (BASELINE.md §4), same (seed, step) -> same output,
    next step -> different mask."""
    from parity import philox_keep_mask
    keep = philox_keep_mask(8 * 1_000_000, 123, 0, 5, 0.1)
    assert abs(keep.mean() - 0.9) < 2e-3
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev).train()
    d = to_dev(bert_ref.synthetic_batch(cfg, 4, 128, 1, padded=False), cuda_dev)

    def run(step):
        model._engine.seed_dropout(5, step)
        with torch.no_grad():
            return model(input_ids=d["input_ids"], attention_mask=d["attention_mask"]).logits.clone()

    a, b, c = run(0), run(0), run(1)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)


@pytest.mark.parametrize("name", ["A", "B", "C"])
def test_full_depth_step0_matches_ddp_fixture(cuda_dev, name):
    """BASELINE.json configs A / B / C at FULL depth (12 / 12 / 24 layers, seq 128 / 512 / 128), dropout off: rank 0's
    step-0 loss, logits and every gradient tensor (norm + 64 strided values) against tests/golden/config_<x>_ddp.pt
    (HF transformers fp32 on CPU, tests/golden/make_golden_full.py).  Weights: the package initialiser under
    set_seed(123), as the fixture generator used."""
    sys_path = os.path.join(GOLD, "config_%s_ddp.pt" % name.lower())
    if not os.path.exists(sys_path):
        pytest.skip("fixture not generated")
    fx = torch.load(sys_path)
    preset = {"A": b2.chinese_bert_wwm_ext_config, "B": b2.bert_base_config, "C": b2.bert_large_config}[name]
    cfg = preset(num_labels=6, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg)
    chk = float(sum(p.detach().double().sum() for p in model.parameters()))
    assert abs(chk - fx["init_checksum"]) <= 1e-6 * max(1.0, abs(fx["init_checksum"])), "initialiser drifted"
    model.to(cuda_dev).train()
    B, S = fx["batch"], fx["seq"]
    batch = bert_ref.synthetic_batch(cfg, B, S, 5000, padded=False)
    assert torch.equal(batch["input_ids"], fx["input_ids_step0_rank0"])
    out, loss = _fwd_bwd(model, batch, cuda_dev)
    w1 = fx["worlds"][1]
    assert abs(float(loss) - float(w1["loss"][0][0])) <= TOL_LOSS
    assert float((out[1].detach().cpu() - w1["logits"][0][0]).abs().max()) <= TOL_LOGITS
    g = model.grad_dict()
    qk_tol = TOL_GRAD_REL if name == "A" else TOL_GRAD_REL_QK     # headline config: 2e-2 on every tensor
    gold = fx["step0_rank0"]
    scale = max(gold["grad_norms"].values())
    worst = {"qk": 0.0, "other": 0.0}
    for k, n in gold["grad_norms"].items():
        got = float(g[k].double().norm())
        rel = abs(got - n) / max(n, 1e-3 * scale)
        worst["qk" if ".query." in k or ".key." in k else "other"] = max(
            worst["qk" if ".query." in k or ".key." in k else "other"], rel)
        assert rel <= grad_tol(k, qk_tol), (k, got, n)
    # strided 64-value samples guard layout / indexing (bf16 noise does not average out over 64 values: 3x tolerance)
    for k, ref in gold["grad_samples"].items():
        f = g[k].flatten()
        if f.numel() > ref.numel():
            f = f[(torch.arange(ref.numel(), dtype=torch.int64) * (f.numel() - 1) // (ref.numel() - 1)).to(f.device)]
        assert float((f.cpu() - ref).norm()) <= 3 * grad_tol(k, qk_tol) * max(float(ref.norm()), 1e-3 * scale), k
    report("full_depth_step0", {"config": name, "dloss": abs(float(loss) - float(w1["loss"][0][0])),
                                "dlogit": float((out[1].detach().cpu() - w1["logits"][0][0]).abs().max()),
                                "worst_norm_rel": worst})


def test_from_pretrained_with_a_checkpoint_directory(cuda_dev, tmp_path):
    """The reference's model construction (multi-gpu-distributed-cls.py:336-338):
        config = BertConfig.from_pretrained(model_path, num_labels=6)
        model  = BertForSequenceClassification.from_pretrained(model_path, config=config)
    against a synthetic HF checkpoint directory (config.json + pytorch_model.bin holding the ENCODER only, as the
    real chinese-bert-wwm-ext checkpoint does: `bert.*` keys plus the pre-training heads `cls.*`, no classifier)."""
    import json
    cfg = tiny_config()
    state = state_from_hf_init(cfg, seed=321)
    ckpt_dir = tmp_path / "model_hub" / "tiny-bert"
    ckpt_dir.mkdir(parents=True)
    with open(ckpt_dir / "config.json", "w") as f:
        json.dump({k: getattr(cfg, k) for k in ("vocab_size", "hidden_size", "num_hidden_layers", "num_attention_heads",
                                                "intermediate_size", "max_position_embeddings", "type_vocab_size",
                                                "hidden_dropout_prob", "attention_probs_dropout_prob",
                                                "layer_norm_eps", "hidden_act", "initializer_range",
                                                "pad_token_id")}, f)
    sd = {k: v for k, v in state.items() if k.startswith("bert.")}
    sd["cls.predictions.bias"] = torch.zeros(cfg.vocab_size)                 # pre-training head: must be ignored
    sd["bert.embeddings.position_ids"] = torch.arange(cfg.max_position_embeddings)[None]
    torch.save(sd, ckpt_dir / "pytorch_model.bin")
    config = b2.BertConfig.from_pretrained(str(ckpt_dir), num_labels=6)
    assert config.num_labels == 6 and config.hidden_size == cfg.hidden_size
    torch.manual_seed(11)
    model = b2.BertForSequenceClassification.from_pretrained(str(ckpt_dir), config=config)
    got = dict(model.named_parameters())
    for k, v in state.items():
        if k.startswith("bert."):
            assert torch.equal(got[k].detach(), v), k                        # encoder: the checkpoint's tensors
    # the classifier is absent from the checkpoint: freshly initialised (N(0, 0.02) weight, zero bias), like HF
    assert got["classifier.weight"].shape == (6, cfg.hidden_size)
    assert 0.005 < float(got["classifier.weight"].std()) < 0.05 and float(got["classifier.bias"].abs().max()) == 0.0
    model.to(cuda_dev).eval()
    batch = bert_ref.synthetic_batch(cfg, 4, 128, 77, padded=True)
    d = to_dev(batch, cuda_dev)
    with torch.no_grad():
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"])
    ref_state = {k: v.detach().cpu() for k, v in model.named_parameters()}
    _, rz = bert_ref.forward(ref_state, cfg, batch["input_ids"], batch["token_type_ids"], batch["attention_mask"])
    assert float((out.logits.cpu() - rz).abs().max()) <= TOL_LOGITS
    with pytest.raises(FileNotFoundError):
        b2.BertForSequenceClassification.from_pretrained(str(tmp_path / "model_hub"), config=config)
