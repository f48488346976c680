"""CPU: BertForTokenClassification's host side -- the token oracle against HF's class, HF naming and checkpoints, the
packed labels, the criterion rules and the token-head entry points' argument checks."""
import ctypes
import json

import pytest
import torch
import torch.nn as nn

import token_oracle as tok
from parity import b2, bert_ref, tiny_config
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import _hf_order, _Layout
from pytorch_distributed_nlp_b200.packing import pack_batch
from pytorch_distributed_nlp_b200.trainer import step_loss


def _cfg(**kw):
    d = dict(num_labels=9, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    d.update(kw)
    return tiny_config(**d)


@pytest.mark.parametrize("classifier_dropout", [None, 0.0])
def test_token_oracle_equals_hf_forward_backward(classifier_dropout):
    """on a padded batch with -100 on padding, on [CLS] and on interior tokens: loss, logits and every gradient"""
    cfg = _cfg(classifier_dropout=classifier_dropout)
    hf = tok.hf_token_model(cfg)
    state = {k: v.detach().clone() for k, v in hf.named_parameters()}
    b = tok.token_batch(cfg, 4, 128, 1000)
    assert (b["label"] == -100).any() and ((b["label"] == -100) & (b["attention_mask"] == 1)).sum() > 4
    out = hf(input_ids=b["input_ids"], token_type_ids=b["token_type_ids"], attention_mask=b["attention_mask"],
             labels=b["label"])
    out[0].backward()
    loss, logits, grads = tok.loss_and_grads(state, cfg, b)
    assert logits.shape == (4, 128, cfg.num_labels)
    assert abs(float(out[0].detach()) - float(loss)) < 2e-6
    assert float((out[1].detach() - logits).abs().max()) < 2e-6
    assert set(grads) == {k for k, _ in hf.named_parameters()}
    for k, p in hf.named_parameters():
        assert float((grads[k] - p.grad).abs().max()) < 2e-6 + 1e-5 * float(p.grad.abs().max()), k


def test_token_oracle_head_dropout_is_mask_over_one_minus_p():
    cfg = _cfg(classifier_dropout=0.25)
    state = tok.token_state_from_hf_init(cfg)
    b = tok.token_batch(cfg, 2, 128, 7)
    m = tok.token_head_mask(cfg, 2, 128, seed=5, step=3)
    assert m.shape == (2, 128, cfg.hidden_size) and 0.6 < m.float().mean() < 0.9
    _, z = tok.forward(state, cfg, b["input_ids"], b["token_type_ids"], b["attention_mask"], head_mask=m)
    _, _, x = bert_ref.forward(dict(state, **{"bert.pooler.dense.weight": torch.zeros(cfg.hidden_size, cfg.hidden_size),
                                              "bert.pooler.dense.bias": torch.zeros(cfg.hidden_size)}),
                               cfg, b["input_ids"], b["token_type_ids"], b["attention_mask"], return_hidden=True)
    ref = (x * m / 0.75) @ state["classifier.weight"].t() + state["classifier.bias"]
    assert torch.allclose(z, ref, atol=1e-6, rtol=1e-6)


@pytest.mark.parametrize("cfg_fn", [lambda: _cfg(), lambda: b2.chinese_bert_wwm_ext_config(num_labels=9)])
def test_named_parameters_are_hf_token_classification(cfg_fn):
    cfg = cfg_fn()
    ours = [(n, tuple(p.shape)) for n, p in b2.BertForTokenClassification(cfg).named_parameters()]
    hf = [(n, tuple(p.shape)) for n, p in tok.hf_token_model(cfg).named_parameters()]
    assert ours == hf
    if cfg.num_hidden_layers == 12:
        assert len(ours) == 199
    assert [n for n, _ in ours] == _hf_order(cfg, "token")


def test_layout_tail_is_the_classifier_in_the_last_layer_bucket():
    cfg = _cfg()
    seq, tk = _Layout(cfg), _Layout(cfg, "token")
    assert not any(k.startswith("bert.pooler") for k in tk.entries)
    assert list(tk.entries)[-2:] == ["classifier.weight", "classifier.bias"]
    # the encoder part of the flat space is the sequence model's, offset for offset
    for k, v in tk.entries.items():
        if k.startswith("bert."):
            assert seq.entries[k] == v
    assert tk.buckets[:-1] == seq.buckets[:-1]
    assert tk.buckets[-1][2].endswith("+head") and tk.buckets[-1][1] == tk.total
    with pytest.raises(ValueError):
        _Layout(cfg, "qa")


def test_hf_state_dict_round_trips_strict():
    cfg = _cfg()
    hf = tok.hf_token_model(cfg)
    m = b2.BertForTokenClassification(cfg)
    m.load_state_dict(hf.state_dict(), strict=True)
    sd = m.state_dict()
    for k, v in hf.state_dict().items():
        assert torch.equal(sd[k], v), k
    # and back into HF (our state dict also carries the position_ids buffer of transformers 4.28)
    hf2 = tok.hf_token_model(cfg, seed=9)
    hf2.load_state_dict({k: sd[k] for k in hf2.state_dict()}, strict=True)


@pytest.mark.parametrize("kind", ["pretraining", "sequence"])
def test_from_pretrained_ignores_the_pooler(tmp_path, kind):
    """as HF's from_pretrained: the encoder loads, the pooler is ignored; the classifier keeps its init when the
    checkpoint has none (pre-training) and loads by name and shape when it has one (sequence classification)"""
    cfg = _cfg()
    from oracle import cpu_step
    seq = cpu_step.build_hf_model(cfg, seed=3)
    ckpt = dict(seq.state_dict())
    if kind == "pretraining":
        ckpt = {k: v for k, v in ckpt.items() if not k.startswith("classifier.")}
        ckpt["cls.predictions.bias"] = torch.zeros(cfg.vocab_size)
    torch.save(ckpt, tmp_path / "pytorch_model.bin")
    torch.manual_seed(11)
    fresh = b2.BertForTokenClassification(cfg)
    torch.manual_seed(11)
    m = b2.BertForTokenClassification.from_pretrained(str(tmp_path), config=cfg)
    sd = m.state_dict()
    for k, v in seq.state_dict().items():
        if k.startswith("bert.") and "pooler" not in k:
            assert torch.equal(sd[k], v), k
    for k in ("classifier.weight", "classifier.bias"):
        want = fresh.state_dict()[k] if kind == "pretraining" else seq.state_dict()[k]
        assert torch.equal(sd[k], want), k
    assert not any("pooler" in k for k in sd)


def test_save_pretrained_round_trip_and_architectures(tmp_path):
    cfg = _cfg()
    m = b2.BertForTokenClassification.from_config(cfg, seed=4)
    m.save_pretrained(str(tmp_path))
    with open(tmp_path / "config.json") as f:
        c = json.load(f)
    assert c["architectures"] == ["BertForTokenClassification"] and c["num_labels"] == 9
    m2 = b2.BertForTokenClassification.from_pretrained(str(tmp_path))
    for (k, a), (k2, b_) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k == k2 and torch.equal(a, b_)
    # the sequence model's config.json is as before: no architectures key
    s = b2.BertForSequenceClassification(cfg)
    s.save_pretrained(str(tmp_path / "seq"))
    with open(tmp_path / "seq" / "config.json") as f:
        assert "architectures" not in json.load(f)


def test_more_labels_than_the_kernel_bound_raise():
    with pytest.raises(ValueError, match="64"):
        b2.BertForTokenClassification(_cfg(num_labels=65))
    b2.BertForTokenClassification(_cfg(num_labels=64))


def test_pack_batch_labels_unpack_to_the_valid_positions():
    cfg = _cfg()
    for bin_len, seq in ((128, 128), (512, 512)):
        b = tok.token_batch(cfg, 16, seq, 77, min_len=4)
        p = pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], bin_len, labels=b["label"])
        assert p["labels"].shape == (p["bins"], bin_len) and p["labels"].dtype == torch.int64
        flat = p["labels"].reshape(-1)
        for i in range(16):
            n = int(p["lengths"][i])
            c = int(p["cls_index"][i])
            assert torch.equal(flat[c:c + n], b["label"][i, :n])
        used = torch.zeros(flat.numel(), dtype=torch.bool)
        for i in range(16):
            c = int(p["cls_index"][i])
            used[c:c + int(p["lengths"][i])] = True
        assert bool((flat[~used] == -100).all())
        # without labels the packed batch is what it was
        q = pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], bin_len)
        assert "labels" not in q
        for k in ("input_ids", "token_type_ids", "position_ids", "segments", "cls_index", "lengths"):
            assert torch.equal(p[k], q[k]), k


def test_pack_batch_labels_other_ignore_index_and_rejections():
    cfg = _cfg()
    b = tok.token_batch(cfg, 4, 128, 5)
    lab = b["label"].clone()
    lab[lab == -100] = -1
    p = pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], 128, labels=lab, ignore_index=-1)
    assert not bool((p["labels"] == -100).any())
    bad = b["label"].clone()
    row = int((b["attention_mask"][0] == 0).nonzero()[0])
    bad[0, row] = 3
    with pytest.raises(ValueError, match="masked position"):
        pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], 128, labels=bad)
    with pytest.raises(ValueError):
        pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], 128, labels=b["label"].float())


def test_criterion_rules_for_a_token_model():
    m = b2.BertForTokenClassification(_cfg())
    plain = step_loss(m)
    assert plain.mode == L.LOSS_CE and plain.plain_ce
    ce = step_loss(m, nn.CrossEntropyLoss(weight=torch.rand(9), ignore_index=-1, label_smoothing=0.1))
    assert ce.mode == L.LOSS_CE and ce.ignore_index == -1 and ce.label_smoothing == pytest.approx(0.1)
    for crit in (nn.MSELoss(), nn.BCEWithLogitsLoss()):
        with pytest.raises(ValueError, match="token-classification"):
            step_loss(m, crit)
    # problem_type is not read: a regression config still trains with cross-entropy, as HF's token model does
    m2 = b2.BertForTokenClassification(_cfg(problem_type="regression"))
    assert step_loss(m2).mode == L.LOSS_CE


def test_token_head_entry_points_are_declared_and_check_arguments():
    for name in ("b2_token_head_fwd", "b2_token_head_bwd_split"):
        assert name in L._SIGNATURES and name in L.EXPORTED_SYMBOLS
    lib = L.load()
    assert lib.b2_token_head_scratch_floats(4096, 768, 9) == 128 * 10 * 768
    assert lib.b2_token_head_scratch_floats(100, 256, 2) == 4 * 3 * 256
    one = ctypes.c_void_p(256)   # never dereferenced: every case fails its checks before a launch
    cases = [(4096, 768, 65, 0.0, "num_labels"), (4096, 300, 9, 0.0, "hidden"), (4096, 768, 9, 1.0, "dropout_p"),
             (4096, 768, 9, float("nan"), "dropout_p"), (0, 768, 9, 0.0, "tokens"), (1 << 20, 768, 9, 0.0, "tokens")]
    for tokens, hidden, C, p, what in cases:
        st = lib.b2_token_head_fwd(one, tokens, hidden, one, one, C, p, one, 7, one, None)
        assert st != 0 and what in L.last_error(), (tokens, hidden, C, p, L.last_error())
        st = lib.b2_token_head_bwd_split(one, one, tokens, hidden, one, C, p, one, 7, one, one, one, one, 1 << 40,
                                         None, None)
        assert st != 0 and what in L.last_error(), (tokens, hidden, C, p, L.last_error())
    st = lib.b2_token_head_bwd_split(one, one, 4096, 768, one, 9, 0.0, one, 7, one, one, one, one, 10, None, None)
    assert st != 0 and "scratch" in L.last_error()
