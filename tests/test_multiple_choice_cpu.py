"""CPU: BertForMultipleChoice's host side -- the multiple-choice oracle against HF's class (loss, logits and every
gradient, over N = 1, 2 and 4 choices, padded rows, ignored labels, label smoothing and class weights), HF naming,
state dicts and checkpoints, packing of [B, N, S] batches, the criterion rules, the argument checks and
synthetic_mc_batch."""
import json

import pytest
import torch
import torch.nn as nn

import mc_oracle as mc
from parity import b2, tiny_config
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import HEAD_KINDS, _hf_order, _Layout
from pytorch_distributed_nlp_b200.packing import bin_length, pack_batch
from pytorch_distributed_nlp_b200.trainer import check_mc_criterion, step_loss

S = 64


def _cfg(**kw):
    d = dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    d.update(kw)
    return tiny_config(**d)


ORACLE_CASES = {   # name: (N, padded, criterion factory)
    "n1": (1, False, None),
    "n2": (2, False, None),
    "n4": (4, False, None),
    "n4_padded": (4, True, None),
    "ignored": (4, True, None),
    "smoothing": (4, True, lambda n: nn.CrossEntropyLoss(label_smoothing=0.1)),
    "weights": (4, True, lambda n: nn.CrossEntropyLoss(weight=torch.linspace(0.5, 2.0, n))),
}


@pytest.mark.parametrize("case", list(ORACLE_CASES))
def test_mc_oracle_equals_hf_forward_backward(case):
    """logits, loss and every gradient of the oracle against transformers.BertForMultipleChoice"""
    N, padded, crit_fn = ORACLE_CASES[case]
    cfg = _cfg()
    hf = mc.hf_mc_model(cfg)
    state = {k: v.detach().clone() for k, v in hf.named_parameters()}
    b = b2.synthetic_mc_batch(cfg, 3, N, S, 11, padded=padded)
    if case == "ignored":
        b["label"][1] = -100
    crit = crit_fn(N) if crit_fn else None
    out = hf(input_ids=b["input_ids"], token_type_ids=b["token_type_ids"], attention_mask=b["attention_mask"])
    hf_loss = (crit or nn.CrossEntropyLoss())(out.logits, b["label"])
    if crit is None:
        # HF's own in-model loss is the same CrossEntropyLoss()
        own = hf(input_ids=b["input_ids"], token_type_ids=b["token_type_ids"], attention_mask=b["attention_mask"],
                 labels=b["label"]).loss
        assert float(own.detach()) == float(hf_loss.detach())
    hf_loss.backward()
    loss, logits, grads = mc.loss_and_grads(state, cfg, b, criterion=crit)
    assert logits.shape == (3, N)
    assert float((out.logits.detach() - logits).abs().max()) < 2e-6
    assert abs(float(hf_loss.detach()) - float(loss)) < 2e-6
    assert set(grads) == {k for k, _ in hf.named_parameters()}
    for k, p in hf.named_parameters():
        assert float((grads[k] - p.grad).abs().max()) < 2e-6 + 1e-5 * float(p.grad.abs().max()), k
    if N == 1 and crit is None:
        # one choice: the softmax is 1, the loss 0 and every gradient 0
        assert float(loss) == 0.0 and all(float(g.abs().max()) == 0.0 for g in grads.values())


@pytest.mark.parametrize("cfg_fn", [lambda: _cfg(num_labels=6), lambda: b2.chinese_bert_wwm_ext_config(num_labels=6)])
def test_named_parameters_are_hf_multiple_choice(cfg_fn):
    """HF's names and order; the classifier has one row whatever num_labels says, and num_labels stays as given"""
    cfg = cfg_fn()
    m = b2.BertForMultipleChoice(cfg)
    names = [k for k, _ in m.named_parameters()]
    assert names == _hf_order(cfg, "multiple_choice")
    assert names[-4:] == ["bert.pooler.dense.weight", "bert.pooler.dense.bias", "classifier.weight",
                          "classifier.bias"]
    assert m.classifier.weight.shape == (1, cfg.hidden_size) and m.classifier.bias.shape == (1,)
    assert cfg.num_labels == 6
    if cfg.num_hidden_layers == 2:
        hf = mc.hf_mc_model(cfg)
        assert names == [k for k, _ in hf.named_parameters()]
        for (k, p), (_k2, q) in zip(m.named_parameters(), hf.named_parameters()):
            assert p.shape == q.shape, k
    else:
        assert len(names) == 201


def test_layout_is_the_sequence_layout_with_one_classifier_row():
    cfg = _cfg(num_labels=6)
    assert HEAD_KINDS[:4] == ("sequence", "token", "mlm", "question_answering") and "multiple_choice" in HEAD_KINDS
    lay = _Layout(cfg, "multiple_choice")
    seq = _Layout(_cfg(num_labels=1), "sequence")
    assert lay.entries == seq.entries and lay.buckets == seq.buckets and lay.total == seq.total
    b, e, label = lay.buckets[-1]
    assert label == "layer1+head" and e == lay.total
    assert b <= lay.off("bert.pooler.dense.weight") < lay.off("classifier.bias") < e
    assert b2.BertForMultipleChoice._anchor == "classifier.bias"
    with pytest.raises(ValueError, match="head="):
        _Layout(cfg, "mc")


def test_hf_state_dict_round_trips_strict():
    cfg = _cfg()
    hf = mc.hf_mc_model(cfg)
    m = b2.BertForMultipleChoice(cfg)
    m.load_state_dict(hf.state_dict(), strict=True)
    sd = m.state_dict()
    for k, v in hf.state_dict().items():
        assert torch.equal(sd[k], v), k
    hf2 = mc.hf_mc_model(cfg, seed=9)
    hf2.load_state_dict({k: sd[k] for k in hf2.state_dict()}, strict=True)


@pytest.mark.parametrize("kind", ["pretraining", "multiple_choice"])
def test_from_pretrained_loads_encoder_and_pooler(tmp_path, kind):
    """the encoder and the pooler load; a pre-training checkpoint's cls.* is ignored and the classifier keeps its
    init, a multiple-choice checkpoint's classifier loads"""
    cfg = _cfg()
    src = mc.hf_mc_model(cfg, seed=3)
    ckpt = dict(src.state_dict())
    if kind == "pretraining":
        ckpt = {k: v for k, v in ckpt.items() if not k.startswith("classifier.")}
        ckpt["cls.predictions.bias"] = torch.zeros(cfg.vocab_size)
        ckpt["cls.seq_relationship.weight"] = torch.zeros(2, cfg.hidden_size)
    torch.save(ckpt, tmp_path / "pytorch_model.bin")
    torch.manual_seed(11)
    fresh = b2.BertForMultipleChoice(cfg)
    torch.manual_seed(11)
    m = b2.BertForMultipleChoice.from_pretrained(str(tmp_path), config=cfg)
    sd = m.state_dict()
    for k, v in src.state_dict().items():
        if k.startswith("bert."):
            assert torch.equal(sd[k], v), k
    assert any(k.startswith("bert.pooler.") for k in sd)
    for k in ("classifier.weight", "classifier.bias"):
        want = fresh.state_dict()[k] if kind == "pretraining" else src.state_dict()[k]
        assert torch.equal(sd[k], want), k
    assert not any(k.startswith("cls.") for k in sd)


def test_sequence_classifier_checkpoint_raises_as_transformers_does(tmp_path):
    """a 6-class sequence classifier's checkpoint: transformers' BertForMultipleChoice.from_pretrained raises on the
    classifier's size mismatch (without ignore_mismatched_sizes), and so does this one"""
    from transformers import BertForMultipleChoice, BertForSequenceClassification
    from oracle import cpu_step
    cfg = _cfg(num_labels=6)
    torch.manual_seed(3)
    BertForSequenceClassification(cpu_step.hf_config(cfg)).save_pretrained(str(tmp_path), safe_serialization=False)
    with pytest.raises(Exception, match="mismatch"):
        BertForMultipleChoice.from_pretrained(str(tmp_path))
    with pytest.raises(RuntimeError, match="size mismatch for classifier.weight"):
        b2.BertForMultipleChoice.from_pretrained(str(tmp_path), config=cfg)


def test_save_pretrained_round_trip_and_architectures(tmp_path):
    cfg = _cfg(num_labels=6)
    m = b2.BertForMultipleChoice.from_config(cfg, seed=4)
    m.save_pretrained(str(tmp_path))
    with open(tmp_path / "config.json") as f:
        c = json.load(f)
    assert c["architectures"] == ["BertForMultipleChoice"] and c["num_labels"] == 6 and c["problem_type"] is None
    m2 = b2.BertForMultipleChoice.from_pretrained(str(tmp_path))
    for (k, a), (k2, b_) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k == k2 and torch.equal(a, b_)


def test_output_is_hf_tuple_order():
    o = b2.MultipleChoiceModelOutput(loss=1, logits=2)
    assert tuple(o) == (1, 2) and o[0] == 1 and o["logits"] == 2 and len(o) == 2 and o.to_tuple() == (1, 2)
    o = b2.MultipleChoiceModelOutput(logits=2)
    assert tuple(o) == (2,) and o[0] == 2 and len(o) == 1


def test_argument_checks():
    m = b2.BertForMultipleChoice(_cfg())
    ids = torch.zeros(2, 3, S, dtype=torch.int64)
    with pytest.raises(ValueError, match=r"\[batch, num_choices, seq\]"):
        m(input_ids=ids[:, 0])
    with pytest.raises(ValueError, match="attention_mask must have input_ids' shape"):
        m(input_ids=ids, attention_mask=ids[:, :2])
    with pytest.raises(ValueError, match="token_type_ids must have input_ids' shape"):
        m(input_ids=ids, token_type_ids=ids.reshape(6, S))
    with pytest.raises(TypeError, match="int64"):
        m(input_ids=ids, labels=torch.zeros(2))
    with pytest.raises(ValueError, match=r"must be \[2\]"):
        m(input_ids=ids, labels=torch.zeros(2, 1, dtype=torch.int64))     # HF rejects [B, 1] too
    with pytest.raises(ValueError, match=r"must be \[2\]"):
        m(input_ids=ids, labels=torch.zeros(6, dtype=torch.int64))
    with pytest.raises(ValueError, match="together"):
        m(input_ids=ids[0], cls_index=torch.zeros(2, 3, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"cls_index .* \[batch, num_choices\]"):
        m(input_ids=ids[0], position_ids=ids[0], segments=ids[0].int(), cls_index=torch.zeros(6, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="CUDA"):
        m(input_ids=ids, labels=torch.zeros(2, dtype=torch.int64))


def test_pack_batch_of_choices():
    """[B, N, S] packs the B·N choice sequences: cls_index and lengths [B, N], sequence labels untouched, and every
    choice's tokens come back from its bin rows"""
    cfg = _cfg()
    b = b2.synthetic_mc_batch(cfg, 5, 4, S, 3, padded=True)
    ids, tt, mask, lab = b["input_ids"], b["token_type_ids"], b["attention_mask"], b["label"]
    assert bin_length(mask, S) == 128
    p = pack_batch(ids, tt, mask, 128, labels=lab)
    assert p["cls_index"].shape == (5, 4) and p["lengths"].shape == (5, 4)
    assert torch.equal(p["lengths"], mask.sum(-1)) and p["labels"] is lab
    flat = pack_batch(ids.view(20, S), tt.view(20, S), mask.view(20, S), 128)
    for k in ("input_ids", "token_type_ids", "position_ids", "segments"):
        assert torch.equal(p[k], flat[k]), k
    assert torch.equal(p["cls_index"].view(-1), flat["cls_index"]) and p["bins"] == flat["bins"]
    rows_ids, rows_tt = p["input_ids"].view(-1), p["token_type_ids"].view(-1)
    for i in range(5):
        for k in range(4):
            n, c = int(p["lengths"][i, k]), int(p["cls_index"][i, k])
            assert torch.equal(rows_ids[c:c + n], ids[i, k, :n]) and torch.equal(rows_tt[c:c + n], tt[i, k, :n])
            assert torch.equal(p["position_ids"].view(-1)[c:c + n], torch.arange(n))
    assert "labels" not in pack_batch(ids, tt, mask, 128)
    with pytest.raises(ValueError, match="multiple-choice labels"):
        pack_batch(ids, tt, mask, 128, labels=lab.float())
    with pytest.raises(ValueError, match="multiple-choice labels"):
        pack_batch(ids, tt, mask, 128, labels=lab[:, None])
    with pytest.raises(ValueError, match="attention_mask must have"):
        pack_batch(ids, tt, mask[:, :2], 128)


def test_criterion_rules_for_a_multiple_choice_model():
    m = b2.BertForMultipleChoice(_cfg(num_labels=6))
    fn = step_loss(m, None, 4)
    assert fn.mode == L.LOSS_CE and fn.C == 4 and fn.plain_ce
    w = torch.tensor([1.0, 2.0, 0.5, 1.5])
    fn = step_loss(m, nn.CrossEntropyLoss(weight=w, ignore_index=-1, label_smoothing=0.2), 4)
    assert fn.C == 4 and torch.equal(fn.weight, w) and fn.ignore_index == -1 and fn.label_smoothing == pytest.approx(0.2)
    with pytest.raises(ValueError, match=r"shape \(4,\)"):
        step_loss(m, nn.CrossEntropyLoss(weight=torch.ones(6)), 4)
    for bad in (nn.MSELoss(), nn.BCEWithLogitsLoss()):
        with pytest.raises(ValueError, match="multiple-choice model"):
            step_loss(m, bad, 4)
        with pytest.raises(ValueError, match="multiple-choice model"):
            check_mc_criterion(bad)
    with pytest.raises(ValueError, match="args.fused = False"):
        step_loss(m, nn.NLLLoss(), 4)
    tr = b2.Trainer(b2.Args(), m.config, m, None, None)
    assert tr.problem_type(torch.zeros(2, dtype=torch.int64)) == "multiple_choice"
    assert getattr(m.config, "problem_type", None) is None
    tr = b2.Trainer(b2.Args(), m.config, m, nn.MSELoss(), None)
    with pytest.raises(ValueError, match="multiple-choice model"):
        tr.compute_loss(torch.zeros(2, 4), torch.zeros(2, dtype=torch.int64))
    tr = b2.Trainer(b2.Args(), m.config, m, nn.CrossEntropyLoss(label_smoothing=0.1), None)
    logits, lab = torch.randn(3, 4), torch.tensor([0, 3, -100])
    assert torch.equal(tr.compute_loss(logits, lab), nn.CrossEntropyLoss(label_smoothing=0.1)(logits, lab))


def test_synthetic_mc_batch_is_reproducible_and_swag_shaped():
    cfg = _cfg()
    a = b2.synthetic_mc_batch(cfg, 16, 4, S, 7, padded=True)
    b = b2.synthetic_mc_batch(cfg, 16, 4, S, 7, padded=True)
    c = b2.synthetic_mc_batch(cfg, 16, 4, S, 8, padded=True)
    assert all(torch.equal(a[k], b[k]) for k in a) and not torch.equal(a["input_ids"], c["input_ids"])
    ids, tt, mask, lab = a["input_ids"], a["token_type_ids"], a["attention_mask"], a["label"]
    assert ids.shape == tt.shape == mask.shape == (16, 4, S) and lab.shape == (16,) and lab.dtype == torch.int64
    assert int(lab.min()) >= 0 and int(lab.max()) < 4
    lens = mask.sum(-1)
    assert bool((mask == (torch.arange(S)[None, None] < lens[..., None])).all())     # right padding
    varied = 0
    for i in range(16):
        ctx = int((tt[i, 0, :lens[i, 0]] == 0).sum()) - 2                          # [CLS] context [SEP]
        varied += len(set(lens[i].tolist())) > 1
        for k in range(4):
            n = int(lens[i, k])
            assert int(ids[i, k, 0]) == 101 and int(ids[i, k, ctx + 1]) == 102 and int(ids[i, k, n - 1]) == 102
            assert torch.equal(ids[i, k, :ctx + 2], ids[i, 0, :ctx + 2])               # one shared context
            assert bool((tt[i, k, :ctx + 2] == 0).all()) and bool((tt[i, k, ctx + 2:n] == 1).all())
            assert bool((tt[i, k, n:] == 0).all()) and bool((ids[i, k, n:] == 0).all())
    assert varied > 8
    full = b2.synthetic_mc_batch(cfg, 2, 3, S, 7)
    assert bool((full["attention_mask"] == 1).all())
