"""CPU: BertForMaskedLM's naming, tied keys and checkpoints, the vocabulary padding of its flat space, mask_tokens
against HF's DataCollatorForLanguageModeling, the criterion rules, and the fp32 masked-LM oracle
(tests/mlm_oracle.py) against the installed transformers.BertForMaskedLM."""
import pytest
import torch
import torch.nn as nn

import mlm_oracle as mlm
from parity import tiny_config
import pytorch_distributed_nlp_b200 as b2
from pytorch_distributed_nlp_b200.modeling import vocab_pad
from pytorch_distributed_nlp_b200.trainer import check_mlm_criterion, step_loss

V_ODD = 1000      # not a multiple of 64: the flat space pads the vocabulary to 1024


def _cfg(**kw):
    return tiny_config(vocab_size=V_ODD, **kw)


def test_hf_names_order_and_count():
    from transformers import BertForMaskedLM
    from oracle import cpu_step
    cfg = _cfg()
    hf = BertForMaskedLM(cpu_step.hf_config(cfg))
    ours = b2.BertForMaskedLM(cfg)
    assert [n for n, _ in ours.named_parameters()] == [n for n, _ in hf.named_parameters()]
    full = b2.BertForMaskedLM(b2.chinese_bert_wwm_ext_config())
    assert len(list(full.named_parameters())) == 202
    for n, p in ours.named_parameters():
        assert tuple(p.shape) == tuple(dict(hf.named_parameters())[n].shape), n


def test_state_dict_tied_keys_and_strict_loading():
    from transformers import BertForMaskedLM
    from oracle import cpu_step
    cfg = _cfg()
    torch.manual_seed(3)
    hf = BertForMaskedLM(cpu_step.hf_config(cfg))
    hsd = hf.state_dict()
    ours = b2.BertForMaskedLM(cfg)
    sd = ours.state_dict()
    for k in ("cls.predictions.decoder.weight", "cls.predictions.decoder.bias"):
        assert k in sd
    assert sd["cls.predictions.decoder.weight"] is sd["bert.embeddings.word_embeddings.weight"]
    assert sd["cls.predictions.decoder.bias"] is sd["cls.predictions.bias"]
    assert set(k for k in hsd if not k.endswith("position_ids")) <= set(sd)
    # with and without the tied keys, strict
    ours.load_state_dict(hsd, strict=True)
    for n, p in ours.named_parameters():
        assert torch.equal(p, hsd[n]), n
    no_tied = {k: v for k, v in hsd.items() if not k.startswith("cls.predictions.decoder")}
    fresh = b2.BertForMaskedLM(cfg)
    fresh.load_state_dict(no_tied, strict=True)
    assert torch.equal(fresh.cls.predictions.bias, hf.cls.predictions.bias)
    with pytest.raises(RuntimeError):
        fresh.load_state_dict({k: v for k, v in no_tied.items() if k != "cls.predictions.bias"}, strict=True)


def test_from_pretrained_pretraining_checkpoint(tmp_path):
    """a BertForPreTraining checkpoint: cls.predictions.* load, bert.pooler.* and cls.seq_relationship.* are ignored"""
    from transformers import BertForPreTraining
    from oracle import cpu_step
    cfg = _cfg()
    torch.manual_seed(5)
    pt = BertForPreTraining(cpu_step.hf_config(cfg))
    sd = pt.state_dict()
    assert any(k.startswith("cls.seq_relationship") for k in sd) and any(k.startswith("bert.pooler") for k in sd)
    torch.save(sd, tmp_path / "pytorch_model.bin")
    m = b2.BertForMaskedLM.from_pretrained(str(tmp_path), config=cfg)
    for n, p in m.named_parameters():
        assert torch.equal(p, sd[n]), n
    m.save_pretrained(str(tmp_path / "out"))
    import json
    assert json.load(open(tmp_path / "out" / "config.json"))["architectures"] == ["BertForMaskedLM"]
    back = b2.BertForMaskedLM.from_pretrained(str(tmp_path / "out"), config=cfg)
    for n, p in back.named_parameters():
        assert torch.equal(p, sd[n]), n


def test_checkpoint_without_head_keeps_hf_init(tmp_path):
    """from_pretrained on an encoder-only (sequence-classification) checkpoint: the encoder loads, the MLM head keeps
    HF's fresh init"""
    cfg = _cfg()
    seq = b2.BertForSequenceClassification(cfg)
    seq.save_pretrained(str(tmp_path))
    torch.manual_seed(0)
    m2 = b2.BertForMaskedLM.from_pretrained(str(tmp_path), config=cfg)
    for n, p in m2.named_parameters():
        if n.startswith("bert."):
            assert torch.equal(p, seq.state_dict()[n]), n
    assert torch.all(m2.cls.predictions.bias == 0)
    assert torch.all(m2.cls.predictions.transform.LayerNorm.weight == 1)
    assert torch.all(m2.cls.predictions.transform.LayerNorm.bias == 0)
    w = m2.cls.predictions.transform.dense.weight
    assert abs(float(w.std()) - cfg.initializer_range) < 0.2 * cfg.initializer_range


def test_vocab_pad_rows_outside_every_view():
    cfg = _cfg()
    m = b2.BertForMaskedLM(cfg)
    lay = m._layout
    Vp, H = vocab_pad(cfg.vocab_size), cfg.hidden_size
    assert Vp == 1024 and lay.vocab_pad == Vp
    off_w, shape_w = lay.entries["bert.embeddings.word_embeddings.weight"]
    off_b, shape_b = lay.entries["cls.predictions.bias"]
    assert shape_w == (cfg.vocab_size, H) and shape_b == (cfg.vocab_size,)
    assert m.bert.embeddings.word_embeddings.weight.shape == (cfg.vocab_size, H)
    # the padding is zero, inside the flat space, and no parameter view reaches it
    assert torch.all(m._flat[off_w + cfg.vocab_size * H:off_w + Vp * H] == 0)
    assert torch.all(m._flat[off_b + cfg.vocab_size:off_b + Vp] == 0)
    covered = torch.zeros(lay.total, dtype=torch.bool)
    for name, (off, shape) in lay.entries.items():
        covered[off:off + int(torch.tensor(shape).prod())] = True
    assert not covered[off_w + cfg.vocab_size * H:off_w + Vp * H].any()
    assert not covered[off_b + cfg.vocab_size:off_b + Vp].any()
    for k, v in m.state_dict().items():
        if "word_embeddings" in k or "decoder.weight" in k:
            assert v.shape[0] == cfg.vocab_size
    # the sequence and token models keep their layout
    seq = b2.BertForSequenceClassification(cfg)
    assert seq._layout.entries["bert.embeddings.word_embeddings.weight"][0] + cfg.vocab_size * H == \
        seq._layout.entries["bert.embeddings.position_embeddings.weight"][0]


class _StubTokenizer:
    mask_token = "[MASK]"
    pad_token = "[PAD]"

    def __init__(self, vocab):
        self.vocab = vocab

    def __len__(self):
        return self.vocab

    def convert_tokens_to_ids(self, tok):
        return 103


@pytest.mark.parametrize("seed,prob,replace,rand,padded", [
    (0, 0.15, 0.8, 0.1, False), (1, 0.15, 0.8, 0.1, True), (7, 0.3, 0.5, 0.25, True), (11, 0.15, 1.0, 0.0, True),
    (13, 0.4, 0.8, 0.0, False), (17, 0.15, 0.0, 0.5, True)])
def test_mask_tokens_matches_hf_collator(seed, prob, replace, rand, padded):
    from transformers import DataCollatorForLanguageModeling
    cfg = tiny_config(vocab_size=21128)
    batch = b2.synthetic_batch(cfg, 8, 128, seed, padded=padded)
    ids, mask = batch["input_ids"], batch["attention_mask"]
    ids[:, 5] = 102
    special = ((ids == 0) | (ids == 101) | (ids == 102) | (mask == 0))
    coll = DataCollatorForLanguageModeling(_StubTokenizer(cfg.vocab_size), mlm_probability=prob,
                                           mask_replace_prob=replace, random_replace_prob=rand)
    coll.generator = torch.Generator().manual_seed(seed)
    hf_in, hf_lab = coll.torch_mask_tokens(ids.clone(), special_tokens_mask=special.clone())
    g = torch.Generator().manual_seed(seed)
    got_in, got_lab = b2.mask_tokens(ids, mask, mlm_probability=prob, mask_replace_prob=replace,
                                     random_replace_prob=rand, vocab_size=cfg.vocab_size, generator=g)
    assert torch.equal(got_in, hf_in) and torch.equal(got_lab, hf_lab)
    # the same with the special positions given as a mask, and the caller's ids untouched
    g = torch.Generator().manual_seed(seed)
    again = b2.mask_tokens(ids, special_tokens_mask=special, mlm_probability=prob, mask_replace_prob=replace,
                           random_replace_prob=rand, vocab_size=cfg.vocab_size, generator=g, special_ids=())
    assert torch.equal(again[0], hf_in) and torch.equal(again[1], hf_lab)
    assert not torch.equal(ids, hf_in) or prob == 0


def test_mask_tokens_arguments():
    ids = torch.randint(200, 300, (2, 16))
    with pytest.raises(ValueError):
        b2.mask_tokens(ids, mlm_probability=1.5, vocab_size=512)
    with pytest.raises(ValueError):
        b2.mask_tokens(ids, mask_replace_prob=0.8, random_replace_prob=0.3, vocab_size=512)
    with pytest.raises(TypeError):
        b2.mask_tokens(ids.float(), vocab_size=512)


def test_synthetic_mlm_batch():
    cfg = tiny_config(vocab_size=V_ODD)
    b = b2.synthetic_mlm_batch(cfg, 4, 128, 3, padded=True)
    lab = b["label"]
    assert lab.shape == (4, 128) and lab.dtype == torch.int64
    assert torch.all(lab[b["attention_mask"] == 0] == -100)
    assert torch.all(lab[:, 0] == -100)
    assert (lab != -100).any()
    assert torch.equal(b2.synthetic_mlm_batch(cfg, 4, 128, 3, padded=True)["input_ids"], b["input_ids"])


def test_criterion_rules():
    check_mlm_criterion(None)
    check_mlm_criterion(nn.CrossEntropyLoss(ignore_index=-1))
    for bad in (nn.MSELoss(), nn.BCEWithLogitsLoss()):
        with pytest.raises(ValueError):
            check_mlm_criterion(bad)
    m = b2.BertForMaskedLM(_cfg())
    fn = step_loss(m, None)
    assert fn.C == V_ODD and fn.ignore_index == -100 and not fn.float_labels
    assert step_loss(m, nn.CrossEntropyLoss(ignore_index=-1)).ignore_index == -1
    for bad in (nn.CrossEntropyLoss(label_smoothing=0.1), nn.CrossEntropyLoss(weight=torch.ones(V_ODD)),
                nn.CrossEntropyLoss(reduction="sum")):
        check_mlm_criterion(bad)                     # the eager path applies it to the full logits
        with pytest.raises(ValueError, match="fused = False"):
            step_loss(m, bad)
    with pytest.raises(ValueError):
        step_loss(m, nn.MSELoss())


def test_model_needs_cuda():
    m = b2.BertForMaskedLM(_cfg())
    with pytest.raises(RuntimeError, match="CUDA"):
        m(input_ids=torch.zeros(1, 128, dtype=torch.int64))


def test_oracle_matches_hf_masked_lm():
    """loss, logits and every gradient of the fp32 oracle against transformers.BertForMaskedLM, the tied table's pad
    row included (its gradient is the decoder's part alone)"""
    cfg = _cfg(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    hf = mlm.hf_mlm_model(cfg, seed=9)
    params = {k: v.detach().clone() for k, v in hf.named_parameters()}
    batch = b2.synthetic_mlm_batch(cfg, 2, 128, 4, padded=True)
    out = hf(input_ids=batch["input_ids"], token_type_ids=batch["token_type_ids"],
             attention_mask=batch["attention_mask"], labels=batch["label"])
    out.loss.backward()
    loss, logits, grads = mlm.loss_and_grads(params, cfg, batch)
    assert abs(float(loss) - float(out.loss)) < 1e-5
    assert torch.allclose(logits, out.logits.detach(), atol=1e-4, rtol=1e-4)
    for n, p in hf.named_parameters():
        ref = p.grad if p.grad is not None else torch.zeros_like(p)
        assert torch.allclose(grads[n], ref, atol=1e-6, rtol=1e-4), n
    pad_row = grads["bert.embeddings.word_embeddings.weight"][0]
    assert float(pad_row.abs().sum()) > 0      # the decoder part reaches the pad row
