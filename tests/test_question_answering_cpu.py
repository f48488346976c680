"""CPU: BertForQuestionAnswering's host side -- the QA oracle against HF's class (logits, loss and gradients under
every clamp case), the packed normaliser against HF run on each sequence unpadded, HF naming and checkpoints, the
packed position checks, the criterion rules, the span loss's argument checks, synthetic_qa_batch and the dev() /
test() span scoring."""
import ctypes
import json

import pytest
import torch
import torch.nn as nn

import qa_oracle as qa
from parity import b2, tiny_config
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import _hf_order, _Layout
from pytorch_distributed_nlp_b200.packing import pack_batch
from pytorch_distributed_nlp_b200.trainer import best_spans, check_qa_criterion, qa_scores, step_loss

S = 128


def _cfg(**kw):
    d = dict(num_labels=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    d.update(kw)
    return tiny_config(**d)


def clamp_case(case, B=4, seed=3):
    """(start_positions, end_positions) of a clamp case, B sequences of S tokens"""
    g = torch.Generator().manual_seed(seed)
    st = torch.randint(1, S // 2, (B,), generator=g)
    en = st + torch.randint(0, 10, (B,), generator=g)
    if case == "minus_one":
        st[0] = -1
    elif case == "minus_100":
        st[1], en[1] = -100, -100
    elif case == "last":
        st[2], en[2] = S - 1, S - 1
    elif case == "S":
        en[0] = S
    elif case == "S_plus_5":
        st[3], en[3] = S + 5, S + 5
    elif case == "all_ignored":
        st[:] = S
        en[:] = S + 7
    elif case == "start_ignored":
        st[:] = S + 1
    elif case == "b1":
        return st[:, None], en[:, None]
    return st, en


CLAMP_CASES = ["plain", "minus_one", "minus_100", "last", "S", "S_plus_5", "all_ignored", "start_ignored", "b1"]


@pytest.mark.parametrize("case", CLAMP_CASES)
def test_qa_oracle_equals_hf_forward_backward(case):
    """logits, loss and every gradient of the oracle against transformers.BertForQuestionAnswering"""
    cfg = _cfg()
    hf = qa.hf_qa_model(cfg)
    state = {k: v.detach().clone() for k, v in hf.named_parameters()}
    b = b2.synthetic_qa_batch(cfg, 4, S, 11, padded=True)
    b["start_positions"], b["end_positions"] = clamp_case(case)
    out = hf(input_ids=b["input_ids"], token_type_ids=b["token_type_ids"], attention_mask=b["attention_mask"],
             start_positions=b["start_positions"], end_positions=b["end_positions"])
    out.loss.backward()
    loss, start, end, grads = qa.loss_and_grads(state, cfg, b)
    assert start.shape == end.shape == (4, S)
    assert float((out.start_logits.detach() - start).abs().max()) < 2e-6
    assert float((out.end_logits.detach() - end).abs().max()) < 2e-6
    if case in ("all_ignored", "start_ignored"):
        assert torch.isnan(out.loss) and torch.isnan(loss)
    else:
        assert abs(float(out.loss.detach()) - float(loss)) < 2e-6
    assert set(grads) == {k for k, _ in hf.named_parameters()}
    for k, p in hf.named_parameters():
        assert torch.isfinite(grads[k]).all(), k
        assert float((grads[k] - p.grad).abs().max()) < 2e-6 + 1e-5 * float(p.grad.abs().max()), k
    if case == "all_ignored":
        # an all-ignored batch: NaN loss and a zero gradient
        assert all(float(g.abs().max()) == 0.0 for g in grads.values())


def test_packed_normaliser_is_hf_on_each_sequence_unpadded():
    """the packed loss -- each sequence's softmax over its own tokens, the two means over the batch -- equals HF's
    model run on every sequence alone, unpadded, with the per-sequence losses averaged as the batch loss does"""
    cfg = _cfg()
    hf = qa.hf_qa_model(cfg).eval()
    state = {k: v.detach().clone() for k, v in hf.named_parameters()}
    b = b2.synthetic_qa_batch(cfg, 6, S, 21, padded=True, ignored=0.3)
    lens = b["attention_mask"].sum(1)
    sp, ep = b["start_positions"], b["end_positions"]
    loss, start, end, _g = qa.loss_and_grads(state, cfg, b, packed=True)
    per_s, per_e = [], []
    with torch.no_grad():
        for i in range(6):
            n = int(lens[i])
            o = hf(input_ids=b["input_ids"][i:i + 1, :n], token_type_ids=b["token_type_ids"][i:i + 1, :n],
                   attention_mask=b["attention_mask"][i:i + 1, :n])
            # HF unpadded ignores positions >= n; packing passes exactly those >= S (the rest it rejects)
            for logit, p, acc in ((o.start_logits[0], sp[i], per_s), (o.end_logits[0], ep[i], per_e)):
                t = int(p.clamp(0, S))
                if t < S:
                    acc.append(torch.logsumexp(logit, 0) - logit[t])
    want = (torch.stack(per_s).mean() + torch.stack(per_e).mean()) / 2
    assert abs(float(loss) - float(want)) < 5e-6
    # and it is not the padded loss, whose softmax spreads mass over the padding logits
    padded = qa.span_loss(start, end, sp, ep)
    assert abs(float(padded) - float(want)) > 1e-3


@pytest.mark.parametrize("cfg_fn", [lambda: _cfg(), lambda: b2.chinese_bert_wwm_ext_config(num_labels=2)])
def test_named_parameters_are_hf_question_answering(cfg_fn):
    cfg = cfg_fn()
    hf = qa.hf_qa_model(cfg) if cfg.num_hidden_layers == 2 else None
    m = b2.BertForQuestionAnswering(cfg)
    names = [k for k, _ in m.named_parameters()]
    assert names == _hf_order(cfg, "question_answering")
    assert names[-2:] == ["qa_outputs.weight", "qa_outputs.bias"] and not any("pooler" in k for k in names)
    if hf is not None:
        assert names == [k for k, _ in hf.named_parameters()]
        for (k, p), (_k2, q) in zip(m.named_parameters(), hf.named_parameters()):
            assert p.shape == q.shape, k
    else:
        assert len(names) == 199


def test_layout_tail_is_qa_outputs_in_the_last_layer_bucket():
    cfg = _cfg()
    lay = _Layout(cfg, "question_answering")
    b, e, label = lay.buckets[-1]
    assert label == "layer1+head" and e == lay.total
    w_off, w_shape = lay.entries["qa_outputs.weight"]
    b_off, b_shape = lay.entries["qa_outputs.bias"]
    assert w_shape == (2, cfg.hidden_size) and b_shape == (2,)
    assert b <= w_off < b_off < e
    assert b2.BertForQuestionAnswering._anchor == "qa_outputs.bias"


def test_hf_state_dict_round_trips_strict():
    cfg = _cfg()
    hf = qa.hf_qa_model(cfg)
    m = b2.BertForQuestionAnswering(cfg)
    m.load_state_dict(hf.state_dict(), strict=True)
    sd = m.state_dict()
    for k, v in hf.state_dict().items():
        assert torch.equal(sd[k], v), k
    hf2 = qa.hf_qa_model(cfg, seed=9)
    hf2.load_state_dict({k: sd[k] for k in hf2.state_dict()}, strict=True)


@pytest.mark.parametrize("kind", ["pretraining", "qa"])
def test_from_pretrained_ignores_pooler_and_cls(tmp_path, kind):
    """the encoder loads; a pre-training checkpoint's pooler and cls.* are ignored and qa_outputs keeps its init, a QA
    checkpoint's qa_outputs loads"""
    cfg = _cfg()
    src = qa.hf_qa_model(cfg, seed=3)
    ckpt = dict(src.state_dict())
    if kind == "pretraining":
        ckpt = {k: v for k, v in ckpt.items() if not k.startswith("qa_outputs.")}
        ckpt["cls.predictions.bias"] = torch.zeros(cfg.vocab_size)
        ckpt["cls.seq_relationship.weight"] = torch.zeros(2, cfg.hidden_size)
        ckpt["bert.pooler.dense.weight"] = torch.zeros(cfg.hidden_size, cfg.hidden_size)
    torch.save(ckpt, tmp_path / "pytorch_model.bin")
    torch.manual_seed(11)
    fresh = b2.BertForQuestionAnswering(cfg)
    torch.manual_seed(11)
    m = b2.BertForQuestionAnswering.from_pretrained(str(tmp_path), config=cfg)
    sd = m.state_dict()
    for k, v in src.state_dict().items():
        if k.startswith("bert."):
            assert torch.equal(sd[k], v), k
    for k in ("qa_outputs.weight", "qa_outputs.bias"):
        want = fresh.state_dict()[k] if kind == "pretraining" else src.state_dict()[k]
        assert torch.equal(sd[k], want), k
    assert not any("pooler" in k or k.startswith("cls.") for k in sd)


def test_save_pretrained_round_trip_and_architectures(tmp_path):
    cfg = _cfg()
    m = b2.BertForQuestionAnswering.from_config(cfg, seed=4)
    m.save_pretrained(str(tmp_path))
    with open(tmp_path / "config.json") as f:
        c = json.load(f)
    assert c["architectures"] == ["BertForQuestionAnswering"] and c["num_labels"] == 2
    m2 = b2.BertForQuestionAnswering.from_pretrained(str(tmp_path))
    for (k, a), (k2, b_) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k == k2 and torch.equal(a, b_)


@pytest.mark.parametrize("n", [1, 3, 6])
def test_num_labels_other_than_two_raise(n):
    with pytest.raises(ValueError, match="exactly 2"):
        b2.BertForQuestionAnswering(_cfg(num_labels=n))


def test_output_is_hf_tuple_order():
    o = b2.QuestionAnsweringModelOutput(loss=1, start_logits=2, end_logits=3)
    assert tuple(o) == (1, 2, 3) and o[0] == 1 and o["end_logits"] == 3 and len(o) == 3
    o = b2.QuestionAnsweringModelOutput(start_logits=2, end_logits=3)
    assert tuple(o) == (2, 3) and o[0] == 2


def test_model_forward_needs_cuda():
    m = b2.BertForQuestionAnswering(_cfg())
    with pytest.raises(RuntimeError, match="CUDA"):
        m(input_ids=torch.zeros(1, S, dtype=torch.int64))


def test_pack_batch_positions_pass_through_and_rejections():
    cfg = _cfg()
    b = b2.synthetic_qa_batch(cfg, 8, S, 5, padded=True)
    ids, tt, mask = b["input_ids"], b["token_type_ids"], b["attention_mask"]
    sp, ep = b["start_positions"].clone(), b["end_positions"].clone()
    sp[0], ep[1] = -3, S + 40                # negative and >= S pass through; the kernel clamps them as HF does
    p = pack_batch(ids, tt, mask, 128, start_positions=sp, end_positions=ep[:, None])
    assert torch.equal(p["start_positions"], sp) and torch.equal(p["end_positions"], ep) and p["seq_len"] == S
    # each sequence's tokens keep their order from cls_index on: a position indexes the same token
    flat = p["input_ids"].view(-1)
    for i in range(8):
        if 0 <= int(sp[i]) < S:
            assert int(flat[p["cls_index"][i] + sp[i]]) == int(ids[i, sp[i]])
    lens = mask.sum(1)
    bad = sp.clone()
    bad[2] = int(lens[2])                   # the first padding token of row 2
    with pytest.raises(ValueError, match="padding token"):
        pack_batch(ids, tt, mask, 128, start_positions=bad, end_positions=ep)
    bad = ep.clone()
    bad[4] = S - 1 if int(lens[4]) < S else 0
    if int(lens[4]) < S:
        with pytest.raises(ValueError, match="end_positions"):
            pack_batch(ids, tt, mask, 128, start_positions=sp, end_positions=bad)
    with pytest.raises(ValueError, match="together"):
        pack_batch(ids, tt, mask, 128, start_positions=sp)
    with pytest.raises(ValueError, match="int64"):
        pack_batch(ids, tt, mask, 128, start_positions=sp.float(), end_positions=ep)
    with pytest.raises(ValueError, match="int64"):
        pack_batch(ids, tt, mask, 128, start_positions=sp[:3], end_positions=ep)
    assert "start_positions" not in pack_batch(ids, tt, mask, 128)


def test_criterion_rules_for_a_qa_model():
    m = b2.BertForQuestionAnswering(_cfg())
    for ok in (None, nn.CrossEntropyLoss()):
        check_qa_criterion(ok)
        assert step_loss(m, ok) is None
    for bad in (nn.MSELoss(), nn.BCEWithLogitsLoss(), nn.CrossEntropyLoss(weight=torch.ones(2)),
                nn.CrossEntropyLoss(label_smoothing=0.1), nn.CrossEntropyLoss(ignore_index=0),
                nn.CrossEntropyLoss(reduction="sum")):
        with pytest.raises(ValueError, match="span loss"):
            step_loss(m, bad)
        with pytest.raises(ValueError, match="span loss"):
            b2.Trainer(b2.Args(), m.config, m, bad, None)
    tr = b2.Trainer(b2.Args(), m.config, m, None, None)
    assert tr.problem_type(None) == "question_answering"
    assert getattr(m.config, "problem_type", None) is None
    assert b2.Args.max_answer_length == 30


def test_span_loss_entry_point_is_declared_and_checks_arguments():
    assert "b2_qa_span_loss" in L._SIGNATURES and "b2_qa_span_loss" in L.EXPORTED_SYMBOLS
    lib = L.load()
    one = ctypes.c_void_p(256)   # never dereferenced: every case fails its checks before a launch
    odd = ctypes.c_void_p(260)
    cases = [  # logits, rows, starts, ends, nseq, ignored, first, len, d_logits, expected message
        (None, 512, one, one, 4, 128, None, None, None, "null pointer"),
        (one, 512, None, one, 4, 128, None, None, None, "null pointer"),
        (odd, 512, one, one, 4, 128, None, None, None, "aligned"),
        (one, 512, one, one, 4, 128, None, None, odd, "aligned"),
        (one, 0, one, one, 4, 128, None, None, None, "rows"),
        (one, 512, one, one, 0, 128, None, None, None, "num_seqs"),
        (one, 512, one, one, 513, 128, None, None, None, "num_seqs"),
        (one, 512, one, one, 4, 0, None, None, None, "ignored_index"),
        (one, 1026, one, one, 2, 513, None, None, None, "ignored_index"),
        (one, 512, one, one, 4, 128, one, None, None, "together"),
        (one, 512, one, one, 4, 128, None, one, None, "together"),
        (one, 500, one, one, 4, 128, None, None, None, "padded rows"),
    ]
    for logits, rows, st, en, nseq, ign, first, ln, dl, what in cases:
        r = lib.b2_qa_span_loss(logits, rows, st, en, nseq, ign, first, ln, None, one, dl, None, None)
        assert r != 0 and what in L.last_error(), (what, L.last_error())


def test_synthetic_qa_batch_is_reproducible_and_squad_shaped():
    cfg = _cfg()
    a = b2.synthetic_qa_batch(cfg, 64, S, 7, padded=True)
    b = b2.synthetic_qa_batch(cfg, 64, S, 7, padded=True)
    c = b2.synthetic_qa_batch(cfg, 64, S, 8, padded=True)
    assert all(torch.equal(a[k], b[k]) for k in a) and not torch.equal(a["input_ids"], c["input_ids"])
    sp, ep, mask, tt, ids = a["start_positions"], a["end_positions"], a["attention_mask"], a["token_type_ids"], \
        a["input_ids"]
    assert sp.dtype == ep.dtype == torch.int64 and sp.shape == (64,)
    lens = mask.sum(1)
    n_null = n_ign = n_span = 0
    for i in range(64):
        n = int(lens[i])
        assert int(ids[i, 0]) == 101 and int(ids[i, n - 1]) == 102 and int(tt[i, 0]) == 0 and int(tt[i, n - 1]) == 1
        q = int((tt[i, :n] == 0).sum()) - 2          # [CLS] q... [SEP]
        assert 2 <= q <= 8 and int(ids[i, q + 1]) == 102
        s, e = int(sp[i]), int(ep[i])
        if s >= S or e >= S:
            n_ign += 1
        elif s == 0 and e == 0:
            n_null += 1
        else:
            n_span += 1
            assert q + 2 <= s <= e <= n - 2 and int(tt[i, s]) == 1
    assert n_null > 0 and n_ign > 0 and n_span > 0
    full = b2.synthetic_qa_batch(cfg, 4, S, 7)
    assert bool((full["attention_mask"] == 1).all())


def test_best_spans_and_scores():
    """run_qa.py's rule: the best start + end with s <= e < s + max_answer_length over valid tokens; (0, 0) wins when
    [CLS] scores best; exact match and position-level F1 by hand"""
    st = torch.full((3, 8), -5.0)
    en = torch.full((3, 8), -5.0)
    st[0, 2], en[0, 4] = 3.0, 3.0          # span (2, 4)
    st[1, 5], en[1, 1] = 9.0, 9.0          # end before start is not a span: the best valid pair
    en[1, 6] = 1.0
    st[2, 0], en[2, 0] = 4.0, 4.0          # no answer
    st[2, 6], en[2, 7] = 9.0, 9.0          # ... unless padding could be chosen: it is masked
    mask = torch.ones(3, 8, dtype=torch.int64)
    mask[2, 5:] = 0
    got = best_spans(st, en, mask, max_answer_length=30)
    assert got.tolist() == [[2, 4], [5, 6], [0, 0]]
    # max_answer_length bounds e - s
    st2, en2 = torch.zeros(1, 8), torch.zeros(1, 8)
    st2[0, 1], en2[0, 7] = 5.0, 5.0
    en2[0, 2] = 1.0
    assert best_spans(st2, en2, None, max_answer_length=3).tolist() == [[1, 2]]
    rows = torch.tensor([[2, 4, 2, 4], [5, 6, 4, 6], [0, 0, 3, 3]])
    em, f1 = qa_scores(rows)
    assert em == pytest.approx(1 / 3)
    # row 2: overlap 2, precision 1, recall 2/3 -> 0.8; row 3: no overlap -> 0
    assert f1 == pytest.approx((1.0 + 0.8 + 0.0) / 3)
