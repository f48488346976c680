"""GPU: BertForMaskedLM -- the masked-LM head kernels (csrc/mlm_head.cu) against float64, the model against the
masked-LM oracle (tests/mlm_oracle.py), the eager full-logit path against the labelled-rows path, the tied
word-embedding gradient, the vocabulary padding under every optimizer, determinism, checkpoints and the Trainer.

Kernel bounds.  fp32 unit roundoff u = 2^-24, bf16 2^-8 relative.  The cross-entropy kernel's log-sum-exp over V
columns adds V terms of at most 1 (each exp within a few u of exact), so lse is off by at most (V + 8) u relative to
the sum, i.e. (V + 8) u absolute in the log; a row loss lse - x_y is then off by that plus u |lse|.  d_logits is one
bf16 rounding (2^-8 |ref|) of a value whose fp32 error is a few u times the scale, plus u |ref| for the one fp32 add of
the dense form's incoming gradient (d_extra).  check_mlm_ce holds these bounds; the training step's stage test
(test_step_stages.py) applies them to the recorded launches.  The kernels are also run at their edges: argmax ties
(torch's first occurrence), logits spanning +-1e4 and all-equal rows, means over rows past the 1024-thread stride,
the 1024-thread compaction chunks, the gather / scatter thread-count limits, the GELU' and bias-fill grid strides,
and every host-side argument rule.  The in-kernel traps (a label out of range, more labelled rows than the capacity)
are not run: the host's mlm_capacity rejects both first.
"""
import numpy as np
import pytest
import torch
import torch.nn as nn

import mlm_oracle as mlm
from parity import TOL_GRAD_REL_QK, TOL_LOSS, assert_grads_within_tolerance, b2, tiny_config
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import vocab_pad
from test_gemm_reference import U, bf_bound, gelu_grad64, gelu_grad_err

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


def _ce(logits, labels, rows, V, n_rows, d_loss=None, with_dl=True, extra=None, n_lab=None):
    """b2_mlm_ce on poisoned outputs; labels None: the extra-only form; n_rows None: every row live; n_lab None: the
    labelled live rows' count"""
    Vp = logits.shape[1]
    dev = logits.device
    lab = None if labels is None else torch.tensor(labels, dtype=torch.int32, device=dev)
    n_rows_t = None if n_rows is None else torch.tensor([n_rows], dtype=torch.int32, device=dev)
    if n_lab is None:
        live = torch.arange(rows, device=dev) < (rows if n_rows is None else n_rows)
        n_lab = int(((lab >= 0) & live).sum())
    n_lab_t = torch.tensor([n_lab], dtype=torch.int32, device=dev)
    row_loss = torch.full((rows,), float("nan"), device=dev)
    pred = torch.full((rows,), -7, dtype=torch.int32, device=dev)
    dl = torch.full((rows, Vp), float("nan"), dtype=torch.bfloat16, device=dev) if with_dl else None
    loss = torch.full((), float("nan"), device=dev)
    L.call("b2_mlm_ce", logits.data_ptr(), rows, V, Vp, L.ptr(lab), L.ptr(n_rows_t), n_lab_t.data_ptr(),
           L.ptr(d_loss), L.ptr(extra), 0 if extra is None else extra.shape[1], row_loss.data_ptr(), pred.data_ptr(),
           L.ptr(dl), loss.data_ptr(), _stream())
    torch.cuda.synchronize()
    return row_loss, pred, dl, loss, n_lab


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        raise AssertionError("%s: %d elements over the bound, worst error / bound %.3g" % (
            what, int(bad.sum()), float((err / bound.clamp_min(1e-300)).max())))


def check_mlm_ce(logits, labels, V, n_lab, d_loss=1.0, extra=None, n_rows=None, row_loss=None, pred=None, dl=None,
                 loss=None, what="mlm ce", check=_within):
    """b2_mlm_ce's outputs against float64 from the fp32 logits [rows, vocab_pad] it read and its int labels [rows]
    (-1: no loss term; None: the extra-only form).  n_rows: rows at or past it are capacity padding (None: every row
    is live); n_lab: the mean's divisor; d_loss: the loss part's scale; extra: the fp32 [rows, V] added onto d_logits.
    Bounds as in the module docstring: row loss (V + 8) u + u |lse|, twice; the mean that plus rows u max |row|;
    d_logits one bf16 rounding of a value within 16 u d_loss / n of the exact one, plus one fp32 add of extra.  pred
    exactly torch's argmax over the first V columns (its first occurrence), d_logits columns V..vocab_pad and the
    padding rows exactly 0.  check: the within(got, ref, bound, what) that asserts and reports."""
    rows, dev = logits.shape[0], logits.device
    x = logits.double()[:, :V]
    live_row = torch.arange(rows, device=dev) < (rows if n_rows is None else n_rows)
    lab = torch.full((rows,), -1, dtype=torch.long, device=dev) if labels is None else labels.long()
    live = live_row & (lab >= 0)
    lse = torch.logsumexp(x, 1)
    zero = torch.zeros_like(lse)
    ref_row = torch.where(live, lse - x.gather(1, lab.clamp(min=0)[:, None])[:, 0], zero)
    bound = torch.where(live, ((V + 8) * U32 + U32 * lse.abs()) * 2, zero)
    if row_loss is not None:
        check(row_loss, ref_row, bound, what + " row_loss")
    if loss is not None:
        ref_loss = (ref_row.sum() / n_lab).reshape(1)
        check(loss.reshape(1), ref_loss, (bound.max() + rows * U32 * ref_row.abs().max()).reshape(1), what + " loss")
    if pred is not None:
        ref_pred = torch.where(live, x.argmax(1), torch.full_like(lab, -1))
        bad = pred.long() != ref_pred
        assert not bool(bad.any()), "%s pred: %d rows differ, first %s" % (what, int(bad.sum()),
                                                                          bad.nonzero()[0].tolist())
    if dl is not None:
        got = dl.double()
        assert bool((got[:, V:] == 0).all()), what + " d_logits: a padding column is not 0"
        assert bool((got[~live_row] == 0).all()), what + " d_logits: a capacity padding row is not 0"
        onehot = torch.zeros_like(x)
        onehot[torch.arange(rows, device=dev), lab.clamp(min=0)] = 1
        ref = torch.where(live[:, None], (torch.softmax(x, 1) - onehot) * (d_loss / n_lab), torch.zeros_like(x))
        E = torch.where(live, zero + 16 * U32 * abs(d_loss) / n_lab, zero)[:, None]
        if extra is not None:
            ref = ref + torch.where(live_row[:, None], extra.double(), torch.zeros_like(x))
            E = E + U32 * ref.abs()            # the one fp32 add of extra
        check(got[:, :V], ref, 2.0 ** -8 * ref.abs() + E, what + " d_logits")


def _tie_logits(rows, V, Vp, gen):
    """integer-valued logits whose maximum 30 repeats: within one thread's float4, at one thread's next 1024-column
    stride, across lanes of a warp, across warps, at columns 0 and V-1; then V-1 alone and 0 alone"""
    x = torch.randint(-20, 21, (rows, Vp), generator=gen).double()
    ties = [(4000, 4001), (4000, 5024), (8, 20), (100, 900), (100, 900, 20000), (0, V - 1), (V - 1,), (0,),
            (1023, 1024), (V - 5, V - 2)]
    for r in range(rows):
        for c in ties[r % len(ties)]:
            x[r, c] = 30
    return x


@gpu
@pytest.mark.parametrize("V, form", [pytest.param(64, "loss", id="64"), pytest.param(21128, "loss", id="21128"),
                                     pytest.param(30522, "loss", id="30522"),
                                     pytest.param(1050, "extra", id="extra-1050"),
                                     pytest.param(1050, "extra_only", id="extra_only-1050"),
                                     pytest.param(21128, "ties", id="ties-21128"),
                                     pytest.param(21128, "wide", id="wide-21128"),
                                     pytest.param(1050, "mean1025", id="mean1025-1050"),
                                     pytest.param(1050, "mean4096", id="mean4096-1050")])
def test_ce_kernel_against_float64(V, form):
    """loss: the labelled-rows form (loss, row losses, argmax, d_logits, capacity padding rows).  extra: the dense
    backward's form, labels + d_loss + extra with some rows ignored, at ld_extra = V with V % 4 = 2 (the column
    break inside a float4); extra_only: the extra alone (labels null).  ties: integer logits whose maximum repeats
    within a thread, across the thread stride, lanes and warps, and at columns 0 and V-1.  wide: rows spanning
    +-1e4, and rows of all-equal logits.  mean1025 / mean4096: the mean over rows past the 1024-thread stride, and
    its bitwise repeatability."""
    torch.manual_seed(V)
    gen = torch.Generator().manual_seed(V + len(form))
    Vp = vocab_pad(V)
    rows, n_rows = 300, 261            # 300 is no multiple of any block size; rows past 261 are capacity padding
    if form.startswith("mean"):
        rows = n_rows = int(form[4:])
    if form == "ties":
        x = _tie_logits(rows, V, Vp, gen)
    elif form == "wide":
        x = (torch.rand(rows, Vp, generator=gen, dtype=torch.float64) * 2 - 1) * 1e4
        x[::3] = 5.0                   # all-equal rows
        x[1::6] = -7.25
    else:
        x = torch.randn(rows, Vp, dtype=torch.float64, generator=gen) * 3
    x[:, V:] = 1e4                     # the padded columns must not be read into the softmax
    labels = torch.randint(0, V, (rows,), generator=gen)
    labels[::7] = -1                   # ignored rows
    lx = x.float().to(DEV)
    d_loss = torch.tensor(1.7, device=DEV)
    extra = None
    if form.startswith("extra"):
        n_rows = None
        extra = (torch.randn(rows, V, generator=gen) * 1e-3).to(DEV)
    if form == "extra_only":
        row_loss, pred, dl, loss, n = _ce(lx, None, rows, V, None, None, extra=extra, n_lab=1)
        check_mlm_ce(lx, None, V, 1, extra=extra, row_loss=row_loss, pred=pred, dl=dl, what="extra only")
        return
    row_loss, pred, dl, loss, n = _ce(lx, labels.tolist(), rows, V, n_rows, d_loss, extra=extra)
    check_mlm_ce(lx, labels.to(DEV), V, n, d_loss=1.7, extra=extra, n_rows=n_rows, row_loss=row_loss, pred=pred,
                 dl=dl, loss=loss, what=form)
    if form == "ties":
        # every tie pattern reached a labelled row (check_mlm_ce asserted each against torch's first occurrence)
        assert set(pred[labels.to(DEV) >= 0].tolist()) >= {4000, 8, 100, 0, V - 1, 1023, V - 5}
    if form.startswith("mean"):
        again = _ce(lx, labels.tolist(), rows, V, n_rows, d_loss, extra=extra)
        for a, b in zip((row_loss, pred, dl, loss), again[:4]):
            assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a,
                               b.view(torch.int16) if b.dtype == torch.bfloat16 else b)


@gpu
def test_ce_kernel_all_ignored_is_nan_with_zero_gradient():
    V, rows = 21128, 128
    lx = torch.randn(rows, vocab_pad(V), device=DEV)
    row_loss, pred, dl, loss, n = _ce(lx, [-1] * rows, rows, V, 100)
    assert n == 0 and torch.isnan(loss)
    assert torch.all(dl.float() == 0) and torch.all(pred == -1) and torch.all(row_loss == 0)


@gpu
def test_compaction_exact():
    """15% of 4096 tokens labelled into a capacity of 768 rows; gather and scatter at H = 256"""
    _compaction_case((4096, 768, -100, "sparse", 256, 256), seed=1)


# (tokens, capacity, ignore_index, labels, gather hidden, scatter hidden): the 1024-thread chunk edges with every token
# labelled (capacity == tokens), labels 0 and V-1, ignore_index -1 and 0, and the gather / scatter thread-count limits
COMPACT_EDGES = [(1, 1, -1, "all", 8, 4096), (1000, 1000, -1, "all", 1024, 1024), (1024, 1024, -1, "all", 8, 4096),
                 (1025, 1025, -1, "all", 1024, 1024), (3073, 3073, -1, "all", 256, 4096),
                 (3073, 3072, 0, "zero_ignored", 8, 1024)]


@gpu
@pytest.mark.parametrize("case", COMPACT_EDGES, ids=lambda c: "%d-%d-%s-%d-%d" % (c[0], c[1], c[3], c[4], c[5]))
def test_compaction_edges(case):
    _compaction_case(case, seed=case[0] + case[1])


def _compaction_case(case, seed):
    """b2_mlm_compact exactly (rows, slots, slot labels, count), then gather and scatter around it"""
    M, cap, ignore, kind, Hg, Hs = case
    torch.manual_seed(seed)
    V = 21128
    if kind == "sparse":
        lab = torch.full((M,), -100, dtype=torch.int64)
        pick = torch.rand(M) < 0.15
        lab[pick] = torch.randint(0, V, (int(pick.sum()),))
    else:
        lab = torch.randint(0, V, (M,))
        lab[::5] = 0
        lab[1::5] = V - 1
        pick = lab != ignore
    n = int(pick.sum())
    assert n <= cap and (kind != "all" or n == cap)
    d = lab.to(DEV)
    rows = torch.full((cap,), -7, dtype=torch.int32, device=DEV)
    slot = torch.full((M,), -7, dtype=torch.int32, device=DEV)
    slab = torch.full((cap,), -7, dtype=torch.int32, device=DEV)
    cnt = torch.full((1,), -7, dtype=torch.int32, device=DEV)
    L.call("b2_mlm_compact", d.data_ptr(), M, ignore, V, cap, rows.data_ptr(), slot.data_ptr(), slab.data_ptr(),
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
    x = torch.randn(M, Hg, device=DEV).to(torch.bfloat16)
    g = torch.full((cap, Hg), float("nan"), dtype=torch.bfloat16, device=DEV)
    L.call("b2_mlm_gather_rows", x.data_ptr(), rows.data_ptr(), cnt.data_ptr(), cap, Hg, g.data_ptr(), _stream())
    src = torch.randn(cap, Hs, device=DEV)
    dx = torch.full((M, Hs), float("nan"), device=DEV)
    L.call("b2_mlm_scatter_rows", src.data_ptr(), slot.data_ptr(), M, Hs, dx.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert torch.equal(g[:n], x[idx.to(DEV)]) and torch.all(g[n:] == 0)
    ref = torch.zeros(M, Hs, device=DEV)
    ref[idx.to(DEV)] = src[:n]
    assert torch.equal(dx, ref)


GELU_BWD_STRIDE = 132 * 16 * 256 * 8      # elements per pass of b2_mlm_gelu_bwd's grid-stride loop


@gpu
@pytest.mark.parametrize("n", [8, 2 * GELU_BWD_STRIDE + 8 * 37])
def test_gelu_bwd_kernel_against_float64(n):
    """du = bf16(dg gelu'(u)) against float64: one fp32 product and one bf16 rounding of the erf GELU' the GEMM's
    EPI_GELU_BWD uses, u over [-10, 10] with 0 and the bf16 extremes, n = 8 and past two grid strides"""
    gen = torch.Generator().manual_seed(n)
    u = (torch.rand(n, generator=gen) * 20 - 10).to(torch.bfloat16)
    edges = torch.tensor([0.0, -0.0, 10.0, -10.0, 3.3895313892515355e38, -3.3895313892515355e38, 1.1754943508222875e-38,
                          -1.1754943508222875e-38], dtype=torch.bfloat16)
    u[:edges.numel()] = edges
    u[-edges.numel():] = edges.flip(0)
    dg = torch.randn(n, generator=gen) * 4
    du = torch.full((n,), float("nan"), dtype=torch.bfloat16, device=DEV)
    ud, dgd = u.to(DEV), dg.to(DEV)
    L.call("b2_mlm_gelu_bwd", dgd.data_ptr(), ud.data_ptr(), n, du.data_ptr(), _stream())
    torch.cuda.synchronize()
    x = ud.double()
    r = dgd.double() * gelu_grad64(x)
    _within(du, r, bf_bound(r, dgd.double().abs() * gelu_grad_err(x) + U * r.abs()), "gelu_bwd n=%d" % n)


@gpu
@pytest.mark.parametrize("rows", [1, 3, 2100])
def test_bias_fill_kernel_exact(rows):
    """logits[r, c] = float(bias[c]) over vocab_pad = 1088 (17 x 64, 8.5 x 128) columns; 2100 rows wrap the
    grid-stride loop"""
    Vp = 1088
    bias = torch.randn(Vp, device=DEV).to(torch.bfloat16)
    logits = torch.full((rows + 1, Vp), float("nan"), device=DEV)
    L.call("b2_mlm_bias_fill", bias.data_ptr(), rows, Vp, logits.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert torch.equal(logits[:rows], bias.float()[None].expand(rows, Vp))
    assert bool(torch.isnan(logits[rows]).all())      # nothing past the rows


@gpu
def test_entry_points_reject_bad_arguments():
    """each argument rule of the b2_mlm_* entry points raises RuntimeError on the host, before any launch"""
    i32, dev = torch.int32, DEV
    lab = torch.zeros(64, dtype=torch.int64, device=dev)
    ib = torch.zeros(256, dtype=i32, device=dev)
    fb = torch.zeros(256 * 1088, device=dev)
    bb = torch.zeros(256 * 64, dtype=torch.bfloat16, device=dev)
    p, s = lambda t: t.data_ptr(), _stream()
    bad = [("b2_mlm_compact", (p(lab), 64, -100, 1000, 65, p(ib), p(ib), p(ib), p(ib), s), "capacity"),
           ("b2_mlm_gather_rows", (p(bb), p(ib), p(ib), 4, 12, p(bb), s), "hidden"),
           ("b2_mlm_scatter_rows", (p(fb), p(ib), 4, 6, p(fb), s), "hidden"),
           ("b2_mlm_bias_fill", (p(bb), 4, 1000, p(fb), s), "vocab_pad"),
           ("b2_mlm_ce", (p(fb), 4, 1000, 1000, p(ib), None, p(ib), None, None, 0, p(fb), None, p(bb), None, s),
            "vocab"),
           ("b2_mlm_ce", (p(fb), 4, 1000, 1088, p(ib), None, p(ib), None, None, 0, p(fb), None, p(bb), None, s),
            "vocab"),
           ("b2_mlm_ce", (p(fb), 4, 1000, 1024, p(ib), None, p(ib), None, p(fb), 1000, p(fb), None, None, None, s),
            "d_extra")]
    torch.cuda.synchronize()
    before = L.launch_count()
    for name, args, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            L.call(name, *args)
    torch.cuda.synchronize()
    assert L.launch_count() == before


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
