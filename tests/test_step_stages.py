"""One training step, stage by stage: every launch of _Engine.forward and _Engine._backward_from_dlogits element-wise
against a float64 restatement computed from that launch's own recorded inputs ("teacher-forced"), so every bound is a
single-kernel bound and no model-depth amplification enters.

Recorder.  _lib.call is replaced for one step.  Every pointer argument is mapped back, by address range, to a
workspace tensor, a parameter span of `shadow` / `grads` (query | key | value as one span), `bias_acc`, the det
buffers or an input tensor; a pointer it cannot map fails the test, so a launch added later cannot go unchecked.
The recorder synchronises the device around every launch and clones what the launch may read and write before and
after it (the clones are done before the launch, which may run on the other stream), so the side stream's operands are
the values present at the fork and its outputs are read once it is done.  The masked-LM backward hands its kernels
the gradients autograd passes the model: tensor hooks on the output's loss and logits register them as step inputs.
One pointer is mapped by exception: the int32 labels the dense masked-LM cross-entropy builds on the fly, whose
values the recorder copies (b2_copy_async) at the launch; any other unmappable pointer still fails.
That serialisation can hide a race between the weight-gradient stream and the main stream; the comparisons against
unrecorded and captured steps (below) are what catch one.

Poison.  Before the recorded step, every workspace tensor of the step's shape, dq_accum, dq_parts, the LayerNorm
partials, the masked-LM head's buffers and decoder part (int32 buffers: -7) and the whole bf16 gradient space are
filled with NaN (rng, owner, bias_acc and the head's column-sum scratch keep their state).  An
element a launch should have rewritten and did not fails its check.  After the step bias_acc must be all zero again.

Wiring.  Each check first asserts which buffers the launch reads and writes (layer l's QKV GEMM reads layer l-1's x2,
its attention reads layer l's qkv, the parity buffer set of layer l is l & 1, ...), and the dropout site and step it
uses (0, 1+3l, 2+3l, 3+3l, 1+3L; seed and step read from eng.rng).  Then its outputs against float64:

  GEMMs           layer A of test_gemm_reference: |acc - A64 B64| <= C_ACC K U S, S = |A64| @ |B64| (the engine's
                  fp32 accumulator is not visible), plus the epilogue terms of that file's layer B: EPI_BIAS one fp32
                  add (U |t|); BIAS_GELU aux_out u that way and h = gelu64(u) at gelu_err(u); BIAS_DROPOUT_RESIDUAL
                  keep sc (E + U |t|) + 2U (|t sc| + |r|); GELU_BWD |acc| gelu_grad_err(u) + E |gelu'| + U |ref|;
                  ACCUM_F32 onto the recorded prior value, E + SPLITS U (|R| + S) with at most SPLITS = 8 split-K
                  slices (choose_config's cap in gemm.cu); the weight gradients, grouped or split, E + SPLITS U S.  Every bf16 store then
                  gets bf_bound(ref, E) = UB |ref| + (1 + UB) E.  The GELU_BWD colsum into bias_acc:
                  gamma(32 + ceil(M / 32)) sum |dU| (test_gemm_reference).
  dense + LN      fused (b2_gemm_ln_fwd): z = keep sc (A W^T + bias) + the previous block's fp32 output, within
                  Ez = keep sc (E + U |t|) + 2U (|t sc| + |r|); D = bf16(z) at bf_bound; statistics, y_f32 and y by
                  test_gemm_ln_reference.stats_bound / ln_fwd_check with ez = Ez; y == bf16(y_f32).  Unfused: the
                  BIAS_DROPOUT_RESIDUAL GEMM as above, then test_step_kernels.ln_fwd_check on its bf16 z.
  attention       test_attention_reference.check_outputs on the recorded qkv, dctx, ctx, lse (its bounds include the
                  nkv fp32 atomics of dQ above 128 tokens, in any order, which also covers the ordered slices); the
                  stored keep bits at 128 tokens bitwise against the Philox replica; the QKV bias accumulator by its
                  gamma(4 + 8 batch) bound.
  LN backward     test_step_kernels.ln_bwd_ref for the fp32 dx; dx_drop == bf16(keep dx sc) bitwise; the three column
                  sums with ln_bwd_sums_check's gamma(depth) bound, into bias_acc (accumulating form) or, det, through
                  the partial rows and b2_colsum_finish (depth + nparts + 9, then one bf16 rounding).
  b2_colsum       any summation order of n terms is within gamma(n - 1) of the sum: gamma(M) sum |x|, one bf16 store.
  b2_accum_finish grads == bf16(accumulator) bitwise and the accumulator zero, for exactly the segments of the layer
                  (the QKV one skipped when S != 128).
  embedding       ids32 / tt32 / pos32 and pre_ln exactly, LayerNorm by ln_fwd_check at site 0; backward as
                  test_step_kernels.check_embed_grads from the recorded dx; unused word / position rows exactly 0.
  head and loss   test_step_kernels.check_head_fwd / check_head_bwd / check_ce, and for the token head
                  test_token_classification.check_token_head_fwd / _bwd, at site 1 + 3L; the logits gradient the head
                  backward reads equals dloss_logits (in-model loss, d_loss = 1).
  masked-LM head  compaction (rows, slots, labels, count), gather (rows, zeros past the count), scatter (rows, zero
                  rows) and the bias fill (every row = the fp32 bias over vocab_pad columns) exactly; the transform
                  GEMM as BIAS_GELU, its LayerNorm by ln_fwd_check on the bf16 h; the projection, d_t, decoder and
                  d_x GEMMs as ACCUM_F32 onto the bias-filled logits or the zero b2_zero left (asserted); b2_mlm_ce
                  by test_masked_lm.check_mlm_ce (pred exact, d_logits columns V..vocab_pad and the capacity padding
                  rows exactly 0; the backward's row losses bitwise the forward's; the dense form's labels exactly
                  the step's with ignore_index -> -1, its incoming d_logits bitwise R); the head's LayerNorm backward
                  by ln_bwd_ref, dh_bf == bf16(dh), its partials through b2_colsum_finish (third target null);
                  b2_mlm_gelu_bwd at bf_bound(r, |dg| gelu_grad_err(u) + U |r|); the two bias column sums at
                  gamma(rows), the decoder bias's padding exactly 0; the split dW_t as a weight gradient; the tied
                  add bitwise bf16(pre + dec) over V H, pre the embedding backward's output, rows V..vocab_pad 0 and
                  the pad row bf16(dec[0]).  Streams: the decoder part, dW_t and the column sums on the
                  weight-gradient stream, the rest on the main one.
Every bound above is computed by the helper named, which takes this file's check as its check= callback.

Coverage ledger.  Every element of the flat gradient space is claimed by exactly one check (padding: zero in the
embedding bucket and in cls.predictions.bias's vocab_pad - V entries, untouched NaN elsewhere; the masked-LM word
table by the tied add, its embedding-backward value by check_embed_grads), and every (launch, workspace tensor) the
launch changed by exactly one check; both are asserted after the step.  expected_grad_claims() builds the ledger
from _Layout alone.

Race sensitivity.  The same step on a model loaded from the same state, with the same warm-up, poison and
seed_dropout(seed, step), runs again without the recorder.  In det mode its activations, gradient space and
embedding-backward input must be bitwise the recorded step's, and so must the gradient space after one replay of the
captured step (FusedTrainStep, or PackedTrainStep for packed bins), built on another such model with AdamW at lr 0
and replayed at the same dropout key (its backward starts from dloss_logits directly, the eager one from
0 + dloss_logits * 1: equal up to the sign of a zero, so gradients are compared by value; the captured masked-LM step
computes d_logits in the forward's cross-entropy launch, the eager one in the backward's).  mlm_dense skips the
captured comparison: the captured step's objective is the loss alone.  With atomics on, the backward's sums have no
fixed order, so only the forward's activations are compared bitwise (the loss, a mean over blocks, is left out).
A split-K vocabulary projection would make the logits and what is read from them non-bitwise; at these shapes the
automatic configuration did not split it, and the masked-LM forward buffers, logits included, compared bitwise.

Planted defects.  On a recorded step the reference side is altered on the host and the named check must fail: layer
l's weight gradients from layer l+2's operands, dropout at the neighbouring sublayer's site and at the previous step,
the bf16 residual in place of x1f on the fused path, one gradient element and one workspace row restored to the
previous step's values, the QKV bias gradient summed over one bin fewer; the tied add against the warm-up step's
decoder part, one gathered row restored to the warm-up step's, the cross-entropy reference on the neighbouring
slot's label.

Configurations, each with torch.use_deterministic_algorithms off and on: tiny (H 256, 3 layers, B 8 x 128, one
sequence of padding only; unfused LayerNorm), hidden768 (4 layers, B 32 x 128, dropout on and off; the cluster
LayerNorm, two parity reuses), large (H 1024, 3 layers, 16 heads, B 8), seq512 (padded B 4 x 512: dq_accum, b2_colsum,
segment seg0 + 1, the ordered dQ), packed128 and packed512 (pack_batch bins; packed attention, embedding, cls rows),
token128 and token512packed (BertForTokenClassification, 9 labels, padded B 16 x 128 and 512-token bins:
b2_token_head_fwd / _bwd_split, the per-token loss with ignored rows); BertForMaskedLM: mlm128 (V 21128, vocab_pad
21184 = 165.5 x 128, 2 layers, padded B 16 x 128 with dropout; the labelled count is no multiple of 128, so the
capacity has padding rows), mlm512packed (the same model, 8 sequences of up to 512 tokens in 512-token bins) and
mlm_dense (H 256, V 1050: vocab_pad 1088 = 17 x 64, V % 4 = 2; B 8 x 128 with one sequence of padding only, every real
token labelled, 768 = capacity; objective loss + (logits R).sum(), so the dense cross-entropy runs with labels,
d_loss and d_logits, and the head's backward writes dxA over every row).

Measured on an H100 80GB HBM3 (700 W power limit): worst error / bound per stage family and configuration, the larger
of the two modes ("-": the configuration has no such stage).  Columns: tiny, hidden768, hidden768 without dropout,
large, seq512, packed128, packed512, token128, token512packed.
                   tiny   h768  h768nd  large   s512   p128   p512   t128  t512p
  GEMM qkv         0.95   0.82   0.81   0.72   0.82   0.82   0.81   0.81   0.81
  GEMM u / h       0.94   0.82   0.81   0.72   0.81   0.82   0.82   0.81   0.82   (h: 0.971 everywhere)
  GEMM dU          0.93   0.81   0.81   0.74   0.83   0.81   0.81   0.81   0.82
  GEMM dctx        0.93   0.85   0.81   0.75   0.81   0.81   0.83   0.82   0.82
  ACCUM_F32 dx     0.028  0.0018 0.0019 0.0015 0.0022 0.0022 0.0022 0.0010 0.0011
  weight grads     0.93   0.76   0.78   0.94   0.89   0.86   0.86   0.88   0.79
  unfused z1 / z2  0.99   -      -      -      -      -      -      -      -
  LN fwd z         -      0.996  0.96   0.996  0.996  0.996  0.996  0.996  0.996
  LN fwd y         0.996  0.996  0.95   0.996  0.996  0.996  0.996  0.996  0.996
  LN fwd y_f32     -      0.46   0.0022 0.39   0.42   0.44   0.41   0.44   0.44
  LN fwd mean      0.012  4e-5   4e-5   2e-5   4e-5   4e-5   5e-5   3e-5   4e-5
  LN fwd rstd      0.12   4e-4   4e-4   2e-4   5e-4   4e-4   5e-4   4e-4   4e-4
  attention ctx    0.77   0.68   0.62   0.65   0.50   0.79   0.63   0.66   0.64
  attention lse    0.055  0.030  0.028  0.020  0.027  0.028  0.024  0.026  0.033
  attention dQ     0.69   0.59   0.71   0.69   0.45   0.86   0.50   0.79   0.61
  attention dK     0.94   0.97   0.94   0.97   0.93   0.95   0.94   0.71   0.59
  attention dV     0.89   0.95   0.96   0.93   0.94   0.95   0.95   0.64   0.60
  QKV bias acc     0.058  0.0089 0.011  0.038  -      0.018  -      0.017  -
  LN bwd dx        0.23   0.19   0.17   0.15   0.17   0.18   0.18   0.20   0.20
  LN bwd sums      0.98   0.98   0.98   0.99   0.99   0.97   0.98   0.98   0.98
  b2_colsum        0.94   0.87   0.86   0.97   0.96   0.92   0.94   0.93   0.93
  embed y          0.996  0.996  0.996  0.996  0.996  0.996  0.996  0.996  0.996
  embed y_f32      -      0.54   0.49   0.53   0.54   0.54   0.54   0.55   0.54
  embed mean       0.0084 0.0071 0.0071 0.0028 0.0089 0.0089 0.010  0.0052 0.0065
  embed rstd       0.10   0.067  0.067  0.045  0.062  0.065  0.063  0.054  0.077
  embed scratch_dx 0.994  0.996  0.995  0.995  0.995  0.996  0.995  0.996  0.996
  d_word / d_pos   0.996  0.996  0.996  0.996  0.996  0.996  0.996  0.996  0.996
  d_type           0.93   0.93   0.92   0.96   0.96   0.95   0.96   0.94   0.83
  d_gamma          0.95   0.93   0.93   0.97   0.96   0.94   0.94   0.98   0.95
  d_beta           0.92   0.95   0.95   0.99   0.97   0.98   0.94   0.95   0.95
  head pooled      0.98   0.99   0.98   0.97   0.94   0.98   0.98   -      -
  head logits      0.018  0.0096 0.0058 0.0071 0.0072 0.011  0.0078 -      -
  head gradients   0.995  0.991  0.993  0.995  0.995  0.991  0.995  -      -
  head d_hidden    0.0089 0.0044 0.0052 0.0031 0.0039 0.0046 0.0048 -      -
  token logits     -      -      -      -      -      -      -      0.016  0.016
  token d_hidden   -      -      -      -      -      -      -      0.40   0.39
  token dW / db    -      -      -      -      -      -      -      0.97   0.98
  loss             0.028  0.026  0.027  0.0096 0.019  0.0043 0.028  0.017  0.0078
  dloss_logits     0.15   0.18   0.19   0.20   0.13   0.32   0.24   0.37   0.30
The masked-LM head, same card and runs (columns mlm128, mlm512packed, mlm_dense; lab / full: the larger of the
labelled-row and every-row launches):
                   m128   m512p  mdense
  transform u      0.80   0.81   0.94
  transform h      0.97   0.97   0.97
  LN fwd y         0.996  0.996  0.996
  LN fwd mean      0.040  0.044  0.022
  LN fwd rstd      0.073  0.076  0.12
  logits           0.0021 0.0019 0.0027
  ce row_loss      4e-4   5e-4   0.0057
  ce loss          2e-5   4e-4   2e-4
  ce d_logits      0.58   0.52   0.996
  d_t              0.0092 0.0091 0.0012
  LN bwd dh        0.13   0.14   0.22
  LN bwd sums      0.98   0.95   0.91
  gelu bwd         0.99   0.99   0.99
  decoder dE       0.032  0.050  0.0012
  bias colsum      0.99   0.99   0.77   (decoder bias; the transform bias 0.91 / 0.88 / 0.74)
  dW_t             0.96   0.92   0.66
  d_x              0.0020 0.0020 0.0037
Compaction, gather, scatter, bias fill, pred and the tied add matched exactly everywhere.
Keep bits and accum_finish matched bitwise everywhere; every row with no visible key kept lse < -1e38.  The bf16
stores reach 0.99 because the half-ulp rounding itself dominates their bound.  Every det step was bitwise the
unrecorded one, and its gradient space bitwise (by value) the captured step's after one replay.  Every atomic-mode
forward was bitwise the unrecorded one.  Every planted defect failed its named check.  No check needed a new slack,
and no library defect showed.
Runtime, from one `pytest -m gpu tests/test_step_stages.py --durations=0` on that card: 25 tests in 76 s as pytest
counts it.  The first test takes 28 s, mostly CUDA start-up; token512packed takes 7 s; the others take 0.1-4 s.  The
masked-LM cases and defects add 9 tests and about 10 s of calls (mlm512packed 2.8 / 1.5 s, mlm128 1.7 / 1.3 s,
mlm_dense 0.3 / 0.3 s atomic / det, the three defects 1 s together, measured with tests/test_masked_lm.py in the same
run).
Every check reports to parity.report under tag "step_stages".
"""
import ctypes
from collections import OrderedDict

import numpy as np
import pytest
import torch

from parity import (b2, full_config, make_model, packed_visibility, padded_visibility, philox_keep_mask, report,
                    state_from_hf_init, tiny_config)
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import _Layout
from pytorch_distributed_nlp_b200.packing import pack_batch
from test_attention_reference import check_outputs
from test_determinism import _bits
from test_gemm_ln_reference import stats_bound
from mlm_oracle import mlm_state_from_hf_init
from test_gemm_reference import (C_ACC, U, bf_bound, drop_scale, gamma, gelu64, gelu_err, gelu_grad64,
                                 gelu_grad_err)
from test_masked_lm import check_mlm_ce
from test_packing import short_batch
from test_packing_long import long_batch
from test_step_kernels import check_ce, check_embed_grads, check_head_bwd, check_head_fwd, ln_bwd_ref, ln_fwd_check
from test_token_classification import check_token_head_bwd, check_token_head_fwd
from token_oracle import token_batch, token_state_from_hf_init

TAG = "step_stages"
bf, f32, f64 = torch.bfloat16, torch.float32, torch.float64
KM, MN = L.MAJOR_K, L.MAJOR_MN
SPLITS = 8                  # most split-K slices the GEMM's automatic configuration picks (gemm.cu)
SEED = 20261017
POISON64 = 0x5A5A5A5A5A5A5A5A   # int64 poison: neither all-keep nor all-drop bits
SCRATCH = ("head_scratch", "dq_accum", "dq_parts", "det_side", "split_ws", "partials")
WORD = "bert.embeddings.word_embeddings.weight"
MLM_BACKWARD = ("dlog", "dt", "dh", "dh_bf", "du", "dx")     # the masked-LM head buffers its backward writes


def f32eq(a, b):
    return np.float32(a) == np.float32(b)


# ======================================================================================================================
# the flat gradient space: spans and the ledger (CPU)
# ======================================================================================================================
def param_spans(lay):
    """OrderedDict name -> (begin, n): the layout's parameters, query | key | value of a layer as one span
    ('...attention.self.qkv.weight' / '.bias'), as the kernels address them"""
    out = OrderedDict()
    for name, (off, shape) in lay.entries.items():
        n = int(np.prod(shape))
        if ".attention.self.key." in name or ".attention.self.value." in name:
            continue
        if ".attention.self.query." in name:
            name = name.replace(".query.", ".qkv.")
            n *= 3
        out[name] = (off, n)
    return out


def family(name):
    if name.startswith("bert.embeddings."):
        return "embedding backward"
    if name.startswith(("bert.pooler.", "classifier.", "cls.")):
        return "head backward"
    if name.endswith(".weight") and "LayerNorm" not in name:
        return "weight gradient"
    if "LayerNorm" in name or name.endswith("output.dense.bias"):
        return "LayerNorm column sums"
    return "bias column sums"


def expected_grad_claims(lay):
    """[(begin, end, family)] tiling [0, lay.total): every parameter span by the check family that owns it, every
    round-8 gap by 'padding'"""
    claims, pos = [], 0
    for name, (b, n) in param_spans(lay).items():
        if b > pos:
            claims.append((pos, b, "padding"))
        claims.append((b, b + n, family(name)))
        pos = b + n
    if pos < lay.total:
        claims.append((pos, lay.total, "padding"))
    return claims


def zero_padding(lay, b, e):
    """whether the padding [b, e) of the gradient space reads exactly 0 after a step: the embedding bucket's (its
    b2_zero clears the whole bucket, the word table's vocab_pad - V masked-LM rows included) and the masked-LM
    cls.predictions.bias's entries V..vocab_pad (b2_colsum writes them; the optimizers rely on a zero gradient there).
    Any other padding is never written."""
    if e <= lay.buckets[0][1]:
        return True
    if lay.head == "mlm":
        ob, (V,) = lay.entries["cls.predictions.bias"]
        return (b, e) == (ob + V, ob + lay.vocab_pad)
    return False


def reserved_spans(lay):
    """param_spans with the masked-LM word table and cls.predictions.bias at their vocab_pad reserve: the span the
    vocabulary GEMMs and b2_colsum address"""
    spans = param_spans(lay)
    if lay.head == "mlm":
        H = lay.entries[WORD][1][1]
        for name, n in ((WORD, lay.vocab_pad * H), ("cls.predictions.bias", lay.vocab_pad)):
            spans[name] = (spans[name][0], n)
    return spans


def assert_tiles(claims, total):
    """the claims cover [0, total) once: no gap, no overlap"""
    pos = 0
    for b, e, what in sorted(claims):
        assert b == pos, "gradient elements [%d, %d) claimed %s" % (min(b, pos), max(b, pos),
                                                                  "twice" if b < pos else "by no check")
        assert e > b, what
        pos = e
    assert pos == total, "gradient elements [%d, %d) claimed by no check" % (pos, total)


class Regions:
    """address ranges -> (name, tensor, kind); the narrowest range containing an address wins"""

    def __init__(self):
        self.items = []

    def add(self, name, t, kind):
        if t is not None and t.numel():
            b = t.data_ptr()
            self.items.append((b, b + t.numel() * t.element_size(), name, t, kind))

    def covers(self, addr):
        return any(it[0] <= addr < it[1] for it in self.items)

    def find(self, addr):
        hits = [it for it in self.items if it[0] <= addr < it[1]]
        if not hits:
            raise AssertionError("pointer 0x%x maps to no tensor the step owns" % addr)
        b, _e, name, t, kind = min(hits, key=lambda it: it[1] - it[0])
        assert (addr - b) % t.element_size() == 0, "pointer 0x%x is inside an element of %s" % (addr, name)
        return name, (addr - b) // t.element_size()


@pytest.mark.parametrize("head", ["sequence", "token", "mlm"])
@pytest.mark.parametrize("layers", [0, 1, 3])
def test_ledger_tiles_the_gradient_space(head, layers):
    V = 1050 if head == "mlm" else 512                  # vocab_pad 1088: padding in the word table and the bias
    lay = _Layout(tiny_config(num_hidden_layers=layers, type_vocab_size=3, vocab_size=V), head=head)
    claims = expected_grad_claims(lay)
    assert_tiles(claims, lay.total)
    spans = param_spans(lay)
    assert sum(n for _b, n in spans.values()) == sum(int(np.prod(s)) for _o, s in lay.entries.values())
    fams = {f for _b, _e, f in claims}
    want = {"embedding backward", "head backward", "padding"}
    if layers:
        want |= {"weight gradient", "LayerNorm column sums", "bias column sums"}
    assert fams == want
    zero = [(b, e) for b, e, f in claims if f == "padding" and zero_padding(lay, b, e)]
    eb, ee, _ = lay.buckets[0]
    if head == "mlm":
        ow, ob, H = lay.off(WORD), lay.off("cls.predictions.bias"), 256
        assert lay.vocab_pad == 1088
        assert (ow + V * H, ow + 1088 * H) in zero and (ob + V, ob + 1088) in zero
        assert [z for z in zero if z[1] > ee] == [(ob + V, ob + 1088)]
        spans = reserved_spans(lay)
        assert spans[WORD] == (ow, 1088 * H) and spans["cls.predictions.bias"] == (ob, 1088)
    else:
        assert all(e <= ee for _b, e in zero)
    with pytest.raises(AssertionError, match="twice"):
        assert_tiles(claims + [claims[1]], lay.total)
    with pytest.raises(AssertionError, match="by no check"):
        assert_tiles(claims[:1] + claims[2:], lay.total)


def test_pointer_map():
    r = Regions()
    flat = torch.zeros(64, dtype=bf)
    r.add("flat", flat, "grad")
    r.add("g:a", flat[8:24], "grad")
    r.add("ws", torch.zeros(10, dtype=f32), "ws")
    assert r.find(flat.data_ptr() + 2 * 10) == ("g:a", 2)
    assert r.find(flat.data_ptr() + 2 * 30) == ("flat", 30)
    ws = [it for it in r.items if it[2] == "ws"][0]
    assert r.find(ws[0] + 36) == ("ws", 9)
    with pytest.raises(AssertionError, match="no tensor"):
        r.find(ws[1])
    with pytest.raises(AssertionError, match="inside an element"):
        r.find(ws[0] + 2)


# ======================================================================================================================
# the recorder
# ======================================================================================================================
class Launch:
    def __init__(self, idx, name, args):
        self.idx, self.name, self.args = idx, name, args
        self.ptrs = {}          # argument key -> (region, element offset)
        self.pre, self.post = {}, {}
        self.g = None           # GemmArgs fields
        self.n_out = None
        self.labels = None      # the dense masked-LM cross-entropy's on-the-fly int32 labels, copied at the launch


_GEMM_PTRS = ("A", "B", "D", "bias", "aux_in", "aux_out", "colsum_out", "rng_state", "workspace")


def gemm_fields(a):
    return {f: getattr(a, f) for f, _t in L.GemmArgs._fields_}


class Recorder:
    def __init__(self, eng):
        self.eng, self.launches, self.orig = eng, [], L.call
        self.reg = Regions()
        self.kind = {}
        self.streams = set()

    def register(self, name, t, kind):
        self.reg.add(name, t, kind)
        if t is not None:
            self.kind[name] = (t, kind)

    def map(self, ln, key, addr):
        if addr is None or addr == 0:
            return
        if addr in self.streams:
            return
        ln.ptrs[key] = self.reg.find(addr)

    def snap(self, ln):
        out = {}
        for reg, _off in ln.ptrs.values():
            t, kind = self.kind[reg]
            if kind in ("ws", "grad", "acc") and reg not in out:
                out[reg] = t.clone()
        return out

    def describe(self, name, args):
        sig = L._SIGNATURES[name]
        if name == "b2_gemm_bf16_grouped":
            lns = []
            for i in range(args[1]):
                ln = Launch(len(self.launches) + len(lns), name, None)
                ln.g = gemm_fields(args[0][i])
                for k in _GEMM_PTRS:
                    self.map(ln, k, ln.g[k])
                lns.append(ln)
            return lns
        ln = Launch(len(self.launches), name, args)
        for i, (a, t) in enumerate(zip(args, sig)):
            if isinstance(a, L.GemmArgs):
                ln.g = gemm_fields(a)
                for k in _GEMM_PTRS:
                    self.map(ln, k, ln.g[k])
            elif t is ctypes.c_void_p:
                if name == "b2_layernorm_bwd" and i == 19:
                    ln.n_out = a            # host address of the partial-row count
                    continue
                if name == "b2_mlm_ce" and i == 4 and args[8] is not None and a and not self.reg.covers(a):
                    # the one pointer no tensor of the step owns: the int32 labels the dense form builds on the fly
                    ln.labels = torch.empty(args[1], dtype=torch.int32, device=self.eng.dev)
                    self.orig("b2_copy_async", ln.labels.data_ptr(), a, 4 * args[1],
                              torch.cuda.current_stream().cuda_stream)
                    torch.cuda.synchronize()
                    continue
                self.map(ln, i, a)
            elif t is not ctypes.c_void_p and not isinstance(a, (int, float)):
                raise AssertionError("%s argument %d: %r is not recorded" % (name, i, a))
        if name == "b2_accum_finish":
            # the grads base pointer addresses the segment table's targets: record those spans
            segs = self.eng.bias_segs.cpu()
            seg0 = ln.ptrs[2][1] // 3
            for j in range(args[3]):
                a_off, g_off, n = (int(v) for v in segs[seg0 + j])
                ln.ptrs["seg%d" % j] = self.reg.find(self.eng.grads.data_ptr() + 2 * g_off)
        return [ln]

    def call(self, name, *args):
        torch.cuda.synchronize()
        lns = self.describe(name, args)
        for ln in lns:
            ln.pre = self.snap(ln)
        # the clones run on the current stream: they must be done before a launch on the weight-gradient stream
        torch.cuda.synchronize()
        self.orig(name, *args)
        torch.cuda.synchronize()
        for ln in lns:
            ln.post = self.snap(ln)
            if ln.n_out is not None:
                ln.n_out = ctypes.c_int32.from_address(ln.n_out).value
        self.launches.extend(lns)


def mlm_bufs(eng):
    """name -> tensor: the masked-LM head's buffers ('mlm.lab.*' over the labelled rows' capacity, 'mlm.full.*' over
    every row, 'mlm.dec' the decoder part of the tied word gradient); none for the other heads"""
    out = {}
    if not eng.mlm:
        return out
    kinds = [full for (_M, _rows, full) in eng._mlm_ws]
    assert len(kinds) == len(set(kinds)), "one masked-LM buffer set of each kind"
    for (_M, _rows, full), hb in eng._mlm_ws.items():
        for k, t in hb.items():
            if isinstance(t, torch.Tensor):
                out["mlm.%s.%s" % ("full" if full else "lab", k)] = t
    if eng._mlm_shared is not None:
        out["mlm.dec"] = eng._mlm_shared["dec"]
    return out


def step_bufs(eng, ws):
    """the step's activations: the workspace and the masked-LM head's buffers"""
    return {**flat_ws(ws), **mlm_bufs(eng)}


def register_step(rec, eng, ws, inputs):
    lay = eng.lay
    for name, (b, n) in reserved_spans(lay).items():
        rec.register("g:" + name, eng.grads[b:b + n], "grad")
        rec.register("w:" + name, eng.shadow[b:b + n], "w")
    for k, v in ws.items():
        if k == "layers":
            for l, d in enumerate(v):
                for kk, t in d.items():
                    rec.register("layers.%d.%s" % (l, kk), t, "ws")
        elif isinstance(v, list):
            for i, t in enumerate(v):
                rec.register("%s.%d" % (k, i), t, "ws")
        else:
            rec.register(k, v, "ws" if k != "zeros_tt" else "in")
    if eng._det_bufs is not None:
        side, parts = eng._det_bufs
        rec.register("det_side", side, "ws")
        for i in range(2):
            for j in range(2):
                rec.register("ln_parts.%d.%d" % (i, j), parts[i][j], "ws")
    for k, t in mlm_bufs(eng).items():
        rec.register(k, t, "ws")
    if eng.mlm:
        sh = eng._mlm_shared
        rec.register("mlm.colsum", sh["colsum"], "scratch")
        rec.register("mlm.ln_parts", sh["ln_parts"], "scratch")
        rec.register("mlm.n_lab_one", sh["n_lab_one"], "state")
    rec.register("bias_acc", eng.bias_acc, "acc")
    for k in ("rng", "owner", "bias_segs"):
        rec.register(k, getattr(eng, k), "state")
    rec.register("split_ws", eng.split_ws, "scratch")
    rec.register("partials", eng.partials, "scratch")
    for k, t in inputs.items():
        rec.register("in:" + k, t, "in")
    rec.streams = {torch.cuda.current_stream().cuda_stream, eng.wgrad_stream.cuda_stream}


def poison(eng, ws):
    """NaN into every workspace tensor the engine allocates with torch.empty, and into the whole gradient space"""
    for k, v in ws.items():
        ts = [t for d in v for t in d.values()] if k == "layers" else (v if isinstance(v, list) else [v])
        for t in ts:
            if t is None or k == "zeros_tt":
                continue
            t.fill_(float("nan") if t.is_floating_point() else -7 if t.dtype == torch.int32 else POISON64)
    if eng._det_bufs is not None:
        side, parts = eng._det_bufs
        for t in [side] + [p for pp in parts for p in pp]:
            t.view(f32).fill_(float("nan"))
    for t in mlm_bufs(eng).values():
        t.fill_(float("nan") if t.is_floating_point() else -7)
    eng.grads.fill_(float("nan"))


# ======================================================================================================================
# the checker
# ======================================================================================================================
_MASKS = {}


def keep64(n_rows, n_cols, seed, step, site, p, dev):
    key = (n_rows, n_cols, seed, step, site, p)
    if key not in _MASKS:
        if len(_MASKS) > 64:
            _MASKS.clear()
        _MASKS[key] = torch.from_numpy(philox_keep_mask(n_rows * n_cols, seed, step, site, p).reshape(n_rows, n_cols))
    return _MASKS[key].to(dev)


class Checker:
    """checks every recorded launch of one step; `defect` alters the reference side (planted-defect tests)"""

    def __init__(self, case, eng, rec, info, defect=None):
        self.case, self.eng, self.rec, self.info, self.defect = case, eng, rec, info, defect
        self.cfg, self.lay, self.dev = eng.cfg, eng.lay, eng.dev
        self.H, self.I, self.nl, self.nh = eng.H, eng.I, eng.nl, eng.heads
        self.seed, self.step = info["seed"], info["step"]
        self.B, self.S = info["B"], info["S"]
        self.M = self.B * self.S
        self.det, self.packed = info["det"], info["packed"]
        self.grad_claims, self.ws_claims = [], []
        self.worst = {}
        self.att_fwd = {}
        self.ln_parts = {}
        self.V, self.Vp = self.cfg.vocab_size, self.lay.vocab_pad

    # ---- reporting -----------------------------------------------------------------------------------------------
    def within(self, got, ref, bound, what):
        err = (got.double() - ref).abs()
        ratio = err / bound.clamp_min(1e-300)
        worst = float(ratio.max()) if err.numel() else 0.0
        fam = what.split(" ", 1)[1] if what.startswith("L") and " " in what else what
        self.worst[fam] = max(self.worst.get(fam, 0.0), worst) if worst == worst else float("nan")
        bad = ~(ratio <= 1.0)
        if bool(bad.any()):
            flat = int(torch.isnan(ratio).flatten().nonzero()[0]) if bool(torch.isnan(ratio).any()) \
                else int(ratio.argmax())
            idx = tuple(int(i) for i in np.unravel_index(flat, tuple(ratio.shape)))
            raise AssertionError("%s %s: worst error is %.3g x its bound at %s (got %r, ref %r, %d over)" % (
                self.case, what, worst, idx, float(got[idx]), float(ref[idx]), int(bad.sum())))

    def same(self, got, ref, what):
        bad = ~((got == ref) | (torch.isnan(got) & torch.isnan(ref))) if got.is_floating_point() else got != ref
        n = int(bad.sum())
        if n:
            raise AssertionError("%s %s: %d elements differ, first at %s" % (
                self.case, what, n, tuple(bad.nonzero()[0].tolist())))

    def finish(self):
        for fam, w in sorted(self.worst.items()):
            report(TAG, {"case": self.case, "family": fam, "err_over_bound": w})

    # ---- operands ----------------------------------------------------------------------------------------------------
    def expect(self, ln, key, region, what):
        got = ln.ptrs.get(key, (None, 0))
        assert got == (region, 0), "%s %s: %s is %s, expected %s" % (self.case, what, key, got, region)

    def region(self, ln, key):
        return ln.ptrs[key][0] if key in ln.ptrs else None

    def flat(self, ln, key, when):
        reg, off = ln.ptrs[key]
        t, kind = self.rec.kind[reg]
        src = (ln.pre if when == "pre" else ln.post)[reg] if kind in ("ws", "grad", "acc") else t
        return src.reshape(-1)[off:]

    def mat(self, ln, key, rows, cols, ld, when="pre"):
        f = self.flat(ln, key, when)
        return f[:(rows - 1) * ld + cols].as_strided((rows, cols), (ld, 1))

    def vec(self, ln, key, n, when="pre"):
        return self.flat(ln, key, when)[:n]

    def keep(self, rows, cols, site, p):
        step = self.step - 1 if self.defect == "previous_step" else self.step
        if self.defect == "neighbour_site" and site >= 2 and site < 1 + 3 * self.nl and site % 3 != 1:
            site = site + 1 if site % 3 == 2 else site - 1
        return keep64(rows, cols, self.seed, step, site, p, self.dev).double()

    def claim_ws(self, ln, *regions):
        for r in regions:
            if r is not None:
                self.ws_claims.append((ln.idx, r))

    def claim_grad(self, name):
        b, n = param_spans(self.lay)[name]
        self.grad_claims.append((b, b + n, family(name)))

    def pname(self, l, what):
        return "bert.encoder.layer.%d.%s" % (l, what)

    def x_in(self, l, f=False):
        if l == 0:
            return "emb_out_f" if f else "emb_out"
        return "layers.%d.%s" % (l - 1, "x2f" if f else "x2")

    # ---- GEMMs -------------------------------------------------------------------------------------------------------
    def gemm_ref(self, ln, defect_ops=None):
        g = ln.g
        M, N, K = g["M"], g["N"], g["K"]
        src = defect_ops or ln
        A = self.mat(src, "A", M, K, g["lda"]) if g["a_major"] == KM else self.mat(src, "A", K, M, g["lda"]).t()
        Bm = self.mat(src, "B", N, K, g["ldb"]).t() if g["b_major"] == KM else self.mat(src, "B", K, N, g["ldb"])
        A, Bm = A.double(), Bm.double()
        return A @ Bm, A.abs() @ Bm.abs()

    def check_gemm(self, ln, what, ref_src=None):
        g = ln.g
        M, N, K = g["M"], g["N"], g["K"]
        epi = g["epilogue"]
        ref, S = self.gemm_ref(ln, ref_src)
        E = C_ACC * K * U * S
        dtype = f32 if epi == L.EPI_ACCUM_F32 else bf
        D = self.mat(ln, "D", M, N, g["ldd"], "post")
        if epi == L.EPI_NONE:
            E = E + (SPLITS * U * S if g["workspace"] else 0.0)
            self.within(D, ref, bf_bound(ref, E), what)
        elif epi == L.EPI_BIAS:
            t = ref + self.vec(ln, "bias", N).double()
            self.within(D, t, bf_bound(t, E + U * t.abs()), what)
        elif epi == L.EPI_BIAS_GELU:
            t = ref + self.vec(ln, "bias", N).double()
            u = self.mat(ln, "aux_out", M, N, g["ld_aux_out"], "post")
            self.within(u, t, bf_bound(t, E + U * t.abs()), what + " u")
            x = u.double()
            h = gelu64(x)
            self.within(D, h, bf_bound(h, gelu_err(x)), what + " h")
        elif epi == L.EPI_BIAS_DROPOUT_RESIDUAL:
            z, Ez = self.dropout_residual(ln, ref, E, self.mat(ln, "aux_in", M, N, g["ld_aux_in"]).double())
            self.within(D, z, bf_bound(z, Ez), what)
        elif epi == L.EPI_GELU_BWD:
            x = self.mat(ln, "aux_in", M, N, g["ld_aux_in"]).double()
            gp = gelu_grad64(x)
            r = ref * gp
            self.within(D, r, bf_bound(r, ref.abs() * gelu_grad_err(x) + E * gp.abs() + U * r.abs()), what)
        elif epi == L.EPI_ACCUM_F32:
            R = self.mat(ln, "D", M, N, g["ldd"], "pre").double()
            self.within(D, R + ref, E + SPLITS * U * (R.abs() + S), what)
        else:
            raise AssertionError("%s: epilogue %d is not restated" % (what, epi))
        assert D.dtype == dtype
        if g["colsum_out"]:
            d = D.double()
            c0 = self.vec(ln, "colsum_out", N, "pre").double()
            c1 = self.vec(ln, "colsum_out", N, "post")
            self.within(c1, c0 + d.sum(0), gamma(32 + -(-M // 32)) * (c0.abs() + d.abs().sum(0)), what + " colsum")

    def dropout_residual(self, ln, ref, E, r):
        g = ln.g
        t = ref + self.vec(ln, "bias", g["N"]).double()
        Et = E + U * t.abs()
        p = g["dropout_p"]
        k = self.keep(g["M"], g["N"], g["rng_site"], p) * drop_scale(p) if p > 0 else 1.0
        ts = t * k
        return ts + r, Et * k + 2 * U * (ts.abs() + r.abs())

    # ---- per-launch checks ------------------------------------------------------------------------------------------
    def run(self, only=None):
        for ln in self.rec.launches:
            if only is None or only(ln):
                getattr(self, "c_" + ln.name)(ln)

    def layer_of(self, ln):
        """the encoder layer a launch belongs to: the layer of the parameters it addresses"""
        for pre in ("w:bert.encoder.layer.", "g:bert.encoder.layer.", "layers."):
            for reg, _o in ln.ptrs.values():
                if reg.startswith(pre):
                    return int(reg[len(pre):].split(".")[0])
        return None

    def c_b2_embed_fwd(self, ln, packed=False):
        a = ln.args
        o = 3 if packed else 0        # position_ids and max_position shift the tail
        B, S, H = a[2 + o - (1 if packed else 0)], a[3 + o - (1 if packed else 0)], self.H
        assert (B, S) == (self.B, self.S)
        names = ["emb_out", "emb_out_f", "emb_pre", "emb_mean", "emb_rstd", "ids32", "tt32"]
        base = 16 + o - (1 if packed else 0)
        for i, nm in enumerate(names):
            if self.rec.kind.get(nm) is not None:
                self.expect(ln, base + i, nm, "embed_fwd")
        assert f32eq(a[base - 3], self.info["p_h"]) and a[base - 1] == 0, "embedding dropout p / site"
        M = self.M
        post = lambda nm: ln.post[nm]
        ids = self.info["inputs"]["ids"].reshape(-1)
        tt = self.info["inputs"]["tt"].reshape(-1)
        self.same(post("ids32").long(), ids, "embed ids32")
        self.same(post("tt32").long(), tt, "embed tt32")
        if packed:
            self.expect(ln, 25, "pos32", "embed_fwd_packed")
            posi = self.info["inputs"]["pos"].reshape(-1)
            self.same(post("pos32").long(), posi, "embed pos32")
        else:
            posi = torch.arange(M, device=self.dev) % S
        W = lambda n: self.rec.kind["w:bert.embeddings." + n][0]
        word = W("word_embeddings.weight").view(-1, H)
        v = (word[ids].float() + W("position_embeddings.weight").view(-1, H)[posi].float()) \
            + W("token_type_embeddings.weight").view(-1, H)[tt].float()
        self.same(post("emb_pre"), v.to(bf), "embed pre_ln")
        p = self.info["p_h"]
        keep = self.keep(M, H, 0, p) * drop_scale(p) if p > 0 else None
        yf = post("emb_out_f") if "emb_out_f" in ln.post else None
        ln_fwd_check(v.double(), post("emb_mean"), post("emb_rstd"), post("emb_out"),
                     W("LayerNorm.weight"), W("LayerNorm.bias"), "embed", keep=keep, y_f32=yf,
                     check=self.within)
        if yf is not None:
            self.same(post("emb_out"), yf.to(bf), "embed y == bf16(y_f32)")
        self.claim_ws(ln, *[n for n in names + (["pos32"] if packed else []) if n in ln.post])

    def c_b2_embed_fwd_packed(self, ln):
        self.c_b2_embed_fwd(ln, packed=True)

    def c_b2_gemm_bf16(self, ln):
        if self.is_mlm(ln):
            return self.mlm_gemm(ln)
        g = ln.g
        l = self.layer_of(ln)
        H, I = self.H, self.I
        epi = g["epilogue"]
        A, Bw, D = self.region(ln, "A"), self.region(ln, "B"), self.region(ln, "D")
        st = l & 1
        w = lambda n: "w:" + self.pname(l, n)
        if epi == L.EPI_BIAS:                                                   # QKV
            want = (self.x_in(l), w("attention.self.qkv.weight"), "layers.%d.qkv" % l)
            what = "L%d qkv" % l
        elif epi == L.EPI_BIAS_GELU:
            want = ("layers.%d.x1" % l, w("intermediate.dense.weight"), "layers.%d.h" % l)
            self.expect(ln, "aux_out", "layers.%d.u" % l, "FFN1")
            what = "L%d u, h" % l
        elif epi == L.EPI_BIAS_DROPOUT_RESIDUAL:                                # unfused dense + residual
            first = A == "layers.%d.ctx" % l
            want = (A, w("attention.output.dense.weight" if first else "output.dense.weight"),
                    "layers.%d.%s" % (l, "z1" if first else "z2"))
            self.expect(ln, "aux_in", self.x_in(l) if first else "layers.%d.x1" % l, "residual")
            assert g["rng_site"] == (2 if first else 3) + 3 * l and f32eq(g["dropout_p"], self.info["p_h"])
            what = "L%d %s" % (l, "z1" if first else "z2")
        elif epi == L.EPI_GELU_BWD:
            want = ("dzd.%d" % st, w("output.dense.weight"), "dU.%d" % st)
            self.expect(ln, "aux_in", "layers.%d.u" % l, "GELU_BWD")
            if not self.det:
                self.expect_acc(ln, "colsum_out", l, 3 * H)
            else:
                assert not g["colsum_out"], "det: GELU_BWD must not accumulate"
            what = "L%d dU" % l
        elif epi == L.EPI_ACCUM_F32:
            if A.startswith("dU."):
                want = ("dU.%d" % st, w("intermediate.dense.weight"), "dxB")
                what = "L%d dx_other += dU W1" % l
            else:
                want = ("dqkv.%d" % st, w("attention.self.qkv.weight"), "dxA")
                what = "L%d dx += dqkv Wqkv" % l
            if self.det:
                assert g["force_splits"] == 1, "det: the dgrads run unsplit"
        elif epi == L.EPI_NONE:
            want = ("dz1d.%d" % st, w("attention.output.dense.weight"), "dctx")
            what = "L%d dctx" % l
        else:
            raise AssertionError("epilogue %d" % epi)
        assert (A, Bw, D) == want, "%s %s: operands %s, expected %s" % (self.case, what, (A, Bw, D), want)
        if epi in (L.EPI_BIAS, L.EPI_BIAS_GELU, L.EPI_BIAS_DROPOUT_RESIDUAL):
            bias = {"qkv": "attention.self.qkv.bias", "u, h": "intermediate.dense.bias",
                    "z1": "attention.output.dense.bias", "z2": "output.dense.bias"}[what.split(" ", 1)[1]]
            self.expect(ln, "bias", w(bias), what)
        self.check_gemm(ln, what)
        self.claim_ws(ln, D, self.region(ln, "aux_out"))

    def expect_acc(self, ln, key, l, slot):
        reg, off = ln.ptrs[key]
        assert reg == "bias_acc" and off == l * self.eng.acc_per_layer + slot, \
            "%s L%d: %s accumulates at bias_acc[%d], expected %d" % (self.case, l, key, off,
                                                                     l * self.eng.acc_per_layer + slot)

    def c_b2_gemm_bf16_grouped(self, ln):
        l = self.layer_of(ln)
        st = l & 1
        D = self.region(ln, "D")
        pre = "g:" + self.pname(l, "")
        want = {pre + "output.dense.weight": ("dzd.%d" % st, "layers.%d.h" % l),
                pre + "intermediate.dense.weight": ("dU.%d" % st, "layers.%d.x1" % l),
                pre + "attention.output.dense.weight": ("dz1d.%d" % st, "layers.%d.ctx" % l),
                pre + "attention.self.qkv.weight": ("dqkv.%d" % st, self.x_in(l))}
        assert D in want and (self.region(ln, "A"), self.region(ln, "B")) == want[D], \
            "%s L%d weight gradient %s from %s" % (self.case, l, D, (self.region(ln, "A"), self.region(ln, "B")))
        ref_src = None
        if self.defect == "parity_race" and l + 2 < self.nl:
            ref_src = self.partner(ln, l + 2)
        self.check_gemm(ln, "L%d %s" % (l, D[len(pre):]), ref_src)
        self.claim_grad(D[2:])

    def partner(self, ln, l2):
        """the grouped problem of layer l2 with the same role (planted parity race)"""
        l = self.layer_of(ln)
        role = self.region(ln, "D")[len("g:" + self.pname(l, "")):]
        for o in self.rec.launches:
            if o.name == ln.name and self.layer_of(o) == l2 and self.region(o, "D") == "g:" + self.pname(l2, role):
                return o
        raise AssertionError("no layer %d partner" % l2)

    def c_b2_gemm_ln_fwd(self, ln):
        g, a = ln.g, ln.args
        l = self.layer_of(ln)
        first = self.region(ln, "A") == "layers.%d.ctx" % l
        tag = "1" if first else "2"
        w = lambda n: "w:" + self.pname(l, n)
        sub = "attention.output." if first else "output."
        want = {"A": "layers.%d.%s" % (l, "ctx" if first else "h"), "B": w(sub + "dense.weight"),
                "bias": w(sub + "dense.bias"), "D": "layers.%d.z%s" % (l, tag),
                "aux_in": self.x_in(l, True) if first else "layers.%d.x1f" % l,
                1: w(sub + "LayerNorm.weight"), 2: w(sub + "LayerNorm.bias"), 4: "layers.%d.x%s" % (l, tag),
                8: "layers.%d.mean%s" % (l, tag), 9: "layers.%d.rstd%s" % (l, tag)}
        yf_name = "layers.%d.x%sf" % (l, tag)
        if self.rec.kind.get(yf_name) is not None:
            want[6] = yf_name
        for k, v in want.items():
            self.expect(ln, k, v, "L%d LN%s" % (l, tag))
        assert g["rng_site"] == (2 if first else 3) + 3 * l and f32eq(g["dropout_p"], self.info["p_h"])
        M, N, K = g["M"], g["N"], g["K"]
        ref, S = self.gemm_ref(ln)
        r = self.mat(ln, "aux_in", M, N, g["ld_aux_in"]).double()
        if self.defect == "bf16_residual":
            r = r.float().to(bf).double()
        z, Ez = self.dropout_residual(ln, ref, C_ACC * K * U * S, r)
        what = "L%d LN%s" % (l, tag)
        self.within(self.mat(ln, "D", M, N, g["ldd"], "post"), z, bf_bound(z, Ez), what + " z")
        e_mu, e_rel = stats_bound(z, Ez)
        y = self.mat(ln, 4, M, N, a[5], "post")
        yf = self.mat(ln, 6, M, N, a[7], "post") if 6 in ln.ptrs else None
        ln_fwd_check(z, self.vec(ln, 8, M, "post"), self.vec(ln, 9, M, "post"), y, self.vec(ln, 1, N),
                     self.vec(ln, 2, N), what, y_f32=yf, stats_bound=(e_mu, e_rel), ev=Ez, check=self.within)
        if yf is not None:
            self.same(y, yf.to(bf), what + " y == bf16(y_f32)")
        self.claim_ws(ln, *[self.region(ln, k) for k in ("D", 4, 6, 8, 9)])

    def c_b2_layernorm_fwd(self, ln):
        if self.is_mlm(ln):
            return self.mlm_ln_fwd(ln)
        l = self.layer_of(ln)
        first = self.region(ln, 0) == "layers.%d.z1" % l
        tag = "1" if first else "2"
        sub = "attention.output." if first else "output."
        for k, v in {0: "layers.%d.z%s" % (l, tag), 1: "w:" + self.pname(l, sub + "LayerNorm.weight"),
                     2: "w:" + self.pname(l, sub + "LayerNorm.bias"), 6: "layers.%d.x%s" % (l, tag),
                     7: "layers.%d.mean%s" % (l, tag), 8: "layers.%d.rstd%s" % (l, tag)}.items():
            self.expect(ln, k, v, "L%d LN%s fwd" % (l, tag))
        M, H = self.M, self.H
        z = self.mat(ln, 0, M, H, H).double()
        ln_fwd_check(z, self.vec(ln, 7, M, "post"), self.vec(ln, 8, M, "post"), self.mat(ln, 6, M, H, H, "post"),
                     self.vec(ln, 1, H), self.vec(ln, 2, H), "L%d LN%s" % (l, tag), check=self.within)
        self.claim_ws(ln, *[self.region(ln, k) for k in (6, 7, 8)])

    # ---- attention -------------------------------------------------------------------------------------------------
    def c_b2_attention_fwd(self, ln):
        l = (ln.args[8] - 1) // 3
        self.att_fwd[l] = ln
        self.expect(ln, 0, "layers.%d.qkv" % l, "L%d attention fwd" % l)
        assert ln.args[8] == 1 + 3 * l and f32eq(ln.args[6], self.info["p_a"])
        self.expect(ln, 9, "layers.%d.ctx" % l, "attention fwd")
        self.expect(ln, 10, "layers.%d.lse" % l, "attention fwd")
        self.claim_ws(ln, "layers.%d.ctx" % l, "layers.%d.lse" % l)

    def c_b2_attention_fwd_packed(self, ln):
        l = (ln.args[7] - 1) // 3
        assert ln.args[7] == 1 + 3 * l and f32eq(ln.args[5], self.info["p_a"])
        self.att_fwd[l] = ln
        self.expect(ln, 0, "layers.%d.qkv" % l, "attention fwd packed")
        self.expect(ln, 8, "layers.%d.ctx" % l, "attention fwd packed")
        self.expect(ln, 9, "layers.%d.lse" % l, "attention fwd packed")
        self.claim_ws(ln, "layers.%d.ctx" % l, "layers.%d.lse" % l)

    def c_b2_attention_fwd_packed_seq(self, ln):
        self.c_b2_attention_fwd(ln)

    def att_bwd(self, ln, site_idx, dqkv_idx, acc_idx=None):
        a = ln.args
        l = (a[site_idx] - 1) // 3
        st = l & 1
        assert a[site_idx] == 1 + 3 * l and f32eq(a[site_idx - 2], self.info["p_a"])
        for k, v in {0: "layers.%d.qkv" % l, 2: "layers.%d.ctx" % l, 3: "dctx", 4: "layers.%d.lse" % l,
                     dqkv_idx: "dqkv.%d" % st}.items():
            self.expect(ln, k, v, "L%d attention bwd" % l)
        fw = self.att_fwd[l]
        B, S, nh, H, M = self.B, self.S, self.nh, self.H, self.M
        qkv = self.mat(ln, 0, M, 3 * H, 3 * H)
        dctx = self.mat(ln, 3, M, H, H)
        ctx = self.mat(fw, 9 if fw.name != "b2_attention_fwd_packed" else 8, M, H, H, "post")
        lse = self.flat(fw, 10 if fw.name != "b2_attention_fwd_packed" else 9, "post")[:B * nh * S].view(B, nh, S)
        if self.packed:
            vis = packed_visibility(self.info["inputs"]["seg"])
        else:
            vis = padded_visibility(self.info["inputs"]["mask"], S)
        p = self.info["p_a"]
        keep = self.keep(B * nh * S, S, 1 + 3 * l, p).view(B, nh, S, S) if p > 0 else None
        dbias = c0 = None
        if acc_idx is not None and a[acc_idx] is not None:
            self.expect_acc(ln, acc_idx, l, 0)
            c0 = self.vec(ln, acc_idx, 3 * H, "pre")
            dbias = self.vec(ln, acc_idx, 3 * H, "post")
        dqkv = self.mat(ln, dqkv_idx, M, 3 * H, 3 * H, "post")
        v = check_outputs("%s L%d" % (self.case, l), qkv, dctx, vis, B, S, nh, p, keep, ctx, lse, dqkv,
                          dbias=dbias, c0=c0)
        for fam, w in v.worst.items():
            self.worst["attention " + fam] = max(self.worst.get("attention " + fam, 0.0), w)
        v.assert_ok()
        kb_idx = 11 if fw.name != "b2_attention_fwd_packed" else 10
        if S == 128 and kb_idx in fw.ptrs and (p > 0 or not torch.equal(fw.pre["layers.%d.keep" % l],
                                                                      fw.post["layers.%d.keep" % l])):
            self.expect(fw, kb_idx, "layers.%d.keep" % l, "keep bits")
            self.claim_ws(fw, "layers.%d.keep" % l)
            kb = self.flat(fw, kb_idx, "post")[:B * nh * S * 2].view(B * nh * S * 2)
            bits = keep.view(-1, 64).long() if keep is not None else torch.ones(B * nh * S * 2, 64, dtype=torch.long,
                                                                                 device=self.dev)
            words = (bits << torch.arange(64, device=self.dev)).sum(1)
            self.same(kb, words, "L%d stored keep bits" % l)
        self.claim_ws(ln, "dqkv.%d" % st)

    def c_b2_attention_bwd(self, ln):
        self.att_bwd(ln, 11, 12, 14)

    def c_b2_attention_bwd_packed(self, ln):
        self.att_bwd(ln, 10, 11, 12)

    def c_b2_attention_bwd_packed_seq(self, ln):
        self.att_bwd(ln, 11, 12)

    def c_b2_attention_bwd_ordered(self, ln):
        self.att_bwd(ln, 11, 12)

    def c_b2_attention_bwd_packed_seq_ordered(self, ln):
        self.att_bwd(ln, 11, 12)

    # ---- LayerNorm backward and the column sums -------------------------------------------------------------------------
    def ln_bwd(self, ln, dy_i, x_i, mean_i, rstd_i, g_i, site_i, dx_i, dxd_i):
        a = ln.args
        l = self.layer_of(ln)
        first = a[site_i] == 2 + 3 * l
        tag = "1" if first else "2"
        st = l & 1
        sub = "attention.output." if first else "output."
        want = {dy_i: "dxB" if first else "dxA", x_i: "layers.%d.z%s" % (l, tag), mean_i: "layers.%d.mean%s" % (l, tag),
                rstd_i: "layers.%d.rstd%s" % (l, tag), g_i: "w:" + self.pname(l, sub + "LayerNorm.weight"),
                dx_i: "dxA" if first else "dxB", dxd_i: ("dz1d.%d" if first else "dzd.%d") % st}
        for k, v in want.items():
            self.expect(ln, k, v, "L%d LN%s bwd" % (l, tag))
        assert a[site_i] in (2 + 3 * l, 3 + 3 * l) and f32eq(a[site_i - 2], self.info["p_h"])
        M, H = self.M, self.H
        dy = self.mat(ln, dy_i, M, H, H)
        x = self.mat(ln, x_i, M, H, H)
        mean, rstd = self.vec(ln, mean_i, M), self.vec(ln, rstd_i, M)
        gam = self.vec(ln, g_i, H)
        ref, E, xh, ex = ln_bwd_ref(dy, x, mean, rstd, gam)
        what = "L%d LN%s bwd" % (l, tag)
        dx = self.mat(ln, dx_i, M, H, H, "post")
        self.within(dx, ref, E, what + " dx")
        p = self.info["p_h"]
        keep = self.keep(M, H, a[site_i], p) != 0 if p > 0 else torch.ones(M, H, dtype=torch.bool, device=self.dev)
        dxd = self.mat(ln, dxd_i, M, H, H, "post")
        self.same(dxd, torch.where(keep, dx * drop_scale(p), torch.zeros_like(dx)).to(bf), what + " dx_drop")
        self.claim_ws(ln, want[dx_i], want[dxd_i])
        return l, tag, sub, (dy, xh, ex, dxd)

    def sums_check(self, got, terms, depth, what, bf_out, offset=None):
        """the column sums got[k] of d_gamma, d_beta and (when dxd is given) d_bias"""
        dy, xh, ex, dxd = terms
        dy = dy.double()
        parts = [(dy * xh, (dy.abs() * ex).sum(0) + 3 * U * (dy * xh).abs().sum(0)), (dy, 0.0)]
        if dxd is not None:
            parts.append((dxd.double(), 0.0))
        assert len(got) == len(parts)
        for k, (t, extra) in enumerate(parts):
            off = offset[k] if offset is not None else 0.0
            ref = t.sum(0) + off
            E = depth * U * (t.abs().sum(0) + (off.abs() if offset is not None else 0.0)) + extra + U * ref.abs()
            self.within(got[k], ref, bf_bound(ref, E) if bf_out else E, "%s sum %d" % (what, k))

    def ln_depth(self):
        nsm = torch.cuda.get_device_properties(self.dev).multi_processor_count
        nb = min(nsm, (self.M + 7) // 8)
        return -(-self.M // (8 * nb)) + 8 + nb + 1

    def c_b2_layernorm_bwd_accum(self, ln):
        l, tag, sub, terms = self.ln_bwd(ln, 0, 1, 2, 3, 4, 9, 10, 11)
        H, I = self.H, self.I
        slot = 3 * H + I if tag == "2" else 6 * H + I
        self.expect_acc(ln, 12, l, slot)
        pre, post = self.vec(ln, 12, 3 * H, "pre").view(3, H), self.vec(ln, 12, 3 * H, "post").view(3, H)
        self.sums_check(post, terms, self.ln_depth(), "L%d LN%s bwd accum" % (l, tag), False,
                        offset=pre.double())

    def c_b2_layernorm_bwd(self, ln):
        if self.is_mlm(ln):
            return self.mlm_ln_bwd(ln)
        assert self.det, "the partial-row LayerNorm backward belongs to the det branch"
        l, tag, sub, terms = self.ln_bwd(ln, 0, 2, 3, 4, 5, 10, 12, 13)
        st = l & 1
        self.expect(ln, 17, "ln_parts.%d.%d" % (st, 0 if tag == "2" else 1), "L%d LN%s partials" % (l, tag))
        self.ln_parts[(l, tag)] = (terms, ln.n_out)

    def c_b2_colsum_finish(self, ln):
        if self.is_mlm(ln):
            return self.mlm_colsum_finish(ln)
        a = ln.args
        reg = self.region(ln, 0)
        st, which = int(reg.split(".")[1]), int(reg.split(".")[2])
        cand = [k for k in self.ln_parts if k[0] & 1 == st and k[1] == ("2" if which == 0 else "1")]
        l, tag = max(cand, key=lambda k: -k[0])          # the most recent (lowest) layer of that parity
        terms, n = self.ln_parts.pop((l, tag))
        assert a[1] == n and a[2] == 3 and a[3] == self.H
        sub = "attention.output." if tag == "1" else "output."
        names = [sub + "LayerNorm.weight", sub + "LayerNorm.bias", sub + "dense.bias"]
        for i, nm in enumerate(names):
            self.expect(ln, 4 + i, "g:" + self.pname(l, nm), "L%d LN%s finish" % (l, tag))
        got = [self.vec(ln, 4 + i, self.H, "post") for i in range(3)]
        self.sums_check(got, terms, -(-self.M // (8 * n)) + 8 + n + 9 + 1, "L%d LN%s bwd det" % (l, tag), True)
        for nm in names:
            self.claim_grad(self.pname(l, nm))

    def c_b2_colsum(self, ln):
        if self.is_mlm(ln):
            return self.mlm_colsum(ln)
        a = ln.args
        l = self.layer_of(ln)
        st = l & 1
        src = self.region(ln, 0)
        if src == "dU.%d" % st:
            want, N = "intermediate.dense.bias", self.I
            assert self.det
        else:
            want, N = "attention.self.qkv.bias", 3 * self.H
            assert src == "dqkv.%d" % st and (self.det or self.S != 128)
        self.expect(ln, 4, "g:" + self.pname(l, want), "L%d colsum" % l)
        assert a[1] == self.M and a[2] == N and a[3] == N
        x = self.mat(ln, 0, self.M, N, N).double()
        if self.defect == "one_bin_fewer":
            x = x[:-self.S]
        ref = x.sum(0)
        self.within(self.vec(ln, 4, N, "post"), ref, bf_bound(ref, gamma(self.M) * x.abs().sum(0)),
                    "L%d %s colsum" % (l, want))
        self.claim_grad(self.pname(l, want))

    def c_b2_accum_finish(self, ln):
        a = ln.args
        assert not self.det
        segs = self.eng.bias_segs.cpu()
        seg0 = ln.ptrs[2][1] // 3
        spl = self.eng.segs_per_layer
        l = seg0 // spl
        assert seg0 == spl * l + (0 if self.S == 128 else 1) and a[3] == spl * (l + 1) - seg0, \
            "%s L%d: accum_finish segments [%d, +%d)" % (self.case, l, seg0, a[3])
        acc_pre, acc_post = ln.pre["bias_acc"], ln.post["bias_acc"]
        for j in range(a[3]):
            a_off, g_off, n = (int(v) for v in segs[seg0 + j])
            reg, off = ln.ptrs["seg%d" % j]
            got = ln.post[reg].reshape(-1)[off:off + n]
            self.same(got, acc_pre[a_off:a_off + n].to(bf), "L%d accum_finish %s" % (l, reg))
            self.same(acc_post[a_off:a_off + n], torch.zeros(n, device=self.dev), "L%d accumulator re-armed" % l)
            name = reg[2:]
            if off == 0 and param_spans(self.lay)[name][1] == n:
                self.claim_grad(name)
            else:
                raise AssertionError("segment %d of layer %d covers part of %s" % (j, l, name))

    # ---- head and loss -----------------------------------------------------------------------------------------------
    def head_w(self, n, shape):
        return self.rec.kind["w:" + n][0].view(*shape)

    def cls_rows(self):
        return self.info["inputs"]["cls"] if self.packed else torch.arange(self.info["Bo"], device=self.dev) * self.S

    def head_keep(self, site, p, rows):
        """the classifier dropout's scaled fp64 keep mask [rows, H] (all ones at p = 0)"""
        if p > 0:
            return self.keep(rows, self.H, site, p) * drop_scale(p)
        return torch.ones(rows, self.H, dtype=f64, device=self.dev)

    def c_b2_head_fwd(self, ln):
        a = ln.args
        H, C, Bo = self.H, self.cfg.num_labels, self.info["Bo"]
        for k, v in {0: self.x_in(self.nl), 4: "w:bert.pooler.dense.weight", 5: "w:bert.pooler.dense.bias",
                     6: "w:classifier.weight", 7: "w:classifier.bias", 12: "pooled", 13: "logits"}.items():
            self.expect(ln, k, v, "head fwd")
        if self.packed:
            self.expect(ln, 1, "in:cls", "head fwd")
        p, site = a[9], a[11]
        assert f32eq(p, self.info["p_c"]) and site == 1 + 3 * self.nl
        params = (self.head_w("bert.pooler.dense.weight", (H, H)), self.head_w("bert.pooler.dense.bias", (H,)),
                  self.head_w("classifier.weight", (C, H)), self.head_w("classifier.bias", (C,)))
        check_head_fwd(self.mat(ln, 0, self.M, H, H), self.cls_rows(), self.vec(ln, 12, Bo * H, "post").view(Bo, H),
                       self.vec(ln, 13, Bo * C, "post").view(Bo, C), params, p, "head", keep=self.head_keep(site, p, Bo),
                       check=self.within)
        self.claim_ws(ln, "pooled", "logits")

    def c_b2_head_fwd_packed(self, ln):
        self.c_b2_head_fwd(ln)

    def c_b2_ce_fwd_bwd(self, ln):
        Bo, C = self.info["Bo"], self.cfg.num_labels
        for k, v in {0: "logits", 1: "in:labels", 4: "loss", 5: "dloss_logits"}.items():
            self.expect(ln, k, v, "loss")
        assert ln.args[2] == Bo and ln.args[3] == C
        dl = self.vec(ln, 5, Bo * C, "post").view(Bo, C)
        check_ce(self.vec(ln, 0, Bo * C).view(Bo, C), self.info["inputs"]["labels"].view(-1),
                 self.vec(ln, 4, 1, "post"), dl, "loss", check=self.within)
        self.dloss = dl.clone()
        self.claim_ws(ln, "loss", "dloss_logits")

    def c_b2_zero(self, ln):
        reg = self.region(ln, 0)
        if reg != "g:" + WORD:
            # the masked-LM head's fp32 GEMM targets: d_t, the decoder part, d_hidden (labelled rows, or dxA dense)
            assert self.eng.mlm and reg in ("mlm.lab.dt", "mlm.full.dt", "mlm.dec", "mlm.lab.dx", "dxA"), \
                "%s: b2_zero of %s" % (self.case, reg)
            t = self.rec.kind[reg][0]
            assert ln.ptrs[0][1] == 0 and ln.args[1] == t.numel() * t.element_size(), "%s: b2_zero covers part of %s" % (
                self.case, reg)
            self.on(ln, 2, reg == "mlm.dec", "b2_zero " + reg)
            self.same(ln.post[reg], torch.zeros_like(ln.post[reg]), "b2_zero " + reg)
            self.claim_ws(ln, reg)
            return
        eb, ee, _ = self.lay.buckets[0]
        self.expect(ln, 0, "g:" + WORD, "embedding bucket clear")
        assert ln.args[1] == 2 * (ee - eb)

    def dlogits(self, ln):
        """the logits gradient the head backward reads: dloss_logits (in-model loss, d_loss = 1), by value"""
        self.expect(ln, 0, "dlogits", "head bwd")
        dl = self.vec(ln, 0, self.dloss.numel()).view(self.dloss.shape)
        self.same(dl, self.dloss + 0.0, "head bwd reads dloss_logits")
        return dl

    def c_b2_head_bwd_split(self, ln):
        a = ln.args
        H, C, Bo, M = self.H, self.cfg.num_labels, self.info["Bo"], self.M
        for k, v in {1: self.x_in(self.nl), 2: "pooled", 8: "w:bert.pooler.dense.weight",
                     9: "w:classifier.weight", 14: "g:bert.pooler.dense.weight", 15: "g:bert.pooler.dense.bias",
                     16: "g:classifier.weight", 17: "g:classifier.bias", 18: "dxA", 20: "head_scratch"}.items():
            self.expect(ln, k, v, "head bwd")
        p, site = a[11], a[13]
        assert f32eq(p, self.info["p_c"]) and site == 1 + 3 * self.nl and a[19] == 1
        names = ("bert.pooler.dense.weight", "bert.pooler.dense.bias", "classifier.weight", "classifier.bias")
        shapes = ((H, H), (H,), (C, H), (C,))
        params = [self.head_w(n, sh) for n, sh in zip(names, shapes)]
        grads = [self.vec(ln, 14 + k, int(np.prod(sh)), "post").view(sh) for k, sh in enumerate(shapes)]
        check_head_bwd(self.dlogits(ln), self.mat(ln, 1, M, H, H), self.cls_rows(),
                       self.vec(ln, 2, Bo * H).view(Bo, H), params, grads, self.mat(ln, 18, M, H, H, "post"), True,
                       self.head_keep(site, p, Bo), "head", check=self.within)
        for n in names:
            self.claim_grad(n)
        self.claim_ws(ln, "dxA")

    def c_b2_token_head_fwd(self, ln):
        a = ln.args
        H, C, M = self.H, self.cfg.num_labels, self.M
        for k, v in {0: self.x_in(self.nl), 3: "w:classifier.weight", 4: "w:classifier.bias", 9: "logits"}.items():
            self.expect(ln, k, v, "token head fwd")
        p, site = a[6], a[8]
        assert a[1] == M and a[2] == H and a[5] == C
        assert f32eq(p, self.info["p_c"]) and site == 1 + 3 * self.nl
        check_token_head_fwd(self.mat(ln, 0, M, H, H), self.head_w("classifier.weight", (C, H)),
                             self.head_w("classifier.bias", (C,)), self.head_keep(site, p, M),
                             self.vec(ln, 9, M * C, "post").view(M, C), "token head", check=self.within)
        self.claim_ws(ln, "logits")

    def c_b2_token_head_bwd_split(self, ln):
        a = ln.args
        H, C, M = self.H, self.cfg.num_labels, self.M
        for k, v in {1: self.x_in(self.nl), 4: "w:classifier.weight", 9: "g:classifier.weight",
                     10: "g:classifier.bias", 11: "dxA", 12: "head_scratch"}.items():
            self.expect(ln, k, v, "token head bwd")
        p, site = a[6], a[8]
        assert a[2] == M and a[3] == H and a[5] == C
        assert f32eq(p, self.info["p_c"]) and site == 1 + 3 * self.nl
        check_token_head_bwd(self.mat(ln, 1, M, H, H), self.head_w("classifier.weight", (C, H)), self.dlogits(ln),
                             self.head_keep(site, p, M), self.mat(ln, 11, M, H, H, "post"),
                             self.vec(ln, 9, C * H, "post").view(C, H), self.vec(ln, 10, C, "post"), "token head",
                             check=self.within)
        self.claim_grad("classifier.weight")
        self.claim_grad("classifier.bias")
        self.claim_ws(ln, "dxA")

    # ---- masked-LM head ----------------------------------------------------------------------------------------------
    def is_mlm(self, ln):
        return any(reg.startswith(("mlm.", "w:cls.", "g:cls.")) for reg, _o in ln.ptrs.values())

    def mlm_kind(self, *regs):
        """'lab' (the labelled rows' capacity) or 'full' (every row): the head buffer set a launch addresses"""
        kinds = {r.split(".")[1] for r in regs if r is not None and r.startswith(("mlm.lab.", "mlm.full."))}
        assert len(kinds) == 1, "%s: head buffers %s" % (self.case, regs)
        return kinds.pop()

    def mlm_rows(self, kind):
        return self.info["cap"] if kind == "lab" else self.M

    def mlm_labels(self):
        """the step's labels [M] and the labelled token indices in token order"""
        lab = self.info["inputs"]["labels"].reshape(-1)
        return lab, torch.nonzero(lab != -100)[:, 0]

    def on(self, ln, i, side, what):
        """the launch's stream argument: the weight-gradient stream (side) or the main stream"""
        want = self.eng.wgrad_stream if side and self.nl > 0 else torch.cuda.current_stream(self.dev)
        assert ln.args[i] == want.cuda_stream, "%s %s: not on the %s stream" % (
            self.case, what, "weight-gradient" if side else "main")

    def c_b2_mlm_compact(self, ln):
        a = ln.args
        names = ("src", "slot", "labels", "count")
        self.expect(ln, 0, "in:labels", "mlm compact")
        for i, k in enumerate(names):
            self.expect(ln, 5 + i, "mlm.lab." + k, "mlm compact")
        cap, M = a[4], self.M
        assert (a[1], a[2], a[3], cap) == (M, -100, self.V, self.info["cap"])
        self.on(ln, 9, False, "mlm compact")
        lab, idx = self.mlm_labels()
        n = idx.numel()
        post = lambda k: ln.post["mlm.lab." + k]
        i32 = dict(dtype=torch.int32, device=self.dev)
        self.same(post("count"), torch.tensor([n], **i32), "mlm compact count")
        rows = torch.zeros(cap, **i32)
        rows[:n] = idx.int()
        self.same(post("src"), rows, "mlm compact rows")
        slab = torch.full((cap,), -1, **i32)
        slab[:n] = lab[idx].int()
        self.same(post("labels"), slab, "mlm compact labels")
        slot = torch.full((M,), -1, **i32)
        slot[idx] = torch.arange(n, **i32)
        self.same(post("slot"), slot, "mlm compact slots")
        self.claim_ws(ln, *["mlm.lab." + k for k in names])

    def c_b2_mlm_gather_rows(self, ln):
        a = ln.args
        for k, v in {0: self.x_in(self.nl), 1: "mlm.lab.src", 2: "mlm.lab.count", 5: "mlm.lab.x"}.items():
            self.expect(ln, k, v, "mlm gather")
        H, cap = self.H, self.info["cap"]
        assert a[3] == cap and a[4] == H
        self.on(ln, 6, False, "mlm gather")
        _lab, idx = self.mlm_labels()
        ref = torch.zeros(cap, H, dtype=bf, device=self.dev)
        ref[:idx.numel()] = self.mat(ln, 0, self.M, H, H)[idx]
        self.same(ln.post["mlm.lab.x"], ref, "mlm gather")
        self.claim_ws(ln, "mlm.lab.x")

    def mlm_gemm(self, ln):
        g = ln.g
        A, Bw, D = self.region(ln, "A"), self.region(ln, "B"), self.region(ln, "D")
        kind = self.mlm_kind(A, Bw, D)
        hb, rows, H, Vp = "mlm.%s." % kind, self.mlm_rows(kind), self.H, self.Vp
        x_in = self.x_in(self.nl) if kind == "full" else hb + "x"
        tw = "w:cls.predictions.transform.dense.weight"
        epi, side = g["epilogue"], False
        if epi == L.EPI_BIAS_GELU:                                              # transform dense + GELU
            want = (x_in, tw, hb + "h", rows, H, H)
            self.expect(ln, "aux_out", hb + "u", "mlm transform")
            self.expect(ln, "bias", "w:cls.predictions.transform.dense.bias", "mlm transform")
            what = "mlm %s u, h" % kind
        elif D == hb + "logits":                                                # onto the bias-filled logits
            want = (hb + "t", "w:" + WORD, D, rows, Vp, H)
            what = "mlm %s logits" % kind
        elif D == hb + "dt":                                                    # d_t = d_logits E, K = vocab_pad
            want = (hb + "dlog", "w:" + WORD, D, rows, H, Vp)
            what = "mlm d_t"
        elif D == "mlm.dec":                                                    # dE = d_logits^T t, M = vocab_pad
            want, side = (hb + "dlog", hb + "t", D, Vp, H, rows), True
            what = "mlm decoder dE"
        elif D == "g:cls.predictions.transform.dense.weight":                   # split weight gradient
            want, side = (hb + "du", x_in, D, H, H, rows), True
            assert epi == L.EPI_NONE and g["workspace"], "mlm dW_t: the split weight-gradient form"
            what = "mlm weight grads"
        else:                                                                   # d_hidden = du W_t
            want = (hb + "du", tw, "dxA" if kind == "full" else hb + "dx", rows, H, H)
            what = "mlm d_x"
        got = (A, Bw, D, g["M"], g["N"], g["K"])
        assert got == want, "%s %s: operands %s, expected %s" % (self.case, what, got, want)
        self.on(ln, 1, side, what)
        if epi == L.EPI_ACCUM_F32:
            if self.det:
                assert g["force_splits"] == 1, "det: the head's GEMMs run unsplit"
            if what != "mlm %s logits" % kind:
                prior = self.mat(ln, "D", g["M"], g["N"], g["ldd"])
                self.same(prior, torch.zeros_like(prior), what + " adds onto zero")
        self.check_gemm(ln, what)
        if D.startswith("g:"):
            self.claim_grad(D[2:])
        else:
            self.claim_ws(ln, D, self.region(ln, "aux_out"))

    def mlm_ln_fwd(self, ln):
        a = ln.args
        kind = self.mlm_kind(self.region(ln, 0))
        hb, rows, H = "mlm.%s." % kind, self.mlm_rows(kind), self.H
        w = "w:cls.predictions.transform.LayerNorm."
        for k, v in {0: hb + "h", 1: w + "weight", 2: w + "bias", 6: hb + "t", 7: hb + "mean", 8: hb + "rstd"}.items():
            self.expect(ln, k, v, "mlm LN fwd")
        assert a[3] == rows and a[4] == H
        self.on(ln, 9, False, "mlm LN fwd")
        ln_fwd_check(self.mat(ln, 0, rows, H, H).double(), self.vec(ln, 7, rows, "post"), self.vec(ln, 8, rows, "post"),
                     self.mat(ln, 6, rows, H, H, "post"), self.vec(ln, 1, H), self.vec(ln, 2, H), "mlm %s LN" % kind,
                     check=self.within)
        self.claim_ws(ln, hb + "t", hb + "mean", hb + "rstd")

    def c_b2_mlm_bias_fill(self, ln):
        a = ln.args
        kind = self.mlm_kind(self.region(ln, 3))
        hb, rows, Vp = "mlm.%s." % kind, self.mlm_rows(kind), self.Vp
        self.expect(ln, 0, "w:cls.predictions.bias", "mlm bias fill")
        self.expect(ln, 3, hb + "logits", "mlm bias fill")
        assert a[1] == rows and a[2] == Vp and ln.post[hb + "logits"].shape == (rows, Vp)
        self.on(ln, 4, False, "mlm bias fill")
        bias = self.vec(ln, 0, Vp).float()
        self.same(ln.post[hb + "logits"], bias[None].expand(rows, Vp), "mlm %s bias fill" % kind)
        self.claim_ws(ln, hb + "logits")

    def c_b2_mlm_ce(self, ln):
        a = ln.args
        kind = self.mlm_kind(self.region(ln, 0))
        hb, rows, V, Vp = "mlm.%s." % kind, self.mlm_rows(kind), self.V, self.Vp
        assert (a[1], a[2], a[3]) == (rows, V, Vp)
        self.on(ln, 14, False, "mlm ce")
        lab, idx = self.mlm_labels()
        n = idx.numel()
        fwd = a[13] is not None
        want = {0: hb + "logits", 10: hb + "row_loss"}
        extra, n_rows = None, None
        if kind == "lab":
            want.update({4: hb + "labels", 5: hb + "count", 6: hb + "count"})
            if fwd:             # the eager forward: loss, row losses and argmax, no d_logits
                want.update({11: hb + "pred", 13: hb + "loss"})
                assert a[7] is None and a[12] is None
            else:               # the backward from the loss: d_logits, the row losses again
                want.update({7: "in:d_loss", 12: hb + "dlog"})
                assert a[11] is None
            assert a[8] is None
            labels, n_rows = self.vec(ln, 4, rows), n
        else:                   # the dense form: every row, the incoming d_logits, the loss's part
            assert not fwd and a[5] is None and a[11] is None and a[9] == V and ln.labels is not None
            want.update({6: "mlm.lab.count", 7: "in:d_loss", 8: "in:d_logits", 12: hb + "dlog"})
            self.same(ln.labels, torch.where(lab == -100, torch.full_like(lab, -1), lab).int(), "mlm dense labels")
            extra = self.mat(ln, 8, rows, V, V)
            self.same(extra, self.info["R"].view(rows, V), "mlm incoming d_logits == R")
            labels = ln.labels
        for k, v in want.items():
            self.expect(ln, k, v, "mlm %s ce" % kind)
        if self.defect == "neighbour_label":
            labels = labels.roll(1)
        d_loss = float(self.vec(ln, 7, 1)) if 7 in want else 1.0
        post = lambda k: ln.post[hb + k] if hb + k in ln.post else None
        back_lab = kind == "lab" and not fwd
        check_mlm_ce(self.mat(ln, 0, rows, Vp, Vp), labels, V, n, d_loss=d_loss, extra=extra, n_rows=n_rows,
                     row_loss=None if back_lab else post("row_loss"), pred=post("pred") if fwd else None,
                     dl=None if fwd else post("dlog"), loss=post("loss") if fwd else None,
                     what="mlm %s ce" % kind, check=self.within)
        if back_lab:
            fw = [o for o in self.rec.launches if o.name == "b2_mlm_ce" and o.idx < ln.idx and o.args[13] is not None]
            self.same(ln.post[hb + "row_loss"], fw[-1].post[hb + "row_loss"], "mlm backward row_loss == forward's")
            self.claim_ws(ln, hb + "dlog")
        elif fwd:
            self.claim_ws(ln, hb + "row_loss", hb + "pred", hb + "loss")
        else:
            self.claim_ws(ln, hb + "row_loss", hb + "dlog")

    def mlm_ln_bwd(self, ln):
        a = ln.args
        kind = self.mlm_kind(self.region(ln, 0))
        hb, rows, H = "mlm.%s." % kind, self.mlm_rows(kind), self.H
        w, gn = "cls.predictions.transform.LayerNorm.weight", "cls.predictions.transform.LayerNorm.bias"
        for k, v in {0: hb + "dt", 2: hb + "h", 3: hb + "mean", 4: hb + "rstd", 5: "w:" + w, 12: hb + "dh",
                     13: hb + "dh_bf", 14: "g:" + w, 15: "g:" + gn, 17: "mlm.ln_parts"}.items():
            self.expect(ln, k, v, "mlm LN bwd")
        # no dropout, the fp32 gradient and its bf16 copy, partial rows in both modes, no third sum
        assert (a[1], a[6], a[7], a[8], a[11], a[16]) == (None, rows, H, 0.0, 1, None)
        self.on(ln, 20, False, "mlm LN bwd")
        dy = self.mat(ln, 0, rows, H, H)
        ref, E, xh, ex = ln_bwd_ref(dy, self.mat(ln, 2, rows, H, H), self.vec(ln, 3, rows), self.vec(ln, 4, rows),
                                    self.vec(ln, 5, H))
        dh = self.mat(ln, 12, rows, H, H, "post")
        self.within(dh, ref, E, "mlm LN bwd dh")
        self.same(self.mat(ln, 13, rows, H, H, "post"), dh.to(bf), "mlm LN bwd dh_bf == bf16(dh)")
        self.ln_parts["mlm"] = ((dy, xh, ex, None), ln.n_out, rows)
        self.claim_ws(ln, hb + "dh", hb + "dh_bf")

    def mlm_colsum_finish(self, ln):
        a = ln.args
        terms, n, rows = self.ln_parts.pop("mlm")
        self.expect(ln, 0, "mlm.ln_parts", "mlm LN finish")
        assert (a[1], a[2], a[3], a[6]) == (n, 3, self.H, None), "mlm LN finish: %s" % (a[:7],)
        names = ["cls.predictions.transform.LayerNorm.weight", "cls.predictions.transform.LayerNorm.bias"]
        for i, nm in enumerate(names):
            self.expect(ln, 4 + i, "g:" + nm, "mlm LN finish")
        self.on(ln, 7, True, "mlm LN finish")
        got = [self.vec(ln, 4 + i, self.H, "post") for i in range(2)]
        self.sums_check(got, terms, -(-rows // (8 * n)) + 8 + n + 9 + 1, "mlm LN bwd", True)
        for nm in names:
            self.claim_grad(nm)

    def mlm_colsum(self, ln):
        a = ln.args
        src = self.region(ln, 0)
        kind = self.mlm_kind(src)
        hb, rows = "mlm.%s." % kind, self.mlm_rows(kind)
        if src == hb + "dlog":
            want, N = "cls.predictions.bias", self.Vp          # every vocab_pad column: the padding sums to 0
        else:
            assert src == hb + "du", "%s: b2_colsum of %s" % (self.case, src)
            want, N = "cls.predictions.transform.dense.bias", self.H
        self.expect(ln, 4, "g:" + want, "mlm colsum")
        self.expect(ln, 5, "mlm.colsum", "mlm colsum")
        assert (a[1], a[2], a[3]) == (rows, N, N)
        self.on(ln, 7, True, "mlm colsum")
        x = self.mat(ln, 0, rows, N, N).double()
        ref = x.sum(0)
        got = self.vec(ln, 4, N, "post")
        self.within(got, ref, bf_bound(ref, gamma(rows) * x.abs().sum(0)), "mlm %s colsum" % want)
        if N == self.Vp:
            self.same(got[self.V:], torch.zeros_like(got[self.V:]), "mlm decoder bias padding")
        self.claim_grad(want)

    def c_b2_mlm_gelu_bwd(self, ln):
        a = ln.args
        kind = self.mlm_kind(self.region(ln, 0))
        hb, rows, H = "mlm.%s." % kind, self.mlm_rows(kind), self.H
        for k, v in {0: hb + "dh", 1: hb + "u", 3: hb + "du"}.items():
            self.expect(ln, k, v, "mlm gelu bwd")
        assert a[2] == rows * H
        self.on(ln, 4, False, "mlm gelu bwd")
        dg, u = self.mat(ln, 0, rows, H, H).double(), self.mat(ln, 1, rows, H, H).double()
        r = dg * gelu_grad64(u)
        self.within(self.mat(ln, 3, rows, H, H, "post"), r, bf_bound(r, dg.abs() * gelu_grad_err(u) + U * r.abs()),
                    "mlm gelu bwd")
        self.claim_ws(ln, hb + "du")

    def c_b2_mlm_scatter_rows(self, ln):
        a = ln.args
        for k, v in {0: "mlm.lab.dx", 1: "mlm.lab.slot", 4: "dxA"}.items():
            self.expect(ln, k, v, "mlm scatter")
        M, H = self.M, self.H
        assert a[2] == M and a[3] == H
        self.on(ln, 5, False, "mlm scatter")
        _lab, idx = self.mlm_labels()
        ref = torch.zeros(M, H, dtype=f32, device=self.dev)
        ref[idx] = self.mat(ln, 0, self.info["cap"], H, H)[:idx.numel()]
        self.same(self.mat(ln, 4, M, H, H, "post"), ref, "mlm scatter")
        self.claim_ws(ln, "dxA")

    def c_b2_mlm_tied_add(self, ln):
        a = ln.args
        V, Vp, H = self.V, self.Vp, self.H
        wreg = "g:" + WORD
        self.expect(ln, 0, "mlm.dec", "mlm tied add")
        self.expect(ln, 1, wreg, "mlm tied add")
        assert a[2] == V * H
        self.on(ln, 3, False, "mlm tied add")
        emb = [o for o in self.rec.launches if o.name.startswith("b2_embed_bwd") and o.idx < ln.idx]
        self.same(ln.pre[wreg], emb[-1].post[wreg], "mlm tied add reads the embedding backward's word gradient")
        pre, post = ln.pre[wreg].view(Vp, H), ln.post[wreg].view(Vp, H)
        dec = ln.pre["mlm.dec"].view(Vp, H)
        self.same(post[:V], (pre[:V].float() + dec[:V]).to(bf), "mlm tied add")
        self.same(post[V:], torch.zeros_like(post[V:]), "mlm tied add: word rows past the vocabulary")
        pad = self.cfg.pad_token_id
        self.same(post[pad], dec[pad].to(bf), "mlm tied add: the pad row")
        self.claim_grad(WORD)

    # ---- embedding backward ------------------------------------------------------------------------------------------
    def c_b2_embed_bwd(self, ln, packed=False):
        a = ln.args
        H, M, S = self.H, self.M, self.S
        o = 1 if packed else 0
        want = {0: "dxA", 2: "emb_pre", 3: "emb_mean", 4: "emb_rstd", 5: "w:bert.embeddings.LayerNorm.weight",
                6: "ids32", 7: "tt32", 17 + o: "g:bert.embeddings.word_embeddings.weight",
                18 + o: "g:bert.embeddings.position_embeddings.weight",
                19 + o: "g:bert.embeddings.token_type_embeddings.weight",
                20 + o: "g:bert.embeddings.LayerNorm.weight", 21 + o: "g:bert.embeddings.LayerNorm.bias",
                22 + o: "emb_dx"}
        if packed:
            want[8] = "pos32"
        for k, v in want.items():
            self.expect(ln, k, v, "embed bwd")
        V, T, pad, p, site = a[11 + o], a[12 + o], a[13 + o], a[14 + o], a[16 + o]
        assert f32eq(p, self.info["p_h"]) and site == 0 and a[1] == 1
        P = self.cfg.max_position_embeddings
        assert (V, T) == (self.cfg.vocab_size, self.cfg.type_vocab_size)
        keep = self.keep(M, H, 0, p) * drop_scale(p) if p > 0 else torch.ones(M, H, dtype=f64, device=self.dev)
        fw = {"pre": self.mat(ln, 2, M, H, H), "mean": self.vec(ln, 3, M), "rstd": self.vec(ln, 4, M),
              "ids32": self.vec(ln, 6, M), "tt32": self.vec(ln, 7, M), "packed": packed}
        if packed:
            fw["pos32"] = self.vec(ln, 8, M)
        rows = lambda i, n: self.flat(ln, i, "post")[:n * H].view(n, H)
        g = {"word": rows(17 + o, V), "pos": rows(18 + o, P), "type": rows(19 + o, T),
             "gamma": self.vec(ln, 20 + o, H, "post"), "beta": self.vec(ln, 21 + o, H, "post"),
             "sdx": self.mat(ln, 22 + o, M, H, H, "post")}
        # every row outside the batch was cleared by the bucket's b2_zero and must still be 0
        check_embed_grads(g, fw, self.mat(ln, 0, M, H, H), keep, self.vec(ln, 5, H), S, H, T, pad, a[24 + o],
                          "embed", vocab=V, max_pos=P, unused=0.0, check=self.within)
        for n in ("word_embeddings.weight", "position_embeddings.weight", "token_type_embeddings.weight",
                  "LayerNorm.weight", "LayerNorm.bias"):
            if not (self.eng.mlm and n == "word_embeddings.weight"):    # the masked-LM tied add owns its final value
                self.claim_grad("bert.embeddings." + n)
        self.claim_ws(ln, "emb_dx")

    def c_b2_embed_bwd_packed(self, ln):
        self.c_b2_embed_bwd(ln, packed=True)

    def c_b2_embed_bwd_ordered(self, ln):
        self.c_b2_embed_bwd(ln)

    def c_b2_embed_bwd_packed_ordered(self, ln):
        self.c_b2_embed_bwd(ln, packed=True)

    # ---- the ledger --------------------------------------------------------------------------------------------------
    def ledger(self):
        grads = self.eng.grads
        eb, ee, _ = self.lay.buckets[0]
        pad = [(b, e) for b, e, f in expected_grad_claims(self.lay) if f == "padding"]
        for b, e in pad:
            t = grads[b:e]
            if zero_padding(self.lay, b, e):
                self.same(t, torch.zeros_like(t), "padding [%d, %d)" % (b, e))
            else:
                assert bool(torch.isnan(t).all()), "%s: padding [%d, %d) was written" % (self.case, b, e)
            self.grad_claims.append((b, e, "padding"))
        assert_tiles(self.grad_claims, self.lay.total)
        assert sorted(self.grad_claims) == sorted(expected_grad_claims(self.lay))
        written = set()
        for ln in self.rec.launches:
            for reg in ln.post:
                if self.rec.kind[reg][1] == "ws" and not reg.startswith(SCRATCH + ("ln_parts",)):
                    if not torch.equal(_bits(ln.pre[reg]), _bits(ln.post[reg])):
                        written.add((ln.idx, reg))
        claims = self.ws_claims
        assert len(claims) == len(set(claims)), "%s: a workspace output is claimed twice" % self.case
        assert set(claims) == written, "%s: written but unchecked %s; claimed but unwritten %s" % (
            self.case, sorted(written - set(claims))[:5], sorted(set(claims) - written)[:5])


# ======================================================================================================================
# one recorded step
# ======================================================================================================================
NO_DROP = dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
# the activations a backward rewrites; the rest of the workspace is the forward's
BACKWARD_WS = ("dxA", "dxB", "emb_dx", "dctx", "dlogits", "dzd.", "dz1d.", "dU.", "dqkv.")


def case_config(case):
    if case == "tiny":
        return tiny_config(num_hidden_layers=3)
    if case == "hidden768":
        return full_config(num_hidden_layers=4)
    if case == "hidden768_nodrop":
        return full_config(num_hidden_layers=4, **NO_DROP)
    if case == "large":
        return full_config(hidden_size=1024, num_hidden_layers=3, num_attention_heads=16, intermediate_size=4096)
    if case.startswith("token"):
        return b2.chinese_bert_wwm_ext_config(num_labels=9, num_hidden_layers=3)
    if case == "mlm_dense":
        return tiny_config(vocab_size=1050, num_hidden_layers=2)        # vocab_pad 1088 = 17 x 64, V % 4 = 2
    if case.startswith("mlm"):
        return b2.chinese_bert_wwm_ext_config(num_hidden_layers=2)      # vocab_pad 21184 = 165.5 x 128
    return full_config(num_hidden_layers=3)


def case_model(case, cfg, state, dev):
    if case.startswith(("token", "mlm")):
        m = (b2.BertForTokenClassification if case.startswith("token") else b2.BertForMaskedLM)(cfg)
        m.load_state_dict(state, strict=True)
        return m.to(dev).train()
    return make_model(cfg, state, dev).train()


def case_state(case, cfg):
    if case.startswith("mlm"):
        return mlm_state_from_hf_init(cfg, 9)
    return token_state_from_hf_init(cfg) if case.startswith("token") else state_from_hf_init(cfg)


def dense_mlm_batch(cfg):
    """B 8 x 128 with one sequence of padding only and every real token labelled: 768 = 6 x 128 labels, so the
    labelled rows fill their capacity with no padding row"""
    b = b2.synthetic_mlm_batch(cfg, 8, 128, 23, padded=True)
    lens = torch.tensor([128, 100, 90, 120, 110, 0, 92, 128])
    mask = (torch.arange(128)[None] < lens[:, None]).to(torch.int64)
    ids = b["input_ids"] * mask
    return {"input_ids": ids, "token_type_ids": torch.zeros_like(ids), "attention_mask": mask,
            "label": torch.where(mask == 1, ids, torch.full_like(ids, -100))}


def case_batch(case, cfg, dev):
    """(model kwargs on the device, host batch, info)"""
    if case == "tiny":
        b = short_batch(cfg, 8, 3, lo=5, hi=128)
        b["input_ids"][5] = 0
        b["attention_mask"][5] = 0           # a sequence of padding only: its rows see no key
        b["token_type_ids"][5] = 0
    elif case.startswith("hidden768"):
        b = short_batch(cfg, 32, 4, lo=20, hi=128)
    elif case == "large":
        b = short_batch(cfg, 8, 5, lo=20, hi=128)
    elif case == "seq512":
        b = short_batch(cfg, 4, 6, lo=100, hi=512, S=512)
    elif case == "packed128":
        b = short_batch(cfg, 48, 7, lo=3, hi=100)
    elif case == "packed512":
        b = long_batch(cfg, 12, 8, lo=16, hi=400, S=512)
    elif case == "token128":
        b = token_batch(cfg, 16, 128, 9)
    elif case == "token512packed":
        b = token_batch(cfg, 12, 512, 10, min_len=16)
    elif case == "mlm128":
        b = b2.synthetic_mlm_batch(cfg, 16, 128, 21, padded=True)
    elif case == "mlm512packed":
        b = b2.synthetic_mlm_batch(cfg, 8, 512, 22, padded=True)
    elif case == "mlm_dense":
        b = dense_mlm_batch(cfg)
    else:
        raise ValueError(case)
    host = {"batch": b}
    token = case.startswith(("token", "mlm"))          # a label per token
    if case.startswith("packed") or case in ("token512packed", "mlm512packed"):
        S = 128 if case == "packed128" else 512
        pk = pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], S,
                        labels=b["label"] if token else None)
        host.update(pk=pk, label=pk["labels"] if token else b["label"])
        kw = dict(input_ids=pk["input_ids"], token_type_ids=pk["token_type_ids"], position_ids=pk["position_ids"],
                  segments=pk["segments"], labels=host["label"])
        if not token:
            kw["cls_index"] = pk["cls_index"]
    else:
        kw = dict(input_ids=b["input_ids"], token_type_ids=b["token_type_ids"], attention_mask=b["attention_mask"],
                  labels=b["label"])
    kw = {k: v.to(dev) for k, v in kw.items()}
    B, S = kw["input_ids"].shape
    inputs = {"ids": kw["input_ids"], "tt": kw["token_type_ids"], "labels": kw["labels"]}
    if "attention_mask" in kw:
        inputs["mask"] = kw["attention_mask"]
    else:
        inputs.update(pos=kw["position_ids"], seg=kw["segments"])
        if not token:
            inputs["cls"] = kw["cls_index"]
    cd = getattr(cfg, "classifier_dropout", None)
    info = dict(B=B, S=S, Bo=kw["labels"].numel(), packed="segments" in kw, inputs=inputs,
                p_h=float(cfg.hidden_dropout_prob), p_a=float(cfg.attention_probs_dropout_prob),
                p_c=float(cd if cd is not None else cfg.hidden_dropout_prob), R=None)
    if case.startswith("mlm"):
        n = int((kw["labels"] != -100).sum())
        info["cap"] = min(B * S, max(128, -(-n // 128) * 128))     # the labelled rows' capacity (mlm_capacity)
        assert (n == info["cap"]) == (case == "mlm_dense"), "%s: %d labelled tokens" % (case, n)
    if case == "mlm_dense":
        # the objective's incoming gradient of the logits: loss + (logits R).sum()
        gen = torch.Generator(device=dev).manual_seed(SEED)
        info["R"] = torch.randn(B, S, cfg.vocab_size, generator=gen, device=dev)
    return kw, host, info


def objective(out, R):
    """the in-model loss; for the dense masked-LM case loss + (logits R).sum(), so d_logits = R and d_loss = 1"""
    return out.loss if R is None else out.loss + (out.logits * R).sum()


def one_step(model, kw, step, R=None):
    """seed the dropout stream at (SEED, step), then forward and the objective's backward"""
    model._engine.seed_dropout(SEED, step)
    objective(model(**kw), R).backward()
    torch.cuda.synchronize()


def run_case(case, det, dev):
    """one recorded step after a warm-up step (dropout step 0) that allocates every buffer; the recorded step runs at
    dropout step 1 on poisoned buffers"""
    cfg = case_config(case)
    state = case_state(case, cfg)
    kw, host, info = case_batch(case, cfg, dev)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        model = case_model(case, cfg, state, dev)
        eng = model._engine
        one_step(model, kw, 0, info["R"])
        ws = eng.workspace(info["B"], info["S"], info["Bo"])
        prev = {"grads": eng.grads.clone(), "ws": {k: v.clone() for k, v in step_bufs(eng, ws).items()}}
        poison(eng, ws)
        rec = Recorder(eng)
        register_step(rec, eng, ws, info["inputs"])
        eng.seed_dropout(SEED, 1)
        rs = eng.rng.cpu()
        info.update(seed=int(rs[0]), step=int(rs[1]), det=det)
        orig = L.call
        L.call = rec.call
        try:
            out = model(**kw)
            if eng.mlm:
                # the masked-LM backward passes d(objective)/d(loss) (and, dense, d_logits) to its kernels: the
                # gradients autograd hands the model become step inputs
                out.loss.register_hook(lambda g: rec.register("in:d_loss", g, "in"))
                if info["R"] is not None:
                    out.logits.register_hook(lambda g: rec.register("in:d_logits", g, "in"))
            objective(out, info["R"]).backward()
        finally:
            L.call = orig
        torch.cuda.synchronize()
        return dict(case=case, cfg=cfg, state=state, kw=kw, host=host, info=info, model=model, rec=rec, ws=ws,
                    prev=prev, grads=eng.grads.clone(), acts={k: v.clone() for k, v in step_bufs(eng, ws).items()},
                    acc_zero=bool((eng.bias_acc == 0).all()))
    finally:
        torch.use_deterministic_algorithms(was)


def flat_ws(ws):
    out = {}
    for k, v in ws.items():
        if k == "layers":
            for l, d in enumerate(v):
                for kk, t in d.items():
                    if t is not None:
                        out["layers.%d.%s" % (l, kk)] = t
        elif isinstance(v, list):
            for i, t in enumerate(v):
                out["%s.%d" % (k, i)] = t
        elif v is not None and k not in SCRATCH:
            out[k] = v
    return out


def check_case(r, defect=None, only=None):
    ck = Checker(r["case"] + (" det" if r["info"]["det"] else ""), r["model"]._engine, r["rec"], r["info"], defect)
    ck.run(only)
    if only is None:
        ck.ledger()
    ck.finish()
    return ck


def unrecorded_step(r, dev):
    """the recorded step again, on a model loaded from the same state, with the same warm-up, poison and dropout
    key, without the recorder; returns (gradient space, workspace)"""
    info = r["info"]
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(info["det"])
    try:
        model = case_model(r["case"], r["cfg"], r["state"], dev)
        eng = model._engine
        one_step(model, r["kw"], 0, info["R"])
        ws = eng.workspace(info["B"], info["S"], info["Bo"])
        poison(eng, ws)
        one_step(model, r["kw"], 1, info["R"])
        return eng.grads.clone(), {k: v.clone() for k, v in step_bufs(eng, ws).items()}
    finally:
        torch.use_deterministic_algorithms(was)


def captured_step(r, dev):
    """the gradient space after one replay of the captured step (FusedTrainStep, PackedTrainStep for packed bins),
    built with AdamW at lr 0 on a model loaded from the same state, the replay at the recorded step's dropout key"""
    info, host = r["info"], r["host"]
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(info["det"])
    try:
        model = case_model(r["case"], r["cfg"], r["state"], dev)
        opt = b2.AdamW(model.parameters(), lr=0.0, weight_decay=0.0)
        if info["packed"]:
            pk = host["pk"]
            step = b2.PackedTrainStep(model, opt, pk["bins"], host["batch"]["input_ids"].shape[0], bin_len=info["S"])
            call = lambda: step(pk, host["label"])
        else:
            step = b2.FusedTrainStep(model, opt, info["B"], info["S"])
            call = lambda: step(host["batch"])
        call()
        call()                                   # the two eager warm-ups
        model.set_dropout_rng_state([SEED, 1])
        call()                                   # capture, then one replay
        torch.cuda.synchronize()
        assert step.graph is not None
        return model._engine.grads.clone()
    finally:
        torch.use_deterministic_algorithms(was)


def assert_same_grads(lay, got, want, what):
    """every parameter span by value (a zero's sign aside): the round-8 padding is not part of the comparison"""
    for name, (b, n) in param_spans(lay).items():
        assert torch.equal(got[b:b + n].float(), want[b:b + n].float()), "%s: the gradient of %s differs" % (what, name)


def assert_same_ws(got, want, names, what):
    for k in names:
        a, b_ = got[k], want[k]
        same = (a == b_) | (torch.isnan(a) & torch.isnan(b_)) if a.is_floating_point() else a == b_
        assert bool(same.all()), "%s: %s differs" % (what, k)


CASES = ["tiny", "hidden768", "hidden768_nodrop", "large", "seq512", "packed128", "packed512", "token128",
         "token512packed", "mlm128", "mlm512packed", "mlm_dense"]


def is_backward_buf(name):
    """a buffer the backward writes (the rest are the forward's activations)"""
    if name.startswith("mlm."):
        return name == "mlm.dec" or name.split(".")[2] in MLM_BACKWARD
    return name.startswith(BACKWARD_WS)


@pytest.mark.gpu
@pytest.mark.parametrize("det", [False, True], ids=["atomic", "det"])
@pytest.mark.parametrize("case", CASES)
def test_step_stages(cuda_dev, case, det):
    r = run_case(case, det, cuda_dev)
    assert r["acc_zero"], "bias_acc is not all zero after the step"
    check_case(r)
    # the recorder serialises the two streams; the same step without it must give what the recorded one gave
    grads, acts = unrecorded_step(r, cuda_dev)
    lay = r["model"]._engine.lay
    if det:
        # every sum in a fixed order: bitwise the activations, the gradient space and the embedding backward's input
        assert_same_ws(acts, r["acts"], acts, case + " unrecorded det step")
        assert_same_grads(lay, grads, r["grads"], case + " unrecorded det step")
        if case != "mlm_dense":         # the captured step's objective is the loss alone
            assert_same_grads(lay, captured_step(r, cuda_dev), r["grads"], case + " captured det step")
    else:
        # atomics order the backward's sums freely; the forward has none but the loss's mean over blocks
        fwd = [k for k in acts if not is_backward_buf(k) and k != "loss"]
        assert_same_ws(acts, r["acts"], fwd, case + " unrecorded step")


# ======================================================================================================================
# planted defects: each must fail its check
# ======================================================================================================================
@pytest.fixture(scope="module")
def recorded(cuda_dev):
    """recorded steps shared by the planted-defect tests, released when the module's tests are done"""
    runs = {}

    def get(case, det):
        if (case, det) not in runs:
            runs[(case, det)] = run_case(case, det, cuda_dev)
        return runs[(case, det)]

    yield get
    runs.clear()
    torch.cuda.empty_cache()


def is_layer(l, *names):
    return lambda ln: ln.name in names and Checker.layer_of(None, ln) == l


# defect -> (recorded case, det, launches it alters, the check that must fail)
DEFECTS = {
    "parity_race": ("hidden768", False, is_layer(0, "b2_gemm_bf16_grouped"), r"L0 \S+weight: worst error"),
    "neighbour_site": ("hidden768", False, is_layer(1, "b2_gemm_ln_fwd"), r"L1 LN1 z: worst error"),
    "previous_step": ("hidden768", False, is_layer(2, "b2_layernorm_bwd_accum"),
                      r"L2 LN2 bwd dx_drop: \d+ elements differ"),
    "bf16_residual": ("hidden768", False, lambda ln: ln.name == "b2_gemm_ln_fwd" and Checker.layer_of(None, ln) == 1
                      and Checker.region(None, ln, "aux_in") == "layers.1.x1f",
                      r"L1 LN2 (z|mean|rstd|y|y_f32): worst error"),
    "stale_gradient": ("hidden768", False, is_layer(1, "b2_gemm_bf16_grouped"), r"L1 \S+weight: worst error"),
    "stale_row": ("hidden768", False, is_layer(2, "b2_gemm_bf16"), r"L2 qkv: worst error"),
    "one_bin_fewer": ("packed128", True, lambda ln: ln.name == "b2_colsum" and Checker.region(None, ln, 0) == "dqkv.1",
                      r"L1 attention.self.qkv.bias colsum: worst error"),
    "stale_dec": ("mlm128", False, lambda ln: ln.name == "b2_mlm_tied_add", r"mlm tied add: \d+ elements differ"),
    "stale_gathered_row": ("mlm128", False, lambda ln: ln.name == "b2_mlm_gather_rows", r"mlm gather: \d+ elements differ"),
    "neighbour_label": ("mlm128", False, lambda ln: ln.name == "b2_mlm_ce" and ln.args[13] is not None,
                        r"mlm lab ce row_loss: worst error"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("defect", list(DEFECTS))
def test_planted_defect_fails(recorded, defect):
    case, det, only, fails = DEFECTS[defect]
    r = recorded(case, det)
    rec, eng, info = r["rec"], r["model"]._engine, r["info"]
    Checker(case + " clean", eng, rec, info).run(only)       # the same launches pass unaltered
    ck = Checker(case + " planted " + defect, eng, rec, info, defect)
    saved = []
    if defect == "stale_gradient":                  # one weight-gradient element back to the warm-up step's value
        ln = [x for x in rec.launches if only(x)][0]
        reg = ln.ptrs["D"][0]
        b, _n = param_spans(ck.lay)[reg[2:]]
        saved.append((ln.post[reg], ln.post[reg].clone()))
        ln.post[reg].view(-1)[5] = r["prev"]["grads"][b + 5]
    elif defect == "stale_row":                     # one row of layer 2's qkv back to the warm-up step's
        ln = [x for x in rec.launches if only(x) and x.g["epilogue"] == L.EPI_BIAS][0]
        saved.append((ln.post["layers.2.qkv"], ln.post["layers.2.qkv"].clone()))
        ln.post["layers.2.qkv"][77] = r["prev"]["ws"]["layers.2.qkv"][77]
    elif defect == "stale_dec":                     # the tied add's reference reads the warm-up step's decoder part
        ln = [x for x in rec.launches if only(x)][0]
        saved.append((ln.pre["mlm.dec"], ln.pre["mlm.dec"].clone()))
        ln.pre["mlm.dec"].copy_(r["prev"]["ws"]["mlm.dec"])
    elif defect == "stale_gathered_row":            # one gathered row back to the warm-up step's
        ln = [x for x in rec.launches if only(x)][0]
        saved.append((ln.post["mlm.lab.x"], ln.post["mlm.lab.x"].clone()))
        ln.post["mlm.lab.x"][3] = r["prev"]["ws"]["mlm.lab.x"][3]
    try:
        with pytest.raises(AssertionError, match=fails):
            ck.run(only)
    finally:
        for t, v in saved:
            t.copy_(v)
