"""The losses of the training step, on the device loss kernel (b2_loss_fwd_bwd, csrc/head.cu).

Two sources pick the loss:
  * the model's ``config.problem_type``, as HF ``BertForSequenceClassification.forward`` does (transformers 5.5):
    "regression" -> ``MSELoss`` (with one label over ``logits.squeeze()`` / ``labels.squeeze()``),
    "single_label_classification" -> ``CrossEntropyLoss``, "multi_label_classification" -> ``BCEWithLogitsLoss``;
    when it is None the first labelled forward infers it (:func:`infer_problem_type`) and stores it on the config;
  * the Trainer's criterion, which the captured steps reproduce when it is exactly one of those three torch losses
    with ``reduction="mean"`` (:func:`loss_from_criterion`); anything else raises there and trains eagerly instead.
"""
import torch
import torch.nn as nn

from . import _lib as L

PROBLEM_TYPES = ("regression", "single_label_classification", "multi_label_classification")
_MODE_OF_PROBLEM_TYPE = {"regression": L.LOSS_MSE, "single_label_classification": L.LOSS_CE,
                         "multi_label_classification": L.LOSS_BCE}
_SUPPORTED = ("torch.nn.CrossEntropyLoss (weight, ignore_index, label_smoothing), torch.nn.MSELoss or "
              "torch.nn.BCEWithLogitsLoss (pos_weight), each exactly that class with reduction='mean'")


def infer_problem_type(num_labels, labels):
    """HF's rule for a config without problem_type: one label is regression, integer labels are single-label
    classification, anything else is multi-label classification."""
    if num_labels == 1:
        return "regression"
    if num_labels > 1 and labels.dtype in (torch.long, torch.int):
        return "single_label_classification"
    return "multi_label_classification"


class Loss:
    """One mean loss of the device kernel: mode ``L.LOSS_CE`` / ``LOSS_MSE`` / ``LOSS_BCE`` over [batch, num_labels]
    logits, with CE's class weights, ignore_index and label smoothing and BCE's pos_weight.  Weight tensors are copied
    to `device` once, here; the kernel reads them from there at every launch (and graph replay)."""

    def __init__(self, mode, num_labels, device=None, weight=None, pos_weight=None, ignore_index=-100,
                 label_smoothing=0.0):
        if mode not in (L.LOSS_CE, L.LOSS_MSE, L.LOSS_BCE):
            raise ValueError("unknown loss mode %r" % (mode,))
        if weight is not None and mode != L.LOSS_CE:
            raise ValueError("class weights apply to cross-entropy only")
        if pos_weight is not None and mode != L.LOSS_BCE:
            raise ValueError("pos_weight applies to BCEWithLogitsLoss only")
        if not 0.0 <= float(label_smoothing) <= 1.0:
            raise ValueError("label_smoothing=%r must be in [0, 1]" % (label_smoothing,))
        self.mode, self.C = mode, int(num_labels)
        self.ignore_index, self.label_smoothing = int(ignore_index), float(label_smoothing)
        self.weight = self._device_vector(weight, "weight", device)
        self.pos_weight = self._device_vector(pos_weight, "pos_weight", device)
        self._params = L.LossParams(L.ptr(self.weight), L.ptr(self.pos_weight), self.ignore_index,
                                    self.label_smoothing)

    def _device_vector(self, t, name, device):
        if t is None:
            return None
        if tuple(t.shape) != (self.C,):
            raise ValueError("%s must have shape (%d,) (one per label), got %s" % (name, self.C, tuple(t.shape)))
        return t.detach().to(device=device, dtype=torch.float32).contiguous().clone()

    @property
    def float_labels(self):
        """MSE / BCE take floating labels, CE int64 class indices"""
        return self.mode != L.LOSS_CE

    @property
    def plain_ce(self):
        """CrossEntropyLoss() with its defaults: the reference's criterion and the parent path (b2_ce_fwd_bwd)"""
        return (self.mode == L.LOSS_CE and self.weight is None and self.ignore_index == -100
                and self.label_smoothing == 0.0)

    def label_shape(self, batch):
        """what a batch of `batch` rows carries: [batch] class indices (CE), [batch] values (one-label regression) or
        [batch, num_labels]"""
        if self.mode == L.LOSS_CE or (self.mode == L.LOSS_MSE and self.C == 1):
            return (batch,)
        return (batch, self.C)

    def check_labels(self, labels, batch):
        """raises TypeError / ValueError when `labels` do not fit this loss over `batch` rows"""
        if self.mode == L.LOSS_CE:
            if labels.dtype != torch.int64:
                raise TypeError("labels must be int64 (as the reference Collate produces)")
            if labels.numel() != batch:
                raise ValueError("labels must be [batch]")
            return
        kind = "regression" if self.mode == L.LOSS_MSE else "multi-label"
        if not labels.is_floating_point():
            raise TypeError("%s labels must be floating point (got %s): MSELoss / BCEWithLogitsLoss take float "
                            "targets" % (kind, labels.dtype))
        shape = tuple(labels.shape)
        if self.mode == L.LOSS_MSE and self.C == 1:
            # HF squeezes both sides: [batch] and [batch, 1] (and a 0-d label for a batch of one)
            ok = shape in ((batch,), (batch, 1)) or (batch == 1 and shape == ())
            want = "[%d] or [%d, 1]" % (batch, batch)
        else:
            ok = shape == (batch, self.C)
            want = "[%d, %d]" % (batch, self.C)
        if not ok:
            raise ValueError("%s labels must be %s, got %s" % (kind, want, list(shape)))

    def device_labels(self, labels, batch):
        """checked labels as the kernel reads them: contiguous int64 [batch] or fp32 [batch * C']"""
        self.check_labels(labels, batch)
        if self.mode == L.LOSS_CE:
            return labels.contiguous().view(-1)
        return labels.to(torch.float32).contiguous().view(-1)

    def launch(self, logits, labels, batch, loss, dlogits, stream):
        """loss (scalar) and dlogits ([batch, C], or None for a forward only) from device pointers `logits` / `loss` /
        `dlogits` and the device_labels() tensor `labels`"""
        if self.plain_ce:
            L.call("b2_ce_fwd_bwd", logits, labels.data_ptr(), batch, self.C, loss, dlogits, stream)
        else:
            L.call("b2_loss_fwd_bwd", logits, labels.data_ptr(), batch, self.C, self.mode, self._params, loss,
                   dlogits, stream)


def problem_type_loss(problem_type, num_labels):
    """HF's loss of a problem type (no weights: no device state)"""
    if problem_type not in _MODE_OF_PROBLEM_TYPE:
        raise ValueError("problem_type=%r: expected one of %s" % (problem_type, PROBLEM_TYPES))
    return Loss(_MODE_OF_PROBLEM_TYPE[problem_type], num_labels)


def loss_from_criterion(criterion, num_labels, device):
    """The device loss equal to `criterion`, or ValueError when the kernel cannot reproduce it."""
    t = type(criterion)
    hint = ("The captured training step reproduces only %s; got %r. Set args.fused = False to train with it through "
            "autograd." % (_SUPPORTED, criterion))
    if t not in (nn.CrossEntropyLoss, nn.MSELoss, nn.BCEWithLogitsLoss) or criterion.reduction != "mean":
        raise ValueError(hint)
    if t is nn.CrossEntropyLoss:
        return Loss(L.LOSS_CE, num_labels, device, weight=criterion.weight, ignore_index=criterion.ignore_index,
                    label_smoothing=criterion.label_smoothing)
    if t is nn.BCEWithLogitsLoss:
        if criterion.weight is not None:
            raise ValueError("BCEWithLogitsLoss(weight=...) is not supported. " + hint)
        return Loss(L.LOSS_BCE, num_labels, device, pos_weight=criterion.pos_weight)
    return Loss(L.LOSS_MSE, num_labels, device)


def check_token_criterion(criterion):
    """A token-classification model's loss is a cross-entropy over every token's C logits (HF's CrossEntropyLoss over
    logits.view(-1, C)); MSELoss / BCEWithLogitsLoss would need float per-token targets, which the tagging path does
    not carry.  Raises ValueError for those two."""
    if isinstance(criterion, (nn.MSELoss, nn.BCEWithLogitsLoss)):
        raise ValueError("%s does not apply to a token-classification model: its labels are one int64 class index per "
                         "token (-100 on ignored ones) and its loss is CrossEntropyLoss over logits.view(-1, C), as HF's "
                         "BertForTokenClassification computes it" % type(criterion).__name__)


def _tensor_key(t):
    return None if t is None else (id(t), t._version)


def criterion_key(criterion):
    """Changes whenever the loss `criterion` stands for may have: its class, reduction and options, and the identity
    and in-place version of its weight tensors (no host sync)"""
    if criterion is None:
        return None
    return (type(criterion), id(criterion), getattr(criterion, "reduction", None),
            getattr(criterion, "ignore_index", None), getattr(criterion, "label_smoothing", None),
            _tensor_key(getattr(criterion, "weight", None)), _tensor_key(getattr(criterion, "pos_weight", None)))
