"""The reference's ``Trainer`` / ``Args`` surface (multi-gpu-distributed-cls.py:113-257) on the H100 step.

Same methods, same argument meaning: ``on_step`` [:126-137], ``loss_reduce`` [:139-143], ``output_reduce`` [:145-155],
``train`` [:157-197], ``dev`` [:199-220], ``test`` [:222-239].  Differences, all on the hot path's periphery:
  * host batches are staged through pinned memory and copied asynchronously (the reference does four pageable,
    synchronous ``.cuda()`` copies per step, :128-131);
  * the per-step ``torch.distributed.barrier()`` [:171] is dropped: ranks are ordered by the device-side flag barriers
    inside the gradient exchange, and a host-blocking barrier only serialises forward/backward across ranks;
  * ``loss_reduce`` / ``output_reduce`` go through the peer-memory kernels when the model is the b200 DDP wrapper;
  * ``train`` uses :class:`FusedTrainStep` (the whole step captured in one CUDA graph) when ``args.fused`` is set.
A learning-rate schedule is a host-side torch ``LRScheduler`` (passed as ``scheduler=`` like fabric-cls.py's Trainer, or
built from ``Args.lr_scheduler_type``), stepped once per optimizer step on every path; the captured steps read the lr
it sets at every replay.
"""
import contextlib
import json
import math
import os
import random
import re
import shutil
import time

import numpy as np
import torch
import torch.nn as nn

from .ddp import DistributedDataParallel
from . import _lib as L
from .losses import Loss, check_token_criterion, criterion_key, infer_problem_type, loss_from_criterion, \
    problem_type_loss
from .optim import clip_grad_norm_
from .packing import MAX_BIN, bin_length, pack_batch
from .schedules import get_scheduler, warmup_steps


class Args:
    model_path = "model_hub/chinese-bert-wwm-ext"
    ckpt_path = "output/multi-gpu-distributed-cls.pt"
    max_seq_len = 128
    ratio = 0.92
    train_batch_size = 32
    dev_batch_size = 32
    weight_decay = 0.01
    epochs = 1
    learning_rate = 3e-5
    eval_step = 50
    local_rank = None
    local_world_size = None
    device_ids = None
    rank = None
    dev = False
    use_amp = False       # the -amp scripts' flag (multi-gpu-distributed-mp-amp-cls.py:160): GradScaler loop on the eager path
    fused = True          # capture fwd + bwd + exchange + AdamW in one CUDA graph
    pack = False          # pack the valid prefixes of padded [B, S <= 512] batches into bins of the shortest multiple of
                          # 128 that holds the batch's longest row (packing.py): the reference pads every row to
                          # max_seq_len although real rows average 18 tokens [:76]
    gradient_accumulation_steps = 1   # k > 1: one optimizer step per k batches, each batch's loss scaled by 1/k (the
                                      # HF Trainer / DeepSpeed name; fabric-cls.py's grad_accumulation)
    max_grad_norm = None  # clip the gradient's 2-norm to this before every optimizer step (HF TrainingArguments'
                          # name); None or 0: no clipping
    lr_scheduler_type = None   # HF TrainingArguments' names: "linear", "cosine", "constant", "constant_with_warmup";
                               # None: a constant lr (HF's default is "linear")
    warmup_steps = 0      # linear warmup from 0 over this many optimizer steps; when 0, ceil(warmup_ratio x total)
    warmup_ratio = 0.0
    optim = "adamw"       # build_optimizer's optimizer: "adamw" (the reference's HF AdamW), "sgd" (fabric-cls.py's
                          # default: torch SGD, no momentum, no weight decay), or "adamw_torch" / "adamw_torch_fused"
                          # (HF's names: torch.optim.AdamW on the reference's two groups, eps 1e-8)
    log_every = 1         # the reference prints every step (forces a D2H sync per step)
    total_step = 0
    output_dir = None     # HF TrainingArguments' checkpoint names: train() writes output_dir/checkpoint-N every save_steps
    save_steps = None     # optimizer steps (None: no checkpoints), keeping the newest save_total_limit of them (None:
    save_total_limit = None   # all); train(resume_from_checkpoint=...) continues from one
    full_determinism = False  # HF TrainingArguments' name: Trainer() calls torch.use_deterministic_algorithms(True), and
                              # every training path then runs its fixed-order backward (bitwise reproducible runs)
    max_answer_length = 30    # run_qa.py's name: a question-answering model's dev() / test() predict spans of at most
                              # this many tokens


def _unwrap(model):
    return model.module if isinstance(model, DistributedDataParallel) else model


def _is_token(model):
    """a BertForTokenClassification (or a wrapper of one): logits and labels per token"""
    return _unwrap(model)._layout.head == "token"


def _is_mlm(model):
    """a BertForMaskedLM (or a wrapper of one)"""
    return _unwrap(model)._layout.head == "mlm"


def _is_qa(model):
    """a BertForQuestionAnswering (or a wrapper of one): start / end positions instead of labels"""
    return _unwrap(model)._layout.head == "question_answering"


def _is_mc(model):
    """a BertForMultipleChoice (or a wrapper of one): [B, N, S] inputs, one logit per choice"""
    return _unwrap(model)._layout.head == "multiple_choice"


def _choices(batch_data):
    """the number of choices of a multiple-choice batch: the middle axis of its [B, N, S] input_ids"""
    ids = batch_data["input_ids"]
    if ids.dim() != 3:
        raise ValueError("a multiple-choice batch's input_ids are [batch, num_choices, seq], got %s" % list(ids.shape))
    return int(ids.shape[1])


TOKEN_PROBLEM_TYPE = "token_classification"     # what Trainer.problem_type reports for a token model (not stored)
MLM_PROBLEM_TYPE = "masked_lm"                  # ... and for a masked-LM model (not stored)
QA_PROBLEM_TYPE = "question_answering"          # ... and for a question-answering model (not stored)
MC_PROBLEM_TYPE = "multiple_choice"             # ... and for a multiple-choice model (not stored)


def check_mc_criterion(criterion):
    """A multiple-choice model's loss is a cross-entropy over each example's N choice logits (HF's CrossEntropyLoss
    over logits.view(-1, N)); MSELoss / BCEWithLogitsLoss would need float targets per choice, which the multiple-choice
    batch does not carry.  Raises ValueError for those two."""
    if isinstance(criterion, (nn.MSELoss, nn.BCEWithLogitsLoss)):
        raise ValueError("%s does not apply to a multiple-choice model: its labels are one int64 choice index per "
                         "example (-100 on ignored ones) and its loss is CrossEntropyLoss over the [batch, num_choices] "
                         "logits, as HF's BertForMultipleChoice computes it" % type(criterion).__name__)


def check_qa_criterion(criterion):
    """HF's question-answering head computes its own span loss and takes no external one: the criterion is None or a
    plain CrossEntropyLoss() (both train that in-model loss); anything else raises ValueError."""
    if criterion is None:
        return
    plain = (type(criterion) is torch.nn.CrossEntropyLoss and criterion.weight is None
             and criterion.ignore_index == -100 and criterion.label_smoothing == 0.0 and criterion.reduction == "mean")
    if not plain:
        raise ValueError("a BertForQuestionAnswering trains HF's in-model span loss (a CrossEntropyLoss over each "
                         "sequence's tokens, ignore_index = the padded length): pass no criterion or a plain "
                         "CrossEntropyLoss(), got %r" % (criterion,))


def qa_positions(batch_data):
    """a question-answering batch's HF keys start_positions / end_positions (int64 [B] or [B, 1]) as one int64
    [2, B] tensor: row 0 the starts, row 1 the ends"""
    st, en = batch_data["start_positions"], batch_data["end_positions"]
    if st.is_floating_point() or en.is_floating_point() or st.numel() != en.numel():
        raise ValueError("start_positions / end_positions must be int64 with one per sequence, got %s %s / %s %s"
                         % (st.dtype, list(st.shape), en.dtype, list(en.shape)))
    return torch.stack([st.reshape(-1), en.reshape(-1)])


def best_spans(start_logits, end_logits, attention_mask, max_answer_length=30):
    """run_qa.py's span choice per sequence, as torch ops on the logits' device: the (s, e) with the largest
    start_logits[s] + end_logits[e] among s <= e < s + max_answer_length, both valid tokens (attention_mask 1;
    position 0 included, so (0, 0) is the no-answer prediction).  int64 [B, 2]."""
    B, S = start_logits.shape
    dev = start_logits.device
    score = start_logits.float()[:, :, None] + end_logits.float()[:, None, :]
    ar = torch.arange(S, device=dev)
    ok = (ar[None, :] >= ar[:, None]) & (ar[None, :] < ar[:, None] + int(max_answer_length))
    valid = torch.ones(B, S, dtype=torch.bool, device=dev) if attention_mask is None else attention_mask.to(dev) != 0
    ok = ok[None] & valid[:, :, None] & valid[:, None, :]
    best = score.masked_fill(~ok, float("-inf")).view(B, S * S).argmax(1)
    return torch.stack([best // S, best % S], 1)


def check_mlm_criterion(criterion, device_loss=False):
    """the criteria of a masked-LM model: CrossEntropyLoss (HF's loss) or none.  device_loss: the loss is the device
    head's over the labelled rows (captured steps, dev()), which computes the mean cross-entropy with an ignore_index
    and nothing else: class weights, label smoothing or another reduction raise ValueError."""
    if criterion is not None and not isinstance(criterion, torch.nn.CrossEntropyLoss):
        raise ValueError("a BertForMaskedLM trains with CrossEntropyLoss (or no criterion: HF's in-model loss), got %s"
                         % type(criterion).__name__)
    if device_loss and criterion is not None and (criterion.weight is not None or criterion.label_smoothing != 0.0
                                                  or criterion.reduction != "mean"):
        raise ValueError("the masked-LM head on the device computes CrossEntropyLoss(reduction='mean') with an "
                         "ignore_index only, not class weights, label smoothing or reduction=%r: set args.fused = "
                         "False to apply this criterion to the full logits" % criterion.reduction)


CHECKPOINT_PREFIX = "checkpoint"     # HF Trainer's PREFIX_CHECKPOINT_DIR: output_dir/checkpoint-{optimizer step}


def sorted_checkpoints(output_dir):
    """the checkpoint-N directories under `output_dir`, oldest (smallest N) first"""
    if output_dir is None or not os.path.isdir(output_dir):
        return []
    found = []
    for name in os.listdir(output_dir):
        m = re.fullmatch(CHECKPOINT_PREFIX + r"-(\d+)", name)
        if m and os.path.isdir(os.path.join(output_dir, name)):
            found.append((int(m.group(1)), os.path.join(output_dir, name)))
    return [path for _n, path in sorted(found)]


def latest_checkpoint(output_dir):
    """HF's get_last_checkpoint: the checkpoint-N directory with the largest N, or None"""
    found = sorted_checkpoints(output_dir)
    return found[-1] if found else None


def rotate_checkpoints(output_dir, save_total_limit):
    """deletes the oldest checkpoint-N directories beyond the newest `save_total_limit` (None or <= 0: keeps all, as
    HF does)"""
    if save_total_limit is None or int(save_total_limit) <= 0:
        return
    found = sorted_checkpoints(output_dir)
    for path in found[:max(0, len(found) - int(save_total_limit))]:
        shutil.rmtree(path)


def step_loss(model, criterion=None, choices=None):
    """The losses.Loss a captured step computes: `criterion`'s when it is one the device kernel reproduces (else
    ValueError), and with no criterion the model's problem-type loss -- single-label cross-entropy when the config has
    no problem_type and more than one label (the step then stages int64 labels, as the reference's Collate yields).
    A multiple-choice model's loss runs over `choices` logits per example."""
    m = _unwrap(model)
    if _is_mc(m):
        check_mc_criterion(criterion)
        if criterion is None:
            return m.choice_loss(choices)
        return loss_from_criterion(criterion, choices, m._engine.dev if m._engine is not None else None)
    if _is_qa(m):
        check_qa_criterion(criterion)
        return None       # the span loss (csrc/qa_head.cu) has no options
    if _is_mlm(m):
        check_mlm_criterion(criterion, device_loss=True)
        return Loss(L.LOSS_CE, m.config.vocab_size, ignore_index=getattr(criterion, "ignore_index", -100))
    if _is_token(m):
        check_token_criterion(criterion)
        if criterion is None:
            return Loss(L.LOSS_CE, m.num_labels)      # HF's in-model loss of the token model
    if criterion is not None:
        return loss_from_criterion(criterion, m.num_labels, m._engine.dev if m._engine is not None else None)
    pt = getattr(m.config, "problem_type", None)
    if pt is None:
        pt = "regression" if m.num_labels == 1 else "single_label_classification"
    return problem_type_loss(pt, m.num_labels)


def qa_scores(spans):
    """(exact match, position-level F1) of int64 [N, 4] rows (pred start, pred end, gold start, gold end): exact match
    is pred == gold; F1 is that of the predicted and gold position ranges [start, end] (an empty predicted range, end <
    start, cannot occur: best_spans keeps start <= end), averaged over the rows.  (nan, nan) for no rows."""
    if spans.shape[0] == 0:
        return float("nan"), float("nan")
    p = spans.double()
    em = float(((spans[:, 0] == spans[:, 2]) & (spans[:, 1] == spans[:, 3])).double().mean())
    overlap = (torch.minimum(p[:, 1], p[:, 3]) - torch.maximum(p[:, 0], p[:, 2]) + 1).clamp(min=0)
    prec = overlap / (p[:, 1] - p[:, 0] + 1)
    rec = overlap / (p[:, 3] - p[:, 2] + 1)
    f1 = torch.where(overlap > 0, 2 * prec * rec / (prec + rec), torch.zeros_like(overlap))
    return em, float(f1.mean())


class _StagedGraphStep:
    """Shared plumbing of the graph-captured steps: one pinned staging buffer for the four host tensors of a batch, one
    async H2D copy, two eager warm-up passes (first launches set kernel attributes), then capture + replay."""

    def __init__(self, model, batch_size, seq_len, use_graph=True, criterion=None, choices=None):
        """choices: a multiple-choice model's N; its steps take [batch_size, N, seq_len] batches and run their
        batch_size x N choice sequences as rows"""
        self.wrapper = model if isinstance(model, DistributedDataParallel) else None
        self.model = _unwrap(model)
        self.eng = self.model._engine
        if self.eng is None:
            raise RuntimeError("%s: model must be on CUDA" % type(self).__name__)
        dev = self.eng.dev
        self.mc = _is_mc(self.model)
        if self.mc != (choices is not None):
            raise ValueError("%s: choices=N is %s" % (type(self).__name__, "required for a multiple-choice model"
                                                       if self.mc else "for multiple-choice models only"))
        self.N = choices
        self.examples = batch_size            # labelled examples (sequences, or multiple-choice examples)
        self.batch_shape = (batch_size, seq_len) if not self.mc else (batch_size, choices, seq_len)
        if self.mc and not isinstance(self, PackedTrainStep):
            batch_size *= choices             # one row per choice sequence
        self.B, self.S = batch_size, seq_len
        self.loss_fn = step_loss(self.model, criterion, choices)
        self.criterion_key = criterion_key(criterion)
        self.token = _is_token(self.model)     # labels per token row: B * S int64 slots
        # masked-LM: the head runs on the labelled rows; the host counts them while staging, and the graphs are kept
        # per capacity (the count rounded up to 128)
        self.mlm = _is_mlm(self.model)
        self.token = self.token or self.mlm
        # question answering: the start and end positions of each sequence, two int64 slots per sequence ([2, B])
        self.qa = _is_qa(self.model)
        self.ignored_index = seq_len      # HF's ignored index of the span loss (a packed step: the padded length)
        self._cap, self._n_lab = None, 0
        z = lambda *s: torch.zeros(*s, dtype=torch.int64, device=dev)
        self.d_ids, self.d_tt, self.d_mask = z(batch_size, seq_len), z(batch_size, seq_len), z(batch_size, seq_len)
        self.d_lab, lab_slots = self._label_buffer(batch_size * seq_len if self.token else self.examples)
        self._alloc_stage(3 * batch_size * seq_len + lab_slots)
        self.loss_out = torch.zeros((), dtype=torch.float32, device=dev)
        self.h_loss = torch.zeros((), dtype=torch.float32).pin_memory()
        self.use_graph = use_graph
        self.graph = None         # the graph of the optimizer-step body (the only one without accumulation)
        self._graphs = {}         # role -> graph, role = (final pass, window already holds gradients), see run_device
        self._warm = {}
        self._graph_hp = {}       # role -> the optimizer hyperparameters its graph was captured with
        self._role = (True, False)
        self.accum_steps = 1
        self.max_grad_norm = None
        self._h2d_done = None
        # The step body -- the critical chain of forward / dgrad kernels -- is issued (and captured) on a HIGH-priority
        # stream, so that when an SM frees up the block scheduler hands it to the critical path before the
        # weight-gradient / optimizer streams (default, i.e. lowest, priority).
        self._prio_stream = torch.cuda.Stream(device=dev, priority=-1)

    def _label_buffer(self, rows):
        """device labels of `rows` sequences for self.loss_fn, and the int64 staging slots they take: int64 [rows]
        class indices, or fp32 [rows] / [rows, C] packed two to a slot"""
        dev = self.eng.dev
        if self.qa:
            return torch.zeros(2, rows, dtype=torch.int64, device=dev), 2 * rows
        shape = self.loss_fn.label_shape(rows)
        if not self.loss_fn.float_labels:
            return torch.zeros(shape, dtype=torch.int64, device=dev), rows
        t = torch.zeros(shape, dtype=torch.float32, device=dev)
        return t, (t.numel() + 1) // 2

    def _stage_labels(self, hs, lab):
        """host labels -> the label slots `hs` of the pinned staging buffer (fp32 labels bit for bit)"""
        fn = self.loss_fn
        if self.qa:
            if lab.is_floating_point() or tuple(lab.shape) != tuple(self.d_lab.shape):
                raise ValueError("%s was built for int64 start / end positions %s, got %s %s"
                                 % (type(self).__name__, list(self.d_lab.shape), lab.dtype, list(lab.shape)))
            hs.copy_(lab.reshape(-1))
            return
        if self.token or self.mc:
            self._check_token_labels(lab)
        if self.mlm:
            n = int((lab != fn.ignore_index).sum())
            self._n_lab = n
            self._cap = min(lab.numel(), max(128, (n + 127) // 128 * 128))
        if not fn.float_labels:
            if lab.is_floating_point():
                raise TypeError("%s was built for int64 class labels, got %s: pass a criterion (or config.problem_type)"
                                " for float labels" % (type(self).__name__, lab.dtype))
            hs.copy_(lab.reshape(-1))
            return
        try:
            fn.check_labels(lab, self.d_lab.shape[0])
        except (TypeError, ValueError) as e:
            raise type(e)("%s was built for %s labels of shape %s: %s"
                          % (type(self).__name__, "fp32", list(self.d_lab.shape), e)) from None
        hs.view(torch.float32)[:self.d_lab.numel()].copy_(lab.reshape(-1))

    def _check_token_labels(self, lab):
        """host token labels: int64, one per staged row, each a class index or the loss's ignore_index (the loss
        kernel traps on anything else; padding must carry the ignore index, as HF's tagging collators put there).
        A multiple-choice step's labels likewise: one choice index per example."""
        what = "choice" if self.mc else "token"
        if lab.is_floating_point():
            raise TypeError("%s labels are int64 class indices (CrossEntropyLoss), got %s" % (what, lab.dtype))
        if lab.numel() != self.d_lab.numel() or (self.mc and lab.dim() != 1):
            raise ValueError("%s was built for %d %s labels, got %s" % (type(self).__name__, self.d_lab.numel(), what,
                                                                        list(lab.shape)))
        fn = self.loss_fn
        bad = (lab != fn.ignore_index) & ((lab < 0) | (lab >= fn.C))
        if bool(bad.any()):
            raise ValueError("%s label %d is outside [0, %d) and is not the ignore_index %d%s"
                             % (what, int(lab[bad].flatten()[0]), fn.C, fn.ignore_index,
                                "" if self.mc else " (padding positions must carry the ignore_index)"))

    def _unstage_labels(self, st):
        if self.qa:
            self.d_lab.view(-1).copy_(st)
        elif self.loss_fn.float_labels:
            self.d_lab.view(-1).copy_(st.view(torch.float32)[:self.d_lab.numel()])
        else:
            self.d_lab.copy_(st)

    def _unstage(self):
        n = self.B * self.S
        st = self.d_stage
        self.d_ids.copy_(st[0:n].view(self.B, self.S))
        self.d_tt.copy_(st[n:2 * n].view(self.B, self.S))
        self.d_mask.copy_(st[2 * n:3 * n].view(self.B, self.S))
        self._unstage_labels(st[3 * n:])

    def _body(self):
        raise NotImplementedError

    def _alloc_stage(self, n):
        """pinned / device staging of n int64 for the batch (h_stage / d_stage), then one slot carrying
        param_groups[0]["lr"] as float64 bits: both travel in the one H2D copy of stage()"""
        self._h_stage_all = torch.zeros(n + 1, dtype=torch.int64).pin_memory()
        self._d_stage_all = torch.zeros_like(self._h_stage_all, device=self.eng.dev)
        self.h_stage, self.d_stage = self._h_stage_all[:n], self._d_stage_all[:n]

    def _head_kw(self, train):
        """the head's forward arguments.  Masked-LM: labelled rows only, this batch's capacity, and in training the
        d_loss scale that makes the loss launch also write d_logits.  Question answering: that d_loss scale, and a
        packed step's ignored index."""
        if self.qa:
            kw = dict(qa_dloss=self._mlm_dloss) if train else {}
            if isinstance(self, PackedTrainStep):
                kw["qa_ignored_index"] = self.ignored_index
            return kw
        if not self.mlm:
            return {}
        kw = dict(mlm_full=False, ignore_index=self.loss_fn.ignore_index, mlm_capacity=self._cap)
        if train:
            kw["mlm_dloss"] = self._mlm_dloss
        return kw

    def _stage_lr(self):
        opt = getattr(self, "opt", None)
        if opt is not None:
            self._h_stage_all[-1:].view(torch.float64).fill_(opt.current_lr())

    def _h2d(self):
        self._d_stage_all.copy_(self._h_stage_all, non_blocking=True)
        self._h2d_done = torch.cuda.Event()
        self._h2d_done.record(torch.cuda.current_stream(self.eng.dev))

    def _unstage_lr(self):
        self.opt._state()["lr"].copy_(self._d_stage_all[-1:].view(torch.float64))

    def stage(self, batch_data):
        """Host batch (the dict the reference Collate yields, int64 tensors) -> pinned staging -> async H2D."""
        n = self.B * self.S
        ids, tt, mask = batch_data["input_ids"], batch_data["token_type_ids"], batch_data["attention_mask"]
        lab = qa_positions(batch_data) if self.qa else batch_data["label"]
        if tuple(ids.shape) != self.batch_shape:
            raise ValueError("%s was built for batch %s, got %s"
                             % (type(self).__name__, "x".join(map(str, self.batch_shape)), tuple(ids.shape)))
        hs = self.h_stage
        if self._h2d_done is not None:
            self._h2d_done.synchronize()  # previous step's copy out of the pinned staging buffer has drained
        hs[0:n].copy_(ids.reshape(-1))
        hs[n:2 * n].copy_(tt.reshape(-1))
        hs[2 * n:3 * n].copy_(mask.reshape(-1))
        self._stage_labels(hs[3 * n:], lab)
        self._stage_lr()
        self._h2d()

    def _run_body(self):
        cur = torch.cuda.current_stream(self.eng.dev)
        self._prio_stream.wait_stream(cur)
        with torch.cuda.stream(self._prio_stream):
            self._body()
        cur.wait_stream(self._prio_stream)

    def run_device(self, final=True):
        """The step with inputs already staged on the device (bench `value` path).  final=False: a micro-batch of a
        gradient-accumulation window (forward, backward, accumulate; no optimizer step)."""
        opt = getattr(self, "opt", None)
        if opt is not None and torch.are_deterministic_algorithms_enabled() != self.deterministic:
            raise RuntimeError("%s was built with torch.use_deterministic_algorithms(%s) and is called with it %s; its "
                               "captured backward keeps the summation order it was built with, so build a new %s in "
                               "this mode" % (type(self).__name__, self.deterministic,
                                              "on" if not self.deterministic else "off", type(self).__name__))
        # the body's accumulation mode (STORE / ADD / FOLD / none) follows from these two, and a graph replay runs no
        # Python: one graph per combination, and the host-side flags are kept current here
        self._role = (final, opt is not None and self.eng.accum_live)
        if self.mlm:
            self._role += (self._cap,)
        self._run_device()
        if opt is not None:
            self.eng.accum_live = not final
            if final:
                # a replay runs no Python: tell the transport the weights moved (under a peer group the next
                # state_dict() pulls the other ranks' slices again)
                opt._transport().stepped()

    def _run_device(self):
        if not self.use_graph:
            self._run_body()
            return
        role = self._role
        g = self._graphs.get(role)
        if g is None:
            if self._warm.get(role, 0) < 2:
                # eager warm-up: first launches set kernel attributes, DDP arms its overlap path
                self._run_body()
                self._warm[role] = self._warm.get(role, 0) + 1
                return
            torch.cuda.synchronize(self.eng.dev)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._run_body()
            self._graphs[role] = g
            if getattr(self, "opt", None) is not None:
                self._graph_hp[role] = self.opt.captured_hparams()
            if role[0]:
                self.graph = g
        elif role in self._graph_hp:
            self._check_hparams(self._graph_hp[role])
        g.replay()

    def _check_hparams(self, captured):
        """a replay reads the lr live; every other optimizer hyperparameter is the one the graph was captured with"""
        now = self.opt.captured_hparams()
        for field, was in captured.items():
            if now[field] != was:
                raise RuntimeError("%s: the optimizer's %s changed from %r to %r after the step was captured; the "
                                   "captured step reads only the lr at each replay, so build a new %s to use it"
                                   % (type(self).__name__, field, was, now[field], type(self).__name__))

    def _arm(self, optimizer, accum_steps, max_grad_norm=None):
        self.opt = optimizer
        # the backward's summation order is baked into the graph: fixed-order under use_deterministic_algorithms
        self.deterministic = torch.are_deterministic_algorithms_enabled()
        self.accum_steps = accum_steps
        self.max_grad_norm = float(max_grad_norm) if max_grad_norm else None
        # the masked-LM and span losses' gradient scale (1/k under accumulation), read by their loss launch
        self._mlm_dloss = torch.full((), 1.0 / accum_steps, dtype=torch.float32, device=self.eng.dev)
        if accum_steps > 1:
            self.eng.ensure_accum()       # outside any capture
        # a valid lr in the device slot before any stage(): run_device() on inputs written straight into d_stage
        # replays at the lr current when the step was built (or last staged)
        self._stage_lr()
        self._d_stage_all[-1:].copy_(self._h_stage_all[-1:])
        # the fused step owns backward + optimizer: each bucket's update (in a peer group, its exchange) may start
        # while backward is still running (optimizer.bucket_ready)
        optimizer._armed = True

    def _train_body(self, forward):
        """forward() -> (logits, loss): the common part of the captured train steps.  A micro-batch body
        (self._role[0] False) accumulates its gradients and bumps the dropout stream instead of stepping; the final
        body folds the window in before the update.  The staged lr goes to the optimizer's device lr first, and every
        update (and step-size prepare) of the body reads it from there, so a replay applies the lr of its own step."""
        self._unstage_lr()
        self.opt._lr_dev_on = True
        try:
            self._train_pass(forward, self._role[0])
        finally:
            self.opt._lr_dev_on = False

    def _train_pass(self, forward, final):
        eng, opt = self.eng, self.opt
        logits, loss = forward()
        B, S, mask, p_h, p_a, p_c, packed = eng._saved
        eng._saved = None
        Bo = eng.head_rows(B, S, packed)
        ws = eng.workspace(B, S, Bo)
        if self.accum_steps > 1 and not (self.mlm or self.qa):
            ws["dloss_logits"].mul_(1.0 / self.accum_steps)     # what an eager loop does with loss / k
        # d(loss)/d(logits) was produced by the loss kernel: the reference's criterion(logits, label) [:169]
        if final and self.max_grad_norm is not None:
            opt._clip_arm(self.max_grad_norm)     # the backward's per-bucket launches become the reduce phase
        eng.start_pass(not final)
        # (masked-LM: the forward's cross-entropy launch left the labelled rows' d_logits for the backward; the span
        # loss's launch left them scaled by 1/k)
        eng._backward_from_dlogits(None if self.mlm else ws["dloss_logits"], B, S, mask, p_h, p_a, p_c, packed)
        eng.end_pass()
        if final:
            opt.step()
        self.loss_out.copy_(loss)

    def loss_to_host(self):
        self.h_loss.copy_(self.loss_out, non_blocking=True)
        torch.cuda.current_stream(self.eng.dev).synchronize()
        return float(self.h_loss)


class FusedTrainStep(_StagedGraphStep):
    """One training step == one CUDA-graph replay: H2D of the batch, embeddings -> 12 layers -> head -> CE, the full
    backward, the peer-HBM gradient exchange fused with AdamW, and the device-side step/RNG bump.  Semantically the body
    of the reference loop [:166-176] without the host round trips.  accum_steps = k > 1: gradient accumulation over k
    micro-batches, the loss scaled by 1/k; call with final=False for the first k - 1 of a window.  max_grad_norm:
    clip the gradient's 2-norm before the update (see clip_grad_norm_); the norm is left in optimizer._clip_buf."""

    def __init__(self, model, optimizer, batch_size, seq_len, use_graph=True, accum_steps=1, max_grad_norm=None,
                 criterion=None, choices=None):
        super().__init__(model, batch_size, seq_len, use_graph, criterion, choices)
        self._arm(optimizer, accum_steps, max_grad_norm)

    # the step body, expressed only with stream-ordered work (capturable)
    def _body(self):
        self._unstage()
        self._train_body(lambda: self.eng.forward(self.d_ids, self.d_tt, self.d_mask, self.d_lab, training=True,
                                                  need_backward=True, loss_fn=self.loss_fn, **self._head_kw(True)))

    def __call__(self, batch_data, final=True):
        """batch_data: the dict the reference Collate yields (host int64 tensors; fp32 labels for regression and
        multi-label).  Returns the device loss scalar (local rank's mean loss, like `loss` at [:169]; unscaled under
        accumulation)."""
        self.stage(batch_data)
        self.run_device(final)
        return self.loss_out


class PackedTrainStep(_StagedGraphStep):
    """FusedTrainStep for PACKED batches (packing.pack_batch): `bins` bins of `bin_len` tokens carrying `batch`
    sequences.  One instance (staging buffers + CUDA graph) per bin count and length; the Trainer keeps a small cache of
    them, since the bins a batch packs into vary with its lengths."""

    def __init__(self, model, optimizer, bins, batch, use_graph=True, accum_steps=1, max_grad_norm=None,
                 criterion=None, bin_len=128, seq_len=None, choices=None):
        """seq_len: a question-answering model's padded length before packing, HF's ignored index (None: bin_len).
        choices: a multiple-choice model's N; the bins then carry batch x N choice sequences"""
        super().__init__(model, bins, bin_len, use_graph, criterion, choices)
        if seq_len is not None:
            self.ignored_index = int(seq_len)
        dev = self.eng.dev
        self.bins, self.batch, self.bin_len = bins, batch, bin_len
        self.ncls = batch * choices if self.mc else batch      # sequences in the bins
        n = bins * bin_len
        # pinned staging: ids | token types | positions | segments (as int64) | cls rows | labels (per sequence or
        # multiple-choice example, or per bin row for a token model: pack_batch's "labels")
        self.d_lab, lab_slots = self._label_buffer(n if self.token else batch)
        self._alloc_stage(4 * n + self.ncls + lab_slots)
        z = lambda *sh: torch.zeros(*sh, dtype=torch.int64, device=dev)
        self.d_pos, self.d_cls = z(bins, bin_len), z(self.ncls)
        self.d_seg = torch.zeros(bins, bin_len, dtype=torch.int32, device=dev)
        self._arm(optimizer, accum_steps, max_grad_norm)

    def _unstage(self):
        n, st, S = self.bins * self.bin_len, self.d_stage, self.bin_len
        self.d_ids.copy_(st[0:n].view(self.bins, S))
        self.d_tt.copy_(st[n:2 * n].view(self.bins, S))
        self.d_pos.copy_(st[2 * n:3 * n].view(self.bins, S))
        self.d_seg.copy_(st[3 * n:4 * n].view(self.bins, S))            # int64 -> int32
        self.d_cls.copy_(st[4 * n:4 * n + self.ncls])
        self._unstage_labels(st[4 * n + self.ncls:])

    def stage(self, packed, label):
        n, hs = self.bins * self.bin_len, self.h_stage
        want = (self.bins, self.bin_len) if self.token else (2, self.batch) if self.qa else (self.batch,)
        if packed["bins"] != self.bins or packed["input_ids"].shape[1] != self.bin_len or \
                tuple(label.shape[:len(want)]) != want or packed["cls_index"].numel() != self.ncls:
            raise ValueError("PackedTrainStep was built for %d bins of %d tokens / %d sequences"
                             % (self.bins, self.bin_len, self.ncls))
        if self._h2d_done is not None:
            self._h2d_done.synchronize()
        hs[0:n].copy_(packed["input_ids"].reshape(-1))
        hs[n:2 * n].copy_(packed["token_type_ids"].reshape(-1))
        hs[2 * n:3 * n].copy_(packed["position_ids"].reshape(-1))
        hs[3 * n:4 * n].copy_(packed["segments"].reshape(-1))
        hs[4 * n:4 * n + self.ncls].copy_(packed["cls_index"].reshape(-1))
        self._stage_labels(hs[4 * n + self.ncls:], label)
        self._stage_lr()
        self._h2d()

    def _body(self):
        self._unstage()
        packed = (self.d_pos, self.d_seg, None if self.token else self.d_cls)
        self._train_body(lambda: self.eng.forward(self.d_ids, self.d_tt, None, self.d_lab, training=True,
                                                  need_backward=True, packed=packed, loss_fn=self.loss_fn,
                                                  **self._head_kw(True)))

    def __call__(self, packed, label, final=True):
        """label: per sequence [batch] (a multiple-choice model: per example), for a token model pack_batch's "labels"
        [bins, bin_len], for a question-answering model the int64 [2, batch] start / end positions
        (trainer.qa_positions of pack_batch's)"""
        self.stage(packed, label)
        self.run_device(final)
        return self.loss_out


class FusedEvalStep(_StagedGraphStep):
    """The reference's eval body (`on_step` + `criterion` under `no_grad`, [:204-208] / [:228-229]) as one CUDA-graph
    replay: H2D of the batch, the dropout-free forward, the mean loss of `criterion` (None: the model's problem-type
    loss).  Returns device tensors that are overwritten by the next call (the callers below consume them before
    staging the next batch)."""

    def __init__(self, model, batch_size, seq_len, use_graph=True, criterion=None, choices=None):
        super().__init__(model, batch_size, seq_len, use_graph, criterion, choices)
        shape = (batch_size, seq_len) if self.token else (batch_size,)
        if self.mlm:
            self.logits_out = None    # no [B, S, V] logits: the labelled rows' (pred, label) pairs instead
            self.pred_out = torch.zeros(batch_size * seq_len, dtype=torch.int32, device=self.eng.dev)
            self.lab_out = torch.zeros_like(self.pred_out)
        else:
            if self.qa:
                shape = (batch_size, seq_len)      # [B, S, 2]: start and end logits
            C = choices if self.mc else self.model.num_labels
            self.logits_out = torch.zeros(*shape, C, dtype=torch.float32, device=self.eng.dev)

    def _body(self):
        self._unstage()
        logits, loss = self.eng.forward(self.d_ids, self.d_tt, self.d_mask, self.d_lab, training=False,
                                        need_backward=False, loss_fn=self.loss_fn, **self._head_kw(False))
        if self.mlm:
            gb, cap = self.eng.mlm_last, self._cap
            self.pred_out[:cap].copy_(gb["pred"])
            self.lab_out[:cap].copy_(gb["labels"])
        else:
            self.logits_out.copy_(logits.view(self.logits_out.shape))
        self.loss_out.copy_(loss)

    def __call__(self, batch_data):
        """(logits, labels, mean loss); a masked-LM model: (predicted ids, labels, mean loss) of the labelled tokens,
        in token order; a question-answering model: ([B, S, 2] start / end logits, [2, B] positions, mean loss)"""
        self.stage(batch_data)
        self.run_device()
        if self.mlm:
            n = self._n_lab
            return self.pred_out[:n].long(), self.lab_out[:n].long(), self.loss_out
        return self.logits_out, self.d_lab.view(self.B, self.S) if self.token else self.d_lab, self.loss_out


class Trainer:
    def __init__(self, args, config, model, criterion, optimizer, scheduler=None):
        """scheduler: a torch LR scheduler of `optimizer` (fabric-cls.py's Trainer argument), stepped once per optimizer
        step; it takes precedence over args.lr_scheduler_type"""
        if scheduler is not None and getattr(scheduler, "optimizer", None) is not optimizer:
            raise ValueError("the scheduler must belong to the Trainer's optimizer")
        if model is not None and _is_qa(model):
            check_qa_criterion(criterion)
        if getattr(args, "full_determinism", False):
            torch.use_deterministic_algorithms(True)      # as HF's enable_full_determinism does
        self.args = args
        self.config = config          # (the reference's `self.config = config,` stores a 1-tuple by accident, :121)
        self.model = model
        self.criterion = criterion
        self.optimizer = optimizer
        self._fused = None
        self._packed = {}     # (bins, batch, bin length, deterministic mode) -> PackedTrainStep
        self._scaler = None
        self._fused_eval = {}
        self._pin = {}
        self._micro = 0       # batches of the open gradient-accumulation window
        self.last_grad_norm = None   # device scalar: the pre-clip gradient norm of the last optimizer step (HF's
                                     # logged `grad_norm`); None when not clipping
        self.lr_scheduler = scheduler
        self.global_step = 0  # optimizer steps taken (HF's global_step; checkpoint-N is named by it)
        # where train() is, for trainer_state.json: batches done, the epoch and the batches of it consumed, best_acc
        self._progress = {"batches": 0, "epoch": 1, "batches_in_epoch": 0, "best_acc": 0.0}
        self._epoch_rng = None     # train(): the CPU RNG state the current epoch's loader iterator was created from
        self._loaded_rng = None    # load_checkpoint(): the RNG states it restored (train() re-applies them after a skip)

    def num_training_steps(self, train_loader):
        """optimizer steps train() takes: epochs x ceil(batches / k).  HF Trainer floors batches / k; this Trainer
        also steps the partial window at the end of an epoch (close_window), so a linear schedule reaches 0 exactly
        after the last step."""
        k = max(1, int(getattr(self.args, "gradient_accumulation_steps", 1)))
        return int(self.args.epochs) * math.ceil(len(train_loader) / k)

    def create_scheduler(self, num_training_steps):
        """HF Trainer.create_scheduler: builds self.lr_scheduler from args.lr_scheduler_type / warmup_steps /
        warmup_ratio, unless a scheduler was passed or built already.  Returns it (None: a constant lr)."""
        name = getattr(self.args, "lr_scheduler_type", None)
        if self.lr_scheduler is None and name is not None:
            warm = warmup_steps(num_training_steps, getattr(self.args, "warmup_steps", 0),
                                getattr(self.args, "warmup_ratio", 0.0))
            self.lr_scheduler = get_scheduler(name, self.optimizer, num_warmup_steps=warm,
                                              num_training_steps=num_training_steps)
        return self.lr_scheduler

    def _to_device(self, batch_data):
        dev = _unwrap(self.model)._engine.dev
        out = {}
        keys = ("start_positions", "end_positions") if _is_qa(self.model) else ("label",)
        for k in keys + ("input_ids", "token_type_ids", "attention_mask"):
            t = batch_data[k]
            if t.is_cuda:
                out[k] = t
                continue
            key = (k, tuple(t.shape))
            if key not in self._pin:
                self._pin[key] = [torch.empty(t.shape, dtype=t.dtype).pin_memory(), None]
            buf, ev = self._pin[key]
            if ev is not None:
                ev.synchronize()          # the previous async copy out of this staging buffer has drained
            buf.copy_(t)
            out[k] = buf.to(dev, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(dev))
            self._pin[key][1] = ev
        return out

    def _forward(self, batch_data):
        """on_step's model call: (output, device label); a question-answering model's label is the int64 [2, B]
        start / end positions"""
        d = self._to_device(batch_data)
        if _is_qa(self.model):
            output = self.model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                                attention_mask=d["attention_mask"], start_positions=d["start_positions"],
                                end_positions=d["end_positions"])
            return output, qa_positions(d)
        label = d["label"]
        # a token model with a criterion leaves the loss to it: its in-model CrossEntropyLoss() would not know the
        # criterion's ignore_index
        model_labels = None if self.criterion is not None and (_is_token(self.model) or _is_mlm(self.model)
                                                               or _is_mc(self.model)) else label
        output = self.model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                            attention_mask=d["attention_mask"], labels=model_labels)
        return output, label

    def on_step(self, batch_data):
        output, label = self._forward(batch_data)
        return self._logits(output), label

    def _logits(self, output):
        """the output's logits; a question-answering model's start and end logits stacked as [B, S, 2]"""
        if _is_qa(self.model):
            return torch.stack([output.start_logits, output.end_logits], -1)
        return output.logits

    def problem_type(self, label):
        """the model's config.problem_type; when None, HF's rule applied to `label` (stored on the config, as the
        model's first labelled forward does)"""
        if _is_mlm(self.model):
            return MLM_PROBLEM_TYPE
        if _is_qa(self.model):
            return QA_PROBLEM_TYPE         # HF's QA model never reads or sets config.problem_type
        if _is_mc(self.model):
            return MC_PROBLEM_TYPE         # nor does HF's multiple-choice model
        if _is_token(self.model):
            return TOKEN_PROBLEM_TYPE      # HF's token model never reads or sets config.problem_type
        cfg = _unwrap(self.model).config
        if getattr(cfg, "problem_type", None) is None:
            cfg.problem_type = infer_problem_type(_unwrap(self.model).num_labels, label)
        return cfg.problem_type

    def compute_loss(self, logits, label, model_loss=None):
        """the criterion on the logits (the reference's criterion(logits, label) [:169]); with one label and float
        labels over the squeezed logits, as HF's regression.  No criterion: the model's own loss `model_loss`."""
        if self.criterion is None:
            if model_loss is None:
                raise ValueError("Trainer has no criterion and the model returned no loss")
            return model_loss
        if _is_qa(self.model):
            check_qa_criterion(self.criterion)      # a plain CrossEntropyLoss() stands for the in-model span loss
            if model_loss is None:
                raise ValueError("a BertForQuestionAnswering's loss is its own: the model returned none")
            return model_loss
        if _is_mlm(self.model):
            check_mlm_criterion(self.criterion)
            return self.criterion(logits.reshape(-1, logits.shape[-1]), label.reshape(-1))
        if _is_token(self.model):
            check_token_criterion(self.criterion)
            C = _unwrap(self.model).num_labels
            return self.criterion(logits.reshape(-1, C), label.reshape(-1))
        if _is_mc(self.model):
            check_mc_criterion(self.criterion)
            return self.criterion(logits, label)
        if _unwrap(self.model).num_labels == 1 and label.is_floating_point():
            return self.criterion(logits.reshape(-1), label.reshape(-1))
        return self.criterion(logits, label)

    def _eager_loss(self, batch_data):
        """the eager loops' forward + loss: on_step and the criterion, or with no criterion the model's own loss"""
        if self.criterion is None or _is_qa(self.model):
            output, _label = self._forward(batch_data)
            return output[0]
        logits, label = self.on_step(batch_data)
        return self.compute_loss(logits, label)

    def _eval_forward(self, batch_data):
        """(logits, label, the model's loss) of a no-grad batch: the graph-captured forward when ``args.fused`` (one
        replay per batch instead of ~100 eager launches), else the eager call"""
        if not getattr(self.args, "fused", True) or batch_data["input_ids"].is_cuda:
            output, label = self._forward(batch_data)
            return self._logits(output), label, output.loss
        self.problem_type(batch_data.get("label"))
        shape = tuple(batch_data["input_ids"].shape)
        m = _unwrap(self.model)
        # a token (or multiple-choice) model's staged labels are checked against its loss's ignore_index: the
        # criterion's
        crit = self.criterion if _is_token(m) or _is_mc(m) else None
        key = (id(m), shape, m.config.problem_type, criterion_key(crit))     # `test` may swap the model [:222-224]
        if key not in self._fused_eval:
            choices = _choices(batch_data) if _is_mc(m) else None
            self._fused_eval[key] = FusedEvalStep(self.model, shape[0], shape[-1], criterion=crit, choices=choices)
        return self._fused_eval[key](batch_data)

    def eval_step(self, batch_data):
        """`on_step` for the no-grad loops.  Returns (logits, label) like `on_step`."""
        logits, label, _loss = self._eval_forward(batch_data)
        return logits, label

    def _captured_loss_key(self, label):
        """what a cached captured step must have been built for: the criterion's loss parameters, or with no
        criterion the model's problem type.  An unset problem type is inferred from this batch's labels either way, as
        the eager path's labelled forward does."""
        problem_type = self.problem_type(label)
        if self.criterion is None:
            return None, problem_type
        return criterion_key(self.criterion), None

    def loss_reduce(self, loss):
        if isinstance(self.model, DistributedDataParallel):
            return self.model.loss_reduce(loss)
        return loss.clone()

    def output_reduce(self, outputs, targets):
        if isinstance(self.model, DistributedDataParallel):
            return self.model.all_gather_rows(outputs), self.model.all_gather_rows(targets)
        return outputs.clone(), targets.clone()

    def train_step(self, batch_data):
        """One step of the reference loop body [:166-176]; returns the rank-averaged loss (device scalar).  With
        args.gradient_accumulation_steps = k > 1 a call is one micro-batch: the first k - 1 of a window accumulate
        (inside no_sync() on the eager paths), the k-th also steps the optimizer; every loss is scaled by 1/k
        (fabric-cls.py:150-157) and the returned loss is the unscaled micro-batch loss."""
        k = max(1, int(getattr(self.args, "gradient_accumulation_steps", 1)))
        if self.lr_scheduler is None and getattr(self.args, "lr_scheduler_type", None) is not None:
            raise RuntimeError("args.lr_scheduler_type is set but no scheduler was built: call "
                               "trainer.create_scheduler(num_training_steps) first (train() does)")
        clip = self._max_grad_norm()
        first, final = self._micro == 0, self._micro >= k - 1
        self._micro = 0 if final else self._micro + 1
        qa = _is_qa(self.model)
        choices = _choices(batch_data) if _is_mc(self.model) else None
        if getattr(self.args, "fused", True) and getattr(self.args, "pack", False) and \
                batch_data["input_ids"].shape[-1] <= MAX_BIN and not batch_data["input_ids"].is_cuda:
            bin_len = bin_length(batch_data["attention_mask"], batch_data["input_ids"].shape[-1])
            token = _is_token(self.model) or _is_mlm(self.model)
            qa_kw = dict(start_positions=batch_data["start_positions"],
                         end_positions=batch_data["end_positions"]) if qa else {}
            packed = pack_batch(batch_data["input_ids"], batch_data["token_type_ids"], batch_data["attention_mask"],
                                bin_len, labels=batch_data["label"] if token else None,
                                ignore_index=self._ignore_index(), **qa_kw)
            key = (packed["bins"], batch_data["input_ids"].shape[0], bin_len,
                   torch.are_deterministic_algorithms_enabled())
            if qa:
                key += (packed["seq_len"],)        # the span loss's ignored index is part of the captured step
            if choices is not None:
                key += (choices,)
            lkey = self._captured_loss_key(batch_data.get("label"))
            if key not in self._packed or (self._packed[key].accum_steps, self._packed[key].max_grad_norm,
                                           self._packed[key].loss_key) != (k, clip, lkey):
                if len(self._packed) >= 16:           # bound the graph cache: drop the oldest entry
                    self._packed.pop(next(iter(self._packed)))
                self._packed[key] = PackedTrainStep(self.model, self.optimizer, key[0], key[1], accum_steps=k,
                                                    max_grad_norm=clip, criterion=self.criterion, bin_len=bin_len,
                                                    seq_len=packed["seq_len"] if qa else None, choices=choices)
                self._packed[key].loss_key = lkey
            self.model.train()
            label = packed["labels"] if token else qa_positions(packed) if qa else batch_data["label"]
            loss = self._packed[key](packed, label, final)
            if final:
                self._scheduler_step()      # after the replay: the next stage() reads the new lr
        elif getattr(self.args, "fused", True):
            shape = tuple(batch_data["input_ids"].shape)
            lkey = self._captured_loss_key(batch_data.get("label"))
            det = torch.are_deterministic_algorithms_enabled()
            if self._fused is None or (self._fused.batch_shape, self._fused.accum_steps, self._fused.max_grad_norm,
                                       self._fused.loss_key, self._fused.deterministic) != (shape, k, clip, lkey, det):
                self._fused = FusedTrainStep(self.model, self.optimizer, shape[0], shape[-1], accum_steps=k,
                                             max_grad_norm=clip, criterion=self.criterion, choices=choices)
                self._fused.loss_key = lkey
            self.model.train()
            loss = self._fused(batch_data, final)
            if final:
                self._scheduler_step()
        elif getattr(self.args, "use_amp", False):
            # the -amp scripts' loop body (multi-gpu-distributed-mp-amp-cls.py:166-171), scaler created once
            if self._scaler is None:
                self._scaler = torch.amp.GradScaler("cuda")
            self.model.train()
            with self._window(final):
                with torch.autocast("cuda"):
                    loss = self._eager_loss(batch_data)
                self._scaler.scale(loss / k if k > 1 else loss).backward()
            if final:
                self._clip(clip)        # no scaler.unscale_: step() takes the scale out of the norm
                self._scaler_step()
        else:
            self.model.train()
            with self._window(final):
                loss = self._eager_loss(batch_data)
                if first:
                    self.optimizer.zero_grad()
                (loss / k if k > 1 else loss).backward()
            if final:
                self._clip(clip)
                self.optimizer.step()
                self._scheduler_step()
        if final:
            self._note_grad_norm(clip)
            self.global_step += 1
        return self.loss_reduce(loss.detach())

    def _ignore_index(self):
        """the token labels' ignore index: the criterion's, else CrossEntropyLoss()'s -100"""
        return int(getattr(self.criterion, "ignore_index", -100))

    def _scheduler_step(self):
        if self.lr_scheduler is not None:
            self.lr_scheduler.step()

    def _scaler_step(self):
        """GradScaler step + update; the scheduler steps only if the optimizer ran (HF Trainer 4.28: the scale did
        not drop).  Reading the scale is one host sync per step, on this eager path only."""
        if self.lr_scheduler is None:
            self._scaler.step(self.optimizer)
            self._scaler.update()
            return
        scale_before = self._scaler.get_scale()
        self._scaler.step(self.optimizer)
        self._scaler.update()
        if scale_before <= self._scaler.get_scale():
            self.lr_scheduler.step()

    def _max_grad_norm(self):
        m = getattr(self.args, "max_grad_norm", None)
        return float(m) if m else None

    def _clip(self, clip):
        if clip is not None:
            clip_grad_norm_(self.model.parameters(), clip)

    def _note_grad_norm(self, clip):
        buf = self.optimizer._clip_buf
        self.last_grad_norm = buf["norm"].clone() if clip is not None and buf is not None else None

    def _window(self, final):
        """the eager loops' micro-batches run inside no_sync(), the final one of a window outside it"""
        return contextlib.nullcontext() if final else self.model.no_sync()

    def close_window(self):
        """Steps the optimizer on a partial accumulation window (end of an epoch, as HF Trainer does); the 1/k scale
        stays.  No-op when no window is open."""
        if self._micro == 0:
            return
        self._micro = 0
        clip = self._max_grad_norm()
        self._clip(clip)
        if self._scaler is not None and not getattr(self.args, "fused", True):
            self._scaler_step()
        else:
            self.optimizer.step()
            self._scheduler_step()
        self._note_grad_norm(clip)
        self.global_step += 1

    # ---- checkpoints (HF Trainer's checkpoint-N layout) -------------------------------------------------------------------
    def _rank(self):
        return self.model.rank if isinstance(self.model, DistributedDataParallel) else 0

    def save_checkpoint(self, output_dir):
        """Writes HF Trainer's checkpoint layout into `output_dir`: ``pytorch_model.bin`` and ``config.json`` of the
        unwrapped model (what ``from_pretrained`` reads), ``optimizer.pt``, ``scheduler.pt``, ``scaler.pt`` (when there
        is a GradScaler), ``trainer_state.json``, and ``rng_state_{rank}.pth`` (python, numpy, torch CPU / CUDA and the
        model's dropout stream, and inside train() the CPU RNG state the epoch's loader iterator was created from).
        Rank 0 writes everything but the RNG files, which every rank writes for itself; under
        DistributedDataParallel every rank must call it.  Only at an optimizer-step boundary."""
        if self._micro != 0:
            raise RuntimeError("save_checkpoint(): a gradient-accumulation window is open (%d of %d batches); "
                               "checkpoints are taken between optimizer steps"
                               % (self._micro, int(getattr(self.args, "gradient_accumulation_steps", 1))))
        m, rank = _unwrap(self.model), self._rank()
        os.makedirs(output_dir, exist_ok=True)
        if rank == 0:
            m.save_pretrained(output_dir)
            torch.save(self.optimizer.state_dict(), os.path.join(output_dir, "optimizer.pt"))
            if self.lr_scheduler is not None:
                torch.save(self.lr_scheduler.state_dict(), os.path.join(output_dir, "scheduler.pt"))
            if self._scaler is not None:
                torch.save(self._scaler.state_dict(), os.path.join(output_dir, "scaler.pt"))
            progress = dict(self._progress, global_step=self.global_step)
            with open(os.path.join(output_dir, "trainer_state.json"), "w") as f:
                json.dump(progress, f, indent=2)
        rng = {"python": random.getstate(), "numpy": np.random.get_state(), "cpu": torch.random.get_rng_state(),
               "cuda": torch.cuda.get_rng_state(m._engine.dev), "dropout": m.dropout_rng_state(),
               "cpu_epoch_start": self._epoch_rng}
        torch.save(rng, os.path.join(output_dir, "rng_state_%d.pth" % rank))

    def load_checkpoint(self, checkpoint_dir, restore_dropout=True):
        """Restores what save_checkpoint wrote, on every rank (each rank its own RNG file): the weights, the optimizer,
        the scheduler and the GradScaler, the random states and the optimizer-step count.  Returns the trainer state
        (trainer_state.json).  restore_dropout=False leaves the model's dropout stream where it is."""
        m, rank = _unwrap(self.model), self._rank()
        f = lambda name: os.path.join(checkpoint_dir, name)
        self._loaded_rng = None
        sd = torch.load(f("pytorch_model.bin"), map_location="cpu")
        if isinstance(self.model, DistributedDataParallel):
            self.model.load_state_dict({"module." + k: v for k, v in sd.items()})
        else:
            m.load_state_dict(sd)
        self.optimizer.load_state_dict(torch.load(f("optimizer.pt"), map_location="cpu"))
        if self.lr_scheduler is not None and os.path.exists(f("scheduler.pt")):
            self.lr_scheduler.load_state_dict(torch.load(f("scheduler.pt"), weights_only=False))
        if os.path.exists(f("scaler.pt")):
            if self._scaler is None:
                self._scaler = torch.amp.GradScaler("cuda")
            self._scaler.load_state_dict(torch.load(f("scaler.pt")))
        if os.path.exists(f("rng_state_%d.pth" % rank)):
            rng = torch.load(f("rng_state_%d.pth" % rank), weights_only=False)
            self._restore_host_rng(rng)
            self._loaded_rng = rng
            if restore_dropout:
                m.set_dropout_rng_state(rng["dropout"])
        with open(f("trainer_state.json")) as fp:
            progress = json.load(fp)
        self.global_step = int(progress["global_step"])
        self._micro = 0
        return progress

    def _restore_host_rng(self, rng):
        random.setstate(rng["python"])
        np.random.set_state(rng["numpy"])
        torch.random.set_rng_state(rng["cpu"])
        torch.cuda.set_rng_state(rng["cuda"], _unwrap(self.model)._engine.dev)

    def _maybe_save(self):
        """train(): checkpoint-{optimizer step} under args.output_dir every args.save_steps optimizer steps, keeping
        the newest args.save_total_limit"""
        every = getattr(self.args, "save_steps", None)
        if not every or self._micro != 0 or self.global_step % int(every) != 0:
            return
        out = getattr(self.args, "output_dir", None)
        if out is None:
            raise ValueError("args.save_steps is set but args.output_dir is None")
        self.save_checkpoint(os.path.join(out, "%s-%d" % (CHECKPOINT_PREFIX, self.global_step)))
        if self._rank() == 0:
            rotate_checkpoints(out, getattr(self.args, "save_total_limit", None))

    def train(self, train_loader, dev_loader=None, train_sampler=None, resume_from_checkpoint=None):
        """resume_from_checkpoint: a checkpoint directory, or True for the newest checkpoint-N under args.output_dir.
        The run continues from it: every state save_checkpoint wrote, and the batches the checkpoint's run consumed in
        its epoch are skipped (the loader is iterated past them, as HF Trainer does).  A shuffling loader gives the
        resumed epoch the order the interrupted one had: its iterator is created from the CPU RNG state that epoch's was,
        and every RNG is set back to the checkpoint's once the consumed batches are skipped."""
        gloabl_step = 1
        best_acc = 0.
        if self.args.local_rank == 0:
            start = time.time()
        if self.lr_scheduler is None and getattr(self.args, "lr_scheduler_type", None) is not None:
            self.create_scheduler(self.num_training_steps(train_loader))
        first_epoch, skip, resume_rng = 1, 0, None
        if resume_from_checkpoint:
            path = resume_from_checkpoint
            if path is True:
                path = latest_checkpoint(getattr(self.args, "output_dir", None))
                if path is None:
                    raise ValueError("resume_from_checkpoint=True: no %s-N directory under args.output_dir (%r)"
                                     % (CHECKPOINT_PREFIX, getattr(self.args, "output_dir", None)))
            progress = self.load_checkpoint(path)
            gloabl_step, best_acc = int(progress["batches"]) + 1, float(progress["best_acc"])
            first_epoch, skip = int(progress["epoch"]), int(progress["batches_in_epoch"])
            resume_rng = self._loaded_rng
        for epoch in range(first_epoch, self.args.epochs + 1):
            if train_sampler is not None:
                train_sampler.set_epoch(epoch)
            if resume_rng is not None and resume_rng.get("cpu_epoch_start") is not None:
                # a DataLoader draws its shuffling seed from the CPU RNG when its iterator starts: the resumed epoch's
                # order is the interrupted epoch's only from the state that epoch started with
                torch.random.set_rng_state(resume_rng["cpu_epoch_start"])
            self._epoch_rng = torch.random.get_rng_state()
            for step, batch_data in enumerate(train_loader):
                if skip:
                    skip -= 1
                    continue
                if resume_rng is not None:
                    self._restore_host_rng(resume_rng)     # past the consumed batches: the checkpoint's RNG states
                    resume_rng = None
                loss = self.train_step(batch_data)
                if self.args.local_rank == 0 and gloabl_step % max(1, getattr(self.args, "log_every", 1)) == 0:
                    print("【train】 epoch：{}/{} step：{}/{} loss：{:.6f}".format(
                        epoch, self.args.epochs, gloabl_step, self.args.total_step, float(loss)
                    ))
                gloabl_step += 1
                if self.args.dev:
                    if gloabl_step % self.args.eval_step == 0:
                        loss, accuracy = self.dev(dev_loader)
                        improved = accuracy > best_acc   # identical on every rank (gathered outputs)
                        if self.args.local_rank == 0:
                            print("【dev】 loss：{:.6f} accuracy：{:.4f}".format(float(loss), accuracy))
                        if improved:
                            best_acc = accuracy
                            if self.args.local_rank == 0:
                                print("【best accuracy】 {:.4f}".format(best_acc))
                                # rank 0 alone, as in the reference [:190-192]: under DDP state_dict() pulls the fp32
                                # slices other ranks own out of their HBM one-sidedly (ddp.py::_gather_master)
                                torch.save(self.model.state_dict(), self.args.ckpt_path)
                self._progress = {"batches": gloabl_step - 1, "epoch": epoch, "batches_in_epoch": step + 1,
                                  "best_acc": float(best_acc)}
                self._maybe_save()
            if resume_rng is not None:       # the checkpoint's run had consumed the whole epoch
                self._restore_host_rng(resume_rng)
                resume_rng = None
            skip = 0
            stepped = self._micro != 0
            self.close_window()
            if stepped:
                self._maybe_save()
        if self.args.local_rank == 0:
            end = time.time()
            print("耗时：{}分钟".format((end - start) / 60))
        if not self.args.dev:
            if self.args.local_rank == 0:
                torch.save(self.model.state_dict(), self.args.ckpt_path)

    def dev(self, dev_loader):
        """(summed rank-mean loss, metric) over the gathered rows.  The metric, higher is better: accuracy
        (single-label; a token model's over the tokens whose label is not the ignore index, a multiple-choice model's
        over the examples whose label is not), subset accuracy -- every column of (logits > 0) equal to (labels >= 0.5) -- (multi-label), or
        the Pearson correlation of predictions and labels (regression)."""
        self.model.eval()
        if _is_mlm(self.model):
            return self._dev_mlm(dev_loader)
        if _is_qa(self.model):
            loss_total, spans = self._qa_spans(dev_loader)
            return loss_total, qa_scores(spans)[0]
        correct_total = 0
        num_total = 0
        loss_total = 0.
        reg_preds, reg_trues = [], []
        problem_type = None
        with torch.no_grad():
            for step, batch_data in enumerate(dev_loader):
                logits, label, model_loss = self._eval_forward(batch_data)
                problem_type = self.problem_type(label)
                loss = self.compute_loss(logits, label, model_loss)
                loss = self.loss_reduce(loss)
                loss_total += loss
                logits, label = self.output_reduce(logits, label)
                logits = logits.detach().cpu().numpy()
                if problem_type in (TOKEN_PROBLEM_TYPE, MC_PROBLEM_TYPE):
                    label = label.reshape(-1).detach().cpu().numpy()
                    keep = label != self._ignore_index()
                    preds = np.argmax(logits.reshape(label.shape[0], -1), axis=1)
                    num_total += int(keep.sum())
                    correct_total += int((preds[keep] == label[keep]).sum())
                    continue
                if problem_type == "regression":
                    reg_preds.append(logits.reshape(-1))
                    reg_trues.append(label.reshape(-1).detach().cpu().numpy())
                    continue
                if problem_type == "multi_label_classification":
                    label = label.detach().cpu().numpy()
                    num_total += len(label)
                    correct_total += ((logits > 0) == (label >= 0.5)).all(axis=1).sum()
                    continue
                label = label.view(-1).detach().cpu().numpy()
                num_total += len(label)
                preds = np.argmax(logits, axis=1).flatten()
                correct_num = (preds == label).sum()
                correct_total += correct_num
        if problem_type == "regression":
            return loss_total, float(np.corrcoef(np.concatenate(reg_preds), np.concatenate(reg_trues))[0, 1])
        return loss_total, correct_total / num_total

    def _dev_mlm(self, dev_loader):
        """dev() of a masked-LM model: (summed rank-mean loss, masked-token accuracy), both from the labelled rows on
        the device (BertForMaskedLM.masked_lm_eval: no [batch, seq, V] logits are built or copied)"""
        check_mlm_criterion(self.criterion, device_loss=True)
        m = _unwrap(self.model)
        ignore = self._ignore_index()
        loss_total, correct, total = 0., None, None
        for batch_data in dev_loader:
            if getattr(self.args, "fused", True) and not batch_data["input_ids"].is_cuda:
                B, S = batch_data["input_ids"].shape
                key = (id(m), B, S, MLM_PROBLEM_TYPE, criterion_key(self.criterion))
                if key not in self._fused_eval:
                    self._fused_eval[key] = FusedEvalStep(self.model, B, S, criterion=self.criterion)
                pred, lab, loss = self._fused_eval[key](batch_data)
            else:
                d = self._to_device(batch_data)
                loss, pred, lab = m.masked_lm_eval(d["input_ids"], d["token_type_ids"], d["attention_mask"],
                                                   d["label"], ignore_index=ignore)
            loss_total += self.loss_reduce(loss)
            c = torch.stack([(pred == lab).sum(), torch.tensor(lab.numel(), device=lab.device)]).double()
            if isinstance(self.model, DistributedDataParallel):
                c = self.model.all_gather_rows(c.view(1, 2)).sum(0)
            correct = c[0] if correct is None else correct + c[0]
            total = c[1] if total is None else total + c[1]
        return loss_total, float(correct / total)

    def _qa_spans(self, loader):
        """(summed rank-mean loss, int64 [N, 4] rows (pred start, pred end, gold start, gold end)) of a
        question-answering model over the gathered sequences whose gold span is not ignored.  Gold is HF's
        clamp(0, S); the prediction is best_spans over the sequence's valid tokens."""
        max_len = int(getattr(self.args, "max_answer_length", 30))
        loss_total, rows = 0., []
        with torch.no_grad():
            for batch_data in loader:
                logits, pos, loss = self._eval_forward(batch_data)
                loss_total += self.loss_reduce(loss)
                S = logits.shape[1]
                mask = batch_data["attention_mask"].to(logits.device)
                pred = best_spans(logits[..., 0], logits[..., 1], mask, max_len)
                gold = pos.to(logits.device).t().clamp(0, S)
                pred, gold = self.output_reduce(pred.contiguous(), gold.contiguous())
                keep = (gold != S).all(1)
                rows.append(torch.cat([pred, gold], 1)[keep].cpu())
        return loss_total, torch.cat(rows) if rows else torch.zeros(0, 4, dtype=torch.int64)

    def test(self, model, test_loader, labels):
        """sklearn's classification_report over the gathered rows: of the argmax class (single-label; a token model's
        over the tokens whose label is not the ignore index, a multiple-choice model's argmax choice over the examples
        whose label is not) or of the
        indicator arrays (logits > 0) against (labels >= 0.5) (multi-label).  Regression raises ValueError."""
        if _is_mlm(model):
            raise ValueError("test() prints a classification report, which is not useful over a vocabulary: use dev() "
                             "for the masked-token accuracy")
        if _is_qa(model):
            # a question-answering model: exact match and position-level F1 of the predicted spans (`labels` unused)
            self.model = model
            self.model.eval()
            _loss, spans = self._qa_spans(test_loader)
            em, f1 = qa_scores(spans)
            print("【test】 exact match：{:.4f} f1：{:.4f}".format(em, f1))
            return em, f1
        self.model = model
        self.model.eval()
        preds = []
        trues = []
        with torch.no_grad():
            for step, batch_data in enumerate(test_loader):
                logits, label = self.eval_step(batch_data)
                problem_type = self.problem_type(label)
                if problem_type == "regression":
                    raise ValueError("test() prints a classification report, which does not apply to regression: "
                                     "use dev() for the Pearson correlation")
                logits, label = self.output_reduce(logits, label)
                logits = logits.detach().cpu().numpy()
                if problem_type in (TOKEN_PROBLEM_TYPE, MC_PROBLEM_TYPE):
                    label = label.reshape(-1).detach().cpu().numpy()
                    keep = label != self._ignore_index()
                    trues.extend(label[keep].tolist())
                    preds.extend(np.argmax(logits.reshape(label.shape[0], -1), axis=1)[keep].tolist())
                    continue
                if problem_type == "multi_label_classification":
                    trues.append(label.detach().cpu().numpy() >= 0.5)
                    preds.append(logits > 0)
                    continue
                label = label.view(-1).detach().cpu().numpy().tolist()
                pred = np.argmax(logits, axis=1).flatten().tolist()
                trues.extend(label)
                preds.extend(pred)
        if preds and isinstance(preds[0], np.ndarray):
            trues, preds = np.concatenate(trues).astype(int), np.concatenate(preds).astype(int)
        from sklearn.metrics import classification_report
        report = classification_report(trues, preds, target_names=labels)
        return report
