"""Drop-in ``BertForSequenceClassification`` whose forward/backward run on the sm_90a kernels of libb2ddpbert.so.

Mirrors the surface `multi-gpu-distributed-cls.py` uses (reference lines in brackets):
  * ``BertConfig(..., num_labels=6)`` / ``BertForSequenceClassification.from_pretrained(path, config=config)`` [:336-338]
  * ``model.cuda()`` [:340], ``model.train()/eval()`` [:166,:200]
  * ``model(input_ids=, token_type_ids=, attention_mask=, labels=)`` -> output with ``[0]`` = loss, ``[1]`` = logits
    [:132-136] and ``.logits`` (`predict.py:133`)
  * ``named_parameters()`` yielding the 201 HF parameter names (the no-decay filter at [:101-107] matches on them)
  * ``state_dict()/load_state_dict()`` in HF naming, fp32 (`test.py:96-101`, [:192,:362])
The arithmetic follows HF ``BertForSequenceClassification`` (SP/transformers/models/bert/modeling_bert.py:53-468,
1077-1154, eager attention) in bf16 with fp32 accumulation/statistics; fp32 master weights stay the parameters
the user sees.  There is no PyTorch fallback: without the CUDA library every call raises.
"""
import contextlib
import ctypes
import os
import weakref
from collections import OrderedDict

import torch
import torch.nn as nn

from . import _lib as L
from .losses import PROBLEM_TYPES, Loss, infer_problem_type, problem_type_loss


class BertConfig:
    """The subset of ``transformers.BertConfig`` the path reads; any object with these attributes works."""

    def __init__(self, vocab_size=21128, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                 intermediate_size=3072, hidden_act="gelu", hidden_dropout_prob=0.1,
                 attention_probs_dropout_prob=0.1, max_position_embeddings=512, type_vocab_size=2,
                 initializer_range=0.02, layer_norm_eps=1e-12, pad_token_id=0, num_labels=2,
                 classifier_dropout=None, problem_type=None, **kwargs):
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.num_hidden_layers = num_hidden_layers
        self.num_attention_heads = num_attention_heads
        self.intermediate_size = intermediate_size
        self.hidden_act = hidden_act
        self.hidden_dropout_prob = hidden_dropout_prob
        self.attention_probs_dropout_prob = attention_probs_dropout_prob
        self.max_position_embeddings = max_position_embeddings
        self.type_vocab_size = type_vocab_size
        self.initializer_range = initializer_range
        self.layer_norm_eps = layer_norm_eps
        self.pad_token_id = pad_token_id
        self.num_labels = num_labels
        self.classifier_dropout = classifier_dropout
        if problem_type is not None and problem_type not in PROBLEM_TYPES:
            raise ValueError("problem_type=%r: expected None or one of %s" % (problem_type, PROBLEM_TYPES))
        self.problem_type = problem_type    # HF's: None is inferred from the first labels (losses.py)
        for k, v in kwargs.items():
            setattr(self, k, v)

    @classmethod
    def from_pretrained(cls, path, **kwargs):
        import json
        cfg = {}
        f = os.path.join(path, "config.json")
        if os.path.exists(f):
            with open(f) as fp:
                cfg = json.load(fp)
        cfg.update(kwargs)
        return cls(**cfg)


# presets named in BASELINE.json
def chinese_bert_wwm_ext_config(num_labels=6, **kw):
    return BertConfig(vocab_size=21128, num_labels=num_labels, **kw)


def bert_base_config(num_labels=6, **kw):
    return BertConfig(vocab_size=30522, num_labels=num_labels, **kw)


def bert_large_config(num_labels=6, **kw):
    return BertConfig(vocab_size=30522, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                      intermediate_size=4096, num_labels=num_labels, **kw)


class SequenceClassifierOutput:
    """Tuple-like output: with labels ``(loss, logits)``, without ``(logits,)`` — as HF's ModelOutput indexes."""

    def __init__(self, loss=None, logits=None):
        self.loss = loss
        self.logits = logits

    def to_tuple(self):
        return tuple(v for v in (self.loss, self.logits) if v is not None)

    def __getitem__(self, i):
        if isinstance(i, str):
            return getattr(self, i)
        return self.to_tuple()[i]

    def __iter__(self):
        return iter(self.to_tuple())

    def __len__(self):
        return len(self.to_tuple())


class QuestionAnsweringModelOutput:
    """HF's QuestionAnsweringModelOutput, tuple-like: ``(loss, start_logits, end_logits)``, the loss left out when it is
    None."""

    def __init__(self, loss=None, start_logits=None, end_logits=None):
        self.loss = loss
        self.start_logits = start_logits
        self.end_logits = end_logits

    def to_tuple(self):
        return tuple(v for v in (self.loss, self.start_logits, self.end_logits) if v is not None)

    __getitem__ = SequenceClassifierOutput.__getitem__
    __iter__ = SequenceClassifierOutput.__iter__
    __len__ = SequenceClassifierOutput.__len__


class MultipleChoiceModelOutput(SequenceClassifierOutput):
    """HF's MultipleChoiceModelOutput, tuple-like: ``(loss, logits)`` with logits [batch, num_choices], the loss left
    out when it is None."""


def _round8(n):
    return (n + 7) // 8 * 8


def vocab_pad(vocab_size):
    """the masked-LM model's vocabulary rows in the flat space: vocab_size rounded up to 64, the GEMM's N granule"""
    return (vocab_size + 63) // 64 * 64


HEAD_KINDS = ("sequence", "token", "mlm", "question_answering", "multiple_choice")   # BertForSequenceClassification's
    # pooler + classifier, a classifier per token, BertForMaskedLM's cls.predictions, BertForQuestionAnswering's
    # qa_outputs, or BertForMultipleChoice's pooler + one-row classifier
MLM_TIED = {"cls.predictions.decoder.weight": "bert.embeddings.word_embeddings.weight",
            "cls.predictions.decoder.bias": "cls.predictions.bias"}    # HF's tied state-dict keys of the MLM head
TOKEN_HEAD_MAX_LABELS = 64             # b2_token_head_fwd's bound


class _Holder(nn.Module):
    """Name-only container so that ``named_parameters()`` reproduces the HF module paths."""


class _Layout:
    """Flat parameter space: HF tensors in forward order, each padded to 8 elements, Q/K/V stacked contiguously.
    Buckets (DDP exchange / AdamW launch units) = embeddings | encoder layer 0..L-2 | last layer + head.  The head
    (pooler + classifier, 0.6 M parameters) rides with the last encoder layer -- they are adjacent in the flat space and
    final within microseconds of each other at the start of backward -- instead of paying a barrier, an exchange and
    a kernel launch of its own.  head "token" (BertForTokenClassification): the tail is the classifier alone.  head
    "mlm" (BertForMaskedLM): the tail is cls.predictions (its decoder is the word-embedding table), and the word table
    and cls.predictions.bias reserve vocab_pad(V) rows / entries, so the vocabulary projection is one GEMM with a
    multiple of 64 columns; the extra rows stay zero and lie outside every parameter view.  head "question_answering"
    (BertForQuestionAnswering): the tail is qa_outputs [2, H] / [2] alone, like the token head's classifier.  head
    "multiple_choice" (BertForMultipleChoice): the sequence layout with a one-row classifier [1, H] / [1]."""

    def __init__(self, cfg, head="sequence"):
        if head not in HEAD_KINDS:
            raise ValueError("head=%r: expected one of %s" % (head, HEAD_KINDS))
        self.head = head
        H, I, L_ = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
        self.entries = OrderedDict()  # hf name -> (offset, shape)
        self.buckets = []             # (begin, end, label)
        off = 0

        def add(name, shape, reserve=None):
            nonlocal off
            n = 1
            for s in shape:
                n *= s
            self.entries[name] = (off, tuple(shape))
            off += _round8(n if reserve is None else reserve)

        mlm = head == "mlm"
        self.vocab_pad = vocab_pad(cfg.vocab_size) if mlm else cfg.vocab_size
        b0 = off
        add("bert.embeddings.word_embeddings.weight", (cfg.vocab_size, H), self.vocab_pad * H if mlm else None)
        add("bert.embeddings.position_embeddings.weight", (cfg.max_position_embeddings, H))
        add("bert.embeddings.token_type_embeddings.weight", (cfg.type_vocab_size, H))
        add("bert.embeddings.LayerNorm.weight", (H,))
        add("bert.embeddings.LayerNorm.bias", (H,))
        self.buckets.append((b0, off, "embeddings"))
        for l in range(L_):
            p = "bert.encoder.layer.%d." % l
            b0 = off
            # stacked [3H, H] weight and [3H] bias: one GEMM for Q, K, V
            add(p + "attention.self.query.weight", (H, H))
            add(p + "attention.self.key.weight", (H, H))
            add(p + "attention.self.value.weight", (H, H))
            add(p + "attention.self.query.bias", (H,))
            add(p + "attention.self.key.bias", (H,))
            add(p + "attention.self.value.bias", (H,))
            add(p + "attention.output.dense.weight", (H, H))
            add(p + "attention.output.dense.bias", (H,))
            add(p + "attention.output.LayerNorm.weight", (H,))
            add(p + "attention.output.LayerNorm.bias", (H,))
            add(p + "intermediate.dense.weight", (I, H))
            add(p + "intermediate.dense.bias", (I,))
            add(p + "output.dense.weight", (H, I))
            add(p + "output.dense.bias", (H,))
            add(p + "output.LayerNorm.weight", (H,))
            add(p + "output.LayerNorm.bias", (H,))
            self.buckets.append((b0, off, "layer%d" % l))
        b0 = off
        if head in ("sequence", "multiple_choice"):
            add("bert.pooler.dense.weight", (H, H))
            add("bert.pooler.dense.bias", (H,))
        if mlm:
            add("cls.predictions.bias", (cfg.vocab_size,), self.vocab_pad)
            add("cls.predictions.transform.dense.weight", (H, H))
            add("cls.predictions.transform.dense.bias", (H,))
            add("cls.predictions.transform.LayerNorm.weight", (H,))
            add("cls.predictions.transform.LayerNorm.bias", (H,))
        elif head == "question_answering":
            add("qa_outputs.weight", (cfg.num_labels, H))
            add("qa_outputs.bias", (cfg.num_labels,))
        else:
            C = 1 if head == "multiple_choice" else cfg.num_labels     # HF's multiple-choice classifier ignores it
            add("classifier.weight", (C, H))
            add("classifier.bias", (C,))
        if L_ > 0:
            lb, _le, lbl = self.buckets[-1]
            self.buckets[-1] = (lb, off, lbl + "+head")
        else:
            self.buckets.append((b0, off, "head"))
        self.head_in_last_layer = L_ > 0
        self.total = off

    def off(self, name):
        return self.entries[name][0]


# HF named_parameters() order (201 tensors for 12 layers, as for the multiple-choice head, 199 without the pooler, 202 for
# the MLM head, 199 for the QA head); differs from the flat order only inside attention.self
def _hf_order(cfg, head="sequence"):
    names = ["bert.embeddings.word_embeddings.weight", "bert.embeddings.position_embeddings.weight",
             "bert.embeddings.token_type_embeddings.weight", "bert.embeddings.LayerNorm.weight",
             "bert.embeddings.LayerNorm.bias"]
    for l in range(cfg.num_hidden_layers):
        p = "bert.encoder.layer.%d." % l
        for m in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense",
                  "attention.output.LayerNorm", "intermediate.dense", "output.dense", "output.LayerNorm"):
            names += [p + m + ".weight", p + m + ".bias"]
    if head in ("sequence", "multiple_choice"):
        names += ["bert.pooler.dense.weight", "bert.pooler.dense.bias"]
    if head == "mlm":
        return names + ["cls.predictions.bias", "cls.predictions.transform.dense.weight",
                        "cls.predictions.transform.dense.bias", "cls.predictions.transform.LayerNorm.weight",
                        "cls.predictions.transform.LayerNorm.bias"]
    if head == "question_answering":
        return names + ["qa_outputs.weight", "qa_outputs.bias"]
    names += ["classifier.weight", "classifier.bias"]
    return names


class _StepFn(torch.autograd.Function):
    """logits (and HF's in-model loss) with a backward that runs the CUDA backward pass."""

    @staticmethod
    def forward(ctx, anchor, model, input_ids, token_type_ids, attention_mask, labels, packed=None, fwd_kw=None):
        eng = model._engine
        logits, loss = eng.forward(input_ids, token_type_ids, attention_mask, labels, training=model.training,
                                   need_backward=True, packed=packed, **(fwd_kw or {}))
        ctx.model = model
        ctx.has_loss = loss is not None
        ctx.set_materialize_grads(False)
        if loss is None:
            return logits.clone(), torch.zeros((), device=logits.device)
        return logits.clone(), loss.clone()

    @staticmethod
    def backward(ctx, d_logits, d_loss):
        model = ctx.model
        eng = model._engine
        if d_logits is None and (d_loss is None or not ctx.has_loss):
            raise RuntimeError("backward reached the model without any gradient")
        accumulate = model._no_sync
        if model._optimizer is not None:
            # gradients are OVERWRITTEN by every backward outside no_sync() (bf16 bucket space, zero_grad is a no-op):
            # a second one before optimizer.step() would silently drop the first one's gradients where torch would
            # accumulate them
            if model._grads_live:
                if accumulate:
                    raise RuntimeError("backward() inside no_sync() after a backward outside it without "
                                       "optimizer.step() in between: run the window's earlier passes inside no_sync()")
                raise RuntimeError("backward() called twice without optimizer.step() in between: gradient "
                                   "accumulation is not supported on this path (gradients are overwritten, not summed)")
            if not accumulate:
                model._grads_live = True
        eng.start_pass(accumulate)
        eng.backward(d_logits, d_loss if ctx.has_loss else None)
        eng.end_pass()
        # Gradients live in the engine's bf16 bucket space, not in `.grad`.  The anchor (classifier.bias, or
        # cls.predictions.bias) gets its true gradient as an fp32 probe: it is the column sum of d_logits, so an
        # inf/nan anywhere upstream
        # of the model shows up in it -- which is what torch.cuda.amp.GradScaler's inf check needs to see.  Autograd
        # sums the probes of an accumulation window's backwards; the final one reads the folded window sum, so the
        # probe is non-finite exactly when some pass of the window was.
        off, shape = ctx.model._layout.entries[model._anchor]
        n = 1
        for d in shape:
            n *= d
        probe = eng.grads[off:off + n].float().view(shape)
        if model._ddp is not None:
            probe = model._ddp.consensus_probe(probe)
        return probe, None, None, None, None, None, None, None


class _BertClassifier(nn.Module):
    """What the classification models share: the HF parameter skeleton over one flat fp32 space, construction,
    device movement, state dicts, the dropout stream and no_sync().  The subclass names its head kind (_Layout)."""
    _head = None
    _anchor = "classifier.bias"   # the parameter _StepFn's autograd output hangs on (its gradient is the probe)
    _config_extra = {}       # written into save_pretrained's config.json over the config's attributes

    def __init__(self, config):
        super().__init__()
        self.config = config
        cfg = config
        assert cfg.hidden_size % cfg.num_attention_heads == 0
        if cfg.hidden_size // cfg.num_attention_heads != 64:
            raise ValueError("only head_dim 64 is on the path (BERT-base / BERT-large)")
        if getattr(cfg, "hidden_act", "gelu") != "gelu":
            raise ValueError("only the erf GELU of the reference config is on the path")
        self.num_labels = cfg.num_labels
        self._layout = _Layout(cfg, self._head)
        lay = self._layout
        # fp32 master weights: ONE flat tensor, every nn.Parameter is a view into it
        self._flat = torch.zeros(lay.total, dtype=torch.float32)
        self._build_skeleton()
        self._init_weights()
        self._engine = None
        self._optimizer = None       # the optimizer whose step schedule the backward drives (the last one built)
        self._optimizers = weakref.WeakSet()   # every live optimizer of the model (their state moves with a wrapper)
        self._ddp = None
        self._grads_live = False     # an eager backward has produced gradients no optimizer.step() has consumed yet
        self._no_sync = False        # inside no_sync(): backwards accumulate
        self._pt_loss = None         # (problem_type, losses.Loss) of the in-model loss

    @contextlib.contextmanager
    def no_sync(self):
        """Gradient accumulation, as ``DistributedDataParallel.no_sync()`` (SP/torch/nn/parallel/distributed.py): a
        backward inside the context adds its gradients into a local fp32 accumulator -- no exchange, no update, no
        barrier.  The first backward after it folds the accumulator into its own gradients, and ``optimizer.step()``
        applies the sum as usual; a step with no such backward applies the accumulator alone (under DDP with world > 1
        it also exchanges, where stock torch DDP would leave the ranks diverged).  Scale the loss by 1/k yourself for
        the mean over k micro-batches.  Also available on the bare model, so one loop runs on 1 and N GPUs."""
        prev = self._no_sync
        self._no_sync = True
        try:
            yield
        finally:
            self._no_sync = prev

    # ---- module skeleton reproducing HF parameter paths -------------------------------------------------------
    def _build_skeleton(self):
        cfg = self.config
        self._params_by_name = OrderedDict()
        root = self

        def holder(parent, path):
            cur = parent
            for part in path:
                if part.isdigit():
                    cur = cur[int(part)]
                    continue
                if not hasattr(cur, part):
                    setattr(cur, part, nn.ModuleList() if part == "layer" else _Holder())
                cur = getattr(cur, part)
            return cur

        # registration order fixes named_parameters() order: embeddings, encoder, pooler (sequence head), classifier
        # (as HF)
        holder(root, ["bert", "embeddings"])
        enc = holder(root, ["bert", "encoder"])
        enc.layer = nn.ModuleList([_Holder() for _ in range(cfg.num_hidden_layers)])
        for name in _hf_order(cfg, self._head):
            off, shape = self._layout.entries[name]
            n = 1
            for s in shape:
                n *= s
            parts = name.split(".")
            mod = holder(root, parts[:-1])
            p = nn.Parameter(self._flat[off:off + n].view(shape))
            p._b2_owner = self
            p._b2_name = name
            mod.register_parameter(parts[-1], p)
            self._params_by_name[name] = p
        # transformers 4.28.1 (the reference's pin) keeps position_ids as a persistent buffer in checkpoints
        emb = holder(root, ["bert", "embeddings"])
        emb.register_buffer("position_ids", torch.arange(cfg.max_position_embeddings).unsqueeze(0), persistent=True)

    def _init_weights(self):
        """HF ``_init_weights``: N(0, initializer_range) for Linear/Embedding weights, zero pad row / biases,
        LayerNorm (1, 0)  (SP/transformers/models/bert/modeling_bert.py `_init_weights`)."""
        cfg = self.config
        with torch.no_grad():
            for name, p in self._params_by_name.items():
                if "LayerNorm.weight" in name:
                    p.fill_(1.0)
                elif name.endswith(".bias") or "LayerNorm.bias" in name:
                    p.zero_()
                else:
                    p.normal_(mean=0.0, std=cfg.initializer_range)
            pad = getattr(cfg, "pad_token_id", None)
            if pad is not None:
                self._params_by_name["bert.embeddings.word_embeddings.weight"][pad].zero_()

    # ---- construction helpers ----------------------------------------------------------------------------------
    @classmethod
    def from_config(cls, config, seed=None):
        if seed is not None:
            torch.manual_seed(seed)
        return cls(config)

    @classmethod
    def from_pretrained(cls, model_path, config=None, **kwargs):
        """Loads HF-format weights (``pytorch_model.bin`` / ``model.safetensors``) when present; like HF, tensors
        absent from the checkpoint (the fresh classifier) keep their random init."""
        if config is None:
            config = BertConfig.from_pretrained(model_path, **kwargs)
        model = cls(config)
        sd = None
        binf = os.path.join(model_path, "pytorch_model.bin")
        sft = os.path.join(model_path, "model.safetensors")
        if os.path.exists(binf):
            sd = torch.load(binf, map_location="cpu")
        elif os.path.exists(sft):
            from safetensors.torch import load_file
            sd = load_file(sft)
        if sd is None:
            raise FileNotFoundError("no pytorch_model.bin / model.safetensors under %s" % model_path)
        model.load_state_dict(sd, strict=False)
        return model

    # ---- device movement keeps the flat storage ---------------------------------------------------------------
    def _apply(self, fn, recurse=True):
        new_flat = fn(self._flat)
        if new_flat.dtype != torch.float32:
            raise TypeError("master weights stay fp32 (the kernels compute in bf16 from a shadow copy)")
        self._flat = new_flat.contiguous()
        for name, p in self._params_by_name.items():
            off, shape = self._layout.entries[name]
            n = p.numel()
            p.data = self._flat[off:off + n].view(shape)
        for mod in self.modules():
            for key, buf in list(mod._buffers.items()):
                if buf is not None:
                    mod._buffers[key] = fn(buf)
        if self._flat.is_cuda:
            self._engine = _Engine(self)
        else:
            self._engine = None
        return self

    def _rebind_flat(self, new_flat):
        """moves the fp32 masters into `new_flat` (same size; e.g. the DDP wrapper's peer-visible buffer) and re-points
        every nn.Parameter view at it"""
        if new_flat.dtype != torch.float32 or new_flat.numel() != self._flat.numel():
            raise ValueError("_rebind_flat: need an fp32 buffer of %d elements" % self._flat.numel())
        new_flat.copy_(self._flat)
        self._flat = new_flat
        for name, p in self._params_by_name.items():
            off, shape = self._layout.entries[name]
            p.data = self._flat[off:off + p.numel()].view(shape)

    # ---- state dict -----------------------------------------------------------------------------------------------
    def load_state_dict(self, state_dict, strict=True, assign=False):
        own = self._params_by_name
        missing = [k for k in own if k not in state_dict]
        unexpected = [k for k in state_dict if k not in own and not k.endswith("position_ids")
                      and not k.endswith("embeddings.token_type_ids")]
        if strict and (missing or unexpected):
            raise RuntimeError("Error(s) in loading state_dict: missing %s unexpected %s" % (missing, unexpected))
        with torch.no_grad():
            for k, p in own.items():
                if k in state_dict:
                    src = state_dict[k]
                    if tuple(src.shape) != tuple(p.shape):
                        raise RuntimeError("size mismatch for %s: %s vs %s" % (k, tuple(src.shape), tuple(p.shape)))
                    p.copy_(src.to(dtype=torch.float32))
        if self._engine is not None:
            self._engine.refresh_shadow()
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def state_dict(self, *args, **kwargs):
        if self._ddp is not None:
            self._ddp._gather_master()
        return super().state_dict(*args, **kwargs)

    def save_pretrained(self, save_directory):
        """HF's layout: ``config.json`` (the config's attributes, problem_type included) and ``pytorch_model.bin``
        (HF-keyed fp32 weights), which ``from_pretrained(save_directory)`` reads back exactly.  Under
        DistributedDataParallel it is one-sided, as state_dict() is: call it on one rank."""
        import json
        os.makedirs(save_directory, exist_ok=True)
        cfg = self.config.to_dict() if hasattr(self.config, "to_dict") else dict(vars(self.config))
        cfg.update(self._config_extra)
        with open(os.path.join(save_directory, "config.json"), "w") as f:
            json.dump(cfg, f, indent=2, sort_keys=True)
        sd = OrderedDict((k, v.detach().cpu().clone()) for k, v in self.state_dict().items())
        torch.save(sd, os.path.join(save_directory, "pytorch_model.bin"))

    # ---- dropout stream -------------------------------------------------------------------------------------------
    def dropout_rng_state(self):
        """the dropout streams' position: CPU int64 [seed, step].  Every optimizer step and every accumulating backward
        moves `step` on; each rank has its own."""
        if self._engine is None:
            raise RuntimeError("the dropout state lives on the GPU: call model.cuda() first")
        return self._engine.rng.cpu()

    def set_dropout_rng_state(self, state):
        """writes a dropout_rng_state() back, stream-ordered and in place (captured train steps keep replaying on it)"""
        if self._engine is None:
            raise RuntimeError("the dropout state lives on the GPU: call model.cuda() first")
        t = torch.as_tensor(state).reshape(-1)
        if t.numel() != 2 or t.is_floating_point():
            raise ValueError("a dropout RNG state is an integer [seed, step] (got %s)" % (state,))
        seed, step = (int(x) for x in t.tolist())
        self._engine.seed_dropout(seed, step)

    # ---- test / tooling helpers -----------------------------------------------------------------------------------------
    def grad_dict(self):
        """fp32 copies of what the next optimizer.step() would apply, keyed by HF parameter name: the (bf16) gradients of
        the last backward, or inside an open accumulation window the fp32 accumulator."""
        if self._engine is None:
            raise RuntimeError("no engine (model not on CUDA)")
        out = OrderedDict()
        g = self._engine.accum if self._engine.accum_live else self._engine.grads
        for name, p in self._params_by_name.items():
            off, shape = self._layout.entries[name]
            out[name] = g[off:off + p.numel()].view(shape).to(torch.float32, copy=True)
        return out


class BertForSequenceClassification(_BertClassifier):
    """HF's BertForSequenceClassification: the pooler's tanh(dense) of each sequence's first token, dropout and a
    linear classifier; the loss follows config.problem_type."""
    _head = "sequence"

    # ---- forward ------------------------------------------------------------------------------------------------------
    def forward(self, input_ids=None, token_type_ids=None, attention_mask=None, labels=None, position_ids=None,
                segments=None, cls_index=None, **unused):
        """`position_ids` / `segments` / `cls_index` (all three or none): the batch is PACKED -- the rows of
        `input_ids` are the bins of `packing.pack_batch` (128, 256, 384 or 512 tokens), logits come back one row per
        original sequence."""
        if self._engine is None:
            raise RuntimeError("BertForSequenceClassification (b200) only runs on CUDA: call model.cuda() first; "
                               "there is no CPU path.")
        if input_ids is None:
            raise ValueError("input_ids is required")
        packed = None
        if segments is not None or cls_index is not None:
            if position_ids is None or segments is None or cls_index is None:
                raise ValueError("a packed batch needs position_ids, segments and cls_index together")
            packed = (position_ids, segments, cls_index)
        elif position_ids is not None:
            raise ValueError("position_ids are only supported for packed batches (with segments and cls_index)")
        if torch.is_grad_enabled() and self.training:
            anchor = self._params_by_name["classifier.bias"]
            logits, loss = _StepFn.apply(anchor, self, input_ids, token_type_ids, attention_mask, labels, packed)
            return SequenceClassifierOutput(loss=loss if labels is not None else None, logits=logits)
        logits, loss = self._engine.forward(input_ids, token_type_ids, attention_mask, labels,
                                            training=self.training, need_backward=False, packed=packed)
        return SequenceClassifierOutput(loss=None if loss is None else loss.clone(), logits=logits.clone())

    def _problem_type_loss(self, labels):
        """The loss of `labels = ...` (HF BertForSequenceClassification.forward): config.problem_type's, inferred from
        these labels and stored on the config when it is None"""
        cfg = self.config
        pt = getattr(cfg, "problem_type", None)
        if pt is None:
            pt = infer_problem_type(self.num_labels, labels)
            cfg.problem_type = pt
        if self._pt_loss is None or self._pt_loss[0] != pt:
            self._pt_loss = (pt, problem_type_loss(pt, self.num_labels))
        return self._pt_loss[1]


class BertForTokenClassification(_BertClassifier):
    """HF's BertForTokenClassification: BertModel without the pooler, dropout (config.classifier_dropout, else
    hidden_dropout_prob) and a linear classifier on every token (csrc/token_head.cu), and with labels HF's
    ``CrossEntropyLoss()`` over ``logits.view(-1, C)`` / ``labels.view(-1)`` (-100 ignored; config.problem_type is not
    read).  Padding positions must carry -100, as HF's tagging collators put there.  Logits are fp32 [batch, seq, C],
    or [bins, bin_len, C] for a packed batch."""
    _head = "token"
    _config_extra = {"architectures": ["BertForTokenClassification"]}

    def __init__(self, config):
        if not 1 <= int(config.num_labels) <= TOKEN_HEAD_MAX_LABELS:
            raise ValueError("BertForTokenClassification: num_labels=%d, the token head supports 1 to %d labels"
                             % (int(config.num_labels), TOKEN_HEAD_MAX_LABELS))
        super().__init__(config)
        self._ce = None

    def forward(self, input_ids=None, token_type_ids=None, attention_mask=None, labels=None, position_ids=None,
                segments=None, **unused):
        """`position_ids` / `segments` (both or neither): the rows of `input_ids` are the bins of
        `packing.pack_batch`, and `labels` its packed "labels" (unused bin rows hold -100)."""
        if self._engine is None:
            raise RuntimeError("BertForTokenClassification (b200) only runs on CUDA: call model.cuda() first; "
                               "there is no CPU path.")
        if input_ids is None:
            raise ValueError("input_ids is required")
        packed = None
        if segments is not None or position_ids is not None:
            if position_ids is None or segments is None:
                raise ValueError("a packed batch needs position_ids and segments together")
            packed = (position_ids, segments, None)
        if labels is not None and labels.is_floating_point():
            raise TypeError("token labels are int64 class indices (CrossEntropyLoss), got %s" % labels.dtype)
        if torch.is_grad_enabled() and self.training:
            anchor = self._params_by_name["classifier.bias"]
            logits, loss = _StepFn.apply(anchor, self, input_ids, token_type_ids, attention_mask, labels, packed)
            return SequenceClassifierOutput(loss=loss if labels is not None else None, logits=logits)
        logits, loss = self._engine.forward(input_ids, token_type_ids, attention_mask, labels,
                                            training=self.training, need_backward=False, packed=packed)
        return SequenceClassifierOutput(loss=None if loss is None else loss.clone(), logits=logits.clone())

    def _problem_type_loss(self, labels):
        """HF's in-model loss of the token model: CrossEntropyLoss() whatever config.problem_type says"""
        if self._ce is None:
            self._ce = Loss(L.LOSS_CE, self.num_labels)
        return self._ce


def _check_mlm_labels(labels, input_ids):
    """masked-LM labels: int64 token ids of the input's shape (the compaction kernel reads them as int64)"""
    if labels.dtype != torch.int64 or tuple(labels.shape) != tuple(input_ids.shape):
        raise TypeError("masked-LM labels are int64 token ids of the input's shape %s (-100: ignored), got %s %s"
                        % (list(input_ids.shape), labels.dtype, list(labels.shape)))


class BertForMaskedLM(_BertClassifier):
    """HF's BertForMaskedLM: BertModel without the pooler, then cls.predictions -- transform (dense, erf GELU,
    LayerNorm) and a decoder tied to the word embeddings, ``logits = transform(x) @ word_embeddings.weight^T +
    cls.predictions.bias`` -- and with labels HF's ``CrossEntropyLoss()`` over ``logits.view(-1, V)`` /
    ``labels.view(-1)`` (-100 ignored; config.problem_type is not read).  Logits are fp32 [batch, seq, V] over every
    row (or [bins, bin_len, V] packed).  The loss, and a backward from the loss alone, run the head on the labelled
    rows only (csrc/mlm_head.cu); a backward that reaches the logits takes their dense gradient."""
    _head = "mlm"
    _anchor = "cls.predictions.bias"
    _config_extra = {"architectures": ["BertForMaskedLM"]}

    def forward(self, input_ids=None, token_type_ids=None, attention_mask=None, labels=None, position_ids=None,
                segments=None, **unused):
        """`position_ids` / `segments` (both or neither): the rows of `input_ids` are the bins of
        `packing.pack_batch`, and `labels` its packed "labels" (unused bin rows hold -100)."""
        if self._engine is None:
            raise RuntimeError("BertForMaskedLM (b200) only runs on CUDA: call model.cuda() first; there is no CPU "
                               "path.")
        if input_ids is None:
            raise ValueError("input_ids is required")
        packed = None
        if segments is not None or position_ids is not None:
            if position_ids is None or segments is None:
                raise ValueError("a packed batch needs position_ids and segments together")
            packed = (position_ids, segments, None)
        if labels is not None:
            _check_mlm_labels(labels, input_ids)
        if torch.is_grad_enabled() and self.training:
            anchor = self._params_by_name[self._anchor]
            logits, loss = _StepFn.apply(anchor, self, input_ids, token_type_ids, attention_mask, labels, packed)
            return SequenceClassifierOutput(loss=loss if labels is not None else None, logits=logits)
        logits, loss = self._engine.forward(input_ids, token_type_ids, attention_mask, labels,
                                            training=self.training, need_backward=False, packed=packed)
        return SequenceClassifierOutput(loss=None if loss is None else loss.clone(), logits=logits.clone())

    def masked_lm_eval(self, input_ids, token_type_ids=None, attention_mask=None, labels=None, ignore_index=-100):
        """The dropout-free forward on the labelled rows only: (mean loss, predicted ids, labels) as device tensors,
        the last two over the labelled tokens in token order.  No [batch, seq, V] logits are built."""
        if self._engine is None:
            raise RuntimeError("BertForMaskedLM (b200) only runs on CUDA: call model.cuda() first")
        if labels is None:
            raise ValueError("masked_lm_eval needs labels: it evaluates the labelled tokens")
        _check_mlm_labels(labels, input_ids)
        with torch.no_grad():
            _logits, loss = self._engine.forward(input_ids, token_type_ids, attention_mask, labels, training=False,
                                                 need_backward=False, mlm_full=False, ignore_index=ignore_index)
        gb = self._engine.mlm_last
        n = int(gb["count"].item())
        return loss.clone(), gb["pred"][:n].long(), gb["labels"][:n].long()

    def state_dict(self, *args, **kwargs):
        """HF's keys, with the tied decoder as HF lists it: cls.predictions.decoder.weight (the word-embedding tensor)
        and cls.predictions.decoder.bias (cls.predictions.bias)"""
        sd = super().state_dict(*args, **kwargs)
        prefix = kwargs.get("prefix", args[1] if len(args) > 1 else "")
        for tied, src in MLM_TIED.items():
            if prefix + src in sd:
                sd[prefix + tied] = sd[prefix + src]
        return sd

    def load_state_dict(self, state_dict, strict=True, assign=False):
        """accepts an HF state dict with or without the tied decoder keys (their tensors are the word embeddings and
        cls.predictions.bias, loaded under those names)"""
        sd = OrderedDict((k, v) for k, v in state_dict.items() if k not in MLM_TIED)
        return super().load_state_dict(sd, strict=strict, assign=assign)

    @classmethod
    def from_pretrained(cls, model_path, config=None, **kwargs):
        """as the classifiers' (a BertForPreTraining checkpoint's bert.pooler.* and cls.seq_relationship.* are
        ignored, as HF ignores them); a checkpoint without cls.predictions keeps HF's fresh init of the head"""
        return super().from_pretrained(model_path, config=config, **kwargs)


def _qa_positions(start_positions, end_positions, nseq, device):
    """HF's start / end positions (int64 [nseq], or [nseq, 1], squeezed) as the one int64 [2, nseq] tensor the span
    loss reads: row 0 the start positions, row 1 the end positions, raw (the kernel applies HF's clamp)"""
    out = []
    for t, nm in ((start_positions, "start_positions"), (end_positions, "end_positions")):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.int64:
            raise TypeError("%s must be an int64 tensor (token positions), got %s"
                            % (nm, getattr(t, "dtype", type(t).__name__)))
        if t.device != device:
            raise RuntimeError("%s is on %s, model on %s" % (nm, t.device, device))
        if tuple(t.shape) not in ((nseq,), (nseq, 1)):
            raise ValueError("%s must be [%d] or [%d, 1] (one per sequence), got %s" % (nm, nseq, nseq, list(t.shape)))
        out.append(t.reshape(nseq))
    return torch.stack(out)


class BertForQuestionAnswering(_BertClassifier):
    """HF's BertForQuestionAnswering: BertModel without the pooler and ``qa_outputs``, a Linear(H, 2) on every token
    with no dropout (the token head's kernels with two labels), split into start and end logits.  With
    ``start_positions`` and ``end_positions`` the loss is HF's: both clamped to [0, S] with S ignored, one
    ``CrossEntropyLoss(ignore_index=S)`` over the sequence axis for each, averaged (csrc/qa_head.cu).  Logits are fp32
    [batch, seq] each, or [bins, bin_len] for a packed batch, where each sequence's softmax runs over its own tokens
    (HF's loss on the sequence unpadded)."""
    _head = "question_answering"
    _anchor = "qa_outputs.bias"
    _config_extra = {"architectures": ["BertForQuestionAnswering"]}

    def __init__(self, config):
        if int(config.num_labels) != 2:
            raise ValueError("BertForQuestionAnswering: num_labels=%d, the span head needs exactly 2 (start and end "
                             "logits)" % int(config.num_labels))
        super().__init__(config)

    def forward(self, input_ids=None, token_type_ids=None, attention_mask=None, start_positions=None,
                end_positions=None, position_ids=None, segments=None, cls_index=None, ignored_index=None, **unused):
        """`position_ids` / `segments` / `cls_index` (all three or none): the rows of `input_ids` are the bins of
        `packing.pack_batch`, and the positions count from each sequence's first token.  `ignored_index` (packed
        only): the padded length the positions were given for, HF's ignored index (None: the bin length); a position
        inside [length, ignored_index) traps, and pack_batch rejects it first."""
        if self._engine is None:
            raise RuntimeError("BertForQuestionAnswering (b200) only runs on CUDA: call model.cuda() first; there is "
                               "no CPU path.")
        if input_ids is None:
            raise ValueError("input_ids is required")
        packed, kw = None, {}
        if segments is not None or cls_index is not None or position_ids is not None:
            if position_ids is None or segments is None or cls_index is None:
                raise ValueError("a packed batch needs position_ids, segments and cls_index together")
            packed = (position_ids, segments, cls_index)
            if ignored_index is not None:
                kw["qa_ignored_index"] = int(ignored_index)
        elif ignored_index is not None:
            raise ValueError("ignored_index applies to packed batches only (a padded batch ignores its length S)")
        positions = None
        if start_positions is not None and end_positions is not None:
            nseq = input_ids.shape[0] if packed is None else cls_index.numel()
            positions = _qa_positions(start_positions, end_positions, nseq, self._engine.dev)
        if torch.is_grad_enabled() and self.training:
            anchor = self._params_by_name[self._anchor]
            logits, loss = _StepFn.apply(anchor, self, input_ids, token_type_ids, attention_mask, positions, packed, kw)
            loss = loss if positions is not None else None
        else:
            logits, loss = self._engine.forward(input_ids, token_type_ids, attention_mask, positions,
                                                training=self.training, need_backward=False, packed=packed, **kw)
            loss = None if loss is None else loss.clone()
        start, end = (t.contiguous() for t in logits.unbind(-1))
        return QuestionAnsweringModelOutput(loss=loss, start_logits=start, end_logits=end)


def check_choice_labels(labels, batch):
    """multiple-choice labels: int64 [batch], one choice index per example (-100: ignored)"""
    if not isinstance(labels, torch.Tensor) or labels.dtype != torch.int64:
        raise TypeError("multiple-choice labels are int64 choice indices, got %s"
                        % getattr(labels, "dtype", type(labels).__name__))
    if tuple(labels.shape) != (batch,):
        raise ValueError("multiple-choice labels must be [%d] (one choice index per example), got %s"
                         % (batch, list(labels.shape)))


class BertForMultipleChoice(_BertClassifier):
    """HF's BertForMultipleChoice: the B·N choice sequences of a [B, N, S] batch run flattened through the sequence
    model's encoder, pooler, dropout (config.classifier_dropout, else hidden_dropout_prob) and a Linear(H, 1) -- the
    sequence head's kernels with one label -- and the [B·N, 1] logits are read as [B, N].  With labels (int64 [B]) the
    loss is HF's ``CrossEntropyLoss()`` over the choices (-100 ignored).  The classifier has one row whatever
    config.num_labels says, and config.problem_type is neither read nor set, as in HF.  from_pretrained loads the
    encoder and pooler and ignores a pre-training checkpoint's cls.*; a classifier of another shape (a sequence
    classifier's [num_labels, H]) raises a size mismatch, as transformers does without ignore_mismatched_sizes."""
    _head = "multiple_choice"
    _config_extra = {"architectures": ["BertForMultipleChoice"]}

    def __init__(self, config):
        super().__init__(config)
        self._ce = {}            # choices -> the in-model CrossEntropyLoss() over them

    def forward(self, input_ids=None, token_type_ids=None, attention_mask=None, labels=None, position_ids=None,
                segments=None, cls_index=None, **unused):
        """Padded: input_ids / token_type_ids / attention_mask int64 [B, N, S].  `position_ids` / `segments` /
        `cls_index` (all three or none): the rows of `input_ids` are the bins of `packing.pack_batch` over the B·N
        choice sequences, and cls_index [B, N] gives the number of choices.  Returns fp32 logits [B, N]."""
        if input_ids is None:
            raise ValueError("input_ids is required")
        packed = None
        if segments is not None or cls_index is not None or position_ids is not None:
            if position_ids is None or segments is None or cls_index is None:
                raise ValueError("a packed batch needs position_ids, segments and cls_index together")
            if cls_index.dim() != 2:
                raise ValueError("cls_index of a packed multiple-choice batch must be [batch, num_choices], got %s"
                                 % list(cls_index.shape))
            B, N = cls_index.shape
            packed = (position_ids, segments, cls_index)
        else:
            if input_ids.dim() != 3:
                raise ValueError("input_ids must be [batch, num_choices, seq], got %s" % list(input_ids.shape))
            B, N, S = input_ids.shape
            for t, nm in ((token_type_ids, "token_type_ids"), (attention_mask, "attention_mask")):
                if t is not None and tuple(t.shape) != (B, N, S):
                    raise ValueError("%s must have input_ids' shape %s, got %s" % (nm, [B, N, S], list(t.shape)))
            flat = lambda t: None if t is None else t.reshape(B * N, S)
            input_ids, token_type_ids, attention_mask = flat(input_ids), flat(token_type_ids), flat(attention_mask)
        if labels is not None:
            check_choice_labels(labels, B)
        if self._engine is None:
            raise RuntimeError("BertForMultipleChoice (b200) only runs on CUDA: call model.cuda() first; there is no "
                               "CPU path.")
        kw = {"loss_fn": self.choice_loss(N)}
        if torch.is_grad_enabled() and self.training:
            anchor = self._params_by_name[self._anchor]
            logits, loss = _StepFn.apply(anchor, self, input_ids, token_type_ids, attention_mask, labels, packed, kw)
            loss = loss if labels is not None else None
        else:
            logits, loss = self._engine.forward(input_ids, token_type_ids, attention_mask, labels,
                                                training=self.training, need_backward=False, packed=packed, **kw)
            logits, loss = logits.clone(), None if loss is None else loss.clone()
        return MultipleChoiceModelOutput(loss=loss, logits=logits.view(B, N))

    def choice_loss(self, num_choices):
        """HF's in-model loss: CrossEntropyLoss() over the num_choices logits of each example"""
        if num_choices not in self._ce:
            self._ce[num_choices] = Loss(L.LOSS_CE, num_choices)
        return self._ce[num_choices]


class _LocalTransport:
    """The facts the optimizer's step schedule (optim._FusedOptimizer: bucket_ready, step, the clip phases) needs about
    where gradients and weights live, on one GPU.  DistributedDataParallel answers the same questions for a peer group
    (world > 1).  A transport holds no policy: it never looks at accumulation, clipping or which buckets are done."""
    world, rank = 1, 0
    background = True            # an update launched under the backward takes the slim kernel form (and its prepare)
    tail_on_side = False         # step() joins the side stream first; the step counter advances on the main stream
    # the backward joins the weight-gradient stream itself at its end.  (It could leave that to the side stream, as
    # the peer path does; that reorders the captured step and is a change to measure on its own.)
    side_carries_wgrad = False

    def __init__(self, eng):
        self.eng = eng
        self.side = torch.cuda.Stream(device=eng.dev)      # runs the per-bucket work of an armed step

    @property
    def overlap(self):
        """may bucket_ready run during backward?  Not under a world-1 DistributedDataParallel wrapper: it keeps the
        whole-range accumulate and update after backward.  (A missed optimisation, kept as it is: lifting it changes
        that configuration's launch order and speed.)"""
        return self.eng.model._ddp is None

    def slice(self, idx):
        """the elements of bucket `idx` this rank reduces and updates"""
        b, e, _label = self.eng.lay.buckets[idx]
        return b, e

    def grad_sources(self, idx, stream):
        """every rank's bf16 gradient buffer, as the reduce kernels index them"""
        return [self.eng.grads.data_ptr()]

    def barrier(self, slot, stream):
        pass

    def norm_exchange(self):
        """(scratch, flags, slot, epoch) of the scalar exchange in the norm finalize"""
        return None, None, 0, None

    def update(self, opt, buckets, stream, background=False):
        eng = self.eng
        # the buckets tile the flat space: all of them are one launch
        whole = len(buckets) == len(eng.lay.buckets)
        for b, e in [(0, eng.lay.total)] if whole else [self.slice(idx) for idx in buckets]:
            opt.update_range(b, e, 1, 0, [eng.grads.data_ptr()], [eng.shadow.data_ptr()], stream,
                             background=background)

    def stepped(self):
        pass


class _Engine:
    """Owns the device-side state of one model replica and drives the kernels (forward, backward)."""

    def __init__(self, model):
        L.load()
        self.model = model
        self.cfg = cfg = model.config
        self.lay = model._layout
        self.dev = model._flat.device
        self.H, self.I = cfg.hidden_size, cfg.intermediate_size
        self.heads, self.nl, self.C = cfg.num_attention_heads, cfg.num_hidden_layers, cfg.num_labels
        # the multiple-choice head is the sequence head with one label over the B·N choice sequences; its loss reads
        # the [B·N, 1] logits as [B, N]
        self.mc = self.lay.head == "multiple_choice"
        if self.mc:
            self.C = 1
        self.p_hidden = float(cfg.hidden_dropout_prob)
        self.p_attn = float(cfg.attention_probs_dropout_prob)
        cd = getattr(cfg, "classifier_dropout", None)
        self.p_cls = float(cd if cd is not None else cfg.hidden_dropout_prob)
        # a classifier on every token row instead of pooler + classifier; the QA head's qa_outputs is one with two labels
        # and no dropout, followed by the span loss (csrc/qa_head.cu)
        self.qa = self.lay.head == "question_answering"
        self.token_head = self.lay.head == "token" or self.qa
        self.cls_w, self.cls_b = ("qa_outputs.weight", "qa_outputs.bias") if self.qa else \
            ("classifier.weight", "classifier.bias")
        if self.qa:
            self.p_cls = 0.0
        self._qa_ws = {}
        self.qa_last = None          # (per-sequence losses, positions [2, sequences], ignored index) of the last span loss
        self.mlm = self.lay.head == "mlm"               # cls.predictions on the labelled rows (csrc/mlm_head.cu)
        self.per_token = self.token_head or self.mlm    # packed bins need no cls_index
        self.V, self.Vp = cfg.vocab_size, self.lay.vocab_pad
        self._mlm_ws = {}
        self._mlm_shared = None
        self._mlm_saved = None
        self._mlm_pending = None     # (head buffers, transform input, labelled-row buffers or None) of the backward
        self.mlm_last = None
        n = self.lay.total
        self.shadow = torch.empty(n, dtype=torch.bfloat16, device=self.dev)   # bf16 copy the GEMMs read
        self.grads = torch.zeros(n, dtype=torch.bfloat16, device=self.dev)    # bf16 gradient bucket space
        self.rng = torch.zeros(2, dtype=torch.int64, device=self.dev)         # {seed, step} for the dropout streams
        self.owner = torch.empty(cfg.vocab_size, dtype=torch.int32, device=self.dev)
        self.split_ws = torch.empty(64 << 20, dtype=torch.uint8, device=self.dev)
        self.partials = torch.empty(32 << 20, dtype=torch.uint8, device=self.dev)   # column-sum partials; the embedding
        # backward's fp32 owner-row accumulators ([tokens + seq*types][H] fp32 = 13.4 MB at config A)
        self._ws = {}
        self._saved = None
        self.wgrad_stream = torch.cuda.Stream(device=self.dev)
        self._local = _LocalTransport(self)
        # gradient accumulation (no_sync(), Trainer gradient_accumulation_steps): fp32 accumulator over the flat space,
        # allocated on first use (local even under DDP); accum_in_use = some backward has accumulated into it;
        # accum_live = the accumulator holds gradients no fold / flush has consumed yet; _pass_op = the
        # b2_grad_accumulate mode of the running backward (None: none)
        self.accum = None
        self.accum_in_use = False
        self.accum_live = False
        self._pass_op = None
        self._pass_stream = None
        # dense + bias + dropout + residual + LayerNorm as ONE cluster kernel (b2_gemm_ln_fwd) for the two N = hidden
        # GEMMs of a layer, when the hidden size has a row-cluster tiling (768, 1024) and the device can co-schedule
        # the 3- / 4-CTA clusters; otherwise the GEMM epilogue + separate LayerNorm launch
        self.fused_ln = self.H in (768, 1024) and int(L.load().b2_gemm_ln_max_clusters(self.H)) > 0
        # fp32 accumulators for the bias gradients that kernels produce as a side effect of their epilogues (QKV bias
        # from attention backward, intermediate bias from the GELU' dgrad): per layer [3H | I]; one finishing launch
        # per step turns them into bf16 gradients and re-zeroes them
        # ... and for the LayerNorm-backward column sums (d_gamma, d_beta, dense-bias gradient of the branch): per
        # layer [3H qkv | I intermediate | 3H output-LN sets | 3H attention-output-LN sets]
        H_, I_ = self.H, self.I
        per = self.acc_per_layer = 9 * H_ + I_
        self.bias_acc = torch.zeros(max(1, self.nl * per), dtype=torch.float32, device=self.dev)
        segs = []
        for l in range(self.nl):
            pre = "bert.encoder.layer.%d." % l
            o = self.lay.off
            segs.append([l * per, o(pre + "attention.self.query.bias"), 3 * H_])
            segs.append([l * per + 3 * H_, o(pre + "intermediate.dense.bias"), I_])
            b2_ = l * per + 3 * H_ + I_
            segs.append([b2_, o(pre + "output.LayerNorm.weight"), H_])
            segs.append([b2_ + H_, o(pre + "output.LayerNorm.bias"), H_])
            segs.append([b2_ + 2 * H_, o(pre + "output.dense.bias"), H_])
            b1_ = b2_ + 3 * H_
            segs.append([b1_, o(pre + "attention.output.LayerNorm.weight"), H_])
            segs.append([b1_ + H_, o(pre + "attention.output.LayerNorm.bias"), H_])
            segs.append([b1_ + 2 * H_, o(pre + "attention.output.dense.bias"), H_])
        self.segs_per_layer = 8
        self.bias_segs = torch.tensor(segs if segs else [[0, 0, 0]], dtype=torch.int64, device=self.dev)
        # fixed-order backward (torch.use_deterministic_algorithms): scratch of its own for the weight-gradient stream's
        # column sums, and the per-block partials of the two LayerNorm backwards of a layer, double-buffered by layer
        # parity like dzd / dU (layer l - 2 reuses a set only after done[l]); allocated on the first such backward
        self._det_bufs = None
        s = self.stream()
        L.call("b2_embed_owner_init", L.ptr(self.owner), cfg.vocab_size, s)
        L.call("b2_rng_seed", L.ptr(self.rng), int(torch.initial_seed()) & ((1 << 63) - 1), 0, s)
        self.refresh_shadow()

    # ---- plumbing ----
    def stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    @property
    def transport(self):
        """whom the optimizer's step schedule asks about ranges, streams and peers"""
        ddp = self.model._ddp
        return ddp if ddp is not None and ddp.world > 1 else self._local

    def rebind(self, shadow, grads):
        """DDP moves the exchanged buffers into IPC-shared allocations."""
        shadow.copy_(self.shadow)
        grads.zero_()
        self.shadow, self.grads = shadow, grads

    def refresh_shadow(self):
        L.call("b2_cast_f32_to_bf16", L.ptr(self.model._flat), L.ptr(self.shadow), self.lay.total, self.stream())

    # ---- gradient accumulation ----
    def ensure_accum(self):
        if self.accum is None:
            self.accum = torch.empty(self.lay.total, dtype=torch.float32, device=self.dev)
        self.accum_in_use = True

    def accumulate_range(self, begin, end, op, stream):
        L.call("b2_grad_accumulate", self.grads.data_ptr(), self.accum.data_ptr(), begin, end, op, stream)

    def start_pass(self, accumulate):
        """Sets the accumulation mode of the next backward: STORE / ADD into the accumulator (accumulate), FOLD it into
        the gradients (the first plain backward after accumulating ones), or nothing."""
        if accumulate:
            self.ensure_accum()
            self._pass_op = L.ACCUM_ADD if self.accum_live else L.ACCUM_STORE
        else:
            self._pass_op = L.ACCUM_FOLD if self.accum_live else None

    def end_pass(self):
        """After the backward: the whole-range accumulate / fold when no per-bucket launch did it, else the join of
        the stream that ran them (the next backward overwrites `grads`, and whoever reads them next is on the main
        stream); an accumulating pass also moves the dropout stream on, as optimizer.step() does for the final one."""
        op, side = self._pass_op, self._pass_stream
        self._pass_op, self._pass_stream = None, None
        if op is None:
            return
        main = torch.cuda.current_stream(self.dev)
        if side is None:
            self.accumulate_range(0, self.lay.total, op, main.cuda_stream)
        else:
            main.wait_stream(side)
        self.accum_live = op != L.ACCUM_FOLD
        if op != L.ACCUM_FOLD:
            L.call("b2_step_advance", None, L.ptr(self.rng), None, main.cuda_stream)

    def flush_accum(self, stream):
        """optimizer.step() with the window still open (no final backward): grads = bf16(accumulator)"""
        if self.accum_live:
            self.accumulate_range(0, self.lay.total, L.ACCUM_FLUSH, stream)
            self.accum_live = False

    def seed_dropout(self, seed, step=0):
        L.call("b2_rng_seed", L.ptr(self.rng), int(seed), int(step), self.stream())

    def head_rows(self, B, S, packed):
        """rows of the head's logits: every token (token head), else one per sequence (packed: its cls rows)"""
        if self.per_token:
            return B * S
        return B if packed is None else packed[1].numel()

    def w(self, name):
        return self.shadow.data_ptr() + 2 * self.lay.off(name)

    def g(self, name):
        return self.grads.data_ptr() + 2 * self.lay.off(name)

    def workspace(self, B, S, Bo=None):
        """B x S token rows; Bo = number of sequences the head sees (packed bins: B bins carry Bo >= B sequences)"""
        Bo = B if Bo is None else Bo
        key = (B, S, Bo)
        ws = self._ws.get(key)
        if ws is not None:
            return ws
        H, I, M, nl = self.H, self.I, B * S, self.nl
        bf, f32, dev = torch.bfloat16, torch.float32, self.dev

        def e(*shape, dtype=bf):
            return torch.empty(*shape, dtype=dtype, device=dev)

        ws = {
            "emb_out": e(M, H), "emb_pre": e(M, H), "emb_mean": e(M, dtype=f32), "emb_rstd": e(M, dtype=f32),
            # fp32 residual stream of the forward (fused dense + LayerNorm path): the LayerNorm outputs are kept
            # unrounded for the NEXT block's residual add; the bf16 copies above / below feed the GEMMs
            "emb_out_f": e(M, H, dtype=f32) if self.fused_ln else None,
            "ids32": e(M, dtype=torch.int32), "tt32": e(M, dtype=torch.int32), "pos32": e(M, dtype=torch.int32),
            "layers": [
                {"qkv": e(M, 3 * H), "ctx": e(M, H), "lse": e(B * self.heads * S, dtype=f32),
                 # attention-dropout decisions of the forward, 1 bit per (b, h, q, k): read back by the backward
                 "keep": e(B * self.heads * S * (S // 64), dtype=torch.int64) if S == 128 else None,
                 "z1": e(M, H),
                 "x1": e(M, H), "mean1": e(M, dtype=f32), "rstd1": e(M, dtype=f32), "u": e(M, I), "h": e(M, I),
                 "z2": e(M, H), "x2": e(M, H), "mean2": e(M, dtype=f32), "rstd2": e(M, dtype=f32),
                 "x1f": e(M, H, dtype=f32) if self.fused_ln else None,
                 "x2f": e(M, H, dtype=f32) if (self.fused_ln and li < nl - 1) else None}
                for li in range(nl)],
            "pooled": None if self.per_token else e(Bo, H), "logits": e(Bo, self.C, dtype=f32),
            "loss": e((), dtype=f32),
            "dlogits": e(Bo, self.C, dtype=f32), "dloss_logits": e(Bo, self.C, dtype=f32),
            # gradient of the residual stream: fp32 (12 layers of residual adds would otherwise each round it to bf16);
            # dzd / dz1d are the bf16 (dropout-masked) copies the tensor cores consume
            "dxA": e(M, H, dtype=f32), "dxB": e(M, H, dtype=f32),
            "emb_dx": e(M, H), "dctx": e(M, H),
            # the token head's fp32 parameter-gradient partials, the sequence head's two [batch, H] planes
            "head_scratch": e(int(L.load().b2_token_head_scratch_floats(M, H, self.C)), dtype=f32) if self.token_head
            else None if self.mlm else e(2 * Bo, H, dtype=f32),
            # operands of the weight-gradient GEMMs, double-buffered by layer parity (see _backward_from_dlogits)
            "dzd": [e(M, H), e(M, H)], "dz1d": [e(M, H), e(M, H)], "dU": [e(M, I), e(M, I)],
            "dqkv": [e(M, 3 * H), e(M, 3 * H)],
            "dq_accum": e(M, H, dtype=f32) if S > 128 else None,
            "zeros_tt": torch.zeros(B, S, dtype=torch.int64, device=dev),
        }
        self._ws[key] = ws
        return ws

    def det_buffers(self):
        """(weight-gradient-stream column-sum scratch, LayerNorm-backward partials [parity][LN2, LN1]) of the
        fixed-order backward.  A partials buffer holds one [3][hidden] fp32 row per block of the LayerNorm backward's
        single wave (one block per SM), as many as the accumulating form launches."""
        if self._det_bufs is None:
            sms = torch.cuda.get_device_properties(self.dev).multi_processor_count
            u8 = dict(dtype=torch.uint8, device=self.dev)
            ln_bytes = sms * 3 * self.H * 4
            side = torch.empty(32 * 4 * max(3 * self.H, self.I), **u8)    # b2_colsum's at most 32 partial rows
            self._det_bufs = (side, [[torch.empty(ln_bytes, **u8) for _ in range(2)] for _ in range(2)])
        return self._det_bufs

    def gemm_grouped(self, problems, stream):
        """independent GEMMs behind one launch where the library can group them (the layer's weight gradients)"""
        arr = (L.GemmArgs * len(problems))(*problems)
        L.call("b2_gemm_bf16_grouped", arr, len(problems), stream)

    def gemm(self, M, N, K, A, lda, a_major, Bm, ldb, b_major, D, ldd, epi=L.EPI_NONE, bias=None, aux_in=None,
             ld_aux_in=0, aux_out=None, ld_aux_out=0, p=0.0, site=0, split=False, stream=None, colsum=None,
             defer=None, splits=0):
        """defer: a list -> the problem is appended to it instead of being launched (see gemm_grouped);
        splits: force_splits (0: the cost model's choice)"""
        a = L.GemmArgs()
        a.M, a.N, a.K = M, N, K
        a.A, a.lda, a.a_major = A, lda, a_major
        a.B, a.ldb, a.b_major = Bm, ldb, b_major
        a.D, a.ldd, a.epilogue = D, ldd, epi
        a.bias, a.aux_in, a.ld_aux_in, a.aux_out, a.ld_aux_out = bias, aux_in, ld_aux_in, aux_out, ld_aux_out
        a.dropout_p, a.rng_state, a.rng_site = p, self.rng.data_ptr(), site
        if split:
            a.workspace, a.workspace_bytes = self.split_ws.data_ptr(), self.split_ws.numel()
        else:
            a.workspace, a.workspace_bytes = None, 0
        a.force_bn = a.force_kernel = 0
        a.force_splits = splits
        a.debug_timing = None
        a.colsum_out = colsum
        if defer is not None:
            defer.append(a)
            return
        L.call("b2_gemm_bf16", a, stream if stream is not None else self.stream())

    def dense_dropout_residual_layernorm(self, M, K, A, W, bias, resid, resid_f, p, site, gamma, beta, z, y, y_f, mean,
                                         rstd):
        """y = LayerNorm(dropout(A W^T + bias) + resid) with z = the pre-LN sum kept for the backward
        (BertSelfOutput / BertOutput, modeling_bert.py:294-298, :352-356).  Fused path: ONE cluster kernel, the
        residual comes in as fp32 (resid_f), the output leaves as bf16 (y) and fp32 (y_f, may be None)."""
        H = self.H
        s = self.stream()
        eps = float(self.cfg.layer_norm_eps)
        if self.fused_ln:
            a = L.GemmArgs()
            a.M, a.N, a.K = M, H, K
            a.A, a.lda, a.a_major = A, K, L.MAJOR_K
            a.B, a.ldb, a.b_major = W, K, L.MAJOR_K
            a.D, a.ldd, a.epilogue = z, H, L.EPI_BIAS_DROPOUT_RESIDUAL
            a.bias, a.aux_in, a.ld_aux_in, a.aux_out, a.ld_aux_out = bias, resid_f, H, None, 0
            a.dropout_p, a.rng_state, a.rng_site = p, self.rng.data_ptr(), site
            a.workspace, a.workspace_bytes = None, 0
            a.force_bn = a.force_splits = a.force_kernel = 0
            a.debug_timing, a.colsum_out = None, None
            L.call("b2_gemm_ln_fwd", a, gamma, beta, eps, y, H, y_f, H if y_f else 0, mean, rstd, s)
            return
        self.gemm(M, H, K, A, K, L.MAJOR_K, W, K, L.MAJOR_K, z, H, L.EPI_BIAS_DROPOUT_RESIDUAL, bias=bias,
                  aux_in=resid, ld_aux_in=H, p=p, site=site)
        L.call("b2_layernorm_fwd", z, gamma, beta, M, H, eps, y, mean, rstd, s)

    # ---- forward --------------------------------------------------------------------------------------------------------
    def forward(self, input_ids, token_type_ids, attention_mask, labels, training, need_backward, packed=None,
                loss_fn=None, mlm_full=True, ignore_index=-100, mlm_capacity=None, mlm_dloss=None,
                qa_ignored_index=None, qa_dloss=None):
        """packed: None, or (position_ids int64 [bins, S], segments int32 [bins, S], cls_index int64 [batch]) -- the
        rows of `input_ids` are then S-token bins produced by packing.pack_batch (S a multiple of 128, at most 512),
        not sequences.
        loss_fn: the losses.Loss of `labels` (None: the model's problem-type loss, HF's in-model loss).
        Multiple-choice head: the rows of `input_ids` are the B·N choice sequences, example-major; loss_fn is
        required, its num_labels is N, and `labels` are int64 [B].
        Masked-LM head: `labels` int64 [B, S] with `ignore_index`; the loss runs on the labelled rows only, in a
        capacity of mlm_capacity rows (None: their count rounded up to 128, read from the device); mlm_full: also
        the logits of every row (returned as [B, S, V]; else None); mlm_dloss: a device scalar d(objective)/d(loss)
        -- the same cross-entropy launch then also writes the labelled rows' d_logits for the backward (the
        captured steps' one pass).
        QA head: `labels` int64 [2, sequences], the raw start / end positions; qa_ignored_index: a packed batch's HF
        ignored index (None: the bin length); qa_dloss: as mlm_dloss, for the span loss."""
        cfg, H, I = self.cfg, self.H, self.I
        if input_ids.dim() != 2:
            raise ValueError("input_ids must be [batch, seq]")
        B, S = input_ids.shape
        Bo = B
        if packed is not None:
            pos_ids, segs, cls_rows = packed
            if attention_mask is not None:
                raise ValueError("packed bins carry their own (block-diagonal) mask: pass attention_mask=None")
            for t, nm, dt, shape in ((pos_ids, "position_ids", torch.int64, (B, S)), (segs, "segments", torch.int32, (B, S)),
                                     (cls_rows, "cls_index", torch.int64, None)):
                if t is None and self.per_token and not self.qa and nm == "cls_index":
                    continue      # the token head reads every bin row (the QA loss needs each sequence's first row)
                if t.device != self.dev or t.dtype != dt or (shape is not None and tuple(t.shape) != shape):
                    raise TypeError("%s must be a %s tensor%s on %s" % (nm, dt, "" if shape is None else " of shape %s"
                                                                        % (shape,), self.dev))
            pos_ids, segs = pos_ids.contiguous(), segs.contiguous()
            if not self.per_token:
                cls_rows = cls_rows.contiguous().view(-1)
                Bo = cls_rows.numel()
            elif self.qa:
                cls_rows = cls_rows.contiguous().view(-1)
        if self.per_token:
            Bo = B * S
        if B == 0 or S == 0:
            raise ValueError("empty batch")
        if S % 128 != 0 or S > 512 or S > cfg.max_position_embeddings:
            raise ValueError("seq_len=%d: the attention kernel covers multiples of 128 up to 512 "
                             "(the reference pads every batch to max_seq_len=128)" % S)
        for t, nm in ((input_ids, "input_ids"), (token_type_ids, "token_type_ids"),
                      (attention_mask, "attention_mask"), (labels, "labels")):
            if t is not None:
                if t.device != self.dev:
                    raise RuntimeError("%s is on %s, model on %s" % (nm, t.device, self.dev))
                if t is not labels and t.dtype != torch.int64:
                    raise TypeError("%s must be int64 (as the reference Collate produces)" % nm)
        loss_rows = Bo
        if labels is not None and not self.mlm and not self.qa:
            if self.mc:
                # loss_fn's labels are the choices: B examples of N choice logits each
                if loss_fn is None or Bo % loss_fn.C != 0:
                    raise ValueError("multiple-choice loss: need the loss over N choices of %d choice sequences"
                                     % Bo)
                loss_rows = Bo // loss_fn.C
            elif loss_fn is None:
                loss_fn = self.model._problem_type_loss(labels)
            labels = loss_fn.device_labels(labels, loss_rows)
        ws = self.workspace(B, S, Bo)
        M = B * S
        s = self.stream()
        ids = input_ids.contiguous()
        tt = (token_type_ids if token_type_ids is not None else ws["zeros_tt"]).contiguous()
        mask = attention_mask.contiguous() if attention_mask is not None else None
        p_h = self.p_hidden if training else 0.0
        p_a = self.p_attn if training else 0.0
        p_c = self.p_cls if training else 0.0
        rng = self.rng.data_ptr()
        w = self.w
        KM, MN = L.MAJOR_K, L.MAJOR_MN

        emb_w = (w("bert.embeddings.word_embeddings.weight"), w("bert.embeddings.position_embeddings.weight"),
                 w("bert.embeddings.token_type_embeddings.weight"), w("bert.embeddings.LayerNorm.weight"),
                 w("bert.embeddings.LayerNorm.bias"))
        emb_out = (L.ptr(ws["emb_out"]), L.ptr(ws["emb_out_f"]), L.ptr(ws["emb_pre"]), L.ptr(ws["emb_mean"]),
                   L.ptr(ws["emb_rstd"]), L.ptr(ws["ids32"]), L.ptr(ws["tt32"]))
        if packed is None:
            L.call("b2_embed_fwd", ids.data_ptr(), tt.data_ptr(), B, S, *emb_w, H, cfg.vocab_size, cfg.type_vocab_size,
                   float(cfg.layer_norm_eps), p_h, rng, 0, *emb_out, s)
        else:
            L.call("b2_embed_fwd_packed", ids.data_ptr(), tt.data_ptr(), pos_ids.data_ptr(),
                   cfg.max_position_embeddings, B, S, *emb_w, H, cfg.vocab_size, cfg.type_vocab_size,
                   float(cfg.layer_norm_eps), p_h, rng, 0, *emb_out, L.ptr(ws["pos32"]), s)
        x, xf = ws["emb_out"], ws["emb_out_f"]
        for l in range(self.nl):
            a = ws["layers"][l]
            pre = "bert.encoder.layer.%d." % l
            self.gemm(M, 3 * H, H, x.data_ptr(), H, KM, w(pre + "attention.self.query.weight"), H, KM,
                      a["qkv"].data_ptr(), 3 * H, L.EPI_BIAS, bias=w(pre + "attention.self.query.bias"))
            if packed is None:
                L.call("b2_attention_fwd", a["qkv"].data_ptr(), L.ptr(mask), B, S, self.heads, 64, p_a, rng, 1 + 3 * l,
                       a["ctx"].data_ptr(), a["lse"].data_ptr(), L.ptr(a["keep"]) if need_backward else None, s)
            elif S == 128:
                L.call("b2_attention_fwd_packed", a["qkv"].data_ptr(), segs.data_ptr(), B, self.heads, 64, p_a, rng,
                       1 + 3 * l, a["ctx"].data_ptr(), a["lse"].data_ptr(),
                       L.ptr(a["keep"]) if need_backward else None, s)
            else:
                L.call("b2_attention_fwd_packed_seq", a["qkv"].data_ptr(), segs.data_ptr(), B, S, self.heads, 64, p_a,
                       rng, 1 + 3 * l, a["ctx"].data_ptr(), a["lse"].data_ptr(), None, s)
            self.dense_dropout_residual_layernorm(
                M, H, a["ctx"].data_ptr(), w(pre + "attention.output.dense.weight"),
                w(pre + "attention.output.dense.bias"), x.data_ptr(), L.ptr(xf), p_h, 2 + 3 * l,
                w(pre + "attention.output.LayerNorm.weight"), w(pre + "attention.output.LayerNorm.bias"),
                a["z1"].data_ptr(), a["x1"].data_ptr(), L.ptr(a["x1f"]), a["mean1"].data_ptr(), a["rstd1"].data_ptr())
            self.gemm(M, I, H, a["x1"].data_ptr(), H, KM, w(pre + "intermediate.dense.weight"), H, KM,
                      a["h"].data_ptr(), I, L.EPI_BIAS_GELU, bias=w(pre + "intermediate.dense.bias"),
                      aux_out=a["u"].data_ptr(), ld_aux_out=I)
            self.dense_dropout_residual_layernorm(
                M, I, a["h"].data_ptr(), w(pre + "output.dense.weight"), w(pre + "output.dense.bias"),
                a["x1"].data_ptr(), L.ptr(a["x1f"]), p_h, 3 + 3 * l, w(pre + "output.LayerNorm.weight"),
                w(pre + "output.LayerNorm.bias"), a["z2"].data_ptr(), a["x2"].data_ptr(), L.ptr(a["x2f"]),
                a["mean2"].data_ptr(), a["rstd2"].data_ptr())
            x, xf = a["x2"], a["x2f"]
        if self.mlm:
            logits, loss = self._mlm_forward(x, M, labels, need_backward, mlm_full, ignore_index, mlm_capacity,
                                             mlm_dloss)
            if need_backward:
                self._saved = (B, S, mask, p_h, p_a, p_c, None if packed is None else (segs, None))
            return (None if logits is None else logits.view(B, S, self.V)), loss
        if self.token_head:
            L.call("b2_token_head_fwd", x.data_ptr(), M, H, w(self.cls_w), w(self.cls_b), self.C, p_c,
                   rng, 1 + 3 * self.nl, ws["logits"].data_ptr(), s)
        elif packed is None:
            head_w = (w("bert.pooler.dense.weight"), w("bert.pooler.dense.bias"), w("classifier.weight"),
                      w("classifier.bias"))
            L.call("b2_head_fwd", x.data_ptr(), B, S, H, *head_w, self.C, p_c, rng, 1 + 3 * self.nl,
                   ws["pooled"].data_ptr(), ws["logits"].data_ptr(), s)
        else:
            head_w = (w("bert.pooler.dense.weight"), w("bert.pooler.dense.bias"), w("classifier.weight"),
                      w("classifier.bias"))
            L.call("b2_head_fwd_packed", x.data_ptr(), cls_rows.data_ptr(), Bo, H, *head_w, self.C, p_c, rng,
                   1 + 3 * self.nl, ws["pooled"].data_ptr(), ws["logits"].data_ptr(), s)
        loss = None
        if labels is not None and self.qa:
            loss = self._qa_loss(ws, M, labels, S, None if packed is None else (segs, cls_rows), need_backward,
                                 qa_ignored_index, qa_dloss)
        elif labels is not None:
            loss_fn.launch(ws["logits"].data_ptr(), labels, loss_rows, ws["loss"].data_ptr(),
                           ws["dloss_logits"].data_ptr() if need_backward else None, s)
            loss = ws["loss"]
        if need_backward:
            self._saved = (B, S, mask, p_h, p_a, p_c, None if packed is None else (segs, cls_rows))
        if self.token_head:
            return ws["logits"].view(B, S, self.C), loss
        return ws["logits"], loss

    # ---- question-answering span loss -----------------------------------------------------------------------------------
    def _qa_loss(self, ws, M, positions, S, packed, need_backward, ignored_index, dloss):
        """b2_qa_span_loss over the head's [M, 2] logits: the loss into ws["loss"] and, for a backward, d(loss)/d(logits)
        into ws["dloss_logits"] (scaled by the device scalar `dloss`, None: 1).  Padded: sequence b is rows
        [b S, (b + 1) S) and S is HF's ignored index.  Packed (segs, cls_rows): sequence b starts at bin row
        cls_rows[b] and its length is the extent of that row's segment."""
        if positions.dtype != torch.int64 or positions.dim() != 2 or positions.shape[0] != 2:
            raise TypeError("QA positions must be int64 [2, sequences] (start row, end row), got %s %s"
                            % (positions.dtype, list(positions.shape)))
        nseq = positions.shape[1]
        pos = positions.contiguous()
        first = lens = None
        if packed is None:
            if nseq * S != M:
                raise ValueError("QA positions: %d sequences for %d rows of %d tokens" % (nseq, M // S, S))
            ignored = S
        else:
            segs, first = packed
            if first.numel() != nseq:
                raise ValueError("QA positions: %d sequences, cls_index has %d" % (nseq, first.numel()))
            seg = segs.view(-1)[first]
            lens = ((seg >> 16) - (seg & 0xFFFF)).to(torch.int64)
            ignored = S if ignored_index is None else int(ignored_index)
        buf = self._qa_ws.get(nseq)
        if buf is None:
            buf = self._qa_ws[nseq] = torch.empty(2 * nseq, dtype=torch.float32, device=self.dev)
        self.qa_last = (buf, pos, ignored)
        L.call("b2_qa_span_loss", ws["logits"].data_ptr(), M, pos.data_ptr(), pos.data_ptr() + 8 * nseq, nseq,
               ignored, L.ptr(first), L.ptr(lens), L.ptr(dloss), buf.data_ptr(),
               ws["dloss_logits"].data_ptr() if need_backward else None, ws["loss"].data_ptr(), self.stream())
        return ws["loss"]

    # ---- masked-LM head (cls.predictions) ---------------------------------------------------------------------------------
    def _mlm_buffers(self, M, rows, full=False):
        """the head's activations over `rows` rows: the labelled rows' capacity, or (full) all M rows, the logits of
        the eager output"""
        key = (M, rows, full)
        hb = self._mlm_ws.get(key)
        if hb is not None:
            return hb
        H, Vp, dev = self.H, self.Vp, self.dev
        e = lambda *shape, dtype=torch.bfloat16: torch.empty(*shape, dtype=dtype, device=dev)
        f32, i32 = torch.float32, torch.int32
        hb = {"rows": rows, "x": None if full else e(rows, H), "u": e(rows, H), "h": e(rows, H), "t": e(rows, H),
              "mean": e(rows, dtype=f32), "rstd": e(rows, dtype=f32), "logits": e(rows, Vp, dtype=f32),
              "row_loss": e(rows, dtype=f32), "pred": e(rows, dtype=i32), "loss": e((), dtype=f32),
              "dlog": None, "dt": None,
              # compaction: source row of each slot, slot of each token, label of each slot (-1: none), count
              "src": e(rows, dtype=i32), "slot": e(M, dtype=i32), "labels": e(rows, dtype=i32),
              "count": e(1, dtype=i32)}
        self._mlm_ws[key] = hb
        return hb

    def _mlm_grad_buffers(self, hb):
        """the backward's buffers over the head's rows, allocated by the first backward that needs them"""
        if hb["dlog"] is None:
            rows, H, dev = hb["rows"], self.H, self.dev
            e = lambda *shape, dtype=torch.bfloat16: torch.empty(*shape, dtype=dtype, device=dev)
            hb.update(dlog=e(rows, self.Vp), dt=e(rows, H, dtype=torch.float32), dh=e(rows, H, dtype=torch.float32),
                      dh_bf=e(rows, H), du=e(rows, H), dx=e(rows, H, dtype=torch.float32))
        if self._mlm_shared is None:
            sms = torch.cuda.get_device_properties(self.dev).multi_processor_count
            self._mlm_shared = {
                # fp32 decoder part of the tied word-embedding gradient [vocab_pad, H]
                "dec": torch.empty(self.Vp, self.H, dtype=torch.float32, device=self.dev),
                # b2_colsum's at most 32 partial rows over vocab_pad columns
                "colsum": torch.empty(32 * self.Vp, dtype=torch.float32, device=self.dev),
                # the transform LayerNorm backward's per-block partials (one block per SM)
                "ln_parts": torch.empty(sms * 3 * self.H, dtype=torch.float32, device=self.dev),
                "n_lab_one": torch.ones(1, dtype=torch.int32, device=self.dev)}
        return hb

    def _mlm_head_fwd(self, x, hb):
        """transform (dense + GELU, LayerNorm) and the fp32 logits over the rows of hb: bias fill, then the product
        with the word-embedding table added by the GEMM (N = vocab_pad)"""
        H, rows, s, w = self.H, hb["rows"], self.stream(), self.w
        KM = L.MAJOR_K
        self.gemm(rows, H, H, x.data_ptr(), H, KM, w("cls.predictions.transform.dense.weight"), H, KM,
                  hb["h"].data_ptr(), H, L.EPI_BIAS_GELU, bias=w("cls.predictions.transform.dense.bias"),
                  aux_out=hb["u"].data_ptr(), ld_aux_out=H)
        L.call("b2_layernorm_fwd", hb["h"].data_ptr(), w("cls.predictions.transform.LayerNorm.weight"),
               w("cls.predictions.transform.LayerNorm.bias"), rows, H, float(self.cfg.layer_norm_eps),
               hb["t"].data_ptr(), hb["mean"].data_ptr(), hb["rstd"].data_ptr(), s)
        L.call("b2_mlm_bias_fill", w("cls.predictions.bias"), rows, self.Vp, hb["logits"].data_ptr(), s)
        self.gemm(rows, self.Vp, H, hb["t"].data_ptr(), H, KM, w("bert.embeddings.word_embeddings.weight"), H, KM,
                  hb["logits"].data_ptr(), self.Vp, L.EPI_ACCUM_F32,
                  splits=1 if torch.are_deterministic_algorithms_enabled() else 0)

    def mlm_capacity(self, labels, ignore_index, M):
        """the labelled rows' capacity for host labels: their count rounded up to 128 (at least 128, at most M).
        Raises ValueError on a label outside [0, V) that is not ignore_index."""
        lab = labels.reshape(-1)
        bad = (lab != ignore_index) & ((lab < 0) | (lab >= self.V))
        n_bad, n = (int(v) for v in torch.stack([bad.sum(), (lab != ignore_index).sum()]).tolist())
        if n_bad:
            raise ValueError("masked-LM label %d is outside [0, %d) and is not the ignore_index %d"
                             % (int(lab[bad][0]), self.V, ignore_index))
        return min(M, max(128, (n + 127) // 128 * 128)), n

    def _mlm_forward(self, x, M, labels, need_backward, full, ignore_index, capacity, dloss=None):
        s, V, Vp = self.stream(), self.V, self.Vp
        loss, logits, gb = None, None, None
        if labels is not None:
            if labels.dtype != torch.int64 or labels.numel() != M:
                raise TypeError("masked-LM labels must be int64 with one per token (%d), got %s %s"
                                % (M, labels.dtype, list(labels.shape)))
            if capacity is None:
                capacity, _n = self.mlm_capacity(labels, ignore_index, M)
            gb = self._mlm_buffers(M, capacity)
            lab = labels.contiguous()
            L.call("b2_mlm_compact", lab.data_ptr(), M, int(ignore_index), V, capacity, gb["src"].data_ptr(),
                   gb["slot"].data_ptr(), gb["labels"].data_ptr(), gb["count"].data_ptr(), s)
            L.call("b2_mlm_gather_rows", x.data_ptr(), gb["src"].data_ptr(), gb["count"].data_ptr(), capacity, self.H,
                   gb["x"].data_ptr(), s)
            self._mlm_head_fwd(gb["x"], gb)
            cnt = gb["count"].data_ptr()
            dlog = None
            if dloss is not None:
                dlog = self._mlm_grad_buffers(gb)["dlog"]
            L.call("b2_mlm_ce", gb["logits"].data_ptr(), capacity, V, Vp, gb["labels"].data_ptr(), cnt, cnt,
                   L.ptr(dloss), None, 0, gb["row_loss"].data_ptr(), gb["pred"].data_ptr(), L.ptr(dlog),
                   gb["loss"].data_ptr(), s)
            loss = gb["loss"]
            if dlog is not None and need_backward:
                # d_logits are final: the captured step's backward starts from them (_backward_from_dlogits)
                self._mlm_pending = (gb, gb["x"], gb)
            self.mlm_last = gb
        fb = None
        if full:
            fb = self._mlm_buffers(M, M, full=True)
            self._mlm_head_fwd(x, fb)
            logits = fb["logits"][:, :V]
        if need_backward:
            # (labelled-row buffers, full-row buffers, the labels and their ignore index, the encoder output)
            self._mlm_saved = (gb, fb, labels, ignore_index, x)
        return logits, loss

    def _mlm_dlogits(self, d_logits, d_loss):
        """the bf16 d_logits of the head's rows: over the labelled rows from the loss alone, else dense over every
        row (the incoming fp32 d_logits plus the loss's part)"""
        gb, fb, labels, ignore_index, x = self._mlm_saved
        s, V, Vp = self.stream(), self.V, self.Vp
        dl_ptr = None if d_loss is None else d_loss.to(torch.float32).contiguous()
        if d_logits is None:
            if gb is None:
                raise RuntimeError("masked-LM backward without labels and without a gradient of the logits")
            hb = self._mlm_grad_buffers(gb)
            cnt = gb["count"].data_ptr()
            L.call("b2_mlm_ce", gb["logits"].data_ptr(), gb["rows"], V, Vp, gb["labels"].data_ptr(), cnt, cnt,
                   L.ptr(dl_ptr), None, 0, gb["row_loss"].data_ptr(), None, hb["dlog"].data_ptr(), None, s)
            self._mlm_pending = (hb, gb["x"], gb)
        else:
            hb = self._mlm_grad_buffers(fb)
            M = fb["rows"]
            extra = d_logits.to(torch.float32).reshape(M, V).contiguous()
            lab32, n_lab = None, self._mlm_shared["n_lab_one"]
            if dl_ptr is not None and gb is not None:
                lab = labels.reshape(-1)
                lab32 = torch.where(lab == ignore_index, torch.full_like(lab, -1), lab).to(torch.int32)
                n_lab = gb["count"]
            L.call("b2_mlm_ce", fb["logits"].data_ptr(), M, V, Vp, L.ptr(lab32), None, n_lab.data_ptr(),
                   L.ptr(dl_ptr), extra.data_ptr(), V, fb["row_loss"].data_ptr(), None, hb["dlog"].data_ptr(), None,
                   s)
            self._mlm_pending = (hb, x, None)
        self._mlm_saved = None

    def _mlm_backward(self, x_last, dxA, det, main, side):
        """the head's backward from the pending d_logits: d_hidden (fp32, every row of dxA) on the main stream, the
        head's parameter gradients and the decoder's part of the tied word gradient on the weight-gradient stream.
        Returns the event after which that decoder part (self._mlm_shared["dec"]) is final."""
        hb, xin, gb = self._mlm_pending
        self._mlm_pending = None
        H, Vp, rows = self.H, self.Vp, hb["rows"]
        w, g = self.w, self.g
        KM, MN = L.MAJOR_K, L.MAJOR_MN
        sh = self._mlm_shared
        s = main.cuda_stream
        side_s = side if self.nl > 0 else main
        ss = side_s.cuda_stream
        splits = 1 if det else 0
        # d_t = d_logits E  (N = H, K = vocab_pad); then the transform's LayerNorm and GELU backward
        L.call("b2_zero", hb["dt"].data_ptr(), hb["dt"].numel() * 4, s)
        self.gemm(rows, H, Vp, hb["dlog"].data_ptr(), Vp, KM, w("bert.embeddings.word_embeddings.weight"), H, MN,
                  hb["dt"].data_ptr(), H, L.EPI_ACCUM_F32, splits=splits)
        nparts = ctypes.c_int32()
        L.call("b2_layernorm_bwd", hb["dt"].data_ptr(), None, hb["h"].data_ptr(), hb["mean"].data_ptr(),
               hb["rstd"].data_ptr(), w("cls.predictions.transform.LayerNorm.weight"), rows, H, 0.0, None, 0, 1,
               hb["dh"].data_ptr(), hb["dh_bf"].data_ptr(), g("cls.predictions.transform.LayerNorm.weight"),
               g("cls.predictions.transform.LayerNorm.bias"), None, sh["ln_parts"].data_ptr(),
               sh["ln_parts"].numel() * 4, ctypes.addressof(nparts), s)
        L.call("b2_mlm_gelu_bwd", hb["dh"].data_ptr(), hb["u"].data_ptr(), rows * H, hb["du"].data_ptr(), s)
        # fork: the parameter gradients (fixed-order column sums in both modes) and the decoder's dense part
        ev = torch.cuda.Event()
        ev.record(main)
        side_s.wait_event(ev)
        L.call("b2_zero", sh["dec"].data_ptr(), sh["dec"].numel() * 4, ss)
        self.gemm(Vp, H, rows, hb["dlog"].data_ptr(), Vp, MN, hb["t"].data_ptr(), H, MN, sh["dec"].data_ptr(), H,
                  L.EPI_ACCUM_F32, splits=splits, stream=ss)
        sc, scn = sh["colsum"].data_ptr(), sh["colsum"].numel() * 4
        L.call("b2_colsum", hb["dlog"].data_ptr(), rows, Vp, Vp, g("cls.predictions.bias"), sc, scn, ss)
        L.call("b2_colsum_finish", sh["ln_parts"].data_ptr(), nparts.value, 3, H,
               g("cls.predictions.transform.LayerNorm.weight"), g("cls.predictions.transform.LayerNorm.bias"), None,
               ss)
        self.gemm(H, H, rows, hb["du"].data_ptr(), H, MN, xin.data_ptr(), H, MN,
                  g("cls.predictions.transform.dense.weight"), H, split=True, stream=ss)
        L.call("b2_colsum", hb["du"].data_ptr(), rows, H, H, g("cls.predictions.transform.dense.bias"), sc, scn, ss)
        dec_done = torch.cuda.Event()
        dec_done.record(side_s)
        # d_hidden = du W_t: straight into dxA over every row, or over the labelled rows and scattered
        out = dxA if gb is None else hb["dx"]
        L.call("b2_zero", out.data_ptr(), out.numel() * 4, s)
        self.gemm(rows, H, H, hb["du"].data_ptr(), H, KM, w("cls.predictions.transform.dense.weight"), H, MN,
                  out.data_ptr(), H, L.EPI_ACCUM_F32, splits=splits)
        if gb is not None:
            L.call("b2_mlm_scatter_rows", out.data_ptr(), gb["slot"].data_ptr(), dxA.shape[0], H, dxA.data_ptr(), s)
        return dec_done

    # ---- backward ---------------------------------------------------------------------------------------------------------
    def backward(self, d_logits, d_loss=None, stream=None):
        """d_logits: fp32 [B, C] gradient wrt the returned logits; d_loss: optional scalar gradient wrt HF's loss."""
        if self._saved is None:
            raise RuntimeError("backward called without a training forward")
        B, S, mask, p_h, p_a, p_c, packed = self._saved
        self._saved = None
        if self.mlm:
            self._mlm_dlogits(d_logits, d_loss)
            return self._backward_from_dlogits(None, B, S, mask, p_h, p_a, p_c, packed)
        Bo = self.head_rows(B, S, packed)
        ws = self.workspace(B, S, Bo)
        dl = ws["dlogits"]
        if d_logits is not None:
            dl.copy_(d_logits.to(torch.float32).reshape(Bo, self.C))
        else:
            dl.zero_()
        if d_loss is not None:
            dl.add_(ws["dloss_logits"] * d_loss.to(torch.float32))
        return self._backward_from_dlogits(dl, B, S, mask, p_h, p_a, p_c, packed)

    def _backward_from_dlogits(self, dl, B, S, mask, p_h, p_a, p_c, packed=None):
        cfg, H, I, M = self.cfg, self.H, self.I, B * S
        Bo = self.head_rows(B, S, packed)
        ws = self.workspace(B, S, Bo)
        s = self.stream()
        rng = self.rng.data_ptr()
        w, g = self.w, self.g
        KM, MN = L.MAJOR_K, L.MAJOR_MN
        scratch, scratch_bytes = self.partials.data_ptr(), self.partials.numel()
        # torch.use_deterministic_algorithms: every sum of the backward in a fixed order.  The bias and LayerNorm
        # column sums leave the atomic epilogues / accumulators for column-sum passes on the weight-gradient stream,
        # the N = hidden dgrads run unsplit (one add onto what the LayerNorm backward left), dQ above 128 tokens
        # goes through per-key-block slices, and the word-embedding rows through the in-order owner scan.
        det = torch.are_deterministic_algorithms_enabled()
        if det:
            side_scratch, ln_parts = self.det_buffers()
            if S > 128 and ws.get("dq_parts") is None:
                ws["dq_parts"] = torch.empty(S // 128, M, H, dtype=torch.float32, device=self.dev)

        # embedding-table gradients are scatter targets: clear the whole bucket (word rows not in the batch, unused
        # position rows and padding must read as zero for the dense DDP/AdamW pass, like the reference's dense grads)
        eb, ee, _ = self.lay.buckets[0]
        L.call("b2_zero", self.grads.data_ptr() + 2 * eb, 2 * (ee - eb), s)

        x_last = ws["layers"][-1]["x2"] if self.nl > 0 else ws["emb_out"]
        # data gradient (d_hidden) on the main stream; the four head parameter gradients on the weight-gradient stream
        # (they belong to the last layer's bucket, whose readiness waits for that stream's marker of the layer anyway).
        # A model without encoder layers announces its head bucket right away: keep everything on one stream there.
        main = torch.cuda.current_stream(self.dev)
        side = self.wgrad_stream
        if self.nl > 0:
            # the side stream may still be busy with the previous step's tail; it must also not overtake this step
            side.wait_stream(main)
        if self.mlm:
            dec_done = self._mlm_backward(x_last, ws["dxA"], det, main, side)
        elif self.token_head:
            # every row of d_hidden is written: no memset
            L.call("b2_token_head_bwd_split", dl.data_ptr(), x_last.data_ptr(), M, H, w(self.cls_w), self.C,
                   p_c, rng, 1 + 3 * self.nl, g(self.cls_w), g(self.cls_b), ws["dxA"].data_ptr(),
                   ws["head_scratch"].data_ptr(), ws["head_scratch"].numel(), s,
                   side.cuda_stream if self.nl > 0 else None)
        else:
            head_g = (g("bert.pooler.dense.weight"), g("bert.pooler.dense.bias"), g("classifier.weight"),
                      g("classifier.bias"))
            L.call("b2_head_bwd_split", dl.data_ptr(), x_last.data_ptr(), ws["pooled"].data_ptr(),
                   None if packed is None else packed[1].data_ptr(), M, Bo, S, H, w("bert.pooler.dense.weight"),
                   w("classifier.weight"), self.C, p_c, rng, 1 + 3 * self.nl, *head_g, ws["dxA"].data_ptr(), 1,
                   ws["head_scratch"].data_ptr(), s, side.cuda_stream if self.nl > 0 else None)
        dx, dx_other = ws["dxA"], ws["dxB"]
        # Weight gradients are off the critical path (only the optimizer consumes them): they run on a second stream,
        # overlapping the dgrad / LayerNorm / attention chain of the main stream.  Their A operands (dzd, dU, dz1d,
        # dqkv) are double-buffered by layer parity; the main stream may reuse a buffer set only after the weight
        # gradients of the layer two steps earlier have drained (done[l + 2]).
        ss = side.cuda_stream
        done = {}

        # An armed step (a captured train step owns backward + optimizer) runs each bucket's share of the optimizer
        # step on the transport's side stream as soon as the bucket's gradients are final: opt.bucket_ready
        opt, transport = self.model._optimizer, self.transport
        per_bucket = opt is not None and opt._armed and transport.overlap
        # an accumulating / folding backward: per bucket on that stream too, else one whole-range launch in end_pass()
        if self._pass_op is not None and per_bucket:
            self._pass_stream = transport.side

        def bucket_ready(idx, wg_event=None):
            if per_bucket:
                opt.bucket_ready(idx, wg_event)

        if not self.lay.head_in_last_layer:
            bucket_ready(len(self.lay.buckets) - 1)     # (a model without encoder layers: the head is its own bucket)
        for l in reversed(range(self.nl)):
            a = ws["layers"][l]
            x_in = ws["layers"][l - 1]["x2"] if l > 0 else ws["emb_out"]
            pre = "bert.encoder.layer.%d." % l
            st = l & 1
            dzd, dU, dz1d, dqkv = ws["dzd"][st], ws["dU"][st], ws["dz1d"][st], ws["dqkv"][st]
            if (l + 2) in done:
                main.wait_event(done[l + 2])
            # --- BertOutput: LN2 backward (+ dropout mask, bias grad), FFN2 wgrad/dgrad(+GELU')
            acc_l = self.bias_acc.data_ptr() + 4 * l * self.acc_per_layer
            ln_out = (g(pre + "output.LayerNorm.weight"), g(pre + "output.LayerNorm.bias"), g(pre + "output.dense.bias"))
            ln_att = (g(pre + "attention.output.LayerNorm.weight"), g(pre + "attention.output.LayerNorm.bias"),
                      g(pre + "attention.output.dense.bias"))
            if det:
                # per-block partials; b2_colsum_finish on the weight-gradient stream turns them into the gradients
                n2 = ctypes.c_int32()
                L.call("b2_layernorm_bwd", dx.data_ptr(), None, a["z2"].data_ptr(), a["mean2"].data_ptr(),
                       a["rstd2"].data_ptr(), w(pre + "output.LayerNorm.weight"), M, H, p_h, rng, 3 + 3 * l, 1,
                       dx_other.data_ptr(), dzd.data_ptr(), *ln_out, ln_parts[st][0].data_ptr(),
                       ln_parts[st][0].numel(), ctypes.addressof(n2), s)
            else:
                # column sums (d_gamma, d_beta, d_bias) are added into this layer's fp32 accumulators by the kernel
                L.call("b2_layernorm_bwd_accum", dx.data_ptr(), a["z2"].data_ptr(), a["mean2"].data_ptr(),
                       a["rstd2"].data_ptr(), w(pre + "output.LayerNorm.weight"), M, H, p_h, rng, 3 + 3 * l,
                       dx_other.data_ptr(), dzd.data_ptr(), acc_l + 4 * (3 * H + I), s)
            # the layer's four weight gradients: collected here and issued as ONE launch on the side stream once the
            # last operand (dqkv) exists
            wgrads = []
            self.gemm(H, I, M, dzd.data_ptr(), H, MN, a["h"].data_ptr(), I, MN, g(pre + "output.dense.weight"), I,
                      split=True, defer=wgrads)
            # dU = (dY2 W2) * gelu'(u); its column sums (= intermediate bias gradient) accumulate in the same epilogue
            # (det: a b2_colsum of dU on the weight-gradient stream)
            self.gemm(M, I, H, dzd.data_ptr(), H, KM, w(pre + "output.dense.weight"), I, MN, dU.data_ptr(), I,
                      L.EPI_GELU_BWD, aux_in=a["u"].data_ptr(), ld_aux_in=I,
                      colsum=None if det else acc_l + 4 * 3 * H)
            # --- BertIntermediate
            self.gemm(I, H, M, dU.data_ptr(), I, MN, a["x1"].data_ptr(), H, MN,
                      g(pre + "intermediate.dense.weight"), H, split=True, defer=wgrads)
            # dX1 = dZ2 + dU W1: LayerNorm backward left dZ2 (fp32) in dx_other and the GEMM adds into it (split-K
            # slices reduce in place at L2)
            self.gemm(M, H, I, dU.data_ptr(), I, KM, w(pre + "intermediate.dense.weight"), H, MN,
                      dx_other.data_ptr(), H, L.EPI_ACCUM_F32, splits=1 if det else 0)
            # --- BertSelfOutput
            if det:
                n1 = ctypes.c_int32()
                L.call("b2_layernorm_bwd", dx_other.data_ptr(), None, a["z1"].data_ptr(), a["mean1"].data_ptr(),
                       a["rstd1"].data_ptr(), w(pre + "attention.output.LayerNorm.weight"), M, H, p_h, rng,
                       2 + 3 * l, 1, dx.data_ptr(), dz1d.data_ptr(), *ln_att, ln_parts[st][1].data_ptr(),
                       ln_parts[st][1].numel(), ctypes.addressof(n1), s)
            else:
                L.call("b2_layernorm_bwd_accum", dx_other.data_ptr(), a["z1"].data_ptr(), a["mean1"].data_ptr(),
                       a["rstd1"].data_ptr(), w(pre + "attention.output.LayerNorm.weight"), M, H, p_h, rng,
                       2 + 3 * l, dx.data_ptr(), dz1d.data_ptr(), acc_l + 4 * (6 * H + I), s)
            self.gemm(H, H, M, dz1d.data_ptr(), H, MN, a["ctx"].data_ptr(), H, MN,
                      g(pre + "attention.output.dense.weight"), H, split=True, defer=wgrads)
            self.gemm(M, H, H, dz1d.data_ptr(), H, KM, w(pre + "attention.output.dense.weight"), H, MN,
                      ws["dctx"].data_ptr(), H)
            # --- BertSelfAttention
            att_in = (a["qkv"].data_ptr(), L.ptr(mask) if packed is None else packed[0].data_ptr(),
                      a["ctx"].data_ptr(), ws["dctx"].data_ptr(), a["lse"].data_ptr())
            qkv_acc = None if det else acc_l     # det: the QKV bias gradient is a b2_colsum of dqkv
            if det and S > 128:
                L.call("b2_attention_bwd_ordered" if packed is None else "b2_attention_bwd_packed_seq_ordered",
                       *att_in, B, S, self.heads, 64, p_a, rng, 1 + 3 * l, dqkv.data_ptr(),
                       ws["dq_parts"].data_ptr(), s)
            elif packed is None:
                L.call("b2_attention_bwd", *att_in, B, S, self.heads, 64, p_a, rng, 1 + 3 * l,
                       dqkv.data_ptr(), L.ptr(ws["dq_accum"]), qkv_acc if S == 128 else None, L.ptr(a["keep"]), s)
            elif S == 128:
                L.call("b2_attention_bwd_packed", *att_in, B, self.heads, 64, p_a, rng, 1 + 3 * l,
                       dqkv.data_ptr(), qkv_acc, L.ptr(a["keep"]), s)
            else:
                L.call("b2_attention_bwd_packed_seq", *att_in, B, S, self.heads, 64, p_a, rng, 1 + 3 * l,
                       dqkv.data_ptr(), ws["dq_accum"].data_ptr(), None, None, s)
            if S != 128 and not det:   # longer sequences or bins: separate column-sum pass into the same accumulator slot
                L.call("b2_colsum", dqkv.data_ptr(), M, 3 * H, 3 * H, g(pre + "attention.self.query.bias"),
                       scratch, scratch_bytes, s)
            self.gemm(3 * H, H, M, dqkv.data_ptr(), 3 * H, MN, x_in.data_ptr(), H, MN,
                      g(pre + "attention.self.query.weight"), H, split=True, defer=wgrads)
            # fork: the side stream waits for every operand of the layer's weight gradients
            ev = torch.cuda.Event()
            ev.record(main)
            side.wait_event(ev)
            # 108 full-K 256x256 tiles (BERT-base) in two waves of one kernel instead of four small split-K GEMMs and
            # their reduce kernels; largest problems first
            wgrads.sort(key=lambda t: -(t.M * t.N))
            self.gemm_grouped(wgrads, ss)
            if det:
                # the layer's bias and LayerNorm gradients in a fixed order, off the critical path; the accumulators
                # stay untouched (zero), so there is nothing for b2_accum_finish to finish
                sb, sn = side_scratch.data_ptr(), side_scratch.numel()
                L.call("b2_colsum", dU.data_ptr(), M, I, I, g(pre + "intermediate.dense.bias"), sb, sn, ss)
                L.call("b2_colsum", dqkv.data_ptr(), M, 3 * H, 3 * H, g(pre + "attention.self.query.bias"), sb, sn,
                       ss)
                L.call("b2_colsum_finish", ln_parts[st][0].data_ptr(), n2.value, 3, H, *ln_out, ss)
                L.call("b2_colsum_finish", ln_parts[st][1].data_ptr(), n1.value, 3, H, *ln_att, ss)
            else:
                # fp32 accumulators -> bf16 bias gradients of this layer (and re-arm them); for S != 128 the QKV
                # segment's accumulator is unused (zero) and must not overwrite the colsum result: finish only the
                # intermediate one.  Every kernel that adds into this layer's accumulators is behind the fork above,
                # and only the optimizer / exchange reads the result: the launch rides the weight-gradient stream,
                # off the critical path.
                spl = self.segs_per_layer
                seg0 = spl * l if S == 128 else spl * l + 1
                L.call("b2_accum_finish", self.bias_acc.data_ptr(), self.grads.data_ptr(),
                       self.bias_segs.data_ptr() + 24 * seg0, spl * (l + 1) - seg0, max(3 * H, I), ss)
            done[l] = torch.cuda.Event()
            done[l].record(side)
            self.gemm(M, H, 3 * H, dqkv.data_ptr(), 3 * H, KM, w(pre + "attention.self.query.weight"), H, MN,
                      dx.data_ptr(), H, L.EPI_ACCUM_F32, splits=1 if det else 0)
            bucket_ready(1 + l, done[l])   # complete only with this layer's weight gradients
        emb_in = (dx.data_ptr(), 1, ws["emb_pre"].data_ptr(), ws["emb_mean"].data_ptr(), ws["emb_rstd"].data_ptr(),
                  w("bert.embeddings.LayerNorm.weight"), ws["ids32"].data_ptr(), ws["tt32"].data_ptr())
        emb_tail = (B, S, H, cfg.vocab_size, cfg.type_vocab_size,
                    -1 if getattr(cfg, "pad_token_id", None) is None else int(cfg.pad_token_id), p_h, rng, 0,
                    g("bert.embeddings.word_embeddings.weight"), g("bert.embeddings.position_embeddings.weight"),
                    g("bert.embeddings.token_type_embeddings.weight"), g("bert.embeddings.LayerNorm.weight"),
                    g("bert.embeddings.LayerNorm.bias"), ws["emb_dx"].data_ptr(), scratch, scratch_bytes,
                    self.owner.data_ptr(), s)
        emb_fn = "b2_embed_bwd" if packed is None else "b2_embed_bwd_packed"
        if det:
            emb_fn += "_ordered"
        if packed is None:
            L.call(emb_fn, *emb_in, *emb_tail)
        else:
            L.call(emb_fn, *emb_in, ws["pos32"].data_ptr(), *emb_tail)
        if self.mlm:
            # the tied decoder's dense part of the word-embedding gradient, on top of the scatter the embedding
            # backward stored (the pad row included: padding_idx only zeroes the scatter part)
            main.wait_event(dec_done)
            L.call("b2_mlm_tied_add", self._mlm_shared["dec"].data_ptr(), g("bert.embeddings.word_embeddings.weight"),
                   self.V * H, s)
        # Whoever consumes the gradients next on the main stream (optimizer.step, grad_dict) must see the weight-gradient
        # stream's work.  Where the per-bucket side stream has taken those dependencies, optimizer.step() (or
        # end_pass) joins it; in every other case join here.
        if not (per_bucket and transport.side_carries_wgrad):
            for l in sorted(done)[:2]:       # the last two layers processed (0 and 1) may still be in flight
                main.wait_event(done[l])
        bucket_ready(0)
