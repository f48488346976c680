"""HF-semantics ``AdamW``, torch-semantics ``SGD``, ``Adam`` and ``TorchAdamW``, and the reference's
``build_optimizer`` on top of the fused CUDA update.

Reference surface: ``build_optimizer(model, args)`` (multi-gpu-distributed-cls.py:100-111) returning an object with
``zero_grad()`` [:172] and ``step()`` [:174].  The arithmetic is transformers 4.28.1 ``optimization.py::AdamW.step``
(eps added to sqrt(v) before the bias correction, weight decay applied after the Adam update with the updated
weight, ``correct_bias=True``) — NOT ``torch.optim.AdamW``.  One kernel updates the whole flat parameter space
(or, under DDP, this rank's slice of every bucket, fused with the gradient mean over peers).  ``SGD`` is
``torch.optim.SGD`` (fabric-cls.py's ``Args.optim = "sgd"`` branch) on the same kernels' gradient path, and ``Adam`` /
``TorchAdamW`` are ``torch.optim.Adam`` / ``torch.optim.AdamW`` with ``fused=True`` (HF transformers 5.5's default).
"""
import copy
import itertools
import os

import torch

from . import _lib as L
from .ddp import _SLOT_BUCKET0, _SLOT_GRADS_READY, _SLOT_UPDATE_DONE

_uids = itertools.count()


class _FusedOptimizer(torch.optim.Optimizer):
    """What every optimizer of a b200 model does around its update kernels: the device state, the GradScaler hooks and
    the schedule of one optimizer step -- in which order, on which stream and over which element ranges accumulate,
    clip-reduce, update, barrier and advance run (``bucket_ready`` during backward, ``step()`` after it, the clip
    phases).  The schedule is written once; what differs between one GPU and a peer group it asks of the engine's
    transport (see modeling._LocalTransport).  A subclass supplies its hyperparameter struct, its state buffers and its
    two kernel forms."""
    # torch.cuda.amp.GradScaler contract for optimizers that unscale themselves (torch/amp/grad_scaler.py `step`):
    # the scaler sets `self.grad_scale` (device fp32 scalar) / `self.found_inf` around step() instead of walking
    # `.grad` tensors -- which do not exist here (gradients live in the bf16 bucket space).  This is what lets the
    # reference's -amp loop (multi-gpu-distributed-mp-amp-cls.py:166-171: autocast, scaler.scale(loss).backward(),
    # scaler.step(optimizer), scaler.update()) run unchanged.  bf16 has fp32's exponent range, so no overflow check
    # is needed: found_inf stays 0 and the scale only has to be divided out (exactly: it is a power of two).
    _step_supports_amp_scaling = True
    _shared_keys = ()     # the group hyperparameters besides lr that every group must share (one kernel, one value)
    _flat_keys = ()       # the subclass's state buffers over the flat space (peer-visible under DistributedDataParallel)

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        owners = {id(getattr(p, "_b2_owner", None)) for g in self.param_groups for p in g["params"]}
        first = self.param_groups[0]["params"][0]
        self._model = getattr(first, "_b2_owner", None)
        if self._model is None or len(owners) != 1:
            raise TypeError("this %s drives the fused CUDA update of ONE b200 BertForSequenceClassification; "
                            "got parameters that do not belong to such a model" % type(self).__name__)
        self._wd, self._decay_flags_cpu = self._group_rules(self.param_groups)
        self._dev_state = None
        # the step schedule's state.  _armed: set by a captured train step, bucket_ready may run during backward;
        # _pending: the buckets bucket_ready has already handled in this step (updated, or in a clipped step reduced)
        # on the transport's side stream; _clip = the clipped step in progress (None: the next step does not clip),
        # _clip_buf = its device buffers, kept across steps (captured graphs replay on them)
        self._armed = False
        self._pending = set()
        self._clip = None
        self._clip_buf = None
        # set by a captured train step for the duration of its body: the kernels read the lr from the device scalar
        # the step refreshes before every replay (see hparams), not the value passed at launch / capture
        self._lr_dev_on = False
        self._uid = next(_uids)
        self._model._optimizer = self
        self._model._optimizers.add(self)    # every optimizer's state follows the model into and out of a peer group
        if self._peer() is not None:
            self._state()       # under a peer group the allocation is collective: every rank is here

    def _group_rules(self, groups):
        """What a grouping of the parameters must satisfy (one kernel: the groups may differ only in weight_decay, and
        cover every parameter).  Returns (the one non-zero weight decay or 0, the decay flag of every 8 elements)."""
        g0 = groups[0]
        key = lambda g: (g["lr"],) + tuple(tuple(v) if isinstance(v, (list, tuple)) else v
                                           for v in (g[k] for k in self._shared_keys))
        for g in groups[1:]:
            if key(g) != key(g0):
                raise ValueError("param groups may differ only in weight_decay (as the reference's two groups do)")
        wds = sorted({float(g["weight_decay"]) for g in groups if g["weight_decay"] > 0})
        if len(wds) > 1:
            raise ValueError("at most one non-zero weight_decay value is supported")
        lay = self._model._layout
        covered = set()
        flags = torch.zeros(lay.total // 8, dtype=torch.uint8)
        for g in groups:
            for p in g["params"]:
                off, _shape = lay.entries[p._b2_name]
                covered.add(p._b2_name)
                if g["weight_decay"] > 0:
                    flags[off // 8:(off + (p.numel() + 7) // 8 * 8) // 8] = 1
        if covered != set(lay.entries):
            raise ValueError("the fused update steps every parameter of the model; %d of %d were passed"
                             % (len(covered), len(lay.entries)))
        return (wds[0] if wds else 0.0), flags

    # -- device state (step counter, lr slot, decay flags, and the subclass's buffers) -------------------------------
    def _peer(self):
        """the DistributedDataParallel wrapper (world > 1) whose peers map the state buffers, else None"""
        ddp = self._model._ddp
        return ddp if ddp is not None and ddp.world > 1 and ddp.comm is not None else None

    def _new_flat(self, key, zero=True):
        """an fp32 buffer over the flat space for the state `key`.  Under a peer group it is peer-visible memory, as the
        masters are, so that state_dict() can pull the slices other ranks update; that allocation is collective, so it
        happens only where every rank is: construction or wrap time, step() and its eager warm-ups, load_state_dict()."""
        n, dev = self._model._layout.total, self._model._engine.dev
        ddp = self._peer()
        if ddp is None:
            return (torch.zeros if zero else torch.empty)(n, dtype=torch.float32, device=dev)
        t = ddp.comm.alloc(self._peer_name(key), 4 * n).tensor(torch.float32, dev)
        return t.zero_() if zero else t

    def _peer_name(self, key):
        """this optimizer's name of the peer buffer of state `key`: every optimizer of a wrapped model has its own (the
        buffers of one that is dropped stay mapped until the wrapper closes)"""
        return "opt%d.%s" % (self._uid, key)

    def _ensure_lazy(self, stream):
        """creates the state buffers that come into use with an update (SGD's momentum, amsgrad's maximum); called
        where every rank of a peer group is, before the updates of a step"""

    def _share_state(self):
        """DistributedDataParallel (world > 1) wrapping the model: the state buffers move into peer-visible memory"""
        if self._dev_state is None or self._dev_state["dev"] != self._model._engine.dev:
            self._state()
            return
        st = self._dev_state
        for k in self._flat_keys:
            if st.get(k) is not None:
                st[k] = self._new_flat(k, zero=False).copy_(st[k])

    def _gather_state(self):
        """Under a peer group each rank updates only its slice of every bucket: pull the other slices of every state
        buffer out of their owners' copies (DistributedDataParallel._pull_slices, one-sided and safe between steps
        for the reason _gather_master gives)."""
        ddp = self._peer()
        if ddp is None or self._dev_state is None:
            return
        for k in self._flat_keys:
            if self._dev_state.get(k) is not None:
                ddp._pull_slices(self._peer_name(k), self._dev_state[k])

    def _unshare_state(self):
        """DistributedDataParallel.close(): private copies of the state buffers, every slice gathered, as the masters get"""
        if self._dev_state is None or self._peer() is None:
            return
        self._gather_state()
        for k in self._flat_keys:
            if self._dev_state.get(k) is not None:
                self._dev_state[k] = self._dev_state[k].clone()

    def _state(self):
        eng = self._model._engine
        if eng is None:
            raise RuntimeError("optimizer.step(): the model is not on CUDA")
        if self._dev_state is None or self._dev_state["dev"] != eng.dev:
            self._dev_state = {
                "dev": eng.dev,
                "step": torch.zeros(1, dtype=torch.int64, device=eng.dev),
                "lr": torch.zeros(1, dtype=torch.float64, device=eng.dev),           # a captured step's lr
                "decay": self._decay_flags_cpu.to(eng.dev),
            }
            self._init_state(self._dev_state, self._model._layout.total)
            self._prepare(eng.stream())
        return self._dev_state

    def _init_state(self, st, n):
        """adds the optimizer's own device buffers to the fresh state `st` (n = elements of the flat space)"""

    def _prepare(self, stream):
        """per-step device values the background kernel reads, for the NEXT update"""

    def flush_pending(self):
        """No-op: every update is applied within the step that produced its gradients, so none is ever left pending.
        Kept for callers that flush before reading the weights."""

    def current_lr(self):
        """The lr of the next update: param_groups' (a torch LR scheduler changes it between steps).  The update is
        one kernel over every parameter, so the groups must agree; they may differ only in weight_decay."""
        lr = self.param_groups[0]["lr"]
        for g in self.param_groups[1:]:
            if g["lr"] != lr:
                raise ValueError("param groups have different learning rates (%s); the fused update applies one lr to "
                                 "every parameter (a LambdaLR with one lambda per group can cause this)"
                                 % ", ".join(repr(x["lr"]) for x in self.param_groups))
        return float(lr)

    def hparams(self):
        hp = self._hparams()
        gs = getattr(self, "grad_scale", None)        # set by GradScaler.step() for the duration of step()
        hp.grad_scale = gs.data_ptr() if gs is not None else None
        if gs is not None and (gs.dtype != torch.float32 or not gs.is_cuda):
            raise TypeError("grad_scale must be a CUDA fp32 scalar (torch.cuda.amp.GradScaler's)")
        hp.found_inf = self._found_inf_ptr()
        if self._clip is not None and self._clip["final"]:
            hp.clip_coef = self._clip_buf["coef"].data_ptr()
        if self._lr_dev_on:
            hp.lr_dev = self._dev_state["lr"].data_ptr()
        return hp

    def _found_inf_ptr(self):
        """what skips the update: the GradScaler's flag, or in a clipped step the finalize's (which includes it)"""
        if self._clip is not None and self._clip["final"]:
            return self._clip_buf["skip"].data_ptr()
        return self._scaler_found_inf_ptr()

    def _scaler_found_inf_ptr(self):
        fi = getattr(self, "found_inf", None)         # GradScaler: 0-dim fp32 tensor (or int 0 when nothing was checked)
        if isinstance(fi, torch.Tensor):
            if fi.dtype != torch.float32 or not fi.is_cuda:
                raise TypeError("found_inf must be a CUDA fp32 scalar (torch.cuda.amp.GradScaler's)")
            self._found_inf_keep = fi                 # keep the tensor alive until the kernels that read it have run
            return fi.data_ptr()
        return None

    def zero_grad(self, set_to_none=True):
        """Gradients live in the bf16 bucket space and are overwritten by every backward: nothing to clear
        (the reference's zero_grad [:172] exists only because torch accumulates into .grad).  The one real `.grad`
        is the small fp32 probe the eager backward leaves on classifier.bias for GradScaler's inf check."""
        self._model._params_by_name[self._model._anchor].grad = None
        return None

    def update_range(self, begin, end, world, rank, peer_grads, peer_shadow, stream, background=False, grad_f32=None):
        """Fused (mean over peers +) update of flat elements [begin, end).  background=True (one GPU, the update of a
        bucket launched while the backward pass is still running): the form shaped to run beside the GEMM CTAs; with
        nothing left to hide behind (the last bucket, or a plain optimizer.step()) the 256-thread kernel is the faster
        one (5.2 vs 3.6 TB/s alone for AdamW).  In a clipped step the gradient is multiplied by the clip coefficient;
        grad_f32: the fp32 mean gradient of the slice (the clip stash) to read instead of the peers' bf16 gradients."""
        if os.environ.get("B2_DEBUG_SKIP_ADAMW") == "1":
            return      # MEASUREMENT ONLY (how much of the optimizer is exposed in the step): weights are not updated
        st = self._state()
        hp = self.hparams()
        hp.grad_f32 = grad_f32
        bg = background and world == 1 and hp.grad_scale is None and hp.found_inf is None and grad_f32 is None
        self._launch(st, hp, begin, end, world, rank, peer_grads, peer_shadow, stream, bg)

    def prepare_background(self, stream):
        """Before the first per-bucket background update of a step: the per-step values from the lr current now, not
        the one of the previous step() (a scheduler has stepped since)"""
        self._state()
        self._prepare(stream)

    def advance(self, stream):
        st = self._state()
        L.call("b2_step_advance", L.ptr(st["step"]), L.ptr(self._model._engine.rng), self._found_inf_ptr(), stream)
        self._prepare(stream)

    # -- the schedule of one optimizer step ----------------------------------------------------------------------------
    def _transport(self):
        return self._model._engine.transport

    def bucket_ready(self, idx, wg_event=None):
        """Called by the backward of an armed step: bucket `idx` holds this rank's final local gradients once the main
        stream reaches this point and `wg_event` (the weight-gradient stream's marker for the layer) has fired.  Its
        share of the step starts on the transport's side stream right away, so it hides behind the rest of backward.
        Only the SIDE stream waits for the weight gradients: the main stream's dgrad chain never parks behind them."""
        eng, t = self._model._engine, self._transport()
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(eng.dev))
        t.side.wait_event(ev)
        if wg_event is not None:
            t.side.wait_event(wg_event)
        s = t.side.cuda_stream
        op = eng._pass_op
        if op is not None:
            # gradient accumulation, on the local gradients of the whole bucket: an accumulating pass stops here (no
            # barrier, no exchange, no update); the final pass folds BEFORE the barrier, so peers read the window's sum
            b, e, _label = self._model._layout.buckets[idx]
            eng.accumulate_range(b, e, op, s)
            if op != L.ACCUM_FOLD:
                return
        if not self._pending:
            self._ensure_lazy(s)
        t.barrier(_SLOT_BUCKET0 + idx, s)
        if self._clip is not None:
            # a clipped step: only the reduce phase hides under the backward; no bucket may move before the norm of
            # the whole gradient is known (step() finalizes and updates)
            self._clip_reduce(idx, s)
        else:
            if t.background and not self._pending:
                self.prepare_background(s)      # the slim form reads the prepared values: those of this step's lr
            # with nothing left to hide behind (bucket 0, the last one produced) the full-size kernel is the faster one
            t.update(self, [idx], s, background=t.background and idx != 0)
        self._pending.add(idx)

    def _finish_step(self):
        """What step() still has to do after the backward: the clip's remaining reduces and its norm, the update of
        every bucket bucket_ready did not update, the step counter; with the side stream joined wherever it worked."""
        eng, t = self._model._engine, self._transport()
        main = torch.cuda.current_stream(eng.dev)
        buckets = range(len(self._model._layout.buckets))
        todo = [idx for idx in buckets if self._clip is not None or idx not in self._pending]
        # nothing left but the closing barrier and the counter: they may stay behind the updates on the side stream
        on_side = t.tail_on_side and not todo
        if self._pending and not on_side:
            main.wait_stream(t.side)
        s = (t.side if on_side else main).cuda_stream
        if self._clip is not None:
            # the reduce phase of every bucket neither bucket_ready nor clip_grad_norm_ has reduced, then the finalize
            # -- again when a GradScaler hands over its scale, since the norm clip_grad_norm_ returned was that of the
            # scaled gradients
            self._clip_reduce_rest(s)
            if not self._clip["final"] or getattr(self, "grad_scale", None) is not None:
                self._clip_finalize(s)
        elif todo:
            t.barrier(_SLOT_GRADS_READY, s)
        if todo:
            self._ensure_lazy(s)
            t.update(self, todo, s)
        t.barrier(_SLOT_UPDATE_DONE, s)
        self.advance(s)
        if on_side:
            main.wait_stream(t.side)
        self._pending = set()
        t.stepped()

    # -- gradient-norm clipping: reduce (+ partial sums of squares) per bucket, one norm, then the update -----------------
    def _clip_arm(self, max_norm):
        """Starts a clipped step: from here until step() no bucket is updated before the norm of the whole gradient is
        known.  The device buffers (and, in a peer group, the fp32 stash of this rank's slices) are allocated on first
        use."""
        if self._clip is not None:
            raise RuntimeError("clip_grad_norm_() called twice before optimizer.step(): the gradients of this step are "
                               "already clipped")
        max_norm = float(max_norm)
        if not max_norm > 0.0:
            raise ValueError("max_norm must be positive (got %r)" % max_norm)
        t = self._transport()
        ranges = [t.slice(idx) for idx in range(len(self._model._layout.buckets))]
        dev = self._model._engine.dev
        key = (t.world, t.rank, tuple(ranges), dev)
        if self._clip_buf is None or self._clip_buf["key"] != key:
            slot_off, stash_off, ns, nst = [], [], 0, 0
            for (b, e) in ranges:
                slot_off.append(ns)
                stash_off.append(nst)
                ns += L.sumsq_slots(max(0, e - b))
                nst += max(0, e - b)
            f32 = dict(dtype=torch.float32, device=dev)
            self._clip_buf = {
                "key": key, "ranges": ranges, "slot_off": slot_off, "stash_off": stash_off, "nslots": ns,
                "partials": torch.zeros(max(ns, 1), dtype=torch.float64, device=dev),
                "stash": torch.empty(max(nst, 8), **f32) if t.world > 1 else None,   # 4 B x total / world
                "norm": torch.zeros((), **f32), "coef": torch.ones((), **f32), "skip": torch.zeros((), **f32),
            }
        self._clip = {"max_norm": max_norm, "reduced": set(), "final": False}

    def clip_stash(self, idx):
        """in a clipped step of a peer group: the fp32 mean gradient of this rank's slice of bucket `idx`, which the
        reduce phase left for the update to read; else None"""
        buf = self._clip_buf
        if self._clip is None or buf["stash"] is None:
            return None
        return buf["stash"].data_ptr() + 4 * buf["stash_off"][idx]

    def _clip_reduce(self, idx, stream):
        """reduce phase of bucket `idx`: the mean over ranks of this rank's slice and its partial sums of squares"""
        buf = self._clip_buf
        b, e = buf["ranges"][idx]
        if e > b:
            sources = self._transport().grad_sources(idx, stream)
            L.call("b2_grad_reduce_sumsq", L.ptr_array(sources), len(sources), self.clip_stash(idx), b, e,
                   buf["partials"].data_ptr() + 8 * buf["slot_off"][idx], stream)
        self._clip["reduced"].add(idx)

    def _clip_reduce_rest(self, stream):
        """the reduce phase of every bucket not reduced yet, behind the barrier that makes every rank's gradients final"""
        todo = [idx for idx in range(len(self._clip_buf["ranges"])) if idx not in self._clip["reduced"]]
        if todo:
            self._transport().barrier(_SLOT_GRADS_READY, stream)
        for idx in todo:
            self._clip_reduce(idx, stream)

    def _clip_finalize(self, stream):
        """the norm and the coefficient (collective in a peer group).  Inside a GradScaler step it divides by the scale, so
        the norm is that of the unscaled gradients, and a non-finite norm skips the step like GradScaler's inf check."""
        buf, t = self._clip_buf, self._transport()
        scratch, flags, slot, epoch = t.norm_exchange()
        gs = getattr(self, "grad_scale", None)
        L.call("b2_grad_norm_finalize", buf["partials"].data_ptr(), buf["nslots"], scratch, flags, t.world, t.rank, slot,
               epoch, self._clip["max_norm"], L.ptr(gs), self._scaler_found_inf_ptr(), buf["norm"].data_ptr(),
               buf["coef"].data_ptr(), buf["skip"].data_ptr(), stream)
        self._clip["final"] = True

    def clip_now(self, max_norm):
        """The eager clip_grad_norm_: flush an open accumulation window, reduce every bucket, finalize; step() then runs
        the update with the coefficient.  Returns the device norm buffer."""
        eng = self._model._engine
        if self._pending:
            raise RuntimeError("clip_grad_norm_(): this step's update already ran during backward (the optimizer is "
                               "armed by a FusedTrainStep); clip through the captured step's max_grad_norm instead")
        s = torch.cuda.current_stream(eng.dev).cuda_stream
        eng.flush_accum(s)
        self._clip_arm(max_norm)
        self._clip_reduce_rest(s)
        self._clip_finalize(s)
        return self._clip_buf["norm"]

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        self.current_lr()
        model = self._model
        eng = model._engine
        if eng is None:
            raise RuntimeError("optimizer.step(): the model is not on CUDA")
        # every pass of an accumulation window ran inside no_sync(): apply the accumulator (torch applies its .grad)
        eng.flush_accum(torch.cuda.current_stream(eng.dev).cuda_stream)
        self._finish_step()
        self._clip = None
        model._grads_live = False
        # the inf-check probe has served its purpose (GradScaler reads it before calling step); the -amp scripts never
        # call zero_grad, so drop it here or it would accumulate
        model._params_by_name[model._anchor].grad = None
        return loss

    def _views(self, flat):
        """`flat` (indexed like the flat parameter space) as views by HF parameter name"""
        out = {}
        for name, p in self._model._params_by_name.items():
            off, shape = self._model._layout.entries[name]
            out[name] = flat[off:off + p.numel()].view(shape)
        return out

    # -- checkpoint: torch's state_dict format over the flat device buffers ----------------------------------------------
    def state_dict(self):
        """torch's format: ``{"state": {i: {...}}, "param_groups": [{..., "params": [i, ...]}]}``, the parameters
        numbered in param_groups order as torch numbers them.  The per-parameter tensors are views into the device
        state buffers (torch also returns live references); ``Optimizer.state`` itself stays empty.  The state is empty
        before the first update, as torch's is.  Under DistributedDataParallel with world > 1 the call is one-sided, as
        ``model.state_dict()`` is: this rank pulls the slices other ranks update out of their memory."""
        for pre_hook in self._optimizer_state_dict_pre_hooks.values():
            pre_hook(self)
        groups, idx = [], 0
        for g in self.param_groups:        # torch's pack_group
            packed = {k: v for k, v in g.items() if k != "params"}
            packed["params"] = list(range(idx, idx + len(g["params"])))
            idx += len(g["params"])
            groups.append(packed)
        sd = {"state": {}, "param_groups": groups}
        if self._dev_state is not None:
            self._gather_state()
            entries = self._export(self._dev_state, int(self._dev_state["step"]))
            if entries:
                idx = 0
                for g in self.param_groups:
                    for p in g["params"]:
                        sd["state"][idx] = entries(p._b2_name)
                        idx += 1
        for post_hook in self._optimizer_state_dict_post_hooks.values():
            out = post_hook(self, sd)
            if out is not None:
                sd = out
        return sd

    def load_state_dict(self, state_dict):
        """Loads a dict of ``state_dict()``'s format -- this class's, or the stock torch class's it restates.  torch's
        checks first, then the group rules of the constructor; the tensors are copied into the existing device buffers
        in place, so a captured train step replays on the loaded state.  Under DistributedDataParallel every rank must
        call it (it may allocate a buffer the dict carries, collectively).  torch's load pre- and post-hooks run."""
        state_dict = state_dict.copy()
        for pre_hook in self._optimizer_load_state_dict_pre_hooks.values():
            out = pre_hook(self, state_dict)
            if out is not None:
                state_dict = out
        groups = self.param_groups
        saved = copy.deepcopy(state_dict["param_groups"])
        if len(groups) != len(saved):
            raise ValueError("loaded state dict has a different number of parameter groups")
        if any(len(g["params"]) != len(s["params"]) for g, s in zip(groups, saved)):
            raise ValueError("loaded state dict contains a parameter group that doesn't match the size of optimizer's "
                             "group")
        names, new_groups = {}, []
        for g, s in zip(groups, saved):
            for p, i in zip(g["params"], s["params"]):
                names[i] = p._b2_name
            s["params"] = g["params"]
            if "param_names" in g and "param_names" not in s:
                s["param_names"] = g["param_names"]
            for k, v in self.defaults.items():      # (as torch's subclasses' __setstate__ fill in newer keys)
                s.setdefault(k, v)
            new_groups.append(s)
        wd, flags = self._group_rules(new_groups)
        state = {names[i]: v for i, v in state_dict["state"].items() if i in names and v}
        if state and len(state) != len(names):
            raise ValueError("the loaded state covers %d of %d parameters: the fused update keeps one state for all of "
                             "them" % (len(state), len(names)))
        step = self._loaded_step(state)
        self._check_loaded(state, step, new_groups[0])
        shapes = {p._b2_name: tuple(p.shape) for g in groups for p in g["params"]}
        for name, entry in state.items():
            for key, v in entry.items():
                if isinstance(v, torch.Tensor) and key != "step" and tuple(v.shape) != shapes[name]:
                    raise ValueError("loaded state %r of %s has shape %s, the parameter %s"
                                     % (key, name, tuple(v.shape), shapes[name]))
        if state and self._model._engine is None:
            raise RuntimeError("load_state_dict: the optimizer state lives on the GPU; call model.cuda() before "
                               "loading a state with steps")
        self.param_groups = new_groups
        self._wd, self._decay_flags_cpu = wd, flags
        if self._model._engine is None:
            self._dev_state = None       # (created from the loaded groups' decay flags by the first step)
        else:
            st = self._state()
            st["decay"].copy_(flags)
            with torch.no_grad():
                self._import(st, state, step)
            self._prepare(self._model._engine.stream())
        for post_hook in self._optimizer_load_state_dict_post_hooks.values():
            post_hook(self)

    def _loaded_step(self, state):
        """the one step count of the loaded per-parameter states (int, float or tensor), 0 without state"""
        steps = set()
        for name, entry in state.items():
            v = entry.get("step")
            if v is None:
                continue
            x = float(v.item() if isinstance(v, torch.Tensor) else v)
            if x != int(x) or x < 0:
                raise ValueError("loaded state of %s has step %r; a step count is a non-negative integer" % (name, v))
            steps.add(int(x))
        if len(steps) > 1:
            raise ValueError("the loaded parameters disagree on step (%s): the fused update keeps one step count"
                             % sorted(steps))
        return steps.pop() if steps else 0

    def _check_loaded(self, state, step, group):
        """raises before anything is changed when the loaded per-parameter states lack what this update needs"""
        first = None
        for name, entry in state.items():
            for key in self._required:
                if key not in entry:
                    raise ValueError("loaded state of %s has no %r" % (name, key))
            have = sorted(k for k in self._flat_keys if k in entry)
            if first is None:
                first = have
            elif have != first:
                raise ValueError("the loaded parameters disagree on which state they have (%s: %s, others: %s): the "
                                 "fused update keeps one set of buffers" % (name, have, first))

    def _load_flat(self, st, key, state):
        """the loaded per-parameter `key` tensors into the flat buffer st[key] (created if the dict carries it and it
        does not exist yet), in place, its 8-element padding zeroed; a buffer the dict does not carry is zeroed"""
        if st.get(key) is None:
            if not state or key not in next(iter(state.values())):
                return
            st[key] = self._new_flat(key, zero=False)
        buf = st[key]
        buf.zero_()
        if state:
            views = self._views(buf)
            for name, entry in state.items():
                views[name].copy_(entry[key])


class AdamW(_FusedOptimizer):
    _shared_keys = ("betas", "eps", "correct_bias")
    _flat_keys = ("exp_avg", "exp_avg_sq")
    _required = ("step", "exp_avg", "exp_avg_sq")

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, correct_bias=True,
                 no_deprecation_warning=True):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr} - should be >= 0.0")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter: {betas[0]} - should be in [0.0, 1.0)")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter: {betas[1]} - should be in [0.0, 1.0)")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps} - should be >= 0.0")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, correct_bias=correct_bias)
        super().__init__(params, defaults)

    def _init_state(self, st, n):
        st["exp_avg"] = self._new_flat("exp_avg")
        st["exp_avg_sq"] = self._new_flat("exp_avg_sq")
        st["step_size"] = torch.zeros(1, dtype=torch.float32, device=st["dev"])   # see b2_adamw_prepare

    def _export(self, st, step):
        """transformers 4.28.1 AdamW.step's state of a parameter: step (a python int), exp_avg, exp_avg_sq"""
        if step == 0:
            return None
        m, v = self._views(st["exp_avg"]), self._views(st["exp_avg_sq"])
        return lambda name: {"step": step, "exp_avg": m[name], "exp_avg_sq": v[name]}

    def _import(self, st, state, step):
        for key in self._flat_keys:
            self._load_flat(st, key, state)
        st["step"].fill_(step)

    def _prepare(self, stream):
        """bias-corrected step size of the NEXT update -> device float (read by the background kernel)"""
        st = self._dev_state
        L.call("b2_adamw_prepare", self.hparams(), L.ptr(st["step"]), L.ptr(st["step_size"]), stream)

    def captured_hparams(self):
        """The hyperparameters a captured step bakes into its graph (all but the lr, which it reads at every replay)"""
        return {"betas": tuple(tuple(float(b) for b in g["betas"]) for g in self.param_groups),
                "eps": tuple(float(g["eps"]) for g in self.param_groups),
                "weight_decay": tuple(float(g["weight_decay"]) for g in self.param_groups),
                "correct_bias": tuple(bool(g["correct_bias"]) for g in self.param_groups)}

    def _hparams(self):
        g = self.param_groups[0]
        hp = L.AdamWHParams()
        hp.lr, hp.beta1, hp.beta2, hp.eps = float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"])
        hp.weight_decay = float(self._wd)
        hp.correct_bias = 1 if g["correct_bias"] else 0
        return hp

    def _launch(self, st, hp, begin, end, world, rank, peer_grads, peer_shadow, stream, background):
        flat = self._model._flat
        if background:
            # one GPU: the form that fits beside the GEMM CTAs (csrc/optim.cu, slim_update_kernel)
            L.call("b2_adamw_background", peer_grads[0], peer_shadow[0], L.ptr(flat), L.ptr(st["exp_avg"]),
                   L.ptr(st["exp_avg_sq"]), L.ptr(st["decay"]), begin, end, hp, L.ptr(st["step_size"]), stream)
            return
        L.call("b2_bucket_reduce_adamw", L.ptr_array(peer_grads), L.ptr_array(peer_shadow), world, rank,
               L.ptr(flat), L.ptr(st["exp_avg"]), L.ptr(st["exp_avg_sq"]), L.ptr(st["decay"]), begin, end,
               hp, L.ptr(st["step"]), stream)

    def moments(self):
        """(exp_avg, exp_avg_sq) fp32 by HF parameter name — for tests/checkpoint tooling (every slice gathered under
        a peer group, as in state_dict())."""
        st = self._state()
        self._gather_state()
        m, v = self._views(st["exp_avg"]), self._views(st["exp_avg_sq"])
        return {name: (m[name], v[name]) for name in m}


class SGD(_FusedOptimizer):
    """``torch.optim.SGD`` (torch 2.11: momentum, dampening, coupled weight decay, Nesterov, maximize) as one fused
    update over the flat parameter space, on every path AdamW runs: the eager loop, the captured steps and DDP.

    The stock ``torch.optim.SGD`` cannot train a b200 model: its gradients live in the model's bf16 bucket space, not
    in ``.grad``.  The momentum buffer is allocated when the first step with ``momentum != 0`` runs; as in torch, that
    step sets it to the gradient.  ``foreach``, ``fused`` and ``differentiable=False`` are accepted and ignored."""
    _shared_keys = ("momentum", "dampening", "nesterov", "maximize")
    _flat_keys = ("momentum_buffer",)
    _required = ()

    def __init__(self, params, lr=1e-3, momentum=0, dampening=0, weight_decay=0, nesterov=False, *, maximize=False,
                 foreach=None, differentiable=False, fused=None):
        if isinstance(lr, torch.Tensor) and lr.numel() != 1:
            raise ValueError("Tensor lr must be 1-element")
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if differentiable:
            raise ValueError("differentiable=True is not supported: the update is a fused kernel outside autograd")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov,
                        maximize=maximize, foreach=foreach, differentiable=differentiable, fused=fused)
        if nesterov and (momentum <= 0 or dampening != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        super().__init__(params, defaults)

    def _init_state(self, st, n):
        st["momentum_buffer"] = None     # allocated by the first step with momentum (torch: `momentum_buffer is None`)

    def _ensure_lazy(self, stream):
        """When the momentum buffer comes into use the step count restarts at 0 on `stream`, the stream of the update
        about to read it: that update initialises the buffer from the gradient."""
        st = self._state()
        if float(self.param_groups[0]["momentum"]) != 0.0 and st["momentum_buffer"] is None:
            st["momentum_buffer"] = self._new_flat("momentum_buffer", zero=False)
            L.call("b2_zero", L.ptr(st["step"]), 8, stream)

    def _buffer(self, st, stream):
        """the momentum buffer, or None without momentum"""
        if float(self.param_groups[0]["momentum"]) == 0.0:
            return None
        self._ensure_lazy(stream)
        return st["momentum_buffer"]

    def _export(self, st, step):
        """torch.optim.SGD's state of a parameter: momentum_buffer once it exists (nothing without momentum)"""
        if st["momentum_buffer"] is None or step == 0:
            return None
        views = self._views(st["momentum_buffer"])
        return lambda name: {"momentum_buffer": views[name]}

    def _import(self, st, state, step):
        self._load_flat(st, "momentum_buffer", state)
        # the device step only decides whether the next update initialises the buffer from the gradient (step 0):
        # torch's `momentum_buffer is None`.  A loaded buffer is used; without one the next update starts it afresh.
        carried = bool(state) and "momentum_buffer" in next(iter(state.values()))
        st["step"].fill_(1 if carried else 0)

    def captured_hparams(self):
        """The hyperparameters a captured step bakes into its graph (all but the lr, which it reads at every replay)"""
        return {"momentum": tuple(float(g["momentum"]) for g in self.param_groups),
                "dampening": tuple(float(g["dampening"]) for g in self.param_groups),
                "weight_decay": tuple(float(g["weight_decay"]) for g in self.param_groups),
                "nesterov": tuple(bool(g["nesterov"]) for g in self.param_groups),
                "maximize": tuple(bool(g["maximize"]) for g in self.param_groups)}

    def _hparams(self):
        g = self.param_groups[0]
        if g["nesterov"] and (g["momentum"] <= 0 or g["dampening"] != 0):
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")
        hp = L.SGDHParams()
        hp.lr, hp.momentum, hp.dampening = float(g["lr"]), float(g["momentum"]), float(g["dampening"])
        hp.weight_decay = float(self._wd)
        hp.nesterov, hp.maximize = (1 if g["nesterov"] else 0), (1 if g["maximize"] else 0)
        return hp

    def _launch(self, st, hp, begin, end, world, rank, peer_grads, peer_shadow, stream, background):
        flat = self._model._flat
        buf = self._buffer(st, stream)
        if background:
            L.call("b2_sgd_background", peer_grads[0], peer_shadow[0], L.ptr(flat), L.ptr(buf), L.ptr(st["decay"]),
                   begin, end, hp, L.ptr(st["step"]), stream)
            return
        L.call("b2_bucket_reduce_sgd", L.ptr_array(peer_grads), L.ptr_array(peer_shadow), world, rank, L.ptr(flat),
               L.ptr(buf), L.ptr(st["decay"]), begin, end, hp, L.ptr(st["step"]), stream)

    def momentum_buffers(self):
        """fp32 momentum buffers by HF parameter name, or {} while there is none (momentum 0, or no step yet) — the
        counterpart of AdamW.moments(), for tests and tooling."""
        buf = self._state()["momentum_buffer"]
        self._gather_state()
        return {} if buf is None else self._views(buf)


class Adam(_FusedOptimizer):
    """``torch.optim.Adam`` (torch 2.11: coupled or decoupled weight decay, amsgrad, maximize) as one fused update over
    the flat parameter space, on every path AdamW runs: the eager loop, the captured steps and DDP.  The arithmetic is
    that of ``fused=True`` (HF transformers 5.5's default ``"adamw_torch_fused"``), bit for bit on the same gradient.

    The stock ``torch.optim.Adam`` / ``AdamW`` cannot train a b200 model: its gradients live in the model's bf16 bucket
    space, not in ``.grad``.  ``foreach``, ``fused`` and ``capturable`` are accepted and ignored (the update is always
    fused and capturable); ``differentiable=True`` raises.  The max_exp_avg_sq buffer is created by the first update
    with ``amsgrad`` set; turning amsgrad on after an update has run raises at ``step()``."""
    _shared_keys = ("betas", "eps", "amsgrad", "maximize", "decoupled_weight_decay")
    _flat_keys = ("exp_avg", "exp_avg_sq", "max_exp_avg_sq")
    _required = ("step", "exp_avg", "exp_avg_sq")

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None,
                 maximize=False, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False):
        # torch 2.11's checks, in its order, with its messages
        if isinstance(lr, torch.Tensor):
            if foreach and not capturable:
                raise ValueError("lr as a Tensor is not supported for capturable=False and foreach=True")
            if lr.numel() != 1:
                raise ValueError("Tensor lr must be 1-element")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if not ((isinstance(betas[0], float) and isinstance(betas[1], float))
                or (isinstance(betas[0], torch.Tensor) and isinstance(betas[1], torch.Tensor))):
            raise ValueError("betas must be either both floats or both Tensors")
        for i in (0, 1):
            if isinstance(betas[i], torch.Tensor):
                if not capturable and foreach:
                    raise ValueError(f"betas[{i}] as a Tensor is not supported for capturable=False and foreach=True")
                if betas[i].numel() != 1:
                    raise ValueError(f"Tensor betas[{i}] must be 1-element")
        if fused:
            if differentiable:
                raise RuntimeError("`fused` does not support `differentiable`")
            if foreach:
                raise RuntimeError("`fused` and `foreach` cannot be `True` together.")
        if differentiable:
            raise ValueError("differentiable=True is not supported: the update is a fused kernel outside autograd")
        if isinstance(betas[0], torch.Tensor):
            raise ValueError("Tensor betas are not supported: the fused update takes the betas by value")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                        maximize=maximize, foreach=foreach, capturable=capturable, differentiable=differentiable,
                        fused=fused, decoupled_weight_decay=decoupled_weight_decay)
        self._updated = False    # an update has run on this state: amsgrad can no longer be turned on
        super().__init__(params, defaults)

    def _group_rules(self, groups):
        wd, flags = super()._group_rules(groups)
        # torch's kernel forms the L2 term by the lane an element takes in its loop (see b2_adam_hparams_t): a tensor
        # whose size is not a multiple of 4 goes through its unaligned loop, where element j is in lane (j % 2048) / 512
        lay = self._model._layout
        for name, (off, shape) in lay.entries.items():
            n = self._model._params_by_name[name].numel()
            if n % 4:
                j = torch.arange(0, n, 8)
                bits = L.ADAM_DECAY_UNALIGNED + L.ADAM_DECAY_LANE0 * ((j % 2048) < 512).to(torch.uint8)
                seg = flags[off // 8:off // 8 + len(j)]
                seg |= seg * bits      # on decayed vectors only
        return wd, flags

    def _init_state(self, st, n):
        st["exp_avg"] = self._new_flat("exp_avg")
        st["exp_avg_sq"] = self._new_flat("exp_avg_sq")
        # with amsgrad on from the start the buffer comes with the state; turned on later, with the first update that
        # reads it (see _ensure_lazy)
        st["max_exp_avg_sq"] = self._new_flat("max_exp_avg_sq") if self.param_groups[0]["amsgrad"] else None
        self._updated = False
        st["prepared"] = torch.zeros(2, dtype=torch.float32, device=st["dev"])   # see b2_adam_prepare

    def _ensure_lazy(self, stream):
        st = self._state()
        if self.param_groups[0]["amsgrad"] and st["max_exp_avg_sq"] is None and not self._updated:
            # before any update (never inside a capture: the captured steps run eager passes first).  After one,
            # _hparams raises.
            st["max_exp_avg_sq"] = self._new_flat("max_exp_avg_sq")
            torch.cuda.current_stream(st["dev"]).synchronize()     # zeroed before another stream's update reads it

    def _export(self, st, step):
        """torch.optim.Adam / AdamW's state of a parameter: step (0-dim fp32), exp_avg, exp_avg_sq, and
        max_exp_avg_sq once amsgrad has run"""
        if step == 0:
            return None
        bufs = [(k, self._views(st[k])) for k in self._flat_keys if st.get(k) is not None]
        return lambda name: dict([("step", torch.tensor(float(step), dtype=torch.float32))]
                                 + [(k, v[name]) for k, v in bufs])

    def _check_loaded(self, state, step, group):
        super()._check_loaded(state, step, group)
        if group["amsgrad"] and step > 0 and "max_exp_avg_sq" not in next(iter(state.values())):
            raise ValueError("amsgrad is on but the loaded state has no max_exp_avg_sq after %d steps: the buffer would "
                             "start from zero mid-run (as when amsgrad is turned on after the first step)" % step)

    def _import(self, st, state, step):
        self._load_flat(st, "exp_avg", state)
        self._load_flat(st, "exp_avg_sq", state)
        carried = bool(state) and "max_exp_avg_sq" in next(iter(state.values()))
        if carried or self.param_groups[0]["amsgrad"]:
            self._load_flat(st, "max_exp_avg_sq", state)
        else:
            st["max_exp_avg_sq"] = None         # as in torch: no amsgrad state without amsgrad having run
        st["step"].fill_(step)
        self._updated = step > 0

    def _prepare(self, stream):
        """the bias corrections of the NEXT update -> device floats (read by the background kernel)"""
        st = self._dev_state
        L.call("b2_adam_prepare", self.hparams(), L.ptr(st["step"]), L.ptr(st["prepared"]), stream)

    def captured_hparams(self):
        """The hyperparameters a captured step bakes into its graph (all but the lr, which it reads at every replay)"""
        return {"betas": tuple(tuple(float(b) for b in g["betas"]) for g in self.param_groups),
                "eps": tuple(float(g["eps"]) for g in self.param_groups),
                "weight_decay": tuple(float(g["weight_decay"]) for g in self.param_groups),
                "amsgrad": tuple(bool(g["amsgrad"]) for g in self.param_groups),
                "maximize": tuple(bool(g["maximize"]) for g in self.param_groups),
                "decoupled_weight_decay": tuple(bool(g["decoupled_weight_decay"]) for g in self.param_groups)}

    def _hparams(self):
        g = self.param_groups[0]
        st = self._dev_state
        if g["amsgrad"] and st is not None and st["max_exp_avg_sq"] is None and self._updated:
            # torch fails here too (a KeyError on the missing state entry)
            raise ValueError("amsgrad was turned on after the first step: the max_exp_avg_sq buffer would start "
                             "from zero mid-run; build the optimizer with amsgrad=True")
        hp = L.AdamHParams()
        hp.lr, hp.beta1, hp.beta2, hp.eps = float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"])
        hp.weight_decay = float(self._wd)
        hp.amsgrad, hp.maximize = (1 if g["amsgrad"] else 0), (1 if g["maximize"] else 0)
        hp.decoupled = 1 if g["decoupled_weight_decay"] else 0
        return hp

    def _launch(self, st, hp, begin, end, world, rank, peer_grads, peer_shadow, stream, background):
        flat = self._model._flat
        if hp.amsgrad:
            self._ensure_lazy(stream)
        vmax = st["max_exp_avg_sq"] if hp.amsgrad else None
        self._updated = True
        if background:
            L.call("b2_adam_background", peer_grads[0], peer_shadow[0], L.ptr(flat), L.ptr(st["exp_avg"]),
                   L.ptr(st["exp_avg_sq"]), L.ptr(vmax), L.ptr(st["decay"]), begin, end, hp, L.ptr(st["prepared"]),
                   stream)
            return
        L.call("b2_bucket_reduce_adam", L.ptr_array(peer_grads), L.ptr_array(peer_shadow), world, rank, L.ptr(flat),
               L.ptr(st["exp_avg"]), L.ptr(st["exp_avg_sq"]), L.ptr(vmax), L.ptr(st["decay"]), begin, end, hp,
               L.ptr(st["step"]), stream)

    moments = AdamW.moments

    def max_exp_avg_sqs(self):
        """amsgrad's fp32 max_exp_avg_sq by HF parameter name, or {} without amsgrad"""
        buf = self._state()["max_exp_avg_sq"]
        self._gather_state()
        return {} if buf is None else self._views(buf)


class TorchAdamW(Adam):
    """``torch.optim.AdamW`` (torch 2.11: decoupled weight decay, default 0.01) on the fused update; see ``Adam``.
    Exported under this name because the package's ``AdamW`` is the reference's HF AdamW, whose arithmetic differs
    (eps before the bias correction, decay after the update)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, *,
                 maximize=False, foreach=None, capturable=False, differentiable=False, fused=None):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, foreach=foreach, maximize=maximize,
                         capturable=capturable, differentiable=differentiable, fused=fused,
                         decoupled_weight_decay=True)


def clip_grad_norm_(parameters, max_norm, norm_type=2.0, error_if_nonfinite=False, foreach=None):
    """``torch.nn.utils.clip_grad_norm_`` for a b200 model: call it between ``backward()`` and ``optimizer.step()``.

    torch's own function cannot be used: the gradients live in the model's bf16 bucket space, not in ``.grad``, so it
    would see only the 6-float probe on ``classifier.bias`` and clip nothing else.  This one computes the 2-norm of the
    gradient the next ``optimizer.step()`` applies (an open ``no_sync()`` window is flushed first) and makes that step
    multiply the gradient by ``min(1, max_norm / (norm + 1e-6))`` (torch's coefficient).

    ``parameters`` must be every parameter of one b200 model (``model.parameters()``, wrapped or not).  Returns the
    total norm as a 0-dim fp32 CUDA tensor without a host sync; ``error_if_nonfinite=True`` syncs and raises
    ``RuntimeError`` on a non-finite norm, and the step is then not clipped.  ``foreach`` is accepted and ignored.

    Under ``DistributedDataParallel`` with world > 1 it is the norm of the DDP-mean gradient, the one torch DDP clips,
    and the call is collective: every rank must make it, and every rank gets the same norm bit for bit.  Under a
    GradScaler step (the package Trainer's ``use_amp``) ``step()`` recomputes the norm from the unscaled gradients."""
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    params = list(parameters)
    if float(norm_type) != 2.0:
        raise ValueError("clip_grad_norm_: only norm_type=2 is supported (got %r)" % (norm_type,))
    owners = {id(getattr(p, "_b2_owner", None)) for p in params}
    model = getattr(params[0], "_b2_owner", None) if params else None
    if model is None or len(owners) != 1:
        raise TypeError("clip_grad_norm_: the parameters must all belong to ONE b200 BertForSequenceClassification")
    names = {p._b2_name for p in params}
    if names != set(model._layout.entries):
        raise ValueError("clip_grad_norm_: clipping covers the whole gradient of the model; pass every parameter "
                         "(%d of %d were passed)" % (len(names), len(model._layout.entries)))
    if model._engine is None:
        raise RuntimeError("clip_grad_norm_: the model is not on CUDA (there is no CPU path): call model.cuda() first")
    opt = model._optimizer
    if opt is None:
        raise RuntimeError("clip_grad_norm_: the clip is applied by the model's optimizer inside optimizer.step(); build "
                           "the optimizer first")
    norm = opt.clip_now(max_norm)
    if error_if_nonfinite and not bool(torch.isfinite(norm)):
        opt._clip = None
        raise RuntimeError("The total norm of order 2.0 for gradients from `parameters` is non-finite, so it cannot be "
                           "clipped. To disable this error and scale the gradients by the non-finite norm anyway, set "
                           "`error_if_nonfinite=False`")
    return norm.clone()


def build_optimizer(model, args):
    """Same grouping rule as the reference (multi-gpu-distributed-cls.py:100-111): no weight decay for names
    containing 'bias' or 'LayerNorm.weight'; lr = args.learning_rate; HF AdamW defaults otherwise.

    ``args.optim = "sgd"`` (fabric-cls.py's default, :281-285) gives that script's optimizer instead:
    ``SGD(model.parameters(), lr=args.learning_rate)``, one group, no momentum and no weight decay.

    ``args.optim = "adamw_torch"`` or ``"adamw_torch_fused"`` (HF TrainingArguments' names; the second is transformers
    5.5's default) gives ``TorchAdamW`` on the same two groups, torch's defaults otherwise (eps 1e-8)."""
    optim = getattr(args, "optim", "adamw")
    if optim == "sgd":
        return SGD(model.parameters(), lr=args.learning_rate)
    if optim not in ("adamw", "adamw_torch", "adamw_torch_fused"):
        raise ValueError("args.optim must be 'adamw', 'adamw_torch', 'adamw_torch_fused' or 'sgd' (got %r)"
                         % (optim,))
    no_decay = ['bias', 'LayerNorm.weight']
    optimizer_grouped_parameters = [
        {'params': [p for n, p in model.named_parameters() if not any(nd in n for nd in no_decay)],
         'weight_decay': args.weight_decay},
        {'params': [p for n, p in model.named_parameters() if any(nd in n for nd in no_decay)],
         'weight_decay': 0.0}
    ]
    if optim != "adamw":
        return TorchAdamW(optimizer_grouped_parameters, lr=args.learning_rate, weight_decay=args.weight_decay)
    optimizer = AdamW(optimizer_grouped_parameters, lr=args.learning_rate)
    return optimizer
