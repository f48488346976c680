"""The stream schedule of one training step: every pair of conflicting accesses on different streams must be ordered
by a recorded happens-before, decided from a log of the step alone.

A step runs on up to five streams: the body stream (the captured steps' high-priority stream, else the caller's),
the engine's weight-gradient stream, the transport's side stream (the per-bucket accumulate, clip-reduce and
update of an armed step), the weight-stream fork inside b2_head_bwd_split / b2_token_head_bwd_split, and the host,
which refills the pinned staging buffers.  Their ordering rests on hand-placed record / wait_event / wait_stream /
synchronize calls.  The stage test (test_step_stages.py) serialises the device around every launch and cannot see
them; a bitwise comparison sees a race only if it fires in that run.

Log.  StepLog records, in program order and without synchronising anything:
  - every library call (_lib.call replaced): the entry point, its stream and every pointer argument.  Each
    *_head_bwd_split call becomes a main-stream part, the fork the C++ code does (record on the main stream, wait
    on the weight stream: head.cu / token_head.cu), and a weight-stream part, with the arguments split as the two
    .cu files split them (HEAD_SPLIT);
  - every torch op on a CUDA or pinned tensor (a TorchDispatchMode): its tensors, the current stream, and which
    tensors it writes (the schema's alias info, plus the tensors it returns new).  An op on pinned host memory
    alone runs on the host; a blocking copy between host and device, or a scalar read, joins the host to its stream;
  - torch.cuda.Event.record / wait / synchronize, Stream.synchronize and torch.cuda.synchronize (wait_event and
    wait_stream reach Event.wait).  A CUDA graph runs its captured work as one unit where it is replayed: the end of
    a capture is logged as a record of the graph on the capture stream, a replay as a wait for it on the replay
    stream.  Every entry keeps its call site in the package, which the planted defects name.

Memory model.  After the log, every pointer resolves by address to a region of the step: what register_step
(test_step_stages.py) registers, the per-layer slices of bias_acc, the optimizer's flat state and scalars, the clip
buffers, the accumulator, and the staging buffers (host and device).  Roles come from include/b2_ddp_bert.h
(parse_header): a const pointer is a read, any other pointer a read + write, `*stream` parameters are skipped; the
GemmArgs, hyperparameter and loss-parameter structs and the pointer arrays have small tables.  Inside the flat spaces
(gradients, shadow and master weights, moments, momentum, amsgrad maximum, accumulator) extents are exact: a pointer
at a parameter span's start (Q | K | V one span; the masked-LM word table and bias at their vocab_pad reserve) covers
that span, the optimizer / accumulate / sum-of-squares / zero / cast / copy entry points cover their own range, and
b2_accum_finish its decoded segments; any other flat-space pointer fails as unmodelled.  Every other region counts
as one unit.  A library pointer in no region fails, except a temporary a logged torch op made (the dense masked-LM
labels, the GradScaler's scale and found_inf): a temporary must stay on the stream that made it.

Check.  Vector clocks per stream and one for the host: an enqueue joins the host's clock into the stream's, a
record copies the stream's clock into the event, a wait joins the event's most recent record at that point of the
log into the stream, a synchronize joins into the host.  Every pair of accesses on different streams that overlap,
one a write, must be ordered; a failure names both entries (entry point and log position) with their streams, the
region, the element range and RAW / WAR / WAW.

Recorded.  Captured steps (FusedTrainStep, PackedTrainStep, armed per bucket): the two eager warm-up bodies back
to back (the same schedule, unserialised, so hazards across steps show) and the capture call, whose body becomes one
graph; sequence, token and masked-LM heads with deterministic algorithms off and on, HF AdamW, TorchAdamW,
Adam(amsgrad), SGD(momentum, nesterov), max_grad_norm, accum_steps 2 (STORE, ADD and FOLD bodies), an lr schedule,
padded 512 and packed 128 / 512 tokens, and a model without encoder layers (its head is its own bucket).  Eager
paths over two steps: autograd + optimizer.step(), clip_grad_norm_, the GradScaler loop, a no_sync() window of two,
a world-1 DistributedDataParallel wrapper, and Trainer.train_step on the staged captured step.  Peer transports at
world > 1 are out of scope: their barriers are cross-device flags, not stream events.

Planted defects, each one edge deleted from a recorded log (the library is unchanged), each failing with its region
and kind: the fork before the top layer's grouped weight-gradient GEMM (RAW on its parity set), the parity-reuse
wait on done[l + 2] (WAR), bucket_ready's wait on the weight-gradient marker (RAW on a gradient span the update
reads), the wait on dec_done before the tied add (RAW on mlm.dec), _finish_step's join of the side stream (the
pending update against the next step), b2_head_bwd_split's internal fork (RAW on head_scratch, where the main part
leaves dropout(pooled) and the logits' gradient terms for the weight part), and the host's wait on _h2d_done
before refilling the pinned staging buffer (WAR on stage.h).  The optimizer's device state is created before a
captured case's log: its creation copies the decay flags with a blocking copy, a host synchronise that would
otherwise order the second step's refill behind the first step's copy.

Part B, the optimizer stage of a captured step at lr > 0 against the step's own gradients: after the warm-ups and
the capture, two replays under an lr schedule (LambdaLR, a new lr every step).  Before each, a snapshot of the master,
the optimizer state, the step counter, the dropout rng and the lr stage() is about to stage; after it, the gradient
space holds what the update read.  Expected: TorchAdamW and Adam (with and without amsgrad) bitwise torch's
_fused_adamw_ / _fused_adam_, SGD(momentum, nesterov, decay) bitwise torch.optim.SGD, HF AdamW at
test_step_kernels.AdamWRef's bound (both run on the decayed and the other elements as two parameters, as
test_torch_adam / test_sgd do); with max_grad_norm the norm within 1e-6 of float64 (test_clip's bound), the
coefficient torch's formula bitwise and that one coefficient applied to every bucket; with accum_steps 2 the FOLD
left bf16(accumulator + g) in the gradient space.  Everywhere: shadow == bf16(master) bitwise, the step counter and
rng[1] one up, the device lr slot this replay's staged lr.  Planted on the reference side, each must fail: the
previous replay's lr, bucket 1's gradients from the previous replay, the step count one too high.

Findings: no hazard in the library.  Every recorded log was ordered; the one report while this file was written
was the log's own (the loss read after a replay, before the log modelled the replay).

Measured on an H100 80GB HBM3 (700 W power limit), `pytest -m gpu tests/test_step_schedule.py`: 44 tests in 21-26 s
as pytest counts it (three runs); the first takes 12-13 s, mostly CUDA start-up, every other one under 1 s.  Ordered
cross-stream conflicting pairs of the warm-up logs: 636-1104 per captured case with encoder layers (8628 with
accumulation), 156 and 184 without; 740-3280 on the eager paths.
"""
import ctypes
import linecache
import os
import re
import sys
from collections import defaultdict

import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode

from parity import b2, tiny_config
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import _Layout
from test_clip import _torch_coef
from test_packing import short_batch
from test_packing_long import long_batch
from test_step_kernels import AdamWRef, within
from test_step_stages import Regions, WORD, register_step, reserved_spans
from token_oracle import token_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b2_ddp_bert.h")
PKG = os.path.dirname(os.path.abspath(b2.__file__))
HOST = "host"
R, RW = "r", "rw"
SEED = 20261018

# ======================================================================================================================
# roles: the C header
# ======================================================================================================================
STRUCTS = {"b2_gemm_args_t": "gemm", "b2_adamw_hparams_t": "hparams", "b2_sgd_hparams_t": "hparams",
           "b2_adam_hparams_t": "hparams", "b2_loss_params_t": "loss_params"}
STRUCT_ROLES = {
    "gemm": {"A": R, "B": R, "bias": R, "aux_in": R, "rng_state": R,
             "D": RW, "aux_out": RW, "colsum_out": RW, "workspace": RW},
    "hparams": {"grad_scale": R, "found_inf": R, "clip_coef": R, "grad_f32": R, "lr_dev": R},
    "loss_params": {"weight": R, "pos_weight": R},
}
HOST_POINTERS = {("b2_layernorm_bwd", "deferred_nparts")}     # a host int32 the call fills (the partial-row count)


def classify(fn, pname, ptype):
    """the role of one header parameter: None (a value), 'skip' (a stream), 'host', r / rw (a pointer), r[] / rw[]
    (an array of pointers), or a struct table's name"""
    if pname.endswith("stream"):
        return "skip"
    if (fn, pname) in HOST_POINTERS:
        return "host"
    for s, role in STRUCTS.items():
        if s in ptype:
            return role
    stars = ptype.count("*") + ptype.count("[")
    if stars == 0:
        return None
    const = ptype.startswith("const")
    if stars >= 2:
        return "r[]" if const else "rw[]"
    return R if const else RW


def parse_header(text):
    """entry point -> [(parameter name, role)] of every int32_t b2_* declaration"""
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    out = {}
    for m in re.finditer(r"int32_t\s+(b2_\w+)\s*\(([^;{]*?)\)\s*;", text):
        name, params = m.group(1), m.group(2)
        roles = []
        for p in params.split(","):
            p = " ".join(p.split())
            if p in ("", "void"):
                continue
            arr = re.search(r"\[[^\]]*\]$", p)
            core = p[:arr.start()].strip() if arr else p
            pname = re.findall(r"(\w+)$", core)[0]
            ptype = core[:len(core) - len(pname)].strip() + ("[" if arr else "")
            roles.append((pname, classify(name, pname, ptype)))
        out[name] = roles
    return out


_ROLES = None


def roles():
    global _ROLES
    if _ROLES is None:
        with open(HEADER) as f:
            _ROLES = parse_header(f.read())
    return _ROLES


# the two split head backwards: parameter index -> role of the main-stream part and of the weight-stream part
# (head.cu head_bwd_impl: k1 reads dlogits, pooled, cls_w and the rng and fills scratch (its second plane is
# dropout(pooled)); the memset and k3 write d_hidden from scratch, pool_w and cls_rows; on the weight stream k1b reads
# dlogits and scratch into d_cls_w / d_cls_b, k2 scratch, hidden_states and cls_rows into d_pool_w / d_pool_b.
# token_head.cu: the data kernel reads dlogits, cls_w and the rng into d_hidden; on the weight stream the partial
# kernel reads dlogits, hidden_states and the rng into scratch, the finish kernel scratch into d_cls_w / d_cls_b)
HEAD_SPLIT = {
    "b2_head_bwd_split": ({0: R, 2: R, 3: R, 8: R, 9: R, 12: R, 18: RW, 20: RW},
                          {0: R, 1: R, 3: R, 14: RW, 15: RW, 16: RW, 17: RW, 20: R}, 21, 22, "head.cu"),
    "b2_token_head_bwd_split": ({0: R, 4: R, 7: R, 11: RW},
                                {0: R, 1: R, 7: R, 9: RW, 10: RW, 12: RW}, 14, 15, "token_head.cu"),
}

# ======================================================================================================================
# the log
# ======================================================================================================================
class Entry:
    """one log entry: kind 'launch' / 'op' (accesses on `stream`), 'record' / 'wait' (event `ev` on `stream`),
    'ev_sync' / 'stream_sync' / 'device_sync' (the host waits)"""

    def __init__(self, kind, name, stream=None, ev=None, site=""):
        self.kind, self.name, self.stream, self.ev, self.site = kind, name, stream, ev, site
        self.acc = []           # (key, address or byte range (lo, hi), write, torch tensor extent?)
        self.scal = {}          # the call's value arguments by header name
        self.idx = None


def call_site():
    """'file:line: source' of the innermost package frame calling into the log; None inside torch.cuda.graph's own
    entry and exit (its generator-state bookkeeping, which no kernel of the step touches)"""
    f = sys._getframe(2)
    while f is not None:
        fn = f.f_code.co_filename
        if fn.endswith(GRAPHS_PY):
            return None
        if fn.startswith(PKG):
            line = linecache.getline(fn, f.f_lineno).strip()
            return "%s:%d: %s" % (os.path.basename(fn), f.f_lineno, line)
        f = f.f_back
    return "(outside the package)"


def tensors_of(v):
    if isinstance(v, torch.Tensor):
        return [v]
    if isinstance(v, (list, tuple)):
        return [t for x in v for t in tensors_of(x)]
    return []


def byte_range(t):
    if t.numel() == 0:
        return None
    span = 1 + sum((s - 1) * abs(st) for s, st in zip(t.shape, t.stride()))
    lo = t.data_ptr()
    return lo, lo + span * t.element_size()


def pinned(t):
    return t.device.type == "cpu" and t.is_pinned()


COPIES = ("copy_", "_to_copy", "_copy_from", "_copy_from_and_resize")
GRAPHS_PY = os.path.join("torch", "cuda", "graphs.py")
_VIEWLESS = {"empty", "empty_strided", "empty_like", "new_empty", "new_empty_strided", "record_stream", "set_",
             "resize_"}


class _OpMode(TorchDispatchMode):
    def __init__(self, log):
        super().__init__()
        self.log = log

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        out = func(*args, **kwargs)
        self.log.op(func, args, kwargs, out)
        return out


class StepLog:
    """records one or more steps; see the module docstring"""

    def __init__(self):
        self.entries = []
        self.events = []            # keeps every logged event alive: ids stay unique
        self.temps = []             # (entry index, lo, hi) of tensors a logged torch op returned new

    def add(self, e):
        e.idx = len(self.entries)
        self.entries.append(e)
        return e

    def sync(self, kind, ev=None, stream=None, site=None):
        if ev is not None:
            self.events.append(ev)
        self.add(Entry(kind, kind, stream, None if ev is None else id(ev), site or call_site() or "torch.cuda.graph"))

    # ---- library calls ----------------------------------------------------------------------------------------------
    def call(self, name, *args):
        rl = roles().get(name)
        if rl is None or len(rl) != len(args):
            raise AssertionError("%s: no header declaration with %d parameters" % (name, len(args)))
        site = call_site()
        if name in HEAD_SPLIT:
            main_r, wgt_r, si, wi, cu = HEAD_SPLIT[name]
            s, ws = args[si], args[wi]
            ws = s if ws is None else ws
            self.launch(name, args, rl, s, main_r, site + " [main part]")
            if ws != s:
                key = object()
                self.events.append(key)
                self.add(Entry("record", "record", s, id(key), "%s: the fork of %s: cudaEventRecord" % (cu, name)))
                self.add(Entry("wait", "wait", ws, id(key), "%s: the fork of %s: cudaStreamWaitEvent" % (cu, name)))
            self.launch(name, args, rl, ws, wgt_r, site + " [weight part]")
            return
        streams = [a for a, (_p, r) in zip(args, rl) if r == "skip"]
        self.launch(name, args, rl, streams[0], None, site)

    def launch(self, name, args, rl, stream, only, site):
        e = Entry("launch", name, stream, site=site)
        for i, (a, (pname, role)) in enumerate(zip(args, rl)):
            if only is not None:
                role = only.get(i) if role not in (None, "skip") else role
            if role is None:
                if isinstance(a, (int, float)):
                    e.scal[pname] = a
                continue
            if role in ("skip", "host") or a is None:
                continue
            if role in (R, RW):
                if a:
                    e.acc.append((pname, int(a), role == RW, False))
            elif role in ("r[]", "rw[]"):
                n = len(a) if hasattr(a, "__len__") else 0
                for j in range(n):
                    if a[j]:
                        e.acc.append(("%s[%d]" % (pname, j), int(a[j]), role == "rw[]", False))
            else:
                table = STRUCT_ROLES[role]
                items = [a] if not hasattr(a, "__len__") else [a[j] for j in range(args[1])]
                for j, st in enumerate(items):
                    pre = "" if len(items) == 1 else "p%d." % j
                    for f, fr in table.items():
                        v = getattr(st, f)
                        if v:
                            e.acc.append((pre + f, int(v), fr == RW, False))
        self.add(e)

    # ---- torch ops --------------------------------------------------------------------------------------------------
    def op(self, func, args, kwargs, out):
        schema = func._schema
        base = schema.name.split("::")[-1]
        if base in _VIEWLESS or any(r.alias_info is not None and not r.alias_info.is_write for r in schema.returns):
            return
        acc, cpu, cuda = [], False, False
        capturing = torch.cuda.is_current_stream_capturing()     # (no host memory is touched inside a capture)
        for i, a in enumerate(schema.arguments):
            v = args[i] if i < len(args) else kwargs.get(a.name)
            w = a.alias_info is not None and a.alias_info.is_write
            for t in tensors_of(v):
                acc.append((t, w))
        ins = {t.untyped_storage().data_ptr() for t, _w in acc if t.device.type != "meta"}
        new = [t for t in tensors_of(out) if t.untyped_storage().data_ptr() not in ins]
        acc += [(t, True) for t in new]
        keep = []
        for t, w in acc:
            if t.is_cuda:
                cuda = True
            elif t.device.type == "cpu":
                cpu = True
                if capturing or not pinned(t):
                    continue
            else:
                continue
            br = byte_range(t)
            if br is not None:
                keep.append((t, br, w))
        if base == "_local_scalar_dense":
            self.sync("stream_sync", stream=torch.cuda.current_stream().cuda_stream, site="scalar read " + call_site())
            return
        site = call_site()
        if not keep or site is None:
            return
        stream = torch.cuda.current_stream().cuda_stream if cuda else HOST
        e = Entry("op", "aten." + base, stream, site=site)
        for t, br, w in keep:
            e.acc.append(("tensor", br, w, True))
        self.add(e)
        for t in new:
            br = byte_range(t)
            if br is not None and (t.is_cuda or pinned(t)):
                self.temps.append((e.idx, br[0], br[1]))
        nb = kwargs.get("non_blocking", args[2] if base == "copy_" and len(args) > 2 else False)
        if cuda and cpu and base in COPIES and not nb:
            self.sync("stream_sync", stream=stream, site="blocking copy " + call_site())

    # ---- recording --------------------------------------------------------------------------------------------------
    def __enter__(self):
        log = self
        ev_record, ev_wait, ev_sync = torch.cuda.Event.record, torch.cuda.Event.wait, torch.cuda.Event.synchronize
        st_sync, dev_sync, call = torch.cuda.Stream.synchronize, torch.cuda.synchronize, L.call
        cap_end, replay = torch.cuda.CUDAGraph.capture_end, torch.cuda.CUDAGraph.replay

        def record(ev, stream=None):
            s = stream if stream is not None else torch.cuda.current_stream()
            log.sync("record", ev, s.cuda_stream)
            return ev_record(ev, stream)

        def wait(ev, stream=None):
            s = stream if stream is not None else torch.cuda.current_stream()
            log.sync("wait", ev, s.cuda_stream)
            return ev_wait(ev, stream)

        def synchronize(ev):
            log.sync("ev_sync", ev)
            return ev_sync(ev)

        def stream_synchronize(s):
            log.sync("stream_sync", stream=s.cuda_stream)
            return st_sync(s)

        def device_synchronize(device=None):
            log.sync("device_sync")
            return dev_sync(device)

        # a graph runs its captured work as one unit on the stream it is replayed on: the end of the capture records
        # the graph like an event, a replay waits for it
        def capture_end(g):
            out = cap_end(g)
            log.sync("record", g, torch.cuda.current_stream().cuda_stream, "capture end")
            return out

        def graph_replay(g):
            log.sync("wait", g, torch.cuda.current_stream().cuda_stream, "graph replay")
            return replay(g)

        def lib_call(name, *args):
            log.call(name, *args)
            return call(name, *args)

        self._saved = (ev_record, ev_wait, ev_sync, st_sync, dev_sync, call, cap_end, replay)
        torch.cuda.CUDAGraph.capture_end, torch.cuda.CUDAGraph.replay = capture_end, graph_replay
        torch.cuda.Event.record, torch.cuda.Event.wait, torch.cuda.Event.synchronize = record, wait, synchronize
        torch.cuda.Stream.synchronize, torch.cuda.synchronize, L.call = stream_synchronize, device_synchronize, lib_call
        self._mode = _OpMode(self)
        self._mode.__enter__()
        return self

    def __exit__(self, *exc):
        self._mode.__exit__(*exc)
        (torch.cuda.Event.record, torch.cuda.Event.wait, torch.cuda.Event.synchronize, torch.cuda.Stream.synchronize,
         torch.cuda.synchronize, L.call, torch.cuda.CUDAGraph.capture_end, torch.cuda.CUDAGraph.replay) = self._saved
        return False


# ======================================================================================================================
# the memory model
# ======================================================================================================================
OPT_RANGE = ("b2_adamw_background", "b2_bucket_reduce_adamw", "b2_sgd_background", "b2_bucket_reduce_sgd",
             "b2_adam_background", "b2_bucket_reduce_adam", "b2_grad_accumulate", "b2_grad_reduce_sumsq")
FLAT_KEYS = ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "momentum_buffer")


class Memory:
    """the regions of a recorded step: flat spaces (exact element extents), parameter spans (their starts), and
    one-unit regions (test_step_stages.Regions, the narrowest containing range wins)"""

    def __init__(self):
        self.flats = []             # (name, lo, hi, element size)
        self.spans = {}             # (flat name, begin) -> (span name, n)
        self.units = Regions()
        self.segs = None            # (bias_segs address, rows [[a_off, g_off, n]], bias_acc address)

    # register_step's interface
    def register(self, name, t, kind):
        if t is None or not t.numel():
            return
        if name.startswith(("g:", "w:")):
            flat = "grads" if name.startswith("g:") else "shadow"
            base = [f for f in self.flats if f[0] == flat][0]
            self.spans[(flat, (t.data_ptr() - base[1]) // base[3])] = (name, t.numel())
            return
        self.units.add(name, t, kind)

    def flat(self, name, t):
        if t is not None:
            self.flats.append((name, t.data_ptr(), t.data_ptr() + t.numel() * t.element_size(), t.element_size()))

    def find_flat(self, addr):
        for f in self.flats:
            if f[1] <= addr < f[2]:
                return f
        return None


def engine_memory(eng, opt=None, step=None, inputs=(), extra=()):
    """the Memory of a recorded step: register_step over the engine's workspace, plus the optimizer's state, the clip
    buffers, the accumulator, the staging buffers and `extra` (name, tensor) pairs"""
    mem = Memory()
    model = eng.model
    mem.flat("grads", eng.grads)
    mem.flat("shadow", eng.shadow)
    mem.flat("master", model._flat)
    mem.flat("accum", eng.accum)
    st = opt._dev_state if opt is not None else None
    if st is not None:
        for k in FLAT_KEYS:
            mem.flat(k, st.get(k))
    wss = list(eng._ws.values())
    assert len(wss) == 1, "one workspace per recorded step"
    register_step(mem, eng, wss[0], dict(inputs))
    for l in range(eng.nl):
        p = eng.acc_per_layer
        mem.units.add("bias_acc.%d" % l, eng.bias_acc[l * p:(l + 1) * p], "acc")
    mem.segs = (eng.bias_segs.data_ptr(), eng.bias_segs.cpu().tolist(), eng.bias_acc.data_ptr())
    if st is not None:
        for k in ("step", "lr", "decay", "step_size", "prepared"):
            mem.units.add("opt." + k, st.get(k), "state")
    cb = opt._clip_buf if opt is not None else None
    if cb is not None:
        for k in ("partials", "norm", "coef", "skip", "stash"):
            mem.units.add("clip." + k, cb.get(k), "state")
    if step is not None:
        mem.units.add("stage.h", step._h_stage_all, "host")
        mem.units.add("stage.d", step._d_stage_all, "in")
        mem.units.add("loss_out", step.loss_out, "out")
        mem.units.add("h_loss", step.h_loss, "host")
        mem.units.add("mlm_dloss", getattr(step, "_mlm_dloss", None), "in")
    for k, t in extra:
        mem.units.add(k, t, "in")
    return mem


class Unmodelled(AssertionError):
    pass


def flat_ranges(e, key, off, esize, mem):
    """[(lo, hi)] of a library pointer at element `off` of a flat space (see the module docstring)"""
    n, sc = e.name, e.scal
    if n in OPT_RANGE:
        return [(sc["begin"], sc["end"])]
    if n == "b2_zero" or n == "b2_copy_async":
        return [(off, off + sc["bytes"] // esize)]
    if n in ("b2_cast_f32_to_bf16", "b2_cast_bf16_to_f32"):
        return [(off, off + sc["n"])]
    if n == "b2_accum_finish" and key == "dst":
        segs_addr, rows, _acc = mem.segs
        seg0 = (e.seg_ptr - segs_addr) // 24
        return [(rows[seg0 + j][1], rows[seg0 + j][1] + rows[seg0 + j][2]) for j in range(sc["n_segments"])]
    return None


class Access:
    __slots__ = ("e", "key", "region", "lo", "hi", "write", "stream", "epoch", "clock")

    def __init__(self, e, key, region, lo, hi, write):
        self.e, self.key, self.region, self.lo, self.hi, self.write = e, key, region, lo, hi, write


def resolve(log, mem):
    """every access of the log as Access objects; raises on a pointer in no region or an unmodelled flat pointer"""
    out = []
    temps = sorted(log.temps, key=lambda t: t[0])
    for e in log.entries:
        if e.kind not in ("launch", "op"):
            continue
        if e.name == "b2_accum_finish":
            e.seg_ptr = dict((k, a) for k, a, _w, _t in e.acc)["segments"]
        for key, a, w, is_t in e.acc:
            lo_b, hi_b = a if is_t else (a, a + 1)
            f = mem.find_flat(lo_b)
            if f is not None:
                name, base, _hi, es = f
                off = (lo_b - base) // es
                if is_t:
                    rng = [(off, (min(hi_b, f[2]) - base + es - 1) // es)]
                else:
                    rng = flat_ranges(e, key, off, es, mem)
                    if rng is None:
                        span = mem.spans.get((name, off))
                        if span is None:
                            raise Unmodelled("%s #%d (%s): %s points at element %d of %s, which starts no parameter "
                                             "span and is not its own range: unmodelled" % (e.name, e.idx, e.site, key,
                                                                                            off, name))
                        rng = [(off, off + span[1])]
                for lo, hi in rng:
                    out.append(Access(e, key, name, lo, hi, w))
                continue
            if e.name == "b2_accum_finish" and key == "src":
                _sa, rows, acc = mem.segs
                seg0 = (e.seg_ptr - _sa) // 24
                for j in range(e.scal["n_segments"]):
                    reg, _o = mem.units.find(acc + 4 * rows[seg0 + j][0])
                    out.append(Access(e, key, reg, 0, 1, w))
                continue
            if mem.units.covers(lo_b):
                reg, _o = mem.units.find(lo_b)
                out.append(Access(e, key, reg, 0, 1, w))
                continue
            made = [t for t in temps if t[0] <= e.idx and t[1] <= lo_b < t[2]]
            if not made:
                raise AssertionError("%s #%d (%s): %s = 0x%x maps to no region of the step" % (e.name, e.idx, e.site,
                                                                                             key, lo_b))
            out.append(Access(e, key, "temp@%d" % made[-1][0], 0, 1, w))
    return out


# ======================================================================================================================
# the check: vector clocks
# ======================================================================================================================
def join(a, b):
    for k, v in b.items():
        if a.get(k, 0) < v:
            a[k] = v


def clocks(entries):
    """entry index -> (stream, epoch, clock snapshot) of every launch / op"""
    vc = defaultdict(dict)
    events = {}
    out = {}
    for e in entries:
        if e.kind in ("launch", "op"):
            s = e.stream
            if s != HOST:
                join(vc[s], vc[HOST])
            vc[s][s] = vc[s].get(s, 0) + 1
            out[e.idx] = (s, vc[s][s], dict(vc[s]))
        elif e.kind == "record":
            join(vc[e.stream], vc[HOST])
            events[e.ev] = dict(vc[e.stream])
        elif e.kind == "wait":
            join(vc[e.stream], vc[HOST])
            join(vc[e.stream], events.get(e.ev, {}))
        elif e.kind == "ev_sync":
            join(vc[HOST], events.get(e.ev, {}))
        elif e.kind == "stream_sync":
            join(vc[HOST], vc[e.stream])
        elif e.kind == "device_sync":
            for s in list(vc):
                join(vc[HOST], vc[s])
    return out


class Result:
    def __init__(self):
        self.hazards, self.ordered, self.streams = [], 0, set()


def check(entries, accesses, names=None):
    """the unordered conflicting pairs of `accesses` under the clocks of `entries`"""
    names = names or {}
    sname = lambda s: names.get(s, HOST if s == HOST else "stream 0x%x" % s)
    ck = clocks(entries)
    res = Result()
    by_region = defaultdict(list)
    for a in accesses:
        if a.e.idx not in ck:
            continue            # (an entry deleted from the log)
        a.stream, a.epoch, a.clock = ck[a.e.idx]
        by_region[a.region].append(a)
        res.streams.add(a.stream)
    for reg, accs in by_region.items():
        if reg.startswith("temp@") and len({a.stream for a in accs}) > 1:
            res.hazards.append("temporary %s (made by entry %s) used on %s" % (
                reg, reg[5:], ", ".join(sorted(sname(a.stream) for a in accs))))
            continue
        accs.sort(key=lambda a: a.e.idx)
        writes = [a for a in accs if a.write]
        seen = set()
        for w in writes:
            for o in accs:
                if o.stream == w.stream or o.e.idx == w.e.idx or not (o.lo < w.hi and w.lo < o.hi):
                    continue
                a, b = (w, o) if w.e.idx < o.e.idx else (o, w)
                pair = (id(a), id(b))
                if pair in seen:
                    continue
                seen.add(pair)
                if b.clock.get(a.stream, 0) >= a.epoch:
                    res.ordered += 1
                    continue
                kind = "WAW" if a.write and b.write else "RAW" if a.write else "WAR"
                res.hazards.append(
                    "%s on %s [%d, %d): %s #%d (%s, %s) on %s and %s #%d (%s, %s) on %s are unordered" % (
                    kind, reg, max(a.lo, b.lo), min(a.hi, b.hi), a.e.name, a.e.idx, a.key, a.e.site, sname(a.stream),
                    b.e.name, b.e.idx, b.key, b.e.site, sname(b.stream)))
    return res


def assert_ordered(res, what):
    if res.hazards:
        raise AssertionError("%s: %d unordered conflicting pairs; first: %s" % (what, len(res.hazards),
                                                                               "\n".join(res.hazards[:4])))


def drop(entries, site_text, nth=0):
    """the log without the nth entry whose call site contains `site_text`"""
    hits = [e for e in entries if site_text in e.site]
    assert len(hits) > nth, "no entry at %r in the log" % site_text
    gone = hits[nth]
    return [e for e in entries if e is not gone]


# ======================================================================================================================
# CPU: the engine on synthetic logs, the header, the extents
# ======================================================================================================================
def synth(*ops):
    """a log from ('L', stream, region, 'r'|'w') / ('R', stream, ev) / ('W', stream, ev) / ('E', ev) / ('S', stream) /
    ('D',) tuples"""
    log = StepLog()
    acc = []
    for op in ops:
        k = op[0]
        if k == "L":
            e = log.add(Entry("launch", "k%d" % len(log.entries), op[1]))
            acc.append(Access(e, "x", op[2], 0, 1, op[3] == "w"))
        elif k in ("R", "W"):
            log.add(Entry("record" if k == "R" else "wait", k, op[1], op[2]))
        elif k == "E":
            log.add(Entry("ev_sync", k, None, op[1]))
        elif k == "S":
            log.add(Entry("stream_sync", k, op[1]))
        elif k == "D":
            log.add(Entry("device_sync", k))
    return log.entries, acc


def test_clock_fork_join():
    ents, acc = synth(("L", 1, "x", "w"), ("R", 1, "e"), ("W", 2, "e"), ("L", 2, "x", "r"), ("L", 2, "y", "w"),
                      ("R", 2, "f"), ("W", 1, "f"), ("L", 1, "y", "r"))
    res = check(ents, acc)
    assert not res.hazards and res.ordered == 2
    res = check([e for e in ents if not (e.kind == "wait" and e.ev == "e")], acc)
    assert len(res.hazards) == 1 and res.hazards[0].startswith("RAW on x")
    res = check([e for e in ents if not (e.kind == "wait" and e.ev == "f")], acc)
    assert len(res.hazards) == 1 and res.hazards[0].startswith("RAW on y")


def test_clock_event_rerecorded_between_record_and_wait():
    # the wait sees the most recent record: the one after stream 1's second write
    ents, acc = synth(("L", 1, "x", "w"), ("R", 1, "e"), ("L", 1, "y", "w"), ("R", 1, "e"), ("W", 2, "e"),
                      ("L", 2, "y", "r"), ("L", 2, "x", "r"))
    assert not check(ents, acc).hazards
    # recorded again after the wait: a later write on stream 1 is not ordered before stream 2's read
    ents, acc = synth(("L", 1, "x", "r"), ("R", 1, "e"), ("W", 2, "e"), ("R", 1, "e"), ("L", 1, "x", "w"),
                      ("L", 2, "x", "r"))
    res = check(ents, acc)
    assert len(res.hazards) == 1 and "RAW on x" in res.hazards[0]
    # a write on 2 after a read on 1 that 2 never waited for
    ents, acc = synth(("L", 1, "x", "r"), ("L", 2, "x", "w"))
    assert check(ents, acc).hazards[0].startswith("WAR on x")
    ents, acc = synth(("L", 1, "x", "w"), ("L", 2, "x", "w"))
    assert check(ents, acc).hazards[0].startswith("WAW on x")


def test_clock_wait_stream_is_transitive():
    # 3 waits 2, which waited 1: 1's write is ordered before 3's read
    ents, acc = synth(("L", 1, "x", "w"), ("R", 1, "a"), ("W", 2, "a"), ("L", 2, "y", "r"), ("R", 2, "b"),
                      ("W", 3, "b"), ("L", 3, "x", "r"))
    assert not check(ents, acc).hazards
    # read-read is never a conflict, and same-stream pairs are stream-ordered
    ents, acc = synth(("L", 1, "x", "r"), ("L", 2, "x", "r"), ("L", 2, "x", "w"), ("L", 2, "x", "r"))
    res = check(ents, acc)
    assert [h.split(" ")[0] for h in res.hazards] == ["WAR"]


def test_clock_host_synchronisation():
    # the host refills a buffer a stream read: ordered by an event synchronize, a stream synchronize or a device one
    for sync in (("E", "e"), ("S", 1), ("D",)):
        ents, acc = synth(("L", 1, "h", "r"), ("R", 1, "e"), sync, ("L", HOST, "h", "w"))
        assert not check(ents, acc).hazards, sync
    ents, acc = synth(("L", 1, "h", "r"), ("R", 1, "e"), ("L", HOST, "h", "w"))
    assert check(ents, acc).hazards[0].startswith("WAR on h")
    # what the host did before an enqueue happens before the enqueued work, on any stream
    ents, acc = synth(("L", HOST, "h", "w"), ("L", 2, "h", "r"))
    assert not check(ents, acc).hazards
    # the host's join carries to a stream it enqueues on later: 1 -> host -> 2
    ents, acc = synth(("L", 1, "x", "w"), ("S", 1), ("L", 2, "x", "r"))
    assert not check(ents, acc).hazards


def test_clock_temporaries_stay_on_their_stream():
    ents, acc = synth(("L", 1, "temp@3", "w"), ("L", 1, "temp@3", "r"))
    assert not check(ents, acc).hazards
    ents, acc = synth(("L", 1, "temp@3", "w"), ("R", 1, "e"), ("W", 2, "e"), ("L", 2, "temp@3", "r"))
    assert check(ents, acc).hazards[0].startswith("temporary temp@3")


def test_drop_names_the_site():
    ents, _acc = synth(("R", 1, "e"), ("W", 2, "e"))
    ents[1].site = "modeling.py:1: side.wait_event(ev)"
    assert len(drop(ents, "side.wait_event(ev)")) == 1
    with pytest.raises(AssertionError, match="no entry"):
        drop(ents, "main.wait_event")


# entry points the recorded steps call
STEP_ENTRY_POINTS = (
    "b2_gemm_bf16", "b2_gemm_bf16_grouped", "b2_gemm_ln_fwd", "b2_embed_fwd", "b2_embed_fwd_packed", "b2_embed_bwd",
    "b2_embed_bwd_packed", "b2_embed_bwd_ordered", "b2_embed_bwd_packed_ordered", "b2_layernorm_fwd",
    "b2_layernorm_bwd", "b2_layernorm_bwd_accum", "b2_colsum_finish", "b2_colsum", "b2_attention_fwd",
    "b2_attention_bwd", "b2_attention_fwd_packed", "b2_attention_bwd_packed", "b2_attention_fwd_packed_seq",
    "b2_attention_bwd_packed_seq", "b2_attention_bwd_ordered", "b2_attention_bwd_packed_seq_ordered",
    "b2_accum_finish", "b2_head_fwd", "b2_head_fwd_packed", "b2_head_bwd_split", "b2_ce_fwd_bwd", "b2_loss_fwd_bwd",
    "b2_token_head_fwd", "b2_token_head_bwd_split", "b2_mlm_compact", "b2_mlm_gather_rows", "b2_mlm_scatter_rows",
    "b2_mlm_gelu_bwd", "b2_mlm_bias_fill", "b2_mlm_ce", "b2_mlm_tied_add", "b2_bucket_reduce_adamw",
    "b2_adamw_prepare", "b2_adamw_background", "b2_bucket_reduce_sgd", "b2_sgd_background", "b2_bucket_reduce_adam",
    "b2_adam_prepare", "b2_adam_background", "b2_grad_accumulate", "b2_grad_reduce_sumsq", "b2_grad_norm_finalize",
    "b2_step_advance", "b2_rng_seed", "b2_cast_f32_to_bf16", "b2_zero", "b2_copy_async")


def test_header_roles_cover_every_entry_point():
    rl = roles()
    for name, sig in L._SIGNATURES.items():
        assert name in rl, "%s is not declared in the header" % name
        assert len(rl[name]) == len(sig), "%s: %d header parameters, %d ctypes arguments" % (name, len(rl[name]),
                                                                                           len(sig))
        for (pname, role), t in zip(rl[name], sig):
            if t in (ctypes.c_void_p, ctypes.c_char_p):
                ok = role in (R, RW, "skip", "host", "r[]", "rw[]")
            elif isinstance(t, type) and issubclass(t, ctypes._Pointer):
                ok = role in STRUCT_ROLES or role in ("r[]", "rw[]")
                if role in STRUCT_ROLES:
                    assert set(STRUCT_ROLES[role]) <= {f for f, _t in t._type_._fields_}, (name, pname)
            else:
                ok = role is None
            assert ok, "%s: parameter %s has role %r for ctypes type %r" % (name, pname, role, t)
    assert set(STEP_ENTRY_POINTS) <= set(rl)
    # each split head's tables cover every pointer parameter but the streams
    for name, (main_r, wgt_r, si, wi, _cu) in HEAD_SPLIT.items():
        ptrs = {i for i, (_p, r) in enumerate(rl[name]) if r in (R, RW)}
        assert set(main_r) | set(wgt_r) == ptrs, name
        assert (rl[name][si][0], rl[name][wi][0]) in (("stream_", "weight_stream_"), ("stream", "weight_stream")), name
        for i, r in list(main_r.items()) + list(wgt_r.items()):
            assert r == R or rl[name][i][1] == RW, "%s: parameter %s is const in the header" % (name, rl[name][i][0])


def test_header_role_examples():
    rl = roles()
    assert rl["b2_mlm_tied_add"] == [("dec", R), ("grad", RW), ("n", None), ("stream", "skip")]
    assert dict(rl["b2_layernorm_bwd"])["deferred_nparts"] == "host"
    ad = dict(rl["b2_bucket_reduce_adamw"])
    assert (ad["peer_grads"], ad["peer_shadow"], ad["hp"], ad["step_counter"], ad["master"]) == \
        ("r[]", "rw[]", "hparams", R, RW)
    assert dict(rl["b2_gemm_bf16_grouped"])["args"] == "gemm"
    assert dict(rl["b2_head_bwd_split"])["weight_stream"] == "skip"
    assert dict(rl["b2_accum_finish"])["segments"] == R and dict(rl["b2_accum_finish"])["dst"] == RW
    assert parse_header("int32_t b2_x(const float* a /* c */, void* b, int64_t n, void* s_stream);") == \
        {"b2_x": [("a", R), ("b", RW), ("n", None), ("s_stream", "skip")]}


def _cpu_memory(lay):
    """a Memory over CPU stand-ins of a layout's flat spaces, with register_step's span registrations"""
    mem = Memory()
    grads = torch.zeros(lay.total, dtype=torch.bfloat16)
    shadow = torch.zeros(lay.total, dtype=torch.bfloat16)
    mem.flat("grads", grads)
    mem.flat("shadow", shadow)
    for name, (b, n) in reserved_spans(lay).items():
        mem.register("g:" + name, grads[b:b + n], "grad")
        mem.register("w:" + name, shadow[b:b + n], "w")
    ws = torch.zeros(64)
    mem.units.add("ws", ws, "ws")
    return mem, grads, shadow, ws


def _launch(name, acc, **scal):
    e = Entry("launch", name, 1)
    e.idx = 0
    e.acc = [(k, a, w, False) for k, a, w in acc]
    e.scal = scal
    return e


@pytest.mark.parametrize("head", ["sequence", "token", "mlm"])
@pytest.mark.parametrize("layers", [0, 1, 3])
def test_extents_on_the_layout(head, layers):
    V = 1050 if head == "mlm" else 512
    lay = _Layout(tiny_config(num_hidden_layers=layers, type_vocab_size=3, vocab_size=V), head=head)
    mem, grads, shadow, ws = _cpu_memory(lay)
    log = StepLog()
    g0, w0 = grads.data_ptr(), shadow.data_ptr()
    spans = reserved_spans(lay)
    # every span start covers exactly its span, in either space; the spans never overlap
    for name, (b, n) in spans.items():
        log.entries = [_launch("b2_gemm_bf16", [("D", g0 + 2 * b, True), ("B", w0 + 2 * b, False)])]
        got = {(a.region, a.lo, a.hi) for a in resolve(log, mem)}
        assert got == {("grads", b, b + n), ("shadow", b, b + n)}, name
    cover = sorted((b, b + n) for b, n in spans.values())
    assert all(e0 <= b1 for (_b0, e0), (b1, _e1) in zip(cover, cover[1:]))
    if head == "mlm":
        assert spans[WORD][1] == lay.vocab_pad * lay.entries[WORD][1][1]
    # a pointer inside a span, or into the padding after one, is unmodelled
    wb, wn = spans[WORD]
    offs = [wb + 8] + [sb + sn for sb, sn in spans.values() if sn % 8]
    for off in offs:
        log.entries = [_launch("b2_gemm_bf16", [("D", g0 + 2 * off, True)])]
        with pytest.raises(Unmodelled, match="unmodelled"):
            resolve(log, mem)
    # the range entry points cover their own range, wherever their pointers start
    eb, ee, _ = lay.buckets[0]
    log.entries = [_launch("b2_zero", [("dst", g0 + 2 * eb, True)], bytes=2 * (ee - eb))]
    assert [(a.region, a.lo, a.hi) for a in resolve(log, mem)] == [("grads", eb, ee)]
    for bi, (bb, be, _l) in enumerate(lay.buckets):
        log.entries = [_launch("b2_adamw_background", [("grads", g0, False), ("shadow", w0, True)], begin=bb, end=be)]
        assert [(a.region, a.lo, a.hi, a.write) for a in resolve(log, mem)] == \
            [("grads", bb, be, False), ("shadow", bb, be, True)]
    log.entries = [_launch("b2_cast_f32_to_bf16", [("dst", w0, True)], n=lay.total)]
    assert [(a.lo, a.hi) for a in resolve(log, mem)] == [(0, lay.total)]
    # a unit is covered whole from any element; an address in no region fails
    log.entries = [_launch("b2_colsum", [("scratch_partials", ws.data_ptr() + 4 * 9, True)])]
    assert [(a.region, a.lo, a.hi) for a in resolve(log, mem)] == [("ws", 0, 1)]
    log.entries = [_launch("b2_colsum", [("scratch_partials", ws.data_ptr() + 4 * 64, True)])]
    with pytest.raises(AssertionError, match="no region"):
        resolve(log, mem)


def test_accum_finish_covers_its_segments():
    lay = _Layout(tiny_config(num_hidden_layers=2), head="sequence")
    mem, grads, _shadow, _ws = _cpu_memory(lay)
    H, I = 256, 512
    per = 9 * H + I
    acc = torch.zeros(2 * per)
    segs = []
    for l in range(2):
        pre = "bert.encoder.layer.%d." % l
        segs += [[l * per, lay.off(pre + "attention.self.query.bias"), 3 * H],
                 [l * per + 3 * H, lay.off(pre + "intermediate.dense.bias"), I]]
    st = torch.tensor(segs, dtype=torch.int64)
    mem.units.add("bias_segs", st, "state")
    for l in range(2):
        mem.units.add("bias_acc.%d" % l, acc[l * per:(l + 1) * per], "acc")
    mem.segs = (st.data_ptr(), segs, acc.data_ptr())
    log = StepLog()
    e = _launch("b2_accum_finish", [("src", acc.data_ptr(), True), ("dst", grads.data_ptr(), True),
                                    ("segments", st.data_ptr() + 24 * 3, False)], n_segments=1)
    log.entries = [e]
    got = sorted((a.region, a.lo, a.hi) for a in resolve(log, mem))
    ob = lay.off("bert.encoder.layer.1.intermediate.dense.bias")
    assert got == [("bias_acc.1", 0, 1), ("bias_segs", 0, 1), ("grads", ob, ob + I)]


# ======================================================================================================================
# GPU: the recorded steps
# ======================================================================================================================
def model_of(head, layers, S=128):
    cfg = tiny_config(num_hidden_layers=layers, max_position_embeddings=max(128, S),
                      vocab_size=1050 if head == "mlm" else 512, num_labels=9 if head == "token" else 6)
    torch.manual_seed(SEED)
    cls = {"sequence": b2.BertForSequenceClassification, "token": b2.BertForTokenClassification,
           "mlm": b2.BertForMaskedLM}[head]
    return cls(cfg).cuda().train(), cfg


def batch_of(head, cfg, B, S, seed):
    if head == "token":
        return token_batch(cfg, B, S, seed)
    if head == "mlm":
        return b2.synthetic_mlm_batch(cfg, B, S, seed, padded=True)
    if S > 128:
        return long_batch(cfg, B, seed, lo=16, hi=S - 40, S=S)
    return short_batch(cfg, B, seed, lo=20, hi=S)


def optimizer_of(kind, model):
    p = model.parameters()
    if kind == "adamw":
        return b2.AdamW(p, lr=1e-3, weight_decay=0.01)
    if kind == "torch_adamw":
        return b2.TorchAdamW(p, lr=1e-3)
    if kind == "adam_amsgrad":
        return b2.Adam(p, lr=1e-3, amsgrad=True, weight_decay=0.01)
    if kind == "sgd":
        return b2.SGD(p, lr=1e-2, momentum=0.9, nesterov=True, weight_decay=0.01)
    raise ValueError(kind)


def stream_names(eng, step=None):
    names = {torch.cuda.default_stream().cuda_stream: "default", eng.wgrad_stream.cuda_stream: "wgrad",
             eng._local.side.cuda_stream: "side"}
    if step is not None:
        names[step._prio_stream.cuda_stream] = "body"
    return names


CAPTURED = {
    "seq_adamw": dict(head="sequence", layers=3, opt="adamw"),
    "seq_adamw_det": dict(head="sequence", layers=3, opt="adamw", det=True),
    "token_torch_adamw": dict(head="token", layers=3, opt="torch_adamw"),
    "token_det": dict(head="token", layers=3, opt="torch_adamw", det=True),
    "mlm_adam_amsgrad": dict(head="mlm", layers=2, opt="adam_amsgrad"),
    "mlm_det": dict(head="mlm", layers=2, opt="adamw", det=True),
    "seq_sgd_nesterov": dict(head="sequence", layers=3, opt="sgd"),
    "seq_clip": dict(head="sequence", layers=3, opt="adamw", clip=1.0),
    "seq_clip_det": dict(head="sequence", layers=3, opt="torch_adamw", clip=0.5, det=True),
    "seq_accum2": dict(head="sequence", layers=3, opt="adamw", accum=2),
    "seq_lr_schedule": dict(head="sequence", layers=3, opt="torch_adamw", sched=True),
    "seq512": dict(head="sequence", layers=2, opt="adamw", S=512),
    "packed128": dict(head="sequence", layers=2, opt="adamw", packed=True),
    "packed512": dict(head="sequence", layers=2, opt="sgd", packed=True, S=512),
    "token_packed512": dict(head="token", layers=2, opt="adamw", packed=True, S=512, det=True),
    "no_layers": dict(head="sequence", layers=0, opt="adamw"),
    "mlm_no_layers": dict(head="mlm", layers=0, opt="torch_adamw"),
}


def run_captured(case):
    """(warm-up log, capture log, Memory, stream names, the step) of one CAPTURED case"""
    c = CAPTURED[case]
    head, layers, S, det = c["head"], c["layers"], c.get("S", 128), c.get("det", False)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        model, cfg = model_of(head, layers, S)
        opt = optimizer_of(c["opt"], model)
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 1.0 / (1 + i)) if c.get("sched") else None
        kw = dict(accum_steps=c.get("accum", 1), max_grad_norm=c.get("clip"))
        if c.get("packed"):
            b = batch_of(head, cfg, 12 if S == 512 else 24, S, 11) if head != "sequence" else \
                (long_batch(cfg, 8, 11, lo=16, hi=400, S=512) if S == 512 else short_batch(cfg, 24, 11, lo=3, hi=60))
            token = head != "sequence"
            pk = b2.pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], S,
                               labels=b["label"] if token else None)
            step = b2.PackedTrainStep(model, opt, pk["bins"], b["input_ids"].shape[0], bin_len=S, **kw)
            label = pk["labels"] if token else b["label"]
            call = lambda final: step(pk, label, final)
            inputs = {"ids": step.d_ids, "tt": step.d_tt, "pos": step.d_pos, "seg": step.d_seg, "cls": step.d_cls,
                      "labels": step.d_lab}
        else:
            B = 4 if S == 512 else 8
            b = batch_of(head, cfg, B, S, 11)
            step = b2.FusedTrainStep(model, opt, B, S, **kw)
            call = lambda final: step(b, final)
            inputs = {"ids": step.d_ids, "tt": step.d_tt, "mask": step.d_mask, "labels": step.d_lab}
        finals = [False, False, True] * 2 if c.get("accum") else [True, True]

        def one(final):
            call(final)
            if sched is not None and final:
                sched.step()

        # the optimizer's device state first: creating it copies the decay flags to the device, a host synchronise
        # that would hide the cross-step host edge (stage()'s wait on _h2d_done) inside the log
        opt._state()
        torch.cuda.synchronize()
        with StepLog() as warm:
            for f in finals:
                one(f)
        with StepLog() as cap:
            one(finals[0])
        assert step._graphs, "%s: the third call did not capture" % case
        torch.cuda.synchronize()
        mem = engine_memory(model._engine, opt, step, inputs)
        return warm, cap, mem, stream_names(model._engine, step), (model, opt, step)
    finally:
        torch.use_deterministic_algorithms(was)


@pytest.fixture(scope="module")
def recorded():
    runs = {}

    def get(case):
        if case not in runs:
            runs[case] = run_captured(case)
        return runs[case]

    yield get
    runs.clear()
    torch.cuda.empty_cache()


# ordered cross-stream conflicting pairs a captured case's warm-up log must have at least (with encoder layers; the
# models without them have one backward launch stream fewer)
MIN_ORDERED, MIN_ORDERED_NO_LAYERS = 500, 150


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CAPTURED))
def test_captured_schedule_is_ordered(cuda_dev, recorded, case):
    warm, cap, mem, names, (model, _opt, _step) = recorded(case)
    for what, log in (("warm-up bodies", warm), ("capture", cap)):
        res = check(log.entries, resolve(log, mem), names)
        assert_ordered(res, "%s %s" % (case, what))
        launch_streams = {e.stream for e in log.entries if e.kind == "launch"}
        assert {e.name for e in log.entries if e.kind == "launch"} <= set(STEP_ENTRY_POINTS)
        assert len(res.streams) >= 3, "%s %s: accesses on %s only" % (case, what, res.streams)
        layers = CAPTURED[case]["layers"]
        assert len(launch_streams) >= (3 if layers else 2), "%s %s: launches on %d streams" % (
            case, what, len(launch_streams))
        if what == "warm-up bodies":
            least = MIN_ORDERED if layers else MIN_ORDERED_NO_LAYERS
            assert res.ordered >= least, "%s: only %d ordered cross-stream conflicting pairs" % (case, res.ordered)
            print("%s: %d entries, %d ordered cross-stream conflicting pairs on %d streams (%d with launches)" % (
                case, len(log.entries), res.ordered, len(res.streams), len(launch_streams)))


# the planted defects: (case, call-site text of the edge deleted, occurrence, the failure)
UPDATES = r"(b2_adamw_background|b2_adam_background|b2_sgd_background|b2_bucket_reduce_\w+)"
DEFECTS = {
    "fork_before_grouped_wgrad": ("seq_adamw", "modeling.py", "side.wait_event(ev)", 0,
                                  r"RAW on (dzd|dU|dz1d|dqkv)\.0 .*b2_gemm_bf16_grouped"),
    "parity_reuse": ("seq_adamw", "modeling.py", "main.wait_event(done[l + 2])", 0,
                     r"WAR on (dzd|dU|dz1d|dqkv)\.0 "),
    "wgrad_marker": ("seq_adamw", "optim.py", "t.side.wait_event(wg_event)", 0,
                     r"RAW on grads \[.*b2_gemm_bf16_grouped.*" + UPDATES),
    "dec_done": ("mlm_adam_amsgrad", "modeling.py", "main.wait_event(dec_done)", 0,
                 r"RAW on mlm\.dec .*b2_mlm_tied_add"),
    "finish_step_join": ("seq_adamw", "optim.py", "main.wait_stream(t.side)", 0, UPDATES + r" #\d+ .* on side and "),
    "head_split_fork": ("seq_adamw", "head.cu", "the fork of b2_head_bwd_split: cudaStreamWaitEvent", 0,
                        r"RAW on head_scratch .*b2_head_bwd_split"),
    "h2d_done": ("seq_adamw", "trainer.py", "self._h2d_done.synchronize()", 0, r"WAR on stage\.h "),
}


@pytest.mark.gpu
@pytest.mark.parametrize("defect", list(DEFECTS))
def test_planted_schedule_defect_fails(cuda_dev, recorded, defect):
    case, where, text, nth, fails = DEFECTS[defect]
    warm, _cap, mem, names, _objs = recorded(case)
    acc = resolve(warm, mem)
    assert_ordered(check(warm.entries, acc, names), case)
    ents = drop(warm.entries, text, nth)
    gone = [e for e in warm.entries if e not in ents][0]
    assert gone.site.startswith(where), gone.site
    res = check(ents, acc, names)
    assert res.hazards, "%s: deleting %r left every conflict ordered; the host waits at: %s" % (
        defect, gone.site, "; ".join("#%d %s %s" % (e.idx, e.kind, e.site) for e in ents
                                     if e.kind in ("ev_sync", "stream_sync", "device_sync")))
    assert any(re.search(fails, h) for h in res.hazards), "%s: no hazard matches %r; got:\n%s" % (
        defect, fails, "\n".join(res.hazards[:6]))


# ---- eager paths, two steps each -------------------------------------------------------------------------------------
EAGER = ("autograd", "clip", "amp", "no_sync", "ddp_world1", "trainer_staged")


def run_eager(kind):
    model, cfg = model_of("sequence", 3)
    opt = b2.AdamW(model.parameters(), lr=1e-3, weight_decay=0.01)
    batches = [short_batch(cfg, 8, 20 + i, lo=20, hi=128) for i in range(6)]
    dev_b = [{k: v.cuda() for k, v in b.items()} for b in batches]
    extra = []
    net = model
    trainer = None
    if kind == "ddp_world1":
        net = b2.DistributedDataParallel(model, overlap=False)
    if kind in ("amp", "trainer_staged"):
        args = b2.Args()
        args.fused = kind == "trainer_staged"
        args.use_amp = kind == "amp"
        trainer = b2.Trainer(args, cfg, model, None, opt)

    def fwd_bwd(d):
        net(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
            labels=d["label"]).loss.backward()

    def one(i):
        if trainer is not None:
            trainer.train_step(batches[i])
            return
        if kind == "no_sync":
            with net.no_sync():
                fwd_bwd(dev_b[2 * i])
            fwd_bwd(dev_b[2 * i + 1])
        else:
            fwd_bwd(dev_b[i])
        if kind == "clip":
            b2.clip_grad_norm_(model.parameters(), 1.0)
        opt.step()
        opt.zero_grad()

    one(0)          # allocations outside the log
    torch.cuda.synchronize()
    with StepLog() as log:
        one(1)
        one(2)
    torch.cuda.synchronize()
    for j, d in enumerate(dev_b):
        for k, v in d.items():
            extra.append(("in%d:%s" % (j, k), v))
    step = None
    if trainer is not None:
        for (k, _shape), (buf, _ev) in trainer._pin.items():
            extra.append(("pin:" + k, buf))
        step = trainer._fused
        if step is not None:
            extra += [("step." + k, getattr(step, k)) for k in ("d_ids", "d_tt", "d_mask", "d_lab")]
        if trainer._scaler is not None:
            extra += [("scaler.scale", trainer._scaler._scale), ("scaler.growth", trainer._scaler._growth_tracker)]
    mem = engine_memory(model._engine, opt, step, extra=extra)
    return log, mem, stream_names(model._engine, step)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", EAGER)
def test_eager_schedule_is_ordered(cuda_dev, kind):
    log, mem, names = run_eager(kind)
    res = check(log.entries, resolve(log, mem), names)
    assert_ordered(res, kind)
    assert {e.name for e in log.entries if e.kind == "launch"} <= set(STEP_ENTRY_POINTS)
    print("%s: %d entries, %d ordered cross-stream conflicting pairs on %d streams" % (
        kind, len(log.entries), res.ordered, len(res.streams)))
    if kind == "trainer_staged":
        assert any("self._h2d_done.synchronize()" in e.site for e in log.entries)


# ======================================================================================================================
# Part B: the optimizer stage of a captured step, against the step's own gradients
# ======================================================================================================================
# A replay consumes the gradient space in place (with accumulation the FOLD leaves bf16(acc + g) there), so after a
# replay `grads` holds exactly what the update read.  From a snapshot of the master, the optimizer state, the step
# counter, the dropout rng and the staged lr taken before the replay, the expected update is computed on every
# bucket.  The schedule updates buckets != 0 with the background (slim) form during the backward and bucket 0 (and
# a clipped step's whole range) with the reduce form; both forms are held to the same reference: torch's fused
# Adam / AdamW op bitwise, torch.optim.SGD bitwise, HF AdamW at test_step_kernels.AdamWRef's bound.
UPDATE_CASES = {
    "adamw": dict(opt="adamw"),
    "torch_adamw": dict(opt="torch_adamw"),
    "adam": dict(opt="adam"),
    "adam_amsgrad": dict(opt="adam_amsgrad"),
    "sgd": dict(opt="sgd"),
    "adamw_clip": dict(opt="adamw", clip=0.05),
    "torch_adamw_clip": dict(opt="torch_adamw", clip=0.05),
    "torch_adamw_accum2": dict(opt="torch_adamw", accum=2),
}
UPDATE_DEFECTS = ("previous_lr", "stale_bucket", "step_off_by_one")


def update_optimizer(kind, model):
    p = model.parameters()
    if kind == "adam":
        return b2.Adam(p, lr=1e-3)                  # coupled decay off: torch's fused kernel varies it by lane
    if kind == "adam_amsgrad":
        return b2.Adam(p, lr=1e-3, amsgrad=True)
    return optimizer_of(kind, model)


def snapshot(model, opt):
    torch.cuda.synchronize()
    eng, st = model._engine, opt._dev_state
    out = {"master": model._flat.clone(), "step": int(st["step"]), "rng": eng.rng.cpu().clone(),
           "grads": eng.grads.clone(), "shadow": eng.shadow.clone(), "lr_slot": float(st["lr"].double())}
    for k in FLAT_KEYS:
        if st.get(k) is not None:
            out[k] = st[k].clone()
    if opt._clip_buf is not None:
        out["norm"], out["coef"] = opt._clip_buf["norm"].clone(), opt._clip_buf["coef"].clone()
    return out


def expected_update(kind, opt, before, g, lr, t, coef=None):
    """the state after one update of `before` with bf16 gradients g at lr and bias-correction step t (1-based):
    name -> (expected, bound or None for bitwise)"""
    dec = (opt._dev_state["decay"] & 1).bool().repeat_interleave(8)
    gf = g.float() if coef is None else g.float() * coef
    w0 = before["master"]
    out = {}
    if kind == "adamw":
        sel = torch.arange(w0.numel(), device=w0.device)
        gr = opt.param_groups[0]
        ref = AdamWRef(w0, dec, sel, lr, opt._wd, gr["correct_bias"], 1, extra=0 if coef is None else 1)
        ref.opt.betas, ref.opt.eps = gr["betas"], gr["eps"]
        for name, m in (("x.weight", dec), ("x.bias", ~dec)):
            ref.opt.state[name] = {"step": t - 1, "exp_avg": before["exp_avg"].double()[m].clone(),
                                   "exp_avg_sq": before["exp_avg_sq"].double()[m].clone()}
        g64 = g.double() if coef is None else g.double() * float(coef)
        m, v, w = ref.step(g64)
        return {"master": (w, ref.ew), "exp_avg": (m, ref.em), "exp_avg_sq": (v, ref.ev)}
    groups = [(m, wd) for m, wd in ((dec, opt._wd), (~dec, 0.0)) if bool(m.any())]
    if kind == "sgd":
        gr = opt.param_groups[0]
        ps = [torch.nn.Parameter(w0[m].clone()) for m, _wd in groups]
        ref = torch.optim.SGD([{"params": [p], "weight_decay": wd} for p, (_m, wd) in zip(ps, groups)], lr=lr,
                              momentum=gr["momentum"], dampening=gr["dampening"], nesterov=gr["nesterov"],
                              foreach=False)
        for p, (m, _wd) in zip(ps, groups):
            p.grad = gf[m].clone()
            if t > 1:
                ref.state[p]["momentum_buffer"] = before["momentum_buffer"][m].clone()
        ref.step()
        out["master"], out["momentum_buffer"] = w0.clone(), before["momentum_buffer"].clone()
        for p, (m, _wd) in zip(ps, groups):
            out["master"][m] = p.detach()
            out["momentum_buffer"][m] = ref.state[p]["momentum_buffer"]
        return {k: (v, None) for k, v in out.items()}
    gr = opt.param_groups[0]
    ams = bool(gr["amsgrad"])
    keys = ["exp_avg", "exp_avg_sq"] + (["max_exp_avg_sq"] if ams else [])
    out = {k: before[k].clone() for k in keys}
    out["master"] = w0.clone()
    fused = torch._fused_adamw_ if gr["decoupled_weight_decay"] else torch._fused_adam_
    for m, wd in groups:
        p, st = w0[m].clone(), {k: before[k][m].clone() for k in keys}
        fused([p], [gf[m].clone()], [st["exp_avg"]], [st["exp_avg_sq"]], [st["max_exp_avg_sq"]] if ams else [],
              [torch.tensor(float(t), device=w0.device)], lr=lr, beta1=gr["betas"][0], beta2=gr["betas"][1],
              weight_decay=wd, eps=gr["eps"], amsgrad=ams, maximize=bool(gr["maximize"]))
        out["master"][m] = p
        for k in keys:
            out[k][m] = st[k]
    return {k: (v, None) for k, v in out.items()}


def compare_update(case, got, want):
    for k, (ref, bound) in want.items():
        if bound is None:
            bad = int((got[k].view(torch.int32) != ref.view(torch.int32)).sum())
            assert bad == 0, "%s %s: %d elements differ from the reference bitwise" % (case, k, bad)
        else:
            within(got[k], ref, bound, "%s %s" % (case, k))


def run_updates(case):
    """the captured step after its warm-ups and capture, then two replays at an lr that changes every step:
    [(before, after, staged lr)] of the two replays and the optimizer"""
    c = UPDATE_CASES[case]
    model, cfg = model_of("sequence", 3)
    opt = update_optimizer(c["opt"], model)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda i: 1.0 / (1 + i))
    k = c.get("accum", 1)
    step = b2.FusedTrainStep(model, opt, 8, 128, accum_steps=k, max_grad_norm=c.get("clip"))
    batches = [short_batch(cfg, 8, 40 + i, lo=20, hi=128) for i in range(8 * k)]
    it = iter(batches)

    def optimizer_step(measure):
        for j in range(k):
            final = j == k - 1
            if final and measure:
                lr = opt.current_lr()
                before = snapshot(model, opt)
            step(next(it), final)
        sched.step()
        if measure:
            return before, snapshot(model, opt), lr

    for _ in range(3):              # two eager warm-ups and the capture (each role of the window has its graph)
        optimizer_step(False)
    assert step.graph is not None
    return [optimizer_step(True) for _ in range(2)], opt


@pytest.fixture(scope="module")
def updated():
    runs = {}

    def get(case):
        if case not in runs:
            runs[case] = run_updates(case)
        return runs[case]

    yield get
    runs.clear()


def check_replay(case, opt, before, after, lr, defect=None, previous=None):
    c = UPDATE_CASES[case]
    g = after["grads"]
    t = before["step"] + 1
    assert after["step"] == before["step"] + 1, "%s: step counter %d -> %d" % (case, before["step"], after["step"])
    assert int(after["rng"][1]) == int(before["rng"][1]) + 1, "%s: dropout step did not advance by one" % case
    assert after["lr_slot"] == lr, "%s: the device lr slot is %r, this replay staged %r" % (case, after["lr_slot"], lr)
    assert torch.equal(after["shadow"], after["master"].to(torch.bfloat16)), "%s: shadow != bf16(master)" % case
    coef = None
    if c.get("clip"):
        norm = float(after["norm"])
        ref = float(g.double().square().sum().sqrt())
        assert abs(norm - ref) <= 1e-6 * ref, "%s: norm %r, float64 %r" % (case, norm, ref)
        want = _torch_coef(after["norm"], c["clip"])
        assert torch.equal(after["coef"].cpu(), want), "%s: clip coefficient %r, torch's %r" % (
            case, after["coef"], want)
        assert float(want) < 1.0, "%s: the clip never bites" % case
        coef = after["coef"]
    if defect == "previous_lr":
        lr = previous[2]
    elif defect == "stale_bucket":
        b, e, _l = opt._model._layout.buckets[1]
        g = g.clone()
        g[b:e] = previous[1]["grads"][b:e]
    elif defect == "step_off_by_one":
        t += 1
    want = expected_update(c["opt"], opt, before, g, lr, t, coef)
    compare_update(case + ("" if defect is None else " planted " + defect), after, want)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(UPDATE_CASES))
def test_captured_update_matches_the_steps_gradients(cuda_dev, updated, case):
    replays, opt = updated(case)
    (b1, a1, lr1), (b2_, a2, lr2) = replays
    assert lr1 != lr2, "the schedule did not change the lr between the replays"
    check_replay(case, opt, b1, a1, lr1)
    check_replay(case, opt, b2_, a2, lr2)


@pytest.mark.gpu
@pytest.mark.parametrize("defect", UPDATE_DEFECTS)
@pytest.mark.parametrize("case", ["torch_adamw", "adamw"])
def test_planted_update_defect_fails(cuda_dev, updated, case, defect):
    replays, opt = updated(case)
    with pytest.raises(AssertionError, match=r"%s planted %s (master|exp_avg\w*): " % (case, defect)):
        check_replay(case, opt, *replays[1], defect=defect, previous=replays[0])
