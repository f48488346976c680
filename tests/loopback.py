"""Test infrastructure: the peer-exchange path of DistributedDataParallel on ONE device.

Two tools, both used by tests/test_peer_loopback.py:

* ``flag_launch`` -- the only way the tests launch a flag kernel (``b2_peer_barrier``, ``b2_allgather_rows``,
  ``b2_scalar_allreduce_mean``, the world > 1 ``b2_grad_norm_finalize``).  Those kernels spin until every flag they poll
  is at least the epoch they use; on one device the other "ranks" never run, so the test posts their flags first and
  the interlock (``interlock``) proves on the host, before the launch, that no poll can wait.  The device is idle before
  and after every launch, so no two flag kernels are ever in flight together.

* ``Group`` -- a loopback peer group: N replicas of one model on one device, each wrapped in the real
  ``DistributedDataParallel``.  The process group is a thread-backed fake (``FakeDist``), an IPC handle is the raw
  device pointer (one process cannot import its own IPC handles), and the flag entry points are replaced by host
  lockstep: synchronize, then meet the other ranks at a ``threading.Barrier`` -- no flag kernel runs at all.  Every
  other library call goes to the real library; a ``Recorder`` keeps the update launches.  One more stand-in, beyond
  those: ``ddp._drain_graveyard`` runs under a lock, because the N ranks share one process's graveyard of parked
  buffers and could otherwise pop from it at the same time (in a real peer group each process has its own).
"""
import ctypes
import threading

import torch

from parity import b2

L = b2._lib
ddp_mod = b2.ddp

REDUCE_ENTRIES = ("b2_bucket_reduce_adamw", "b2_bucket_reduce_sgd", "b2_bucket_reduce_adam")
SLOT_NAMES = {ddp_mod._SLOT_GRADS_READY: "_SLOT_GRADS_READY", ddp_mod._SLOT_UPDATE_DONE: "_SLOT_UPDATE_DONE",
              ddp_mod._SLOT_LOSS: "_SLOT_LOSS", ddp_mod._SLOT_GATHER: "_SLOT_GATHER", ddp_mod._SLOT_INF: "_SLOT_INF",
              ddp_mod._SLOT_CLIP: "_SLOT_CLIP"}


def slot_name(slot):
    if slot in SLOT_NAMES:
        return "slot %d (%s)" % (slot, SLOT_NAMES[slot])
    return "slot %d (_SLOT_BUCKET0 + %d)" % (slot, slot - ddp_mod._SLOT_BUCKET0)


# ======================================================================================================================
# raw device memory
# ======================================================================================================================
def raw(ptr, n, dtype, device):
    """a tensor view of n elements of `dtype` at the raw device address `ptr` (no copy)"""
    class _Iface:
        pass
    o = _Iface()
    nbytes = n * torch.empty((), dtype=dtype).element_size()
    o.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (int(ptr), False), "version": 2,
                                  "strides": None}
    return torch.as_tensor(o, device=device).view(dtype)


class CommBuf:
    """a zeroed b2_comm_alloc buffer as a uint32 / fp32 tensor view; freed by free()"""

    def __init__(self, nbytes, device):
        p = ctypes.c_void_p()
        L.call("b2_comm_alloc", nbytes, ctypes.byref(p))
        self.ptr, self.nbytes, self.device = p.value, nbytes, device

    def u32(self):
        return raw(self.ptr, self.nbytes // 4, torch.int32, self.device)

    def f32(self):
        return raw(self.ptr, self.nbytes // 4, torch.float32, self.device)

    def free(self):
        if self.ptr:
            torch.cuda.synchronize()
            L.call("b2_comm_free", self.ptr)
            self.ptr = 0


# ======================================================================================================================
# the interlock of a flag-kernel launch
# ======================================================================================================================
def ready(flag, epoch):
    """the kernels' wait condition, (int32)(flag - epoch) >= 0 on uint32 values"""
    d = (int(flag) - int(epoch)) & 0xFFFFFFFF
    return d < 0x80000000


def interlock(counter, polled):
    """The epoch a flag kernel will use (counter + 1, uint32) if every flag it polls already satisfies its wait, else
    AssertionError naming the first flag that would make it spin.  `polled`: {description: flag value}."""
    e = (int(counter) + 1) & 0xFFFFFFFF
    for what, v in polled.items():
        if not ready(v, e):
            raise AssertionError("interlock: %s = %#010x does not satisfy epoch %#010x: the kernel would wait; "
                                 "not launched" % (what, int(v) & 0xFFFFFFFF, e))
    return e


def flag_launch(entry, args, epoch_ctr, polled_flags, world):
    """Launches the flag kernel `entry` of one rank with every flag it polls already posted: the device is idle before
    (so no other flag kernel is in flight), the interlock passes on the host (else nothing is launched), and the call
    is synchronized before it returns.  epoch_ctr: (int32 tensor, slot) of the rank's epoch counter; polled_flags:
    (uint32 view of the rank's flag pad, slot) -- the kernel polls words slot * world + q for every q."""
    torch.cuda.synchronize()
    ctr, slot = epoch_ctr
    flags, fslot = polled_flags
    c = int(ctr[slot].item()) & 0xFFFFFFFF
    pad = flags.cpu()
    e = interlock(c, {"flags[%d]" % (fslot * world + q): int(pad[fslot * world + q]) & 0xFFFFFFFF
                      for q in range(world)})
    L.call(entry, *args)
    torch.cuda.synchronize()
    return e


# ======================================================================================================================
# the loopback peer group
# ======================================================================================================================
class Divergence(AssertionError):
    pass


class FakeDist:
    """torch.distributed as DistributedDataParallel uses it, over N threads of one process: rank = the calling thread's"""

    def __init__(self, world, timeout=120.0):
        self.world = world
        self.local = threading.local()
        self.bar = threading.Barrier(world, timeout=timeout)
        self.box = [None] * world

    def is_available(self):
        return True

    def is_initialized(self):
        return True

    def get_world_size(self, group=None):
        return self.world

    def get_rank(self, group=None):
        return self.local.rank

    def barrier(self, group=None):
        self.bar.wait()

    def _exchange(self, obj):
        r = self.local.rank
        self.box[r] = obj
        self.bar.wait()
        out = list(self.box)
        self.bar.wait()
        return out

    def all_gather_object(self, out, obj, group=None):
        out[:] = self._exchange(obj)

    def broadcast(self, tensor, src=0, group=None):
        torch.cuda.synchronize()
        got = self._exchange(tensor.clone() if self.local.rank == src else None)
        tensor.copy_(got[src])
        torch.cuda.synchronize()


class Recorder:
    """What the loopback saw of the library: every reduce-form update launch with its rank, range, world and pointer
    tables, every flag entry point, and every update-form launch by name"""

    def __init__(self):
        self.lock = threading.Lock()
        self.updates = []        # dicts: entry, rank, world, begin, end, grads, shadow, coef, grad_f32
        self.names = []
        self.flags = []          # (rank, entry, slot)
        self.snap_accum = False  # keep every b2_grad_accumulate's (rank, mode, bf16 gradients it reads) in `accum`
        self.accum = []

    def clear(self):
        with self.lock:
            self.updates, self.names, self.flags, self.accum = [], [], [], []


def _reduce_fields(name, args):
    """(world, rank, begin, end, grads, shadow, the clip coefficient and fp32 gradient pointers) of a b2_bucket_reduce_* call"""
    sig = L._SIGNATURES[name]
    i64s = [i for i, t in enumerate(sig) if t is L.i64]
    world, rank = int(args[2]), int(args[3])
    return dict(world=world, rank=rank, begin=int(args[i64s[0]]), end=int(args[i64s[1]]),
                grads=[args[0][q] for q in range(world)], shadow=[args[1][q] for q in range(world)],
                coef=args[i64s[1] + 1].clip_coef, grad_f32=args[i64s[1] + 1].grad_f32)


class Group:
    """N replicas of one model on one device in a loopback peer group.  Use as a context manager: it installs the fake
    process group, the IPC stand-ins and the host lockstep, and removes them on exit.

    plant (Part D of the loopback tests, the library stays unchanged): {"shift_slice": (rank, bucket, elements)} moves
    one rank's slice table; {"drop_shadow": (rank, peer)} drops a peer's shadow pointer from a rank's update tables;
    {"skip_slot": (rank, slot)} makes one rank skip a barrier."""

    def __init__(self, world, plant=None, timeout=120.0):
        self.world = world
        self.fake = FakeDist(world, timeout)
        self.rec = Recorder()
        self.plant = dict(plant or {})
        self.seq = [[] for _ in range(world)]       # every rank's (entry, slot) sequence
        self.box = [None] * world
        self.bar = threading.Barrier(world, timeout=timeout)
        self._saved = []
        self.wrappers = []
        self.driving = None          # the rank whose forward / backward the main thread runs
        self.dev = torch.device("cuda", 0)

    # -- installation ---------------------------------------------------------------------------------------------------
    def __enter__(self):
        orig_call = L.call
        self._orig_call = orig_call
        lock = threading.Lock()
        orig_drain = ddp_mod._drain_graveyard

        def drain():
            with lock:           # every rank shares the one process's graveyard: drain it under a lock
                orig_drain()

        patches = [(ddp_mod, "dist", self.fake), (L, "call", self._call),
                   (ddp_mod._DevBuf, "handle", lambda buf: int(buf.ptr).to_bytes(8, "little")),
                   (ddp_mod, "_import_handle", lambda h: int.from_bytes(bytes(h)[:8], "little")),
                   (ddp_mod, "_drain_graveyard", drain)]
        for obj, name, val in patches:
            self._saved.append((obj, name, getattr(obj, name)))
            setattr(obj, name, val)
        return self

    def __exit__(self, *exc):
        try:
            self.close()         # the stand-ins must outlive the wrappers: close() unmaps through them
        finally:
            self._restore()
        return False

    def _restore(self):
        for obj, name, val in reversed(self._saved):
            setattr(obj, name, val)
        self._saved = []

    # -- the library as the loopback sees it ----------------------------------------------------------------------------
    def _call(self, name, *args):
        if name == "b2_comm_unimport":
            return            # a loopback "mapping" is the owner's pointer itself: nothing to unmap
        if name == "b2_comm_export" or name == "b2_comm_import":
            raise AssertionError("the loopback imports no IPC handle (one process cannot open its own)")
        if name in ("b2_peer_barrier", "b2_scalar_allreduce_mean", "b2_allgather_rows"):
            return self._lockstep(name, args)
        if name == "b2_grad_norm_finalize" and int(args[4]) > 1:
            return self._lockstep(name, args)
        if name == "b2_grad_accumulate" and self.rec.snap_accum:
            torch.cuda.synchronize()
            begin, end = int(args[2]), int(args[3])
            g = raw(int(args[0]) + 2 * begin, end - begin, torch.bfloat16, self.dev).clone()
            with self.rec.lock:
                # (the backward runs in autograd's device thread: the rank is the one the driver is stepping)
                self.rec.accum.append((self.driving, int(args[4]), begin, end, g))
        if name in REDUCE_ENTRIES:
            f = _reduce_fields(name, args)
            args = self._planted_tables(f, args)
            with self.rec.lock:
                self.rec.updates.append(dict(f, entry=name))
        with self.rec.lock:
            self.rec.names.append(name)
        return self._orig_call(name, *args)

    def _planted_tables(self, f, args):
        if "drop_shadow" in self.plant:
            rank, peer = self.plant["drop_shadow"]
            if f["rank"] == rank:
                tab = L.ptr_array([None if q == peer else f["shadow"][q] for q in range(f["world"])])
                args = (args[0], tab) + tuple(args[2:])
        return args

    def _meet(self, rank, entry, slot):
        """host lockstep: every rank posts its (entry, slot) and its sequence so far, meets the others; a rank whose
        sequence differs fails every rank, naming both"""
        self.seq[rank].append((entry, slot))
        torch.cuda.synchronize()          # everything this rank enqueued before the barrier is complete
        self.box[rank] = list(self.seq[rank])
        self.bar.wait()
        seqs = list(self.box)
        self.bar.wait()
        for q in range(self.world):
            if seqs[q] != seqs[rank]:
                a, b = seqs[rank], seqs[q]
                i = next((k for k in range(min(len(a), len(b))) if a[k] != b[k]), min(len(a), len(b)))
                ea = "%s %s" % (a[i][0], slot_name(a[i][1])) if i < len(a) else "nothing"
                eb = "%s %s" % (b[i][0], slot_name(b[i][1])) if i < len(b) else "nothing"
                raise Divergence("lockstep divergence at flag call %d: rank %d reached %s, rank %d reached %s"
                                 % (i, rank, ea, q, eb))

    def _lockstep(self, name, args):
        if name == "b2_peer_barrier":
            world, rank, slot = int(args[1]), int(args[2]), int(args[3])
        elif name == "b2_grad_norm_finalize":
            world, rank, slot = int(args[4]), int(args[5]), int(args[6])
        else:
            world, rank, slot = int(args[4]), int(args[5]), int(args[6])
        assert world == self.world, (name, world)
        with self.rec.lock:
            self.rec.flags.append((rank, name, slot))
        if "skip_slot" in self.plant and self.plant["skip_slot"] == (rank, slot):
            return
        if name == "b2_scalar_allreduce_mean" and slot == ddp_mod._SLOT_INF:
            # the GradScaler consensus probe runs in every backward, and the backward of the loopback runs rank by rank
            # on one thread: no lockstep is possible there.  It is answered from this rank's own value, which is exact
            # while every rank's probe is finite (each posts 0) -- required here; a non-finite probe needs the peers
            self.seq[rank].append((name, slot))
            torch.cuda.synchronize()
            v = float(raw(args[0], 1, torch.float32, self.dev)[0])
            assert v == 0.0, "rank %d's probe is non-finite: the loopback cannot answer the consensus probe" % rank
            raw(args[1], 1, torch.float32, self.dev).fill_(0.0)
            torch.cuda.synchronize()
            return
        self._meet(rank, name, slot)
        if name == "b2_peer_barrier":
            return
        if name == "b2_allgather_rows":
            raise AssertionError("the loopback does not run b2_allgather_rows (eval gathers stay with the 2-GPU worker)")
        if name == "b2_scalar_allreduce_mean":
            v = raw(args[0], 1, torch.float32, self.dev).cpu()
            vals = self._share(rank, v)
            raw(args[1], 1, torch.float32, self.dev).copy_(rank_mean(vals))
        else:
            self._finalize_on_host(rank, args)
        torch.cuda.synchronize()
        self.bar.wait()

    def _share(self, rank, value):
        self.box[rank] = value
        self.bar.wait()
        vals = list(self.box)
        self.bar.wait()
        return vals

    def _finalize_on_host(self, rank, args):
        """b2_grad_norm_finalize at world > 1, restated on the host from the ranks' actual partial sums"""
        partials, nslots = args[0], int(args[1])
        max_norm, gs, fi, out_norm, out_coef, out_skip = args[8], args[9], args[10], args[11], args[12], args[13]
        # the loopback runs no GradScaler (its consensus probe cannot be exchanged here, see _lockstep)
        assert not gs and not fi, "the loopback restates the finalize without a GradScaler only"
        s = float(raw(partials, nslots, torch.float64, self.dev).cpu().sum()) if nslots else 0.0
        shares = self._share(rank, torch.tensor([s], dtype=torch.float64).to(torch.float32))
        mean = rank_mean(shares)
        norm = torch.tensor(float(mean) * self.world, dtype=torch.float64).sqrt().to(torch.float32)
        coef = torch_clip_coef(norm, float(max_norm))
        raw(out_norm, 1, torch.float32, self.dev).copy_(norm.reshape(1))
        raw(out_coef, 1, torch.float32, self.dev).copy_(coef.reshape(1))
        if out_skip:
            raw(out_skip, 1, torch.float32, self.dev).fill_(0.0)     # without a GradScaler nothing skips

    # -- driving --------------------------------------------------------------------------------------------------------
    def run(self, fn):
        """fn(rank) in N threads, one per rank; the first exception is re-raised (a broken barrier lets the others end)"""
        errs = [None] * self.world
        out = [None] * self.world

        def body(r):
            self.fake.local.rank = r
            torch.cuda.set_device(self.dev)
            try:
                out[r] = fn(r)
            except BaseException as e:       # noqa: BLE001 -- handed to the main thread
                errs[r] = e
                self.bar.abort()
                self.fake.bar.abort()

        ts = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        first = [e for e in errs if e is not None and not isinstance(e, threading.BrokenBarrierError)]
        if first:
            raise first[0]
        if any(e is not None for e in errs):
            raise [e for e in errs if e is not None][0]
        return out

    def close(self):
        """closes every wrapper still open, in N threads (collective), with fresh barriers and no planted defect"""
        self.plant = {}
        self.bar = threading.Barrier(self.world, timeout=self.bar._timeout)
        self.fake.bar = threading.Barrier(self.world, timeout=self.fake.bar._timeout)
        torch.cuda.synchronize()
        by_rank = {w.rank: w for w in self.wrappers if not w._closed}
        if len(by_rank) == self.world:
            self.run(lambda r: by_rank[r].close())
        self.wrappers = []

    def wrap(self, models, make_opt):
        """the N DistributedDataParallel wrappers and their optimizers, built in N threads"""
        def body(r):
            w = b2.DistributedDataParallel(models[r], device_ids=[0])
            self.wrappers.append(w)
            if "shift_slice" in self.plant:
                pr, idx, d = self.plant["shift_slice"]
                if pr == r:
                    sb, se = w._slices[idx]
                    w._slices[idx] = (sb + d, se + d)
            return w, make_opt(w)
        res = self.run(body)
        return [x[0] for x in res], [x[1] for x in res]

    def step(self, opts):
        self.run(lambda r: opts[r].step())
        torch.cuda.synchronize()


def rank_mean(values):
    """the flag kernels' mean of one fp32 value per rank: fp32 sum in rank order, divided by (float)world"""
    s = torch.zeros((), dtype=torch.float32)
    for v in values:
        s = s + v.reshape(()).to(torch.float32)
    return s / torch.tensor(float(len(values)), dtype=torch.float32)


def torch_clip_coef(norm, max_norm):
    """torch.nn.utils.clip_grads_with_norm_'s coefficient in fp32: clamp(max_norm / (norm + 1e-6), max=1)"""
    norm = torch.as_tensor(norm, dtype=torch.float32)
    return torch.clamp(max_norm / (norm + 1e-6), max=1.0)
