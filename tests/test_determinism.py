"""torch.use_deterministic_algorithms: the fixed-order backward.

With the flag on, two runs of the same program from the same state give bitwise-identical losses, gradients, fp32
masters, optimizer state and dropout RNG state on every training path (the engine's backward routes every
order-dependent sum to a fixed-order form: column-sum passes instead of atomic bias / LayerNorm epilogues, unsplit
N = hidden dgrads, the ordered long-attention dQ and the in-order word-embedding scatter).

CPU: Args.full_determinism sets the flag; the new entry points are declared, exported, and reject bad arguments (in a
child process that sees no device, as test_packing_long does).
GPU:
* reproducibility: each case runs twice from identical state (weights, optimizer, dropout RNG, batches; dropout 0.1)
  and every result is compared as integer bits and checked finite;
* accuracy: mode-on gradients of config A against the fp32 oracle at DESIGN §2's per-tensor bounds, and mode-on against
  mode-off on the same state;
* kernels: the ordered long attention backward (stable, dK / dV equal to the atomic form, dQ within the reordering
  bound of test_attention_packed_long) and the ordered embedding backward with heavy duplicates;
* the mode switch: a captured step raises in the other mode, and Trainer.train_step rebuilds across a flip.
The fixture below turns the flag on and restores it, and keeps torch's fill of uninitialised memory on: a buffer read
before it is written (an unvisited dQ slice) would show up as NaN.
"""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from parity import (TOL_GRAD_REL, TOL_GRAD_REL_QK, assert_grads_within_tolerance, b2, bert_ref, full_config,
                    make_model, state_from_hf_init, tiny_config, to_dev)
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.packing import pack_batch
from test_packing import short_batch
from test_packing_long import long_batch, long_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
bf = torch.bfloat16
NEW_ENTRY_POINTS = ("b2_attention_bwd_ordered", "b2_attention_bwd_packed_seq_ordered", "b2_embed_bwd_ordered",
                    "b2_embed_bwd_packed_ordered")


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_args_full_determinism_sets_the_flag():
    assert b2.Args.full_determinism is False
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        b2.Trainer(b2.Args(), None, None, None, None)
        assert not torch.are_deterministic_algorithms_enabled()
        args = b2.Args()
        args.full_determinism = True
        b2.Trainer(args, None, None, None, None)
        assert torch.are_deterministic_algorithms_enabled()
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


def test_entry_points_are_declared_and_exported():
    with open(os.path.join(ROOT, "include", "b2_ddp_bert.h")) as f:
        header = f.read()
    for name in NEW_ENTRY_POINTS:
        assert name in L._SIGNATURES and name in L.EXPORTED_SYMBOLS
        assert hasattr(L.load(), name)
        assert "int32_t %s(" % name in header
    assert L.ABI_VERSION == 23 and L.load().b2_abi_version() == 23


_CHILD = r"""
import importlib.util, json, sys
spec = importlib.util.spec_from_file_location("b2_lib_child", sys.argv[1])
L = importlib.util.module_from_spec(spec)
spec.loader.exec_module(L)
lib = L.load()
a = [(1 << 24) + i * 0x100000 for i in range(24)]
out = {}
for call in json.loads(sys.argv[2]):
    name, seq, null = call
    arg = lambda i, what: None if null == what else a[i]
    if name == "att":
        st = lib.b2_attention_bwd_ordered(a[0], arg(1, "mask"), a[2], a[3], a[4], 2, seq, 4, 64, 0.1, a[5], 4, a[6],
                                          arg(7, "parts"), None)
    elif name == "att_packed":
        st = lib.b2_attention_bwd_packed_seq_ordered(a[0], arg(1, "seg"), a[2], a[3], a[4], 2, seq, 4, 64, 0.1, a[5],
                                                     4, a[6], arg(7, "parts"), None)
    elif name == "emb":
        st = lib.b2_embed_bwd_ordered(a[0], 1, a[1], a[2], a[3], a[4], arg(5, "ids"), a[6], 2, seq, 256, 512, 2, 0,
                                      0.1, a[7], 0, a[8], a[9], a[10], a[11], a[12], a[13], a[14], 1 << 24, a[15],
                                      None)
    else:
        st = lib.b2_embed_bwd_packed_ordered(a[0], 1, a[1], a[2], a[3], a[4], a[5], a[6], arg(16, "pos"), 2, seq, 256,
                                             512, 2, 0, 0.1, a[7], 0, a[8], a[9], a[10], a[11], a[12], a[13], a[14],
                                             1 << 24, a[15], None)
    out[json.dumps(call)] = [int(st), L.last_error()]
print(json.dumps(out))
"""
BAD = [(("att", 128, None), "seq=128"), (("att", 256, "parts"), "dq_partials"),
       (("att_packed", 128, None), "seq=128"), (("att_packed", 512, "parts"), "dq_partials"),
       (("att_packed", 256, "seg"), "null segments"), (("att", 640, None), "seq=640"),
       (("emb", 128, "ids"), "null pointer"), (("emb_packed", 256, "pos"), "null pos32")]
GOOD = [("att", 256, None), ("att", 512, "mask"), ("att_packed", 384, None), ("emb", 128, None),
        ("emb_packed", 512, None)]


@pytest.fixture(scope="module")
def arg_results():
    env = dict(os.environ)
    env["CUDA_VISIBLE_DEVICES"] = ""
    calls = [list(c) for c, _ in BAD] + [list(c) for c in GOOD]
    r = subprocess.run([sys.executable, "-c", _CHILD, os.path.join(ROOT, "pytorch-distributed-nlp_b200", "_lib.py"),
                        json.dumps(calls)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("call,why", BAD, ids=lambda c: "-".join(map(str, c)) if isinstance(c, tuple) else c)
def test_bad_arguments_are_rejected(arg_results, call, why):
    st, err = arg_results[json.dumps(list(call))]
    assert st != 0 and why in err, err


@pytest.mark.parametrize("call", GOOD, ids=lambda c: "-".join(map(str, c)))
def test_good_arguments_pass_the_checks(arg_results, call):
    """valid arguments get past the checks (and then fail for want of a device)"""
    st, err = arg_results[json.dumps(list(call))]
    assert st != 0 and "null" not in err and "seq=" not in err and "dq_partials" not in err, err


# ---- GPU: reproducibility -------------------------------------------------------------------------------------------------
def _bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32 if t.element_size() == 4 else torch.int64) \
        if t.is_floating_point() else t


def _tensors(prefix, obj, out):
    """every tensor of a nested state_dict, keyed by its path"""
    if torch.is_tensor(obj):
        out[prefix] = obj.detach().cpu().clone()
    elif isinstance(obj, dict):
        for k, v in obj.items():
            _tensors("%s.%s" % (prefix, k), v, out)
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            _tensors("%s.%d" % (prefix, i), v, out)
    return out


def _snapshot(model, opt, losses):
    torch.cuda.synchronize()
    out = {"loss.%d" % i: l.detach().float().cpu().reshape(1) for i, l in enumerate(losses)}
    _tensors("grad", dict(model.grad_dict()), out)
    _tensors("master", dict(model.state_dict()), out)
    _tensors("opt", opt.state_dict(), out)
    out["rng"] = model.dropout_rng_state()
    return out


def assert_bitwise_equal(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        x, y = a[k], b[k]
        assert x.dtype == y.dtype and x.shape == y.shape, k
        if x.is_floating_point():
            assert bool(torch.isfinite(x).all()), k
        assert torch.equal(_bits(x), _bits(y)), k


OPTIMS = {"adamw": lambda m: b2.AdamW(m.parameters(), lr=1e-4, weight_decay=0.01),
          "torch_adamw": lambda m: b2.TorchAdamW(m.parameters(), lr=1e-4, weight_decay=0.01),
          "adam": lambda m: b2.Adam(m.parameters(), lr=1e-4, weight_decay=0.01),
          "sgd": lambda m: b2.SGD(m.parameters(), lr=1e-2, momentum=0.9)}


def _fresh(cfg, state, dev, optim="adamw"):
    model = make_model(cfg, state, dev).train()
    model.set_dropout_rng_state([77, 0])
    return model, OPTIMS[optim](model)


def _captured(cfg, state, dev, batches, optim="adamw", **kw):
    model, opt = _fresh(cfg, state, dev, optim)
    B, S = batches[0]["input_ids"].shape
    step = b2.FusedTrainStep(model, opt, B, S, **kw)
    k = kw.get("accum_steps", 1)
    losses = [step(b, final=(i + 1) % k == 0).clone() for i, b in enumerate(batches)]
    return _snapshot(model, opt, losses)


def _trainer(cfg, state, dev, batches, **kw):
    model, _ = _fresh(cfg, state, dev)
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank = 0, 1, 0
    for k, v in kw.items():
        setattr(args, k, v)
    opt = b2.build_optimizer(model, args)
    tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)
    losses = [tr.train_step(b).clone() for b in batches]
    return _snapshot(model, opt, losses)


def _twice(fn):
    a = fn()
    b = fn()
    assert_bitwise_equal(a, b)
    return a


def _batches(cfg, B, n, seed, S=128, **kw):
    return [short_batch(cfg, B, seed + i, S=S, **kw) for i in range(n)]


@pytest.mark.gpu
def test_captured_hidden768_cluster_layernorm(cuda_dev, deterministic):
    """config-A shapes at 2 layers, M = 32 x 128 = 4096 rows: the fused dense + LayerNorm cluster kernels"""
    cfg = full_config(num_hidden_layers=2)
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 32, 2, 10, lo=20, hi=128)
    _twice(lambda: _captured(cfg, state, cuda_dev, batches))


@pytest.mark.gpu
def test_captured_tiny_unfused(cuda_dev, deterministic):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 16, 3, 20)
    _twice(lambda: _captured(cfg, state, cuda_dev, batches))


@pytest.mark.gpu
def test_captured_padded_512(cuda_dev, deterministic):
    """the long attention backward's ordered dQ"""
    cfg = long_config()
    state = state_from_hf_init(cfg)
    batches = [long_batch(cfg, 6, 30 + i, lo=100, hi=512) for i in range(2)]
    _twice(lambda: _captured(cfg, state, cuda_dev, batches))


@pytest.mark.gpu
def test_eager_grad_scaler(cuda_dev, deterministic):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 8, 3, 40)
    _twice(lambda: _trainer(cfg, state, cuda_dev, batches, fused=False, use_amp=True))


@pytest.mark.gpu
@pytest.mark.parametrize("S", [128, 512])
def test_trainer_packed(cuda_dev, deterministic, S):
    cfg = long_config()
    state = state_from_hf_init(cfg)
    batches = ([long_batch(cfg, 8, 50 + i, lo=60, hi=400, long_rows=[(0, 480)]) for i in range(2)] if S == 512
               else _batches(cfg, 16, 2, 50))
    _twice(lambda: _trainer(cfg, state, cuda_dev, batches, pack=True))


@pytest.mark.gpu
def test_trainer_accumulation(cuda_dev, deterministic):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 8, 4, 60)
    _twice(lambda: _trainer(cfg, state, cuda_dev, batches, gradient_accumulation_steps=2))


@pytest.mark.gpu
def test_trainer_max_grad_norm(cuda_dev, deterministic):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 8, 3, 70)
    _twice(lambda: _trainer(cfg, state, cuda_dev, batches, max_grad_norm=0.05))


@pytest.mark.gpu
def test_eager_no_sync_accumulation(cuda_dev, deterministic):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 8, 4, 75)
    _twice(lambda: _trainer(cfg, state, cuda_dev, batches, fused=False, gradient_accumulation_steps=2))


@pytest.mark.gpu
@pytest.mark.parametrize("optim", sorted(OPTIMS))
def test_each_optimizer(cuda_dev, deterministic, optim):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 8, 2, 80)
    _twice(lambda: _captured(cfg, state, cuda_dev, batches, optim=optim))


@pytest.mark.gpu
def test_repeated_word_rows(cuda_dev, deterministic):
    """ids from 50 tokens: every word row occurs many times"""
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 16, 2, 90, lo=60, hi=128)
    for b in batches:
        b["input_ids"] = (b["input_ids"] % 50 + 1) * b["attention_mask"]
    _twice(lambda: _captured(cfg, state, cuda_dev, batches))


# ---- GPU: accuracy --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_full_size_gradients_vs_oracle(cuda_dev, deterministic):
    """config A (12 layers, batch 32 x 128), dropout off, mode on: every gradient tensor within DESIGN §2's per-tensor
    rel-L2 bound of the fp32 oracle"""
    from oracle import cpu_step
    cfg = full_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    model = make_model(cfg, state, cuda_dev).train()
    batch = bert_ref.synthetic_batch(cfg, 32, 128, 1000, padded=True)
    d = to_dev(batch, cuda_dev)
    out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                labels=d["label"])
    F.cross_entropy(out[1], d["label"]).backward()
    torch.cuda.synchronize()
    torch.set_num_threads(cpu_step.usable_cores())
    _, _, ref = bert_ref.loss_and_grads(state, cfg, batch)
    qk, other = assert_grads_within_tolerance(model.grad_dict(), ref)
    print("config A, mode on: worst grad rel-L2 q/k %.2e, others %.2e" % (qk, other))


@pytest.mark.gpu
@pytest.mark.parametrize("S", [128, 512])
def test_mode_on_agrees_with_mode_off(cuda_dev, S):
    """the same backward in both modes, hidden 768: the two differ only by the order of fp32 sums (and the bf16
    roundings they move), so every gradient tensor agrees to well within the oracle bound (a quarter of it)"""
    cfg = full_config(num_hidden_layers=2, max_position_embeddings=512, hidden_dropout_prob=0.0,
                      attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    batch = long_batch(cfg, 8, 5, lo=S // 4, hi=S, S=S)
    model = make_model(cfg, state, cuda_dev).train()
    d = to_dev(batch, cuda_dev)
    grads = {}
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                        attention_mask=d["attention_mask"], labels=d["label"])
            F.cross_entropy(out[1], d["label"]).backward()
            torch.cuda.synchronize()
            grads[det] = model.grad_dict()
    finally:
        torch.use_deterministic_algorithms(was)
    scale = max(float(v.double().norm()) for v in grads[False].values())
    for k, off in grads[False].items():
        on = grads[True][k]
        assert bool(torch.isfinite(on).all()), k
        n = max(float(off.double().norm()), 1e-3 * scale)
        rel = float((on.double() - off.double()).norm()) / n
        assert rel <= 0.25 * (TOL_GRAD_REL_QK if ("query" in k or "key" in k) else TOL_GRAD_REL), (k, rel)


# ---- GPU: kernels ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("S", [256, 512])
def test_ordered_long_attention_backward(cuda_dev, S, packed):
    """stable across launches whatever the partials buffer held (never-visited slices are not read: NaN there changes
    nothing); dK, dV bitwise the atomic form's; dQ within the atomic form's reordering bound plus one bf16 step"""
    from test_attention import SEED, SITE, STEP, attn_fwd, stream
    from test_attention_packed_long import _bf16_step, dq_reorder_bound, fwd, long_layout
    from parity import packed_visibility, padded_visibility
    torch.manual_seed(S + packed)
    nh, p = 4, 0.1
    H = nh * 64
    if packed:
        seg = long_layout(S).to(cuda_dev)            # includes bins whose CTAs skip query blocks
        B = seg.shape[0]
        mask = None
    else:
        B = 3
        mask = (torch.arange(S)[None] < torch.tensor([[S], [S - 130], [70]])).to(torch.int64).to(cuda_dev)
    qkv = torch.randn(B * S, 3 * H, device=cuda_dev).to(bf)
    dctx = torch.randn(B * S, H, device=cuda_dev).to(bf)
    ctx, lse = fwd(qkv, seg, S, nh, p) if packed else attn_fwd(qkv, B, S, nh, p, mask=mask)
    rs = torch.tensor([SEED, STEP], dtype=torch.int64, device=cuda_dev)
    first = seg.data_ptr() if packed else L.ptr(mask)

    def atomic():
        dqkv = torch.zeros(B * S, 3 * H, dtype=bf, device=cuda_dev)
        acc = torch.empty(B * S, H, dtype=torch.float32, device=cuda_dev)
        name = "b2_attention_bwd_packed_seq" if packed else "b2_attention_bwd"
        L.call(name, qkv.data_ptr(), first, ctx.data_ptr(), dctx.data_ptr(), lse.data_ptr(), B, S, nh, 64, p,
               rs.data_ptr(), SITE, dqkv.data_ptr(), acc.data_ptr(), None, None, stream())
        return dqkv

    def ordered(fill):
        dqkv = torch.zeros(B * S, 3 * H, dtype=bf, device=cuda_dev)
        parts = torch.full((S // 128, B * S, H), fill, dtype=torch.float32, device=cuda_dev)
        name = "b2_attention_bwd_packed_seq_ordered" if packed else "b2_attention_bwd_ordered"
        L.call(name, qkv.data_ptr(), first, ctx.data_ptr(), dctx.data_ptr(), lse.data_ptr(), B, S, nh, 64, p,
               rs.data_ptr(), SITE, dqkv.data_ptr(), parts.data_ptr(), stream())
        return dqkv

    a = atomic()
    o1, o2, o3 = ordered(float("nan")), ordered(0.0), ordered(float("nan"))
    torch.cuda.synchronize()
    assert bool(torch.isfinite(o1.float()).all())
    assert torch.equal(o1, o2) and torch.equal(o1, o3)
    assert torch.equal(o1[:, H:], a[:, H:])                      # dK | dV
    vis = packed_visibility(seg) if packed else padded_visibility(mask, S)
    bound = dq_reorder_bound(qkv, dctx, vis, B, S, nh, p)
    err = (o1[:, :H].double() - a[:, :H].double()).abs()
    tol = bound + _bf16_step(a[:, :H].double().abs() + bound).double()
    assert bool((err <= tol).all()), float((err / tol).max())


@pytest.mark.gpu
@pytest.mark.parametrize("packed", [False, True])
def test_ordered_embedding_backward(cuda_dev, packed):
    """heavy duplicates (ids from 20 tokens): d_word bitwise stable and within one bf16 rounding (plus fp32 summation
    error) of the float64 sum of the token rows; position, type and LayerNorm gradients stable too"""
    torch.manual_seed(3 + packed)
    B, S, H, V, T = 8, 256, 256, 512, 2
    M = B * S
    dev = cuda_dev
    dy = torch.randn(M, H, device=dev)
    pre = torch.randn(M, H, device=dev).to(bf)
    mean = pre.float().mean(1)
    rstd = torch.rsqrt(pre.float().var(1, unbiased=False) + 1e-12)
    gamma = (1 + 0.1 * torch.randn(H, device=dev)).to(bf)
    ids32 = torch.randint(1, 21, (M,), dtype=torch.int32, device=dev)
    ids32[::37] = 0                                      # pad rows get no gradient
    tt32 = torch.randint(0, T, (M,), dtype=torch.int32, device=dev)
    pos32 = torch.randint(0, S, (M,), dtype=torch.int32, device=dev)
    owner = torch.empty(V, dtype=torch.int32, device=dev)
    L.call("b2_embed_owner_init", owner.data_ptr(), V, torch.cuda.current_stream().cuda_stream)
    rs = torch.tensor([5, 0], dtype=torch.int64, device=dev)

    def run():
        outs = [torch.zeros(n, H, dtype=bf, device=dev) for n in (V, S, T, 1, 1)]
        dx = torch.empty(M, H, dtype=bf, device=dev)
        scratch = torch.empty(8 << 20, dtype=torch.uint8, device=dev)
        head = (dy.data_ptr(), 1, pre.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(), ids32.data_ptr(),
                tt32.data_ptr())
        tail = (B, S, H, V, T, 0, 0.1, rs.data_ptr(), 0, *[o.data_ptr() for o in outs], dx.data_ptr(),
                scratch.data_ptr(), scratch.numel(), owner.data_ptr(), torch.cuda.current_stream().cuda_stream)
        if packed:
            L.call("b2_embed_bwd_packed_ordered", *head, pos32.data_ptr(), *tail)
        else:
            L.call("b2_embed_bwd_ordered", *head, *tail)
        torch.cuda.synchronize()
        return outs, dx

    (w1, *r1), dx1 = run()
    (w2, *r2), dx2 = run()
    assert torch.equal(w1.view(torch.int16), w2.view(torch.int16)) and torch.equal(dx1, dx2)
    for x, y in zip(r1, r2):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16))
    ref = torch.zeros(V, H, dtype=torch.float64, device=dev)
    ref.index_put_((ids32.long(),), dx1.double(), accumulate=True)
    ref[0] = 0
    absum = torch.zeros(V, H, dtype=torch.float64, device=dev)
    absum.index_put_((ids32.long(),), dx1.double().abs(), accumulate=True)
    n = torch.bincount(ids32.long(), minlength=V).double()[:, None]
    got = w1.double()
    tol = 2.0 ** -8 * ref.abs() + n * 2.0 ** -24 * absum + 2.0 ** -133
    assert bool(((got - ref).abs() <= tol).all())
    assert bool((w1[0] == 0).all()) and bool(torch.isfinite(w1.float()).all())


# ---- GPU: the mode switch ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_captured_step_raises_in_the_other_mode(cuda_dev):
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batch = _batches(cfg, 8, 1, 95)[0]
    was = torch.are_deterministic_algorithms_enabled()
    try:
        for built in (False, True):
            torch.use_deterministic_algorithms(built)
            model, opt = _fresh(cfg, state, cuda_dev)
            step = b2.FusedTrainStep(model, opt, 8, 128)
            step(batch)
            torch.use_deterministic_algorithms(not built)
            with pytest.raises(RuntimeError, match="use_deterministic_algorithms"):
                step(batch)
    finally:
        torch.use_deterministic_algorithms(was)


@pytest.mark.gpu
def test_trainer_recovers_across_a_flip(cuda_dev):
    """train_step in mode off, on, off: each mode gets its own captured step, and the mode-on steps reproduce"""
    cfg = tiny_config()
    state = state_from_hf_init(cfg)
    batches = _batches(cfg, 8, 3, 97)
    was = torch.are_deterministic_algorithms_enabled()

    def run():
        model, _ = _fresh(cfg, state, cuda_dev)
        args = b2.Args()
        args.local_rank, args.local_world_size, args.rank = 0, 1, 0
        opt = b2.build_optimizer(model, args)
        tr = b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)
        losses = []
        for det, b in zip((False, True, True), batches):
            torch.use_deterministic_algorithms(det)
            losses.append(tr.train_step(b).clone())
            assert tr._fused.deterministic == det
        torch.use_deterministic_algorithms(False)
        losses.append(tr.train_step(batches[0]).clone())
        return model, opt, losses

    try:
        m, o, l = run()
        assert int(o._state()["step"]) == 4
        assert all(bool(torch.isfinite(x).all()) for x in l)
    finally:
        torch.use_deterministic_algorithms(was)


# ---- DDP ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_ddp_runs_reproduce_per_rank():
    world = 2
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29611", os.path.join(ROOT, "tests", "ddp_determinism_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_determinism_worker: OK" in r.stdout
