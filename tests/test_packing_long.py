"""Packing past 128 tokens: bins of 256, 384 and 512 tokens (packing.bin_length) through the packed attention entry
points b2_attention_{fwd,bwd}_packed_seq, the packed step, Trainer(pack=True) and DDP.

CPU: pack_batch's layout at bin_len 256 / 512, the bin length the Trainer picks from a batch's lengths, and the
arguments the new entry points reject (in a child process that sees no device, as test_attention_reference does).
GPU: the packed step at bins of 256 and 512 against the fp32 oracle run on the PADDED batch and against the padded
CUDA step; Trainer(pack=True) on 512-padded long-text batches against the oracle's trajectory, with accumulation, with
clipping, and next to 128-padded batches; a world-2 DDP worker (skipped with fewer than 2 GPUs).
"""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from parity import (TOL_GRAD_REL_QK, TOL_LOGITS, TOL_LOSS, TOL_TRAJ, assert_grads_within_tolerance, b2, bert_ref,
                    full_config, make_model, state_from_hf_init, tiny_config, to_dev)
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.packing import bin_length, pack_batch
from test_packing import short_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def long_batch(cfg, B, seed, lo=16, hi=512, S=512, long_rows=()):
    """short_batch's rows padded to S with lengths ~ U{lo..hi}; `long_rows`: (row, length) overrides"""
    b = short_batch(cfg, B, seed, lo=lo, hi=hi, S=S)
    for r, n in long_rows:
        b["attention_mask"][r] = (torch.arange(S) < n).to(torch.int64)
    g = torch.Generator().manual_seed(seed + 1)
    ids = torch.randint(1, cfg.vocab_size, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0] = min(101, cfg.vocab_size - 1)
    b["input_ids"] = ids * b["attention_mask"]
    b["token_type_ids"] = b["token_type_ids"] * b["attention_mask"]
    return b


def long_config(**kw):
    return tiny_config(max_position_embeddings=512, **kw)


# ---- CPU: layout ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bin_len", [256, 512])
def test_pack_batch_long_bins(bin_len):
    cfg = long_config()
    b = long_batch(cfg, 23, bin_len, lo=1, hi=bin_len // 2, S=bin_len, long_rows=[(4, bin_len), (9, 300 % bin_len + 1)])
    p = pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], bin_len)
    lens = b["attention_mask"].sum(1)
    NB = p["bins"]
    assert p["input_ids"].shape == (NB, bin_len) and p["segments"].shape == (NB, bin_len)
    assert NB * bin_len >= int(lens.sum()) and NB < 23
    seen = torch.zeros(NB, bin_len, dtype=torch.bool)
    for i in range(23):
        k, lo = divmod(int(p["cls_index"][i]), bin_len)
        n = int(lens[i])
        assert lo + n <= bin_len and not seen[k, lo:lo + n].any()
        seen[k, lo:lo + n] = True
        assert torch.equal(p["input_ids"][k, lo:lo + n], b["input_ids"][i, :n])
        assert torch.equal(p["token_type_ids"][k, lo:lo + n], b["token_type_ids"][i, :n])
        assert torch.equal(p["position_ids"][k, lo:lo + n], torch.arange(n))
        seg = p["segments"][k, lo:lo + n]
        assert bool(((seg & 0xffff) == lo).all()) and bool(((seg >> 16) == lo + n).all())
    un = ~seen
    rows = torch.arange(bin_len).repeat(NB, 1)[un]
    assert bool((p["input_ids"][un] == 0).all()) and bool((p["position_ids"][un] == 0).all())
    assert bool(((p["segments"][un] & 0xffff) == rows).all()) and bool(((p["segments"][un] >> 16) == rows + 1).all())


def test_a_300_token_sequence_fills_one_512_bin():
    cfg = long_config()
    b = long_batch(cfg, 5, 3, lo=10, hi=50, long_rows=[(2, 300)])
    p = pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], 512)
    k, lo = divmod(int(p["cls_index"][2]), 512)
    assert lo == 0                                               # longest first: it opens a bin
    assert bool((p["segments"][k, :300] == (0 | (300 << 16))).all())
    assert torch.equal(p["position_ids"][k, :300], torch.arange(300))
    assert p["bins"] == 1                                        # the short rows fill the rest of that bin


def test_bin_length_follows_the_longest_row():
    cfg = long_config()
    assert bin_length(short_batch(cfg, 8, 1)["attention_mask"], 128) == 128                      # 128-padded
    assert bin_length(long_batch(cfg, 8, 2, lo=5, hi=120)["attention_mask"], 512) == 128         # 512-padded, short
    assert bin_length(long_batch(cfg, 8, 3, lo=5, hi=60, long_rows=[(3, 300)])["attention_mask"], 512) == 384
    assert bin_length(long_batch(cfg, 8, 4, lo=5, hi=60, long_rows=[(0, 129)])["attention_mask"], 512) == 256
    assert bin_length(long_batch(cfg, 8, 5, lo=5, hi=60, long_rows=[(7, 512)])["attention_mask"], 512) == 512
    assert bin_length(short_batch(cfg, 8, 6, hi=64, S=64)["attention_mask"], 64) == 128          # max_seq_len = 64
    assert bin_length(None, 200) == 256


# ---- CPU: the entry points' argument checks ---------------------------------------------------------------------------
_CHILD = r"""
import importlib.util, json, sys
spec = importlib.util.spec_from_file_location("b2_lib_child", sys.argv[1])
L = importlib.util.module_from_spec(spec)
spec.loader.exec_module(L)
lib = L.load()
a = [(1 << 24) + i * 0x100000 for i in range(10)]   # qkv, seg, ctx, d_ctx, lse, rng, keep_bits, d_qkv, dq_accum, dbias
out = {}
for name, seg, seq, dq, db in json.loads(sys.argv[2]):
    s = a[1] if seg else None
    if name == "fwd":
        st = lib.b2_attention_fwd_packed_seq(a[0], s, 2, seq, 4, 64, 0.1, a[5], 4, a[2], a[4], a[6], None)
    else:
        st = lib.b2_attention_bwd_packed_seq(a[0], s, a[2], a[3], a[4], 2, seq, 4, 64, 0.1, a[5], 4, a[7],
                                             a[8] if dq else None, a[9] if db else None, a[6], None)
    out[json.dumps([name, seg, seq, dq, db])] = [int(st), L.last_error()]
print(json.dumps(out))
"""
BAD = [("fwd", False, 256, True, False, "null segments"), ("bwd", False, 256, True, False, "null segments"),
       ("fwd", True, 100, True, False, "seq=100"), ("bwd", True, 100, True, False, "seq=100"),
       ("fwd", True, 640, True, False, "seq=640"), ("bwd", True, 640, True, False, "seq=640"),
       ("fwd", True, 0, True, False, "empty"), ("bwd", True, 0, True, False, "empty"),
       ("bwd", True, 256, False, False, "dq_accum"), ("bwd", True, 512, True, True, "fused QKV bias")]
GOOD = [("fwd", True, 128, False, False), ("fwd", True, 256, False, False), ("fwd", True, 512, False, False),
        ("bwd", True, 128, False, True), ("bwd", True, 384, True, False), ("bwd", True, 512, True, False)]


@pytest.fixture(scope="module")
def arg_results():
    env = dict(os.environ)
    env["CUDA_VISIBLE_DEVICES"] = ""
    calls = [c[:5] for c in BAD] + list(GOOD)
    r = subprocess.run([sys.executable, "-c", _CHILD, os.path.join(ROOT, "pytorch-distributed-nlp_b200", "_lib.py"),
                        json.dumps(calls)], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_entry_points_are_declared_and_exported():
    for name in ("b2_attention_fwd_packed_seq", "b2_attention_bwd_packed_seq"):
        assert name in L._SIGNATURES and name in L.EXPORTED_SYMBOLS
        assert hasattr(L.load(), name)
    assert L.ABI_VERSION == 23 and L.load().b2_abi_version() == 23


@pytest.mark.parametrize("call", BAD, ids=lambda c: "%s-seg%d-seq%d-dq%d-db%d" % c[:5])
def test_bad_arguments_are_rejected(arg_results, call):
    st, err = arg_results[json.dumps(list(call[:5]))]
    assert st != 0 and call[5] in err, err


@pytest.mark.parametrize("call", GOOD, ids=lambda c: "%s-seq%d" % (c[0], c[2]))
def test_good_arguments_pass_the_checks(arg_results, call):
    """the same calls with valid arguments get past the checks (and then fail for want of a device)"""
    st, err = arg_results[json.dumps(list(call))]
    assert st != 0 and "null" not in err and "seq=" not in err and "dq_accum" not in err and "bias" not in err, err


# ---- GPU: the packed step ---------------------------------------------------------------------------------------------
def _run(model, dev, batch, packed=None):
    if packed is None:
        d = to_dev(batch, dev)
        out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"], attention_mask=d["attention_mask"],
                    labels=d["label"])
    else:
        out = model(input_ids=packed["input_ids"].to(dev), token_type_ids=packed["token_type_ids"].to(dev),
                    labels=batch["label"].to(dev), position_ids=packed["position_ids"].to(dev),
                    segments=packed["segments"].to(dev), cls_index=packed["cls_index"].to(dev))
    loss = F.cross_entropy(out[1], batch["label"].to(dev))
    loss.backward()
    torch.cuda.synchronize()
    return out, loss


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["tiny", "hidden768"])
@pytest.mark.parametrize("bin_len", [256, 512])
def test_long_packed_step_equals_padded_step(cuda_dev, which, bin_len):
    """dropout off: a 512-padded batch packed into bins of `bin_len`; logits, loss and every gradient against the fp32
    oracle on the PADDED batch (DESIGN §2's tolerances, seq-512 exception for the q/k projections), and against the
    padded CUDA step on the same weights"""
    kw = dict(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    cfg, B = (long_config(**kw), 12) if which == "tiny" else (full_config(num_hidden_layers=3, **kw), 16)
    state = state_from_hf_init(cfg)
    rows = [(0, bin_len), (5, bin_len - 77)]
    batch = long_batch(cfg, B, 40 + bin_len, lo=8, hi=bin_len // 2, long_rows=rows)
    assert bin_length(batch["attention_mask"], 512) == bin_len
    packed = pack_batch(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"], bin_len)
    assert packed["bins"] < B
    rl, rz, rg = bert_ref.loss_and_grads(state, cfg, batch)
    model = make_model(cfg, state, cuda_dev).train()
    out_p, loss_p = _run(model, cuda_dev, batch, packed)
    g_packed = model.grad_dict()
    assert out_p[1].shape == (B, cfg.num_labels)
    assert abs(float(loss_p) - float(rl)) <= TOL_LOSS and abs(float(out_p[0]) - float(rl)) <= TOL_LOSS
    assert float((out_p[1].detach().cpu() - rz).abs().max()) <= TOL_LOGITS
    qk, other = assert_grads_within_tolerance(g_packed, rg, qk_tol=TOL_GRAD_REL_QK)
    print("%s bins of %d: worst grad rel-L2 q/k %.2e, others %.2e" % (which, bin_len, qk, other))
    out_d, loss_d = _run(model, cuda_dev, batch)                   # the padded step on the same weights
    g_padded = model.grad_dict()
    assert float((out_d[1].detach() - out_p[1].detach()).abs().max()) <= TOL_LOGITS
    assert abs(float(loss_d) - float(loss_p)) <= TOL_LOSS
    assert_grads_within_tolerance(g_packed, {k: v.detach().cpu() for k, v in g_padded.items()},
                                  qk_tol=TOL_GRAD_REL_QK)


# ---- GPU: the Trainer -------------------------------------------------------------------------------------------------
def _trainer(cfg, state, dev, **kw):
    model = make_model(cfg, state, dev)
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank, args.pack = 0, 1, 0, True
    for k, v in kw.items():
        setattr(args, k, v)
    opt = b2.build_optimizer(model, args)
    return model, opt, b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)


def _oracle(state, cfg, steps, max_norm=None, lr=3e-5):
    """ddp_ref.train's loop (HF AdamW on the mean gradient of each step's micro-batches), with torch's
    clip_grad_norm_ (coef = max_norm / (norm + 1e-6), at most 1) before the update when max_norm is set"""
    from oracle import adamw_ref, ddp_ref
    params = {k: v.clone() for k, v in state.items()}
    opt = adamw_ref.HFAdamW(params, lr=lr, weight_decay=0.01)
    losses = []
    for micro in steps:
        out = [bert_ref.loss_and_grads(params, cfg, b) for b in micro]
        losses.append([float(o[0]) for o in out])
        g = ddp_ref.mean_grads([o[2] for o in out])
        if max_norm:
            norm = torch.sqrt(sum((v.double() ** 2).sum() for v in g.values()))
            coef = min(1.0, max_norm / (float(norm) + 1e-6))
            g = {k: v * coef for k, v in g.items()}
        opt.step(g)
    return losses, params


LONG_TEXT = [dict(lo=20, hi=200, long_rows=[(1, 480)]), dict(lo=8, hi=60), dict(lo=100, hi=400),
             dict(lo=8, hi=100, long_rows=[(3, 200)]), dict(lo=200, hi=512)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "accum2", "clip"])
def test_trainer_packs_512_padded_batches(cuda_dev, mode):
    """Trainer(pack=True) on 512-padded long-text batches (bins of 128 to 512 tokens) follows the oracle's loss
    trajectory on the PADDED batches; with gradient_accumulation_steps = 2 and with max_grad_norm"""
    cfg = long_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    k = 2 if mode == "accum2" else 1
    clip = 0.5 if mode == "clip" else None
    batches = [long_batch(cfg, 8, 700 + i, **LONG_TEXT[i % 5]) for i in range(5 * k)]
    lens = {bin_length(b["attention_mask"], 512) for b in batches}
    assert len(lens) >= 3, lens
    ref_losses, ref = _oracle(state, cfg, [batches[i * k:(i + 1) * k] for i in range(5)], clip)
    model, opt, tr = _trainer(cfg, state, cuda_dev, gradient_accumulation_steps=k, max_grad_norm=clip)
    for i, b in enumerate(batches):
        loss = float(tr.train_step(b))
        want = ref_losses[i // k][i % k]
        assert abs(loss - want) <= TOL_TRAJ, (mode, i, loss, want)
    assert int(opt._state()["step"]) == 5
    assert {key[2] for key in tr._packed} == lens                # one captured step per bin length in use
    sd = model.state_dict()
    for name, v in ref.items():
        assert float((sd[name].cpu() - v).abs().max()) <= 2e-4, name


@pytest.mark.gpu
def test_trainer_mixes_128_and_512_padded_batches(cuda_dev):
    """128- and 512-padded batches alternate: each (bins, batch, bin length) gets its own graph, and the loss follows the
    oracle; max_seq_len = 64 batches pack into 128-token bins instead of raising"""
    cfg = long_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    batches = [short_batch(cfg, 8, 800), long_batch(cfg, 8, 801, lo=100, hi=250, long_rows=[(0, 300)]),
               short_batch(cfg, 8, 802, hi=60, S=64),
               long_batch(cfg, 8, 803, lo=5, hi=100), short_batch(cfg, 8, 804)]
    ref_losses, ref = _oracle(state, cfg, [[b] for b in batches])
    model, opt, tr = _trainer(cfg, state, cuda_dev)
    for i, b in enumerate(batches):
        loss = float(tr.train_step(b))
        assert abs(loss - ref_losses[i][0]) <= TOL_TRAJ, (i, loss, ref_losses[i][0])
    assert {key[2] for key in tr._packed} == {128, 384}
    assert len(tr._packed) >= 3
    sd = model.state_dict()
    for name, v in ref.items():
        assert float((sd[name].cpu() - v).abs().max()) <= 2e-4, name


@pytest.mark.gpu
def test_128_padded_batches_pack_as_before(cuda_dev):
    """a 128-padded batch takes bin length 128, and Trainer(pack=True) computes on it what it computed before bins
    could be longer: one step from the initial weights leaves the bf16 gradient of every weight matrix and embedding
    table bit for bit what that build computed (golden/pack128_trainer_grads.json, sha256 of grad_dict's fp32 copies,
    per batch).  The gradients of the biases and LayerNorm weights are fp32 column sums added by atomics in no fixed
    order, so they differ between runs of either build in the last bits; they are not fingerprinted."""
    import hashlib
    with open(os.path.join(ROOT, "tests", "golden", "pack128_trainer_grads.json")) as f:
        gold = json.load(f)["sha256_16"]
    cfg = tiny_config(hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    state = state_from_hf_init(cfg)
    batches = [short_batch(cfg, 16, 900 + i, hi=(30 if i % 2 else 90)) for i in range(4)]
    colsum = lambda k: k.endswith(".bias") or k.endswith("LayerNorm.weight")
    digest = lambda t: hashlib.sha256(t.detach().float().cpu().contiguous().numpy().tobytes()).hexdigest()[:16]
    for b, want in zip(batches, gold):
        model, _, tr = _trainer(cfg, state, cuda_dev)
        tr.train_step(b)
        torch.cuda.synchronize()
        assert [key[2] for key in tr._packed] == [128]
        got = {k: digest(v) for k, v in model.grad_dict().items() if not colsum(k)}
        assert sorted(got) == sorted(want)
        for name, h in want.items():
            assert got[name] == h, name


@pytest.mark.gpu
def test_ddp_packs_long_batches_per_rank():
    world = 2
    if not torch.cuda.is_available() or torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29605", os.path.join(ROOT, "tests", "ddp_pack_long_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "ddp_pack_long_worker: OK" in r.stdout
