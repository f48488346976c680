"""CPU: the C-ABI library loads and exports what include/b2_ddp_bert.h declares; host-side logic of the drop-in layer
(parameter naming/layout, optimizer grouping, bucket slicing, error behaviour without a GPU)."""
import ctypes
import os
import re

import pytest
import torch

from parity import b2, tiny_config, full_config
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.modeling import _Layout, _hf_order

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_loads_and_exports_every_declared_symbol():
    lib = L.load()
    assert lib.b2_abi_version() == L.ABI_VERSION
    hdr = open(os.path.join(ROOT, "include", "b2_ddp_bert.h")).read()
    declared = set(re.findall(r"\b(b2_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    raw = ctypes.CDLL(L.LIB_PATH)
    for sym in sorted(declared):
        assert hasattr(raw, sym), "library does not export %s" % sym
    assert declared == set(L.EXPORTED_SYMBOLS), declared ^ set(L.EXPORTED_SYMBOLS)


def test_error_convention_without_gpu():
    a = L.GemmArgs()
    with pytest.raises(RuntimeError, match="empty problem"):
        L.call("b2_gemm_bf16", a, None)
    assert "empty problem" in L.last_error()


def test_no_cpu_fallback():
    model = b2.BertForSequenceClassification(tiny_config())
    ids = torch.zeros(2, 128, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="no CPU path"):
        model(input_ids=ids)


def test_parameter_names_order_and_count_match_hf():
    from oracle import cpu_step
    cfg = full_config()
    names = _hf_order(cfg)
    assert len(names) == 201
    lay = _Layout(cfg)
    assert set(lay.entries) == set(names)
    n_params = sum(int(torch.tensor(s).prod()) for _, s in lay.entries.values())
    assert n_params == 102_272_262                      # SURVEY.md §2.2 K14
    assert lay.total % 8 == 0 and all(off % 8 == 0 for off, _ in lay.entries.values())
    assert len(lay.buckets) == 13                       # embeddings | layers 0..10 | layer 11 + head
    assert lay.buckets[0][0] == 0 and lay.buckets[-1][1] == lay.total
    for (b0, e0, _), (b1, _e1, _) in zip(lay.buckets, lay.buckets[1:]):
        assert e0 == b1
    tcfg = tiny_config()
    m = b2.BertForSequenceClassification(tcfg)
    hf = cpu_step.build_hf_model(tcfg)
    assert [n for n, _ in m.named_parameters()] == [n for n, _ in hf.named_parameters()]
    for (n, p), (_, q) in zip(m.named_parameters(), hf.named_parameters()):
        assert tuple(p.shape) == tuple(q.shape), n
    # Q/K/V are adjacent in the flat space so one [3H, H] GEMM serves them
    q, k, v = (lay.off("bert.encoder.layer.3.attention.self.%s.weight" % t) for t in ("query", "key", "value"))
    H = cfg.hidden_size
    assert k - q == H * H and v - k == H * H


def test_parameters_are_views_of_one_flat_buffer_and_init_is_hf_like():
    torch.manual_seed(0)
    cfg = tiny_config()
    m = b2.BertForSequenceClassification(cfg)
    base = m._flat.data_ptr()
    for n, p in m.named_parameters():
        off, _ = m._layout.entries[n]
        assert p.data_ptr() == base + 4 * off
    sd = m.state_dict()
    assert float(sd["bert.embeddings.word_embeddings.weight"][0].abs().max()) == 0.0      # pad row
    assert float(sd["bert.embeddings.LayerNorm.weight"].min()) == 1.0
    assert float(sd["classifier.bias"].abs().max()) == 0.0
    std = float(sd["bert.encoder.layer.0.intermediate.dense.weight"].std())
    assert 0.018 < std < 0.022
    with pytest.raises(RuntimeError, match="size mismatch"):
        m.load_state_dict({**sd, "classifier.weight": torch.zeros(3, 3)})
    with pytest.raises(RuntimeError, match="missing"):
        m.load_state_dict({})


def test_build_optimizer_grouping_matches_reference_rule():
    class A:
        weight_decay, learning_rate = 0.01, 3e-5
    cfg = tiny_config()
    m = b2.BertForSequenceClassification(cfg)
    opt = b2.build_optimizer(m, A)
    assert len(opt.param_groups) == 2
    decay_names = {p._b2_name for p in opt.param_groups[0]["params"]}
    nodecay_names = {p._b2_name for p in opt.param_groups[1]["params"]}
    assert all(("bias" not in n and "LayerNorm.weight" not in n) for n in decay_names)
    assert all(("bias" in n or "LayerNorm.weight" in n) for n in nodecay_names)
    assert opt.param_groups[0]["eps"] == 1e-6 and opt.param_groups[0]["betas"] == (0.9, 0.999)
    flags = opt._decay_flags_cpu
    for n, (off, shape) in m._layout.entries.items():
        want = 1 if n in decay_names else 0
        assert int(flags[off // 8]) == want, n
    with pytest.raises(ValueError, match="every parameter"):
        b2.AdamW([m._params_by_name["classifier.weight"]], lr=1e-3)
    with pytest.raises(TypeError, match="b200"):
        b2.AdamW([torch.nn.Parameter(torch.zeros(3))], lr=1e-3)
    with pytest.raises(RuntimeError, match="not on CUDA"):
        opt.step()


def test_bucket_slices_partition_every_bucket():
    """the per-rank slices the DDP wrapper hands to b2_bucket_reduce_adamw tile each bucket exactly, 8-aligned"""
    from pytorch_distributed_nlp_b200.ddp import DistributedDataParallel as D
    lay = _Layout(full_config())
    for world in (2, 4, 8):
        for (b, e, _label) in lay.buckets:
            covered = 0
            prev = b
            for r in range(world):
                fake = type("F", (), {})()
                fake.module = type("M", (), {"_layout": type("L", (), {"buckets": [(b, e, "x")]})()})()
                fake.world, fake.rank = world, r
                (sb, se), = D._make_slices(fake)
                assert sb % 8 == 0 and se % 8 == 0 and sb == prev and se >= sb
                covered += se - sb
                prev = se
            assert covered == e - b and prev == e


def test_output_object_indexing():
    o = b2.SequenceClassifierOutput(loss=torch.tensor(1.0), logits=torch.zeros(2, 6))
    assert o[0] is o.loss and o[1] is o.logits and len(o) == 2 and o["logits"] is o.logits
    o2 = b2.SequenceClassifierOutput(logits=torch.zeros(2, 6))
    assert o2[0] is o2.logits and len(o2) == 1


def test_package_synthetic_batch_is_the_oracles():
    """bench.py's b200 arm draws its inputs from the package (nothing of oracle/ on that arm); the parity tests draw
    theirs from the oracle: same generator, same tensors"""
    from oracle import bert_ref
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    for padded in (False, True):
        a = b2.synthetic_batch(cfg, 5, 128, 1234, padded=padded)
        b = bert_ref.synthetic_batch(cfg, 5, 128, 1234, padded=padded)
        assert set(a) == set(b) == {"input_ids", "token_type_ids", "attention_mask", "label"}
        for k in a:
            assert a[k].dtype == torch.int64 and torch.equal(a[k], b[k])


def test_philox_replica_known_answers():
    """The numpy Philox4x32-10 that the GPU dropout masks are compared with (tests/parity.py) reproduces the
    known-answer vectors published with Random123 (kat_vectors: philox4x32, 10 rounds) -- so "the kernels' masks equal
    the replica's" (asserted bit for bit in the -m gpu tests) means "the kernels run the published generator"."""
    import numpy as np
    from parity import philox4x32_10
    kat = [
        ((0x00000000,) * 4, (0x00000000,) * 2, (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
        ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
        ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
         (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
    ]
    for ctr, key, want in kat:
        c = [np.array([v], dtype=np.uint64) for v in ctr]
        out = philox4x32_10(c[0], c[1], c[2], c[3], key[0], key[1])
        assert tuple(int(o[0]) for o in out) == want, (ctr, [hex(int(o[0])) for o in out])


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the driver's CPU arm): rank 0 prints ONE JSON line with the contract's keys, any
    other rank exits 0 silently (the driver launches the arm under torchrun for N > 1)."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, RANK="1", WORLD_SIZE="2", LOCAL_RANK="1")
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--gpus", "2",
                        "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0 and r.stdout.strip() == "", r.stdout[-500:] + r.stderr[-500:]
    env = dict(os.environ, RANK="0", WORLD_SIZE="1", LOCAL_RANK="0")
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--gpus", "1",
                        "--steps", "1", "--warmup", "0"], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "samples/s" and d["higher_is_better"] is True
    assert d["metric"] == "training samples/sec (seq_len=128)" and d["scaling"] == "weak" and d["vs_baseline"] is None
    assert d["value"] > 0 and d["steps"] == 1 and d["n_gpus"] == 1 and d["gpu_launches"] == 0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"] == {"value": d["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    # the `config` object has the same keys (and, for N = 1, values) on both arms: the driver's same_config check
    sys.path.insert(0, root)
    import bench
    assert d["config"] == bench.config_dict(bench.CONFIGS["A"], 1)
    assert set(d["config"]) == {"workload", "global_batch", "seq_len", "parallelism", "dropout", "optimizer"}


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_bench_b200_arm_fails_loudly_without_a_gpu():
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr and r.stdout.strip() == ""


def test_fused_adamw_skip_flags_cover_exactly_the_encoder_matrices():
    """the vectors the (experimental) fused weight-gradient epilogue updates itself -- and the per-bucket AdamW launch
    must then skip -- are the six weight matrices of every encoder layer, nothing else"""
    class A:
        weight_decay, learning_rate = 0.01, 3e-5
    cfg = tiny_config()
    m = b2.BertForSequenceClassification(cfg)
    opt = b2.build_optimizer(m, A)
    flags = opt._fused_skip_flags()
    want = torch.zeros_like(flags)
    for n, (off, shape) in m._layout.entries.items():
        is_enc_matrix = n.startswith("bert.encoder.layer.") and n.endswith(".weight") and "LayerNorm" not in n
        numel = 1
        for d in shape:
            numel *= d
        if is_enc_matrix:
            assert numel % 8 == 0
            want[off // 8:(off + numel) // 8] = 1
    assert torch.equal(flags, want)
    assert int(flags.sum()) * 8 == cfg.num_hidden_layers * (4 * cfg.hidden_size ** 2 +
                                                          2 * cfg.hidden_size * cfg.intermediate_size)


def test_sass_carries_wgmma_and_tma():
    """what the compiler actually emitted for sm_90a (cuobjdump -sass of the in-tree library): the GEMM and attention
    kernels issue warpgroup MMAs (HGMMA), move tiles with TMA (UTMALDG; UTMASTG for the attention stores) and wait on
    mbarriers (SYNCS); the LayerNorm-fused GEMM synchronises its cluster (UCGABAR_*).  mma.sync (HMMA) must not appear
    in them."""
    import shutil
    import subprocess
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([exe, "-sass", L.LIB_PATH], capture_output=True, text=True, timeout=600).stdout
    per_fn, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = per_fn.setdefault(m.group(1), set())
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
        if m and cur is not None:
            cur.add(m.group(1))

    def ops(fragment):
        hit = [v for k, v in per_fn.items() if fragment in k]
        assert hit, "no kernel matching %s in the library" % fragment
        return hit

    for frag in ("gemm_bf16_kernel", "gemm_grouped_tn_kernel", "gemm_ln_kernel"):
        for o in ops(frag):
            assert {"HGMMA", "UTMALDG", "SYNCS"} <= o, (frag, sorted(o))
            assert "HMMA" not in o
    for o in ops("gemm_ln_kernel"):
        assert "UCGABAR_ARV" in o and "UCGABAR_WAIT" in o
    for frag in ("attention_fwd_kernel", "attention_fwd128_kernel", "attention_bwd_kernel"):
        for o in ops(frag):
            assert {"HGMMA", "UTMALDG", "UTMASTG", "SYNCS"} <= o, (frag, sorted(o))
            assert "HMMA" not in o
