"""The fixed-order backward (torch.use_deterministic_algorithms), measured: three rounds, each alternating the modes.

Steps (samples/s of the captured step replayed on staged inputs, as tools/pack_long_bench.py's device_rate):
  A  config A: bert-base, batch 32 padded to 128
  B  config B: bert-base, batch 16 padded to 512
  P  pack_long_bench's case (a): config B's batch with lengths ~ U{16..512}, packed into 512-token bins
Sites (device time per launch, CUDA events around a captured loop), each fixed-order form against the form it
replaces, at config A's shapes (dQ at config B's):
  colsum   b2_colsum of dU [4096, 3072] vs the same GELU' dgrad's epilogue column sums (dgrad without - with them)
  ln       b2_layernorm_bwd with partials + b2_colsum_finish vs b2_layernorm_bwd_accum
  split    the N = hidden EPI_ACCUM_F32 dgrad (K = 3072) unsplit vs the cost model's split
  embed    b2_embed_bwd_ordered vs b2_embed_bwd (word rows: in-order owner scan vs fp32 owner-row reductions)
  dq       b2_attention_bwd_ordered vs b2_attention_bwd at seq 512 (both with their dQ conversion)
The GPU's name, power limit and max SM clock are read in the same run.  One JSON line (--out also writes it).
    python tools/determinism_bench.py [--rounds 3] [--steps 20] [--out /tmp/determinism_bench.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch

import pytorch_distributed_nlp_b200 as b2
from pytorch_distributed_nlp_b200 import _lib as L
from pytorch_distributed_nlp_b200.packing import pack_batch
from accum_bench import gpu_info
from attention_bench import timed_loop
from pack_long_bench import uniform_batch

bf, f32 = torch.bfloat16, torch.float32


def step_rate(cfg, batch, det, steps, pack=False):
    """samples/s of one captured step built and replayed with the flag set to `det`"""
    torch.use_deterministic_algorithms(det)
    try:
        b2.set_seed(123)
        model = b2.BertForSequenceClassification(cfg).cuda().train()
        opt = b2.build_optimizer(model, b2.Args())
        B, S = batch["input_ids"].shape
        if pack:
            p = pack_batch(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"], S)
            st = b2.PackedTrainStep(model, opt, p["bins"], B, bin_len=S, criterion=torch.nn.CrossEntropyLoss())
            st.stage(p, batch["label"])
        else:
            st = b2.FusedTrainStep(model, opt, B, S, criterion=torch.nn.CrossEntropyLoss())
            st.stage(batch)
        for _ in range(4):
            st.run_device()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            st.run_device()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        del model, opt, st
        torch.cuda.empty_cache()
        return steps * B / dt
    finally:
        torch.use_deterministic_algorithms(False)


def site_times(rep=20):
    """{site: (fixed-order us, replaced form us)}"""
    dev = "cuda"
    s = lambda: torch.cuda.current_stream().cuda_stream
    H, I, M, V = 768, 3072, 32 * 128, 21128
    g = torch.Generator(device=dev).manual_seed(5)
    rnd = lambda *sh: (torch.randn(*sh, device=dev, generator=g) * 0.1).to(bf)
    out = {}
    # colsum of dU vs the GELU' epilogue's column sums
    dz, w2, u, dU = rnd(M, H), rnd(H, I), rnd(M, I), torch.empty(M, I, dtype=bf, device=dev)
    acc = torch.zeros(I, dtype=f32, device=dev)
    bias = torch.empty(I, dtype=bf, device=dev)
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device=dev)

    def gelu_dgrad(colsum):
        a = L.GemmArgs()
        a.M, a.N, a.K = M, I, H
        a.A, a.lda, a.a_major = dz.data_ptr(), H, L.MAJOR_K
        a.B, a.ldb, a.b_major = w2.data_ptr(), I, L.MAJOR_MN
        a.D, a.ldd, a.epilogue = dU.data_ptr(), I, L.EPI_GELU_BWD
        a.aux_in, a.ld_aux_in = u.data_ptr(), I
        a.colsum_out = colsum
        L.call("b2_gemm_bf16", a, s())
    t_with = timed_loop(lambda _: gelu_dgrad(acc.data_ptr()), [0], rep)
    t_without = timed_loop(lambda _: gelu_dgrad(None), [0], rep)
    t_col = timed_loop(lambda _: L.call("b2_colsum", dU.data_ptr(), M, I, I, bias.data_ptr(), scratch.data_ptr(),
                                        scratch.numel(), s()), [0], rep)
    out["colsum"] = (t_col, t_with - t_without)
    # LayerNorm backward: partials + finish vs accum
    dy, dx = torch.randn(M, H, device=dev), torch.empty(M, H, dtype=f32, device=dev)
    z, gam = rnd(M, H), (1 + rnd(H).float()).to(bf)
    mean, rstd = z.float().mean(1), torch.rsqrt(z.float().var(1) + 1e-12)
    dxd, lnacc = torch.empty(M, H, dtype=bf, device=dev), torch.zeros(3 * H, dtype=f32, device=dev)
    grads = torch.empty(3, H, dtype=bf, device=dev)
    parts = torch.empty(132 * 3 * H * 4, dtype=torch.uint8, device=dev)
    rs = torch.tensor([1, 0], dtype=torch.int64, device=dev)

    def ln_partials(_):
        n = ctypes.c_int32()
        L.call("b2_layernorm_bwd", dy.data_ptr(), None, z.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gam.data_ptr(),
               M, H, 0.1, rs.data_ptr(), 3, 1, dx.data_ptr(), dxd.data_ptr(), grads[0].data_ptr(),
               grads[1].data_ptr(), grads[2].data_ptr(), parts.data_ptr(), parts.numel(), ctypes.addressof(n), s())
        L.call("b2_colsum_finish", parts.data_ptr(), n.value, 3, H, grads[0].data_ptr(), grads[1].data_ptr(),
               grads[2].data_ptr(), s())
    t_parts = timed_loop(ln_partials, [0], rep)
    t_accum = timed_loop(lambda _: L.call("b2_layernorm_bwd_accum", dy.data_ptr(), z.data_ptr(), mean.data_ptr(),
                                          rstd.data_ptr(), gam.data_ptr(), M, H, 0.1, rs.data_ptr(), 3, dx.data_ptr(),
                                          dxd.data_ptr(), lnacc.data_ptr(), s()), [0], rep)
    out["ln"] = (t_parts, t_accum)
    # the N = hidden accumulating dgrad, one split vs the cost model's
    w1 = rnd(I, H)

    def accum_dgrad(splits):
        a = L.GemmArgs()
        a.M, a.N, a.K = M, H, I
        a.A, a.lda, a.a_major = dU.data_ptr(), I, L.MAJOR_K
        a.B, a.ldb, a.b_major = w1.data_ptr(), H, L.MAJOR_MN
        a.D, a.ldd, a.epilogue = dx.data_ptr(), H, L.EPI_ACCUM_F32
        a.force_splits = splits
        L.call("b2_gemm_bf16", a, s())
    out["split"] = (timed_loop(lambda _: accum_dgrad(1), [0], rep), timed_loop(lambda _: accum_dgrad(0), [0], rep))
    # embedding backward
    ids = torch.randint(1, V, (M,), dtype=torch.int32, device=dev)
    tt = torch.zeros(M, dtype=torch.int32, device=dev)
    owner = torch.empty(V, dtype=torch.int32, device=dev)
    L.call("b2_embed_owner_init", owner.data_ptr(), V, s())
    eg = [torch.zeros(n, H, dtype=bf, device=dev) for n in (V, 512, 2, 1, 1)]
    edx, escr = torch.empty(M, H, dtype=bf, device=dev), torch.empty(32 << 20, dtype=torch.uint8, device=dev)

    def embed(name):
        L.call(name, dy.data_ptr(), 1, z.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gam.data_ptr(), ids.data_ptr(),
               tt.data_ptr(), 32, 128, H, V, 2, 0, 0.1, rs.data_ptr(), 0, *[t.data_ptr() for t in eg], edx.data_ptr(),
               escr.data_ptr(), escr.numel(), owner.data_ptr(), s())
    out["embed"] = (timed_loop(lambda _: embed("b2_embed_bwd_ordered"), [0], rep),
                    timed_loop(lambda _: embed("b2_embed_bwd"), [0], rep))
    # dQ at config B's attention shapes
    B, S, nh = 16, 512, 12
    qkv, dctx = rnd(B * S, 3 * H), rnd(B * S, H)
    ctx, lse = torch.empty(B * S, H, dtype=bf, device=dev), torch.empty(B * nh * S, dtype=f32, device=dev)
    L.call("b2_attention_fwd", qkv.data_ptr(), None, B, S, nh, 64, 0.1, rs.data_ptr(), 1, ctx.data_ptr(),
           lse.data_ptr(), None, s())
    dqkv, dq_acc = torch.empty(B * S, 3 * H, dtype=bf, device=dev), torch.empty(B * S, H, dtype=f32, device=dev)
    dq_parts = torch.empty(S // 128, B * S, H, dtype=f32, device=dev)
    common = (qkv.data_ptr(), None, ctx.data_ptr(), dctx.data_ptr(), lse.data_ptr(), B, S, nh, 64, 0.1, rs.data_ptr(),
              1, dqkv.data_ptr())
    out["dq"] = (timed_loop(lambda _: L.call("b2_attention_bwd_ordered", *common, dq_parts.data_ptr(), s()), [0], rep),
                 timed_loop(lambda _: L.call("b2_attention_bwd", *common, dq_acc.data_ptr(), None, None, s()), [0],
                            rep))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("determinism_bench needs a GPU")
    cfg_a = b2.chinese_bert_wwm_ext_config(num_labels=2)
    cfg_b = b2.chinese_bert_wwm_ext_config(num_labels=2, max_position_embeddings=512)
    batch_a = b2.synthetic_batch(cfg_a, 32, 128, 1000, padded=True)
    batch_b = uniform_batch(cfg_b, 16, 512, 11, lo=512)
    batch_p = uniform_batch(cfg_b, 16, 512, 7)
    arms = {"A": (cfg_a, batch_a, False), "B": (cfg_b, batch_b, False), "P": (cfg_b, batch_p, True)}
    rates = {k: {"off": [], "on": []} for k in arms}
    sites = {}
    for r in range(a.rounds):
        order = ("off", "on") if r % 2 == 0 else ("on", "off")
        for name, (cfg, batch, pack) in arms.items():
            for mode in order:
                rates[name][mode].append(step_rate(cfg, batch, mode == "on", a.steps, pack))
        for k, (on, off) in site_times().items():
            sites.setdefault(k, {"fixed_order_us": [], "replaced_us": []})
            sites[k]["fixed_order_us"].append(on)
            sites[k]["replaced_us"].append(off)
    res = {"gpu": gpu_info(), "rounds": a.rounds, "steps": a.steps,
           "samples_per_s": {k: {m: [round(x, 1) for x in v[m]] for m in v} for k, v in rates.items()},
           "median_on_over_off": {k: round(statistics.median(v["on"]) / statistics.median(v["off"]), 4)
                                  for k, v in rates.items()},
           "sites_us": {k: {m: [round(x, 2) for x in v[m]] for m in v} for k, v in sites.items()}}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
