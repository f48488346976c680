"""BertForMaskedLM, measured at config A's shapes (chinese-bert-wwm-ext, batch 32, seq 128, 15 % masking) and at 32
sequences of 8 to 512 tokens (uniform lengths) packed into 512-token bins.

  (a) the captured training step (FusedTrainStep / PackedTrainStep replayed on staged inputs, host clock around a
      synchronised window) of the masked-LM model against the sequence-classification model on the same ids; the arms
      alternate within each round.
  (b) stock HF BertForMaskedLM (transformers, sdpa attention, bf16 autocast, fused torch.optim.AdamW) at config A,
      when transformers imports.
  (c) each launch of the masked-LM head alone (CUDA events around a captured loop) at config A's labelled-row
      capacity: the compaction, the transform (EPI_BIAS_GELU GEMM + LayerNorm), the three vocabulary GEMMs (logits,
      d_transform, d_decoder) and the cross-entropy.  FLOP/s and the share of the larger of the compute floor (989
      TFLOP/s dense bf16) and the HBM floor (3.35 TB/s), both H100 SXM data-sheet figures, are computed from the
      shapes below.
The card's name, power limit and max SM clock are read in the same run.  One JSON line.
    python tools/mlm_bench.py [--rounds 3] [--steps 20]
"""
import argparse
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
from accum_bench import HBM_BYTES_PER_S, gpu_info
from attention_bench import timed_loop

B = 32
BF16_FLOPS = 989e12


def batches(cfg, S, n, packed):
    out = []
    for i in range(n):
        bt = b2.synthetic_mlm_batch(cfg, B, S, 300 + i, padded=packed)
        bt["seq_label"] = torch.randint(0, 6, (B,), generator=torch.Generator().manual_seed(i))
        out.append(bt)
    return out


def step_arm(kind, S, bts):
    """a callable replaying the captured step of `kind` on the staged batch (the model's own labels)"""
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    b2.set_seed(123)
    model = (b2.BertForMaskedLM if kind == "mlm" else b2.BertForSequenceClassification)(cfg).cuda().train()
    opt = b2.build_optimizer(model, b2.Args())
    bt = bts[0]
    lab = bt["label"] if kind == "mlm" else bt["seq_label"]
    if S == 128:
        st = b2.FusedTrainStep(model, opt, B, S)
        st.stage(dict(bt, label=lab))
    else:
        p = b2.pack_batch(bt["input_ids"], bt["token_type_ids"], bt["attention_mask"], S,
                          labels=lab if kind == "mlm" else None)
        st = b2.PackedTrainStep(model, opt, p["bins"], B, bin_len=S)
        st.stage(p, p["labels"] if kind == "mlm" else lab)
    for _ in range(4):
        st.run_device()
    return (lambda: st.run_device()), model


def time_steps(run, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        run()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def hf_arm(bts):
    from transformers import BertConfig, BertForMaskedLM
    cfg = BertConfig(vocab_size=21128, attn_implementation="sdpa")
    torch.manual_seed(123)
    model = BertForMaskedLM(cfg).cuda().train()
    opt = torch.optim.AdamW(model.parameters(), lr=3e-5, fused=True)
    d = {k: v.cuda() for k, v in bts[0].items() if k != "seq_label"}

    def run():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(input_ids=d["input_ids"], token_type_ids=d["token_type_ids"],
                        attention_mask=d["attention_mask"], labels=d["label"])
        out.loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    for _ in range(3):
        run()
    return run


def kernel_times(model, bt, rep=20):
    """each launch of the head at the batch's capacity, from the engine's own buffers after a training step"""
    eng = model._engine
    H, V, Vp = eng.H, eng.V, eng.Vp
    lab = bt["label"].cuda()
    M = lab.numel()
    cap, n = eng.mlm_capacity(lab, -100, M)
    gb = eng._mlm_buffers(M, cap)
    hb = eng._mlm_grad_buffers(gb)
    x = torch.randn(M, H, device="cuda").to(torch.bfloat16)
    dscale = torch.ones((), device="cuda")
    sh = eng._mlm_shared
    s = lambda: torch.cuda.current_stream().cuda_stream
    w = eng.w
    one = [None]

    def compact(_):
        L.call("b2_mlm_compact", lab.data_ptr(), M, -100, V, cap, gb["src"].data_ptr(), gb["slot"].data_ptr(),
               gb["labels"].data_ptr(), gb["count"].data_ptr(), s())
        L.call("b2_mlm_gather_rows", x.data_ptr(), gb["src"].data_ptr(), gb["count"].data_ptr(), cap, H,
               gb["x"].data_ptr(), s())

    def transform(_):
        eng.gemm(cap, H, H, gb["x"].data_ptr(), H, L.MAJOR_K, w("cls.predictions.transform.dense.weight"), H,
                 L.MAJOR_K, gb["h"].data_ptr(), H, L.EPI_BIAS_GELU, bias=w("cls.predictions.transform.dense.bias"),
                 aux_out=gb["u"].data_ptr(), ld_aux_out=H)
        L.call("b2_layernorm_fwd", gb["h"].data_ptr(), w("cls.predictions.transform.LayerNorm.weight"),
               w("cls.predictions.transform.LayerNorm.bias"), cap, H, 1e-12, gb["t"].data_ptr(), gb["mean"].data_ptr(),
               gb["rstd"].data_ptr(), s())

    def logits(_):
        L.call("b2_mlm_bias_fill", w("cls.predictions.bias"), cap, Vp, gb["logits"].data_ptr(), s())
        eng.gemm(cap, Vp, H, gb["t"].data_ptr(), H, L.MAJOR_K, w("bert.embeddings.word_embeddings.weight"), H,
                 L.MAJOR_K, gb["logits"].data_ptr(), Vp, L.EPI_ACCUM_F32)

    def ce(_):
        c = gb["count"].data_ptr()
        L.call("b2_mlm_ce", gb["logits"].data_ptr(), cap, V, Vp, gb["labels"].data_ptr(), c, c, dscale.data_ptr(),
               None, 0, gb["row_loss"].data_ptr(), gb["pred"].data_ptr(), hb["dlog"].data_ptr(),
               gb["loss"].data_ptr(), s())

    def d_transform(_):
        eng.gemm(cap, H, Vp, hb["dlog"].data_ptr(), Vp, L.MAJOR_K, w("bert.embeddings.word_embeddings.weight"), H,
                 L.MAJOR_MN, hb["dt"].data_ptr(), H, L.EPI_ACCUM_F32)

    def d_decoder(_):
        eng.gemm(Vp, H, cap, hb["dlog"].data_ptr(), Vp, L.MAJOR_MN, gb["t"].data_ptr(), H, L.MAJOR_MN,
                 sh["dec"].data_ptr(), H, L.EPI_ACCUM_F32)

    def tied_add(_):
        L.call("b2_mlm_tied_add", sh["dec"].data_ptr(), eng.g("bert.embeddings.word_embeddings.weight"), V * H, s())

    vocab_flop = 2 * cap * Vp * H
    work = {  # (flop, bytes) each launch needs at least
        "compaction+gather": (0, M * 8 + M * 4 + cap * 12 + 2 * cap * H * 2),
        "transform": (2 * cap * H * H, cap * H * 2 * 4 + H * H * 2 + cap * 8),
        "logits (bias fill + GEMM)": (vocab_flop, Vp * H * 2 + cap * H * 2 + 2 * cap * Vp * 4),
        "cross_entropy": (0, cap * Vp * 4 + cap * Vp * 2 + cap * 16),
        "d_transform GEMM": (vocab_flop, cap * Vp * 2 + Vp * H * 2 + 2 * cap * H * 4),
        "d_decoder GEMM": (vocab_flop, cap * Vp * 2 + cap * H * 2 + 2 * Vp * H * 4),
        "tied_add": (0, V * H * (4 + 2 + 2)),
    }
    fns = {"compaction+gather": compact, "transform": transform, "logits (bias fill + GEMM)": logits,
           "cross_entropy": ce, "d_transform GEMM": d_transform, "d_decoder GEMM": d_decoder, "tied_add": tied_add}
    out = {"capacity": cap, "labelled": n, "vocab_pad": Vp}
    for name, fn in fns.items():
        t_us = timed_loop(fn, one, rep)
        flop, byt = work[name]
        floor_us = 1e6 * max(flop / BF16_FLOPS, byt / HBM_BYTES_PER_S)
        out[name] = {"us": round(t_us, 2), "tflop_s": round(flop / t_us / 1e6, 1) if flop else None,
                     "floor_us": round(floor_us, 2),
                     "bound": "compute" if flop / BF16_FLOPS > byt / HBM_BYTES_PER_S else "hbm",
                     "share_of_floor": round(floor_us / t_us, 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mlm_bench needs a GPU")
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    res = {"gpu": gpu_info()}
    for S, name in ((128, "config_a_32x128"), (512, "packed_32x512")):
        bts = batches(cfg, S, 1, S == 512)
        arms, models = {}, {}
        for kind in ("sequence", "mlm"):
            arms[kind], models[kind] = step_arm(kind, S, bts)
        if S == 128:
            try:
                arms["hf_bert_for_masked_lm"] = hf_arm(bts)
            except ImportError as e:
                res["hf"] = "not measured: %s" % e
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, run in arms.items():
                times[k].append(time_steps(run, args.steps))
        med = {k: statistics.median(v) for k, v in times.items()}
        r = {k: {"median_ms": round(1e3 * t, 3), "samples_per_s": round(B / t, 1),
                 "rounds_ms": [round(1e3 * x, 3) for x in times[k]]} for k, t in med.items()}
        r["mlm_vs_sequence_time"] = round(med["mlm"] / med["sequence"], 3)
        if "hf_bert_for_masked_lm" in med:
            r["mlm_speedup_vs_hf"] = round(med["hf_bert_for_masked_lm"] / med["mlm"], 2)
        r["labelled_tokens"] = int((bts[0]["label"] != -100).sum())
        if S == 128:
            r["head_kernels"] = kernel_times(models["mlm"], bts[0])
        res[name] = r
        del arms, models
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
