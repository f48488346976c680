"""BertForTokenClassification, measured at config A's shapes (chinese-bert-wwm-ext, batch 32, seq 128, C 9).

  (a) the captured training step (FusedTrainStep replayed on staged inputs, host clock around a synchronised window)
      of the sequence model against the token model, padded to 128 and packed (PackedTrainStep, 128-token bins), on
      rows whose lengths follow synthetic.REFERENCE_LENGTH_HISTOGRAM; the arms alternate within each round.
  (b) each token-head kernel and the loss kernel alone (CUDA events around a captured loop), at M = 4 096 and 16 384
      token rows, against the HBM floor of the bytes each launch must move once (3.35 TB/s, the H100 SXM data sheet):
        forward        x (M H bf16) + W + logits (M C fp32)
        data grad      dlogits (M C fp32) + W + d_hidden (M H fp32)
        parameter grad x (M H bf16) + dlogits, per label group of 8, + partials written and read back + dW / db
        loss           logits (M C fp32) + labels (M int64) + dlogits (M C fp32)
The card's name, power limit and max SM clock are read in the same run.  One JSON line.
    python tools/token_cls_bench.py [--rounds 3] [--steps 30]
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
from pytorch_distributed_nlp_b200.losses import Loss
from pytorch_distributed_nlp_b200.synthetic import reference_length_batch
from accum_bench import HBM_BYTES_PER_S, gpu_info
from attention_bench import timed_loop

B, S, C = 32, 128, 9


def token_labels(batch, seed):
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, C, batch["input_ids"].shape, generator=g, dtype=torch.int64)
    lab[batch["attention_mask"] == 0] = -100
    lab[:, 0] = -100
    return lab


def step_arm(kind, packed, batches):
    """a callable running one replay of the captured step for the next batch"""
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=C)
    b2.set_seed(123)
    cls = b2.BertForTokenClassification if kind == "token" else b2.BertForSequenceClassification
    model = cls(cfg).cuda().train()
    args = b2.Args()
    opt = b2.build_optimizer(model, args)
    if not packed:
        st = b2.FusedTrainStep(model, opt, B, S)
        for bt in batches:
            st.stage(bt if kind == "sequence" else dict(bt, label=bt["token_label"]))
            st.run_device()
        return lambda i: st.run_device()
    # one packed batch (its bin count fixes the graph): the captured step replayed on it
    bt = batches[0]
    lab = bt["token_label"] if kind == "token" else None
    p = b2.pack_batch(bt["input_ids"], bt["token_type_ids"], bt["attention_mask"], 128, labels=lab)
    st = b2.PackedTrainStep(model, opt, p["bins"], B)
    st.stage(p, p["labels"] if kind == "token" else bt["label"])
    for _ in range(3):
        st.run_device()
    return lambda i: st.run_device()


def time_steps(run, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        run(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def kernel_times(M, H=768, rep=50):
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(M)
    sets = []
    for s in range(4):     # rotate operand sets so each launch reads from HBM rather than a warm L2
        x = torch.randn(M, H, generator=g).to(torch.bfloat16).to(dev)
        dl = (torch.randn(M, C, generator=g) / M).to(dev)
        lab = torch.randint(0, C, (M,), generator=g).to(dev)
        sets.append(dict(x=x, dl=dl, lab=lab, logits=torch.empty(M, C, device=dev), dh=torch.empty(M, H, device=dev)))
    W = (0.05 * torch.randn(C, H, generator=g)).to(torch.bfloat16).to(dev)
    bvec = torch.zeros(C, dtype=torch.bfloat16, device=dev)
    dW, db = torch.empty(C, H, dtype=torch.bfloat16, device=dev), torch.empty(C, dtype=torch.bfloat16, device=dev)
    n = int(L.load().b2_token_head_scratch_floats(M, H, C))
    scratch = torch.empty(n, device=dev)
    rng = torch.tensor([1, 0], dtype=torch.int64, device=dev)
    loss = torch.empty((), device=dev)
    ce = Loss(L.LOSS_CE, C)
    p = 0.1

    def stream():
        return torch.cuda.current_stream().cuda_stream

    def fwd(s):
        L.call("b2_token_head_fwd", s["x"].data_ptr(), M, H, W.data_ptr(), bvec.data_ptr(), C, p, rng.data_ptr(),
               37, s["logits"].data_ptr(), stream())

    def bwd(s):
        L.call("b2_token_head_bwd_split", s["dl"].data_ptr(), s["x"].data_ptr(), M, H, W.data_ptr(), C, p,
               rng.data_ptr(), 37, dW.data_ptr(), db.data_ptr(), s["dh"].data_ptr(), scratch.data_ptr(), n, stream(),
               None)

    def ce_launch(s):
        ce.launch(s["logits"].data_ptr(), s["lab"], M, loss.data_ptr(), s["dl"].data_ptr(), stream())

    for s in sets:
        fwd(s)
    torch.cuda.synchronize()
    groups = -(-C // 8)
    nblk = n // ((C + 1) * H)
    bytes_ = {"token_head_fwd": M * H * 2 + C * H * 2 + M * C * 4,
              "token_head_bwd_split": (M * C * 4 + C * H * 2 + M * H * 4) +
              (groups * (M * H * 2 + M * C * 4) + 2 * nblk * (C + 1) * H * 4 + (C * H + C) * 2),
              "ce_fwd_bwd": M * C * 4 + M * 8 + M * C * 4}
    out = {}
    for name, fn in (("token_head_fwd", fwd), ("token_head_bwd_split", bwd), ("ce_fwd_bwd", ce_launch)):
        t_us = timed_loop(fn, sets, rep)
        floor_us = 1e6 * bytes_[name] / HBM_BYTES_PER_S
        out[name] = {"us": round(t_us, 2), "bytes": bytes_[name], "hbm_floor_us": round(floor_us, 2),
                     "share_of_hbm_floor": round(floor_us / t_us, 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("token_cls_bench needs a GPU")
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=C)
    batches = []
    for i in range(4):
        bt = reference_length_batch(cfg, B, 100 + i, S)
        bt["token_label"] = token_labels(bt, 200 + i)
        batches.append(bt)
    arms = {}
    for kind in ("sequence", "token"):
        for packed in (False, True):
            arms["%s_%s" % (kind, "packed" if packed else "padded")] = step_arm(kind, packed, batches)
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, run in arms.items():
            times[k].append(time_steps(run, args.steps))
    steps = {k: {"median_ms": round(1e3 * statistics.median(v), 3), "samples_per_s": round(B / statistics.median(v), 1),
                 "rounds_ms": [round(1e3 * t, 3) for t in v]} for k, v in times.items()}
    del arms
    torch.cuda.empty_cache()
    res = {"gpu": gpu_info(), "config": "A (chinese-bert-wwm-ext, batch 32, seq 128, C 9)", "captured_step": steps,
           "token_vs_sequence_padded": round(steps["token_padded"]["median_ms"] / steps["sequence_padded"]["median_ms"], 3),
           "token_vs_sequence_packed": round(steps["token_packed"]["median_ms"] / steps["sequence_packed"]["median_ms"], 3),
           "kernels": {str(M): kernel_times(M) for M in (4096, 16384)}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
