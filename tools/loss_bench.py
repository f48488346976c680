"""The training losses on one GPU, BASELINE config A (seq 128, batch 32, 6 labels, dropout on).

  * captured, device-resident training steps with CrossEntropyLoss() (the default path), weighted and label-smoothed
    CrossEntropyLoss, BCEWithLogitsLoss(pos_weight) and MSELoss, alternated in rounds within this one run: ms per step
    and samples/s for each;
  * the loss kernel alone (b2_ce_fwd_bwd / b2_loss_fwd_bwd, one block over batch x labels) for each loss, in us.
The GPU's name and power limit are read in the same run and printed with the numbers (one JSON line; --out also writes
it to a file).
    python tools/loss_bench.py [--steps 50] [--rounds 3] [--out /tmp/loss_bench.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch
import torch.nn as nn

import pytorch_distributed_nlp_b200 as b2
from accum_bench import gpu_info
from clip_bench import time_kernel, time_steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="timed steps per loss and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    B, S, C = 32, 128, 6
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg).cuda().train()
    opt = b2.build_optimizer(model, b2.Args())
    res = {"config": "A", "batch": B, "seq": S, "num_labels": C, "gpu": gpu_info()}
    w = torch.tensor([0.2, 1.0, 3.0, 0.5, 2.0, 1.0], device=dev)
    crits = {"ce": None, "ce_weight_smoothing": nn.CrossEntropyLoss(weight=w, label_smoothing=0.1),
             "bce_pos_weight": nn.BCEWithLogitsLoss(pos_weight=w), "mse": nn.MSELoss()}
    batch = b2.synthetic_batch(cfg, B, S, 1000, padded=True)
    g = torch.Generator().manual_seed(7)
    float_labels = {"bce_pos_weight": (torch.rand(B, C, generator=g) < 0.4).float(), "mse": torch.randn(B, C, generator=g)}
    steps = {}
    for k, crit in crits.items():
        st = b2.FusedTrainStep(model, opt, B, S, criterion=crit)
        bt = dict(batch, label=float_labels.get(k, batch["label"]))
        st.stage(bt)
        for _ in range(5):             # warm-up and capture
            st.run_device()
        steps[k] = st
    torch.cuda.synchronize()
    ms = {k: [] for k in steps}
    for _ in range(a.rounds):
        for k, st in steps.items():
            ms[k].append(time_steps(st, a.steps))
    res["steps"] = {k: {"ms_per_step": [round(x, 4) for x in v], "median_ms": round(sorted(v)[len(v) // 2], 4),
                        "samples_per_s": round(B / (sorted(v)[len(v) // 2] / 1e3), 1)} for k, v in ms.items()}
    logits = torch.randn(B, C, device=dev)
    loss, dl = torch.empty((), device=dev), torch.empty(B, C, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    res["kernel_us"] = {}
    for k, st in steps.items():
        fn, lab = st.loss_fn, st.d_lab

        def launch():
            fn.launch(logits.data_ptr(), lab.view(-1), B, loss.data_ptr(), dl.data_ptr(), s)
        res["kernel_us"][k] = round(time_kernel(launch, a.kernel_iters) * 1e6, 2)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
