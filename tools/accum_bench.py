"""Gradient accumulation on one GPU, BASELINE config A (seq 128, batch 32, dropout on).

  * captured, device-resident training windows for k = 1, 2, 4, 8 micro-batches (k - 1 accumulating replays + one
    final replay with the optimizer step): ms per window, ms per micro-batch, samples/s;
  * each b2_grad_accumulate mode alone over the whole flat parameter space: kernel time, achieved GB/s from the bytes
    the mode must move (STORE 6, ADD 10, FOLD 8, FLUSH 6 bytes per parameter) and the fraction of the H100 SXM's
    3.35 TB/s data-sheet HBM3 bandwidth.
The GPU's name and power limit are read in the same run and printed with the numbers (one JSON line; --out also writes
it to a file).
    python tools/accum_bench.py [--micro-batches 64] [--out /tmp/accum_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

import pytorch_distributed_nlp_b200 as b2
from pytorch_distributed_nlp_b200 import _lib as L

HBM_BYTES_PER_S = 3.35e12
MODES = {"store": (L.ACCUM_STORE, 6), "add": (L.ACCUM_ADD, 10), "fold": (L.ACCUM_FOLD, 8), "flush": (L.ACCUM_FLUSH, 6)}


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    parts = [p.strip() for p in line.split(",")] if line else []
    return {"name": torch.cuda.get_device_name(0), "power_limit": parts[1] if len(parts) > 1 else None,
            "max_sm_clock": parts[2] if len(parts) > 2 else None}


def time_windows(step, k, windows):
    def window():
        for i in range(k):
            step.run_device(final=(i == k - 1))
    for _ in range(3):                     # every role warmed up and captured
        window()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(windows):
        window()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / windows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--micro-batches", type=int, default=64, help="timed per k (rounded up to whole windows)")
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    B, S = 32, 128
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg).cuda().train()
    opt = b2.build_optimizer(model, b2.Args())
    res = {"config": "A", "batch": B, "seq": S, "gpu": gpu_info(), "steps": {}, "kernel": {}}
    batch = b2.synthetic_batch(cfg, B, S, 1000, padded=True)
    for k in (1, 2, 4, 8):
        step = b2.FusedTrainStep(model, opt, B, S, accum_steps=k)
        step.stage(batch)
        windows = -(-a.micro_batches // k)
        ms = time_windows(step, k, windows)
        res["steps"][k] = {"windows": windows, "ms_per_window": round(ms, 4), "ms_per_micro_batch": round(ms / k, 4),
                           "samples_per_s": round(B * k / (ms / 1e3), 1)}
        del step
    eng = model._engine
    n = model._layout.total
    s = torch.cuda.current_stream().cuda_stream
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, (op, bpp) in MODES.items():
        for _ in range(3):
            eng.accumulate_range(0, n, op, s)
        torch.cuda.synchronize()
        t0.record()
        for _ in range(a.kernel_iters):
            eng.accumulate_range(0, n, op, s)
        t1.record()
        torch.cuda.synchronize()
        sec = t0.elapsed_time(t1) / 1e3 / a.kernel_iters
        res["kernel"][name] = {"us": round(sec * 1e6, 1), "bytes": bpp * n, "GB_per_s": round(bpp * n / sec / 1e9, 1),
                               "fraction_of_3.35TB_s": round(bpp * n / sec / HBM_BYTES_PER_S, 3)}
    res["parameters"] = n
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
