"""Gradient-norm clipping on one GPU, BASELINE config A (seq 128, batch 32, dropout on).

  * captured, device-resident training steps without and with max_grad_norm, alternated in rounds within this one run:
    ms per step and samples/s for each, and the difference -- the part of the update that no longer hides under the
    backward (with clipping the update waits for the norm of the whole gradient);
  * the reduce phase (b2_grad_reduce_sumsq, world 1: 2 bytes per parameter in) and the norm finalize alone over the
    whole flat parameter space: kernel time, achieved GB/s and the fraction of the H100 SXM's 3.35 TB/s data-sheet
    HBM3 bandwidth.
The GPU's name and power limit are read in the same run and printed with the numbers (one JSON line; --out also writes
it to a file).
    python tools/clip_bench.py [--steps 50] [--rounds 3] [--out /tmp/clip_bench.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch

import pytorch_distributed_nlp_b200 as b2
from pytorch_distributed_nlp_b200 import _lib as L
from accum_bench import HBM_BYTES_PER_S, gpu_info


def time_steps(step, n):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        step.run_device()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / n


def time_kernel(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="timed steps per form and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--max-grad-norm", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    B, S = 32, 128
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg).cuda().train()
    opt = b2.build_optimizer(model, b2.Args())
    res = {"config": "A", "batch": B, "seq": S, "gpu": gpu_info(), "max_grad_norm": a.max_grad_norm}
    batch = b2.synthetic_batch(cfg, B, S, 1000, padded=True)
    steps = {"plain": b2.FusedTrainStep(model, opt, B, S),
             "clipped": b2.FusedTrainStep(model, opt, B, S, max_grad_norm=a.max_grad_norm)}
    for st in steps.values():
        st.stage(batch)
        for _ in range(5):             # warm-up and capture
            st.run_device()
    torch.cuda.synchronize()
    ms = {k: [] for k in steps}
    for _ in range(a.rounds):
        for k, st in steps.items():
            ms[k].append(time_steps(st, a.steps))
    res["steps"] = {k: {"ms_per_step": [round(x, 4) for x in v], "median_ms": round(sorted(v)[len(v) // 2], 4),
                        "samples_per_s": round(B / (sorted(v)[len(v) // 2] / 1e3), 1)} for k, v in ms.items()}
    res["clip_cost_ms"] = round(res["steps"]["clipped"]["median_ms"] - res["steps"]["plain"]["median_ms"], 4)
    res["last_grad_norm"] = float(opt._clip_buf["norm"])
    del steps
    eng, n = model._engine, model._layout.total
    s = torch.cuda.current_stream().cuda_stream
    ns = L.sumsq_slots(n)
    partials = torch.zeros(ns, dtype=torch.float64, device=eng.dev)
    out = [torch.zeros((), device=eng.dev) for _ in range(3)]
    grads = L.ptr_array([eng.grads.data_ptr()])

    def reduce():
        L.call("b2_grad_reduce_sumsq", grads, 1, None, 0, n, partials.data_ptr(), s)

    def finalize():
        L.call("b2_grad_norm_finalize", partials.data_ptr(), ns, None, None, 1, 0, 0, None, 1.0, None, None,
               out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), s)

    sec = time_kernel(reduce, a.kernel_iters)
    res["kernel"] = {"reduce_sumsq_world1": {"us": round(sec * 1e6, 1), "bytes": 2 * n,
                                             "GB_per_s": round(2 * n / sec / 1e9, 1),
                                             "fraction_of_3.35TB_s": round(2 * n / sec / HBM_BYTES_PER_S, 3)},
                     "finalize": {"us": round(time_kernel(finalize, a.kernel_iters) * 1e6, 1), "slots": ns}}
    res["parameters"] = n
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
