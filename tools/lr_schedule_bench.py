"""Learning-rate schedules on one GPU, BASELINE config A (seq 128, batch 32, dropout on).

  * the captured, device-resident training step without a scheduler and with a "linear" schedule (a torch LambdaLR
    stepped after every step, its lr staged with the batch and read by the graph at every replay), alternated in
    rounds within this one run: ms per step (median of rounds) and samples/s;
  * b2_bucket_reduce_adamw and b2_adamw_background over the whole flat parameter space with the lr passed by value
    and read from the device (b2_adamw_hparams_t.lr_dev): kernel time of each.
The GPU's name and power limit are read in the same run and printed with the numbers (one JSON line; --out also writes
it to a file).
    python tools/lr_schedule_bench.py [--steps 50] [--rounds 3] [--out /tmp/lr_schedule_bench.json]
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
from accum_bench import gpu_info
from clip_bench import time_kernel


def time_steps(step, batch, sched, n):
    """host staging included: the scheduled form's cost is the lr staged with the batch and the scheduler's step()"""
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        step(batch)
        if sched is not None:
            sched.step()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="timed steps per form and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    B, S = 32, 128
    b2.set_seed(123)
    res = {"config": "A", "batch": B, "seq": S, "gpu": gpu_info()}
    batch = b2.synthetic_batch(cfg, B, S, 1000, padded=True)
    forms = {}
    for name in ("constant", "linear"):
        model = b2.BertForSequenceClassification(cfg).cuda().train()
        opt = b2.build_optimizer(model, b2.Args())
        total = 10 + a.rounds * a.steps + 1
        sched = b2.get_scheduler("linear", opt, num_warmup_steps=total // 10, num_training_steps=total) \
            if name == "linear" else None
        st = b2.FusedTrainStep(model, opt, B, S)
        for _ in range(5):             # warm-up and capture
            st(batch)
            if sched is not None:
                sched.step()
        forms[name] = (st, sched, model, opt)
    torch.cuda.synchronize()
    ms = {k: [] for k in forms}
    for _ in range(a.rounds):
        for k, (st, sched, _m, _o) in forms.items():
            ms[k].append(time_steps(st, batch, sched, a.steps))
    res["steps"] = {k: {"ms_per_step": [round(x, 4) for x in v], "median_ms": round(sorted(v)[len(v) // 2], 4),
                        "samples_per_s": round(B / (sorted(v)[len(v) // 2] / 1e3), 1)} for k, v in ms.items()}
    res["schedule_cost_ms"] = round(res["steps"]["linear"]["median_ms"] - res["steps"]["constant"]["median_ms"], 4)
    _st, _sched, model, opt = forms.pop("linear")
    forms.clear()
    eng, n = model._engine, model._layout.total
    state = opt._state()
    s = torch.cuda.current_stream().cuda_stream
    grads, shadow = L.ptr_array([eng.grads.data_ptr()]), L.ptr_array([eng.shadow.data_ptr()])

    def kernels(lr_dev):
        hp = opt.hparams()
        hp.lr_dev = state["lr"].data_ptr() if lr_dev else None

        def reduce():
            L.call("b2_bucket_reduce_adamw", grads, shadow, 1, 0, L.ptr(model._flat), L.ptr(state["exp_avg"]),
                   L.ptr(state["exp_avg_sq"]), L.ptr(state["decay"]), 0, n, hp, L.ptr(state["step"]), s)

        def background():
            L.call("b2_adamw_background", eng.grads.data_ptr(), eng.shadow.data_ptr(), L.ptr(model._flat),
                   L.ptr(state["exp_avg"]), L.ptr(state["exp_avg_sq"]), L.ptr(state["decay"]), 0, n, hp,
                   L.ptr(state["step_size"]), s)
        return reduce, background

    res["kernel_us"] = {}
    for lr_dev in (False, True):
        reduce, background = kernels(lr_dev)
        key = "lr_dev" if lr_dev else "lr_by_value"
        res["kernel_us"][key] = {"bucket_reduce_adamw": round(time_kernel(reduce, a.kernel_iters) * 1e6, 1),
                                 "adamw_background": round(time_kernel(background, a.kernel_iters) * 1e6, 1)}
    res["parameters"] = n
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
