"""torch's AdamW against HF AdamW on one GPU, BASELINE config A (seq 128, batch 32, dropout on).

  * captured, device-resident training steps with build_optimizer's HF AdamW, TorchAdamW ("adamw_torch") and
    TorchAdamW(amsgrad=True), on the reference's two groups, alternated in rounds within this one run: ms per step and
    samples/s;
  * each update kernel alone over the whole flat parameter space, in both forms (the 256-thread reduce form at world 1
    and the 128-thread background form): kernel time, bytes per parameter (28 for both AdamWs, 36 with amsgrad),
    achieved TB/s and the fraction of the H100 SXM's 3.35 TB/s data-sheet HBM3 bandwidth.
The GPU's name, power limit and max SM clock are read in the same run and printed with the numbers (one JSON line;
--out also writes it to a file).
    python tools/adam_bench.py [--steps 30] [--rounds 3] [--out /tmp/adam_bench.json]
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
from accum_bench import HBM_BYTES_PER_S, gpu_info
from clip_bench import time_kernel, time_steps


def _args(**kw):
    args = b2.Args()
    for k, v in kw.items():
        setattr(args, k, v)
    return args


def _amsgrad(model, args):
    """TorchAdamW(amsgrad=True) on build_optimizer's two groups (no decay for bias and LayerNorm.weight)"""
    nd = lambda n: "bias" in n or "LayerNorm.weight" in n
    named = list(model.named_parameters())
    groups = [{"params": [p for n, p in named if not nd(n)], "weight_decay": args.weight_decay},
              {"params": [p for n, p in named if nd(n)], "weight_decay": 0.0}]
    return b2.TorchAdamW(groups, lr=args.learning_rate, amsgrad=True)


FORMS = {   # name: (optimizer of a model, bytes per parameter of the update at world 1)
    "hf_adamw": (lambda m: b2.build_optimizer(m, _args()), 28),
    "torch_adamw": (lambda m: b2.build_optimizer(m, _args(optim="adamw_torch")), 28),
    "torch_adamw_amsgrad": (lambda m: _amsgrad(m, _args()), 36),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per optimizer and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    B, S = 32, 128
    res = {"config": "A", "batch": B, "seq": S, "gpu": gpu_info()}
    batch = b2.synthetic_batch(cfg, B, S, 1000, padded=True)
    models, opts, steps = {}, {}, {}
    for name, (make, _bpp) in FORMS.items():
        b2.set_seed(123)
        models[name] = b2.BertForSequenceClassification(cfg).cuda().train()
        opts[name] = make(models[name])
        steps[name] = b2.FusedTrainStep(models[name], opts[name], B, S)
        steps[name].stage(batch)
        for _ in range(5):             # warm-up and capture
            steps[name].run_device()
    torch.cuda.synchronize()
    assert opts["torch_adamw_amsgrad"].max_exp_avg_sqs() != {}
    ms = {k: [] for k in steps}
    for _ in range(a.rounds):
        for k, st in steps.items():
            ms[k].append(time_steps(st, a.steps))
    res["steps"] = {k: {"ms_per_step": [round(x, 4) for x in v], "median_ms": round(sorted(v)[len(v) // 2], 4),
                        "samples_per_s": round(B / (sorted(v)[len(v) // 2] / 1e3), 1)} for k, v in ms.items()}
    del steps
    s = torch.cuda.current_stream().cuda_stream
    res["kernel"] = {}
    for name, opt in opts.items():
        model = models[name]
        eng, n = model._engine, model._layout.total
        bpp = FORMS[name][1]
        g, sh = [eng.grads.data_ptr()], [eng.shadow.data_ptr()]
        for form, bg in (("reduce", False), ("background", True)):
            if bg:
                opt.prepare_background(s)     # the per-step values the background form reads
            sec = time_kernel(lambda: opt.update_range(0, n, 1, 0, g, sh, s, background=bg), a.kernel_iters)
            res["kernel"]["%s_%s" % (name, form)] = {
                "us": round(sec * 1e6, 1), "bytes_per_param": bpp, "TB_per_s": round(bpp * n / sec / 1e12, 3),
                "fraction_of_3.35TB_s": round(bpp * n / sec / HBM_BYTES_PER_S, 3)}
        res["lower_bound_us_%d_B" % bpp] = round(bpp * n / HBM_BYTES_PER_S * 1e6, 1)
    res["parameters"] = n
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
