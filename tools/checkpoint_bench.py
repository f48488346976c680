"""Checkpoint cost on one GPU, BASELINE config A (seq 128, batch 32, dropout on), build_optimizer's HF AdamW.

  * optimizer.state_dict() + torch.save into a temporary directory (the moments: 8 B per parameter);
  * optimizer.load_state_dict() of that file (torch.load to the CPU included, and without it);
  * Trainer.save_checkpoint() (weights, config, optimizer, scheduler, RNG files, trainer state);
  * the median captured step (FusedTrainStep replays of one graph) over --rounds rounds before, and as many after, a
    load of the saved optimizer and weights into the same objects, in this one run: the loaded state must cost the
    step nothing.
Wall-clock times of the host calls (median of --reps), CUDA-event times of the steps.  The GPU's name, power limit and
max SM clock are read in the same run and printed with the numbers (one JSON line; --out also writes it to a file).
Writes only under a temporary directory, removed at the end.
    python tools/checkpoint_bench.py [--steps 30] [--rounds 3] [--reps 3] [--out /tmp/checkpoint_bench.json]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch

import pytorch_distributed_nlp_b200 as b2
from accum_bench import gpu_info
from clip_bench import time_steps


def _wall(fn, reps):
    """median wall-clock seconds of fn() with the device idle before and after"""
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return sorted(out)[len(out) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30, help="timed steps per round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    B, S = 32, 128
    res = {"config": "A", "batch": B, "seq": S, "optimizer": "hf_adamw", "gpu": gpu_info()}
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg).cuda().train()
    args = b2.Args()
    args.local_rank = 0
    opt = b2.build_optimizer(model, args)
    tr = b2.Trainer(args, cfg, model, None, opt)
    step = b2.FusedTrainStep(model, opt, B, S)
    step.stage(b2.synthetic_batch(cfg, B, S, 1000, padded=True))
    for _ in range(5):                 # warm-up and capture
        step.run_device()
    torch.cuda.synchronize()
    graph = step.graph
    tmp = tempfile.mkdtemp(prefix="b2-ckpt-bench-")
    try:
        f = os.path.join(tmp, "optimizer.pt")
        res["state_dict_save_s"] = round(_wall(lambda: torch.save(opt.state_dict(), f), a.reps), 4)
        res["optimizer_file_MB"] = round(os.path.getsize(f) / 2 ** 20, 1)
        res["load_state_dict_with_torch_load_s"] = round(
            _wall(lambda: opt.load_state_dict(torch.load(f, map_location="cpu")), a.reps), 4)
        sd = torch.load(f, map_location="cpu")
        res["load_state_dict_s"] = round(_wall(lambda: opt.load_state_dict(sd), a.reps), 4)
        res["save_checkpoint_s"] = round(_wall(lambda: tr.save_checkpoint(os.path.join(tmp, "checkpoint-1")), a.reps), 4)
        res["checkpoint_MB"] = round(sum(os.path.getsize(os.path.join(tmp, "checkpoint-1", x))
                                         for x in os.listdir(os.path.join(tmp, "checkpoint-1"))) / 2 ** 20, 1)
        before, after = [], []
        for _ in range(a.rounds):
            before.append(time_steps(step, a.steps))
        opt.load_state_dict(torch.load(f, map_location="cpu"))
        model.load_state_dict(torch.load(os.path.join(tmp, "checkpoint-1", "pytorch_model.bin")))
        for _ in range(a.rounds):
            after.append(time_steps(step, a.steps))
        assert step.graph is graph
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    med = lambda v: sorted(v)[len(v) // 2]
    res["step_ms_before_load"] = {"rounds": [round(x, 4) for x in before], "median": round(med(before), 4)}
    res["step_ms_after_load"] = {"rounds": [round(x, 4) for x in after], "median": round(med(after), 4)}
    res["parameters"] = model._layout.total
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fp:
            fp.write(line + "\n")


if __name__ == "__main__":
    main()
