"""BertForMultipleChoice, measured at config A's encoder (chinese-bert-wwm-ext): B = 8 examples of N = 4 choices of 128
tokens, the same 32 x 128 token rows as config A's step.

  (a) the captured training step (FusedTrainStep replayed on staged inputs, host clock around a synchronised window)
      of the multiple-choice model against config A's captured sequence step (C 6) on the same flattened rows;
  (b) the same two steps packed (PackedTrainStep, 128-token bins) on rows whose lengths follow
      synthetic.REFERENCE_LENGTH_HISTOGRAM;
  (c) stock transformers.BertForMultipleChoice (sdpa attention, torch fused AdamW) under bf16 autocast, one eager step
      per call on the padded batches.
The arms alternate within each round.  The card's name, power limit and max SM clock are read in the same run.  One
JSON line.
    python tools/mc_bench.py [--rounds 5] [--steps 20]
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
from pytorch_distributed_nlp_b200.synthetic import reference_length_batch
from accum_bench import gpu_info

B, N, S = 8, 4, 128


def as_choices(flat, seed):
    """a [B·N, S] batch as [B, N, S] choices with one choice label per example"""
    g = torch.Generator().manual_seed(seed)
    bt = {k: flat[k].reshape(B, N, S) for k in ("input_ids", "token_type_ids", "attention_mask")}
    bt["label"] = torch.randint(0, N, (B,), generator=g, dtype=torch.int64)
    return bt


def step_arm(kind, packed, flats):
    """a captured step of the multiple-choice model (kind "mc") or config A's sequence model ("sequence") on `flats`"""
    mc = kind == "mc"
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    b2.set_seed(123)
    model = (b2.BertForMultipleChoice if mc else b2.BertForSequenceClassification)(cfg).cuda().train()
    opt = b2.build_optimizer(model, b2.Args())
    batches = [as_choices(f, 300 + i) if mc else f for i, f in enumerate(flats)]
    if not packed:
        st = b2.FusedTrainStep(model, opt, B if mc else B * N, S, choices=N if mc else None)
        for bt in batches:
            st.stage(bt)
            st.run_device()
        return lambda: st.run_device()
    bt = batches[0]
    p = b2.pack_batch(bt["input_ids"], bt["token_type_ids"], bt["attention_mask"], 128)
    st = b2.PackedTrainStep(model, opt, p["bins"], B if mc else B * N, choices=N if mc else None)
    st.stage(p, bt["label"])
    for _ in range(3):
        st.run_device()
    return lambda: st.run_device()


def hf_arm(flats):
    """stock HF BertForMultipleChoice, one eager bf16-autocast step per call"""
    from transformers import BertConfig, BertForMultipleChoice
    torch.manual_seed(123)
    m = BertForMultipleChoice(BertConfig(vocab_size=21128)).cuda().train()
    opt = torch.optim.AdamW(m.parameters(), lr=3e-5, fused=True)
    dev = []
    for i, f in enumerate(flats):
        bt = as_choices(f, 400 + i)
        dev.append({"input_ids": bt["input_ids"].cuda(), "token_type_ids": bt["token_type_ids"].cuda(),
                    "attention_mask": bt["attention_mask"].cuda(), "labels": bt["label"].cuda()})
    it = [0]

    def run():
        d = dev[it[0] % len(dev)]
        it[0] += 1
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = m(**d)
        out.loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    for _ in range(3):
        run()
    return run


def time_steps(run, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        run()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mc_bench needs a GPU")
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    full = []
    for i in range(3):
        bt = b2.synthetic_mc_batch(cfg, B, N, S, 100 + i)
        full.append({k: v.reshape(B * N, S) for k, v in bt.items() if k != "label"})
        full[-1]["label"] = torch.randint(0, 6, (B * N,), generator=torch.Generator().manual_seed(i))
    ref = [reference_length_batch(cfg, B * N, 100 + i, S) for i in range(3)]
    arms = {"mc_padded": step_arm("mc", False, full), "sequence_padded": step_arm("sequence", False, full),
            "mc_packed": step_arm("mc", True, ref), "sequence_packed": step_arm("sequence", True, ref),
            "hf_mc_bf16_autocast": hf_arm(full)}
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, run in arms.items():
            times[k].append(time_steps(run, args.steps))
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"gpu": gpu_info(), "examples": B, "choices": N, "seq": S,
           "steps": {k: {"median_ms": round(1e3 * med[k], 3), "examples_per_s": round(B / med[k], 1),
                         "rounds_ms": [round(1e3 * t, 3) for t in v]} for k, v in times.items()},
           "mc_vs_sequence_padded": round(med["mc_padded"] / med["sequence_padded"], 3),
           "mc_vs_sequence_packed": round(med["mc_packed"] / med["sequence_packed"], 3),
           "hf_vs_mc_padded": round(med["hf_mc_bf16_autocast"] / med["mc_padded"], 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
