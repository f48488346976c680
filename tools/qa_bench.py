"""BertForQuestionAnswering, measured at config A (chinese-bert-wwm-ext, batch 32, seq 128) and at SQuAD's shape (batch
32, seq 384).

  (a) the captured training step (FusedTrainStep replayed on staged inputs, host clock around a synchronised window)
      of the QA model against the token model (C 9) and the sequence model (C 6), at both shapes; the arms alternate
      within each round;
  (b) the same steps packed (PackedTrainStep, 128-token bins) on rows whose lengths follow
      synthetic.REFERENCE_LENGTH_HISTOGRAM;
  (c) stock transformers.BertForQuestionAnswering (sdpa attention, torch fused AdamW) under bf16 autocast, one
      eager step at each shape;
  (d) the span-loss kernel alone (CUDA events around a captured loop) at 32 x 128 and 32 x 384 rows, against the HBM
      floor of the bytes it must move once: logits (M x 2 fp32) read twice, positions, d_logits (M x 2 fp32) written.
The card's name, power limit and max SM clock are read in the same run.  One JSON line.
    python tools/qa_bench.py [--rounds 3] [--steps 20]
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
from pytorch_distributed_nlp_b200.synthetic import reference_length_batch
from accum_bench import HBM_BYTES_PER_S, gpu_info
from attention_bench import timed_loop

B = 32
LABELS = {"qa": 2, "token": 9, "sequence": 6}
CLASSES = {"qa": "BertForQuestionAnswering", "token": "BertForTokenClassification",
           "sequence": "BertForSequenceClassification"}


def batch_for(kind, base, seed):
    """`base` (input ids / types / mask) with the labels of `kind`"""
    g = torch.Generator().manual_seed(seed)
    bt = {k: base[k] for k in ("input_ids", "token_type_ids", "attention_mask")}
    lens = bt["attention_mask"].sum(1)
    if kind == "qa":
        s = (torch.rand(B, generator=g) * lens).long()
        bt["start_positions"] = s
        bt["end_positions"] = torch.minimum(s + torch.randint(0, 8, (B,), generator=g), lens - 1)
    elif kind == "token":
        lab = torch.randint(0, 9, bt["input_ids"].shape, generator=g, dtype=torch.int64)
        lab[bt["attention_mask"] == 0] = -100
        bt["label"] = lab
    else:
        bt["label"] = torch.randint(0, 6, (B,), generator=g, dtype=torch.int64)
    return bt


def step_arm(kind, S, packed, bases):
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=LABELS[kind])
    b2.set_seed(123)
    model = getattr(b2, CLASSES[kind])(cfg).cuda().train()
    opt = b2.build_optimizer(model, b2.Args())
    batches = [batch_for(kind, bs, 300 + i) for i, bs in enumerate(bases)]
    if not packed:
        st = b2.FusedTrainStep(model, opt, B, S)
        for bt in batches:
            st.stage(bt)
            st.run_device()
        return lambda: st.run_device()
    bt = batches[0]
    kw = dict(start_positions=bt["start_positions"], end_positions=bt["end_positions"]) if kind == "qa" else {}
    p = b2.pack_batch(bt["input_ids"], bt["token_type_ids"], bt["attention_mask"], 128,
                      labels=bt["label"] if kind == "token" else None, **kw)
    st = b2.PackedTrainStep(model, opt, p["bins"], B, seq_len=S if kind == "qa" else None)
    label = p["labels"] if kind == "token" else \
        torch.stack([p["start_positions"], p["end_positions"]]) if kind == "qa" else bt["label"]
    st.stage(p, label)
    for _ in range(3):
        st.run_device()
    return lambda: st.run_device()


def hf_arm(S, bases):
    """stock HF BertForQuestionAnswering, one eager bf16-autocast step per call"""
    from transformers import BertConfig, BertForQuestionAnswering
    hc = BertConfig(vocab_size=21128, num_labels=2)
    torch.manual_seed(123)
    m = BertForQuestionAnswering(hc).cuda().train()
    opt = torch.optim.AdamW(m.parameters(), lr=3e-5, fused=True)
    dev = [{k: v.cuda() for k, v in batch_for("qa", bs, 400 + i).items()} for i, bs in enumerate(bases)]
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


def kernel_time(S, rep=200):
    dev = torch.device("cuda")
    M = B * S
    g = torch.Generator().manual_seed(S)
    sets = []
    for _ in range(4):
        sets.append(dict(x=torch.randn(M, 2, generator=g).to(dev), dl=torch.empty(M, 2, device=dev),
                         pos=torch.randint(0, S, (2, B), generator=g).to(dev)))
    seq_loss, loss = torch.empty(2 * B, device=dev), torch.empty((), device=dev)

    def launch(s):
        L.call("b2_qa_span_loss", s["x"].data_ptr(), M, s["pos"].data_ptr(), s["pos"].data_ptr() + 8 * B, B, S, None,
               None, None, seq_loss.data_ptr(), s["dl"].data_ptr(), loss.data_ptr(),
               torch.cuda.current_stream().cuda_stream)
    for s in sets:
        launch(s)
    torch.cuda.synchronize()
    t_us = timed_loop(launch, sets, rep)
    bytes_ = 2 * M * 8 + 2 * B * 8 * 2 + M * 8 + 2 * B * 4
    floor_us = 1e6 * bytes_ / HBM_BYTES_PER_S
    return {"us": round(t_us, 2), "bytes": bytes_, "hbm_floor_us": round(floor_us, 3),
            "share_of_hbm_floor": round(floor_us / t_us, 4), "launches": 2}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qa_bench needs a GPU")
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=2)
    res = {"gpu": gpu_info(), "batch": B}
    for S in (128, 384):
        full = [b2.synthetic_qa_batch(cfg, B, S, 100 + i) for i in range(3)]
        ref = [reference_length_batch(cfg, B, 100 + i, S) for i in range(3)]
        arms = {}
        for kind in ("qa", "token", "sequence"):
            arms["%s_padded" % kind] = step_arm(kind, S, False, full)
            arms["%s_packed" % kind] = step_arm(kind, S, True, ref)
        arms["hf_qa_bf16_autocast"] = hf_arm(S, full)
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, run in arms.items():
                times[k].append(time_steps(run, args.steps))
        med = {k: statistics.median(v) for k, v in times.items()}
        res["seq%d" % S] = {
            "steps": {k: {"median_ms": round(1e3 * med[k], 3), "samples_per_s": round(B / med[k], 1),
                          "rounds_ms": [round(1e3 * t, 3) for t in v]} for k, v in times.items()},
            "qa_vs_token_padded": round(med["qa_padded"] / med["token_padded"], 3),
            "qa_vs_sequence_padded": round(med["qa_padded"] / med["sequence_padded"], 3),
            "qa_vs_token_packed": round(med["qa_packed"] / med["token_packed"], 3),
            "hf_vs_qa_padded": round(med["hf_qa_bf16_autocast"] / med["qa_padded"], 3),
            "span_loss_kernel": kernel_time(S)}
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
