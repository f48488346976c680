"""Context number (SURVEY.md §8d, last row): the reference's loop body in stock torch eager on ONE GPU -- HF
BertForSequenceClassification (eager attention, as transformers 4.28.1 computes it), the restated HF AdamW run the
way the original runs it (a python loop of per-tensor ops), cuBLAS/cuDNN kernels, no graph.  Three precisions:
fp32 (what multi-gpu-distributed-cls.py runs), TF32 matmuls, bf16 autocast (what the -amp scripts run, minus the
GradScaler).  NOT a pytest module (no test_ prefix), not part of bench.py's contract; run it by hand:

    python tests/context_torch_eager.py > torch_eager.json

Lives under tests/ because it drives oracle/ code (test infrastructure); nothing in the product imports it.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import pytorch_distributed_nlp_b200 as b2  # noqa: E402
from oracle import bert_ref, cpu_step  # noqa: E402

BATCH, SEQ, WARM, STEPS = 32, 128, 10, 30


def run(mode):
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    torch.backends.cudnn.allow_tf32 = mode == "tf32"
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    model = cpu_step.build_hf_model(cfg).cuda().train()
    opt = cpu_step._HFOpt(model, 3e-5, 0.01)
    crit = torch.nn.CrossEntropyLoss()
    ring = [{k: v.cuda() for k, v in bert_ref.synthetic_batch(cfg, BATCH, SEQ, 1000 + i).items()} for i in range(8)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    loss = None
    for i in range(WARM + STEPS):
        if i == WARM:
            torch.cuda.synchronize()
            e0.record()
        b = ring[i % len(ring)]
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "bf16_autocast")):
            out = model(input_ids=b["input_ids"], token_type_ids=b["token_type_ids"],
                        attention_mask=b["attention_mask"], labels=b["label"])
            loss = crit(out[1].float(), b["label"])
        opt.zero_grad()
        loss.backward()
        opt.step()
        loss.item()                      # the reference formats the loss every step (:179)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / STEPS
    return {"mode": mode, "ms_per_step": round(ms, 3), "samples_per_s": round(BATCH / ms * 1e3, 1),
            "final_loss": round(float(loss), 5)}


if __name__ == "__main__":
    res = {"what": "stock torch-eager HF BERT-base step on one GPU (context, SURVEY 8d)", "batch": BATCH, "seq": SEQ,
           "steps": STEPS, "warmup": WARM, "torch": torch.__version__, "runs": [run(m) for m in
                                                                              ("fp32", "tf32", "bf16_autocast")]}
    print(json.dumps(res))
