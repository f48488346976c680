"""The seq-128 fused attention kernels alone, at BASELINE config A's shapes and in the form the training step issues
them (batch 32, seq 128, 12 heads of 64, dropout 0.1 with the keep-bit cache, the reference's padding mask, the
fused QKV-bias sums in the backward), and in the packed form on the bins of the same reference-shaped batch.

Each launch form is timed as bench.py's GEMM table times its kernels: a loop of launches captured once in a CUDA
graph, bracketed by CUDA events.  "cold" rotates operand sets spanning more than twice the 50 MB L2, "warm" reuses one.
Printed per form: us per launch, the bytes the launch must move (the floor at the H100 SXM's 3.35 TB/s data-sheet
HBM3 bandwidth) and the achieved fraction of it, with the GPU's name, power limit and max SM clock read in the same
run (one JSON line; --out also writes it to a file).
    python tools/attention_bench.py [--rep 50] [--out /tmp/attention_bench.json]
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
from pytorch_distributed_nlp_b200.packing import pack_batch
from pytorch_distributed_nlp_b200.synthetic import reference_length_batch
from accum_bench import HBM_BYTES_PER_S, gpu_info

L2_BYTES = 50 * 2 ** 20
B, S, NH, P = 32, 128, 12, 0.1
H = NH * 64
bf = torch.bfloat16


def timed_loop(launch_one, sets, rep):
    """mean device time of one launch over rep x len(sets) launches captured in one graph"""
    for s in sets:
        launch_one(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(rep):
            for s in sets:
                launch_one(s)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (rep * len(sets))


def make_set(rows, gen):
    """one operand set of `rows` token rows: qkv, dO, and the forward's ctx / lse / keep bits / dbias buffers"""
    dev = "cuda"
    s = {"qkv": (torch.randn(rows, 3 * H, device=dev, generator=gen) * 0.5).to(bf),
         "dctx": torch.randn(rows, H, device=dev, generator=gen).to(bf),
         "ctx": torch.empty(rows, H, dtype=bf, device=dev),
         "lse": torch.empty(rows * NH, dtype=torch.float32, device=dev),
         "kb": torch.zeros(rows * NH * 2, dtype=torch.int64, device=dev),
         "dqkv": torch.empty(rows, 3 * H, dtype=bf, device=dev),
         "dbias": torch.zeros(3 * H, dtype=torch.float32, device=dev)}
    return s


def forms():
    cfg = b2.chinese_bert_wwm_ext_config(num_labels=6)
    batch = reference_length_batch(cfg, B, 1000, S)
    mask = batch["attention_mask"].cuda()
    seg = pack_batch(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"])["segments"].cuda()
    return {"padded": (B, mask, None), "packed": (seg.shape[0], None, seg.contiguous())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rep", type=int, default=50, help="launches per operand set in the timed graph")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    stream = lambda: torch.cuda.current_stream().cuda_stream
    rs = torch.tensor([1234, 5], dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(0)
    res = {"config": "A", "batch": B, "seq": S, "heads": NH, "dropout": P, "gpu": gpu_info(), "kernels": {}}
    for name, (nb, mask, seg) in forms().items():
        rows = nb * S
        items = nb * NH

        def fwd(s):
            if seg is None:
                L.call("b2_attention_fwd", s["qkv"].data_ptr(), mask.data_ptr(), nb, S, NH, 64, P, rs.data_ptr(), 4,
                       s["ctx"].data_ptr(), s["lse"].data_ptr(), s["kb"].data_ptr(), stream())
            else:
                L.call("b2_attention_fwd_packed", s["qkv"].data_ptr(), seg.data_ptr(), nb, NH, 64, P, rs.data_ptr(), 4,
                       s["ctx"].data_ptr(), s["lse"].data_ptr(), s["kb"].data_ptr(), stream())

        def bwd(s):
            if seg is None:
                L.call("b2_attention_bwd", s["qkv"].data_ptr(), mask.data_ptr(), s["ctx"].data_ptr(),
                       s["dctx"].data_ptr(), s["lse"].data_ptr(), nb, S, NH, 64, P, rs.data_ptr(), 4,
                       s["dqkv"].data_ptr(), 0, s["dbias"].data_ptr(), s["kb"].data_ptr(), stream())
            else:
                L.call("b2_attention_bwd_packed", s["qkv"].data_ptr(), seg.data_ptr(), s["ctx"].data_ptr(),
                       s["dctx"].data_ptr(), s["lse"].data_ptr(), nb, NH, 64, P, rs.data_ptr(), 4,
                       s["dqkv"].data_ptr(), s["dbias"].data_ptr(), s["kb"].data_ptr(), stream())

        # bytes each launch must move: qkv 3 tiles in; ctx, lse, keep bits out (fwd); qkv, dO, O, lse, keep bits in,
        # dqkv out (bwd); the mask / segment words are negligible
        tile = rows * 64 * 2 * NH            # one [rows, hidden] bf16 matrix
        lse_b, kb_b = rows * NH * 4, rows * NH * 16
        nbytes = {"fwd": 3 * tile + tile + lse_b + kb_b, "bwd": 3 * tile + 2 * tile + lse_b + kb_b + 3 * tile}
        set_bytes = 8 * tile + lse_b + kb_b
        nsets = max(2, -(-2 * L2_BYTES // set_bytes) + 1)
        sets = [make_set(rows, gen) for _ in range(nsets)]
        for s in sets:
            fwd(s)
        torch.cuda.synchronize()
        for kname, fn in (("fwd", fwd), ("bwd", bwd)):
            cold = timed_loop(fn, sets, a.rep)
            warm = timed_loop(fn, sets[:1], a.rep * nsets)
            floor = nbytes[kname] / HBM_BYTES_PER_S * 1e6
            res["kernels"]["%s_%s" % (kname, name)] = {
                "us": round(cold, 2), "us_warm": round(warm, 2), "MB": round(nbytes[kname] / 1e6, 1),
                "floor_us": round(floor, 2), "fraction_of_3.35TB_s": round(floor / cold, 3),
                "fraction_warm": round(floor / warm, 3), "items": items, "rotated_sets": nsets,
                "rotated_mb": round(nsets * set_bytes / 2 ** 20)}
        del sets
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
