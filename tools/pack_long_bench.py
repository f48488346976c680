"""Packing past 128 tokens, measured: three rounds, each alternating its arms in one run.

  (a) config B's model and batch (bert-base, batch 16) padded to 512, valid lengths ~ U{16..512} (seeded): padded vs
      packed through Trainer.train_step with host batches (packing included), and the device-resident captured step
      (FusedTrainStep / PackedTrainStep replayed on staged inputs).
  (b) config A's model, batch 32, lengths from synthetic.REFERENCE_LENGTH_HISTOGRAM padded to 256 (max_seq_len = 256).
      The histogram caps its rows at 128 tokens; a row in its 128 bucket is given a length ~ U{129..256} here, the
      rare long row a 256-token max_seq_len no longer truncates.  Padded-256 vs packed (the Trainer's bin lengths:
      128, or 256 for a batch holding a long row) vs today's packed-128 on the same rows truncated to 128.
  (c) the attention kernels alone at (a)'s shapes, padded vs packed into 512-token bins (dropout 0.1, the backward
      with its dQ accumulator and conversion), cold (operand sets rotated past twice the 50 MB L2) and warm.  Bytes
      and flops each launch must move, counted from the masks / segments: HBM bytes are what the launch reads and
      writes once; flops count the 128 x 128 x 64 products of the blocks it visits (2 per key block in the forward,
      5 per query block in the backward).  Shares are of the larger of the HBM floor (3.35 TB/s) and the tensor
      floor (989 TFLOP/s dense BF16), the H100 SXM data-sheet figures.

Steps are timed with a host clock around work that ends in a device synchronise; kernels with CUDA events around a
captured loop (tools/attention_bench.py's timed_loop).  The GPU's name, power limit and max SM clock are read in the
same run.  One JSON line (--out also writes it to a file).
    python tools/pack_long_bench.py [--rounds 3] [--steps 20] [--out /tmp/pack_long_bench.json]
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
from pytorch_distributed_nlp_b200.packing import bin_length, pack_batch
from pytorch_distributed_nlp_b200.synthetic import reference_length_batch
from accum_bench import HBM_BYTES_PER_S, gpu_info
from attention_bench import L2_BYTES, timed_loop

TENSOR_FLOPS = 989e12
BLOCK_FLOPS = 2 * 128 * 128 * 64      # one 128 x 128 x 64 product
bf = torch.bfloat16


# ---- inputs -----------------------------------------------------------------------------------------------------------
def uniform_batch(cfg, B, S, seed, lo=16):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(lo, S + 1, (B,), generator=g)
    ids = torch.randint(1, cfg.vocab_size, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0] = min(101, cfg.vocab_size - 1)
    mask = (torch.arange(S)[None] < lens[:, None]).to(torch.int64)
    return {"input_ids": ids * mask, "token_type_ids": torch.zeros(B, S, dtype=torch.int64), "attention_mask": mask,
            "label": torch.randint(0, cfg.num_labels, (B,), generator=g, dtype=torch.int64)}


def histogram_batch(cfg, B, seed, S=256):
    """reference_length_batch at seq 128, its capped rows (length 128) given a length ~ U{129..S}, padded to S"""
    b = reference_length_batch(cfg, B, seed, 128)
    g = torch.Generator().manual_seed(seed + 7)
    lens = b["attention_mask"].sum(1)
    lens = torch.where(lens == 128, torch.randint(129, S + 1, (B,), generator=g), lens)
    ids = torch.randint(1, cfg.vocab_size, (B, S), generator=g, dtype=torch.int64)
    ids[:, 0] = min(101, cfg.vocab_size - 1)
    mask = (torch.arange(S)[None] < lens[:, None]).to(torch.int64)
    return {"input_ids": ids * mask, "token_type_ids": torch.zeros(B, S, dtype=torch.int64), "attention_mask": mask,
            "label": b["label"]}


def truncated(batch, S=128):
    return {k: (v[:, :S].contiguous() if v.dim() == 2 else v) for k, v in batch.items()}


# ---- step arms --------------------------------------------------------------------------------------------------------
def make_trainer(cfg, pack):
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg).cuda()
    args = b2.Args()
    args.local_rank, args.local_world_size, args.rank, args.pack = 0, 1, 0, pack
    opt = b2.build_optimizer(model, args)
    return model, opt, b2.Trainer(args, cfg, model, torch.nn.CrossEntropyLoss(), opt)


def trainer_rate(cfg, batches, pack, steps):
    """samples/s of Trainer.train_step over `steps` host batches (every batch's graph built in the warmup)"""
    model, opt, tr = make_trainer(cfg, pack)
    for b in batches:
        tr.train_step(b)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        loss = tr.train_step(batches[i % len(batches)])
    float(loss)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    B = batches[0]["input_ids"].shape[0]
    bins = sorted({k[2] for k in tr._packed}) if pack else None
    del model, opt, tr
    torch.cuda.empty_cache()
    return steps * B / dt, bins


def device_rate(cfg, batches, pack, steps):
    """samples/s of the captured step replayed on staged inputs (no host work, no H2D in the timed window)"""
    b2.set_seed(123)
    model = b2.BertForSequenceClassification(cfg).cuda()
    args = b2.Args()
    opt = b2.build_optimizer(model, args)
    model.train()
    runs = []
    for b in batches:
        B, S = b["input_ids"].shape
        if pack:
            bl = bin_length(b["attention_mask"], S)
            p = pack_batch(b["input_ids"], b["token_type_ids"], b["attention_mask"], bl)
            st = b2.PackedTrainStep(model, opt, p["bins"], B, bin_len=bl, criterion=torch.nn.CrossEntropyLoss())
            st.stage(p, b["label"])
        else:
            st = b2.FusedTrainStep(model, opt, B, S, criterion=torch.nn.CrossEntropyLoss())
            st.stage(b)
        for _ in range(4):      # two eager warm-up runs, the capture, one replay: the timed loop only replays
            st.run_device()
        runs.append(st)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        runs[i % len(runs)].run_device()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    B = batches[0]["input_ids"].shape[0]
    del model, opt, runs
    torch.cuda.empty_cache()
    return steps * B / dt


# ---- kernel arm -------------------------------------------------------------------------------------------------------
def visited_blocks(seg, S):
    """(fwd key blocks, bwd query blocks) the packed kernels visit, summed over bins, from the segment words"""
    lo, hi = (seg & 0xffff).long(), (seg >> 16).long()
    nb = S // 128
    fwd = bwd = 0
    for b in range(seg.shape[0]):
        for k in range(nb):
            rows = slice(128 * k, 128 * k + 128)
            fwd += (int(hi[b, rows].max()) + 127) // 128 - int(lo[b, rows].min()) // 128
            bwd += (int(hi[b, 128 * k + 127]) + 127) // 128 - int(lo[b, 128 * k]) // 128
    return fwd, bwd


def kernel_round(cfg, batch, rep):
    B, S = batch["input_ids"].shape
    NH, H = cfg.num_attention_heads, cfg.hidden_size
    P = 0.1
    dev = "cuda"
    stream = lambda: torch.cuda.current_stream().cuda_stream
    rs = torch.tensor([1234, 5], dtype=torch.int64, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    mask = batch["attention_mask"].to(dev)
    seg = pack_batch(batch["input_ids"], batch["token_type_ids"], batch["attention_mask"], S)["segments"].to(dev)
    out = {}
    for name, nb in (("padded", B), ("packed", seg.shape[0])):
        rows = nb * S
        sets_needed = None

        def make(rows=rows):
            return {"qkv": (torch.randn(rows, 3 * H, device=dev, generator=gen) * 0.5).to(bf),
                    "dctx": torch.randn(rows, H, device=dev, generator=gen).to(bf),
                    "ctx": torch.empty(rows, H, dtype=bf, device=dev),
                    "lse": torch.empty(rows * NH, dtype=torch.float32, device=dev),
                    "dqkv": torch.empty(rows, 3 * H, dtype=bf, device=dev),
                    "dq": torch.empty(rows, H, dtype=torch.float32, device=dev)}

        def fwd(s, nb=nb, name=name):
            if name == "padded":
                L.call("b2_attention_fwd", s["qkv"].data_ptr(), mask.data_ptr(), nb, S, NH, 64, P, rs.data_ptr(), 4,
                       s["ctx"].data_ptr(), s["lse"].data_ptr(), None, stream())
            else:
                L.call("b2_attention_fwd_packed_seq", s["qkv"].data_ptr(), seg.data_ptr(), nb, S, NH, 64, P,
                       rs.data_ptr(), 4, s["ctx"].data_ptr(), s["lse"].data_ptr(), None, stream())

        def bwd(s, nb=nb, name=name):
            if name == "padded":
                L.call("b2_attention_bwd", s["qkv"].data_ptr(), mask.data_ptr(), s["ctx"].data_ptr(),
                       s["dctx"].data_ptr(), s["lse"].data_ptr(), nb, S, NH, 64, P, rs.data_ptr(), 4,
                       s["dqkv"].data_ptr(), s["dq"].data_ptr(), None, None, stream())
            else:
                L.call("b2_attention_bwd_packed_seq", s["qkv"].data_ptr(), seg.data_ptr(), s["ctx"].data_ptr(),
                       s["dctx"].data_ptr(), s["lse"].data_ptr(), nb, S, NH, 64, P, rs.data_ptr(), 4,
                       s["dqkv"].data_ptr(), s["dq"].data_ptr(), None, None, stream())

        if name == "padded":
            nbk = S // 128
            v_fwd = v_bwd = B * nbk * nbk
        else:
            v_fwd, v_bwd = visited_blocks(seg.cpu(), S)
        mat = rows * H * 2                                   # one [rows, hidden] bf16 matrix
        lse_b = rows * NH * 4
        nbytes = {"fwd": 3 * mat + mat + lse_b,
                  # qkv, dO, O, lse in; dqkv out; the fp32 dQ accumulator cleared, added into, read back
                  "bwd": 3 * mat + 2 * mat + lse_b + 3 * mat + 3 * rows * H * 4}
        flops = {"fwd": NH * v_fwd * 2 * BLOCK_FLOPS, "bwd": NH * v_bwd * 5 * BLOCK_FLOPS}
        set_bytes = 9 * mat + lse_b + rows * H * 4
        nsets = max(2, -(-2 * L2_BYTES // set_bytes) + 1)
        sets_needed = [make() for _ in range(nsets)]
        for s in sets_needed:
            fwd(s)
        torch.cuda.synchronize()
        for kname, fn in (("fwd", fwd), ("bwd", bwd)):
            cold = timed_loop(fn, sets_needed, rep)
            warm = timed_loop(fn, sets_needed[:1], rep * nsets)
            floor_hbm = nbytes[kname] / HBM_BYTES_PER_S * 1e6
            floor_tc = flops[kname] / TENSOR_FLOPS * 1e6
            floor = max(floor_hbm, floor_tc)
            out["%s_%s" % (kname, name)] = {
                "us": round(cold, 2), "us_warm": round(warm, 2), "MB": round(nbytes[kname] / 1e6, 1),
                "GFLOP": round(flops[kname] / 1e9, 2), "floor_us": round(floor, 2),
                "bound": "hbm" if floor_hbm >= floor_tc else "tensor", "share": round(floor / cold, 3),
                "share_warm": round(floor / warm, 3), "bins": nb, "visited_blocks": v_fwd if kname == "fwd" else v_bwd}
        del sets_needed
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the arms")
    ap.add_argument("--steps", type=int, default=20, help="timed steps per arm and round")
    ap.add_argument("--rep", type=int, default=20, help="launches per operand set in the kernel loops")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"gpu": gpu_info(), "rounds": a.rounds, "steps": a.steps}

    cfg_b = b2.bert_base_config(num_labels=6)
    batches_b = [uniform_batch(cfg_b, 16, 512, 100 + i) for i in range(4)]
    cfg_a = b2.chinese_bert_wwm_ext_config(num_labels=6, max_position_embeddings=512)
    batches_a = [histogram_batch(cfg_a, 32, 200 + i) for i in range(8)]
    arms = {
        "a_trainer_padded512": lambda: trainer_rate(cfg_b, batches_b, False, a.steps)[0],
        "a_trainer_packed": lambda: trainer_rate(cfg_b, batches_b, True, a.steps)[0],
        "a_device_padded512": lambda: device_rate(cfg_b, batches_b, False, a.steps),
        "a_device_packed": lambda: device_rate(cfg_b, batches_b, True, a.steps),
        "b_trainer_padded256": lambda: trainer_rate(cfg_a, batches_a, False, a.steps)[0],
        "b_trainer_packed": lambda: trainer_rate(cfg_a, batches_a, True, a.steps)[0],
        "b_trainer_packed128_truncated": lambda: trainer_rate(cfg_a, [truncated(b) for b in batches_a], True,
                                                              a.steps)[0],
    }
    rates = {k: [] for k in arms}
    for r in range(a.rounds):
        for k, fn in arms.items():
            rates[k].append(fn())
            print("round %d %s: %.1f samples/s" % (r, k, rates[k][-1]), file=sys.stderr, flush=True)
    res["samples_per_s"] = {k: {"median": round(statistics.median(v), 1), "runs": [round(x, 1) for x in v]}
                            for k, v in rates.items()}
    res["b_bin_lengths"] = [bin_length(b["attention_mask"], 256) for b in batches_a]
    res["a_mean_valid_tokens"] = round(float(torch.cat([b["attention_mask"].sum(1) for b in batches_b]).float().mean()), 1)
    res["b_mean_valid_tokens"] = round(float(torch.cat([b["attention_mask"].sum(1) for b in batches_a]).float().mean()), 1)
    res["kernels"] = kernel_round(cfg_b, batches_b[0], a.rep)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
