"""Summarises an `ncu --csv` metric log of one training step into per-kernel evidence (JSON on stdout):
tensor-pipe utilisation for the wgmma kernels, DRAM bytes and achieved GB/s for the memory-bound ones.

    ncu --metrics gpu__time_duration.sum,sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed,\\
sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_elapsed,\\
sm__ops_path_tensor_op_hmma_src_bf16_dst_fp32.sum,dram__bytes_read.sum,dram__bytes_write.sum \\
        --clock-control none -s <first launch of the step> -c <launches per step> --csv --log-file counters.csv \\
        python tools/profile_step.py 3
    python tools/ncu_counters.py counters.csv [peaks.json] > ncu_counters.json
Times under ncu are cold-cache and serialised: shares and per-launch counters are the evidence, not the absolute step.
"""
import csv
import json
import re
import sys
from collections import OrderedDict


def parse(path):
    rows = []
    with open(path, newline="") as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    rd = csv.DictReader(lines)
    for r in rd:
        rows.append(r)
    return rows


def short(name):
    name = re.sub(r"^void\s+", "", name)
    name = re.sub(r"\(.*$", "", name)
    return name.replace("b2::", "").replace("(anonymous namespace)::", "")


def main():
    rows = parse(sys.argv[1])
    peaks = json.load(open(sys.argv[2])) if len(sys.argv) > 2 else {}
    launches = OrderedDict()      # launch id -> dict
    for r in rows:
        lid = r.get("ID")
        d = launches.setdefault(lid, {"kernel": short(r.get("Kernel Name", "?"))})
        try:
            v = float(str(r.get("Metric Value", "")).replace(",", ""))
        except ValueError:
            continue
        unit = r.get("Metric Unit", "")
        name = r.get("Metric Name", "")
        if name == "gpu__time_duration.sum":
            v = v / 1e3 if unit in ("nsecond", "ns") else (v * 1e3 if unit in ("msecond", "ms") else v)   # -> us
        if name.startswith("dram__bytes"):
            scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1.0)
            v *= scale
        d[name] = v
    # one step = the launches after the second-to-last step_advance_kernel up to and including the last one
    seq = list(launches.values())
    marks = [i for i, d in enumerate(seq) if "step_advance_kernel" in d["kernel"]]
    if len(marks) >= 2:
        seq = seq[marks[-2] + 1: marks[-1] + 1]
    per = OrderedDict()
    for d in seq:
        k = per.setdefault(d["kernel"], {"launches": 0, "us": 0.0, "tensor_pct": [], "hmma_pct": [], "rd": 0.0, "wr": 0.0,
                                         "ops": 0.0})
        k["launches"] += 1
        k["us"] += d.get("gpu__time_duration.sum", 0.0)
        for key, dst in (("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor_pct"),
                         ("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_elapsed", "hmma_pct")):
            if key in d:
                k[dst].append((d[key], d.get("gpu__time_duration.sum", 0.0)))
        k["rd"] += d.get("dram__bytes_read.sum", 0.0)
        k["wr"] += d.get("dram__bytes_write.sum", 0.0)
        k["ops"] += d.get("sm__ops_path_tensor_op_hmma_src_bf16_dst_fp32.sum", 0.0)
    total_us = sum(k["us"] for k in per.values()) or 1.0
    out = []
    for name, k in sorted(per.items(), key=lambda kv: -kv[1]["us"]):
        def wavg(lst):
            w = sum(t for _v, t in lst)
            return round(sum(v * t for v, t in lst) / w, 2) if w > 0 else None
        n = k["launches"]
        row = {"kernel": name, "launches": n, "total_us": round(k["us"], 1), "avg_us": round(k["us"] / n, 2),
               "share_pct": round(100 * k["us"] / total_us, 1),
               "tensor_pipe_pct_of_peak": wavg(k["tensor_pct"]), "hmma_subpipe_pct_of_peak": wavg(k["hmma_pct"]),
               "dram_read_mb_per_launch": round(k["rd"] / n / 1e6, 2), "dram_write_mb_per_launch": round(k["wr"] / n / 1e6, 2),
               "dram_gbs": round((k["rd"] + k["wr"]) / (k["us"] * 1e-6) / 1e9, 1) if k["us"] > 0 else None}
        if k["ops"] > 0:
            row["tensor_tflops"] = round(k["ops"] / (k["us"] * 1e-6) / 1e12, 1)   # counter counts FMA-halves as ops
        if peaks.get("hbm_gbs") and row["dram_gbs"] is not None:
            row["dram_frac_of_measured_peak"] = round(row["dram_gbs"] / peaks["hbm_gbs"], 3)
        out.append(row)
    print(json.dumps({"source": "ncu --metrics ... --clock-control none, one eager training step (tools/profile_step.py)",
                      "note": "cold-cache serialised launches: shares and per-launch counters are the evidence",
                      "total_us": round(total_us, 1), "kernels": out}, indent=1))


if __name__ == "__main__":
    main()
