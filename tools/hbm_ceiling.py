#!/usr/bin/env python3
"""Measures the read-only HBM stream rate of GPU 0: the ceiling the substring scan's roofline is set against.

    python tools/hbm_ceiling.py [--gib 32] [--runs 10]

Compiles tools/hbm_read.cu for sm_90a into a temporary directory, runs it (a persistent grid of 16-byte loads over a buffer of --gib GiB,
the median of --runs CUDA-event-timed passes after two warm-up passes) and prints one JSON line: GB/s with the card's name, its power
limit and the SM clock nvidia-smi reports while the passes run.  Nothing is written to the repository."""
import argparse
import json
import os
import statistics
import subprocess
import tempfile
import threading

HERE = os.path.dirname(os.path.abspath(__file__))


def smi(*fields):
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + ",".join(fields), "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
    return [x.strip() for x in out.strip().split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=32.0)
    ap.add_argument("--runs", type=int, default=10)
    args = ap.parse_args()
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "hbm_read")
        subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe, os.path.join(HERE, "hbm_read.cu")])
        samples = []
        sampler = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-lms", "100"],
                                   stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        reader = threading.Thread(target=lambda: samples.extend(line.strip() for line in sampler.stdout), daemon=True)
        reader.start()
        try:
            line = subprocess.run([exe, str(args.gib), str(args.runs)], capture_output=True, text=True, check=True).stdout.strip()
        finally:
            sampler.terminate()
            sampler.wait(timeout=5)
    res = dict(kv.split("=", 1) for kv in line.split(" ", 6))
    name, power_limit, sm_max = smi("name", "power.limit", "clocks.max.sm")
    sm = [float(s) for s in samples if s.replace(".", "").isdigit()]
    # the samples include the allocation and fill; the busiest samples are the timed passes
    busy = sorted(sm)[len(sm) // 2:] if sm else []
    print(json.dumps({"hbm_read_gbs": float(res["gbs"]), "bytes": int(res["bytes"]), "runs": args.runs, "median_ms": float(res["median_ms"]),
                      "min_ms": float(res["min_ms"]), "max_ms": float(res["max_ms"]), "grid": int(res["grid"]), "device": res["device"],
                      "card": name, "power_limit_w": power_limit, "sm_clock_mhz": statistics.median(busy) if busy else None, "sm_clock_max_mhz": sm_max}))


if __name__ == "__main__":
    main()
