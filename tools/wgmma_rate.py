#!/usr/bin/env python
"""
Issue rate of wgmma.m64nNk32.s32.u8.s8 (A from registers, B from shared memory), the MMA of the int8 decode-GEMM.

    python tools/wgmma_rate.py [--iters 20000] [--out FILE]

Compiles tools/wgmma_rate.cu with nvcc into a temporary directory, runs it on GPU 0 and prints one JSON line per
configuration (N = 8 / 16, one / four warpgroups per SM, 8 MMAs per commit group into one accumulator or 8 independent
ones, wait_group 0 or 1 after each group) with the SM clocks per wgmma per SM over all SMs, then one summary line with the
card's name and power limit.
"""
from __future__ import annotations
import argparse, json, os, shutil, subprocess, sys, tempfile

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20000, help="batches of 8 wgmma per warpgroup")
    ap.add_argument("--out", default=None, help="also write the results (JSON) here")
    args = ap.parse_args()
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    rows = []
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "wgmma_rate")
        subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        os.path.join(HERE, "wgmma_rate.cu"), "-o", exe], check=True)
        p = subprocess.run([exe, str(args.iters)], capture_output=True, text=True)
        if p.returncode != 0:
            sys.exit(f"wgmma_rate failed (exit {p.returncode}):\n{p.stdout}\n{p.stderr}")
        for ln in p.stdout.splitlines():
            if ln.startswith("{"):
                rows.append(json.loads(ln))
                print(ln, flush=True)
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    summary = {"gpu": gpu, "results": rows}
    print(json.dumps({"gpu": gpu}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
