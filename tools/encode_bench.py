#!/usr/bin/env python
"""
Times the trellis encoder, ext.quantize_tiles, against the reference's kernel (oracle/_ref, built by oracle/build_ref_encode.py) in
the same process: K = 1..8 with the mul1 codebook and K = 4 with 3inst (cb0) and mcg (cb1), at 256, 896 and 8192 tiles
(one LDLQ strip of a 4096- and a 14336-wide matrix, and a batched call).  The reference gets temp buffers sized as its
converter's get_temp_buffers does (modules/quant/exl3_lib/quantize.py:53-63).  Inputs are randn(n, 256) x 1.24371 (cb0 / cb1)
or x 1.0 (mul1).

    python tools/encode_bench.py [--runs 5] [--warmup 1] [--sizes 256,896,8192] [--out DIR]

Each configuration warms both kernels up, then alternates them `runs` times, each run timed with CUDA events, and reports
the median: tiles/s, the projected seconds for the 229,376 tiles of a 4096 x 14336 matrix, and the mean squared error per
value of both kernels' results.  Prints one JSON line per configuration and a summary line with the card and power limit.
"""
from __future__ import annotations
import argparse, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

MATRIX_TILES = 4096 * 14336 // 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sizes", default="256,896,8192")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    from exllamav3_b200 import ext
    from oracle import encode_oracle as enc
    import exl3_ref_encode as ref
    assert torch.cuda.is_available(), "encode_bench needs a CUDA device"
    dev = torch.device("cuda:0")
    power = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    configs = [(K, 2) for K in range(1, 9)] + [(4, 0), (4, 1)]
    sizes = [int(s) for s in a.sizes.split(",")]
    rows = []
    for K, cb in configs:
        B = max(256, 2 * sms) if K >= 4 else 256
        tc = torch.zeros((B, 2, 65536 >> K), dtype=torch.half, device=dev)
        te = torch.zeros((B, 256, 65536 >> K), dtype=torch.short, device=dev)
        for n in sizes:
            x = enc.encode_inputs(n, cb, 4242 + n)
            xt = torch.from_numpy(x).to(dev)
            outs = {s: (torch.empty_like(xt), torch.empty(xt.shape, dtype=torch.short, device=dev)) for s in ("ours", "ref")}
            fns = {"ours": lambda: ext.quantize_tiles(xt, *outs["ours"], tc, te, K, cb == 1, cb == 2),
                   "ref": lambda: ref.quantize_tiles(xt, *outs["ref"], tc, te, K, cb == 1, cb == 2)}
            for _ in range(a.warmup):
                for f in fns.values():
                    f()
            times = {s: [] for s in fns}
            for _ in range(a.runs):
                for s, f in fns.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(); f(); e1.record()
                    torch.cuda.synchronize()
                    times[s].append(e0.elapsed_time(e1) / 1e3)
            row = {"K": K, "cb": cb, "tiles": n}
            for s in fns:
                t = float(np.median(times[s]))
                mse = float(enc.tile_sq_error(x, outs[s][1].cpu().numpy(), cb).sum() / x.size)
                row[s] = {"median_s": t, "tiles_per_s": n / t, "projected_4096x14336_s": MATRIX_TILES * t / n, "mse": mse}
            row["speedup"] = row["ref"]["median_s"] / row["ours"]["median_s"]
            rows.append(row)
            print(json.dumps(row), flush=True)
        del tc, te
        torch.cuda.empty_cache()
    summary = {"device": power, "runs": a.runs, "configs": len(rows)}
    print(json.dumps(summary), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "encode_bench.json"), "w") as f:
            json.dump({"summary": summary, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
