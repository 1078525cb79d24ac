#!/usr/bin/env python
"""
Phase split of the int8 decode-GEMM (tag 210) launches of the flagship token, from the in-kernel timeline stamps of the
bring-up build:

    EXL3B_LIB_SUFFIX=_dbg EXL3B_TC_DEBUG=1 python -m exllamav3_b200.build
    python tools/i8_phase_profile.py --library exllamav3_b200/libexl3b200_dbg.so [--reps 20] [--out FILE]

Runs the launches of one Llama-3.1-8B layer as bench.py issues them (q+k+v fan-out, o, gate+up exl3_mgemm, down) and the
lm_head, each `reps` times after a warm-up, with the timeline buffer set (exl3b_debug_tc_timeline).  Per CTA it splits a
launch into
    ramp    kernel start -> the first decode warp has its first unit's weights   (stamps 0 -> 3)
    steady  decode and MMA of the CTA's units, up to the last unit's MMAs        (stamps 3 -> 10)
    tail    epilogue and split-K exchange                                         (stamps 10 -> 8)
and prints one JSON line per launch with the median and the max over CTAs (pooled over the repetitions), in microseconds
(%globaltimer), plus the steady time per unit: the median steady time over the mean units per CTA.
"""
from __future__ import annotations
import argparse, ctypes, json, os, statistics, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLOTS = 64                                       # u64 stamps per CTA (gemm_tc_i8_body.cuh: p.dbg[blockIdx.x * 64 + slot])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--library", required=True, help="bring-up build of libexl3b200 (EXL3B_TC_DEBUG)")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the results (JSON) here")
    args = ap.parse_args()
    os.environ["EXL3B_LIBRARY"] = os.path.abspath(args.library)
    sys.path.insert(0, ROOT)
    import torch
    import bench
    from exllamav3_b200 import ext

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = dict(bench.MODELS["llama-3.1-8b"], layers=1)
    tok = bench.Token(cfg, 1, 0, dev)
    num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
    buf = torch.zeros((4 * num_sms, SLOTS), dtype=torch.int64, device=dev)
    results = []
    for ln in tok.launches:
        mats = ln["mats"]
        name = "+".join(m["name"] for m in mats)
        units = sum((m["k"] // 128) * (m["n"] // 128) for m in mats)
        for _ in range(3):
            tok.run([ln])
        torch.cuda.synchronize()
        ramp, steady, tail, total, ctas = [], [], [], [], []
        ext.lib.exl3b_debug_tc_timeline(ctypes.c_void_p(buf.data_ptr()))
        try:
            for _ in range(args.reps):
                buf.zero_()
                tok.run([ln])
                torch.cuda.synchronize()
                st = buf.cpu()
                rows = [r for r in st.tolist() if r[0] and r[3] and r[10] and r[8]]
                ctas.append(len(rows))
                for r in rows:
                    ramp.append((r[3] - r[0]) / 1e3)
                    steady.append((r[10] - r[3]) / 1e3)
                    tail.append((r[8] - r[10]) / 1e3)
                    total.append((r[8] - r[0]) / 1e3)
        finally:
            ext.lib.exl3b_debug_tc_timeline(ctypes.c_void_p(0))
        torch.cuda.synchronize()
        assert ramp, f"{name}: no timeline stamps (is {args.library} the EXL3B_TC_DEBUG build?)"
        n_cta = statistics.median(ctas)
        q = lambda v: {"median": round(statistics.median(v), 2), "max": round(max(v), 2)}
        res = {"launch": name, "k": mats[0]["k"], "n": [m["n"] for m in mats], "K": mats[0]["K"], "units": units,
               "ctas": n_cta, "ramp_us": q(ramp), "steady_us": q(steady), "tail_us": q(tail), "cta_total_us": q(total),
               "steady_us_per_unit": round(statistics.median(steady) / (units / n_cta), 3)}
        results.append(res)
        print(json.dumps(res), flush=True)
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "library": os.path.basename(args.library)}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "library": os.path.basename(args.library), "launches": results}, f, indent=1)


if __name__ == "__main__":
    main()
