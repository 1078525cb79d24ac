#!/usr/bin/env python
"""
A/B of two builds of libexl3b200.so on the flagship workload: runs bench.py alternately against a baseline and a candidate
library (selected with EXL3B_LIBRARY), several times each in one process tree, and compares what both builds computed.

    python tools/ab_bench.py --baseline exllamav3_b200/libexl3b200_base.so [--candidate exllamav3_b200/libexl3b200.so]
                             [--mode ops|blocks|layer|token] [--runs 3] [--steps 400] [--warmup 50] [--out DIR]

The baseline library is built from the old sources into its own directory and copied next to the candidate, e.g.
    git worktree add /tmp/base <commit>; (cd /tmp/base && EXL3B_LIB_SUFFIX=_base python -m exllamav3_b200.build)
    cp /tmp/base/exllamav3_b200/libexl3b200_base.so exllamav3_b200/
(a build product like the candidate, so git ignores it).  Every run writes its outputs with --dump-outputs; the script requires
them to be bit-identical across all runs of both builds (the int8 path accumulates integers, so a reordering of the MMAs changes
no bit).  It prints one
JSON line: per build the tok/s of every run, the per-launch qgemm times of gate, down and lm_head, of the batch-8 / 32 decode
and of the other two codebooks, and the reference's own kernels timed in the same bench runs.
"""
from __future__ import annotations
import argparse, glob, json, os, statistics, subprocess, sys, tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(lib, mode, steps, warmup, dump_dir):
    env = dict(os.environ, EXL3B_LIBRARY=os.path.abspath(lib))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--mode", mode, "--dump-outputs", dump_dir]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    if p.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py failed with {lib} (exit {p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")
    return json.loads(lines[-1])


def summary(res):
    qg = res.get("qgemm") or {}
    q = qg.get("decode_hbm", {})
    ref = (qg.get("reference_cuda") or {}).get("shapes", {})
    times = lambda d: {k: {"us": v["us_per_launch"], "GBps": v["GBps"]} for k, v in d.items()}
    # decode_batch (m = 8 / 32) and decode_codebooks (3inst / mcg at m = 1) are where bench.py times the fp16 path (tag 200)
    return {"value": res["value"],
            "decode_hbm": {k: v for k, v in times(q).items() if k in ("gate", "down", "lm_head")},
            "decode_batch": times(qg.get("decode_batch", {})), "decode_codebooks": times(qg.get("decode_codebooks", {})),
            "reference_cuda": ref}


def outputs_equal(a_dir, b_dir):
    names = sorted(os.path.basename(f) for f in glob.glob(os.path.join(a_dir, "*.npy")))
    assert names, f"no outputs in {a_dir}"
    assert names == sorted(os.path.basename(f) for f in glob.glob(os.path.join(b_dir, "*.npy"))), "different output sets"
    diff = []
    for n in names:
        x, y = np.load(os.path.join(a_dir, n)), np.load(os.path.join(b_dir, n))
        if x.dtype != y.dtype or x.shape != y.shape or x.tobytes() != y.tobytes():
            diff.append(n)
    return len(names), diff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", required=True)
    ap.add_argument("--candidate", default=os.path.join(ROOT, "exllamav3_b200", "libexl3b200.so"))
    ap.add_argument("--mode", default="ops", help="bench.py --mode (blocks / layer / token run the chain kernel)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    args = ap.parse_args()
    builds = {"baseline": args.baseline, "candidate": args.candidate}
    for name, lib in builds.items():
        assert os.path.exists(lib), f"{name} library {lib} not found"
    runs = {name: [] for name in builds}
    with tempfile.TemporaryDirectory() as td:
        dumps = []
        for i in range(args.runs):
            order = list(builds) if i % 2 == 0 else list(reversed(builds))     # alternate which build goes first
            for name in order:
                d = os.path.join(td, f"{name}_{i}")
                runs[name].append(summary(run_bench(builds[name], args.mode, args.steps, args.warmup, d)))
                dumps.append(d)
                print(f"run {i} {name}: {runs[name][-1]['value']:.1f} tok/s", file=sys.stderr, flush=True)
        n_out, diffs = 0, {}
        for d in dumps[1:]:
            n_out, diff = outputs_equal(dumps[0], d)
            if diff:
                diffs[os.path.basename(d)] = diff
    vals = {name: [r["value"] for r in rs] for name, rs in runs.items()}
    med = {name: statistics.median(v) for name, v in vals.items()}
    line = {"mode": args.mode, "runs": runs,
            "tok_s": {name: {"median": round(med[name], 1), "min": round(min(v), 1), "max": round(max(v), 1)} for name, v in vals.items()},
            "speedup_median": round(med["candidate"] / med["baseline"], 3),
            "outputs_compared": n_out, "outputs_bit_identical": not diffs, "differing_outputs": diffs}
    try:
        line["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                     capture_output=True, text=True).stdout.strip()
    except OSError:
        pass
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)
    sys.exit(0 if not diffs else 1)


if __name__ == "__main__":
    main()
