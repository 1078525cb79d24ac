#!/usr/bin/env python
"""
Times the library's RMSNorm (exllamav3_b200.ext.rms_norm / rms_norm_res_in) against the reference's own kernel
(oracle/_ref/exl3_ref_norm.so, built by oracle/build_ref_norm.py) in one process, alternating the two, and checks both outputs
against the fp64 model within the bars of tests/test_norm_gpu.py.

    python tools/norm_bench.py [--iters 200] [--out norm_bench.json]

Shapes: fp16 x / w / y decode rows 1, 8 and 32 at dim 4096 and 8192 (as isolated calls, and as a CUDA graph of 64 calls, the norms
of one token through a 32-layer model); prefill rows 4096 and 32768 at dim 4096; head norms (32 tokens x 8 heads at dim 128);
the fused residual form (RES_IN, fp32 residual) at decode.  Isolated calls: CUDA events around each call, median of --iters calls
after a warm-up.  Graphs: events around one replay, median over --iters / 4 replays, divided by 64.  GB/s counts the algorithmic
bytes (x, w, y, and r twice in RES_IN) over the median time, against the H100 SXM's 3.35 TB/s.  Prints one JSON line with the
card's name, power limit and max SM clock read in the same run.
"""
from __future__ import annotations
import argparse, json, os, statistics, subprocess, sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
from oracle import norm_oracle as no  # noqa: E402

HBM_PEAK = 3.35e12


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return dict(zip(q.split(","), (s.strip() for s in out.splitlines()[0].split(","))))


def time_calls(fn, iters):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return statistics.median(a.elapsed_time(b) for a, b in ev) * 1e3


def graph_of(fn, n):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(n):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    return g


def bar_ratio(y, v):
    """largest error in units of the bar: fp16 ulps of fp16(model), or multiples of 4e-6 |v| for fp32"""
    y, v = y.cpu(), v.cpu().double()
    if y.dtype == torch.half:
        return ((y.double() - v.half().double()).abs() / no.ulp16(v)).max().item()
    return ((y.double() - v).abs() / (4e-6 * v.abs()).clamp(min=1e-300)).max().item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "norm_bench.py needs a GPU"
    from exllamav3_b200 import ext
    import exl3_ref_norm as ref
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    res = {"card": card(), "iters": a.iters, "shapes": {}}

    def case(name, rows, dim, mode="none", graph=False):
        x = torch.randn(rows, dim, device=dev, generator=gen).half()
        w = (torch.randn(dim, device=dev, generator=gen) * 0.1 + 1).half()
        y = torch.empty_like(x)
        r = torch.randn(rows, dim, device=dev, generator=gen) if mode == "in" else None
        nbytes = x.numel() * 2 + w.numel() * 2 + y.numel() * 2 + (2 * r.numel() * 4 if r is not None else 0)
        out = {"rows": rows, "dim": dim, "mode": mode, "bytes": nbytes}
        for lib_name, lib in (("ours", ext), ("reference", ref)):
            if mode == "in":
                r0 = r.clone()
                fn = lambda lib=lib: lib.rms_norm_res_in(x, w, y, r, 1e-6, 0.0, 1.0)
                rc = r0.clone()
                lib.rms_norm_res_in(x, w, y, rc, 1e-6, 0.0, 1.0)
                torch.cuda.synchronize()
                assert torch.equal(rc.cpu(), no.res_in_sum(x.cpu(), r0.cpu())), f"{name} {lib_name}: residual"
                out[f"{lib_name}_bar"] = bar_ratio(y, no.rms_norm_f64(rc.cpu(), w.cpu(), 1e-6))
            else:
                fn = lambda lib=lib: lib.rms_norm(x, w, y, 1e-6, 0.0, 1.0, False, False)
                fn()
                torch.cuda.synchronize()
                sel = slice(None) if rows <= 512 else slice(0, rows, max(1, rows // 256))
                out[f"{lib_name}_bar"] = bar_ratio(y[sel], no.rms_norm_f64(x[sel].cpu(), w.cpu(), 1e-6))
            out[f"_{lib_name}_fn"] = fn
        for _ in range(20):
            out["_ours_fn"](); out["_reference_fn"]()
        torch.cuda.synchronize()
        ts = {"ours": [], "reference": []}
        if graph:
            gs = {k: graph_of(out[f"_{k}_fn"], 64) for k in ts}
            for _ in range(max(4, a.iters // 4)):
                for k in ts:
                    ts[k].append(time_calls(gs[k].replay, 1) / 64)
        else:
            for _ in range(max(1, a.iters // 50)):
                for k in ts:
                    ts[k].append(time_calls(out[f"_{k}_fn"], 50))
        for k in ts:
            us = statistics.median(ts[k])
            out[f"{k}_us"] = round(us, 3)
            out[f"{k}_GBps"] = round(nbytes / us / 1e3, 1)
            out[f"{k}_peak_frac"] = round(nbytes / us / 1e-6 / HBM_PEAK, 3)
        out["speedup"] = round(out["reference_us"] / out["ours_us"], 3)
        for k in ("_ours_fn", "_reference_fn"):
            del out[k]
        res["shapes"][name] = out
        print(name, {k: v for k, v in out.items() if k.endswith(("_us", "_bar")) or k == "speedup"}, flush=True)

    for dim in (4096, 8192):
        for rows in (1, 8, 32):
            case(f"decode_{rows}x{dim}", rows, dim)
            case(f"decode_{rows}x{dim}_graph64", rows, dim, graph=True)
        case(f"res_in_1x{dim}", 1, dim, mode="in")
    case("prefill_4096x4096", 4096, 4096)
    case("prefill_32768x4096", 32768, 4096)
    case("head_norm_256x128", 32 * 8, 128)
    case("head_norm_256x128_graph64", 32 * 8, 128, graph=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
