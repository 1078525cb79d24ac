#!/usr/bin/env python
"""
Times Llama-3.1-8B's MLP decode block (hidden 4096, intermediate 2 x 14336, K = 4, mul1 codebook, synthetic weights) at 1, 2, 4
and 8 tokens, two ways on this library:
  * fused    BC_GatedMLP.run_bszN: exl3_mgemm(gate, up), then exl3_gemm_gated(down) with SiLU in its input stage -- 2 launches
             at <= 4 tokens (the int8 path); at 5..8 tokens gate / up and down run on the exact path (tag 200), 6 launches
  * ref-seq  the reference's sequence (exllamav3_ext/libtorch/mlp.cpp:14-91): exl3_mgemm, silu_mul, exl3_gemm -- 3 launches at
             <= 4 tokens, 7 at 5..8
Each side is captured in a CUDA graph of `--calls` block calls and replayed; CUDA events time `--reps` replays, the median per
call is reported.  Both sides run alternately in one process and their outputs are checked to be bit-identical.

    python tools/mlp_bench.py [--tokens 1,2,4,8] [--calls 20] [--reps 25] [--out DIR]

Prints one JSON line: device name, power limit, launches and median microseconds per block call of each side, and their ratio.
"""
from __future__ import annotations
import argparse, json, os, statistics, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HIDDEN, INTER, K = 4096, 14336, 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", default="1,2,4,8")
    ap.add_argument("--calls", type=int, default=20, help="block calls per graph replay")
    ap.add_argument("--reps", type=int, default=25, help="timed replays per side")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from exllamav3_b200 import ext
    assert torch.cuda.is_available(), "mlp_bench needs a CUDA device"
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    g = torch.Generator(device=dev); g.manual_seed(0)

    def mat(k, n):
        tr = torch.randint(-32768, 32767, (k // 16, n // 16, 16 * K), dtype=torch.int16, device=dev, generator=g)
        suh = ((torch.rand(k, device=dev, generator=g) + 0.5) * torch.sign(torch.randn(k, device=dev, generator=g)) / k ** 0.5).half()
        svh = ((torch.rand(n, device=dev, generator=g) + 0.5) * torch.sign(torch.randn(n, device=dev, generator=g))).half()
        return tr, suh, svh

    gate, up, down = mat(HIDDEN, INTER), mat(HIDDEN, INTER), mat(INTER, HIDDEN)
    tabs = [torch.tensor([gate[i].data_ptr(), up[i].data_ptr()], dtype=torch.long, device=dev) for i in range(3)]
    dn = ext.BC_LinearEXL3(down[0], down[1], down[2], K, None, False, True, None)
    guh = torch.empty((2, 8, HIDDEN), dtype=torch.half, device=dev)
    gu = torch.empty((2, 8, INTER), dtype=torch.half, device=dev)
    a8 = torch.empty((1, 8, INTER), dtype=torch.half, device=dev)
    bc = ext.BC_GatedMLP(guh, gu, a8, torch.empty_like(a8), *tabs, K, False, True, True, False, False, None, None, dn, 0.0)

    res = {"device": gpu, "model": "Llama-3.1-8B MLP", "hidden": HIDDEN, "intermediate": INTER, "K": K, "codebook": "mul1",
           "calls_per_replay": a.calls, "reps": a.reps, "tokens": {}}
    for n in [int(t) for t in a.tokens.split(",")]:
        x = torch.randn((1, n, HIDDEN), device=dev, generator=g).half()
        d_f = torch.empty((1, n, HIDDEN), dtype=torch.half, device=dev)
        d_r = torch.empty_like(d_f)
        gu_r = torch.empty((2, n, INTER), dtype=torch.half, device=dev)
        guh_r = torch.empty((2, n, HIDDEN), dtype=torch.half, device=dev)
        a_r = torch.empty((1, n, INTER), dtype=torch.half, device=dev)
        ah_r = torch.empty_like(a_r)

        def fused():
            bc.run_bszN(x, d_f)

        def refseq():
            ext.exl3_mgemm(x, tabs[0], gu_r, tabs[1], guh_r, tabs[2], None, None, K, -1, False, True, -1, -1, 0)
            ext.silu_mul(gu_r[0].unsqueeze(0), gu_r[1].unsqueeze(0), a_r, 0.0)
            ext.exl3_gemm(a_r, down[0], d_r, down[1], ah_r, down[2], -1, False, True, 0)

        sides = {"fused": fused, "ref_seq": refseq}
        graphs, launches = {}, {}
        for name, fn in sides.items():
            fn(); torch.cuda.synchronize()                       # buffers, host tables, kernel attributes outside capture
            l0 = ext.launch_count(); fn(); launches[name] = ext.launch_count() - l0
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                for _ in range(a.calls):
                    fn()
            graphs[name] = gr
        torch.cuda.synchronize()
        assert torch.equal(d_f.view(torch.int16), d_r.view(torch.int16)), f"outputs differ at {n} tokens"
        times = {k: [] for k in sides}
        for name in sides:
            graphs[name].replay()                                # warm-up replay
        torch.cuda.synchronize()
        for _ in range(a.reps):
            for name in sides:                                   # alternate the sides
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); graphs[name].replay(); e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1) * 1000.0 / a.calls)
        med = {k: statistics.median(v) for k, v in times.items()}
        res["tokens"][str(n)] = {"fused_us": round(med["fused"], 2), "ref_seq_us": round(med["ref_seq"], 2),
                                 "fused_launches": launches["fused"], "ref_seq_launches": launches["ref_seq"],
                                 "speedup": round(med["ref_seq"] / med["fused"], 3),
                                 "spread_us": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()}}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "mlp_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
