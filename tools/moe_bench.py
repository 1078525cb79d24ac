#!/usr/bin/env python
"""
Times exl3_moe (the fused routed-expert MLP, tag 230) against the composition of verified operators it replaces: per expert
exl3_gemm for gate and up (exact tensor-core path), the activation in torch, exl3_gemm for down, a weighted index_add.
Shapes: Qwen3-30B-A3B (hidden 2048, intermediate 768, 128 experts, top-8) and Mixtral-8x7B (4096, 14336, 8 experts, top-2)
at bsz 8, 64 and 512, mul1 codebook, K = 4, every expert under the temp-row limit (T = bsz: every expert is processed).
Synthetic weights (random trellis bits are valid tensors); routing is uniform random top-k.

    python tools/moe_bench.py [--iters 50] [--warmup 5] [--out DIR]

Both sides are timed with CUDA events over `iters` calls after `warmup` calls.  The composition reads the routing on the
host once, outside the timed region (its per-expert loop needs the counts there), so its time is its GPU work plus its launch
overhead.  Prints one JSON line: device name, power limit, and per shape the median ms of each side and their ratio.
"""
from __future__ import annotations
import argparse, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"qwen3-30b-a3b": (2048, 768, 128, 8), "mixtral-8x7b": (4096, 14336, 8, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bsz", default="8,64,512")
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from exllamav3_b200 import ext
    assert torch.cuda.is_available(), "moe_bench needs a CUDA device"
    dev = torch.device("cuda:0")
    K, cb_mul1 = 4, True
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    res = {"device": torch.cuda.get_device_name(0), "power_limit_max_sm_clock": power, "K": K, "codebook": "mul1",
           "iters": a.iters, "shapes": {}}
    g = torch.Generator(device=dev); g.manual_seed(0)
    for name in a.shapes.split(","):
        hidden, inter, E, topk = SHAPES[name]
        mats = {}
        for proj, (k, n) in (("gate", (hidden, inter)), ("up", (hidden, inter)), ("down", (inter, hidden))):
            tr = [torch.randint(-32768, 32767, (k // 16, n // 16, 16 * K), dtype=torch.int16, device=dev, generator=g) for _ in range(E)]
            suh = [((torch.rand(k, device=dev, generator=g) + 0.5) * torch.sign(torch.randn(k, device=dev, generator=g)) / k ** 0.5).half() for _ in range(E)]
            svh = [((torch.rand(n, device=dev, generator=g) + 0.5) * torch.sign(torch.randn(n, device=dev, generator=g))).half() for _ in range(E)]
            mats[proj] = (tr, suh, svh, [torch.tensor([t.data_ptr() for t in ts], dtype=torch.long, device=dev) for ts in (tr, suh, svh)])
        for bsz in [int(b) for b in a.bsz.split(",")]:
            x = torch.randn(bsz, hidden, device=dev, generator=g).half()
            sel = torch.rand(bsz, E, device=dev, generator=g).topk(topk, dim=1).indices
            wt = torch.rand(bsz, topk, device=dev, generator=g).half()
            fe = sel.reshape(-1)
            order = torch.argsort(fe, stable=True)
            tok = torch.arange(bsz, device=dev).repeat_interleave(topk)[order].contiguous()
            wts = wt.reshape(-1)[order].contiguous()
            count = torch.cat([torch.bincount(fe, minlength=E), torch.zeros(1, dtype=torch.long, device=dev)])
            T = bsz
            conc = ext.exl3_moe_max_concurrency(0)
            tsg = torch.empty((conc, T, hidden), dtype=torch.half, device=dev)
            tig = torch.empty((conc, T, inter), dtype=torch.half, device=dev)
            out = torch.zeros(bsz, hidden, device=dev)
            G, U, D = mats["gate"][3], mats["up"][3], mats["down"][3]

            def fused():
                ext.exl3_moe(x, out, count, tok, wts, tsg, tsg, tig, tig, 0, K, K, K, *G, *U, *D,
                             False, cb_mul1, False, cb_mul1, False, cb_mul1, 0.0, -1)

            c_host = count.cpu().tolist()
            starts = [sum(c_host[:e]) for e in range(E)]
            groups = [(e, tok[starts[e]:starts[e] + c_host[e]], wts[starts[e]:starts[e] + c_host[e]].float()[:, None])
                      for e in range(E) if c_host[e] > 0]
            bufs = {e: (torch.empty(len(t), hidden, dtype=torch.half, device=dev), torch.empty(len(t), inter, dtype=torch.half, device=dev),
                        torch.empty(len(t), inter, dtype=torch.half, device=dev), torch.empty(len(t), inter, dtype=torch.half, device=dev),
                        torch.empty(len(t), hidden, device=dev)) for e, t, _ in groups}
            out2 = torch.zeros(bsz, hidden, device=dev)

            def composition():
                for e, t, w in groups:
                    xh, gg, uu, hh, yy = bufs[e]
                    xe = x.index_select(0, t)
                    ext.exl3_gemm(xe, mats["gate"][0][e], gg, mats["gate"][1][e], xh, mats["gate"][2][e], 2, False, cb_mul1, 0)
                    ext.exl3_gemm(xe, mats["up"][0][e], uu, mats["up"][1][e], xh, mats["up"][2][e], 2, False, cb_mul1, 0)
                    h = (torch.nn.functional.silu(gg.float()) * uu.float()).half()
                    ext.exl3_gemm(h, mats["down"][0][e], yy, mats["down"][1][e], hh, mats["down"][2][e], 2, False, cb_mul1, 0)
                    out2.index_add_(0, t, yy * w)

            def timeit(fn):
                for _ in range(a.warmup):
                    fn()
                torch.cuda.synchronize()
                ts = []
                for _ in range(a.iters):
                    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s0.record(); fn(); s1.record()
                    s1.synchronize()
                    ts.append(s0.elapsed_time(s1))
                ts.sort()
                return ts[len(ts) // 2]

            tf, tc = timeit(fused), timeit(composition)
            # same result within the parity bars (outputs accumulated over different numbers of calls: compare one call each)
            out.zero_(); out2.zero_(); fused(); composition(); torch.cuda.synchronize()
            err = ((out - out2).abs().max() / out2.abs().max()).item()
            res["shapes"][f"{name}/bsz{bsz}"] = {"fused_ms": round(tf, 4), "composition_ms": round(tc, 4),
                                                 "speedup": round(tc / tf, 3), "max_rel_diff": err}
            print(f"{name} bsz={bsz}: fused {tf:.3f} ms, composition {tc:.3f} ms, x{tc / tf:.2f}, diff {err:.1e}",
                  file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "moe_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
