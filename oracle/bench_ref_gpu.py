"""
TEST/MEASUREMENT INFRASTRUCTURE.  Times the UNMODIFIED reference kernels (oracle/_ref) and this repo's kernels on the
same GPU, same shapes, same method: per shape, >= 512 MB of rotated weight copies to defeat L2 (as the reference's
science/qgemm_benchmark.py:74-82), 10 warm-up + 60 timed calls, CUDA events.

    python oracle/bench_ref_gpu.py [mma|gemv|int8|ours]      (no arg: runs all four in fresh processes)
    -> $REF_BENCH_OUT/ref_bench_<mode>.json
"""
import os, sys, json, subprocess
HERE = os.path.dirname(os.path.abspath(__file__)); ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

MODES = {"mma": {"EXL3_INT8_GEMV": "0", "EXL3_GEMV": "0"}, "gemv": {"EXL3_INT8_GEMV": "0"}, "int8": {}, "ours": {}}
SHAPES = [("q/o", 4096, 4096, 4, 1), ("k/v", 4096, 1024, 4, 1), ("gate/up", 4096, 14336, 4, 1), ("down", 14336, 4096, 4, 1),
          ("lm_head", 4096, 128256, 6, 1), ("q/o m=8", 4096, 4096, 4, 8), ("gate/up m=32", 4096, 14336, 4, 32),
          ("q/o K=2", 4096, 4096, 2, 1), ("q/o K=3", 4096, 4096, 3, 1), ("q/o K=6", 4096, 4096, 6, 1),
          ("gate/up m=128", 4096, 14336, 4, 128)]
# the other two codebooks (same bytes, different decode): the 3INST default of older conversions and the MCG variant, batch 1
CB_SHAPES = [("q/o 3inst", 4096, 4096, 4, 1, "3inst"), ("gate/up 3inst", 4096, 14336, 4, 1, "3inst"), ("q/o mcg", 4096, 4096, 4, 1, "mcg")]


def main(mode):
    import torch
    global SHAPES
    if os.environ.get("REF_BENCH_SHAPES") == "decode":       # bench.py's same-run leg: the Llama decode shapes only
        SHAPES = SHAPES[:7] + CB_SHAPES
    else:
        SHAPES = SHAPES + CB_SHAPES
    dev = torch.device("cuda:0")
    if mode == "ours":
        from exllamav3_b200 import ext as e
        gemm_cb = lambda A, B, C, su, Ah, sv, mcg, mul1: e.exl3_gemm(A, B, C, su, Ah, sv, -1, mcg, mul1, 0)
    else:
        sys.path.insert(0, os.path.join(HERE, "_ref"))
        import exl3_ref_ext as r
        gemm_cb = lambda A, B, C, su, Ah, sv, mcg, mul1: r.exl3_gemm(A, B, C, su, Ah, sv, -1, mcg, mul1, 0)
    res = []
    g = torch.Generator(device=dev); g.manual_seed(0)
    for shp in SHAPES:
        (name, k, n, K, m), cbn = shp[:5], (shp[5] if len(shp) > 5 else "mul1")
        gemm = lambda A, B, C, su, Ah, sv, mcg=(cbn == "mcg"), mul1=(cbn == "mul1"): gemm_cb(A, B, C, su, Ah, sv, mcg, mul1)
        nbytes = k * n * K // 8
        copies = max(2, min(64, (512 << 20) // nbytes + 1))
        Bs = [torch.randint(0, 65536, (k // 16, n // 16, 16 * K), generator=g, device=dev, dtype=torch.int32).to(torch.int16)
              for _ in range(copies)]
        su = (torch.randn(k, generator=g, device=dev) / k ** 0.5).half(); sv = torch.randn(n, generator=g, device=dev).half()
        A = torch.randn((m, k), generator=g, device=dev).half(); Ah = torch.empty_like(A)
        C = torch.empty((m, n), dtype=torch.half, device=dev)
        tag = None
        for i in range(10):
            tag = gemm(A, Bs[i % copies], C, su, Ah, sv)
        torch.cuda.synchronize()
        iters = 60
        # kernels only: replay a CUDA graph of the 60 calls (the reference's own decode path replays graphs,
        # libtorch/mlp.cpp:93-147); eager launches measure host launch overhead instead
        graph, mode_used = None, "eager"
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=st):
                    for i in range(iters):
                        gemm(A, Bs[i % copies], C, su, Ah, sv)
            mode_used = "graph"
        except Exception as ex:
            print("graph capture failed:", type(ex).__name__, str(ex)[:200], flush=True)
            graph = None
            torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if graph is not None:
            graph.replay(); torch.cuda.synchronize()
            e0.record(); graph.replay(); e1.record(); e1.synchronize()
        else:
            e0.record()
            for i in range(iters):
                gemm(A, Bs[i % copies], C, su, Ah, sv)
            e1.record(); e1.synchronize()
        us = e0.elapsed_time(e1) * 1000 / iters
        alg = nbytes + 2 * m * k + 2 * m * n + 2 * (k + n)
        res.append(dict(timing=mode_used, shape=name, k=k, n=n, K=K, m=m, codebook=cbn, us=us, gbps=alg / us / 1e3, tag=int(tag) if tag is not None else None))
        print(mode, res[-1], flush=True)
        del Bs
        torch.cuda.empty_cache()
    out_dir = os.environ.get("REF_BENCH_OUT") or os.path.join(ROOT, "ref_bench_out")
    os.makedirs(out_dir, exist_ok=True)
    json.dump(res, open(os.path.join(out_dir, f"ref_bench_{mode}.json"), "w"), indent=1)


if __name__ == "__main__":
    if len(sys.argv) > 1:
        main(sys.argv[1])
    else:
        for mode, env in MODES.items():
            e = dict(os.environ); e.update(env); e.setdefault("EXLLAMAV3_TUNE_CACHE", "/tmp/exl3_ref_tune")
            r = subprocess.run([sys.executable, os.path.abspath(__file__), mode], env=e)
            print("mode", mode, "rc", r.returncode, flush=True)
