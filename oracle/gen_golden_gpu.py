"""
TEST INFRASTRUCTURE (oracle).  Runs the UNMODIFIED reference CUDA kernels (oracle/_ref/exl3_ref_ext.so, built by
oracle/build_ref.py from $EXLLAMAV3_SOURCE) on a GPU and records their outputs on seeded inputs as golden vectors.

    python oracle/gen_golden_gpu.py            # driver: runs the three modes below in fresh processes
    -> $GOLDEN_OUT/ref_gpu_mma.npz    EXL3_INT8_GEMV=0 EXL3_GEMV=0   (tensor-core mma.sync kernel only)   == GOLDEN
       $GOLDEN_OUT/ref_gpu_gemv.npz   EXL3_INT8_GEMV=0               (fp16-accumulate GEMV heuristics on)
       $GOLDEN_OUT/ref_gpu_int8.npz   defaults                       (int8-activation GEMV for mul1, ~0.9% RMS by design)

tests/golden/ref_gpu.npz is a copy of ref_gpu_mma.npz (committed).  Inputs are NOT stored: they are regenerated
from oracle.exl3_oracle.make_synthetic / case_inputs with the same seeds at test time (a checksum of every input is
stored to prove identity).
"""
import os, sys, subprocess, zlib
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import exl3_oracle as orc   # noqa: E402

MODES = {
    "mma": {"EXL3_INT8_GEMV": "0", "EXL3_GEMV": "0"},
    "gemv": {"EXL3_INT8_GEMV": "0"},
    "int8": {},
}


def crc(*arrs):
    c = 0
    for a in arrs:
        c = zlib.crc32(np.ascontiguousarray(a).tobytes(), c)
    return np.uint32(c)


# ---- case tables (shared with tests/test_golden_gpu.py) -------------------------------------------------------

def reconstruct_cases():
    return [(K, cb, 32, 128) for cb in range(3) for K in range(1, 9)] + [(4, 2, 128, 384), (3, 0, 64, 256)]


def gemm_cases():
    cases = [(1, 256, 256, K, 2, False) for K in range(1, 9)]
    for cb in range(3):
        for m in (1, 4, 16, 17, 33):
            for fp32 in (False, True):
                cases.append((m, 256, 256, 4, cb, fp32))
    cases += [(2, 512, 128, 3, 0, False), (8, 128, 512, 6, 1, True), (1, 1024, 384, 2, 2, True)]
    return cases


def had_cases():
    return [(dt, mode, scale) for dt in ("f16", "f32") for mode in ("none", "pre", "post") for scale in (1.0, 0.5)]


def had_inputs(dt):
    rng = np.random.default_rng(99)
    x = rng.standard_normal((3, 256)).astype(np.float16 if dt == "f16" else np.float32)
    sc = (np.sign(rng.standard_normal(256)) * rng.uniform(0.5, 2.0, 256)).astype(np.float16)
    return x, sc


def mgemm_inputs():
    k, n, K, m = 256, 128, 4, 3
    mats = [orc.make_synthetic(k, n, K, seed=1000 + e, m=m) for e in range(4)]
    rng = np.random.default_rng(5)
    A = rng.standard_normal((4, m, k)).astype(np.float16)
    w = rng.uniform(0.1, 1.0, 4).astype(np.float16)
    return k, n, K, m, mats, A, w


def main_mode(mode):
    import torch
    sys.path.insert(0, os.path.join(HERE, "_ref"))
    import exl3_ref_ext as ref
    dev = "cuda:0"
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = {}

    for (K, cb, k, n) in reconstruct_cases():
        tr, suh, svh, _ = orc.make_synthetic(k, n, K)
        w = torch.empty((k, n), dtype=torch.half, device=dev)
        ref.reconstruct(w, T(tr), K, cb == 1, cb == 2)
        out[f"rec_{K}_{cb}_{k}_{n}"] = w.cpu().numpy()
        out[f"rec_{K}_{cb}_{k}_{n}_crc"] = crc(tr)
    # slice + fused
    for (K, cb, k, n, off, nout) in [(4, 2, 128, 384, 128, 256), (3, 0, 128, 256, 0, 256)]:
        tr, suh, svh, _ = orc.make_synthetic(k, n, K)
        w = torch.empty((k, nout), dtype=torch.half, device=dev)
        ref.reconstruct_slice(w, T(tr), K, cb == 1, cb == 2, off)
        out[f"recslice_{K}_{cb}_{k}_{n}_{off}_{nout}"] = w.cpu().numpy()
        w2 = torch.empty((k, nout), dtype=torch.half, device=dev)
        ref.reconstruct_had_slice(w2, T(tr), T(suh), T(svh[off:]), K, cb == 1, cb == 2, off)
        out[f"rechad_{K}_{cb}_{k}_{n}_{off}_{nout}"] = w2.cpu().numpy()

    for (dt, hmode, scale) in had_cases():
        x, sc = had_inputs(dt)
        xi = T(x); yo = torch.empty_like(xi)
        ref.had_r_128(xi, yo, T(sc) if hmode == "pre" else None, T(sc) if hmode == "post" else None, scale)
        out[f"had_{dt}_{hmode}_{scale}"] = yo.cpu().numpy()

    for (m, k, n, K, cb, fp32) in gemm_cases():
        tr, suh, svh, x = orc.make_synthetic(k, n, K, m=m)
        A = T(x); C = torch.empty((m, n), dtype=torch.float if fp32 else torch.half, device=dev)
        A_had = torch.empty_like(A)
        tag = ref.exl3_gemm(A, T(tr), C, T(suh), A_had, T(svh), -1, cb == 1, cb == 2, 0)
        torch.cuda.synchronize()
        key = f"gemm_{m}_{k}_{n}_{K}_{cb}_{int(fp32)}"
        out[key] = C.cpu().numpy()
        out[key + "_xh"] = A_had.cpu().numpy()
        out[key + "_tag"] = np.int32(tag)
        out[key + "_crc"] = crc(tr, suh, svh, x)

    # mgemm: (a) one input, 4 outputs; (b) indices incl. a skipped slot; (c) weighted reduction; (d) range filter
    k, n, K, m, mats, A, wts = mgemm_inputs()
    trs = [T(t[0]) for t in mats]; suhs = [T(t[1]) for t in mats]; svhs = [T(t[2]) for t in mats]
    P = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.long, device=dev)
    pB, pU, pV = P(trs), P(suhs), P(svhs)
    mul = 0x83DCD12D
    for fp32 in (False, True):
        dt = torch.float if fp32 else torch.half
        C = torch.zeros((4, m, n), dtype=dt, device=dev); Ah = torch.empty((4, m, k), dtype=torch.half, device=dev)
        ref.exl3_mgemm(T(A[:1]), pB, C, pU, Ah, pV, None, None, K, -1, 0, mul, -1, -1, 0)
        out[f"mgemm_a_{int(fp32)}"] = C.cpu().numpy()
        C = torch.zeros((4, m, n), dtype=dt, device=dev)
        idx = torch.tensor([[2, -1, 0, 3]], dtype=torch.long, device=dev)
        ref.exl3_mgemm(T(A), pB, C, pU, Ah, pV, idx, None, K, -1, 0, mul, -1, -1, 0)
        out[f"mgemm_b_{int(fp32)}"] = C.cpu().numpy()
        C = torch.zeros((4, m, n), dtype=dt, device=dev)
        idx = torch.tensor([[3, 1, 0, 2]], dtype=torch.long, device=dev)
        ref.exl3_mgemm(T(A[:1]), pB, C, pU, Ah, pV, idx, T(wts).view(1, 4), K, -1, 0, mul, -1, -1, 0)
        out[f"mgemm_c_{int(fp32)}"] = C[0].cpu().numpy()
        C = torch.zeros((4, m, n), dtype=dt, device=dev)
        ref.exl3_mgemm(T(A[:1]), pB[1:3].contiguous(), C, pU[1:3].contiguous(), Ah, pV[1:3].contiguous(),
                       idx, T(wts).view(1, 4), K, -1, 0, mul, 1, 3, 0)
        out[f"mgemm_d_{int(fp32)}"] = C[0].cpu().numpy()
    torch.cuda.synchronize()

    out_dir = os.environ.get("GOLDEN_OUT") or os.path.join(ROOT, "golden_out")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, f"ref_gpu_{mode}.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    if len(sys.argv) > 1:
        main_mode(sys.argv[1])
    else:
        for mode, env in MODES.items():
            e = dict(os.environ); e.update(env)
            e.setdefault("EXLLAMAV3_TUNE_CACHE", "/tmp/exl3_ref_tune")
            r = subprocess.run([sys.executable, os.path.abspath(__file__), mode], env=e)
            print("mode", mode, "rc", r.returncode, flush=True)
