"""
Full-size parity of the DEFAULT product path (automatic kernel selection, through the C ABI) on the shapes BASELINE.json names,
closing the holes the round-1 review listed: lm_head 4096 x 128256 at 6 bpw, the Llama-3.1-8B shapes at 2 / 3 / 6 bpw (config 3),
8 and 32 rows at full size, every Llama-3.1-70B shard shape at TP 2 / 4 / 8 including k = 28672 (224 k-blocks: beyond the
96-unit int32 accumulation chunk), dense multi-matrix calls at 8 / 32 rows, per-matrix output widths (size_n_list / c_ptrs), and
the dense wgmma GEMM at 8192 x 4096 x 14336.

Method at sizes the fp64 oracle cannot afford in full: random 128-column blocks of the output against the oracle restricted to
those columns (a 128-column block of an EXL3 linear is itself a complete EXL3 linear: trellis[:, 8b:8b+8], svh[128b:128b+128]),
tolerances of README.md, Parity (max-abs <= 2e-3 max|y| (+1 fp16 ulp), rel-RMS <= 1e-3).
"""
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc

pytestmark = pytest.mark.gpu


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(got, ref):
    got = np.asarray(got, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
    d = got - ref
    return np.abs(d).max() / max(np.abs(ref).max(), 1e-30), np.sqrt((d ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def synth_gpu(k, n, K, dev, seed):
    """Synthetic tensor built on the GPU (the numpy generator needs minutes at lm_head size), copied back for the oracle."""
    g = torch.Generator(device=dev); g.manual_seed(seed)
    tr = torch.randint(0, 65536, (k // 16, n // 16, 16 * K), generator=g, device=dev, dtype=torch.int32).to(torch.int16)
    sgn = lambda sz: (torch.randint(0, 2, (sz,), generator=g, device=dev) * 2 - 1).float()
    suh = (sgn(k) * (0.5 + 1.5 * torch.rand(k, generator=g, device=dev)) / k ** 0.5).half()
    svh = (sgn(n) * (0.5 + 1.5 * torch.rand(n, generator=g, device=dev))).half()
    return tr, suh, svh


def check_blocks(y, x_np, tr, suh, svh, K, cb, blocks, tol=(2e-3, 1e-3), tag=""):
    suh_np = suh.cpu().numpy()
    for blk in blocks:
        sl = slice(blk * 128, blk * 128 + 128)
        tr_b = tr[:, blk * 8: blk * 8 + 8, :].contiguous().cpu().numpy()
        ref = orc.exl3_gemm_f64(x_np, tr_b, suh_np, svh[sl].cpu().numpy(), K, cb)
        mx, rms = rel_err(y[..., sl].float().cpu().numpy().reshape(ref.shape), ref)
        ulp = 2.0 ** -10 if y.dtype == torch.half else 0.0
        assert mx <= tol[0] + ulp and rms <= tol[1], (tag, blk, mx, rms)


def run_default(ext, x, tr, suh, svh, fp32=True, mul1=True, mcg=False):
    m, n = x.shape[0], tr.shape[1] * 16
    y = torch.zeros((m, n), dtype=torch.float if fp32 else torch.half, device=x.device)
    xh = torch.empty_like(x)
    tag = ext.exl3_gemm(x, tr, y, suh, xh, svh, -1, mcg, mul1, 0)
    torch.cuda.synchronize()
    return y, tag


def test_lm_head_6bpw_full_size(cuda):
    from exllamav3_b200 import ext
    k, n, K = 4096, 128256, 6
    tr, suh, svh = synth_gpu(k, n, K, cuda, 11)
    rng = np.random.default_rng(1)
    for m, fp32 in ((1, True), (1, False), (3, True)):
        x = torch.from_numpy(rng.standard_normal((m, k)).astype(np.float16)).to(cuda)
        y, tag = run_default(ext, x, tr, suh, svh, fp32)
        assert tag in (ext.EXL3B_TAG_TC_I8, ext.EXL3B_TAG_TC_I8_CHAIN)
        blocks = list(rng.choice(n // 128, 8, replace=False)) + [0, n // 128 - 1]
        check_blocks(y, x.cpu().numpy(), tr, suh, svh, K, 2, blocks, tag=f"lm_head m={m} fp32={fp32}")
        assert torch.isfinite(y.float()).all()


@pytest.mark.parametrize("K", [2, 3, 6])
@pytest.mark.parametrize("shape", [(4096, 4096), (4096, 14336), (14336, 4096)])
def test_llama_shapes_other_bitrates(cuda, K, shape):
    """BASELINE config 3: the 2.5 bpw model is a K = 2 / K = 3 mix, 6.0 bpw is K = 6."""
    from exllamav3_b200 import ext
    k, n = shape
    tr, suh, svh = synth_gpu(k, n, K, cuda, 100 + K)
    rng = np.random.default_rng(K)
    x = torch.from_numpy(rng.standard_normal((1, k)).astype(np.float16)).to(cuda)
    y, _ = run_default(ext, x, tr, suh, svh, True)
    check_blocks(y, x.cpu().numpy(), tr, suh, svh, K, 2, rng.choice(n // 128, 3, replace=False), tag=f"{shape} K={K}")
    # the other codebooks take the exact tensor-core kernel at one row: same bar
    for (mcg, cb) in ((False, 0), (True, 1)):
        y, tag = run_default(ext, x, tr, suh, svh, True, mul1=False, mcg=mcg)
        assert tag == ext.EXL3B_TAG_TC
        check_blocks(y, x.cpu().numpy(), tr, suh, svh, K, cb, rng.choice(n // 128, 2, replace=False), tag=f"{shape} K={K} cb={cb}")


@pytest.mark.parametrize("m", [8, 32])
@pytest.mark.parametrize("shape", [(4096, 4096), (4096, 14336), (14336, 4096)])
def test_llama_shapes_batch_8_and_32(cuda, m, shape):
    """Batch 8 / 32 decode (BASELINE config 3) on the default path; the row list of the reference's own kernel test
    (tests/test_qgemm.py:31-53) is covered at test size by test_gpu_parity.py."""
    from exllamav3_b200 import ext
    k, n = shape
    K = 4
    tr, suh, svh = synth_gpu(k, n, K, cuda, 200 + m)
    rng = np.random.default_rng(m)
    x = torch.from_numpy(rng.standard_normal((m, k)).astype(np.float16)).to(cuda)
    for fp32 in (True, False):
        y, tag = run_default(ext, x, tr, suh, svh, fp32)
        assert tag != ext.EXL3B_TAG_SIMT                              # batch 8 / 32 runs on the tensor cores
        check_blocks(y, x.cpu().numpy(), tr, suh, svh, K, 2, rng.choice(n // 128, 2, replace=False), tag=f"{shape} m={m}")


# Llama-3.1-70B shards as modules/quant/exl3.py:284-330 cuts them (hidden 8192, intermediate 28672, kv 1024):
#   column-parallel: q (8192 -> 8192 / tp), k / v (8192 -> max(128, 1024 / tp)), gate / up (8192 -> 28672 / tp)
#   row-parallel:    o (8192 / tp -> 8192), down (28672 / tp -> 8192)
def _shards_70b():
    s = set()
    for tp in (1, 2, 4, 8):
        s |= {(8192, 8192 // tp), (8192, max(128, 1024 // tp)), (8192, 28672 // tp), (8192 // tp, 8192), (28672 // tp, 8192)}
    return sorted(s)


@pytest.mark.parametrize("shape", _shards_70b())
def test_llama_70b_shard_shapes(cuda, shape):
    from exllamav3_b200 import ext
    k, n = shape
    K = 4
    tr, suh, svh = synth_gpu(k, n, K, cuda, k + n)
    rng = np.random.default_rng(k * 7 + n)
    x = torch.from_numpy(rng.standard_normal((1, k)).astype(np.float16)).to(cuda)
    y, tag = run_default(ext, x, tr, suh, svh, True)
    assert tag in (ext.EXL3B_TAG_TC_I8, ext.EXL3B_TAG_TC_I8_CHAIN)
    nb = n // 128
    check_blocks(y, x.cpu().numpy(), tr, suh, svh, K, 2, rng.choice(nb, min(nb, 2), replace=False), tag=f"70b shard {shape}")
    if k >= 14336:                                                    # long rows also on the chain kernel and with 4 rows
        x4 = torch.from_numpy(rng.standard_normal((4, k)).astype(np.float16)).to(cuda)
        prev = ext.set_gemm_path(ext.EXL3B_TAG_TC_I8_CHAIN)
        try:
            y4, tag = run_default(ext, x4, tr, suh, svh, True)
            assert tag == ext.EXL3B_TAG_TC_I8_CHAIN
        finally:
            ext.set_gemm_path(prev)
        check_blocks(y4, x4.cpu().numpy(), tr, suh, svh, K, 2, rng.choice(nb, 2, replace=False), tag=f"70b shard {shape} chain m=4")


@pytest.mark.parametrize("m", [8, 32])
def test_dense_mgemm_batch_8_and_32_default_path(cuda, m):
    """The model's fused k+v / gate+up call at batch 8 / 32 (modules/attn.py:603, modules/mlp.py:726 fuse up to 32 rows)."""
    from exllamav3_b200 import ext
    K = 4
    for (k, n, mats) in ((4096, 1024, 2), (1024, 512, 3)):
        ts = [synth_gpu(k, n, K, cuda, 300 + i) for i in range(mats)]
        ptr = lambda j: torch.tensor([t[j].data_ptr() for t in ts], dtype=torch.long, device=cuda)
        rng = np.random.default_rng(m + k)
        x = torch.from_numpy(rng.standard_normal((1, m, k)).astype(np.float16)).to(cuda)
        for fp32 in (True, False):
            C = torch.zeros((mats, m, n), dtype=torch.float if fp32 else torch.half, device=cuda)
            Ah = torch.empty((mats, m, k), dtype=torch.half, device=cuda)
            tag = ext.exl3_mgemm(x, ptr(0), C, ptr(1), Ah, ptr(2), None, None, K, -1, False, True, -1, -1, 0)
            torch.cuda.synchronize()
            assert tag != ext.EXL3B_TAG_SIMT, "dense multi-matrix calls up to 32 rows must run on the tensor cores"
            for j, (tr, suh, svh) in enumerate(ts):
                check_blocks(C[j], x[0].cpu().numpy(), tr, suh, svh, K, 2, rng.choice(n // 128, 2, replace=False), tag=f"mgemm m={m} mat {j}")


@pytest.mark.parametrize("m", [1, 5])
def test_mgemm_per_matrix_widths(cuda, m):
    """size_n_list + c_ptrs: matrices of different output widths in one call (exl3_gemm.cu:341-381; SURVEY 8 a9)."""
    from exllamav3_b200 import ext
    K, k = 4, 512
    widths = [256, 128, 640]
    ts = [synth_gpu(k, n, K, cuda, 400 + n) for n in widths]
    ptr = lambda j: torch.tensor([t[j].data_ptr() for t in ts], dtype=torch.long, device=cuda)
    rng = np.random.default_rng(9)
    x = torch.from_numpy(rng.standard_normal((1, m, k)).astype(np.float16)).to(cuda)
    for fp32 in (True, False):
        outs = [torch.zeros((m, n), dtype=torch.float if fp32 else torch.half, device=cuda) for n in widths]
        C = torch.zeros((len(widths), m, max(widths)), dtype=outs[0].dtype, device=cuda)      # shape carrier; results go to c_ptrs
        Ah = torch.empty((len(widths), m, k), dtype=torch.half, device=cuda)
        snl = torch.tensor(widths, dtype=torch.int, device=cuda)
        cp = torch.tensor([o.data_ptr() for o in outs], dtype=torch.long, device=cuda)
        ext.exl3_mgemm(x, ptr(0), C, ptr(1), Ah, ptr(2), None, None, K, -1, False, True, -1, -1, 0, 1, snl, cp)
        torch.cuda.synchronize()
        for (tr, suh, svh), o, n in zip(ts, outs, widths):
            ref = orc.exl3_gemm_f64(x[0].cpu().numpy(), tr.cpu().numpy(), suh.cpu().numpy(), svh.cpu().numpy(), K, 2)
            mx, rms = rel_err(o.float().cpu().numpy(), ref)
            assert mx <= 2e-3 + (2.0 ** -10 if not fp32 else 0) and rms <= 1e-3, (n, fp32, mx, rms)


def test_hgemm_prefill_size(cuda):
    """Dense wgmma GEMM at a prefill shape (8192 x 4096 x 14336):
    sampled rows / columns against an fp64 dot product of the same fp16 operands."""
    from exllamav3_b200 import ext
    m, k, n = 8192, 4096, 14336
    g = torch.Generator(device=cuda); g.manual_seed(3)
    a = (torch.randn((m, k), generator=g, device=cuda) * 0.5).half()
    b = (torch.randn((k, n), generator=g, device=cuda) * 0.05).half()
    rng = np.random.default_rng(4)
    for dt in (torch.half, torch.float):
        c = torch.zeros((m, n), dtype=dt, device=cuda)
        ext.hgemm(a, b, c)
        torch.cuda.synchronize()
        rows = rng.choice(m, 6, replace=False); cols = rng.choice(n, 512, replace=False)
        ref = a[rows].double().cpu().numpy() @ b[:, cols].double().cpu().numpy()
        got = c[rows][:, cols].double().cpu().numpy()
        err = np.abs(got - ref).max() / np.abs(ref).max()
        assert err <= (2e-3 if dt == torch.half else 2e-5), (dt, err)
        # edges: first / last row and column tiles
        for r0, c0 in ((0, 0), (m - 1, n - 1), (m - 129, 255)):
            ref1 = float(a[r0].double() @ b[:, c0].double())
            assert abs(float(c[r0, c0]) - ref1) <= 2e-3 * max(1.0, abs(ref1))
