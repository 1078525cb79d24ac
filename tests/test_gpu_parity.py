"""
GPU parity tests (H100): the CUDA path, called through the C ABI (exllamav3_b200.ext -> libexl3b200.so), against the
CPU oracle on the same seeded inputs, against the committed golden outputs of the reference's own CUDA kernels, and
-- at BASELINE.json's full sizes -- through size-independent properties.

Tolerances (stated per north_star):
  reconstruct, had_r_128 (fp16 and fp32)   : bit-exact
  exl3_gemm / exl3_mgemm vs fp64 oracle    : max-abs <= 2e-3 * max|y| + 1 output ulp,  rel-RMS <= 1e-3
  tags 100 / 200 vs their exact model      : test_edges_host.check_f16_model (oracle.exl3_gemm_f16_model, exl3_mgemm_f16_model)
  exl3_gemm vs reference exl3_gemm (golden): max-abs <= 4e-3 * max|y|,  rel-RMS <= 2e-3 (the reference carries fp16
                                             split-K partial rounding, exl3_gemm_inner.cuh:501-503)
  reconstruct_had vs fp64                  : max-abs <= 2e-3 * max|W|   (reference test: tests/test_reconstruct_had.py:56-58)
  kernel path vs reconstruct+hgemm path    : rtol = atol = 0.05         (reference test: tests/test_qgemm.py:52-53)
"""
import os
import numpy as np
import pytest
import torch
from conftest import GOLDEN
from oracle import exl3_oracle as orc
from oracle import gen_golden_gpu as gg
from test_edges_host import check_f16_gemm, check_f16_model

pytestmark = pytest.mark.gpu


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(y, ref):
    y = y.astype(np.float64); ref = ref.astype(np.float64)
    err = np.abs(y - ref)
    return err.max() / max(np.abs(ref).max(), 1e-30), np.sqrt((err ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def run_gemm(ext, dev, x, tr, suh, svh, K, cb, fp32, a_had=True):
    m, n = x.shape[0], tr.shape[1] * 16
    A = T(x, dev)
    C = torch.full((m, n), float("nan"), dtype=torch.float if fp32 else torch.half, device=dev)
    A_had = torch.empty_like(A) if a_had else None
    tag = ext.exl3_gemm(A, T(tr, dev), C, T(suh, dev), A_had, T(svh, dev), -1, cb == 1, cb == 2, 0)
    torch.cuda.synchronize()
    return C.cpu().numpy(), (A_had.cpu().numpy() if a_had else None), tag


# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", range(1, 9))
@pytest.mark.parametrize("cb", range(3))
def test_reconstruct_bitexact(cuda, K, cb):
    from exllamav3_b200 import ext
    k, n = 64, 256
    tr, _, _, _ = orc.make_synthetic(k, n, K)
    w = torch.empty((k, n), dtype=torch.half, device=cuda)
    ext.reconstruct(w, T(tr, cuda), K, cb == 1, cb == 2)
    ref = orc.reconstruct(tr, K, cb)
    assert (w.cpu().numpy().view(np.uint16) == ref.view(np.uint16)).all()


def test_reconstruct_slice_and_edge_cases(cuda):
    from exllamav3_b200 import ext
    K, cb, k, n = 5, 1, 32, 512
    tr, _, _, _ = orc.make_synthetic(k, n, K)
    ref = orc.reconstruct(tr, K, cb)
    for off, nout in ((0, 128), (128, 256), (384, 128)):
        w = torch.empty((k, nout), dtype=torch.half, device=cuda)
        ext.reconstruct_slice(w, T(tr, cuda), K, True, False, off)
        assert (w.cpu().numpy().view(np.uint16) == ref[:, off:off + nout].view(np.uint16)).all()
    # empty output is a no-op (reconstruct.cu:113-114)
    ext.reconstruct_slice(torch.empty((k, 0), dtype=torch.half, device=cuda), T(tr, cuda), K, True, False, 0)
    with pytest.raises(RuntimeError, match="divisible by 128"):
        ext.reconstruct_slice(torch.empty((k, 64), dtype=torch.half, device=cuda), T(tr, cuda), K, True, False, 0)
    with pytest.raises(RuntimeError, match="exceeds packed tensor bounds"):
        ext.reconstruct_slice(torch.empty((k, 256), dtype=torch.half, device=cuda), T(tr, cuda), K, True, False, 384)


@pytest.mark.parametrize("dt", ["f16", "f32"])
@pytest.mark.parametrize("mode", ["none", "pre", "post"])
def test_had_r_128_bitexact(cuda, dt, mode):
    from exllamav3_b200 import ext
    rng = np.random.default_rng(3)
    x = rng.standard_normal((37, 384)).astype(np.float16 if dt == "f16" else np.float32)
    sc = (np.sign(rng.standard_normal(384)) * rng.uniform(0.5, 2, 384)).astype(np.float16)
    for scale in (1.0, 0.37):
        xi = T(x, cuda); yo = torch.empty_like(xi)
        ext.had_r_128(xi, yo, T(sc, cuda) if mode == "pre" else None, T(sc, cuda) if mode == "post" else None, scale)
        ref = orc.had_r_128(x, sc if mode == "pre" else None, sc if mode == "post" else None, scale)
        got = yo.cpu().numpy()
        view = np.uint16 if dt == "f16" else np.uint32
        assert (got.view(view) == ref.view(view)).all()
    # in place
    xi = T(x, cuda)
    ext.had_r_128(xi, xi, None, None, 1.0)
    assert (xi.cpu().numpy().view(view) == orc.had_r_128(x).view(view)).all()


@pytest.fixture(params=["tc", "simt"])
def gemm_path(request):
    """Run the test once per kernel path: tensor cores (default product path) and the CUDA-core path."""
    from exllamav3_b200 import ext
    prev = ext.set_gemm_path(ext.EXL3B_TAG_TC if request.param == "tc" else ext.EXL3B_TAG_SIMT)
    yield request.param
    ext.set_gemm_path(prev)


@pytest.mark.parametrize("K,cb", [(1, 2), (2, 2), (3, 0), (4, 2), (4, 0), (4, 1), (5, 2), (6, 2), (7, 1), (8, 2)])
@pytest.mark.parametrize("m", [1, 5, 16, 17])
def test_gemm_vs_oracle(cuda, gemm_path, K, cb, m):
    from exllamav3_b200 import ext
    k, n = 512, 384
    tr, suh, svh, x = orc.make_synthetic(k, n, K, m=m)
    ref = orc.exl3_gemm_f64(x, tr, suh, svh, K, cb)
    for fp32 in (False, True):
        y, xh, tag = run_gemm(ext, cuda, x, tr, suh, svh, K, cb, fp32)
        assert tag == (ext.EXL3B_TAG_TC if gemm_path == "tc" else ext.EXL3B_TAG_SIMT)
        assert not np.isnan(y.astype(np.float32)).any()
        if gemm_path == "simt":      # the tensor-core path keeps its transformed input in a private tiled buffer
            xh_ref = orc.had_r_128(x, pre_scale=suh)
            assert (xh.view(np.uint16) == xh_ref.view(np.uint16)).all()      # input transform bit-exact
        mx, rms = rel_err(y, ref)
        ulp = 2.0 ** -10 if not fp32 else 0.0
        assert mx <= 2e-3 + ulp, (K, cb, m, fp32, mx)
        assert rms <= 1e-3, (K, cb, m, fp32, rms)
        check_f16_gemm(y, x, tr, suh, svh, K, cb, fp32, (gemm_path, K, cb, m))


def test_gemm_without_scratch_and_ragged_rows(cuda, gemm_path):
    from exllamav3_b200 import ext
    K, cb, k, n = 4, 2, 256, 256
    for m in (1, 3, 8, 9, 31, 33, 144, 300):          # rows up to the reconstruct threshold (modules/quant/exl3.py:10)
        tr, suh, svh, x = orc.make_synthetic(k, n, K, m=m)
        ref = orc.exl3_gemm_f64(x, tr, suh, svh, K, cb)
        y, _, tag = run_gemm(ext, cuda, x, tr, suh, svh, K, cb, True, a_had=False)
        mx, rms = rel_err(y, ref)
        assert mx <= 2e-3 and rms <= 1e-3, (m, mx, rms)
        if tag in (ext.EXL3B_TAG_SIMT, ext.EXL3B_TAG_TC):
            check_f16_gemm(y, x, tr, suh, svh, K, cb, True, (gemm_path, m))
    # A_had aliasing A is allowed (science/qgemm_benchmark.py:85)
    tr, suh, svh, x = orc.make_synthetic(k, n, K, m=4)
    A = T(x, cuda); C = torch.empty((4, n), dtype=torch.half, device=cuda)
    tag = ext.exl3_gemm(A, T(tr, cuda), C, T(suh, cuda), A, T(svh, cuda), -1, False, True, 0)
    mx, rms = rel_err(C.cpu().numpy(), orc.exl3_gemm_f64(x, tr, suh, svh, K, cb))
    assert mx <= 3e-3 and rms <= 1e-3
    if tag in (ext.EXL3B_TAG_SIMT, ext.EXL3B_TAG_TC):
        check_f16_gemm(C.cpu().numpy(), x, tr, suh, svh, K, cb, False, (gemm_path, "aliased A_had"))


def test_gemm_vs_reference_cuda_golden(cuda, gemm_path):
    p = os.path.join(GOLDEN, "ref_gpu.npz")
    if not os.path.exists(p):
        pytest.skip("tests/golden/ref_gpu.npz not generated yet")
    from exllamav3_b200 import ext
    g = np.load(p)
    for (m, k, n, K, cb, fp32) in gg.gemm_cases():
        tr, suh, svh, x = orc.make_synthetic(k, n, K, m=m)
        key = f"gemm_{m}_{k}_{n}_{K}_{cb}_{int(fp32)}"
        y, xh, _ = run_gemm(ext, cuda, x, tr, suh, svh, K, cb, fp32)
        if gemm_path == "simt":
            assert (xh.view(np.uint16) == g[key + "_xh"].view(np.uint16)).all(), key
        mx, rms = rel_err(y, g[key])
        assert mx <= 4e-3 and rms <= 2e-3, (key, mx, rms)
    for (K, cb, k, n) in gg.reconstruct_cases():
        tr, _, _, _ = orc.make_synthetic(k, n, K)
        w = torch.empty((k, n), dtype=torch.half, device=cuda)
        ext.reconstruct(w, T(tr, cuda), K, cb == 1, cb == 2)
        assert (w.cpu().numpy().view(np.uint16) == g[f"rec_{K}_{cb}_{k}_{n}"].view(np.uint16)).all()


@pytest.mark.parametrize("K,cb", [(3, 0), (4, 2), (2, 1), (6, 2)])
def test_reconstruct_had(cuda, K, cb):
    # tests/test_reconstruct_had.py:45-68: fused W vs explicit Sylvester, max|err|/max|ref| < 2e-3, incl. slice path
    from exllamav3_b200 import ext
    k, n = 256, 384
    tr, suh, svh, _ = orc.make_synthetic(k, n, K)
    ref = orc.get_weight_tensor_f64(tr, suh, svh, K, cb)
    w = torch.empty((k, n), dtype=torch.half, device=cuda)
    ext.reconstruct_had_slice(w, T(tr, cuda), T(suh, cuda), T(svh, cuda), K, cb == 1, cb == 2, 0)
    got = w.cpu().numpy().astype(np.float64)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 2e-3
    w2 = torch.empty((k, 256), dtype=torch.half, device=cuda)
    ext.reconstruct_had_slice(w2, T(tr, cuda), T(suh, cuda), T(svh[128:], cuda), K, cb == 1, cb == 2, 128)
    assert torch.equal(w2.cpu(), w[:, 128:].cpu())


@pytest.mark.parametrize("K,cb", [(1, 0), (2, 1), (3, 2), (4, 2), (5, 0), (6, 2), (7, 1), (8, 2)])
def test_reconstruct_had_tensor_core_and_cuda_core_twins(cuda, K, cb):
    # reconstruct_tc.cu (both Hadamards as wgmma GEMMs, the default) against the oracle and against the CUDA-core
    # kernel of kernels_basic.cu on a shape with more blocks than one wave of the persistent grid covers per CTA
    from exllamav3_b200 import ext
    k, n = 1024, 5120 if K <= 4 else 2560
    tr, suh, svh, _ = orc.make_synthetic(k, n, K, seed=K * 10 + cb)
    outs = {}
    try:
        for mode in (1, 2):                          # CUDA cores, tensor cores
            ext.lib.exl3b_debug_reconstruct_had(mode)
            w = torch.full((k, n), float("nan"), dtype=torch.half, device=cuda)
            ext.reconstruct_had_slice(w, T(tr, cuda), T(suh, cuda), T(svh, cuda), K, cb == 1, cb == 2, 0)
            outs[mode] = w.cpu().numpy().astype(np.float64)
            # column window of the packed tensor (modules/quant/exl3.py:199-211)
            w2 = torch.empty((k, 384), dtype=torch.half, device=cuda)
            ext.reconstruct_had_slice(w2, T(tr, cuda), T(suh, cuda), T(svh[256:640], cuda), K, cb == 1, cb == 2, 256)
            assert torch.equal(w2.cpu(), w[:, 256:640].cpu())
    finally:
        ext.lib.exl3b_debug_reconstruct_had(0)
    # oracle on the first 256 rows (the transform is block-diagonal over 128-row blocks)
    ref = orc.get_weight_tensor_f64(tr[:16], suh[:256], svh, K, cb)
    for mode in outs:
        assert np.isfinite(outs[mode]).all()
        assert np.abs(outs[mode][:256] - ref).max() / np.abs(ref).max() < 2e-3, mode
    # the two kernels round at the same places (fp16 tile between the passes, fp16 scale multiplies): they differ by
    # the summation order inside the 128-term sums only, i.e. by a few fp16 ulps on few elements
    d = np.abs(outs[1] - outs[2])
    assert d.max() <= 4e-3 * np.abs(outs[1]).max()
    assert (d > 0).mean() < 0.05


def test_reconstruct_had_vs_reference_cuda_golden_and_fp32_model(cuda):
    """Both reconstruct_had kernels on the cases captured from the reference's own kernel: within the reference's tolerance of its
    output (which adds in fp16), and equal to the fp32-sum model (oracle.reconstruct_had_fp32_model) up to the order of the fp32
    additions: a few fp16 ulps on few elements."""
    p = os.path.join(GOLDEN, "ref_gpu.npz")
    if not os.path.exists(p):
        pytest.skip("tests/golden/ref_gpu.npz not generated yet")
    from exllamav3_b200 import ext
    g = np.load(p)
    try:
        for mode in (1, 2):
            ext.lib.exl3b_debug_reconstruct_had(mode)
            for (K, cb, k, n, off, nout) in [(4, 2, 128, 384, 128, 256), (3, 0, 128, 256, 0, 256)]:
                tr, suh, svh, _ = orc.make_synthetic(k, n, K)
                w = torch.empty((k, nout), dtype=torch.half, device=cuda)
                ext.reconstruct_had_slice(w, T(tr, cuda), T(suh, cuda), T(svh[off:], cuda), K, cb == 1, cb == 2, off)
                got = w.cpu().numpy()
                gold = g[f"rechad_{K}_{cb}_{k}_{n}_{off}_{nout}"].astype(np.float64)
                assert np.abs(got.astype(np.float64) - gold).max() <= 2.5e-3 * np.abs(gold).max(), (mode, K, cb)
                model = orc.reconstruct_had_fp32_model(tr[:, off // 16:(off + nout) // 16], suh, svh[off:off + nout], K, cb)
                same = (got.view(np.uint16) == model.view(np.uint16)).mean()
                d = np.abs(got.astype(np.float64) - model.astype(np.float64)).max()
                assert same >= 0.97 and d <= 2e-3 * np.abs(gold).max(), (mode, K, cb, same, d)
    finally:
        ext.lib.exl3b_debug_reconstruct_had(0)


def test_hgemm(cuda):
    from exllamav3_b200 import ext
    rng = np.random.default_rng(0)
    for (m, k, n) in ((1, 128, 128), (37, 256, 384), (300, 512, 256)):
        a = rng.standard_normal((m, k)).astype(np.float16); b = rng.standard_normal((k, n)).astype(np.float16)
        ref = a.astype(np.float64) @ b.astype(np.float64)
        for dt in (torch.half, torch.float):
            c = torch.empty((m, n), dtype=dt, device=cuda)
            ext.hgemm(T(a, cuda), T(b, cuda), c)
            mx, rms = rel_err(c.cpu().numpy(), ref)
            assert mx <= (2e-3 if dt == torch.half else 1e-4), (m, k, n, dt, mx)
    # strided C rows (hgemm.cu:52-54), as used by the sliced lm_head path (modules/quant/exl3.py:199-211)
    a = rng.standard_normal((5, 128)).astype(np.float16); b = rng.standard_normal((128, 128)).astype(np.float16)
    cfull = torch.zeros((5, 384), dtype=torch.half, device=cuda)
    ext.hgemm(T(a, cuda), T(b, cuda), cfull[:, 128:256])
    ref = (a.astype(np.float64) @ b.astype(np.float64))
    assert rel_err(cfull[:, 128:256].cpu().numpy(), ref)[0] <= 2e-3 and float(cfull[:, :128].abs().max()) == 0.0


def test_hgemm_tensor_core_tiles(cuda):
    """The dense wgmma GEMM (128 x 128 tiles, persistent CTAs) -- ragged m / n / k, a single tile, several tiles per CTA, strided C,
    both output types; against an fp64 product of the fp16 operands (the reference's hgemm is cuBLAS, hgemm.cu:19-102)."""
    from exllamav3_b200 import ext
    rng = np.random.default_rng(1)
    for (m, k, n) in ((300, 512, 256), (129, 72, 264), (1, 128, 128), (513, 200, 520), (1024, 1024, 768), (4096, 256, 4352)):
        a = rng.standard_normal((m, k)).astype(np.float16); b = rng.standard_normal((k, n)).astype(np.float16)
        ref = a.astype(np.float64) @ b.astype(np.float64)
        for dt in (torch.half, torch.float):
            c = torch.full((m, n), float("nan"), dtype=dt, device=cuda)
            ext.hgemm(T(a, cuda), T(b, cuda), c)
            torch.cuda.synchronize()
            assert not torch.isnan(c.float()).any(), (m, k, n, dt)
            mx, rms = rel_err(c.cpu().numpy(), ref)
            assert mx <= (2e-3 if dt == torch.half else 1e-4), (m, k, n, dt, mx)
    a = rng.standard_normal((260, 128)).astype(np.float16); b = rng.standard_normal((128, 128)).astype(np.float16)
    cfull = torch.zeros((260, 384), dtype=torch.half, device=cuda)
    ext.hgemm(T(a, cuda), T(b, cuda), cfull[:, 128:256])
    assert rel_err(cfull[:, 128:256].cpu().numpy(), a.astype(np.float64) @ b.astype(np.float64))[0] <= 2e-3
    assert float(cfull[:, :128].abs().max()) == 0.0 and float(cfull[:, 256:].abs().max()) == 0.0


def test_linear_exl3_kernel_vs_reconstruct_path(cuda):
    # the reference's own pin of this path: tests/test_qgemm.py:31-53 (rtol = atol = 0.05), m list from there
    from exllamav3_b200 import QLinear
    K, k, n = 3, 1024, 512
    tr, suh, svh, _ = orc.make_synthetic(k, n, K)
    lin = QLinear(T(tr, cuda), T(suh, cuda), T(svh, cuda), mul1=True)
    torch.manual_seed(0)
    for m in (1, 2, 8, 16, 17, 31, 32, 33, 256, 2048):
        x = torch.randn((1, m, k), dtype=torch.half, device=cuda)
        a = lin.forward(x, {"reconstruct": False}) if m <= 144 else lin.forward(x, {})
        b = lin.forward(x, {"reconstruct": True})
        torch.testing.assert_close(a, b, rtol=0.05, atol=0.05)
        assert a.shape == (1, m, n)
        ref = orc.exl3_gemm_f64(x.view(m, k).cpu().numpy(), tr, suh, svh, K, 2)
        mx, rms = rel_err(b.view(m, n).cpu().numpy(), ref)
        assert mx <= 5e-3 and rms <= 2e-3, (m, mx, rms)
    # fp32 output + bias
    bias = torch.randn(n, dtype=torch.half, device=cuda)
    lin2 = QLinear(T(tr, cuda), T(suh, cuda), T(svh, cuda), mul1=True, bias=bias, out_dtype=torch.float)
    x = torch.randn((4, k), dtype=torch.half, device=cuda)
    y = lin2.forward(x, {})
    assert y.dtype == torch.float
    torch.testing.assert_close(y, lin.forward(x, {}, torch.float) + bias, rtol=1e-3, atol=1e-3)
    # original-basis W (fused reconstruct kernel)
    W = lin.weight().cpu().numpy().astype(np.float64)
    Wref = orc.get_weight_tensor_f64(tr, suh, svh, K, 2)
    assert np.abs(W - Wref).max() / np.abs(Wref).max() < 2e-3


def test_mgemm_modes(cuda):
    """The four modes of exl3_mgemm on the default path and on the CUDA-core kernels (tag 100), which are also held to their
    exact model."""
    from exllamav3_b200 import ext, QLinear, pointer_tables
    from types import SimpleNamespace
    k, n, K, m, mats, A, wts = gg.mgemm_inputs()
    lins = [QLinear(T(t[0], cuda), T(t[1], cuda), T(t[2], cuda), mul1=True) for t in mats]
    pt = pointer_tables(cuda, lins)
    ml = SimpleNamespace(ptrs_trellis=pt[0], ptrs_suh=pt[1], ptrs_svh=pt[2], mcg=False, mul1=True)
    trs = [t[0] for t in mats]; suhs = [t[1] for t in mats]; svhs = [t[2] for t in mats]
    golden = np.load(os.path.join(GOLDEN, "ref_gpu.npz")) if os.path.exists(os.path.join(GOLDEN, "ref_gpu.npz")) else None
    tags = set()

    def model(tag, C, A_, npdt, what, slots=slice(None), **kw):
        """C of a tag-100 / 200 call against oracle.exl3_mgemm_f16_model"""
        tags.add(tag)
        if tag in (ext.EXL3B_TAG_SIMT, ext.EXL3B_TAG_TC):
            ref, tol = orc.exl3_mgemm_f16_model(A_, trs, suhs, svhs, K, 2, npdt, bszm_out=4, **kw)
            check_f16_model(C.cpu().numpy()[slots], ref[slots], None if tol is None else tol[slots], what)

    for path in (0, ext.EXL3B_TAG_SIMT):
        prev = ext.set_gemm_path(path)
        try:
            for fp32 in (False, True):
                dt = torch.float if fp32 else torch.half
                npdt = np.float32 if fp32 else np.float16
                Ah = torch.empty((4, m, k), dtype=torch.half, device=cuda)
                tol = 3e-3
                # (a) one input, four outputs
                C = torch.zeros((4, m, n), dtype=dt, device=cuda)
                tag = ext.exl3_mgemm(T(A[:1], cuda), ml.ptrs_trellis, C, ml.ptrs_suh, Ah, ml.ptrs_svh, None, None, K, -1,
                                     ml.mcg, ml.mul1, -1, -1, 0)
                ref = orc.exl3_mgemm(A[:1], trs, suhs, svhs, K, 2, npdt, bszm_out=4)
                assert rel_err(C.cpu().numpy(), ref)[0] <= tol
                model(tag, C, A[:1], npdt, (path, "a", fp32))
                if golden is not None:
                    assert rel_err(C.cpu().numpy(), golden[f"mgemm_a_{int(fp32)}"])[0] <= 5e-3
                # (b) indices with a skipped slot
                C = torch.zeros((4, m, n), dtype=dt, device=cuda)
                idx = torch.tensor([[2, -1, 0, 3]], dtype=torch.long, device=cuda)
                tag = ext.exl3_mgemm(T(A, cuda), ml.ptrs_trellis, C, ml.ptrs_suh, Ah, ml.ptrs_svh, idx, None, K, -1,
                                     ml.mcg, ml.mul1, -1, -1, 0)
                ref = orc.exl3_mgemm(A, trs, suhs, svhs, K, 2, npdt, indices=[2, -1, 0, 3], bszm_out=4)
                assert rel_err(C.cpu().numpy(), ref)[0] <= tol and float(C[1].abs().max()) == 0.0
                model(tag, C, A, npdt, (path, "b", fp32), indices=[2, -1, 0, 3])
                if golden is not None:
                    assert rel_err(C.cpu().numpy(), golden[f"mgemm_b_{int(fp32)}"])[0] <= 5e-3
                # (c) weighted reduction into C[0]
                C = torch.zeros((4, m, n), dtype=dt, device=cuda)
                idx = torch.tensor([[3, 1, 0, 2]], dtype=torch.long, device=cuda)
                tag = ext.exl3_mgemm(T(A[:1], cuda), ml.ptrs_trellis, C, ml.ptrs_suh, Ah, ml.ptrs_svh, idx,
                                     T(wts, cuda).view(1, 4), K, -1, ml.mcg, ml.mul1, -1, -1, 0)
                ref = orc.exl3_mgemm(A[:1], trs, suhs, svhs, K, 2, npdt, indices=[3, 1, 0, 2], weights=wts, bszm_out=4)
                assert rel_err(C[0].cpu().numpy(), ref[0])[0] <= tol
                model(tag, C, A[:1], npdt, (path, "c", fp32), slots=slice(0, 1), indices=[3, 1, 0, 2], weights=wts)
                if golden is not None:
                    assert rel_err(C[0].cpu().numpy(), golden[f"mgemm_c_{int(fp32)}"])[0] <= 5e-3
                # (d) expert-range filter [1, 3) with local tables
                C = torch.zeros((4, m, n), dtype=dt, device=cuda)
                tag = ext.exl3_mgemm(T(A[:1], cuda), ml.ptrs_trellis[1:3].contiguous(), C, ml.ptrs_suh[1:3].contiguous(), Ah,
                                     ml.ptrs_svh[1:3].contiguous(), idx, T(wts, cuda).view(1, 4), K, -1, ml.mcg, ml.mul1, 1, 3, 0)
                ref = orc.exl3_mgemm(A[:1], trs[1:3], suhs[1:3], svhs[1:3], K, 2, npdt, indices=[3, 1, 0, 2], weights=wts,
                                     min_index=1, max_index=3, bszm_out=4)
                assert rel_err(C[0].cpu().numpy(), ref[0])[0] <= tol
                if golden is not None:
                    assert rel_err(C[0].cpu().numpy(), golden[f"mgemm_d_{int(fp32)}"])[0] <= 5e-3
        finally:
            ext.set_gemm_path(prev)
    assert ext.EXL3B_TAG_SIMT in tags


@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("m", [1, 2, 4, 5, 8])
def test_gemm_i8_tensor_core_path(cuda, K, m):
    """
    mul1 int8 tensor-core codebook path (tag 210, default for mul1 at m <= 4, and at m <= 8 while the transformed rows fit
    the kernel's shared-memory cache).  Two bars:
      * implementation: agrees with the exact integer model of the path (oracle.exl3_gemm_i8_model) to fp32 round-off
      * approximation: distance to the fp64 oracle of the reference math  max-abs <= 2e-3 max|y|, rel-RMS <= 1e-3
        (the skipped per-weight fp16 rounding; the reference's own default int8 GEMV deviates ~9e-3, exl3_gemv_int8.cu:19-20)
    """
    from exllamav3_b200 import ext
    prev = ext.set_gemm_path(ext.EXL3B_TAG_TC_I8)
    try:
        for (k, n) in ((512, 384), (2048, 128), (128, 1024)):
            tr, suh, svh, x = orc.make_synthetic(k, n, K, m=m)
            model = orc.exl3_gemm_i8_model(x, tr, suh, svh, K)
            ref = orc.exl3_gemm_f64(x, tr, suh, svh, K, 2)
            for fp32 in (True, False):
                y, _, tag = run_gemm(ext, cuda, x, tr, suh, svh, K, 2, fp32)
                assert tag == ext.EXL3B_TAG_TC_I8
                mx, rms = rel_err(y, model)
                assert mx <= (2e-5 if fp32 else 1.5e-3) and rms <= (1e-5 if fp32 else 5e-4), (K, m, k, n, fp32, mx, rms)
                mx, rms = rel_err(y, ref)
                assert mx <= 2e-3 + (2.0 ** -10 if not fp32 else 0) and rms <= 1e-3, (K, m, k, n, fp32, mx, rms)
        # zero rows and huge dynamic range do not break the per-row activation scale
        tr, suh, svh, x = orc.make_synthetic(512, 256, 4, m=3)
        x[1] = 0
        x[2] *= np.float16(100.0)
        y, _, _ = run_gemm(ext, cuda, x, tr, suh, svh, 4, 2, True)
        ref = orc.exl3_gemm_f64(x, tr, suh, svh, 4, 2)
        assert float(np.abs(y[1]).max()) == 0.0
        for r in (0, 2):
            assert rel_err(y[r:r + 1], ref[r:r + 1])[0] <= 2e-3
        # forcing the path outside its domain (m > 8) is an error, not a silent fallback
        with pytest.raises(RuntimeError, match="int8 tensor-core path forced"):
            ext.exl3_gemm(T(np.zeros((9, 512), np.float16), cuda), T(tr, cuda),
                          torch.empty((9, 256), dtype=torch.half, device=cuda), T(suh, cuda), None, T(svh, cuda),
                          -1, False, True, 0)
    finally:
        ext.set_gemm_path(prev)


@pytest.mark.parametrize("nm,per_mat_input", [(2, False), (2, True), (3, False), (7, False)])
def test_mgemm_i8_tensor_core_single_launch(cuda, nm, per_mat_input):
    """
    Dense exl3_mgemm (the reference's fused k+v / gate+up call, modules/attn.py:603-631, modules/mlp.py:726-760) on the
    mul1 int8 tensor-core path: ONE launch (tag 210), CTA groups per matrix, per-CTA patched tensor maps.  Each
    matrix's output must equal the single-matrix i8 kernel bit for bit when the CTA group size matches, and must
    meet the exl3_gemm tolerances against the fp64 oracle in every case.
    """
    from exllamav3_b200 import ext
    prev = ext.set_gemm_path(0)
    try:
        for (k, n, K, m) in ((512, 384, 4, 1), (1024, 256, 3, 4), (256, 1152, 5, 2)):
            mats = [orc.make_synthetic(k, n, K, seed=77 + 13 * e, m=m) for e in range(nm)]
            rng = np.random.default_rng(nm * 100 + m)
            A = rng.standard_normal((nm if per_mat_input else 1, m, k)).astype(np.float16)
            trs = [T(t[0], cuda) for t in mats]; suhs = [T(t[1], cuda) for t in mats]; svhs = [T(t[2], cuda) for t in mats]
            pt = torch.tensor([t.data_ptr() for t in trs], dtype=torch.long, device=cuda)
            ps = torch.tensor([t.data_ptr() for t in suhs], dtype=torch.long, device=cuda)
            pv = torch.tensor([t.data_ptr() for t in svhs], dtype=torch.long, device=cuda)
            for fp32 in (True, False):
                C = torch.full((nm, m, n), float("nan"), dtype=torch.float if fp32 else torch.half, device=cuda)
                Ah = torch.empty((nm, m, k), dtype=torch.half, device=cuda)
                before = ext.launch_count()
                tag = ext.exl3_mgemm(T(A, cuda), pt, C, ps, Ah, pv, None, None, K, -1, False, True, -1, -1, 0)
                assert tag == ext.EXL3B_TAG_TC_I8
                assert ext.launch_count() - before == 1
                Cn = C.float().cpu().numpy()
                assert np.isfinite(Cn).all()
                for j in range(nm):
                    a = A[j] if per_mat_input else A[0]
                    ref = orc.exl3_gemm_f64(a, mats[j][0], mats[j][1], mats[j][2], K, 2)
                    mx, rms = rel_err(Cn[j], ref)
                    assert mx <= 2e-3 + (2.0 ** -10 if not fp32 else 0) and rms <= 1e-3, (nm, k, n, K, m, j, fp32, mx, rms)
                    model = orc.exl3_gemm_i8_model(a, mats[j][0], mats[j][1], mats[j][2], K)
                    mx, rms = rel_err(Cn[j], model)
                    assert mx <= (2e-5 if fp32 else 1.5e-3), (nm, k, n, K, m, j, fp32, mx)
                # repeated launches are bit-identical (fixed-order split-K inside every CTA group)
                C2 = torch.empty_like(C)
                ext.exl3_mgemm(T(A, cuda), pt, C2, ps, Ah, pv, None, None, K, -1, False, True, -1, -1, 0)
                assert torch.equal(C, C2)
    finally:
        ext.set_gemm_path(prev)


def test_tc_determinism_and_stream_k(cuda):
    """Split-K partials are combined in a fixed order: repeated launches are bit-identical; shapes chosen so that
    strips are split across CTAs (k large, n small) and so that CTAs span several strips (n large)."""
    from exllamav3_b200 import ext
    prev = ext.set_gemm_path(0)
    try:
        for (k, n, m, path) in ((8192, 128, 1, ext.EXL3B_TAG_TC), (4096, 256, 3, ext.EXL3B_TAG_TC), (128, 8192, 2, ext.EXL3B_TAG_TC),
                                (1024, 2048, 16, ext.EXL3B_TAG_TC), (16384, 128, 1, ext.EXL3B_TAG_TC_I8),
                                (4096, 256, 3, ext.EXL3B_TAG_TC_I8), (128, 8192, 2, ext.EXL3B_TAG_TC_I8)):
            ext.set_gemm_path(path)
            tr, suh, svh, x = orc.make_synthetic(k, n, 4, m=m)
            ref = orc.exl3_gemm_f64(x, tr, suh, svh, 4, 2)
            outs = [run_gemm(ext, cuda, x, tr, suh, svh, 4, 2, True)[0] for _ in range(3)]
            assert (outs[0].view(np.uint32) == outs[1].view(np.uint32)).all()
            assert (outs[0].view(np.uint32) == outs[2].view(np.uint32)).all()
            mx, rms = rel_err(outs[0], ref)
            assert mx <= 2e-3 and rms <= 1e-3, (k, n, m, mx, rms)
    finally:
        ext.set_gemm_path(prev)


def test_i8_split_k_exchange_ring(cuda):
    """
    The int8 path exchanges split-K partial sums through a buffer that must be all-sentinel between launches (contributors
    store, the strip's reducer reads and re-arms; 8 rotating slot sets).  Interleave shapes with different grids, strip
    splits and row counts -- single-matrix and multi-matrix launches, back to back without host synchronisation, several
    times around the slot ring -- and require every result to stay bit-identical to its first computation: a slot left
    un-armed (or armed too early) would be consumed as a stale partial sum by a later launch.
    """
    from exllamav3_b200 import ext
    prev = ext.set_gemm_path(0)
    try:
        cases = []
        for (k, n, m) in ((16384, 128, 1), (4096, 256, 3), (2048, 1024, 4), (8192, 384, 2), (128, 2048, 1)):
            tr, suh, svh, x = orc.make_synthetic(k, n, 4, m=m)
            cases.append(dict(k=k, n=n, m=m, x=T(x, cuda), tr=T(tr, cuda), suh=T(suh, cuda), svh=T(svh, cuda),
                              xh=torch.empty((m, k), dtype=torch.half, device=cuda), ref=orc.exl3_gemm_f64(x, tr, suh, svh, 4, 2)))
        # one multi-matrix case (two matrices sharing the input)
        k, n, m = 4096, 512, 2
        mats = [orc.make_synthetic(k, n, 4, seed=900 + e, m=m) for e in range(2)]
        trs = [T(t[0], cuda) for t in mats]; suhs = [T(t[1], cuda) for t in mats]; svhs = [T(t[2], cuda) for t in mats]
        ptr = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.long, device=cuda)
        mg = dict(x=T(mats[0][3], cuda).view(1, m, k), B=ptr(trs), suh=ptr(suhs), svh=ptr(svhs),
                  xh=torch.empty((2, m, k), dtype=torch.half, device=cuda))
        first = {}
        for rnd in range(6):                                   # 6 x 6 launches = 4.5 times around the 8-deep ring
            outs = []
            for i, c in enumerate(cases):
                y = torch.empty((c["m"], c["n"]), dtype=torch.float, device=cuda)
                tag = ext.exl3_gemm(c["x"], c["tr"], y, c["suh"], c["xh"], c["svh"], -1, False, True, 0)
                assert tag == ext.EXL3B_TAG_TC_I8
                outs.append((i, y))
            y2 = torch.empty((2, m, n), dtype=torch.float, device=cuda)
            assert ext.exl3_mgemm(mg["x"], mg["B"], y2, mg["suh"], mg["xh"], mg["svh"], None, None, 4, -1, False, True, -1, -1, 0) == ext.EXL3B_TAG_TC_I8
            outs.append(("mg", y2))
            torch.cuda.synchronize()
            for key, y in outs:
                if key not in first:
                    first[key] = y.clone()
                else:
                    assert torch.equal(first[key], y), (rnd, key)
        for i, c in enumerate(cases):
            mx, rms = rel_err(first[i].cpu().numpy(), c["ref"])
            assert mx <= 2e-3 and rms <= 1e-3, (c["k"], c["n"], c["m"], mx, rms)
        for j in range(2):
            ref = orc.exl3_gemm_f64(mats[0][3], mats[j][0], mats[j][1], mats[j][2], 4, 2)
            mx, rms = rel_err(first["mg"][j].cpu().numpy(), ref)
            assert mx <= 2e-3 and rms <= 1e-3, (j, mx, rms)
    finally:
        ext.set_gemm_path(prev)


def test_full_size_properties(cuda):
    """
    BASELINE.json sizes (Llama-3.1-8B shapes, K=4, mul1) where the numpy oracle is too slow for a dense check:
      * linearity in x:  f(a x1 + b x2) ~= a f(x1) + b f(x2)
      * column-split == slice of the full result; row-split partial sums == full result  (TP shard identity, 8e)
      * spot check of 256 random output columns against the fp64 oracle restricted to those columns' 128-blocks
    """
    from exllamav3_b200 import ext, QLinear, tp
    K, cb = 4, 2
    for (k, n) in ((4096, 4096), (4096, 14336), (14336, 4096)):
        tr, suh, svh, _ = orc.make_synthetic(k, n, K)
        lin = QLinear(T(tr, cuda), T(suh, cuda), T(svh, cuda), mul1=True, out_dtype=torch.float)
        torch.manual_seed(k + n)
        x1 = torch.randn((1, k), dtype=torch.half, device=cuda); x2 = torch.randn((1, k), dtype=torch.half, device=cuda)
        y1, y2 = lin.forward(x1, {}), lin.forward(x2, {})
        xs = (0.5 * x1.float() + 0.25 * x2.float()).half()
        ys = lin.forward(xs, {})
        lin_err = (ys - (0.5 * y1 + 0.25 * y2)).abs().max() / ys.abs().max()
        assert float(lin_err) < 5e-3, (k, n, float(lin_err))
        # TP identities
        half_n = (n // 256) * 128
        ca = tp.tp_slice(lin, (True, 0, half_n)); cb_ = tp.tp_slice(lin, (True, half_n, n))
        ycat = torch.cat((ca.forward(x1, {}), cb_.forward(x1, {})), dim=-1)
        assert float((ycat - y1).abs().max() / y1.abs().max()) < 1e-3
        half_k = (k // 256) * 128
        ra = tp.tp_slice(lin, (False, 0, half_k)); rb = tp.tp_slice(lin, (False, half_k, k))
        ysum = ra.forward(x1[:, :half_k].contiguous(), {}) + rb.forward(x1[:, half_k:].contiguous(), {})
        assert float((ysum - y1).abs().max() / y1.abs().max()) < 2e-3
        # spot check: two random 128-column blocks against the oracle
        rng = np.random.default_rng(n)
        for blk in rng.choice(n // 128, 2, replace=False):
            sl = slice(blk * 128, blk * 128 + 128)
            ref = orc.exl3_gemm_f64(x1.cpu().numpy(), tr[:, blk * 8: blk * 8 + 8, :], suh, svh[sl], K, cb)
            mx, rms = rel_err(y1[:, sl].cpu().numpy(), ref)
            assert mx <= 2e-3 and rms <= 1e-3, (k, n, blk, mx, rms)
