"""
Oracle self-checks and pinning (CPU only).  The oracle (oracle/exl3_oracle.py) is the checker for the CUDA path;
these tests pin the checker itself:
  * fixtures produced by importing the reference's own Python helpers (tests/golden/ref_py.npz, oracle/gen_golden_py.py)
  * outputs of the reference's own CUDA kernels (tests/golden/ref_gpu.npz, oracle/gen_golden_gpu.py)
  * format invariants the reference's tests assert (tests/test_quant_fn.py:82-87,100-128)
  * the C restatement (oracle/exl3_oracle.c) against the numpy one
"""
import os, ctypes, subprocess, sys
import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from oracle import exl3_oracle as orc
from oracle import gen_golden_gpu as gg


def test_perm_matches_reference_python():
    g = np.load(os.path.join(GOLDEN, "ref_py.npz"))
    assert (orc.tensor_core_perm() == g["tensor_core_perm"]).all()


def test_hadamard_matrix_matches_reference_python():
    g = np.load(os.path.join(GOLDEN, "ref_py.npz"))
    assert (orc.hadamard_matrix_128() == g["had128"]).all()
    # butterfly == matrix
    x = np.random.default_rng(1).standard_normal((5, 128)).astype(np.float32)
    ref = x.astype(np.float64) @ orc.hadamard_matrix_128()
    assert np.allclose(orc.fwht128_f32(x), ref, rtol=1e-5, atol=1e-4)


def test_preapply_had_matches_reference_python():
    # reference: fp32 matmul with the scaled fp32 Hadamard, rounded to fp16 (quantize.py:340-357)
    g = np.load(os.path.join(GOLDEN, "ref_py.npz"))
    w = g["had_in"]
    H = (orc.hadamard_matrix_128() / np.sqrt(128.0))
    l = (H @ w.astype(np.float64).reshape(2, 128, 256)).reshape(256, 256)
    r = (w.astype(np.float64).reshape(256, 2, 128) @ H).reshape(256, 256)
    # fp32 matmul vs fp64: allow 1 fp16 ulp on a handful of elements
    for ours, ref in ((l, g["had_l"]), (r, g["had_r"])):
        d = np.abs(ours - ref.astype(np.float64))
        assert d.max() <= 2.0 ** -9 * max(1.0, np.abs(ref).max())
        assert (ours.astype(np.float16) != ref).mean() < 0.01


def test_unpack_bf_matches_reference_python():
    g = np.load(os.path.join(GOLDEN, "ref_py.npz"))
    bits = g["bf_in"].view(np.uint16).astype(np.int64)
    exp = ((bits[:, None] >> np.arange(16)) & 1).reshape(-1)
    assert ((1.0 - 2.0 * exp).astype(np.float16) == g["bf_out"]).all()


@pytest.mark.parametrize("K", range(1, 9))
def test_pack_unpack_roundtrip_and_tailbiting(K):
    # construction of a valid tail-biting state sequence as tests/test_quant_fn.py:100-113
    rng = np.random.default_rng(K)
    sym = rng.integers(0, 1 << K, size=(7, 256 + 16), dtype=np.uint64)
    stream = np.zeros((7, 256), dtype=np.uint16)
    for t in range(256):
        acc = np.zeros(7, dtype=np.uint64)
        # state t = last 16 bits of the symbol stream ending at symbol t (cyclic)
        nsym = -(-16 // K)
        for j in range(nsym, -1, -1):
            acc = (acc << np.uint64(K)) | sym[:, (t - j) % 256]
        stream[:, t] = (acc & np.uint64(0xffff)).astype(np.uint16)
    packed = orc.pack_states(stream, K)
    assert packed.shape == (7, 16 * K)
    un = orc.unpack_states(packed, K)
    assert (un == stream).all()
    assert ((un[:, 0] >> K) == (un[:, 255] & ((1 << (16 - K)) - 1))).all()      # test_quant_fn.py:82-87
    # shift relation st[t+1] = (st[t] << K | new) & 0xffff
    nxt = ((un[:, :-1].astype(np.uint32) << K) & 0xffff) >> K
    assert (nxt == (un[:, 1:] >> K)).all()


def test_any_bitstream_is_valid_and_repacks():
    for K in (1, 3, 4, 8):
        tr = np.random.default_rng(K).integers(0, 65536, size=(3, 2, 16 * K), dtype=np.uint16)
        st = orc.unpack_states(tr, K)
        assert (orc.pack_states(st, K) == tr).all()


def test_codebook_statistics():
    # constants quoted by the reference: quantize.py:16 (1.24371088), SURVEY.md 0
    st = np.arange(65536, dtype=np.uint16)
    for cb, std in ((0, 1.24371088), (1, 1.2441), (2, 1.0003)):
        v = orc.decode_values(st, cb).astype(np.float64)
        assert abs(v.std() - std) < 2e-4
    # single known values: cb2(0) = fp16(1024*k_inv + k_bias)
    assert orc.decode_values(np.array([0], np.uint16), 2).view(np.uint16)[0] == 0xc2e8


def test_mul1_matches_reference_cpu_formula():
    # the reference's own scalar CPU decode (cpu/moe_mul1.cpp:174-179): (bytesum - 510) * k_inv in fp32;
    # differs from the GPU fp16 fma by at most the documented ~0.002 (SURVEY.md 0)
    st = np.arange(65536, dtype=np.uint64)
    x = (st * np.uint64(0x83DCD12D)) & np.uint64(0xffffffff)
    s = (x & 0xff) + ((x >> 8) & 0xff) + ((x >> 16) & 0xff) + (x >> 24)
    k_inv = float(np.array([0x1eee], np.uint16).view(np.float16)[0])
    cpu = (s.astype(np.float64) - 510.0) * k_inv
    gpu = orc.decode_values(st.astype(np.uint16), 2).astype(np.float64)
    assert np.abs(cpu - gpu).max() < 4e-3


def test_reconstruct_layout_against_scalar_walk():
    # independent slow restatement: per position t of tile (kt, nt): state by bit arithmetic on the MSB-first stream
    K, cb = 3, 0
    tr, _, _, _ = orc.make_synthetic(32, 128, K)
    w = orc.reconstruct(tr, K, cb)
    u = tr.view(np.uint16)
    perm = orc.tensor_core_perm()
    for (kt, nt) in ((0, 0), (1, 5)):
        words = u[kt, nt].view(np.uint32)
        bits = np.array([(int(words[i // 32]) >> (31 - i % 32)) & 1 for i in range(256 * K)])
        for t in (0, 1, 7, 100, 255):
            e = (t + 1) * K
            st = 0
            for b in range(e - 16, e):
                st = (st << 1) | int(bits[b % (256 * K)])
            v = orc.decode_values(np.array([st], np.uint16), cb)[0]
            r, c = divmod(int(perm[t]), 16)
            assert w[kt * 16 + r, nt * 16 + c] == v


def test_gemm_definition_consistency():
    # y == x @ W  with W = diag(suh) H W_hat H diag(svh)  (tests/test_reconstruct_had.py:70-95, tol 2e-2 there)
    K, cb = 4, 2
    tr, suh, svh, x = orc.make_synthetic(256, 128, K, m=5)
    y = orc.exl3_gemm_f64(x, tr, suh, svh, K, cb)
    W = orc.get_weight_tensor_f64(tr, suh, svh, K, cb)
    y2 = x.astype(np.float64) @ W
    assert np.abs(y - y2).max() <= 2e-3 * np.abs(y2).max()
    y16 = orc.exl3_gemm(x, tr, suh, svh, K, cb, np.float16).astype(np.float64)
    assert np.abs(y16 - y).max() <= 2e-3 * np.abs(y).max() + 1e-3


# ---- C restatement -------------------------------------------------------------------------------------------------

def _c_oracle():
    so = os.path.join(ROOT, "oracle", "libexl3oracle.so")
    src = os.path.join(ROOT, "oracle", "exl3_oracle.c")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "libexl3oracle.so"])
    lib = ctypes.CDLL(so)
    lib.exl3o_reconstruct.argtypes = [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5
    return lib


@pytest.mark.parametrize("K,cb", [(K, cb) for K in range(1, 9) for cb in range(3)])
def test_c_oracle_matches_numpy(K, cb):
    lib = _c_oracle()
    tr, _, _, _ = orc.make_synthetic(32, 128, K)
    out = np.empty((32, 128), dtype=np.float16)
    lib.exl3o_reconstruct(out.ctypes.data, tr.ctypes.data, 32, 128, K, cb, 2)
    assert (out.view(np.uint16) == orc.reconstruct(tr, K, cb).view(np.uint16)).all()


# ---- pinned against the reference's CUDA kernels (captured outputs) ------------------------------------------------

def _gpu_golden():
    p = os.path.join(GOLDEN, "ref_gpu.npz")
    if not os.path.exists(p):
        pytest.skip("tests/golden/ref_gpu.npz not generated yet (oracle/gen_golden_gpu.py on a GPU box)")
    return np.load(p)


def test_oracle_reconstruct_bitexact_vs_reference_cuda():
    g = _gpu_golden()
    for (K, cb, k, n) in gg.reconstruct_cases():
        tr, _, _, _ = orc.make_synthetic(k, n, K)
        assert gg.crc(tr) == g[f"rec_{K}_{cb}_{k}_{n}_crc"]
        ours = orc.reconstruct(tr, K, cb)
        assert (ours.view(np.uint16) == g[f"rec_{K}_{cb}_{k}_{n}"].view(np.uint16)).all(), (K, cb)


RECHAD_CASES = [(4, 2, 128, 384, 128, 256), (3, 0, 128, 256, 0, 256)]        # oracle/gen_golden_gpu.py: K, cb, k, n, column offset, columns


def test_reconstruct_had_vs_reference_cuda_golden():
    """The fused reconstruction as the reference's OWN kernel computed it: the fp64 restatement reproduces it within the
    reference's test bound (its kernel adds in fp16), and the fp32-sum model the CUDA kernels of this repo follow is closer to fp64
    than the reference's output is."""
    g = _gpu_golden()
    for (K, cb, k, n, off, nout) in RECHAD_CASES:
        tr, suh, svh, _ = orc.make_synthetic(k, n, K)
        gold = g[f"rechad_{K}_{cb}_{k}_{n}_{off}_{nout}"].astype(np.float64)
        f64 = orc.get_weight_tensor_f64(tr, suh, svh, K, cb)[:, off:off + nout]
        model = orc.reconstruct_had_fp32_model(tr[:, off // 16:(off + nout) // 16], suh, svh[off:off + nout], K, cb).astype(np.float64)
        mx = np.abs(f64).max()
        rms = lambda a: np.sqrt(((a - f64) ** 2).mean()) / np.sqrt((f64 ** 2).mean())
        assert np.abs(gold - f64).max() <= 2e-3 * mx                      # tests/test_reconstruct_had.py:56-58
        assert np.abs(model - f64).max() <= 1.2e-3 * mx
        assert np.abs(model - gold).max() <= 2.5e-3 * mx
        assert rms(model) < 0.6 * rms(gold) and rms(gold) < 1.2e-3


def test_oracle_had_bitexact_vs_reference_cuda():
    g = _gpu_golden()
    for (dt, mode, scale) in gg.had_cases():
        x, sc = gg.had_inputs(dt)
        ours = orc.had_r_128(x, sc if mode == "pre" else None, sc if mode == "post" else None, scale)
        ref = g[f"had_{dt}_{mode}_{scale}"]
        if dt == "f16":
            assert (ours.view(np.uint16) == ref.view(np.uint16)).all(), (dt, mode, scale)
        else:
            assert (ours.view(np.uint32) == ref.view(np.uint32)).all(), (dt, mode, scale)


def test_oracle_gemm_vs_reference_cuda():
    # xh bit-exact; outputs: reference accumulates on tensor cores in fp32 (order unspecified) and passes split-K
    # partials through C's dtype (exl3_gemm_inner.cuh:501-503,545-547) => tolerance, SURVEY.md 8(c)
    g = _gpu_golden()
    for (m, k, n, K, cb, fp32) in gg.gemm_cases():
        tr, suh, svh, x = orc.make_synthetic(k, n, K, m=m)
        key = f"gemm_{m}_{k}_{n}_{K}_{cb}_{int(fp32)}"
        assert gg.crc(tr, suh, svh, x) == g[key + "_crc"]
        y, xh = orc.exl3_gemm(x, tr, suh, svh, K, cb, np.float32 if fp32 else np.float16, return_xh=True)
        assert (xh.view(np.uint16) == g[key + "_xh"].view(np.uint16)).all(), key
        ref = g[key].astype(np.float64)
        err = np.abs(y.astype(np.float64) - ref)
        scale = np.abs(ref).max()
        rms = np.sqrt((err ** 2).mean()) / np.sqrt((ref ** 2).mean())
        assert err.max() <= 4e-3 * scale, (key, err.max() / scale)
        assert rms <= 2e-3, (key, rms)
