"""
C-ABI checks that need no GPU: libexl3b200.so loads, exports every symbol include/exl3b200.h declares, and its
argument validation (the reference's TORCH_CHECKs) fires before any CUDA work.  No compute is attempted.
"""
import ctypes, os, re
import numpy as np
import pytest
import torch
from conftest import ROOT


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "exl3b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(exl3b_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from exllamav3_b200 import ext
    syms = _declared_symbols()
    assert len(syms) >= 12
    for s in syms:
        assert hasattr(ext.lib, s), f"{s} declared in include/exl3b200.h but not exported"
    assert ext.lib.exl3b_abi_version() == 1


def test_validation_errors_without_gpu():
    from exllamav3_b200 import ext
    lib = ext.lib
    one = ctypes.c_void_p(16)      # never dereferenced: validation fails first
    # K out of range
    assert lib.exl3b_gemm(None, one, one, one, one, one, one, 1, 128, 128, 9, 0, 0, -1, 0) == -2
    assert b"K must be 1..8" in lib.exl3b_last_error()
    # n not divisible by 128  (exl3_gemm.cu:37-39 "n % 128 == 0")
    assert lib.exl3b_gemm(None, one, one, one, one, one, one, 1, 128, 64, 4, 0, 0, -1, 0) == -1
    assert b"divisible by 128" in lib.exl3b_last_error()
    # reconstruct: offsets (reconstruct.cu:117-120)
    assert lib.exl3b_reconstruct(None, one, one, 16, 128, 8, 4, 0, 64) == -1
    assert b"n_offset must be divisible by 128" in lib.exl3b_last_error()
    assert lib.exl3b_reconstruct(None, one, one, 16, 256, 8, 4, 0, 0) == -1
    assert b"exceeds packed tensor bounds" in lib.exl3b_last_error()
    # had_r_128 (hadamard.cu:101)
    assert lib.exl3b_had_r_128(None, one, one, None, None, 1.0, 1, 100, 0) == -1
    # mgemm argument rules (exl3_gemm.cu:408-410,441-446)
    r = lib.exl3b_mgemm(None, one, one, one, one, one, one, one, 2, None, 1, 2, 1, 128, 128, 4, 0, 0,
                        0, 1, 2, None, None, 0, -1, 0)
    assert r == -2 and b"num_tokens > 1" in lib.exl3b_last_error()
    # empty problems are no-ops, not errors
    assert lib.exl3b_gemm(None, None, None, None, None, None, None, 0, 128, 128, 4, 0, 0, -1, 0) == 0


def test_python_surface_rejects_cpu_tensors_and_bad_dtypes():
    from exllamav3_b200 import ext
    a = torch.zeros(1, 128, dtype=torch.half)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ext.had_r_128(a, a, None, None, 1.0)
    with pytest.raises(RuntimeError, match="no CPU path"):
        ext.exl3_gemm(a, torch.zeros(8, 8, 64, dtype=torch.int16), torch.zeros(1, 128, dtype=torch.half),
                      None, None, None, -1, False, True, 0)


def test_reference_named_surface_is_complete():
    # every binding of exllamav3_ext the qgemm path uses (SURVEY.md 8b)
    from exllamav3_b200 import ext
    for name in ["exl3_gemm", "exl3_mgemm", "reconstruct", "reconstruct_slice", "reconstruct_had_slice",
                 "had_r_128", "hgemm", "BC_LinearEXL3", "g_get_cc", "g_get_num_sms",
                 "exl3_gemm_num_kernel_shapes", "exl3_gemm_shape_compat", "exl3_gemv_int8_max_k", "exl3_gemv"]:
        assert hasattr(ext, name), name


def test_use_mgemm_policy_through_the_shim():
    """model/config.py:48-64 (use_mgemm): for mul1 tensors the reference fuses k+v / gate+up into one exl3_mgemm iff
    K >= ext.exl3_gemv_int8_max_k(device) + 1 or the output is narrow.  The shim reports 0 => fused for every K."""
    from exllamav3_b200 import ext
    import inspect
    src = inspect.getsource(ext.exl3_gemv_int8_max_k)
    assert "return 0" in src
    k_thr = 0 + 1
    assert all(K >= k_thr for K in range(1, 9))


def test_linear_exl3_tp_slice_host_logic():
    # slicing rules of LinearEXL3.tp_import_split (modules/quant/exl3.py:284-330) on CPU tensors: no kernels run
    from exllamav3_b200 import QLinear, tp
    from oracle import exl3_oracle as orc
    k, n, K = 256, 384, 3
    tr, suh, svh, _ = orc.make_synthetic(k, n, K)
    bias = torch.arange(n, dtype=torch.half)
    lin = QLinear(torch.from_numpy(tr), torch.from_numpy(suh), torch.from_numpy(svh), mul1=True, bias=bias)
    col = tp.tp_slice(lin, (True, 128, 384))
    assert col.in_features == k and col.out_features == 256
    assert torch.equal(col.trellis, lin.trellis[:, 8:24, :]) and torch.equal(col.svh, lin.svh[128:384])
    assert torch.equal(col.suh, lin.suh) and torch.equal(col.bias, bias[128:384]) and col.mul1 and not col.mcg
    row0 = tp.tp_slice(lin, (False, 0, 128)); row1 = tp.tp_slice(lin, (False, 128, 256))
    assert row0.in_features == 128 and row0.out_features == n
    assert torch.equal(row1.trellis, lin.trellis[8:16]) and torch.equal(row1.suh, lin.suh[128:256])
    assert row0.bias is not None and row1.bias is None            # bias only on the shard with first == 0
    assert row0.bias_in_group and row1.bias_in_group and col.bias_in_group     # ... but every shard knows the group has one
    assert col.trellis.is_contiguous() and row1.trellis.is_contiguous()


def test_mgemm_split_host_logic(monkeypatch):
    """EXL3B_MGEMM_SPLIT: a dense exl3_mgemm the int8 kernel cannot take becomes one exl3b_gemm per matrix with the right
    pointers (tables read back once per tensor object, cache invalidated by modification).  Recording stand-in, no kernels."""
    import contextlib
    from exllamav3_b200 import ext
    calls = []

    class FakeLib:
        def exl3b_gemm(self, stream, A, B, C, suh, A_had, svh, m, k, n, K, cb, c_fp32, fsi, fns):
            calls.append(("gemm", A, B, C, suh, A_had, svh, m, k, n, K, cb, c_fp32)); return 200
        def exl3b_mgemm(self, *a):
            calls.append(("mgemm",)); return 100
        def exl3b_last_error(self): return b""

    monkeypatch.setattr(ext, "_lib", FakeLib())
    monkeypatch.setattr(ext, "_need_cuda", lambda *a: None)
    monkeypatch.setattr(ext, "_stream", lambda t: 0)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(ext, "_MGEMM_SPLIT", True)
    m, k, n, K = 8, 256, 384, 4
    A = torch.zeros((1, m, k), dtype=torch.half); C = torch.zeros((2, m, n), dtype=torch.float)
    Ah = torch.zeros((2, m, k), dtype=torch.half)
    B = torch.tensor([1000, 2000]); su = torch.tensor([3000, 4000]); sv = torch.tensor([5000, 6000])
    tag = ext.exl3_mgemm(A, B, C, su, Ah, sv, None, None, K, -1, False, True, -1, -1, 0)      # mul1 but 8 rows -> split
    assert tag == 200 and [c[0] for c in calls] == ["gemm", "gemm"]
    g0, g1 = calls
    assert g0[1] == g1[1] == A.data_ptr()                                   # shared input
    assert (g0[2], g0[4], g0[6]) == (1000, 3000, 5000) and (g1[2], g1[4], g1[6]) == (2000, 4000, 6000)
    assert g1[3] - g0[3] == m * n * 4 and g1[5] - g0[5] == m * k * 2        # C[j], A_had[j]
    assert g0[7:] == (m, k, n, K, 2, 1)
    # table modified in place -> re-read
    calls.clear(); B[1] = 2222
    ext.exl3_mgemm(A, B, C, su, Ah, sv, None, None, K, -1, False, True, -1, -1, 0)
    assert calls[1][2] == 2222
    # per-matrix inputs; 3INST codebook at one row also splits (the int8 kernel is mul1 only)
    calls.clear()
    A2 = torch.zeros((2, 1, k), dtype=torch.half); C2 = torch.zeros((2, 1, n), dtype=torch.half)
    ext.exl3_mgemm(A2, B, C2, su, Ah, sv, None, None, K, -1, False, False, -1, -1, 0)
    assert [c[0] for c in calls] == ["gemm", "gemm"] and calls[1][1] - calls[0][1] == k * 2 and calls[0][11] == 0 and calls[0][12] == 0
    # what stays on exl3b_mgemm: int8-eligible calls, routed calls, and everything when the switch is off
    calls.clear()
    ext.exl3_mgemm(A[:, :4], B, C[:, :4], su, Ah, sv, None, None, K, -1, False, True, -1, -1, 0)
    idx = torch.zeros((1, 2), dtype=torch.long)
    ext.exl3_mgemm(A, B, C, su, Ah, sv, idx, None, K, -1, False, True, -1, -1, 0)
    monkeypatch.setattr(ext, "_MGEMM_SPLIT", False)
    ext.exl3_mgemm(A, B, C, su, Ah, sv, None, None, K, -1, False, True, -1, -1, 0)
    assert [c[0] for c in calls] == ["mgemm", "mgemm", "mgemm"]
    # the cache does not outlive the tensor
    n_before = len(ext._table_cache); del B, su, sv
    import gc; gc.collect()
    assert len(ext._table_cache) <= n_before - 3


def test_force_shape_idx_validation_without_gpu():
    """force_shape_idx selects the kernel per call like the reference's (1 = CUDA-core twin, 2 = exact tensor-core kernel); an index
    beyond exl3_gemm_num_kernel_shapes() is an argument error raised before any CUDA work."""
    from exllamav3_b200 import ext
    one = ctypes.c_void_p(16)
    assert ext.exl3_gemm_num_kernel_shapes() == 2
    assert ext.lib.exl3b_gemm(None, one, one, one, one, one, one, 1, 128, 128, 4, 2, 0, 3, 0) == -2
    assert b"force_shape_idx 3 out of range" in ext.lib.exl3b_last_error()
    assert ext.exl3_gemm_shape_compat(1, 1, 4096, 4096, 4) and ext.exl3_gemm_shape_compat(2, 32, 4096, 4096, 4)
    assert not ext.exl3_gemm_shape_compat(3, 1, 4096, 4096, 4) and not ext.exl3_gemm_shape_compat(1, 1, 4000, 4096, 4)
