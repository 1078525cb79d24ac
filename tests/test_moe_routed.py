"""
Routed / weighted exl3_mgemm (the reference's MoE decode calls, modules/block_sparse_mlp.py:1362-1421) on the wgmma int8
path (csrc/gemm_tc_i8_routed.cu, tag 212), against the CPU oracle's restatement of the mgemm semantics
(exllamav3_ext/quant/exl3_gemm.cu:341-381) and against the verified default path (CUDA-core kernels, tag 100) on the same
inputs.

Routed mul1 calls at <= 4 rows take this path automatically; the tests also force it explicitly and compare with the CUDA-core twin (EXL3B_TAG_SIMT).
"""
import os
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc



def test_routed_tag_is_declared_and_distinct():
    from exllamav3_b200 import ext
    assert ext.EXL3B_TAG_TC_I8_ROUTED == 212
    assert len({ext.EXL3B_TAG_SIMT, ext.EXL3B_TAG_TC, ext.EXL3B_TAG_TC_I8, ext.EXL3B_TAG_TC_I8_AR, ext.EXL3B_TAG_TC_I8_ROUTED}) == 5
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "exl3b200.h")).read()
    assert "#define EXL3B_TAG_TC_I8_ROUTED 212" in hdr


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(y, ref):
    y = y.astype(np.float64); ref = ref.astype(np.float64)
    err = np.abs(y - ref)
    return err.max() / max(np.abs(ref).max(), 1e-30), np.sqrt((err ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def _setup(cuda, E, k, n, K, m, seed):
    mats = [orc.make_synthetic(k, n, K, seed=seed + 17 * e, m=m) for e in range(E)]
    trs = [T(t[0], cuda) for t in mats]; suhs = [T(t[1], cuda) for t in mats]; svhs = [T(t[2], cuda) for t in mats]
    ptr = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.long, device=cuda)
    return mats, (trs, suhs, svhs), (ptr(trs), ptr(suhs), ptr(svhs))


@pytest.mark.gpu
@pytest.mark.parametrize("K,m", [(4, 1), (3, 2), (6, 1), (4, 4)])
def test_routed_i8_mgemm_moe_modes(cuda, K, m):
    from exllamav3_b200 import ext
    E, k, n, topk = 8, 512, 384, 3
    mats, keep, (pt, ps, pv) = _setup(cuda, E, k, n, K, m, seed=500 + K)
    trl = [t[0] for t in mats]; sul = [t[1] for t in mats]; svl = [t[2] for t in mats]
    rng = np.random.default_rng(K * 10 + m)
    x1 = rng.standard_normal((1, m, k)).astype(np.float16)           # gate / up: one broadcast input
    xs = rng.standard_normal((topk, m, k)).astype(np.float16)        # down: one input per selected expert
    wts = rng.uniform(0.1, 1.0, topk).astype(np.float16)
    prev = ext.set_gemm_path(ext.EXL3B_TAG_TC_I8_ROUTED)
    try:
        for fp32 in (True, False):
            dt, npdt = (torch.float, np.float32) if fp32 else (torch.half, np.float16)
            tol = 2e-3 + (0 if fp32 else 2.0 ** -9)
            Ah = torch.empty((topk, m, k), dtype=torch.half, device=cuda)

            def run(A, idx, w, mn=-1, mx=-1, tables=(pt, ps, pv)):
                C = torch.zeros((topk, m, n), dtype=dt, device=cuda)
                it = torch.tensor([idx], dtype=torch.long, device=cuda)
                wt = None if w is None else T(w, cuda).view(1, -1)
                before = ext.launch_count()
                tag = ext.exl3_mgemm(T(A, cuda), tables[0], C, tables[1], Ah, tables[2], it, wt, K, -1, False, True, mn, mx, 0)
                torch.cuda.synchronize()
                return C.float().cpu().numpy(), tag, ext.launch_count() - before

            # (a) gate / up: selected experts, broadcast input, separate outputs: resolve + ONE tensor-core launch
            idx = [5, 0, 7]
            C, tag, nl = run(x1, idx, None)
            assert tag == ext.EXL3B_TAG_TC_I8_ROUTED and nl == 2
            ref = orc.exl3_mgemm(x1, trl, sul, svl, K, 2, npdt, indices=idx, bszm_out=topk)
            assert rel_err(C, ref)[0] <= tol
            # (b) a skipped slot (negative index) stays untouched
            idx = [2, -1, 4]
            C, tag, _ = run(x1, idx, None)
            ref = orc.exl3_mgemm(x1, trl, sul, svl, K, 2, npdt, indices=idx, bszm_out=topk)
            assert rel_err(C, ref)[0] <= tol and np.abs(C[1]).max() == 0.0
            # (c) down: per-slot inputs, routing weights, reduced into C[0] (resolve + GEMM + reduce)
            idx = [6, 1, 3]
            C, tag, nl = run(xs, idx, wts)
            assert tag == ext.EXL3B_TAG_TC_I8_ROUTED and nl == 3
            ref = orc.exl3_mgemm(xs, trl, sul, svl, K, 2, npdt, indices=idx, weights=wts, bszm_out=topk)
            assert rel_err(C[0], ref[0])[0] <= tol
            # (d) expert-parallel shard: experts [2, 6) live here, local pointer tables, other selections filtered out
            lo, hi = 2, 6
            sub = tuple(t[lo:hi].contiguous() for t in (pt, ps, pv))
            idx = [7, 3, 5]
            C, tag, _ = run(xs, idx, wts, lo, hi, sub)
            ref = orc.exl3_mgemm(xs, trl[lo:hi], sul[lo:hi], svl[lo:hi], K, 2, npdt, indices=idx, weights=wts,
                                 min_index=lo, max_index=hi, bszm_out=topk)
            assert rel_err(C[0], ref[0])[0] <= tol
            # (e) nothing selected on this shard: no slot is active, C[0] must come out as the empty sum
            C, tag, _ = run(xs, [0, 1, 7], wts, lo, hi, sub)
            assert np.abs(C[0]).max() == 0.0
            # same calls on the verified CUDA-core path agree (different arithmetic: fp16 codebook values there)
            ext.set_gemm_path(ext.EXL3B_TAG_SIMT)
            Cs, tag_s, _ = run(xs, [6, 1, 3], wts)
            assert tag_s == ext.EXL3B_TAG_SIMT
            ext.set_gemm_path(ext.EXL3B_TAG_TC_I8_ROUTED)
            Ct, _, _ = run(xs, [6, 1, 3], wts)
            assert rel_err(Ct[0], Cs[0])[0] <= 2 * tol
    finally:
        ext.set_gemm_path(prev)


@pytest.mark.gpu
def test_routed_i8_mgemm_mixtral_shapes_properties(cuda):
    """Mixtral expert shapes (BASELINE config 5), top-2 of 8: weighted down-projection is linear in the routing weights, and
    the routed result equals the single-matrix kernel's per-expert outputs combined on the host."""
    from exllamav3_b200 import ext
    E, k, n, K, m, topk = 8, 14336, 4096, 4, 1, 2
    mats, keep, (pt, ps, pv) = _setup(cuda, E, k, n, K, m, seed=900)
    rng = np.random.default_rng(1)
    xs = rng.standard_normal((topk, m, k)).astype(np.float16)
    idx = torch.tensor([[6, 2]], dtype=torch.long, device=cuda)
    Ah = torch.empty((topk, m, k), dtype=torch.half, device=cuda)
    prev = ext.set_gemm_path(ext.EXL3B_TAG_TC_I8_ROUTED)
    try:
        outs = []
        for w in ([0.5, 0.25], [1.0, 0.0], [0.0, 1.0]):
            C = torch.zeros((topk, m, n), dtype=torch.float, device=cuda)
            tag = ext.exl3_mgemm(T(xs, cuda), pt, C, ps, Ah, pv, idx, T(np.array(w, dtype=np.float16), cuda).view(1, 2), K, -1,
                                 False, True, -1, -1, 0)
            assert tag == ext.EXL3B_TAG_TC_I8_ROUTED
            outs.append(C[0].clone())
        torch.cuda.synchronize()
        lin = 0.5 * outs[1] + 0.25 * outs[2]
        assert float((outs[0] - lin).abs().max() / lin.abs().max()) < 1e-5
        ext.set_gemm_path(0)
        for j, e in enumerate((6, 2)):
            y = torch.empty((m, n), dtype=torch.float, device=cuda)
            ext.exl3_gemm(T(xs[j], cuda), keep[0][e], y, keep[1][e], torch.empty((m, k), dtype=torch.half, device=cuda), keep[2][e],
                          -1, False, True, 0)
            assert float((outs[1 + j] - y).abs().max() / y.abs().max()) < 1e-5
    finally:
        ext.set_gemm_path(prev)


@pytest.mark.gpu
@pytest.mark.parametrize("m,cb", [(8, 2), (32, 2), (1, 0), (17, 1)])
def test_mgemm_split_matches_fused_default(cuda, monkeypatch, m, cb):
    """EXL3B_MGEMM_SPLIT (ext.py): dense multi-matrix calls the int8 kernel cannot take, issued as one exact tensor-core exl3_gemm
    per matrix, against the default (CUDA-core multi-matrix kernels) and the fp64 oracle."""
    from exllamav3_b200 import ext
    k, n, K, nm = 512, 384, 4, 2
    mats = [orc.make_synthetic(k, n, K, seed=300 + 7 * e, m=m) for e in range(nm)]
    trs = [T(t[0], cuda) for t in mats]; suhs = [T(t[1], cuda) for t in mats]; svhs = [T(t[2], cuda) for t in mats]
    ptr = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.long, device=cuda)
    pt, ps, pv = ptr(trs), ptr(suhs), ptr(svhs)
    x = np.random.default_rng(m).standard_normal((1, m, k)).astype(np.float16)
    Ah = torch.empty((nm, m, k), dtype=torch.half, device=cuda)
    outs = {}
    for split in (False, True):
        monkeypatch.setattr(ext, "_MGEMM_SPLIT", split)
        C = torch.full((nm, m, n), float("nan"), dtype=torch.float, device=cuda)
        before = ext.launch_count()
        tag = ext.exl3_mgemm(T(x, cuda), pt, C, ps, Ah, pv, None, None, K, -1, cb == 1, cb == 2, -1, -1, 0)
        torch.cuda.synchronize()
        assert tag == (ext.EXL3B_TAG_TC if split else ext.EXL3B_TAG_SIMT)
        outs[split] = C.cpu().numpy()
    for j in range(nm):
        ref = orc.exl3_gemm_f64(x[0], mats[j][0], mats[j][1], mats[j][2], K, cb)
        for split in (False, True):
            mx, rms = rel_err(outs[split][j], ref)
            assert mx <= 2e-3 and rms <= 1e-3, (split, j, mx, rms)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [5, 8])
def test_dense_mgemm_i8_eight_row_variant(cuda, m):
    """The 8-row instantiation of the int8 kernel (verified for single matrices, test_gpu_parity.py::test_gemm_i8_tensor_core_path)
    in its multi-matrix mode (verified for <= 4 rows): the combination is what a batch-5..8 decode step's fused k+v / gate+up
    would use if exl3b_mgemm auto-selected tag 210 up to 8 rows instead of falling back to the CUDA-core kernels."""
    from exllamav3_b200 import ext
    k, n, K, nm = 1024, 384, 4, 2
    mats, keep, (pt, ps, pv) = _setup(cuda, nm, k, n, K, m, seed=40 + m)
    x = np.random.default_rng(m).standard_normal((1, m, k)).astype(np.float16)
    Ah = torch.empty((nm, m, k), dtype=torch.half, device=cuda)
    prev = ext.set_gemm_path(ext.EXL3B_TAG_TC_I8)
    try:
        C = torch.full((nm, m, n), float("nan"), dtype=torch.float, device=cuda)
        before = ext.launch_count()
        tag = ext.exl3_mgemm(T(x, cuda), pt, C, ps, Ah, pv, None, None, K, -1, False, True, -1, -1, 0)
        torch.cuda.synchronize()
        assert tag == ext.EXL3B_TAG_TC_I8 and ext.launch_count() - before == 1
        for j in range(nm):
            ref = orc.exl3_gemm_f64(x[0], mats[j][0], mats[j][1], mats[j][2], K, 2)
            mx, rms = rel_err(C[j].cpu().numpy(), ref)
            assert mx <= 2e-3 and rms <= 1e-3, (j, mx, rms)
    finally:
        ext.set_gemm_path(prev)
