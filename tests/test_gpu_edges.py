"""
Decode-GEMM kernels at the geometry edges (H100): every template instantiation, every accumulator row group and pass count,
forced persistent grids that produce every split-K pattern, the uncached int8 activations, the int32 accumulation chunks at
their worst case and CUDA-graph replay.  Which branch each shape reaches is asserted on the host
in tests/test_edges_host.py, which also holds the shared tables and input builders.  The oracle is given each decoded weight
(exl3_gemm_f64's w, exl3_gemm_i8_model's bsum) so that it decodes once per matrix, not once per call.

Every call writes into the middle rows of a larger C filled with a sentinel bit pattern and reads A through a view whose
trailing rows are NaN: the rows around the output must keep their bits and every valid output must stay finite.

Bars (README.md, Parity): vs oracle.exl3_gemm_f64 max-abs <= 2e-3 max|y| (+1 fp16 ulp), rel-RMS <= 1e-3; the int8 path vs its
exact model oracle.exl3_gemm_i8_model max-abs <= 2e-5 max|y|, rel-RMS <= 1e-5 (fp32 C), 1.5e-3 / 5e-4 (fp16 C); tags 100 and 200
vs their exact model oracle.exl3_gemm_f16_model with test_edges_host.check_f16_gemm.
"""
import contextlib
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc
from test_edges_host import CACHE_PAIRS, FORCED_GRIDS, WORST_KQ, check_f16_gemm, gemm_plan, worst_case_inputs

pytestmark = pytest.mark.gpu

TAG_SIMT, TAG_TC, TAG_I8, TAG_CHAIN = 100, 200, 210, 220
SENTINEL = {torch.half: (torch.int16, 0x7E5A), torch.float: (torch.int32, 0x7FA5A5A5)}     # NaN payloads nobody writes


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(y, ref):
    y = y.astype(np.float64); ref = ref.astype(np.float64)
    err = np.abs(y - ref)
    return err.max() / max(np.abs(ref).max(), 1e-30), np.sqrt((err ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def check_f64(y, ref, fp32, what):
    mx, rms = rel_err(y, ref)
    assert mx <= 2e-3 + (0.0 if fp32 else 2.0 ** -10) and rms <= 1e-3, (what, fp32, mx, rms)


def check_model(y, ref, fp32, what):
    mx, rms = rel_err(y, ref)
    assert mx <= (2e-5 if fp32 else 1.5e-3) and rms <= (1e-5 if fp32 else 5e-4), (what, fp32, mx, rms)


@contextlib.contextmanager
def gemm_path(tag):
    from exllamav3_b200 import ext
    prev = ext.set_gemm_path(tag)
    try:
        yield
    finally:
        ext.set_gemm_path(prev)


class Mat:
    """One quantized matrix on the host and on the device."""

    def __init__(self, dev, tr, suh, svh, K, cb):
        self.tr, self.suh, self.svh, self.K, self.cb = tr, suh, svh, K, cb
        self.k, self.n = tr.shape[0] * 16, tr.shape[1] * 16
        self.d_tr, self.d_suh, self.d_svh = T(tr, dev), T(suh, dev), T(svh, dev)

    def cols(self, dev, n):
        """The first n output columns as a matrix of its own."""
        return Mat(dev, self.tr[:, :n // 16], self.suh, self.svh[:n], self.K, self.cb)


def launch(ext, dev, x, mt, fp32, force=0):
    """exl3_gemm into rows 1..m of a sentinel-filled (m + 2, n) C, from rows 0..m-1 of an A whose trailing rows are NaN."""
    m, k = x.shape
    A = torch.full((m + 3, k), float("nan"), dtype=torch.half, device=dev)
    A[:m] = T(x, dev)
    dt = torch.float if fp32 else torch.half
    C = torch.empty((m + 2, mt.n), dtype=dt, device=dev)
    C.view(SENTINEL[dt][0]).fill_(SENTINEL[dt][1])
    tag = ext.exl3_gemm(A[:m], mt.d_tr, C[1:m + 1], mt.d_suh, torch.empty((m, k), dtype=torch.half, device=dev), mt.d_svh,
                        -1, mt.cb == 1, mt.cb == 2, force)
    return C, tag


def finish(C, what):
    """Canary checks after the launch; returns the m valid rows as float64."""
    torch.cuda.synchronize()
    itype, bits = SENTINEL[C.dtype]
    raw = C.view(itype).cpu().numpy()
    assert (raw[0] == bits).all() and (raw[-1] == bits).all(), ("rows outside C written", what)
    y = C[1:-1].double().cpu().numpy()
    assert np.isfinite(y).all(), ("non-finite output", what)
    return y


def run(ext, dev, x, mt, fp32, force=0):
    C, tag = launch(ext, dev, x, mt, fp32, force)
    return finish(C, (x.shape, mt.k, mt.n, mt.K, mt.cb, fp32, force)), tag


# ---- 1. every (K, codebook) instantiation ------------------------------------------------------------------------------

@pytest.mark.parametrize("path", [TAG_TC, TAG_SIMT])
@pytest.mark.parametrize("cb", range(3))
@pytest.mark.parametrize("K", range(1, 9))
def test_every_instantiation(cuda, K, cb, path):
    """gemm_tc_kernel<K, cb> (tag 200) and its CUDA-core twin (tag 100) for all 24 pairs; k = 128 is a single k-block."""
    from exllamav3_b200 import ext
    with gemm_path(path):
        for (k, n) in ((512, 384), (128, 1024)):
            tr, suh, svh, x = orc.make_synthetic(k, n, K, m=17, seed=100 * K + 10 * cb + k // 128)
            mt = Mat(cuda, tr, suh, svh, K, cb)
            w = orc.reconstruct(tr, K, cb)
            for m in (1, 17):
                ref = orc.exl3_gemm_f64(x[:m], tr, suh, svh, K, cb, w=w)
                for fp32 in (False, True):
                    y, tag = run(ext, cuda, x[:m], mt, fp32)
                    assert tag == path
                    check_f64(y, ref, fp32, (K, cb, k, n, m))
                    check_f16_gemm(y, x[:m], tr, suh, svh, K, cb, fp32, (K, cb, k, n, m), w=w)


_RECON_HAD_COVERED = {(1, 0), (2, 1), (3, 2), (4, 2), (5, 0), (6, 2), (7, 1), (8, 2)}       # test_gpu_parity.py


@pytest.mark.parametrize("K,cb", sorted({(K, cb) for K in range(1, 9) for cb in range(3)} - _RECON_HAD_COVERED))
def test_reconstruct_had_remaining_instantiations(cuda, K, cb):
    """The (K, cb) pairs of reconstruct_had that test_reconstruct_had_tensor_core_and_cuda_core_twins does not run, same bars."""
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
            w2 = torch.empty((k, 384), dtype=torch.half, device=cuda)
            ext.reconstruct_had_slice(w2, T(tr, cuda), T(suh, cuda), T(svh[256:640], cuda), K, cb == 1, cb == 2, 256)
            assert torch.equal(w2.cpu(), w[:, 256:640].cpu())
    finally:
        ext.lib.exl3b_debug_reconstruct_had(0)
    ref = orc.get_weight_tensor_f64(tr[:16], suh[:256], svh, K, cb)
    for mode in outs:
        assert np.isfinite(outs[mode]).all()
        assert np.abs(outs[mode][:256] - ref).max() / np.abs(ref).max() < 2e-3, mode
    d = np.abs(outs[1] - outs[2])
    assert d.max() <= 4e-3 * np.abs(outs[1]).max()
    assert (d > 0).mean() < 0.05


# ---- 2. rows across accumulator row groups and passes -------------------------------------------------------------------

SWEEP_ROWS = (1, 8, 9, 15, 16, 17, 31, 33, 48, 49, 64, 65, 80, 95, 97, 112, 113, 127, 128, 129, 143, 256, 257)


@pytest.mark.parametrize("K,cb", [(4, 2), (3, 0), (8, 1)])
def test_row_sweep_exact_path(cuda, K, cb):
    """Every NT = 16 .. 128 of a pass, and one, two and three passes (C and A offsets of later passes)."""
    from exllamav3_b200 import ext
    k, n = 512, 256
    tr, suh, svh, x = orc.make_synthetic(k, n, K, m=max(SWEEP_ROWS), seed=300 + K)
    mt = Mat(cuda, tr, suh, svh, K, cb)
    w = orc.reconstruct(tr, K, cb)
    with gemm_path(TAG_TC):
        for m in SWEEP_ROWS:
            ref = orc.exl3_gemm_f64(x[:m], tr, suh, svh, K, cb, w=w)
            for fp32 in (False, True):
                y, tag = run(ext, cuda, x[:m], mt, fp32)
                assert tag == TAG_TC
                check_f64(y, ref, fp32, (K, cb, m))
                check_f16_gemm(y, x[:m], tr, suh, svh, K, cb, fp32, (K, cb, m), w=w)


def test_canaries_int8_and_cuda_core_paths(cuda):
    from exllamav3_b200 import ext
    k, n = 512, 256
    tr, suh, svh, x = orc.make_synthetic(k, n, 4, m=130, seed=310)
    mt = Mat(cuda, tr, suh, svh, 4, 2)
    w, bs = orc.reconstruct(tr, 4, 2), orc.mul1_bytesum(tr, 4)
    with gemm_path(TAG_I8):                               # rows 5..8 exist on the int8 path only when forced
        for m in range(1, 9):
            ref = orc.exl3_gemm_f64(x[:m], tr, suh, svh, 4, 2, w=w)
            model = orc.exl3_gemm_i8_model(x[:m], tr, suh, svh, 4, bsum=bs)
            for fp32 in (False, True):
                y, tag = run(ext, cuda, x[:m], mt, fp32)
                assert tag == TAG_I8
                check_model(y, model, fp32, m)
                check_f64(y, ref, fp32, m)
    tr, suh, svh, _ = orc.make_synthetic(k, n, 3, seed=311)
    mt = Mat(cuda, tr, suh, svh, 3, 0)
    w = orc.reconstruct(tr, 3, 0)
    with gemm_path(TAG_SIMT):
        for m in (1, 9, 33, 130):
            ref = orc.exl3_gemm_f64(x[:m], tr, suh, svh, 3, 0, w=w)
            for fp32 in (False, True):
                y, tag = run(ext, cuda, x[:m], mt, fp32)
                assert tag == TAG_SIMT
                check_f64(y, ref, fp32, m)
                check_f16_gemm(y, x[:m], tr, suh, svh, 3, 0, fp32, m, w=w)


# ---- 3. forced persistent grids ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k,n,grids", FORCED_GRIDS)
def test_forced_grids_exact_path(cuda, k, n, grids):
    """Tag 200 on every split pattern of the table: against the oracle, and bit-identical when repeated with the same grid."""
    from exllamav3_b200 import ext
    with gemm_path(TAG_TC):
        for cb in (2, 0):
            tr, suh, svh, x = orc.make_synthetic(k, n, 4, m=130, seed=400 + cb)
            mt = Mat(cuda, tr, suh, svh, 4, cb)
            w = orc.reconstruct(tr, 4, cb)
            for m in (1, 17, 130):
                ref = orc.exl3_gemm_f64(x[:m], tr, suh, svh, 4, cb, w=w)
                for G in grids:
                    assert gemm_plan(m, k, n, 4, cb, force=G).grid == G
                    y, tag = run(ext, cuda, x[:m], mt, False, force=G)
                    assert tag == TAG_TC
                    check_f64(y, ref, False, (cb, m, G))
                    check_f16_gemm(y, x[:m], tr, suh, svh, 4, cb, False, (cb, m, G), w=w)
                    y1, _ = run(ext, cuda, x[:m], mt, True, force=G)
                    y2, _ = run(ext, cuda, x[:m], mt, True, force=G)
                    assert np.array_equal(y1, y2), (cb, m, G)
                    check_f64(y1, ref, True, (cb, m, G))
                    check_f16_gemm(y1, x[:m], tr, suh, svh, 4, cb, True, (cb, m, G), w=w)


@pytest.mark.parametrize("k,n,grids", FORCED_GRIDS)
def test_forced_grids_int8_path(cuda, k, n, grids):
    """
    Tag 210 on every split pattern of the table, launched back to back without synchronisation and interleaved with default-grid
    launches of other shapes (the pattern of test_i8_split_k_exchange_ring): forced-grid and default-grid launches share the
    rotating exchange-buffer slots, so a slot left un-armed by either would corrupt the other.
    """
    from exllamav3_b200 import ext
    tr, suh, svh, x = orc.make_synthetic(k, n, 4, m=4, seed=500)
    mt = Mat(cuda, tr, suh, svh, 4, 2)
    w, bs = orc.reconstruct(tr, 4, 2), orc.mul1_bytesum(tr, 4)
    ring = []
    for (rk, rn, rm) in ((16384, 128, 1), (4096, 256, 3), (2048, 1024, 4), (128, 2048, 1)):
        rtr, rsuh, rsvh, rx = orc.make_synthetic(rk, rn, 4, m=rm)
        ring.append((rx, Mat(cuda, rtr, rsuh, rsvh, 4, 2)))
    first = [run(ext, cuda, rx, rmt, True)[0] for (rx, rmt) in ring]
    pending, ring_out = [], []
    for m in (1, 4):
        for G in grids:
            assert gemm_plan(m, k, n, 4, 2, force=G).grid == G
            for (fp32, rep) in ((True, 0), (True, 1), (False, 0)):         # fp32 twice: the repeat must be bit-identical
                pending.append(((m, G, fp32, rep),) + launch(ext, cuda, x[:m], mt, fp32, force=G))
                i = len(ring_out) % len(ring)
                ring_out.append((i,) + launch(ext, cuda, ring[i][0], ring[i][1], True))
    for (i, C, tag) in ring_out:
        assert tag == TAG_I8
        assert np.array_equal(finish(C, ("ring", i)), first[i]), i
    ys = {}
    for ((m, G, fp32, rep), C, tag) in pending:
        assert tag == TAG_I8
        y = finish(C, (m, G, fp32))
        if fp32:
            ys[(m, G, rep)] = y
        if rep:
            assert np.array_equal(y, ys[(m, G, 0)]), (m, G)
        check_model(y, orc.exl3_gemm_i8_model(x[:m], tr, suh, svh, 4, bsum=bs), fp32, (m, G))
        check_f64(y, orc.exl3_gemm_f64(x[:m], tr, suh, svh, 4, 2, w=w), fp32, (m, G))


# ---- 4. uncached int8 activations ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", (2, 4, 6))
def test_int8_both_sides_of_the_activation_cache(cuda, K):
    """(m, k) pairs just inside and just outside the 64 KiB activation cache, incl. a zero row and a row scaled by 100."""
    from exllamav3_b200 import ext
    for (m, k, cached) in CACHE_PAIRS:
        tr, suh, svh, x = orc.make_synthetic(k, 384, K, m=m, seed=600 + K)
        full = Mat(cuda, tr, suh, svh, K, 2)
        w, bs = orc.reconstruct(tr, K, 2), orc.mul1_bytesum(tr, K)
        if m >= 2:
            xz = x.copy(); xz[1] = 0; xz[-1 if m > 2 else 0] *= np.float16(100.0)
            variants = [x, xz]
        else:
            variants = [x, np.zeros_like(x), x * np.float16(100.0)]
        for n in (128, 384):
            mt = full.cols(cuda, n)
            for xv in variants:
                model = orc.exl3_gemm_i8_model(xv, mt.tr, suh, mt.svh, K, bsum=bs[:, :n])
                ref = orc.exl3_gemm_f64(xv, mt.tr, suh, mt.svh, K, 2, w=w[:, :n])
                for fp32 in (True, False):
                    y, tag = run(ext, cuda, xv, mt, fp32)
                    assert tag == TAG_I8
                    for r in range(m):
                        what = (m, k, cached, n, K, r, fp32)
                        if not xv[r].any():
                            assert not y[r].any(), what
                        else:
                            check_model(y[r:r + 1], model[r:r + 1], fp32, what)
                            check_f64(y[r:r + 1], ref[r:r + 1], fp32, what)


def test_int8_uncached_dense_mgemm(cuda):
    """Two matrices sharing an uncached input (m = 4, k = 8320): one launch of the int8 kernel."""
    from exllamav3_b200 import ext
    k, n, K, m = 8320, 256, 4, 4
    mats = [orc.make_synthetic(k, n, K, seed=700 + j, m=m) for j in range(2)]
    x = mats[0][3]
    trs = [T(t[0], cuda) for t in mats]; suhs = [T(t[1], cuda) for t in mats]; svhs = [T(t[2], cuda) for t in mats]
    ptr = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.long, device=cuda)
    for fp32 in (True, False):
        C = torch.full((2, m, n), float("nan"), dtype=torch.float if fp32 else torch.half, device=cuda)
        before = ext.launch_count()
        tag = ext.exl3_mgemm(T(x, cuda).view(1, m, k), ptr(trs), C, ptr(suhs), torch.empty((2, m, k), dtype=torch.half, device=cuda),
                             ptr(svhs), None, None, K, -1, False, True, -1, -1, 0)
        assert tag == TAG_I8 and ext.launch_count() - before == 1
        torch.cuda.synchronize()
        Cn = C.double().cpu().numpy()
        for j, (tr, suh, svh, _) in enumerate(mats):
            check_model(Cn[j], orc.exl3_gemm_i8_model(x, tr, suh, svh, K), fp32, j)
            check_f64(Cn[j], orc.exl3_gemm_f64(x, tr, suh, svh, K, 2), fp32, j)


# ---- 5. worst-case int32 accumulation ------------------------------------------------------------------------------------

def test_int8_worst_case_int32_accumulation(cuda):
    """
    Every u8 x s8 product of a column has the same sign and one CTA walks the whole 640-block strip: an accumulator that is not
    handed to the epilogue every 96 units wraps (the sharpness of this input is asserted in test_edges_host.py).
    """
    from exllamav3_b200 import ext
    tr, suh, svh, x = worst_case_inputs(4)
    mt = Mat(cuda, tr, suh, svh, WORST_KQ, 2)
    w, bs = orc.reconstruct(tr, WORST_KQ, 2), orc.mul1_bytesum(tr, WORST_KQ)
    for m in (1, 4):
        model = orc.exl3_gemm_i8_model(x[:m], tr, suh, svh, WORST_KQ, bsum=bs)
        ref = orc.exl3_gemm_f64(x[:m], tr, suh, svh, WORST_KQ, 2, w=w)
        for force in (1, 0):
            y, tag = run(ext, cuda, x[:m], mt, True, force=force)
            assert tag == TAG_I8
            check_model(y, model, True, (m, force))
        # the chain kernel (tag 220) accumulates in chunks of its own; its activation scale rule differs from the int8
        # kernel's, so it is held to the oracle bar
        with gemm_path(TAG_CHAIN):
            y, tag = run(ext, cuda, x[:m], mt, True, force=1)
        assert tag == TAG_CHAIN
        check_f64(y, ref, True, (m, "chain"))


# ---- 6. CUDA-graph replay ------------------------------------------------------------------------------------------------

def test_graph_replay_matches_eager(cuda):
    """
    A three-pass tag-200 call and cached / uncached tag-210 calls, each captured on its own stream and replayed three times with new
    inputs copied into the captured buffers and eager calls of other shapes in between: every replay equals the eager call on the
    same input bit for bit (self-resetting split-K counters, re-armed exchange slots).
    """
    from exllamav3_b200 import ext
    rng = np.random.default_rng(9)
    cases = []
    for (m, k, n, tag) in ((300, 512, 256, TAG_TC), (1, 4096, 256, TAG_I8), (4, 8320, 256, TAG_I8)):
        tr, suh, svh, _ = orc.make_synthetic(k, n, 4, seed=900 + m)
        mt = Mat(cuda, tr, suh, svh, 4, 2)
        xs = [rng.standard_normal((m, k)).astype(np.float16) for _ in range(3)]
        A = T(xs[0], cuda)
        Ah = torch.empty_like(A)
        C = torch.empty((m, n), dtype=torch.float, device=cuda)
        gemm = lambda A=A, mt=mt, C=C, Ah=Ah: ext.exl3_gemm(A, mt.d_tr, C, mt.d_suh, Ah, mt.d_svh, -1, False, True, 0)
        assert gemm() == tag                              # eager first: kernel attributes and tensor maps outside capture
        torch.cuda.synchronize()
        st = torch.cuda.Stream()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.stream(st):
            with torch.cuda.graph(gr, stream=st):
                assert gemm() == tag
        cases.append(dict(mt=mt, xs=xs, A=A, C=C, st=st, gr=gr, tag=tag))
    others = []
    for (m, k, n, force) in ((2, 2048, 512, 0), (20, 512, 256, 0), (1, 1152, 1152, 7), (3, 4096, 128, 31)):
        tr, suh, svh, x = orc.make_synthetic(k, n, 4, m=m, seed=950 + m)
        others.append((x, Mat(cuda, tr, suh, svh, 4, 2), force))
    for rnd in range(3):
        for c in cases:
            c["A"].copy_(T(c["xs"][rnd], cuda))
            torch.cuda.synchronize()
            with torch.cuda.stream(c["st"]):
                c["gr"].replay()
            c["st"].synchronize()
            got = c["C"].clone()
            for (x, mt, force) in others:
                launch(ext, cuda, x, mt, True, force)
            y, tag = run(ext, cuda, c["xs"][rnd], c["mt"], True)
            assert tag == c["tag"]
            assert np.array_equal(got.double().cpu().numpy(), y), (rnd, c["tag"], c["xs"][0].shape)
            if c["tag"] == TAG_TC:
                mt = c["mt"]
                check_f16_gemm(y, c["xs"][rnd], mt.tr, mt.suh, mt.svh, 4, 2, True, ("replay", rnd))
