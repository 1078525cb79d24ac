"""
Host logic of the tensor-core launchers, checked WITHOUT a GPU through exl3b_gemm_plan / exl3b_plan_* (the same functions the
launchers call): path selection, shared-memory / workspace budgets and the persistent stream-K partition, for every
shape of BASELINE.json's configs -- Llama-3.1-8B and 70B, their tensor-parallel shards at 2/4/8 ranks (SURVEY.md 8d) and
the Mixtral expert shapes -- and every bitrate, i.e. also for shapes no GPU test runs at full size.

The partition invariants are what the kernels' split-K combine relies on (gemm_tc_i8_body.cuh epilogue, gemm_tc.cu):
  * every 128x128 unit belongs to exactly one CTA, ranges are contiguous and non-empty (grid <= units);
  * cta_of_unit inverts unit_begin; the CTAs contributing to a column strip are the contiguous range
    [cta_of_unit(first unit), cta_of_unit(last unit)], and the first of them is the one that meets the strip LAST in its own
    unit order (so it is the natural reducer);
  * the i8 path's exchange buffer has one slot per CTA (DevCtx::I8_PART_CTAS = 256) and the counters one per strip.
"""
import ctypes
import pytest

SMS = 132
TAG_SIMT, TAG_TC, TAG_I8 = 100, 200, 210


class Plan(ctypes.Structure):
    _fields_ = [("path", ctypes.c_int32), ("passes", ctypes.c_int32), ("rows", ctypes.c_int32), ("grid", ctypes.c_int32),
                ("stages", ctypes.c_int32), ("smem_bytes", ctypes.c_int32), ("a_stages", ctypes.c_int32),
                ("d_bufs", ctypes.c_int32), ("tmem_cols", ctypes.c_int32), ("reserved", ctypes.c_int32),
                ("units", ctypes.c_int64)]


@pytest.fixture(scope="module")
def lib():
    from exllamav3_b200 import ext
    L = ext.lib
    L.exl3b_gemm_plan.argtypes = [ctypes.c_int] * 7 + [ctypes.POINTER(Plan)]
    L.exl3b_gemm_plan.restype = ctypes.c_int
    L.exl3b_plan_unit_range.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64)]
    L.exl3b_plan_unit_range.restype = ctypes.c_int
    L.exl3b_plan_cta_of_unit.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int64]
    L.exl3b_plan_cta_of_unit.restype = ctypes.c_int
    ext.set_gemm_path(0)
    return L


def plan(lib, m, k, n, K, cb, sms=SMS, force=0):
    p = Plan()
    r = lib.exl3b_gemm_plan(m, k, n, K, cb, sms, force, ctypes.byref(p))
    assert r == 0, lib.exl3b_last_error()
    return p


def model_shapes():
    """(k, n) of every quantized linear in BASELINE.json's configs, unsharded and as per-rank TP shards."""
    shapes = set()
    for hidden, inter, q, kv in ((4096, 14336, 4096, 1024), (8192, 28672, 8192, 1024)):
        for tp in (1, 2, 4, 8):
            sh = lambda x: max(128, (x // tp) // 128 * 128)
            shapes |= {(hidden, sh(q)), (hidden, sh(kv)), (sh(q), hidden), (hidden, sh(inter)), (sh(inter), hidden),
                       (hidden, sh(128256))}
    shapes |= {(4096, 14336), (14336, 4096)}          # Mixtral experts
    return sorted(shapes)


def test_path_selection_rules(lib):
    # mul1 at m <= 4 -> int8 tensor-core path; everything else the exact tensor-core path (api.cu select_gemm_path)
    assert plan(lib, 1, 4096, 4096, 4, 2).path == TAG_I8
    assert plan(lib, 4, 4096, 4096, 4, 2).path == TAG_I8
    assert plan(lib, 5, 4096, 4096, 4, 2).path == TAG_TC
    assert plan(lib, 1, 4096, 4096, 4, 0).path == TAG_TC
    assert plan(lib, 1, 4096, 4096, 4, 1).path == TAG_TC
    p = plan(lib, 1000, 4096, 4096, 4, 2)
    assert p.path == TAG_TC and p.passes == 8 and p.rows == 128
    # forced paths (exl3b_set_gemm_path), including the refusal when the forced path cannot take the call
    from exllamav3_b200 import ext
    try:
        ext.set_gemm_path(TAG_I8)
        assert plan(lib, 8, 4096, 4096, 4, 2).path == TAG_I8 and plan(lib, 8, 4096, 4096, 4, 2).rows == 8
        q = Plan()
        assert lib.exl3b_gemm_plan(8, 8192, 4096, 4, 2, SMS, 0, ctypes.byref(q)) == -4        # 8 x 8192 fp16 > 64 KB cache
        assert lib.exl3b_gemm_plan(1, 4096, 4096, 4, 0, SMS, 0, ctypes.byref(q)) == -4        # not mul1
        ext.set_gemm_path(TAG_SIMT)
        assert plan(lib, 1, 4096, 4096, 4, 2).path == TAG_SIMT
        ext.set_gemm_path(TAG_TC)
        assert plan(lib, 1, 4096, 4096, 4, 2).path == TAG_TC
    finally:
        ext.set_gemm_path(0)
    q = Plan()
    assert lib.exl3b_gemm_plan(1, 4096, 4000, 4, 2, SMS, 0, ctypes.byref(q)) == -1
    assert lib.exl3b_gemm_plan(1, 4096, 4096, 0, 2, SMS, 0, ctypes.byref(q)) == -2


def test_known_geometry_of_the_bench_shapes(lib):
    """The launch geometry of the bench's decode shapes: K = 4, m = 1."""
    p = plan(lib, 1, 4096, 4096, 4, 2)
    # stage = 8192 B weights + 4096 + 64 B digits; accumulator hand-off 16512 B; activation cache 8192 B
    # -> (204800 - 16512 - 8192) // 12352 = 14 stages; no tensor memory on sm_90a (accumulators in registers)
    assert (p.rows, p.grid, p.units, p.stages, p.a_stages, p.d_bufs, p.tmem_cols) == (4, 132, 1024, 14, 0, 2, 0)
    assert p.smem_bytes == 14 * 12352 + 16 * 128 * 4 + 1024 + 16512 + 8192
    p = plan(lib, 1, 4096, 128256 // 128 * 128, 6, 2)          # lm_head, 6 bpw
    assert p.grid == 132 and p.units == 32 * 1002 and p.stages == (204800 - 16512 - 8192) // (12288 + 4160)
    p = plan(lib, 1, 128, 128, 4, 2)                            # a single unit: one CTA
    assert p.grid == 1 and p.units == 1
    p = plan(lib, 1, 4096, 4096, 4, 2, force=64)                # force_num_sms caps the persistent grid
    assert p.grid == 64


@pytest.mark.parametrize("K", range(1, 9))
def test_budgets_for_every_model_shape(lib, K):
    for (k, n) in model_shapes():
        for (m, cb) in ((1, 2), (4, 2), (1, 0), (8, 1), (32, 2), (256, 0)):
            p = plan(lib, m, k, n, K, cb)
            assert p.path in (TAG_I8, TAG_TC)
            assert 2 <= p.stages <= 16
            assert p.smem_bytes <= 220 * 1024                   # cudaFuncAttributeMaxDynamicSharedMemorySize set by the launchers
            assert 1 <= p.grid <= min(SMS, p.units) and p.units == (k // 128) * (n // 128)
            assert n // 128 <= 32768                            # DevCtx::COUNTERS_PER_SLOT
            assert (p.a_stages, p.tmem_cols) == (0, 0)         # no tensor memory on sm_90a
            if p.path == TAG_I8:
                assert p.grid <= 256                            # DevCtx::I8_PART_CTAS exchange slots
                assert p.d_bufs == 2                            # two shared-memory accumulator hand-off buffers
            else:
                assert p.rows <= 128                            # fp32 accumulators of one pass live in registers
                assert 2 * p.grid * p.rows * 128 * 4 <= 40 << 20   # DevCtx::WS_BYTES_PER_SLOT


def _partition(lib, U, G):
    b, e = ctypes.c_int64(), ctypes.c_int64()
    out = []
    for c in range(G):
        assert lib.exl3b_plan_unit_range(U, G, c, ctypes.byref(b), ctypes.byref(e)) == 0
        out.append((b.value, e.value))
    return out


def test_stream_k_partition_invariants(lib):
    cases = set()
    for (k, n) in model_shapes():
        U = (k // 128) * (n // 128)
        cases.add((k // 128, n // 128, min(SMS, U)))
    cases |= {(1, 1, 1), (3, 5, 15), (3, 5, 7), (32, 32, 74), (7, 11, 76), (112, 32, 148), (32, 1002, 132)}
    for (KB, strips, G) in sorted(cases):
        U = KB * strips
        rng = _partition(lib, U, G)
        assert rng[0][0] == 0 and rng[-1][1] == U
        for c in range(G):
            assert rng[c][1] > rng[c][0], "empty CTA"
            if c:
                assert rng[c][0] == rng[c - 1][1]
        # cta_of_unit inverts the ranges (sampled at the boundaries of every CTA and of every strip)
        probes = {u for (b, e) in rng for u in (b, e - 1)} | {s * KB for s in range(strips)} | {s * KB + KB - 1 for s in range(strips)}
        owner = {}
        for u in probes:
            c = lib.exl3b_plan_cta_of_unit(U, G, u)
            assert rng[c][0] <= u < rng[c][1]
            owner[u] = c
        for s in range(strips):
            c_a, c_b = owner[s * KB], owner[s * KB + KB - 1]
            assert c_a <= c_b
            # contributors are exactly the CTAs whose range intersects the strip
            inter = [c for c in range(c_a, c_b + 1) if rng[c][0] < (s + 1) * KB and rng[c][1] > s * KB]
            assert inter == list(range(c_a, c_b + 1))
            if c_a > 0:
                assert rng[c_a - 1][1] <= s * KB
            if c_b < G - 1:
                assert rng[c_b + 1][0] >= (s + 1) * KB
            if c_b > c_a:
                # split strip: the reducer c_a meets this strip as the LAST segment of its range (its range ends inside
                # the strip), every other contributor meets it first -- so contributors never wait for the reducer
                assert s * KB < rng[c_a][1] < (s + 1) * KB
                for c in range(c_a + 1, c_b + 1):
                    assert rng[c][0] > s * KB and rng[c][0] < (s + 1) * KB


def test_plan_argument_validation(lib):
    b, e = ctypes.c_int64(), ctypes.c_int64()
    assert lib.exl3b_plan_unit_range(10, 11, 0, ctypes.byref(b), ctypes.byref(e)) == -2       # grid > units
    assert lib.exl3b_plan_unit_range(10, 5, 5, ctypes.byref(b), ctypes.byref(e)) == -2
    assert lib.exl3b_plan_cta_of_unit(10, 5, 10) == -2
    assert lib.exl3b_gemm_plan(1, 4096, 4096, 4, 2, 0, 0, ctypes.byref(Plan())) == -2
