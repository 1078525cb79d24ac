"""
Host side of the decode-GEMM edge tests (tests/test_gpu_edges.py), no GPU needed.

The GPU file runs the exact tensor-core kernel (tag 200) and the int8 codebook kernel (tag 210) at shapes and persistent grids
chosen to reach particular branches: split-K slot choice, multi-strip CTAs, uncached int8 activations, int32 accumulation
chunks.  Whether a shape reaches a branch is decided by the host planner (exl3b_gemm_plan) and the stream-K partition
(exl3b_plan_unit_range / exl3b_plan_cta_of_unit), so this file asserts, with the same functions the launchers call, that every
row of those tables still hits the regime it is there for.  A planner change that shrinks the coverage fails here instead of
letting the GPU tests pass without testing anything.

It also owns what both files share: the tables, the worst-case int32 input and the plan helpers, and the checker of the fp16
paths (tags 100 and 200, exl3_moe) against their exact models, with its bars, which every GPU file that reaches those paths uses.
"""
import ctypes
import numpy as np
import pytest
from oracle import exl3_oracle as orc

SMS = 132
TAG_SIMT, TAG_TC, TAG_I8, TAG_CHAIN = 100, 200, 210, 220
INT32_MAX = 2 ** 31 - 1
I8_SUB_UNITS = 96                     # gemm_tc_i8_body.cuh: units per int32 accumulation chunk
I8_CACHE_MAX_BYTES = 64 * 1024        # gemm_tc_i8_body.cuh: largest activation cached in shared memory

# forced persistent grids (force_num_sms): (k, n, grids).  Regimes asserted in test_forced_grid_table_hits_its_regimes.
FORCED_GRIDS = (
    (384, 640, (1, 2, 4, 7, 15)),     # 3 x 5 units: one CTA for all; CTAs with partials of two strips; one unit per CTA
    (1152, 1152, (2, 7, 10, 80)),     # 9 x 9: a CTA spanning >= 3 strips with partial first and last strips
    (4096, 128, (2, 31, 32)),         # 32 x 1: one strip reduced from >= 31 contributors
    (128, 8192, (5,)),                # 1 x 64: every strip full, ~13 strips per CTA
)

# (m, k, cached) on both sides of the int8 path's 64 KiB activation cache
CACHE_PAIRS = ((4, 8192, True), (4, 8320, False), (3, 10880, True), (3, 11008, False),
               (2, 16384, True), (2, 16512, False), (1, 32896, False))

# worst-case int32 accumulation: one CTA walks one strip of 640 k-blocks
WORST_K, WORST_N, WORST_KQ = 81920, 128, 4


class Plan(ctypes.Structure):
    _fields_ = [("path", ctypes.c_int32), ("passes", ctypes.c_int32), ("rows", ctypes.c_int32), ("grid", ctypes.c_int32),
                ("stages", ctypes.c_int32), ("smem_bytes", ctypes.c_int32), ("a_stages", ctypes.c_int32),
                ("d_bufs", ctypes.c_int32), ("tmem_cols", ctypes.c_int32), ("reserved", ctypes.c_int32),
                ("units", ctypes.c_int64)]


def _lib():
    from exllamav3_b200 import ext
    L = ext.lib
    L.exl3b_gemm_plan.argtypes = [ctypes.c_int] * 7 + [ctypes.POINTER(Plan)]
    L.exl3b_gemm_plan.restype = ctypes.c_int
    L.exl3b_plan_unit_range.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int64),
                                        ctypes.POINTER(ctypes.c_int64)]
    L.exl3b_plan_unit_range.restype = ctypes.c_int
    L.exl3b_plan_cta_of_unit.argtypes = [ctypes.c_int64, ctypes.c_int, ctypes.c_int64]
    L.exl3b_plan_cta_of_unit.restype = ctypes.c_int
    return L


def gemm_plan(m, k, n, K, cb, force=0, sms=SMS):
    L = _lib()
    p = Plan()
    r = L.exl3b_gemm_plan(m, k, n, K, cb, sms, force, ctypes.byref(p))
    assert r == 0, L.exl3b_last_error()
    return p


def stream_k_regimes(KB, strips, G):
    """What the split-K combine sees when KB x strips units are spread over G CTAs (the kernels' own partition)."""
    L = _lib()
    U = KB * strips
    b, e = ctypes.c_int64(), ctypes.c_int64()
    rng = []
    for c in range(G):
        assert L.exl3b_plan_unit_range(U, G, c, ctypes.byref(b), ctypes.byref(e)) == 0
        rng.append((b.value, e.value))
    contrib = []
    for s in range(strips):
        c_a, c_b = L.exl3b_plan_cta_of_unit(U, G, s * KB), L.exl3b_plan_cta_of_unit(U, G, s * KB + KB - 1)
        contrib.append((c_a, c_b))
    split = [c_b > c_a for (c_a, c_b) in contrib]
    first_last = [(lo // KB, (hi - 1) // KB) for (lo, hi) in rng]
    return dict(
        all_full=not any(split),
        one_unit_per_cta=all(hi - lo == 1 for (lo, hi) in rng),
        max_contributors=max(c_b - c_a + 1 for (c_a, c_b) in contrib),
        strips_per_cta=[l - f + 1 for (f, l) in first_last],
        # a CTA stores partials of two different strips: its first strip (slot 0) and a later one (slot 1)
        both_slots=any(f != l and split[f] and split[l] for (f, l) in first_last),
        # the strip's first contributor began in an earlier strip: its partial sits in its second slot
        first_contributor_second_slot=any(split[s] and rng[c_a][0] < s * KB for s, (c_a, _) in enumerate(contrib)),
        span3_partial_ends=any(l - f >= 2 and split[f] and split[l] for (f, l) in first_last),
    )


def worst_case_inputs(m, k=WORST_K, n=WORST_N, K=WORST_KQ, s0=0.5):
    """
    Inputs that drive every int32 accumulator of the int8 path up as fast as possible: suh[128 b] = s0 > 0 and x = 1 at every
    block start, 0 elsewhere, so x * suh is s0 * e_0 per block and its Hadamard is s0 / sqrt(128) in EVERY position.  Every row's
    q is then I8_QMAX = 127 * 256 + 0 (hi digit 127, lo digit 0) and every u8 x s8 product of a column has the same sign.
    """
    tr, suh, svh, _ = orc.make_synthetic(k, n, K, seed=4242)
    suh = suh.copy()
    suh[::128] = np.float16(s0)
    x = np.zeros((m, k), dtype=np.float16)
    x[:, ::128] = 1.0
    return tr, suh, svh, x


# ---- the fp16 paths against their exact models -----------------------------------------------------------------------------
# oracle.exl3_gemm_f16_model / exl3_mgemm_f16_model / exl3_moe_model are these paths' arithmetic up to the order of the fp32
# accumulation (README.md, Parity).  The kernels accumulate in fp32 along k, so their distance to the model grows like
# 2^-24 sqrt(k) max|y|: measured on an H100 (80 GB HBM3, 700 W) over the GPU suite, fp32 C is at most 5.0e-6 max|y| max-abs and
# 4.3e-6 rel-RMS from the model (k = 14336, tag 200; 3e-7 at k = 512).
#   fp32 C: max-abs / max|y| and rel-RMS <= F16_MODEL_BAR, the int8 paths' bars.
#   fp16 C: every element within F16_MODEL_STEPS x oracle.f16_model_tol of the model (roundings of the pre-svh value and of C
#           that went the other way) plus F16_MODEL_BAR[0] max|y| (the accumulation order, as for fp32 C), and at least
#           F16_MODEL_SAME of the elements bit-identical to the model.  Measured: at most 1.0 x f16_model_tol + 2e-5 max|y| (tag 100);
#           1.9 % of the elements differ at k = 14336 (4096 x 14336 down, 32 rows), 0.5 % at k = 512.  svh applied in fp32
#           before the one fp16 rounding changes 26 %.
#   exl3_moe: the same accumulation noise flips ~2 % of the fp16 roundings of g and u, and so of h, before the down projection;
#           measured at most 3.4e-4 max-abs and 1.6e-4 rel-RMS from exl3_moe_model (Mixtral widths, several chunks).
F16_MODEL_BAR = (2e-5, 1e-5)
F16_MODEL_SAME = 0.925
F16_MODEL_STEPS = 4
MOE_MODEL_BAR = (1.4e-3, 6.5e-4)


def rel_err(y, ref):
    y = np.asarray(y, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(y - ref)
    return err.max() / max(np.abs(ref).max(), 1e-30), np.sqrt((err ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def f16_model_ratios(y, model, tol):
    """fp16 C against its model: (largest |y - model| over its bound, share of elements that are not bit-identical)."""
    y64, m64 = np.asarray(y, dtype=np.float64), np.asarray(model, dtype=np.float64)
    bound = F16_MODEL_STEPS * tol + F16_MODEL_BAR[0] * np.abs(m64).max()
    d = np.abs(y64 - m64)
    worst = float(np.max(np.where(d > 0, d / np.maximum(bound, 1e-300), 0.0)))
    return worst, float((np.asarray(y, dtype=np.float16) != np.asarray(model, dtype=np.float16)).mean())


def check_f16_model(y, model, tol, what, bar=F16_MODEL_BAR):
    """
    C of an fp16-path call against its model.  tol None: fp32 C, held to `bar`; else fp16 C, held element-wise to
    F16_MODEL_STEPS x tol (f16_model_tol, or the mgemm model's sum of it) plus F16_MODEL_BAR[0] max|y|, and to F16_MODEL_SAME
    bit-identical elements.
    """
    if tol is None:
        mx, rms = rel_err(y, model)
        assert mx <= bar[0] and rms <= bar[1], ("fp16-path model", what, mx, rms)
        return
    worst, changed = f16_model_ratios(y, model, tol)
    assert worst <= 1.0 and changed <= 1 - F16_MODEL_SAME, ("fp16-path model, fp16 C", what, worst, changed)


def check_f16_gemm(y, x, tr, suh, svh, K, cb, fp32, what, w=None):
    """One exl3_gemm call on tag 100 or 200 (C as float64 or its own dtype) against oracle.exl3_gemm_f16_model."""
    model, pre = orc.exl3_gemm_f16_model(x, tr, suh, svh, K, cb, np.float32 if fp32 else np.float16, w=w)
    check_f16_model(y, model, None if fp32 else orc.f16_model_tol(model, pre, svh), what)


def check_moe_model(y, model, what):
    check_f16_model(y, model, None, what, MOE_MODEL_BAR)


# ---- tests -----------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module", autouse=True)
def auto_path():
    from exllamav3_b200 import ext
    prev = ext.set_gemm_path(0)
    yield
    ext.set_gemm_path(prev)


def test_forced_grid_table_hits_its_regimes():
    (r1, r2, r3, r4) = [{G: stream_k_regimes(k // 128, n // 128, G) for G in grids} for (k, n, grids) in FORCED_GRIDS]
    # 384 x 640: one CTA holds every strip whole; some grid gives a CTA partials of two strips (both workspace slots) and a
    # strip whose first contributor holds its partial in the second slot; G = U gives one unit per CTA
    assert r1[1]["all_full"] and r1[1]["strips_per_cta"] == [5]
    assert any(r["both_slots"] for r in r1.values())
    assert any(r["first_contributor_second_slot"] for r in r1.values())
    assert r1[15]["one_unit_per_cta"] and r1[15]["max_contributors"] == 3
    # 1152 x 1152: a CTA spans >= 3 strips and shares the first and the last of them
    assert any(r["span3_partial_ends"] for r in r2.values())
    assert r2[80]["max_contributors"] >= 2 and not r2[80]["all_full"]
    # 4096 x 128: one strip, >= 31 contributors
    assert max(r["max_contributors"] for r in r3.values()) >= 31
    assert r3[32]["one_unit_per_cta"]
    # 128 x 8192: every strip whole, 12..13 strips per CTA
    assert r4[5]["all_full"] and min(r4[5]["strips_per_cta"]) >= 12


@pytest.mark.parametrize("k,n,grids", FORCED_GRIDS)
def test_forced_grids_are_launched_as_asked(k, n, grids):
    from exllamav3_b200 import ext
    U = (k // 128) * (n // 128)
    for G in grids:
        assert G <= U
        try:
            ext.set_gemm_path(TAG_TC)                          # mul1 at m <= 4 would go to the int8 path
            for m in (1, 17, 130):
                for cb in (0, 2):
                    p = gemm_plan(m, k, n, 4, cb, force=G)
                    assert (p.path, p.grid, p.units, p.passes) == (TAG_TC, G, U, (m + 127) // 128), (k, n, G, m, cb)
        finally:
            ext.set_gemm_path(0)
        for m in (1, 4):
            p = gemm_plan(m, k, n, 4, 2, force=G)
            assert (p.path, p.grid, p.units) == (TAG_I8, G, U), (k, n, G, m)


@pytest.mark.parametrize("K", (2, 4, 6))
@pytest.mark.parametrize("n", (128, 384))
def test_int8_cache_boundary(K, n):
    """The activation cache is part of the shared-memory total: cached shapes carry m * k * 2 bytes more than the ring needs."""
    for (m, k, cached) in CACHE_PAIRS:
        assert (m * k * 2 <= I8_CACHE_MAX_BYTES) == cached
        p = gemm_plan(m, k, n, K, 2)
        assert p.path == TAG_I8 and p.rows == 4 and p.grid == min(SMS, (k // 128) * (n // 128))
        stage = 2048 * K + 4096 + 64                           # weights + digit tile + digit sums
        fixed = 16 * 128 * 4 + 1024 + 16512                    # epilogue tile, barriers, accumulator hand-off (MR = 4)
        cache = p.smem_bytes - p.stages * stage - fixed
        assert cache == ((m * k * 2 + 127) // 128 * 128 if cached else 0), (m, k, K, n, cache)
        assert p.stages == min(16, (200 * 1024 - 16512 - cache) // stage)


def test_worst_case_int32_input_is_sharp():
    """
    The worst-case input really gives every row digits (127, 0), and an accumulator that is never handed over would wrap: the
    largest per-decode-group column sum over the strip exceeds 2^31 - 1, while every 96-unit chunk (both groups together, as the
    epilogue adds them in int32) stays below it.
    """
    for m in (1, 4):
        tr, suh, svh, x = worst_case_inputs(m)
        xh = orc.had_r_128(x, pre_scale=suh)
        assert (xh == xh[0, 0]).all() and xh[0, 0] > 0
        q, _ = orc.i8_activation_q(x, suh)
        assert (q == 32512).all()
        hi, lo = (q + 128) >> 8, q - (((q + 128) >> 8) << 8)
        assert (hi == 127).all() and (lo == 0).all()
    bs = orc.mul1_bytesum(tr, WORST_KQ)                        # (k, n), every product 127 * bytesum >= 0
    KB = WORST_K // 128
    per_block = 127 * bs.reshape(KB, 128, WORST_N).sum(axis=1)             # (KB, n) int64
    # with one CTA the unit index is the k-block; decode group g takes the units of parity g
    group_total = np.stack([per_block[g::2].sum(axis=0) for g in (0, 1)])
    assert group_total.max() > INT32_MAX, group_total.max()
    assert group_total.max() > 2.5e9                          # ~ 320 * 128 * 127 * 510
    chunk = np.stack([per_block[c:c + I8_SUB_UNITS].sum(axis=0) for c in range(0, KB, I8_SUB_UNITS)])
    assert chunk.max() < INT32_MAX, chunk.max()
    # the plans the GPU test relies on: one CTA, one strip, uncached activations (recomputed per unit)
    for m in (1, 4):
        p = gemm_plan(m, WORST_K, WORST_N, WORST_KQ, 2, force=1)
        assert (p.path, p.grid, p.units) == (TAG_I8, 1, KB)
        assert m * WORST_K * 2 > I8_CACHE_MAX_BYTES


def test_worst_case_chain_plan():
    """The chain kernel (tag 220) takes the worst-case shape as one op on one CTA."""
    from exllamav3_b200 import ext
    for m in (1, 4):
        op = (ext._ChainOp * 1)()
        op[0].A = op[0].B = op[0].C = op[0].suh = op[0].svh = 4096
        op[0].m, op[0].k, op[0].n, op[0].K, op[0].cb, op[0].c_fp32 = m, WORST_K, WORST_N, WORST_KQ, 2, 1
        pl = ext._ChainPlan()
        assert ext.lib.exl3b_chain_plan(op, 1, 1, ctypes.byref(pl)) == 0, ext.lib.exl3b_last_error()
        assert (pl.grid, pl.units, pl.cache_bytes) == (1, WORST_K // 128, 0)
