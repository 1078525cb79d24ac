"""
Work partition of exl3_moe (csrc/moe_tc.cu), host only: exl3b_moe_plan runs the same planner the route kernel runs on the
device.  Every (processed expert, row, 128-column block) is covered exactly once, skipped experts and the sentinel bucket are
never touched, the scratch bounds hold, and the unit counts fit 32 bits.  Also the exl3b_moe argument checks that need no GPU.
"""
import ctypes
import numpy as np
import pytest


def ext():
    from exllamav3_b200 import ext as e
    return e


def check(count, T, N, hidden=256, inter=384):
    count = np.asarray(count, dtype=np.int64)
    plan, passes, codes = ext().exl3_moe_plan(count, T, N, hidden, inter)
    E = len(count) - 1
    starts = np.concatenate([[0], np.cumsum(count[:-1])])
    owner = np.full(N, -1)
    want_codes = np.full(N, -1)
    rows_seen = set()
    last = (-1, -1)
    for p, (e, pos0, rows, row0, chunk) in enumerate(passes):
        assert 0 <= e < E and 0 < count[e] <= T and 1 <= rows <= 128
        assert starts[e] <= pos0 and pos0 + rows <= starts[e] + count[e] <= N
        assert (chunk, pos0) > last, "passes are in position order, chunks ascending"
        last = (chunk, pos0)
        assert 0 <= chunk < plan.chunks <= plan.max_chunks
        assert row0 % 16 == 0 and row0 + (rows + 15) // 16 * 16 <= min(plan.rows, plan.chunk_rows)
        assert (owner[pos0:pos0 + rows] == -1).all(), "position covered twice"
        owner[pos0:pos0 + rows] = e
        want_codes[pos0:pos0 + rows] = 128 * p + np.arange(rows)
        for r in range(row0, row0 + rows):
            assert (chunk, r) not in rows_seen, "row of a chunk used twice"
            rows_seen.add((chunk, r))
    expected = np.full(N, -1)
    lo = 0
    for e in range(E):
        s, c = int(starts[e]), int(count[e])
        if 0 < c <= T and s >= lo and s + c <= N:
            expected[s:s + c] = e
            lo = s + c
    assert (owner == expected).all()
    assert (codes == want_codes).all(), "position codes of the route kernel disagree with the passes"
    assert plan.passes == len(passes) <= plan.max_passes
    # (pass, 128-column strip) items of each GEMM: each strip of each pass once; 32-bit work lists
    assert plan.units_gate_up == plan.passes * (inter // 128) < 2 ** 31
    assert plan.units_down == plan.passes * (hidden // 128) < 2 ** 31
    assert 128 * plan.max_passes < 2 ** 31
    return plan, passes


def test_plan_edge_cases():
    # empty experts, exactly T, more than T, the sentinel bucket
    plan, passes = check([0, 4, 5, 0, 3, 7], T=4, N=23)
    assert [p[0] for p in passes] == [1, 4]
    # a second and third pass when T > 128
    plan, passes = check([300, 2, 129], T=300, N=431)
    assert [(p[0], p[2]) for p in passes] == [(0, 128), (0, 128), (0, 44), (1, 2)]
    assert passes[1][3] == 128 and passes[2][3] == 256 and passes[3][3] == 256 + 48
    # all experts skipped, and no positions at all
    assert check([9, 9, 0], T=8, N=18)[0].passes == 0
    assert check([0, 0, 0], T=8, N=0)[0].passes == 0
    # counts running past the positions given: the experts that do not fit are skipped
    assert [p[0] for p in check([2, 3, 4, 0], T=8, N=6)[1]] == [0, 1]


@pytest.mark.parametrize("seed", range(12))
def test_plan_random(seed):
    rng = np.random.default_rng(seed)
    E = int(rng.choice([8, 64, 128, 256]))
    topk = int(rng.choice([1, 2, 8]))
    bsz = int(rng.choice([1, 5, 64, 300, 2048]))
    ex = np.stack([rng.choice(E, min(topk, E), replace=False) for _ in range(bsz)])
    ex[rng.random(ex.shape) < 0.1] = E
    count = np.bincount(ex.reshape(-1), minlength=E + 1)
    T = int(rng.choice([1, 16, 128, 200, 1000]))
    hidden, inter = [(2048, 768), (4096, 14336), (7168, 2048), (384, 640)][seed % 4]
    check(count, T, ex.size, hidden, inter)


def test_plan_chunks():
    # Mixtral-8x7B widths: a chunk holds chunk_rows rows of the fixed work area; a long prefill runs in several chunks, each
    # filled beyond chunk_rows - 112 rows before the next starts, within the launcher's bound
    plan, passes = check([2000] * 8 + [0], T=2000, N=16000, hidden=4096, inter=14336)
    assert plan.chunk_rows >= 2048 and plan.chunks >= 6 and plan.chunks <= plan.max_chunks
    used = {}
    for e, pos0, rows, row0, chunk in passes:
        used[chunk] = max(used.get(chunk, 0), row0 + (rows + 15) // 16 * 16)
    assert all(used[c] > plan.chunk_rows - 128 for c in range(plan.chunks - 1))
    # the bound counts only positions that can be processed: min(N, E * T)
    assert ext().exl3_moe_plan([0] * 8 + [0], 128, 16000, 4096, 14336)[0].max_passes <= 8 + 8


def test_plan_bounds_worst_case():
    # one row per expert maximises padding; one huge expert maximises passes
    N = 2048
    plan, _ = check([1] * N + [0], T=1, N=N)
    assert plan.rows == 16 * N
    plan, _ = check([N, 0], T=N, N=N)
    assert plan.passes == N // 128


def test_plan_rejects_bad_arguments():
    e = ext()
    with pytest.raises(RuntimeError):
        e.exl3_moe_plan([1, 2, 0], 0, 3, 256, 384)         # T < 1
    with pytest.raises(RuntimeError):
        e.exl3_moe_plan([1, 2, 0], 4, 3, 192, 384)         # hidden % 128
    with pytest.raises(RuntimeError):
        e.exl3_moe_plan([1, 2, 0], 4, 2 ** 20 + 1, 256, 384)   # more positions than the work list holds


def test_moe_abi_validation_without_gpu():
    lib = ext().lib
    one = ctypes.c_void_p(16)                             # never dereferenced: validation fails first

    def call(**kw):
        a = dict(bsz=4, hidden=256, inter=384, E=8, N=8, T=16, conc=1, act=0, Kg=4, Ku=4, Kd=4,
                 cb=(0, 1, 0, 1, 0, 1), limit=0.0, num_active=-1)
        a.update(kw)
        return lib.exl3b_moe(None, one, one, one, one, one, a["bsz"], a["hidden"], a["inter"], a["E"], a["N"], a["T"],
                             a["conc"], a["act"], a["Kg"], a["Ku"], a["Kd"], *([one] * 9), *a["cb"], a["limit"],
                             a["num_active"])

    assert call(num_active=0) == 0                        # nothing to do: no launch, no check
    assert call(cb=(0, 1, 0, 1, 1, 0)) == -2 and b"same codebook" in lib.exl3b_last_error()
    assert call(cb=(0, 0, 0, 0, 0, 0)) == -2 and b"Only mcg and mul1" in lib.exl3b_last_error()
    assert call(cb=(1, 1, 1, 1, 1, 1)) == -2 and b"Only mcg and mul1" in lib.exl3b_last_error()
    assert call(Kd=9) == -2 and b"K must be 1..8" in lib.exl3b_last_error()
    assert call(act=3) == -2
    assert call(hidden=192) == -1 and b"divisible by 128" in lib.exl3b_last_error()
    assert call(inter=320) == -1 and b"divisible by 128" in lib.exl3b_last_error()
    assert call(E=4096) == -4
    bad = ctypes.c_void_p(16 + 4)
    r = lib.exl3b_moe(None, bad, one, one, one, one, 4, 256, 384, 8, 8, 16, 1, 0, 4, 4, 4, *([one] * 9), 0, 1, 0, 1, 0, 1, 0.0, -1)
    assert r == -2 and b"aligned" in lib.exl3b_last_error()
    r = lib.exl3b_moe(None, one, ctypes.c_void_p(16 + 8), one, one, one, 4, 256, 384, 8, 8, 16, 1, 0, 4, 4, 4, *([one] * 9),
                      0, 1, 0, 1, 0, 1, 0.0, -1)
    assert r == -2 and b"aligned" in lib.exl3b_last_error()
