"""
Drop-in check at the Python level against what the REFERENCE'S OWN Python modules do, recorded once by
oracle/gen_golden_callsites.py into tests/golden/ref_callsites.json.gz: the reference's LinearEXL3 (modules/quant/exl3.py), run
with its `ext` import bound to this repo's shim (`exllamav3_b200.ext`, exactly what INTEGRATION.md's patch does), issued the
recorded extension calls; its MultiLinear built the recorded pointer tables; its use_mgemm policy gave the recorded answers;
its tp_import_split built the recorded shards; and its Python tree calls the qgemm surface at the recorded call sites.  Here
this repo's own caller (QLinear, pointer_tables, tp.tp_slice) must do the same on the same inputs, and every recorded call
must bind against the shim's real signatures.  No kernel runs: the shim's entry points are wrapped by recorders.
"""
import gzip, inspect, json, os
import pytest
import torch

import refstubs

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_callsites.json.gz")


@pytest.fixture(scope="module")
def gold():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


@pytest.fixture()
def recorder(monkeypatch):
    from exllamav3_b200 import ext
    calls = []

    def wrap(name):
        sig = inspect.signature(getattr(ext, name))

        def f(*a, **kw):
            sig.bind(*a, **kw)
            calls.append([name, [refstubs.encode(t) for t in a], sorted(kw)])
            return 210
        return f

    for name in refstubs.RECORDED_OPS:
        monkeypatch.setattr(ext, name, wrap(name))
    return calls


def _qlin(t, **kw):
    from exllamav3_b200 import QLinear
    return QLinear(t["trellis"], t["suh"], t["svh"], mul1=True, **kw)


def _binds(call):
    from exllamav3_b200 import ext
    name, args, kws = call
    inspect.signature(getattr(ext, name)).bind(*([None] * len(args)), **{k: None for k in kws})


def test_reference_linear_exl3_runs_on_the_shim_and_matches_the_mirror(gold, recorder):
    from exllamav3_b200 import qlinear, ext
    g = gold["linear"]
    assert g["AUTO_RECONSTRUCT_THRESHOLD"] == qlinear.KERNEL_MAX_ROWS == 144
    assert g["MAX_RECONSTRUCT_SLICE_N"] == qlinear.DENSE_WINDOW_COLS == 32768
    assert g["bc_type"] == ext.BC_LinearEXL3.__name__ and (g["K"], g["mcg"], g["mul1"]) == (4, False, True)
    k, n = 256, 384
    mir = _qlin(refstubs.tensors(k, n))
    assert len(g["cases"]) == len(refstubs.LINEAR_CASES)
    for (shape, params, odt), case in zip(refstubs.LINEAR_CASES, g["cases"]):
        recorder.clear()
        y = mir.forward(torch.zeros(shape, dtype=torch.half), params, getattr(torch, odt) if odt else None)
        assert recorder == case["calls"] and len(case["calls"]) >= 1, (shape, params)     # same calls, same argument shapes
        assert list(y.shape) == case["y_shape"] and str(y.dtype) == case["y_dtype"], (shape, params)
        for c in case["calls"]:
            _binds(c)
    # the kernel path hands exl3_gemm the reference's 10 arguments: (A, B, C, suh, A_had, svh, -1, mcg, mul1, 0)
    last = g["cases"][-1]["calls"][0]
    assert last[0] == "exl3_gemm" and last[1][6:] == [-1, False, True, 0]


def test_reference_wide_output_slicing_matches_the_mirror(gold, recorder, monkeypatch):
    from exllamav3_b200 import qlinear
    monkeypatch.setattr(qlinear, "DENSE_WINDOW_COLS", 256)
    k, n = 128, 640
    mir = _qlin(refstubs.tensors(k, n))
    for rows, ref_calls in zip(refstubs.SLICING_ROWS, gold["slicing"]):
        recorder.clear()
        mir.forward(torch.zeros((rows, k), dtype=torch.half), {})
        assert recorder == ref_calls and sum(c[0] == "hgemm" for c in ref_calls) == 3, rows


def test_reference_multilinear_tables_match_the_mirror(gold):
    """modules/multilinear.py builds the pointer tables exl3_mgemm reads; pointer_tables must build the same ones."""
    from exllamav3_b200 import pointer_tables
    g = gold["multilinear"]
    k, n = 128, 256
    inners = [_qlin(refstubs.tensors(k, n)) for _ in range(3)]
    where = {getattr(i, a).data_ptr(): [j, a] for j, i in enumerate(inners) for a in ("trellis", "suh", "svh")}
    tables = dict(zip(("ptrs_trellis", "ptrs_suh", "ptrs_svh"), pointer_tables("cpu", inners)))
    for a, t in tables.items():
        assert [where[int(p)] for p in t.tolist()] == g["tables"][a] and str(t.dtype) == g["dtype"], a
    i0 = inners[0]
    assert [i0.K, bool(i0.mcg), bool(i0.mul1), i0.in_features, i0.out_features] == g["fields"]


def test_every_reference_call_site_of_the_qgemm_surface_fits_the_shim(gold):
    """Every `ext.<op>(...)` call site of the qgemm surface in the reference's Python tree (recorded by an AST audit) binds,
    by positional count and keyword names, against the shim's signature.  SURVEY.md 8b lists these callers."""
    from exllamav3_b200 import ext
    seen = {o: 0 for o in refstubs.AUDIT_OPS}
    for path, line, op, nargs, kws in gold["audit"]:
        try:
            inspect.signature(getattr(ext, op)).bind(*([None] * nargs), **{kw: None for kw in kws})
        except TypeError as e:
            raise AssertionError(f"{path}:{line}: ext.{op} call does not fit the shim: {e}")
        seen[op] += 1
    assert seen["exl3_gemm"] >= 1 and seen["exl3_gemm_num_kernel_shapes"] >= 1 and seen["exl3_gemm_shape_compat"] >= 1
    assert seen["exl3_mgemm"] >= 8 and seen["hgemm"] >= 3 and seen["had_r_128"] >= 2 and seen["reconstruct"] >= 2
    assert seen["reconstruct_had_slice"] >= 2 and seen["reconstruct_slice"] >= 1 and seen["exl3_gemv_int8_max_k"] >= 1


def test_reference_use_mgemm_policy_with_the_shims_answer(gold, monkeypatch):
    """model/config.py:48-64, the reference's OWN policy, recorded for the shim's exl3_gemv_int8_max_k answer (0) and for the
    reference extension's answer on Hopper (6): with the shim, k+v and gate+up stay fused for every bitrate -- the launch list
    bench.py times -- whereas with 6 the wide 4-bpw gate+up pair is unfused (bench.py --no-fuse)."""
    from exllamav3_b200 import ext
    monkeypatch.setattr(ext, "_check", lambda rc: 132)                      # no device here: the index check is not under test
    assert ext.exl3_gemv_int8_max_k(0) == 0
    policy = {(mk, K, n, mul1): fused for mk, K, n, mul1, fused in gold["use_mgemm"]}
    for K in range(1, 9):
        for n in (1024, 14336):
            for mul1 in (True, False):
                assert policy[(ext.exl3_gemv_int8_max_k(0), K, n, mul1)], (K, n, mul1)     # fused at every bitrate
    assert not policy[(6, 4, 14336, True)]                                  # wide 4 bpw pair: unfused with the reference's answer
    assert policy[(6, 4, 1024, True)] and policy[(6, 7, 14336, True)] and policy[(6, 4, 14336, False)]


def test_reference_tp_import_split_equals_tp_slice(gold):
    """The reference's OWN shard construction (LinearEXL3.tp_export / tp_import_split, modules/quant/exl3.py:268-330) for every
    split of world 3, against this repo's tp.tp_slice on the same inputs."""
    from exllamav3_b200 import tp
    g = gold["tp"]
    k, n = 512, 768
    tens, bias = refstubs.tp_tensors(k, n)
    assert {a: refstubs.digest(tens[a]) for a in ("trellis", "suh", "svh")} | {"bias": refstubs.digest(bias)} == g["inputs"]
    mir = _qlin(tens, bias=bias, out_dtype=torch.float)
    world = 3
    splits = [[True, a, b] for (a, b) in tp.split_ranges(n, world)] + [[False, a, b] for (a, b) in tp.split_ranges(k, world)] + [None]
    assert splits == [s["split"] for s in g["shards"]]
    for split, ref in zip(splits, g["shards"]):
        m = tp.tp_slice(mir, tuple(split) if split else None)
        assert [m.in_features, m.out_features, m.K, bool(m.mcg), bool(m.mul1), str(m.out_dtype)] == ref["fields"], split
        for a in ("trellis", "suh", "svh", "bias"):
            assert refstubs.digest(getattr(m, a)) == ref[a], (split, a)
        assert m.trellis.is_contiguous()
