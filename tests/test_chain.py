"""
GEMM chains (csrc/chain_i8.cu, include/exl3b200.h "GEMM chains"): one persistent launch for the quantized linears of a decode
block -- the launch sequences of the reference's BC_GatedMLP (libtorch/mlp.cpp:14-91: exl3_mgemm(gate, up) -> silu_mul ->
exl3_gemm(down)) and of BC_Attention's projections (libtorch/attention.cpp:286-365).

CPU part: the kernel's own unit cursor replayed on the host (every unit of every stage visited exactly once over the grid, run
and accumulation-chunk bounds, quad ownership), launch geometry, argument validation.
GPU part: parity with the fp64 oracle (tolerances of README.md, Parity: max-abs <= 2e-3 max|y|, rel-RMS <= 1e-3) and with separate
exl3_gemm calls, for single ops (every K, 1..4 rows, fp16 / fp32 outputs), same-input stages, dependent stages with the
gated activation in between, at test sizes and at the Llama shapes; single ops also against the exact model of the kernel's
arithmetic (oracle.exl3_gemm_i8_model, rule="blocknorm"; the rest of the chain's exact tests are in tests/test_chain_exact.py).
"""
import ctypes
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc


def _ops(specs):
    """specs: (m, k, n, K, in_mode, new_stage) -> ctypes array with dummy non-null pointers (host-only entry points)."""
    from exllamav3_b200 import ext
    arr = (ext._ChainOp * len(specs))()
    for a, (m, k, n, K, in_mode, new_stage) in zip(arr, specs):
        a.A = a.B = a.C = a.suh = a.svh = 4096
        a.A2 = 4096 if in_mode else None
        a.m, a.k, a.n, a.K, a.cb, a.c_fp32, a.in_mode, a.new_stage = m, k, n, K, 2, 1, in_mode, new_stage
    return arr


def _walk(arr, num_sms):
    from exllamav3_b200 import ext
    plan = ext._ChainPlan()
    assert ext.lib.exl3b_chain_plan(arr, len(arr), num_sms, ctypes.byref(plan)) == 0, ext.lib.exl3b_last_error()
    per_cta = []
    for cta in range(plan.grid):
        buf = np.zeros((4096, 8), dtype=np.int32)
        n = ext.lib.exl3b_chain_walk(arr, len(arr), num_sms, cta, buf.ctypes.data, 4096)
        assert 0 <= n <= 4096
        per_cta.append(buf[:n].copy())
    return plan, per_cta


LLAMA_LAYER = [(1, 4096, 4096, 4, 0, 0), (1, 4096, 1024, 4, 0, 0), (1, 4096, 1024, 4, 0, 0), (1, 4096, 4096, 4, 0, 1),
               (1, 4096, 14336, 4, 0, 1), (1, 4096, 14336, 4, 0, 0), (1, 14336, 4096, 4, 1, 1)]


@pytest.mark.parametrize("specs,num_sms", [
    (LLAMA_LAYER, 148),
    ([(1, 4096, 128256, 6, 0, 0)], 148),
    ([(1, 128, 128, 4, 0, 0), (2, 256, 384, 3, 0, 1), (4, 128, 1024, 8, 0, 0)], 148),       # stages smaller than the grid
    ([(1, 512, 4096, 4, 0, 0), (1, 28672, 8192, 4, 0, 1)], 148),                            # 224 k-blocks: chunks of 96 units
    ([(3, 1024, 512, 2, 0, 0)], 5),
])
def test_cursor_walk_covers_every_unit_once(specs, num_sms):
    arr = _ops(specs)
    plan, per_cta = _walk(arr, num_sms)
    # stage structure
    stage_of, off, stage_units = [], [], []
    for i, sp in enumerate(specs):
        if i == 0 or sp[5]:
            stage_units.append(0)
        stage_of.append(len(stage_units) - 1); off.append(stage_units[-1])
        stage_units[-1] += (sp[1] // 128) * (sp[2] // 128)
    assert plan.stages == len(stage_units) and plan.units == sum(stage_units)
    assert plan.grid == min(num_sms, max(stage_units)) and 2 <= plan.ring_stages <= 16 and plan.smem_bytes <= 220 * 1024
    seen = set()
    for cta, w in enumerate(per_cta):
        assert (w[:, 4] == np.arange(len(w))).all()                          # seq is the running index
        prev = None
        for row in w:
            st, op, strip, kb, seq, rb, re, chunk = [int(v) for v in row]
            assert stage_of[op] == st
            key = (op, strip, kb)
            assert key not in seen
            seen.add(key)
            # stream-K order inside the stage: unit index in the stage's space ascends by one
            g = off[op] + strip * (specs[op][1] // 128) + kb
            if prev is not None and prev[0] == st:
                assert g == prev[1] + 1
            prev = (st, g)
            # the stage-space range of this CTA is [U c / Gs, U (c + 1) / Gs), Gs = min(grid, U): no CTA range in between is empty
            U = stage_units[st]
            Gs = min(plan.grid, U)
            assert cta < Gs and U * cta // Gs <= g < U * (cta + 1) // Gs
            # run = this CTA's units inside (op, strip); chunk = <= 96 consecutive units of the run holding seq
            assert rb <= seq < re
            sb, ln = chunk >> 16, chunk & 0xffff
            assert rb <= sb <= seq < sb + ln <= re and ln <= 96 and (sb - rb) % 96 == 0
        # runs: all units of a run share (op, strip) and are k-consecutive
        for rb in set(int(v) for v in w[:, 5]):
            rows = w[w[:, 5] == rb]
            assert len(set((int(r[1]), int(r[2])) for r in rows)) == 1
            assert (np.diff(rows[:, 3]) == 1).all() and int(rows[0, 4]) == rb and int(rows[-1, 4]) == int(rows[0, 6]) - 1
    total = sum((sp[1] // 128) * (sp[2] // 128) for sp in specs)
    assert len(seen) == total


def test_cta_of_unit_formula_holds_when_the_grid_exceeds_the_units():
    """The chain's grid is fixed while stage sizes vary, so a stage may have fewer units than CTAs: the split-K owner formula
    ((g + 1) G - 1) / U must still invert the partition [U c / G, U (c + 1) / G)."""
    for U in (1, 2, 3, 7, 32, 147, 148, 149, 1000):
        for G in (1, 2, 4, 148, 150):
            owner = {}
            for c in range(G):
                for g in range(U * c // G, U * (c + 1) // G):
                    owner[g] = c
            assert len(owner) == U
            for g in range(U):
                assert ((g + 1) * G - 1) // U == owner[g], (U, G, g)


def test_chain_validation_and_plan():
    from exllamav3_b200 import ext
    lib = ext.lib
    plan = ext._ChainPlan()
    bad = lambda specs, cb=2: lib.exl3b_chain_plan(_patch_cb(_ops(specs), cb), len(specs), 148, ctypes.byref(plan))
    assert bad([(1, 4096, 4096, 4, 0, 0)]) == 0 and plan.grid == 148 and plan.stages == 1 and plan.cache_bytes == 8192
    assert bad([(5, 4096, 4096, 4, 0, 0)]) == -4 and b"m <= 4" in lib.exl3b_last_error()
    assert bad([(1, 4096, 4096, 4, 0, 0)], cb=0) == -4 and b"mul1" in lib.exl3b_last_error()
    assert bad([(1, 4000, 4096, 4, 0, 0)]) == -4 and b"multiples of 128" in lib.exl3b_last_error()
    assert bad([(1, 4096, 4096, 9, 0, 0)]) == -4
    assert bad([(4, 14336, 4096, 4, 1, 0)]) == -4 and b"gated input" in lib.exl3b_last_error()
    assert bad([(4, 28672, 8192, 4, 0, 0)]) == 0 and plan.cache_bytes == 0                   # rows too long for the cache: recomputed per unit
    assert lib.exl3b_chain_plan(None, 0, 148, ctypes.byref(plan)) == -2
    # whole token: 32 layers + head in one chain
    specs = LLAMA_LAYER + ([(1, 4096, 4096, 4, 0, 1)] + LLAMA_LAYER[1:]) * 31 + [(1, 4096, 128256, 6, 0, 1)]
    assert bad(specs) == 0 and plan.stages == 4 * 32 + 1 and plan.ring_stages >= 8
    with pytest.raises(RuntimeError, match="empty"):
        ext.GemmChain([])
    with pytest.raises(RuntimeError, match="CUDA"):
        ext.GemmChain([dict(x=torch.zeros((1, 128), dtype=torch.half), trellis=torch.zeros((8, 8, 64), dtype=torch.int16),
                            y=torch.zeros((1, 128)), mul1=True)])


def _patch_cb(arr, cb):
    for a in arr:
        a.cb = cb
    return arr


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------

def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(got, ref):
    got = np.asarray(got, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
    d = got - ref
    return np.abs(d).max() / max(np.abs(ref).max(), 1e-30), np.sqrt((d ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def _mk(k, n, K, m, dev, seed=0):
    tr, suh, svh, x = orc.make_synthetic(k, n, K, m=m, seed=seed) if "seed" in orc.make_synthetic.__code__.co_varnames else orc.make_synthetic(k, n, K, m=m)
    return dict(tr=tr, suh=suh, svh=svh, x=x, d_tr=T(tr, dev), d_suh=T(suh, dev), d_svh=T(svh, dev), d_x=T(x, dev))


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_chain_single_op_vs_oracle(cuda, K, m):
    from exllamav3_b200 import ext
    for (k, n, fp32) in ((512, 384, True), (1024, 256, False), (128, 128, True)):
        t = _mk(k, n, K, m, cuda)
        y = torch.zeros((m, n), dtype=torch.float if fp32 else torch.half, device=cuda)
        ch = ext.GemmChain([dict(x=t["d_x"], trellis=t["d_tr"], suh=t["d_suh"], svh=t["d_svh"], y=y, mul1=True)])
        assert ch.run() == ext.EXL3B_TAG_TC_I8_CHAIN
        torch.cuda.synchronize()
        ref = orc.exl3_gemm_f64(t["x"], t["tr"], t["suh"], t["svh"], K, 2)
        mx, rms = rel_err(y.cpu().numpy(), ref)
        tol = (2e-3, 1e-3) if fp32 else (4e-3, 2e-3)                     # fp16 C: + output rounding
        assert mx <= tol[0] and rms <= tol[1], (K, m, k, n, mx, rms)
        # the exact model of the kernel's arithmetic (block-norm activation scale), per row
        model = orc.exl3_gemm_i8_model(t["x"], t["tr"], t["suh"], t["svh"], K, rule="blocknorm")
        for r in range(m):
            mx, rms = rel_err(y[r:r + 1].cpu().numpy(), model[r:r + 1])
            assert mx <= (2e-5 if fp32 else 1.5e-3) and rms <= (1e-5 if fp32 else 5e-4), (K, m, k, n, r, mx, rms)
        # replay: counters and exchange buffers re-armed
        y.zero_(); ch.run(); torch.cuda.synchronize()
        assert rel_err(y.cpu().numpy(), ref)[0] <= tol[0]
        ch.close()


@pytest.mark.gpu
def test_exl3_gemm_on_the_chain_kernel_matches_the_default_path(cuda):
    from exllamav3_b200 import ext
    for (k, n, K, m) in ((4096, 4096, 4, 1), (4096, 1024, 4, 3), (14336, 4096, 4, 1), (4096, 14336, 3, 2), (2048, 512, 6, 4)):
        t = _mk(k, n, K, m, cuda)
        xh = torch.empty_like(t["d_x"])
        y0 = torch.zeros((m, n), dtype=torch.float, device=cuda); y1 = torch.zeros_like(y0)
        assert ext.exl3_gemm(t["d_x"], t["d_tr"], y0, t["d_suh"], xh, t["d_svh"], -1, False, True, 0) == ext.EXL3B_TAG_TC_I8
        prev = ext.set_gemm_path(ext.EXL3B_TAG_TC_I8_CHAIN)
        try:
            assert ext.exl3_gemm(t["d_x"], t["d_tr"], y1, t["d_suh"], xh, t["d_svh"], -1, False, True, 0) == ext.EXL3B_TAG_TC_I8_CHAIN
        finally:
            ext.set_gemm_path(prev)
        torch.cuda.synchronize()
        mx, rms = rel_err(y1.cpu().numpy(), y0.cpu().numpy())
        assert mx <= 2e-3 and rms <= 5e-4, (k, n, K, m, mx, rms)          # same arithmetic up to the activation scale rule


@pytest.mark.gpu
def test_chain_same_input_stage_and_dependent_stage(cuda):
    """q + k + v style stage (three ops, one input) and a dependent stage reading an earlier output."""
    from exllamav3_b200 import ext
    k, K, m = 1024, 4, 2
    a = _mk(k, 512, K, m, cuda); b = _mk(k, 256, K, m, cuda); c = _mk(k, 256, 3, m, cuda)
    ya = torch.zeros((m, 512), dtype=torch.half, device=cuda)
    yb = torch.zeros((m, 256), dtype=torch.float, device=cuda); yc = torch.zeros((m, 256), dtype=torch.float, device=cuda)
    d = _mk(512, 384, 5, m, cuda)                                       # consumes ya (fp16 rows)
    yd = torch.zeros((m, 384), dtype=torch.float, device=cuda)
    x = a["d_x"]
    ch = ext.GemmChain([
        dict(x=x, trellis=a["d_tr"], suh=a["d_suh"], svh=a["d_svh"], y=ya, mul1=True),
        dict(x=x, trellis=b["d_tr"], suh=b["d_suh"], svh=b["d_svh"], y=yb, mul1=True),
        dict(x=x, trellis=c["d_tr"], suh=c["d_suh"], svh=c["d_svh"], y=yc, mul1=True),
        dict(x=ya, trellis=d["d_tr"], suh=d["d_suh"], svh=d["d_svh"], y=yd, mul1=True, new_stage=True),
    ])
    for _ in range(3):
        ya.zero_(); yd.zero_()
        ch.run()
    torch.cuda.synchronize()
    xa = a["x"]
    ra = orc.exl3_gemm_f64(xa, a["tr"], a["suh"], a["svh"], K, 2)
    assert rel_err(ya.cpu().numpy(), ra)[0] <= 4e-3
    assert rel_err(yb.cpu().numpy(), orc.exl3_gemm_f64(xa, b["tr"], b["suh"], b["svh"], K, 2))[0] <= 2e-3
    assert rel_err(yc.cpu().numpy(), orc.exl3_gemm_f64(xa, c["tr"], c["suh"], c["svh"], 3, 2))[0] <= 2e-3
    rd = orc.exl3_gemm_f64(ya.cpu().numpy(), d["tr"], d["suh"], d["svh"], 5, 2)       # from the kernel's own fp16 ya
    mx, rms = rel_err(yd.cpu().numpy(), rd)
    assert mx <= 2e-3 and rms <= 1e-3, (mx, rms)


def _silu_mul_ref(g, u):
    g = g.astype(np.float64); u = u.astype(np.float64)
    return (g / (1.0 + np.exp(-g)) * u).astype(np.float16)             # the reference rounds the product to fp16 (activation_kernels.cuh:200-240)


@pytest.mark.gpu
@pytest.mark.parametrize("fp32_gu", [True, False])
def test_chain_gated_mlp_block(cuda, fp32_gu):
    """gate + up -> silu * mul -> down in one launch == exl3_mgemm(gate, up), silu_mul, exl3_gemm(down) (mlp.cpp:38-90)."""
    from exllamav3_b200 import ext
    hid, inter, K, m = 512, 1792, 4, 1
    g = _mk(hid, inter, K, m, cuda); u = _mk(hid, inter, K, m, cuda); dn = _mk(inter, hid, K, m, cuda)
    u["tr"] = np.roll(u["tr"], 7, axis=1).copy(); u["d_tr"] = T(u["tr"], cuda)
    dt = torch.float if fp32_gu else torch.half
    yg = torch.zeros((m, inter), dtype=dt, device=cuda); yu = torch.zeros_like(yg)
    yd = torch.zeros((m, hid), dtype=torch.float, device=cuda)
    ch = ext.GemmChain([
        dict(x=g["d_x"], trellis=g["d_tr"], suh=g["d_suh"], svh=g["d_svh"], y=yg, mul1=True),
        dict(x=g["d_x"], trellis=u["d_tr"], suh=u["d_suh"], svh=u["d_svh"], y=yu, mul1=True),
        dict(gate=yg, up=yu, trellis=dn["d_tr"], suh=dn["d_suh"], svh=dn["d_svh"], y=yd, mul1=True, new_stage=True),
    ])
    for _ in range(2):
        yd.zero_(); ch.run()
    torch.cuda.synchronize()
    rg = orc.exl3_gemm_f64(g["x"], g["tr"], g["suh"], g["svh"], K, 2)
    assert rel_err(yg.cpu().numpy(), rg)[0] <= (2e-3 if fp32_gu else 4e-3)
    a = _silu_mul_ref(yg.cpu().numpy(), yu.cpu().numpy())              # activation of the kernel's own gate / up outputs
    rd = orc.exl3_gemm_f64(a, dn["tr"], dn["suh"], dn["svh"], K, 2)
    mx, rms = rel_err(yd.cpu().numpy(), rd)
    assert mx <= 3e-3 and rms <= 1.5e-3, (mx, rms)                      # + fast-math silu (__expf / __fdividef, as the reference's fp32 kernel)


@pytest.mark.gpu
def test_chain_llama_layer_shapes_blocks_vs_oracle(cuda):
    """The three launches a Llama-3.1-8B layer becomes (q+k+v | o | gate+up -> down) at full size: spot-checked 128-column blocks
    against the fp64 oracle, and against separate exl3_gemm calls on the default path."""
    from exllamav3_b200 import ext
    K, m = 4, 1
    hid, inter, kv = 4096, 14336, 1024
    rng = np.random.default_rng(5)
    mats = {nm: _mk(k, n, K, m, cuda) for nm, (k, n) in dict(q=(hid, hid), k=(hid, kv), v=(hid, kv), o=(hid, hid), gate=(hid, inter),
                                                             up=(hid, inter), down=(inter, hid)).items()}
    for nm in ("k", "v", "up"):
        mats[nm]["tr"] = np.roll(mats[nm]["tr"], 3 + len(nm), axis=0).copy(); mats[nm]["d_tr"] = T(mats[nm]["tr"], cuda)
    x = mats["q"]["d_x"]
    out = {nm: torch.zeros((m, t["tr"].shape[1] * 16), dtype=torch.half if nm in ("q", "k", "v") else torch.float, device=cuda) for nm, t in mats.items()}
    op = lambda nm, **kw: dict(trellis=mats[nm]["d_tr"], suh=mats[nm]["d_suh"], svh=mats[nm]["d_svh"], y=out[nm], mul1=True, **kw)
    chains = [ext.GemmChain([op("q", x=x), op("k", x=x), op("v", x=x)]),
              ext.GemmChain([op("o", x=out["q"])]),
              ext.GemmChain([op("gate", x=x), op("up", x=x), op("down", gate=out["gate"], up=out["up"], new_stage=True)])]
    for _ in range(2):
        for ch in chains:
            ch.run()
    torch.cuda.synchronize()
    xin = mats["q"]["x"]
    ins = dict(q=xin, k=xin, v=xin, gate=xin, up=xin, o=out["q"].cpu().numpy(),
               down=_silu_mul_ref(out["gate"].cpu().numpy(), out["up"].cpu().numpy()))
    for nm, t in mats.items():
        n = t["tr"].shape[1] * 16
        for blk in rng.choice(n // 128, 3, replace=False):
            sl = slice(blk * 128, blk * 128 + 128)
            ref = orc.exl3_gemm_f64(ins[nm], t["tr"][:, blk * 8: blk * 8 + 8, :], t["suh"], t["svh"][sl], K, 2)
            mx, rms = rel_err(out[nm][:, sl].cpu().numpy(), ref)
            tol = (4e-3, 2e-3) if out[nm].dtype == torch.half else (3e-3, 1.5e-3)
            assert mx <= tol[0] and rms <= tol[1], (nm, blk, mx, rms)
    # against the default single-GEMM path on the same input
    y_ref = torch.zeros_like(out["o"]); xh = torch.empty_like(out["q"])
    ext.exl3_gemm(out["q"], mats["o"]["d_tr"], y_ref, mats["o"]["d_suh"], xh, mats["o"]["d_svh"], -1, False, True, 0)
    torch.cuda.synchronize()
    assert rel_err(out["o"].cpu().numpy(), y_ref.cpu().numpy())[1] <= 5e-4
