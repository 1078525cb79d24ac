"""
Host side of the GEMM-chain exactness tests (tests/test_chain_exact.py), no GPU needed.

The chain kernel (csrc/chain_i8.cu, tag 220) quantises activations like the single-GEMM int8 kernel but takes its scale from a
block-norm bound instead of the row maximum; oracle.exl3_gemm_i8_model(rule="blocknorm") models that rule bit for bit.  This
file checks the model's own properties, asserts with the kernel's planner and cursor (exl3b_chain_plan / exl3b_chain_walk)
that the GPU file's layer, token and relay chains reach the regimes they are there for (scale-slot reuse, split-K exchange
buffers of both parities, stages smaller than the grid, the stage and op limits), and checks the pointer-alignment
validation.  It also owns what both files share: the chain tables and the adversarial inputs.
"""
import ctypes
import numpy as np
import pytest
from oracle import exl3_oracle as orc

SMS = 132
QMAX = 32512
CH_SCALE_SLOTS = 32                   # chain_i8.cu: scale slots, indexed by op % 32
CH_MAX_STAGES = 255

# ---- chain tables: ops as dicts (name, k, n, K, src, new_stage, fp32); src = "x" (external fp16 rows), the name of an earlier
# fp16 output, or ("gate name", "up name") for the gated input silu(gate) * up -----------------------------------------------

def layer_ops(l, H, I, KV, src, K=(4,), gu_fp32=True):
    """One decoder layer at reduced width: q + k + v | o (reads q) | gate + up (read o) | down (gated): 7 ops in 4 stages."""
    Ks = lambda j: K[(7 * l + j) % len(K)]
    p = f"{l}."
    return [dict(name=p + "q", k=H, n=H, K=Ks(0), src=src, new_stage=True, fp32=False),
            dict(name=p + "k", k=H, n=KV, K=Ks(1), src=src, new_stage=False, fp32=True),
            dict(name=p + "v", k=H, n=KV, K=Ks(2), src=src, new_stage=False, fp32=False),
            dict(name=p + "o", k=H, n=H, K=Ks(3), src=p + "q", new_stage=True, fp32=False),
            dict(name=p + "gate", k=H, n=I, K=Ks(4), src=p + "o", new_stage=True, fp32=gu_fp32),
            dict(name=p + "up", k=H, n=I, K=Ks(5), src=p + "o", new_stage=False, fp32=gu_fp32),
            dict(name=p + "down", k=I, n=H, K=Ks(6), src=(p + "gate", p + "up"), new_stage=True, fp32=False,
                 in_mode=1 if gu_fp32 else 2)]


LAYER = dict(H=512, I=1024, KV=256, m=4)
TOKEN = dict(H=512, I=1024, KV=256, V=8192, layers=8, m=1)      # one row: rows of one op drift apart through silu


def layer_chain():
    return layer_ops(0, LAYER["H"], LAYER["I"], LAYER["KV"], "x")


def token_chain():
    """TOKEN["layers"] layers and a head, bitrates 2..6 mixed (the kernel's any-K instantiation), gate / up outputs alternating
    between fp32 and fp16 (both gated input modes)."""
    H, I, KV = TOKEN["H"], TOKEN["I"], TOKEN["KV"]
    ops, src = [], "x"
    for l in range(TOKEN["layers"]):
        ops += layer_ops(l, H, I, KV, src, K=(2, 3, 4, 5, 6), gu_fp32=l % 2 == 0)
        src = f"{l}.down"
    ops.append(dict(name="head", k=H, n=TOKEN["V"], K=4, src=src, new_stage=True, fp32=True))
    return ops


def relay_chain(n_stages=CH_MAX_STAGES):
    """n_stages ops, each reading the previous op's fp16 output: a wide first stage (so that the grid is the SM count), a
    16-unit second stage, then one-unit stages."""
    ops = [dict(name="r0", k=2048, n=2048, K=4, src="x", new_stage=True, fp32=False),
           dict(name="r1", k=2048, n=128, K=3, src="r0", new_stage=True, fp32=False)]
    for i in range(2, n_stages):
        ops.append(dict(name=f"r{i}", k=128, n=128, K=2 + i % 5, src=f"r{i - 1}", new_stage=True, fp32=i == n_stages - 1))
    return ops


def plan_array(ops, m, ptrs=None):
    """ctypes op table for the host-only entry points: dummy aligned pointers, or per-op overrides ptrs[i] = dict(A=..)."""
    from exllamav3_b200 import ext
    arr = (ext._ChainOp * len(ops))()
    for i, (a, o) in enumerate(zip(arr, ops)):
        in_mode = o.get("in_mode", 0)
        a.A = a.B = a.C = a.suh = a.svh = 4096
        a.A2 = 4096 if in_mode else None
        for nm, v in (ptrs[i] if ptrs else {}).items():
            setattr(a, nm, v)
        a.m, a.k, a.n, a.K, a.cb, a.c_fp32 = o.get("m", m), o["k"], o["n"], o["K"], 2, int(o["fp32"])
        a.in_mode, a.new_stage = in_mode, int(o["new_stage"])
    return arr


def chain_plan(arr, sms=SMS):
    from exllamav3_b200 import ext
    plan = ext._ChainPlan()
    r = ext.lib.exl3b_chain_plan(arr, len(arr), sms, ctypes.byref(plan))
    return r, plan


def chain_regimes(ops, m, sms=SMS):
    """Per stage: units, and whether some output strip is split over more than one CTA (split-K through the exchange buffer
    of parity stage & 1), from the kernel's own cursor."""
    from exllamav3_b200 import ext
    arr = plan_array(ops, m)
    r, plan = chain_plan(arr, sms)
    assert r == 0, ext.lib.exl3b_last_error()
    owners = {}
    for cta in range(plan.grid):
        buf = np.zeros((8192, 8), dtype=np.int32)
        n = ext.lib.exl3b_chain_walk(arr, len(arr), sms, cta, buf.ctypes.data, 8192)
        assert 0 <= n <= 8192
        for st, op, strip in buf[:n, :3]:
            owners.setdefault((int(st), int(op), int(strip)), set()).add(cta)
    units = [0] * plan.stages
    split = [False] * plan.stages
    st = -1
    for o in ops:
        st += bool(o["new_stage"]) or st < 0
        units[st] += (o["k"] // 128) * (o["n"] // 128)
    for (s, _, _), ctas in owners.items():
        split[s] |= len(ctas) > 1
    return plan, units, split


# ---- adversarial inputs ----------------------------------------------------------------------------------------------

def pow2_suh(k, seed):
    """suh = +-2^e, e in {-5, -4, -3}: products x * suh of power-of-two-scaled values are exact in fp16."""
    rng = np.random.default_rng(seed)
    return (np.sign(rng.standard_normal(k)) * np.exp2(rng.integers(-5, -2, k))).astype(np.float16)


def hadamard_aligned_row(k, suh, seed, c=0.25):
    """x with x * suh = c * (a Hadamard row) in every 128-block, exactly: xh has one entry c sqrt(128) per block and zeros,
    and the block-norm bound equals max |xh| up to the 1.002 margin."""
    H = orc.hadamard_matrix_128()
    j = np.random.default_rng(seed).integers(0, 128, k // 128)
    t = np.concatenate([c * H[jj] for jj in j])
    return (t / suh.astype(np.float64)).astype(np.float16)


def adversarial_rows(k, suh, seed):
    """Four rows: zero; Hadamard-aligned (tight bound); Gaussian with one block x 300 (outlier block); x * suh fp16-subnormal."""
    rng = np.random.default_rng(seed)
    x = np.zeros((4, k), dtype=np.float16)
    x[1] = hadamard_aligned_row(k, suh, seed)
    g = rng.standard_normal(k)
    b = rng.integers(0, k // 128)
    g[b * 128:(b + 1) * 128] *= 300.0
    x[2] = g.astype(np.float16)
    sub = rng.standard_normal(k) * 2.0 ** -18 / np.abs(suh.astype(np.float64))        # |x * suh| ~ 2^-18 < 2^-14
    x[3] = sub.astype(np.float16)
    return x


def exact_gates(shape, seed):
    """Gates in {0} u [20, 60]: the kernel's fast-math silu returns exactly g or 0 there, so the gated input is exact."""
    rng = np.random.default_rng(seed)
    g = rng.uniform(20.0, 60.0, shape)
    g[rng.random(shape) < 0.3] = 0.0
    return g


# ---- tests: the model ------------------------------------------------------------------------------------------------

def _xh(x, suh):
    return orc.had_r_128(np.ascontiguousarray(x, dtype=np.float16), pre_scale=suh).astype(np.float32)


def test_rowmax_rule_is_the_default():
    tr, suh, svh, x = orc.make_synthetic(512, 256, 3, m=4)
    for a, b in zip(orc.i8_activation_q(x, suh), orc.i8_activation_q(x, suh, rule="rowmax")):
        assert np.array_equal(a, b)
    mx = np.abs(_xh(x, suh)).max(axis=1, keepdims=True)
    q, scale = orc.i8_activation_q(x, suh)
    assert np.abs(q).max() == QMAX and np.array_equal(scale, (mx / np.float32(QMAX)).astype(np.float64))
    with pytest.raises(ValueError):
        orc.i8_activation_q(x, suh, rule="max")


def test_blocknorm_bound_follows_the_kernel_reduction():
    """The bound is the fp32 butterfly of the kernel, not an fp64 norm: it matches a direct scalar restatement of chain_i8.cu
    bit for bit and is within fp32 round-off of sqrt(max block ||x * suh||^2) * 1.002."""
    k = 1024
    _, suh, _, _ = orc.make_synthetic(k, 128, 4, seed=3)
    x = (np.random.default_rng(4).standard_normal((3, k)) * [[1.0], [1e-3], [50.0]]).astype(np.float16)
    b = orc.i8_blocknorm_bound(x, suh)
    t = (x.astype(np.float64) * suh.astype(np.float64)).astype(np.float16).astype(np.float32)
    for r in range(3):
        n2 = np.float32(0)
        for kb in range(k // 128):
            s = [np.float32(0)] * 32
            for l in range(32):
                v = t[r, kb * 128 + 4 * l: kb * 128 + 4 * l + 4]
                s[l] = np.float32(np.float32(np.float32(v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]) + v[3] * v[3])
            for d in (16, 8, 4, 2, 1):
                s = [np.float32(s[l] + s[l ^ d]) for l in range(32)]
            assert len(set(float(v) for v in s)) == 1
            n2 = max(n2, s[0])
        assert b[r, 0] == np.float32(np.sqrt(n2, dtype=np.float32) * np.float32(1.002))
        exact = np.sqrt((t[r].astype(np.float64).reshape(-1, 128) ** 2).sum(axis=1).max()) * 1.002
        assert abs(b[r, 0] / exact - 1) < 1e-6
    assert orc.i8_blocknorm_bound(np.zeros((1, k), np.float16), suh)[0, 0] == 0


def test_blocknorm_q_stays_in_range_on_adversarial_rows():
    """|q| <= 32512 (hi digit in [-127, 127]) on every row shape that pushes max |xh| towards its block norm."""
    k = 2048
    rng = np.random.default_rng(11)
    suh_r = orc.make_synthetic(k, 128, 4, seed=12)[1]
    for suh in (suh_r, pow2_suh(k, 13)):
        rows = [adversarial_rows(k, suh, s) for s in range(3)]
        rows.append(np.stack([hadamard_aligned_row(k, suh, s, c) for s, c in ((20, 1.0), (21, 2.0 ** -6), (22, 8.0))]))
        spike = np.zeros((3, k)); spike[0, 5] = 60000.0; spike[1, ::128] = 1.0; spike[2, :] = 1.0
        rows.append(spike.astype(np.float16))
        rows.append(np.clip(rng.standard_cauchy((8, k)), -6e4, 6e4).astype(np.float16))
        rows.append((rng.standard_normal((8, k)) * np.exp2(rng.integers(-20, 10, (8, 1)))).astype(np.float16))
        for x in rows:
            xh = _xh(x, suh)
            b = orc.i8_blocknorm_bound(x, suh)
            assert (b[:, 0] >= np.abs(xh).max(axis=1)).all()
            q, scale = orc.i8_activation_q(x, suh, rule="blocknorm")
            assert np.abs(q).max() <= QMAX
            hi = (q + 128) >> 8
            assert np.abs(hi).max() <= 127
            assert np.array_equal(scale, (b / np.float32(QMAX)).astype(np.float64))
        assert (orc.i8_activation_q(rows[0], suh, rule="blocknorm")[0][0] == 0).all()        # zero row: q = 0, scale 0


def test_blocknorm_bound_is_tight_on_a_hadamard_aligned_row():
    for k in (128, 1024, 4096):
        suh = pow2_suh(k, k)
        x = np.stack([hadamard_aligned_row(k, suh, s) for s in range(4)])
        xh = _xh(x, suh)
        b = orc.i8_blocknorm_bound(x, suh)[:, 0]
        ratio = b / np.abs(xh).max(axis=1)
        assert (ratio >= 1.0).all() and (ratio <= 1.003).all(), ratio
        q, _ = orc.i8_activation_q(x, suh, rule="blocknorm")
        assert (np.abs(q).max(axis=1) >= 0.99 * QMAX).all() and np.abs(q).max() <= QMAX
        # the 1.002 margin is what keeps q in range: without it the largest |q| would exceed the hi digit's range
        assert (np.abs(xh).max(axis=1) * np.float32(QMAX) / (b / np.float32(1.002) * np.float32(0.99)) > QMAX + 128).all()


def test_blocknorm_costs_about_two_bits_on_gaussian_rows():
    """On Gaussian rows the bound is ~3.5x the row maximum (the header comment of chain_i8.cu), i.e. ~14 of 16 bits."""
    for k, lo, hi in ((512, 3.4, 4.1), (4096, 3.2, 3.8), (14336, 3.1, 3.6)):
        _, suh, _, _ = orc.make_synthetic(k, 128, 4, seed=k + 1)
        x = np.random.default_rng(k).standard_normal((256, k)).astype(np.float16)
        ratio = orc.i8_blocknorm_bound(x, suh)[:, 0] / np.abs(_xh(x, suh)).max(axis=1)
        assert lo <= np.median(ratio) <= hi and ratio.min() >= 2.0 and ratio.max() <= 5.0, (k, np.median(ratio), ratio.min(), ratio.max())


def test_exact_gates_make_the_gated_input_exact():
    g = exact_gates((4, 1024), 5)
    u = np.random.default_rng(6).standard_normal((4, 1024))
    for dt in (np.float32, np.float16):
        gg, uu = g.astype(dt), u.astype(dt)
        h = orc.chain_gated_input(gg, uu)
        want = (gg.astype(np.float32) * uu.astype(np.float32)).astype(np.float32).astype(np.float16)
        want[gg == 0] = 0
        assert np.array_equal(h.view(np.uint16) & 0x7fff, want.view(np.uint16) & 0x7fff)


def test_blocknorm_model_agrees_with_the_f64_oracle():
    """The model is the kernel's arithmetic: within the path's approximation error of the fp64 oracle (README, Parity)."""
    for K in (2, 4, 7):
        tr, suh, svh, x = orc.make_synthetic(1024, 256, K, m=4)
        y = orc.exl3_gemm_i8_model(x, tr, suh, svh, K, rule="blocknorm")
        ref = orc.exl3_gemm_f64(x, tr, suh, svh, K, 2)
        d = y - ref
        assert np.abs(d).max() <= 2e-3 * np.abs(ref).max() and np.sqrt((d ** 2).mean()) <= 1e-3 * np.sqrt((ref ** 2).mean())


# ---- tests: regimes of the GPU tables --------------------------------------------------------------------------------

def test_layer_chain_plan():
    ops = layer_chain()
    plan, units, split = chain_regimes(ops, LAYER["m"])
    assert len(ops) == 7 and plan.stages == 4 and plan.units == sum(units)
    assert all(split) and plan.grid == min(SMS, max(units))


def test_token_chain_reaches_slot_reuse_both_exchange_buffers_and_small_stages():
    ops = token_chain()
    plan, units, split = chain_regimes(ops, TOKEN["m"])
    assert len(ops) > CH_SCALE_SLOTS                                     # op % 32 reuses scale slots
    assert plan.stages == 4 * TOKEN["layers"] + 1 and plan.stages > 2     # stage counters past index 1
    assert plan.grid == SMS and any(u < plan.grid for u in units)         # stages with fewer units than the grid
    assert any(split[s] for s in range(0, plan.stages, 2)) and any(split[s] for s in range(1, plan.stages, 2))
    assert len(set(o["K"] for o in ops)) > 1                               # mixed bitrates: the any-K instantiation


def test_relay_chain_reaches_the_stage_limit():
    ops = relay_chain()
    plan, units, split = chain_regimes(ops, 1)
    assert plan.stages == CH_MAX_STAGES and plan.grid == SMS
    assert units[0] > plan.grid and all(u < plan.grid for u in units[1:]) and split[1]
    r, _ = chain_plan(plan_array(relay_chain(CH_MAX_STAGES + 1), 1))
    assert r == -4


def test_stage_and_op_limits():
    from exllamav3_b200 import ext
    one = dict(k=128, n=128, K=2, src="x", fp32=True)
    assert chain_plan(plan_array([dict(one, new_stage=False)] * 4096, 1))[0] == 0
    r, _ = chain_plan(plan_array([dict(one, new_stage=False)] * 4097, 1))
    assert r == -2 and b"too many ops" in ext.lib.exl3b_last_error()
    ops = [dict(one, new_stage=i % 16 == 0) for i in range(255 * 16)]
    r, plan = chain_plan(plan_array(ops, 1))
    assert r == 0 and plan.stages == 255
    r, _ = chain_plan(plan_array(ops + [dict(one, new_stage=True)], 1))
    assert r == -4 and b"255 stages" in ext.lib.exl3b_last_error()


def test_mixed_m_chain_plans():
    ops = [dict(k=512, n=256, K=4, src="x", new_stage=False, fp32=True, m=m) for m in (4, 1, 3)]
    ops.append(dict(k=256, n=512, K=3, src="x", new_stage=True, fp32=False, m=1))
    assert chain_plan(plan_array(ops, 4))[0] == 0


# ---- tests: alignment validation -------------------------------------------------------------------------------------

ALIGN_CASES = [
    # (in_mode, c_fp32, field, offset, accepted, message)
    (0, 1, "A", 8, True, None),                       # 8-byte aligned rows: supported, read uncached
    (0, 1, "A", 4, False, b"A must be 8-byte aligned"),
    (0, 1, "A", 2, False, b"A must be 8-byte aligned"),
    (1, 1, "A", 8, False, b"gate (A) must be 16-byte aligned"),
    (1, 1, "A2", 8, False, b"up (A2) must be 16-byte aligned"),
    (1, 1, "A2", 4, False, b"up (A2) must be 16-byte aligned"),
    (2, 1, "A", 8, True, None),
    (2, 1, "A", 4, False, b"gate (A) must be 8-byte aligned"),
    (2, 1, "A2", 2, False, b"up (A2) must be 8-byte aligned"),
    (0, 1, "suh", 8, True, None),                     # suh at 8 bytes: read from global memory instead of the bulk copy
    (0, 1, "suh", 4, False, b"suh must be 8-byte aligned"),
    (0, 1, "svh", 2, False, b"svh must be 8-byte aligned"),
    (0, 1, "svh", 8, True, None),
    (0, 1, "C", 8, False, b"C must be 16-byte aligned"),
    (0, 0, "C", 8, True, None),
    (0, 0, "C", 4, False, b"C must be 8-byte aligned"),
]


@pytest.mark.parametrize("in_mode,c_fp32,field,offset,accepted,message", ALIGN_CASES)
def test_misaligned_pointers_are_rejected(in_mode, c_fp32, field, offset, accepted, message):
    from exllamav3_b200 import ext
    op = dict(k=1024, n=256, K=4, src="x", new_stage=False, fp32=bool(c_fp32), in_mode=in_mode)
    ok = dict(k=512, n=128, K=4, src="x", new_stage=False, fp32=True)
    ptrs = [{}, {"A2": 4096 if in_mode else None, field: 4096 + offset}]
    r, _ = chain_plan(plan_array([ok, op], 2, ptrs))
    if accepted:
        assert r == 0, ext.lib.exl3b_last_error()
    else:
        assert r == -2 and b"op 1: " + message in ext.lib.exl3b_last_error()
