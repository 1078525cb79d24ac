"""
Host side of tests/test_bench_token_exact.py, no GPU needed.

The GPU file holds every output of bench.py's decode token to the int8 path's exact model (oracle.exl3_gemm_i8_model), with the
integer contraction of the model run on the GPU by oracle.exl3_oracle_torch.  This file checks that restatement against the numpy
model (exactly, on the CPU device), the W_hat table against reconstruct, and -- with the planners the launchers call -- that the
tokens the GPU file runs really reach the schedules a fault of the int8 decode-GEMM's unit walk would hide in: single-GEMM CTAs
with more than one 96-unit accumulation chunk, CTAs that start and end inside a strip, strips reduced from several CTAs, decode
groups with an odd unit count, and fan-out CTA groups with a 128-column member.  A planner change that drops one of these fails
here instead of leaving the GPU test with nothing to test.

It also owns what both files share: the token list, the per-launch geometry, the strip -> CTA / unit map of failure messages and
the fault sites.
"""
import ctypes
import sys
import numpy as np
import pytest
import torch
from conftest import ROOT
from oracle import exl3_oracle as orc
from oracle import exl3_oracle_torch as ot
from test_edges_host import I8_SUB_UNITS, SMS, TAG_I8, _lib, gemm_plan

sys.path.insert(0, ROOT)
import bench

# the tokens the GPU file runs: bench.py's token, and the rank-0 shards `bench.py --tp-shapes N` runs
TOKENS = (("llama-3.1-8b", 1), ("llama-3.1-8b", 2), ("llama-3.1-8b", 4), ("llama-3.1-8b", 8), ("llama-3.1-70b", 8))
TINY = dict(hidden=256, inter=512, q=256, kv=128, layers=2, vocab=640, K=4, head_K=6)


# ---- launch geometry --------------------------------------------------------------------------------------------------------

def token_launches(cfg, tp):
    """bench.Token's default launch list (q + k + v fan-out, o, gate + up, down per layer, then lm_head) from the shapes alone:
    [(kind, ((name, k, n, K), ...))] with kind "fanout", "mgemm" or "gemm"; one entry per distinct layer (every layer is alike)."""
    layer, head = bench.token_plan(cfg, tp)
    s = {name: (name, k, n, K) for (name, k, n, K, _, _) in layer}
    return [("fanout", (s["q"], s["k"], s["v"])), ("gemm", (s["o"],)), ("mgemm", (s["gate"], s["up"])), ("gemm", (s["down"],)),
            ("gemm", (head[:4],))]


def launch_kind(ln):
    """The kind of a launch of bench.Token's lists in the terms of token_launches."""
    return ln["kind"] if ln["kind"] == "gemm" else ("fanout" if ln["cp"] is not None else "mgemm")


def matrix_grids(kind, mats, m=1, sms=SMS):
    """[(U, G, KB)] per matrix of a launch: its units, the CTAs of its group and its k-blocks, as the launchers plan them."""
    k, K = mats[0][1], mats[0][3]
    KB = k // 128
    U = [KB * (n // 128) for (_, _, n, _) in mats]
    if kind == "gemm":
        return [(U[0], gemm_plan(m, k, mats[0][2], K, 2, sms=sms).grid, KB)]
    if kind == "mgemm":                                       # gemm_tc_i8.cu launch_mgemm_tc_i8: sms / mats CTAs each
        return [(u, min(sms // len(mats), u), KB) for u in U]
    from exllamav3_b200 import ext
    cta0 = ext.plan_fanout(k, [n for (_, _, n, _) in mats], sms)
    assert cta0 is not None, ("fan-out not eligible", mats)
    return [(u, cta0[j + 1] - cta0[j], KB) for j, u in enumerate(U)]


def unit_ranges(U, G):
    L = _lib()
    b, e = ctypes.c_int64(), ctypes.c_int64()
    out = []
    for c in range(G):
        assert L.exl3b_plan_unit_range(U, G, c, ctypes.byref(b), ctypes.byref(e)) == 0
        out.append((b.value, e.value))
    return out


def strip_writers(U, G, KB, strip):
    """The CTAs that wrote a 128-column strip and their units of it: [(cta, first unit, last unit)] (unit = strip * KB + kb)."""
    L = _lib()
    c_a, c_b = L.exl3b_plan_cta_of_unit(U, G, strip * KB), L.exl3b_plan_cta_of_unit(U, G, strip * KB + KB - 1)
    rng = unit_ranges(U, G)
    return [(c, max(rng[c][0], strip * KB), min(rng[c][1], strip * KB + KB) - 1) for c in range(c_a, c_b + 1)]


def sub_segments(b, e, KB):
    """The epilogue's sub-segments of a CTA's units [b, e): strip ends and every I8_SUB_UNITS units (gemm_tc_i8_body.cuh)."""
    out, u = [], b
    while u < e:
        seg_end = min(e, (u // KB + 1) * KB)
        while u < seg_end:
            out.append((u, min(seg_end, u + I8_SUB_UNITS)))
            u = out[-1][1]
    return out


def fault_unit(k, n, K, m=1, sms=SMS):
    """Where the catalog puts a one-unit fault of a single-GEMM launch: the last unit of the last sub-segment of the CTA with the
    most units.  Returns (strip, kb, cta, units of that CTA, sub-segments of that CTA)."""
    U, G, KB = matrix_grids("gemm", (("", k, n, K),), m, sms)[0]
    rng = unit_ranges(U, G)
    cta = max(range(G), key=lambda c: rng[c][1] - rng[c][0])
    segs = sub_segments(*rng[cta], KB)
    u = segs[-1][1] - 1
    return u // KB, u % KB, cta, rng[cta][1] - rng[cta][0], segs


def census(tokens=TOKENS, sms=SMS):
    """What the launches of the tokens reach, per regime: a list of (model, tp, launch kind, matrix name) that reach it."""
    seen = {r: [] for r in ("gemm_cta_over_96_units", "cta_starts_and_ends_inside_a_strip", "strip_from_several_ctas",
                            "odd_units_per_decode_group", "fanout_with_128_column_member")}
    for (model, tp) in tokens:
        for kind, mats in token_launches(bench.MODELS[model], tp):
            where = lambda j: (model, tp, kind, mats[j][0])
            if kind == "fanout" and any(n == 128 for (_, _, n, _) in mats):
                seen["fanout_with_128_column_member"].append(where(0))
            for j, (U, G, KB) in enumerate(matrix_grids(kind, mats, sms=sms)):
                rng = unit_ranges(U, G)
                if kind == "gemm" and max(e - b for (b, e) in rng) > I8_SUB_UNITS:
                    seen["gemm_cta_over_96_units"].append(where(j))
                if any(b % KB and e % KB and b // KB == (e - 1) // KB for (b, e) in rng):
                    seen["cta_starts_and_ends_inside_a_strip"].append(where(j))
                if any(len(strip_writers(U, G, KB, s)) > 1 for s in range(0, U // KB, max(1, U // KB // 64))):
                    seen["strip_from_several_ctas"].append(where(j))
                # decode group g takes the CTA's units of parity g: (n_units - g + 1) // 2 of them
                if any(((e - b - g + 1) // 2) % 2 for (b, e) in rng for g in (0, 1)):
                    seen["odd_units_per_decode_group"].append(where(j))
    return seen


# ---- faults of the unit walk, applied to the model --------------------------------------------------------------------------

K_INV = float(orc._half_from_bits(orc.MUL1_K_INV_BITS))
C1 = 1534.0 * K_INV + float(orc._half_from_bits(orc.MUL1_K_BIAS_BITS))          # i8_math.cuh i8_assemble's c1


def _unit_bsum(trellis_host, K, strip, kb):
    """(128, 128) byte sums of unit (strip, kb) of a trellis (numpy, or a tensor on any device)."""
    t = trellis_host[kb * 8:kb * 8 + 8, strip * 8:strip * 8 + 8]
    t = t.cpu().numpy() if isinstance(t, torch.Tensor) else t
    return orc.mul1_bytesum(np.ascontiguousarray(t), K)


def unit_faults(x, trellis_host, suh, svh, K, pre, strip, kb, fp32):
    """
    {fault: C of a kernel with that fault} of the int8 decode-GEMM at one 128 x 128 unit (strip, kb), from the model's pieces: pre
    is the model before the svh multiply (exl3_gemm_i8_model with svh None), the fault's change to the unit's accumulators goes
    through the same scale and output Hadamard.  trellis_host: the matrix's trellis (numpy or a tensor), only its units around
    (strip, kb) are read.
    """
    q, scale = orc.i8_activation_q(x, suh)
    KB = q.shape[1] // 128
    H = orc.hadamard_matrix_128() * float(orc.R_SCALE_F32)
    cols = slice(strip * 128, strip * 128 + 128)
    out = lambda y_pre, s=svh: orc.i8_model_output(y_pre, s, np.float32 if fp32 else np.float16)

    def with_acc_delta(d_qb, d_t):
        """the unit's contraction changed by d_qb (m, 128) and its digit sums by d_t (m, 1)"""
        y = pre.copy()
        d = np.broadcast_to((K_INV * d_qb + C1 * d_t) * scale, (pre.shape[0], 128))
        y[:, cols] += d @ H
        return out(y)

    qk = q[:, kb * 128:kb * 128 + 128]
    bs = _unit_bsum(trellis_host, K, strip, kb)
    u_qb, u_t = qk @ (bs - 510), qk.sum(axis=1, keepdims=True)
    g = strip * KB + kb
    bs_prev = _unit_bsum(trellis_host, K, (g - 1) // KB, (g - 1) % KB) if g > 0 else np.full_like(bs, 510)
    kb_n = kb + 1 if kb + 1 < KB else kb - 1
    hi = (qk + 128) >> 8                                                  # i8_math.cuh i8_digits
    bs_d = bs.copy(); bs_d[64:] = bs[:64]
    svh_g = svh.copy()
    nb = strip + 1 if (strip + 1) * 128 < svh.shape[0] else strip - 1
    svh_g[cols] = svh[nb * 128:nb * 128 + 128]
    f = {
        "(a) unit skipped": with_acc_delta(-u_qb, -u_t),
        "(b) split-K partial added twice": with_acc_delta(u_qb, u_t),
        "(c) unit decoded from the previous ring stage": with_acc_delta(qk @ (bs_prev - bs), 0),
        "(d) k-half 1 decoded from k-half 0's words": with_acc_delta(qk @ (bs_d - bs), 0),
        "(e) lo digit dropped": with_acc_delta((256 * hi - qk) @ (bs - 510), (256 * hi - qk).sum(axis=1, keepdims=True)),
        "(f) digit sums of the neighbouring k-block": with_acc_delta(0, q[:, kb_n * 128:kb_n * 128 + 128].sum(axis=1, keepdims=True) - u_t),
        "(g) svh of the neighbouring strip": out(pre, svh_g),
    }
    if not fp32:
        f["(h) svh applied before the fp16 rounding"] = (pre * svh.astype(np.float64)[None, :]).astype(np.float16)
    return f


# ---- tests ------------------------------------------------------------------------------------------------------------------

def _constant_state_trellis(tk, tn, K, state):
    """A trellis whose every tile position has the given state (a 16-bit window of a K-periodic bitstream)."""
    tr = orc.pack_states(np.full((tk, tn, 256), state, dtype=np.uint16), K).view(np.int16)
    assert (orc.unpack_states(tr, K) == state).all()
    return tr


def _extreme_states(K):
    """The constant-window states of K-bit symbols with the smallest and the largest byte sum."""
    def window(p):
        bits = [(p >> (K - 1 - i)) & 1 for i in range(K)] * (16 // K + 2)
        return int("".join(map(str, bits[-16:])), 2)
    states = sorted({window(p) for p in range(2 ** K)})
    sums = [int(orc.mul1_bytesum(_constant_state_trellis(8, 8, K, s), K)[0, 0]) for s in states]
    return states[int(np.argmin(sums))], states[int(np.argmax(sums))], min(sums), max(sums)


@pytest.mark.parametrize("K", range(1, 9))
def test_contraction_equals_numpy(K):
    """The torch byte sums and contraction equal the numpy model's q @ (mul1_bytesum - 510) exactly (CPU device)."""
    rng = np.random.default_rng(K)
    k, n = 512, 384
    tr = rng.integers(0, 65536, size=(k // 16, n // 16, 16 * K), dtype=np.uint16).view(np.int16)
    lo, hi, s_lo, s_hi = _extreme_states(K)
    assert s_lo == 0 and s_hi >= 400
    tr[:8, :8] = _constant_state_trellis(8, 8, K, lo)                 # unit (0, 0): byte sum 0 everywhere
    tr[8:16, 8:16] = _constant_state_trellis(8, 8, K, hi)             # unit (1, 1): the largest byte sum K-bit symbols reach
    q = rng.integers(-orc.I8_QMAX, orc.I8_QMAX + 1, size=(4, k))
    q[0] = orc.I8_QMAX; q[1] = -orc.I8_QMAX                               # rows at |q| = 32512
    t = torch.from_numpy(tr)
    bs = ot.mul1_bytesum(t, K).numpy()
    want_bs = orc.mul1_bytesum(tr, K)
    assert np.array_equal(bs, want_bs) and (want_bs[:128, :128] == 0).all() and (want_bs[128:256, 128:256] == s_hi).all()
    assert np.array_equal(ot.unpack_states(t, K).numpy(), orc.unpack_states(tr, K).astype(np.int64))
    # in chunks of one strip and in one chunk
    for elems in (1, ot.CHUNK_ELEMS):
        qb = ot.i8_contract(t, K, q, elems=elems)
        assert qb.dtype == np.float64 and np.array_equal(qb, (q @ (want_bs - 510)).astype(np.float64))


def test_contraction_exact_at_the_bound():
    """At the arithmetic bound of the argument in i8_contract -- |q| = 32512 of one sign, byte sums 0 or 1020, k = 28672 -- the
    fp64 contraction is the exact integer (a 1020 byte sum is not reachable from 16-bit states, 1005 is the largest)."""
    k = 28672
    rng = np.random.default_rng(5)
    q = np.stack([np.full(k, orc.I8_QMAX), np.full(k, -orc.I8_QMAX), rng.integers(-orc.I8_QMAX, orc.I8_QMAX + 1, k)])
    bs = np.stack([np.zeros(k, np.int64), np.full(k, 1020), rng.integers(0, 1021, k)], axis=1)
    got = ot.centred_contract(torch.from_numpy(q.astype(np.float64)), torch.from_numpy(bs)).numpy()
    want = q @ (bs - 510)
    assert np.abs(want).max() == orc.I8_QMAX * 510 * k and np.array_equal(got, want.astype(np.float64))
    # the same through i8_contract at k = 28672 (the 70B down projection's rows)
    tr = rng.integers(0, 65536, size=(k // 16, 8, 64), dtype=np.uint16).view(np.int16)
    qb = ot.i8_contract(torch.from_numpy(tr), 4, q)
    assert np.array_equal(qb, (q @ (orc.mul1_bytesum(tr, 4) - 510)).astype(np.float64))


@pytest.mark.parametrize("fp32", (True, False))
def test_split_model_is_bit_identical(fp32):
    """exl3_gemm_i8_model(..., qb=i8_contract(...)) and the f64 oracle from the device contraction equal the unsplit models."""
    K, k, n, m = 4, 1024, 512, 2
    tr, suh, svh, x = orc.make_synthetic(k, n, K, m=m)
    q, _ = orc.i8_activation_q(x, suh)
    xh = orc.had_r_128(x, pre_scale=suh)
    qb, acc = ot.i8_contract(torch.from_numpy(tr), K, q, xh)
    assert np.array_equal(orc.exl3_gemm_i8_model(x, None, suh, svh, K, qb=qb), orc.exl3_gemm_i8_model(x, tr, suh, svh, K))
    pre = orc.exl3_gemm_i8_model(x, None, suh, None, K, qb=qb)
    dt = np.float32 if fp32 else np.float16
    a, b = orc.i8_model_output(pre, svh, dt), orc.i8_model_output(orc.exl3_gemm_i8_model(x, tr, suh, None, K), svh, dt)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    # the f64 oracle: same W_hat bits, the fp64 sums may only be reordered
    ref = orc.exl3_gemm_f64(x, tr, suh, svh, K, 2)
    assert np.abs(orc.exl3_gemm_f64(None, None, None, svh, K, 2, acc=acc) - ref).max() <= 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("K", (2, 4, 6))
def test_w_table_equals_reconstruct(K):
    """W_hat from the byte-sum table is reconstruct(trellis, K, 2) bit for bit; the table is decode_values' arithmetic."""
    tr, _, _, _ = orc.make_synthetic(512, 640, K)
    w = ot.mul1_weights(torch.from_numpy(tr), K, elems=512 * 256)
    assert np.array_equal(w.view(np.uint16), orc.reconstruct(tr, K, 2).view(np.uint16))
    st = np.arange(65536, dtype=np.uint16)
    x = (st.astype(np.uint64) * np.uint64(orc.CB_MUL1_MUL)) & np.uint64(0xffffffff)
    s = sum((x >> np.uint64(8 * i)) & np.uint64(0xff) for i in range(4)).astype(np.int64)
    assert np.array_equal(ot.MUL1_W_TABLE[s].view(np.uint16), orc.decode_values(st, 2).view(np.uint16))


def test_column_chunks():
    for (k, n) in ((4096, 128256), (28672, 1024), (14336, 128), (128, 640)):
        ch = ot.column_chunks(k, n)
        assert ch[0][0] == 0 and ch[-1][1] == n and all(a[1] == b[0] for a, b in zip(ch, ch[1:]))
        assert all(c0 % 128 == 0 and (c1 - c0) % 128 == 0 and k * (c1 - c0) <= max(ot.CHUNK_ELEMS, 128 * k) for c0, c1 in ch)


@pytest.mark.parametrize("tp", (1, 2, 8))
def test_launch_walk_is_the_tokens(tp):
    """token_launches (shapes only) describes bench.Token's default launch list, layer by layer, at a tiny config."""
    tok = bench.Token(TINY, tp, 0, torch.device("cpu"))
    want = token_launches(TINY, tp)
    per_layer, head = want[:4], want[4]
    got = [(launch_kind(ln), tuple((mt["name"], mt["k"], mt["n"], mt["K"]) for mt in ln["mats"])) for ln in tok.launches]
    assert got == per_layer * TINY["layers"] + [head]


def test_token_census_reaches_every_regime():
    """The tokens of the GPU file reach every schedule the unit walk's faults depend on (see the module docstring)."""
    seen = census()
    assert all(seen.values()), {r: len(v) for r, v in seen.items()}
    # lm_head at TP 1: about 243 units per CTA, more than two 96-unit accumulation chunks
    assert ("llama-3.1-8b", 1, "gemm", "lm_head") in seen["gemm_cta_over_96_units"]
    # the 70B TP 8 k / v projections are 128 columns wide and share a fan-out launch with q
    assert ("llama-3.1-70b", 8, "fanout", "q") in seen["fanout_with_128_column_member"]
    assert seen["strip_from_several_ctas"] and seen["odd_units_per_decode_group"]
    # every launch of every token is on the int8 decode-GEMM at one row
    for (model, tp) in TOKENS:
        layer, head = bench.token_plan(bench.MODELS[model], tp)
        for (_, k, n, K, _, _) in layer + [head]:
            assert gemm_plan(1, k, n, K, 2).path == TAG_I8


def test_fault_sites():
    """The catalog's units: lm_head's lies past the CTA's 96-unit hand-offs, at the end of its last sub-segment."""
    cfg = bench.MODELS["llama-3.1-8b"]
    layer, head = bench.token_plan(cfg, 1)
    strip, kb, cta, units, segs = fault_unit(*head[1:4])
    assert units > 2 * I8_SUB_UNITS and len(segs) >= 3 and segs[-1][0] > segs[0][0] + I8_SUB_UNITS - 1
    KB = head[1] // 128
    assert (strip * KB + kb) == segs[-1][1] - 1 and 0 < kb
    d = dict((nm, (k, n, K)) for (nm, k, n, K, _, _) in layer)["down"]
    strip, kb, cta, units, segs = fault_unit(*d)
    assert units > 1 and kb > 0


def test_unit_faults_change_only_their_strip():
    """Faults (a)-(g) of unit_faults touch the 128 columns of their strip only, and each changes something."""
    K, k, n = 4, 512, 384
    tr, suh, svh, x = orc.make_synthetic(k, n, K)
    pre = orc.exl3_gemm_i8_model(x, tr, suh, None, K)
    for fp32 in (True, False):
        model = orc.i8_model_output(pre, svh, np.float32 if fp32 else np.float16)
        for name, y in unit_faults(x, tr, suh, svh, K, pre, 1, 2, fp32).items():
            d = np.asarray(y, np.float64) != np.asarray(model, np.float64)
            assert d.any(), name
            if not name.startswith("(h)"):
                assert not d[:, :128].any() and not d[:, 256:].any(), name
