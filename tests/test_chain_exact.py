"""
The GEMM-chain kernel (csrc/chain_i8.cu, tag 220) held to its exact model, oracle.exl3_gemm_i8_model(rule="blocknorm") (H100).

The model reproduces the kernel's activation integers bit for bit (block-norm scale, digits, integer contraction); the kernel
must agree with it to fp32 round-off: max-abs <= 2e-5 max|y|, rel-RMS <= 1e-5 for fp32 C, 1.5e-3 / 5e-4 for fp16 C
(test_gpu_edges.check_model).  Every op is checked against the model on the input it actually read -- for a dependent stage
that is the kernel's own upstream output -- and against the fp64 oracle (README.md, Parity).  Gated ops (silu(gate) * up) are
exact where the gates are in {0} u [20, 60]; elsewhere the kernel's fast-math silu differs from the model's and the bar is 3e-3.

Covered: every split-K pattern of the forced grids on the exl3_gemm entry (inline op), repeats and interleaving bit for bit;
adversarial rows; the uncached fallbacks (A or suh not 16-byte aligned, rows too long for the cache) bit for bit against the
cached runs; layer- and token-shaped chains (scale-slot reuse, both split-K exchange buffers, stage counters past 1); a
255-stage relay; CUDA-graph replay of bench.py's blocks-mode chains; the gated stage's dependency on gate + up; mixed row
counts. The inline op and the device table are compared bit for bit at the default grid (the reduce order depends on the grid).
Which regime each table reaches is asserted on the host in tests/test_chain_host.py.

Every output is written into the middle rows of a sentinel-filled C, and every fp16 input is read through a view whose trailing
rows are NaN: the rows around the output must keep their bits and every output must be finite.
"""
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc
from test_edges_host import FORCED_GRIDS
from test_gpu_edges import SENTINEL, T, Mat as EdgeMat, check_f64, check_model, finish, gemm_path, launch, rel_err
from test_chain_host import (LAYER, TOKEN, adversarial_rows, exact_gates, layer_chain, pow2_suh, relay_chain, token_chain)

pytestmark = pytest.mark.gpu

TAG_CHAIN = 220


# ---- helpers -----------------------------------------------------------------------------------------------------------

class Mat:
    """One quantized matrix (mul1) on the host and on the device, with its decoded forms for the two references."""

    def __init__(self, dev, k, n, K, seed, suh=None, svh_gain=1.0):
        tr, suh0, svh, _ = orc.make_synthetic(k, n, K, seed=seed)
        self.tr, self.K, self.k, self.n = tr, K, k, n
        self.suh = suh0 if suh is None else suh
        self.svh = (svh.astype(np.float64) * svh_gain).astype(np.float16)
        self.w, self.bsum = orc.reconstruct(tr, K, 2), orc.mul1_bytesum(tr, K)
        self.dev = dev
        self.d_tr, self.d_suh, self.d_svh = T(tr, dev), T(self.suh, dev), T(self.svh, dev)

    def set_gain(self, g):
        self.svh = (self.svh.astype(np.float64) * g).astype(np.float16)
        self.d_svh = T(self.svh, self.dev)

    def model(self, x):
        return orc.exl3_gemm_i8_model(x, self.tr, self.suh, self.svh, self.K, bsum=self.bsum, rule="blocknorm")

    def f64(self, x):
        return orc.exl3_gemm_f64(x, self.tr, self.suh, self.svh, self.K, 2, w=self.w)

    def op(self, **kw):
        return dict(trellis=self.d_tr, suh=self.d_suh, svh=self.d_svh, mul1=True, **kw)


def canvas(m, n, fp32, dev):
    """Sentinel-filled (m + 2, n) C and the view of its rows 1..m."""
    dt = torch.float if fp32 else torch.half
    C = torch.empty((m + 2, n), dtype=dt, device=dev)
    C.view(SENTINEL[dt][0]).fill_(SENTINEL[dt][1])
    return C, C[1:m + 1]


def nan_tail(x, dev, dtype=torch.half):
    """x on the device as rows 0..m-1 of a buffer whose 3 trailing rows are NaN."""
    m, k = x.shape
    A = torch.full((m + 3, k), float("nan"), dtype=dtype, device=dev)
    A[:m] = torch.from_numpy(np.ascontiguousarray(x)).to(dev, dtype)
    return A[:m]


def bits(C):
    return C.view(SENTINEL[C.dtype][0]).cpu().numpy().copy()


def check_op(y, x, mt, fp32, what, exact=True):
    """y against the model on the input x the op read (per row: rows of one op carry independent scales), and the oracle."""
    model = mt.model(x)
    for r in range(y.shape[0]):
        if not np.any(model[r]):
            assert not np.any(y[r]), ("zero row not exactly 0", what, r)
            continue
        if exact:
            check_model(y[r:r + 1], model[r:r + 1], fp32, (what, r))
        else:
            mx, rms = rel_err(y[r:r + 1], model[r:r + 1])
            assert mx <= 3e-3 and rms <= 1.5e-3, (what, r, mx, rms)
    if exact:
        check_f64(y, mt.f64(x), fp32, what)


def build_table(ext, dev, ops, m, x, seed, gains=None):
    """Matrices for a chain table, each svh scaled so that the op's output (on the host run of the fp64 oracle along the
    chain) has RMS gains.get(name, 1): values stay in fp16 range over any chain length, and per-layer gains give every layer
    input its own scale.  Returns (GemmChain, mats, canvases)."""
    mats, host, outs, spec = {}, {"x": x}, {}, []
    for i, o in enumerate(ops):
        nm, mi = o["name"], o.get("m", m)
        mt = Mat(dev, o["k"], o["n"], o["K"], seed=seed + 7 * i)
        src = o["src"]
        inp = orc.chain_gated_input(host[src[0]], host[src[1]]) if isinstance(src, tuple) else host[src][:mi]
        y = mt.f64(inp)
        mt.set_gain((gains or {}).get(nm, 1.0) / max(np.sqrt((y ** 2).mean()), 1e-30))
        y = mt.f64(inp)
        host[nm] = y.astype(np.float32 if o["fp32"] else np.float16)
        mats[nm] = mt
        C, yv = canvas(mi, o["n"], o["fp32"], dev)
        outs[nm] = (C, yv)
        d = mt.op(y=yv, new_stage=o["new_stage"])
        if isinstance(src, tuple):
            d.update(gate=outs[src[0]][1], up=outs[src[1]][1])
        else:
            d["x"] = nan_tail(x[:mi], dev) if src == "x" else outs[src][1][:mi]
        spec.append(d)
    return ext.GemmChain(spec), mats, outs


def check_table(ops, m, x, mats, outs):
    """Every op against the model on what the kernel itself produced upstream; returns the outputs' bits."""
    host, raw = {"x": x}, {}
    for o in ops:
        nm, mi, src = o["name"], o.get("m", m), o["src"]
        C = outs[nm][0]
        y = finish(C, nm)
        raw[nm] = bits(C)
        host[nm] = y.astype(np.float32 if o["fp32"] else np.float16)
        if isinstance(src, tuple):
            check_op(y, orc.chain_gated_input(host[src[0]], host[src[1]]), mats[nm], o["fp32"], nm, exact=False)
        else:
            check_op(y, host[src][:mi], mats[nm], o["fp32"], nm)
    return raw


def run_table_twice(ch, ops, m, x, mats, outs):
    ch.run()
    torch.cuda.synchronize()
    first = check_table(ops, m, x, mats, outs)
    for C, _ in outs.values():
        C[1:-1].zero_()
    ch.run()                                                            # counters and exchange buffers re-armed
    torch.cuda.synchronize()
    second = check_table(ops, m, x, mats, outs)
    for nm in first:
        assert np.array_equal(first[nm], second[nm]), ("replay differs", nm)


def rows(m, k, seed, scale=1.0):
    return (np.random.default_rng(seed).standard_normal((m, k)) * scale).astype(np.float16)


# ---- 1. every split-K pattern, inline op (exl3_gemm) and device table (GemmChain) ------------------------------------------

@pytest.mark.parametrize("k,n,grids", FORCED_GRIDS)
def test_forced_grids_bit_stable_and_exact(cuda, k, n, grids):
    """exl3_gemm on the chain kernel (the op inline in the kernel parameters) at every forced grid: each against the model,
    and its repeat (launched after another chain, no synchronisation in between) bit for bit.  The split-K reduce order
    depends on the grid and GemmChain has no grid cap, so the inline op is compared bit for bit with the device-table entry
    (a one-op GemmChain) at the default grid only."""
    from exllamav3_b200 import ext
    tr, suh, svh, _ = orc.make_synthetic(k, n, 4, seed=k + n)
    mt = Mat(cuda, k, n, 4, seed=k + n)
    emt = EdgeMat(cuda, tr, suh, svh, 4, 2)
    # another chain launched in between: two stages, split-K in both, its own scale slots and counters
    a, b = Mat(cuda, 1024, 256, 3, seed=1), Mat(cuda, 256, 512, 5, seed=2)
    xo = rows(4, 1024, 3)
    Ca, ya = canvas(4, 256, False, cuda); Cb, yb = canvas(4, 512, True, cuda)
    other = ext.GemmChain([a.op(x=nan_tail(xo, cuda), y=ya), b.op(x=ya, y=yb, new_stage=True)])
    for m in (1, 4):
        x = rows(m, k, 10 * m + k)
        for fp32 in (True, False):
            runs = []
            with gemm_path(TAG_CHAIN):
                for G in grids:                                         # back to back, no synchronisation
                    C1, t1 = launch(ext, cuda, x, emt, fp32, force=G)
                    other.run()
                    C2, t2 = launch(ext, cuda, x, emt, fp32, force=G)
                    assert t1 == t2 == TAG_CHAIN
                    runs.append((G, C1, C2))
                C0, _ = launch(ext, cuda, x, emt, fp32)
            Cc, yc = canvas(m, n, fp32, cuda)
            ch = ext.GemmChain([mt.op(x=nan_tail(x, cuda), y=yc)])
            ch.run()
            torch.cuda.synchronize()
            for G, C1, C2 in runs:
                y = finish(C1, (k, n, m, fp32, G))
                finish(C2, (k, n, m, fp32, G))
                assert np.array_equal(bits(C1), bits(C2)), ("repeat differs", k, n, m, fp32, G)
                check_op(y, x, mt, fp32, (k, n, m, fp32, G))
            finish(C0, "default grid"); finish(Cc, "GemmChain")
            assert np.array_equal(bits(C0), bits(Cc)), ("inline op != device table", k, n, m, fp32)
            ch.close()
    torch.cuda.synchronize()
    yo = finish(Ca, "other"); finish(Cb, "other")
    check_op(yo, xo, a, False, "other chain, stage 0")
    check_op(finish(Cb, "other").astype(np.float64), yo.astype(np.float16), b, True, "other chain, stage 1")
    other.close()


# ---- 2. adversarial rows -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fp32", [True, False])
def test_adversarial_rows(cuda, fp32):
    """One op: a zero row (output exactly 0), a Hadamard-aligned row (bound tight to 1.002: |q| reaches 0.99 * 32512), an
    outlier block, fp16-subnormal x * suh; a second op of the stage: rows whose scales are 100x apart."""
    from exllamav3_b200 import ext
    k, n = 1024, 384
    suh = pow2_suh(k, 5)
    mt = Mat(cuda, k, n, 4, seed=6, suh=suh)
    xa = adversarial_rows(k, suh, 7)
    xb = (rows(4, k, 8) * np.array([[1e-3], [1e-1], [1e1], [1e3]])).astype(np.float16)
    q, _ = orc.i8_activation_q(xa, suh, rule="blocknorm")
    assert np.abs(q[1]).max() >= 0.99 * 32512 and np.abs(q).max() <= 32512
    Ca, ya = canvas(4, n, fp32, cuda); Cb, yb = canvas(4, n, fp32, cuda)
    ch = ext.GemmChain([mt.op(x=nan_tail(xa, cuda), y=ya), mt.op(x=nan_tail(xb, cuda), y=yb)])
    ch.run()
    torch.cuda.synchronize()
    y = finish(Ca, "adversarial")
    assert (y[0] == 0).all()
    check_op(y, xa, mt, fp32, "adversarial")
    check_op(finish(Cb, "scales 100x apart"), xb, mt, fp32, "scales 100x apart")
    ch.close()


# ---- 3. fallback branches, bit for bit ---------------------------------------------------------------------------------

def test_uncached_fallbacks_match_the_cached_runs(cuda):
    from exllamav3_b200 import ext
    k, n, m = 1024, 384, 4
    mt = Mat(cuda, k, n, 5, seed=21)
    x = rows(m, k, 22)
    # A 8-byte but not 16-byte aligned (read from global memory, not bulk-copied), trailing rows NaN
    buf = torch.full((m * k + 4 + 3 * k,), float("nan"), dtype=torch.half, device=cuda)
    a8 = buf[4:4 + m * k].view(m, k)
    a8.copy_(T(x, cuda))
    assert a8.data_ptr() % 16 == 8
    sbuf = torch.zeros(k + 4, dtype=torch.half, device=cuda)
    s8 = sbuf[4:]
    s8.copy_(mt.d_suh)
    assert s8.data_ptr() % 16 == 8
    variants = dict(aligned=(nan_tail(x, cuda), mt.d_suh), a8=(a8, mt.d_suh), suh8=(nan_tail(x, cuda), s8), both=(a8, s8))
    res = {}
    for fp32 in (True, False):
        for nm, (A, suh) in variants.items():
            C, y = canvas(m, n, fp32, cuda)
            ch = ext.GemmChain([dict(x=A, trellis=mt.d_tr, suh=suh, svh=mt.d_svh, y=y, mul1=True)])
            ch.run()
            torch.cuda.synchronize()
            yy = finish(C, (nm, fp32))
            res[nm, fp32] = bits(C)
            if nm == "aligned":
                check_op(yy, x, mt, fp32, (nm, fp32))
            ch.close()
        for nm in variants:
            assert np.array_equal(res[nm, fp32], res["aligned", fp32]), (nm, fp32)
    # misaligned pointers are refused before anything runs
    with pytest.raises(RuntimeError, match="A must be 8-byte aligned"):
        ext.GemmChain([dict(x=buf[2:2 + m * k].view(m, k), trellis=mt.d_tr, suh=mt.d_suh, svh=mt.d_svh, y=y, mul1=True)])
    with pytest.raises(RuntimeError, match="C must be 16-byte aligned"):
        yf = torch.zeros(m * n + 2, device=cuda)[2:].view(m, n)
        ext.GemmChain([dict(x=a8, trellis=mt.d_tr, suh=mt.d_suh, svh=mt.d_svh, y=yf, mul1=True)])


def test_rows_too_long_for_the_cache_match_single_rows(cuda):
    """m * k * 2 > 64 KiB: the digit warps recompute x * suh per unit from global memory; the same rows one at a time are cached.
    Rows are independent (own scale, same unit partition), so the results agree bit for bit."""
    from exllamav3_b200 import ext
    k, n, m = 8320, 256, 4
    mt = Mat(cuda, k, n, 3, seed=31)
    x = rows(m, k, 32) * np.float16(2.0)
    for fp32 in (True, False):
        C, y = canvas(m, n, fp32, cuda)
        singles = [canvas(1, n, fp32, cuda) for _ in range(m)]
        # one chain each: the same unit partition over the same grid
        chains = [ext.GemmChain([mt.op(x=nan_tail(x, cuda), y=y)])]
        chains += [ext.GemmChain([mt.op(x=nan_tail(x[r:r + 1], cuda), y=singles[r][1])]) for r in range(m)]
        for ch in chains:
            ch.run()
        torch.cuda.synchronize()
        yy = finish(C, ("uncached", fp32))
        check_op(yy, x, mt, fp32, ("uncached", fp32))
        b = bits(C)
        for r in range(m):
            finish(singles[r][0], ("single row", r))
            assert np.array_equal(bits(singles[r][0])[1], b[1 + r]), (fp32, r)
        for ch in chains:
            ch.close()


# ---- 4. gated ops with exact gates ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("gu_dtype", [torch.float, torch.half])
def test_gated_ops_with_exact_gates(cuda, gu_dtype):
    from exllamav3_b200 import ext
    for (m, k, n) in ((4, 1024, 384), (3, 4096, 256), (1, 256, 128)):
        mt = Mat(cuda, k, n, 4, seed=m + k)
        npdt = np.float32 if gu_dtype == torch.float else np.float16
        g = exact_gates((m, k), k).astype(npdt)
        u = (np.random.default_rng(k + 1).standard_normal((m, k)) * 0.5).astype(npdt)
        G, U = nan_tail(g, cuda, gu_dtype), nan_tail(u, cuda, gu_dtype)
        x = rows(m, k, k + 2)
        C0, y0 = canvas(m, n, True, cuda)
        C, y = canvas(m, n, gu_dtype == torch.float, cuda)
        ch = ext.GemmChain([mt.op(x=nan_tail(x, cuda), y=y0), mt.op(gate=G, up=U, y=y)])
        ch.run()
        torch.cuda.synchronize()
        check_op(finish(C0, "plain"), x, mt, True, "plain")
        h = orc.chain_gated_input(g, u)
        check_op(finish(C, ("gated", m, k)), h, mt, gu_dtype == torch.float, ("gated", m, k, gu_dtype))
        ch.close()


# ---- 5. layer-, token- and relay-shaped chains ---------------------------------------------------------------------------

def test_layer_chain_exact(cuda):
    from exllamav3_b200 import ext
    ops, m = layer_chain(), LAYER["m"]
    x = rows(m, LAYER["H"], 41)
    ch, mats, outs = build_table(ext, cuda, ops, m, x, seed=400)
    run_table_twice(ch, ops, m, x, mats, outs)
    ch.close()


def test_token_chain_exact(cuda):
    """8 layers + head (57 ops, 33 stages, bitrates 2..6): scale slots reused (op % 32), both exchange buffers, stage
    counters up to 32; every layer's input has its own scale."""
    from exllamav3_b200 import ext
    ops, m = token_chain(), TOKEN["m"]
    gains = {f"{l}.down": 4.0 ** ((l % 3) - 1) for l in range(TOKEN["layers"])}
    x = rows(m, TOKEN["H"], 51)
    ch, mats, outs = build_table(ext, cuda, ops, m, x, seed=500, gains=gains)
    run_table_twice(ch, ops, m, x, mats, outs)
    ch.close()


def test_relay_chain_255_stages(cuda):
    from exllamav3_b200 import ext
    ops, m = relay_chain(), 3
    x = rows(m, 2048, 61)
    ch, mats, outs = build_table(ext, cuda, ops, m, x, seed=600)
    run_table_twice(ch, ops, m, x, mats, outs)
    ch.close()


# ---- 6. CUDA-graph replay and mixed row counts ---------------------------------------------------------------------------

def _layer_specs(ext, dev, seed):
    ops, m = layer_chain(), LAYER["m"]
    x = rows(m, LAYER["H"], seed)
    _, mats, outs = build_table(ext, dev, ops, m, x, seed=10 * seed)
    specs = []
    for o in ops:
        mt, src = mats[o["name"]], o["src"]
        d = mt.op(y=outs[o["name"]][1], new_stage=o["new_stage"])
        if isinstance(src, tuple):
            d.update(gate=outs[src[0]][1], up=outs[src[1]][1])
        else:
            d["x"] = nan_tail(x, dev) if src == "x" else outs[src][1]
        specs.append(d)
    return ops, m, x, mats, outs, specs


def test_graph_replay_of_block_chains_is_bit_identical(cuda):
    """The blocks mode of bench.py: a layer as three chains (q + k + v | o | gate + up -> down, the last with the gated down in
    a second stage), eager, then captured in a CUDA graph and replayed: bit-identical outputs."""
    from exllamav3_b200 import ext
    ops, m, x, mats, outs, specs = _layer_specs(ext, cuda, 70)
    chains = [ext.GemmChain(specs[0:3]), ext.GemmChain(specs[3:4]), ext.GemmChain(specs[4:7])]
    for ch in chains:
        ch.run()
    torch.cuda.synchronize()
    eager = check_table(ops, m, x, mats, outs)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for ch in chains:
            ch.run()
    for _ in range(2):
        for C, _ in outs.values():
            C[1:-1].zero_()
        g.replay()
        torch.cuda.synchronize()
        for o in ops:
            finish(outs[o["name"]][0], o["name"])
            assert np.array_equal(bits(outs[o["name"]][0]), eager[o["name"]]), ("graph replay differs", o["name"])
    del g
    for ch in chains:
        ch.close()


def test_gated_stage_reads_the_outputs_of_its_first_stage(cuda):
    """gate + up -> down as one chain (bench.py's blocks mode), gate / up buffers pre-filled with 0.5 before the launch: the
    down op, in the second stage, must see the values the first stage wrote, not what the buffers held before."""
    from exllamav3_b200 import ext
    ops, m, x, mats, outs, specs = _layer_specs(ext, cuda, 70)
    xo = rows(m, LAYER["H"], 72) * np.float16(0.3)
    outs["0.o"][1].copy_(T(xo, cuda))
    for nm in ("0.gate", "0.up"):
        outs[nm][1].fill_(0.5)
    ch = ext.GemmChain(specs[4:7])
    ch.run()
    torch.cuda.synchronize()
    host = {"0.o": xo}
    for o in ops[4:7]:
        nm, src = o["name"], o["src"]
        y = finish(outs[nm][0], nm)
        host[nm] = y.astype(np.float32 if o["fp32"] else np.float16)
        inp = orc.chain_gated_input(host[src[0]], host[src[1]]) if isinstance(src, tuple) else host[src]
        check_op(y, inp, mats[nm], o["fp32"], nm, exact=not isinstance(src, tuple))
    ch.close()


def test_mixed_row_counts_in_one_chain(cuda):
    from exllamav3_b200 import ext
    ops = [dict(name="a", k=1024, n=512, K=4, src="x", new_stage=True, fp32=False, m=4),
           dict(name="b", k=1024, n=256, K=3, src="x", new_stage=False, fp32=True, m=1),
           dict(name="c", k=512, n=384, K=5, src="a", new_stage=True, fp32=True, m=1),
           dict(name="d", k=512, n=256, K=2, src="a", new_stage=False, fp32=False, m=4),
           dict(name="e", k=256, n=512, K=6, src="d", new_stage=True, fp32=True, m=3)]
    x = rows(4, 1024, 81)
    ch, mats, outs = build_table(ext, cuda, ops, 4, x, seed=800)
    run_table_twice(ch, ops, 4, x, mats, outs)
    ch.close()
