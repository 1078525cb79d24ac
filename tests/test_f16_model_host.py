"""
The exact models of the fp16 paths (oracle.exl3_gemm_f16_model, exl3_mgemm_f16_model, exl3_moe_model), no GPU needed: what
they are (fp32 round-off of the fp64 oracle, the epilogue's rounding points, the mgemm reduce, the MoE sum), and a catalog of
kernel faults applied to them.  Every fault must miss the bars of test_edges_host.check_f16_model / check_moe_model by at least
3x at the shapes the GPU tests run; the faults the fp64-oracle bars let through are asserted to pass those, which is the gap
the model bars close.
"""
import numpy as np
import pytest
from oracle import exl3_oracle as orc
from test_edges_host import F16_MODEL_BAR, F16_MODEL_SAME, MOE_MODEL_BAR, check_f16_model, f16_model_ratios, rel_err

# (k, n, m) of the GPU tests that reach the fp16 paths: a single k-block, the instantiation and parity shapes, the row sweep,
# the forced-grid shapes, the full-size 128-column blocks at batch 1 / 8 / 32 (k = 14336: the down projection)
SHAPES = ((128, 1024, 1), (512, 384, 17), (512, 256, 257), (1152, 1152, 130), (4096, 128, 8), (4096, 256, 3),
          (14336, 128, 1), (14336, 128, 32))
MARGIN = 3.0


def f64_bars(y, ref, fp32):
    """The fp64-oracle bars of the GPU tests (README.md, Parity)."""
    mx, rms = rel_err(y, ref)
    return mx <= 2e-3 + (0.0 if fp32 else 2.0 ** -10) and rms <= 1e-3


def setup(k, n, m, K=4, cb=2):
    tr, suh, svh, _ = orc.make_synthetic(k, n, K, seed=k + n + m)
    x = np.random.default_rng(m).standard_normal((m, k)).astype(np.float16)
    return x, tr, suh, svh, orc.reconstruct(tr, K, cb)


def epilogue(acc, svh, fp32):
    return orc.had_out_from_f32(acc.astype(np.float32), svh, np.float32 if fp32 else np.float16)


# ---- the model --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k,n,m", SHAPES)
def test_model_is_fp32_round_off_of_the_fp64_oracle(k, n, m):
    x, tr, suh, svh, w = setup(k, n, m)
    ref = orc.exl3_gemm_f64(x, tr, suh, svh, 4, 2, w=w)
    y, pre = orc.exl3_gemm_f16_model(x, tr, suh, svh, 4, 2, np.float32, w=w)
    mx, rms = rel_err(y, ref)
    assert mx <= 1e-6 and rms <= 3e-7, (mx, rms)
    assert np.array_equal(y, orc.exl3_gemm(x, tr, suh, svh, 4, 2, np.float32))
    y16, pre16 = orc.exl3_gemm_f16_model(x, tr, suh, svh, 4, 2, np.float16, w=w)
    assert pre16.dtype == np.float16 and y16.dtype == np.float16
    # fp16 C: rounded before the svh multiply, which is one fp16 multiply (csrc/epilogue.cuh output_row_128)
    assert np.array_equal(y16.view(np.uint16), orc._hmul(pre16, svh[None, :]).view(np.uint16))
    assert np.array_equal(pre16, pre.astype(np.float16))
    # fp32 C: the pre-svh value times float(svh)
    assert np.array_equal(y, (pre * svh.astype(np.float32)[None, :]).astype(np.float32))
    check_f16_model(y16, y16, orc.f16_model_tol(y16, pre16, svh), (k, n, m))


def test_model_scale_is_the_epilogue_out_scale():
    x, tr, suh, svh, w = setup(512, 256, 3)
    s = float(np.float16(0.37))
    y, pre = orc.exl3_gemm_f16_model(x, tr, suh, svh, 4, 2, np.float32, w=w, scale=s)
    y1, pre1 = orc.exl3_gemm_f16_model(x, tr, suh, svh, 4, 2, np.float32, w=w)
    assert rel_err(y, s * y1)[0] <= 1e-6
    r = np.float32(np.float32(s) * orc.R_SCALE_F32)            # fp32(R_SCALE * out_scale), one multiply per element
    acc = (orc.had_r_128(x, pre_scale=suh).astype(np.float64) @ w.astype(np.float64)).astype(np.float32)
    h = orc.fwht128_f32(acc.reshape(3, 2, 128)).reshape(3, 256)
    assert np.array_equal(pre, (h * r).astype(np.float32))


def test_fp16_order_noise_stays_inside_the_fp16_bar():
    """fp32 accumulation in another order (2^-22 relative noise on the sums) passes the fp16-C check; it changes < 1 % of C."""
    for (k, n, m) in ((512, 384, 17), (4096, 128, 8)):
        x, tr, suh, svh, w = setup(k, n, m)
        acc = orc.had_r_128(x, pre_scale=suh).astype(np.float64) @ w.astype(np.float64)
        y, pre = orc.exl3_gemm_f16_model(x, tr, suh, svh, 4, 2, np.float16, w=w)
        rng = np.random.default_rng(k)
        noisy = epilogue(acc * (1 + rng.choice([-1.0, 1.0], acc.shape) * 2.0 ** -22), svh, False)
        check_f16_model(noisy, y, orc.f16_model_tol(y, pre, svh), (k, n, m))
        assert (noisy != y).mean() < 0.01


@pytest.mark.parametrize("fp32", (True, False))
@pytest.mark.parametrize("num_tokens", (1, 2))
def test_mgemm_model_is_the_per_slot_model_reduced(fp32, num_tokens):
    k, n, K, E = 512, 256, 3, 4
    mats = [orc.make_synthetic(k, n, K, seed=30 + e) for e in range(E)]
    trl, sul, svl = [t[0] for t in mats], [t[1] for t in mats], [t[2] for t in mats]
    rng = np.random.default_rng(num_tokens)
    idx = [3, 1, 0, 2]
    A = rng.standard_normal((4, 2, k)).astype(np.float16)
    wts = rng.uniform(0.1, 1.0, 4).astype(np.float16)
    dt = np.float32 if fp32 else np.float16
    C, tol = orc.exl3_mgemm_f16_model(A, trl, sul, svl, K, 1, dt, indices=idx, weights=wts, num_tokens=num_tokens)
    per = np.stack([orc.exl3_gemm_f16_model(A[j], trl[q], sul[q], svl[q], K, 1, dt, scale=float(wts[j]))[0]
                    for j, q in enumerate(idx)])
    assert C.dtype == dt
    assert np.array_equal(C.view(np.uint8), orc.mgemm_reduce(per, 4, num_tokens).view(np.uint8))
    assert (tol is None) == fp32
    # unweighted, one shared input, a skipped slot: the per-slot model, the skipped slot untouched
    C, tol = orc.exl3_mgemm_f16_model(A[:1], trl, sul, svl, K, 1, dt, indices=[2, -1, 0, 3], bszm_out=4)
    for j, q in enumerate((2, -1, 0, 3)):
        if q < 0:
            assert not C[j].any() and (tol is None or not tol[j].any())
            continue
        y, pre = orc.exl3_gemm_f16_model(A[0], trl[q], sul[q], svl[q], K, 1, dt)
        assert np.array_equal(C[j], y)
        if not fp32:
            assert np.array_equal(tol[j], orc.f16_model_tol(y, pre, svl[q]))


# ---- exl3_moe -------------------------------------------------------------------------------------------------------------

def moe_setup(act, limit, seed=0, E=6, bsz=12, topk=2, hidden=256, inter=384):
    rng = np.random.default_rng(seed)
    mats = {}
    for i, (name, k, n, K) in enumerate((("gate", hidden, inter, 3), ("up", hidden, inter, 4), ("down", inter, hidden, 2))):
        mats[name] = [orc.make_synthetic(k, n, K, seed=seed + 100 * i + e)[:3] + (K,) for e in range(E)]
        mats[name] = [(tr, suh, svh, K, orc.reconstruct(tr, K, 2)) for (tr, suh, svh, K) in mats[name]]
    ex = np.stack([rng.choice(E, topk, replace=False) for _ in range(bsz)])
    ex[0, 0] = E                                                     # choices in the sentinel bucket: token 1 has none here
    ex[1, :] = E
    wt = rng.uniform(0.05, 1.0, ex.shape).astype(np.float16)
    order = np.argsort(ex.reshape(-1), kind="stable")
    count = np.bincount(ex.reshape(-1), minlength=E + 1).astype(np.int64)
    tok = np.repeat(np.arange(bsz), topk)[order].astype(np.int64)
    x = rng.standard_normal((bsz, hidden)).astype(np.float16)
    out0 = (rng.standard_normal((bsz, hidden)) * 0.5).astype(np.float32)
    T_ = int(count[:-1].max()) - 1                                   # the largest experts are over the limit: not processed
    return dict(x=x, out=out0, count=count, token_sorted=tok, weight_sorted=wt.reshape(-1)[order], max_tokens=T_, act=act,
                limit=limit, mats=mats, cb=2)


@pytest.mark.parametrize("act", (0, 1, 2))
@pytest.mark.parametrize("limit", (0.0, 0.4))
def test_moe_model_is_the_sum_of_its_expert_models(act, limit):
    c = moe_setup(act, limit, seed=act + 3)
    y = orc.exl3_moe_model(**c)
    procs = orc.moe_processed(c["count"][:-1], c["max_tokens"], len(c["token_sorted"]))
    assert len(procs) < len(c["count"]) - 1                          # some expert is not processed
    ref = c["out"].copy()
    touched = np.zeros(len(ref), dtype=bool)
    terms = {}
    for e, s, n in procs:
        for j in range(s, s + n):
            t = c["token_sorted"][j]
            xr = c["x"][t:t + 1]
            gemm = lambda name, a, dt: orc.exl3_gemm_f16_model(a, *c["mats"][name][e][:4], 2, dt)[0]
            u = gemm("up", xr, np.float16)
            g = u if act == 2 else gemm("gate", xr, np.float16)
            terms[j] = (t, np.float32(c["weight_sorted"][j]) * gemm("down", orc.moe_act(g, u, act, limit), np.float32)[0])
            touched[t] = True
    for j in sorted(terms):                                          # one row at a time: the GEMM rows are independent
        t, v = terms[j]
        ref[t] = ref[t] + v
    assert np.array_equal(y.view(np.uint32), ref.view(np.uint32))
    assert np.array_equal(y[~touched].view(np.uint32), c["out"][~touched].view(np.uint32))
    assert touched.any() and not touched.all()


def test_moe_act_rounding_points():
    g = np.array([0.0, 1.5, -3.0, 20.0, -60000.0], dtype=np.float16)
    u = np.array([1.0, -0.75, 2.0, 0.5, 1.0], dtype=np.float16)
    h = orc.moe_act(g, u, 0, 0.0)
    assert h.dtype == np.float16 and h[0] == 0 and h[3] == np.float16(10.0) and h[4] == 0
    gf, uf = g.astype(np.float32), u.astype(np.float32)
    assert np.array_equal(h, (gf / (np.float32(1) + np.exp(-gf)) * uf).astype(np.float16))
    # the limit clamps u and the activation, before the product; ReLU^2 gates u with itself
    hl = orc.moe_act(g, u, 2, 0.6)
    a = np.minimum(np.maximum(uf, 0), np.float32(0.6))
    assert np.array_equal(hl, (a * np.clip(uf, -0.6, 0.6).astype(np.float32)).astype(np.float16))


# ---- fault catalog ------------------------------------------------------------------------------------------------------

def split_k_fp16(xh, w):
    """split-K partials stored as fp16: the two halves of the k-blocks summed separately, each rounded to fp16"""
    h = (w.shape[0] // 128 + 1) // 2 * 128
    parts = [xh[:, s].astype(np.float64) @ w[s].astype(np.float64) for s in (slice(0, h), slice(h, None))]
    return sum(p.astype(np.float16).astype(np.float32) for p in parts)


def faulty_outputs(x, suh, svh, w, fp32):
    """{fault: C of a kernel with that fault} for the fp16 GEMM; a fault that cannot occur at a shape is absent."""
    m, k = x.shape
    n = w.shape[1]
    xh = orc.had_r_128(x, pre_scale=suh)
    dot = lambda a, b: a.astype(np.float64) @ b.astype(np.float64)
    f = {}
    wf = w.copy(); wf[k // 3, n // 3] = -wf[k // 3, n // 3]
    f["one weight's sign flipped"] = epilogue(dot(xh, wf), svh, fp32)
    if k >= 256:
        f["split-K partials stored as fp16"] = epilogue(split_k_fp16(xh, w), svh, fp32)
    xs = (x.astype(np.float32) * suh.astype(np.float32)[None, :]).reshape(m, k // 128, 128)
    xh32 = (orc.fwht128_f32(xs).reshape(m, k) * orc.R_SCALE_F32).astype(np.float16)
    f["x * suh in fp32, unrounded"] = epilogue(dot(xh32, w), svh, fp32)
    wf = w.copy(); wf[5, 16:32] = w[5, 32:48]
    f["16 weights of a tile row from the next tile"] = epilogue(dot(xh, wf), svh, fp32)
    wf = w.copy(); wf[k - 16:k, :64] = 0
    f["one k16 slice missing from a 64-column half"] = epilogue(dot(xh, wf), svh, fp32)
    xf = xh.copy(); xf[m - 1, k - 16:] = xh[m - 2, k - 16:] if m > 1 else 0
    f["last k-tile of the last row from the wrong row"] = epilogue(dot(xf, w), svh, fp32)
    if not fp32:
        acc = dot(xh, w).astype(np.float32)
        hh = orc.fwht128_f32(acc.reshape(m, n // 128, 128)).reshape(m, n) * orc.R_SCALE_F32
        f["svh in fp32 before the fp16 rounding"] = (hh * svh.astype(np.float32)[None, :]).astype(np.float16)
    return f


def fault_ratio(y, model, pre, svh, fp32):
    """How far a faulty C is outside the model bar (> 1: caught)."""
    if fp32:
        mx, rms = rel_err(y, model)
        return max(mx / F16_MODEL_BAR[0], rms / F16_MODEL_BAR[1])
    over, changed = f16_model_ratios(y, model, orc.f16_model_tol(model, pre, svh))
    return max(over, changed / (1 - F16_MODEL_SAME))


@pytest.mark.parametrize("k,n,m", SHAPES)
@pytest.mark.parametrize("fp32", (True, False))
def test_fault_catalog_gemm(k, n, m, fp32):
    x, tr, suh, svh, w = setup(k, n, m)
    dt = np.float32 if fp32 else np.float16
    model, pre = orc.exl3_gemm_f16_model(x, tr, suh, svh, 4, 2, dt, w=w)
    ref = orc.exl3_gemm_f64(x, tr, suh, svh, 4, 2, w=w)
    for name, y in faulty_outputs(x, suh, svh, w, fp32).items():
        r = fault_ratio(y, model, pre, svh, fp32)
        assert r >= MARGIN, (name, k, n, m, fp32, r)
    # the model itself passes the fp64-oracle bars
    assert f64_bars(model, ref, fp32)


def test_fault_catalog_escapes_today():
    """The table's cases that pass the fp64-oracle bars (the gap): one wrong weight of a 14336-wide down projection, split-K
    partials in fp16, the unrounded pre-scale, and svh applied before the fp16 rounding."""
    for (k, n, m, fp32, names) in ((14336, 256, 5, True, ("one weight's sign flipped", "split-K partials stored as fp16")),
                                   (4096, 1024, 8, True, ("split-K partials stored as fp16", "x * suh in fp32, unrounded")),
                                   (512, 384, 17, True, ("split-K partials stored as fp16", "x * suh in fp32, unrounded")),
                                   (512, 384, 17, False, ("svh in fp32 before the fp16 rounding",))):
        tr, suh, svh, x = orc.make_synthetic(k, n, 4, m=m)
        w = orc.reconstruct(tr, 4, 2)
        ref = orc.exl3_gemm_f64(x, tr, suh, svh, 4, 2, w=w)
        f = faulty_outputs(x, suh, svh, w, fp32)
        for name in names:
            assert f64_bars(f[name], ref, fp32), (name, k, n, m, fp32, rel_err(f[name], ref))


MOE_FAULTS = ("GELU in erf form", "activation from unrounded fp32 g / u", "limit after the multiply")
# Faults of exl3_moe's activation stage that change h by about as much as the kernel's own fp32 accumulation order does (it flips
# ~2 % of the fp16 roundings of g and u, and with them h): they sit at 0.1-1.3x MOE_MODEL_BAR here, so no bar that passes the
# kernel can catch them from the operator's output.
MOE_FAULTS_IN_THE_NOISE = {"GELU in erf form", "activation from unrounded fp32 g / u"}


def moe_fault(name, c, monkeypatch):
    """exl3_moe_model with the fault applied to its activation stage, or None where the fault changes nothing."""
    from scipy.special import erf
    act_ok, gemm_ok = orc.moe_act, orc.exl3_gemm_f16_model
    if name == "GELU in erf form":
        if c["act"] != 1:
            return None

        def act(g, u, a, limit):
            gf, uf = g.astype(np.float32), u.astype(np.float32)
            av = (0.5 * gf * (1 + erf(gf / np.sqrt(2)))).astype(np.float32)
            if limit:
                uf = np.clip(uf, -limit, limit).astype(np.float32); av = np.minimum(av, np.float32(limit))
            return (av * uf).astype(np.float16)
        monkeypatch.setattr(orc, "moe_act", act)
    elif name == "activation from unrounded fp32 g / u":
        monkeypatch.setattr(orc, "exl3_gemm_f16_model",
                            lambda *a, **kw: gemm_ok(*a[:6], np.float32, **kw) if a[6] == np.float16 else gemm_ok(*a, **kw))
    else:
        if not c["limit"]:
            return None

        def act(g, u, a, limit):
            return np.clip(act_ok(g, u, a, 0.0).astype(np.float32), -limit, limit).astype(np.float16)
        monkeypatch.setattr(orc, "moe_act", act)
    try:
        return orc.exl3_moe_model(**c)
    finally:
        monkeypatch.setattr(orc, "moe_act", act_ok)
        monkeypatch.setattr(orc, "exl3_gemm_f16_model", gemm_ok)


@pytest.mark.parametrize("act,limit", [(0, 0.0), (1, 0.0), (2, 0.0), (0, 0.4), (1, 0.5), (2, 0.6)])
def test_fault_catalog_moe(monkeypatch, act, limit):
    c = moe_setup(act, limit, seed=10 + act)
    model = orc.exl3_moe_model(**c)
    touched = (model != c["out"]).any(axis=1)
    for name in MOE_FAULTS:
        y = moe_fault(name, c, monkeypatch)
        if y is None:
            continue
        mx, rms = rel_err(y[touched], model[touched])
        r = max(mx / MOE_MODEL_BAR[0], rms / MOE_MODEL_BAR[1])
        assert (r < MARGIN) if name in MOE_FAULTS_IN_THE_NOISE else (r >= MARGIN), (name, act, limit, mx, rms)
