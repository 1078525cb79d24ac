"""
The RMSNorm operators on the GPU (rms_norm, rms_norm_res_in, gated_rms_norm), held to the fp64 model of oracle/norm_oracle.py
and to the reference kernel's outputs in tests/golden/ref_norm.npz (oracle/gen_golden_norm.py).  Bars:
  fp16 y     within 1 fp16 ulp of fp16(model); RES_POST adds 2^-20 (|y_old| + |v|) for cancellation (v: the normalized term)
  fp32 y     |y - model| <= 4e-6 |v| (+ 4e-6 |y_old| in RES_POST);  gated operator 1e-5 |v|
  RES_IN     the residual written back is bit-identical to (x_clamped.float() + r.float()).to(r.dtype)
Beyond the bars: results are bit-identical in place and out of place, for a row alone and inside a 257-row call, over repeated
calls and under CUDA-graph replay; memory around y and r keeps its bits.
"""
import json, os
import numpy as np
import pytest
import torch

from oracle import norm_oracle as no
from oracle import gen_golden_norm as gg

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_norm.npz")


@pytest.fixture(scope="module")
def ext(cuda):
    from exllamav3_b200 import ext
    return ext


def assert_bars(y, v, y_old=None, gated=False, what=""):
    """y (the kernel's, any device) against the model value v (+ y_old in RES_POST), with the bar of y's dtype"""
    y, v = y.cpu(), v.cpu().double()
    yo = torch.zeros_like(v) if y_old is None else y_old.cpu().double()
    model = v + yo
    if y.dtype == torch.half:
        tol = no.ulp16(model) + 2.0 ** -20 * (yo.abs() + v.abs()) * (y_old is not None)
        err = (y.double() - model.half().double()).abs()
    else:
        tol = (1e-5 if gated else 4e-6) * v.abs() + 4e-6 * yo.abs()
        err = (y.double() - model).abs()
    bad = err > tol
    assert not bad.any(), f"{what}: {int(bad.sum())} elements over the bar, worst {err[bad].max().item():.3g} (model {model[bad][0].item():.6g})"


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale).to(dtype)


# ---- every dtype combination, residual mode, w / bias / scale, against the model and the reference kernel -------------------

def _golden():
    if not os.path.exists(GOLDEN):
        pytest.fail(f"{GOLDEN} missing: run oracle/gen_golden_norm.py on a GPU machine")
    z = np.load(GOLDEN)
    return z, json.loads(bytes(z["meta"]).decode())


def test_golden_cases(ext, cuda):
    z, cases = _golden()
    assert len(cases) == len(gg.case_list())
    for i, c in enumerate(cases):
        t = {k: gg.from_np(z[f"{i}_{k}"], c[{"y0": "y", "r0": "r"}.get(k, k)]) for k in ("x", "w", "y0", "r0", "g") if f"{i}_{k}" in z}
        y, r = gg.run(ext, c, t, cuda)
        y_ref = gg.from_np(z[f"{i}_y"], c["y"])
        what = f"case {i} {c}"
        if c["op"] == "gated_rms_norm":
            v = no.gated_rms_norm_f64(t["x"], t["w"], t["g"], c["eps"], c["bias"], c["w_groups"], c["gate_first"])
            assert_bars(y, v, gated=True, what=what)
            assert_bars(y_ref, v, gated=True, what="reference " + what)
            assert_bars(y, y_ref.double(), gated=True, what="against the reference, " + what)
            continue
        x = t["x"]
        if c["mode"] == "in":
            r_new = no.res_in_sum(x, t["r0"])
            assert torch.equal(r, r_new), what
            assert torch.equal(gg.from_np(z[f"{i}_r"], c["r"]), r_new), "reference " + what
            x = r_new
        v = no.rms_norm_f64(x, t.get("w"), c["eps"], c["bias"], c["scale"])
        y_old = t.get("y0")
        assert_bars(y, v, y_old, what=what)
        assert_bars(y_ref, v, y_old, what="reference " + what)
        if y.dtype == torch.half:                  # the two kernels one fp16 step apart, plus RES_POST's cancellation term
            tol = no.ulp16(y_ref.double()) + (0 if y_old is None else 2.0 ** -20 * (y_old.double().abs() + v.abs()))
            assert ((y.double() - y_ref.double()).abs() <= tol).all(), "against the reference, " + what


# ---- sizes: decode, head norms, prefill ------------------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [4096, 8192])
@pytest.mark.parametrize("rows", [1, 2, 3, 4, 5, 6, 7, 8])
def test_decode_sizes(ext, cuda, rows, dim):
    x = _rand((rows, dim), torch.half, rows * dim, 3.0).to(cuda)
    w = _rand(dim, torch.half, 7, 0.1).add(1).to(cuda)
    y = torch.empty_like(x)
    ext.rms_norm(x, w, y, 1e-6, 0.0, 1.0, False, False)
    assert_bars(y, no.rms_norm_f64(x.cpu(), w.cpu(), 1e-6), what=f"NONE {rows}x{dim}")
    r = _rand((rows, dim), torch.float, 11, 5.0).to(cuda)
    r0 = r.clone()
    ext.rms_norm_res_in(x, w, y, r, 1e-6, 0.0, 1.0)
    r_new = no.res_in_sum(x.cpu(), r0.cpu())
    assert torch.equal(r.cpu(), r_new)
    assert_bars(y, no.rms_norm_f64(r_new, w.cpu(), 1e-6), what=f"IN {rows}x{dim}")


def test_head_norms(ext, cuda):
    # per-head norm of (tokens, heads, head_dim) and the span_heads form over the last two dimensions
    x = _rand((8, 32, 128), torch.half, 21, 2.0).to(cuda)
    w = _rand(128, torch.bfloat16, 22, 0.1).to(cuda)
    y = torch.empty(8, 32, 128, dtype=torch.float, device=cuda)
    ext.rms_norm(x, w, y, 1e-6, 1.0, 1.0, False, False)
    assert_bars(y, no.rms_norm_f64(x.cpu(), w.cpu(), 1e-6, 1.0), what="head norm")
    xs = _rand((4, 8, 2, 128), torch.half, 23, 2.0).to(cuda)
    ws = _rand(256, torch.half, 24, 0.1).add(1).to(cuda)
    ys = torch.empty_like(xs)
    ext.rms_norm(xs, ws, ys, 1e-6, 0.0, 1.0, True, False)
    v = no.rms_norm_f64(xs.cpu().flatten(-2), ws.cpu(), 1e-6).view(4, 8, 2, 128)
    assert_bars(ys, v, what="span_heads")
    # gated head norm with weight groups, both gate orders
    xg = _rand((256, 128), torch.bfloat16, 25).to(cuda)
    gg_ = _rand((256, 128), torch.bfloat16, 26, 2.0).to(cuda)
    wg = _rand(4 * 128, torch.float, 27, 0.1).add(1).to(cuda)
    for gate_first in (False, True):
        yg = torch.empty(256, 128, dtype=torch.float, device=cuda)
        ext.gated_rms_norm(xg, wg, yg, gg_, 1e-5, 0.0, 4, gate_first)
        assert_bars(yg, no.gated_rms_norm_f64(xg.cpu(), wg.cpu(), gg_.cpu(), 1e-5, 0.0, 4, gate_first), gated=True,
                    what=f"gated head norm gate_first={gate_first}")


def test_prefill_size(ext, cuda):
    x = _rand((32768, 4096), torch.half, 31).to(cuda)
    w = _rand(4096, torch.half, 32, 0.1).add(1).to(cuda)
    y = torch.empty_like(x)
    ext.rms_norm(x, w, y, 1e-6, 0.0, 1.0, False, False)
    sel = torch.arange(0, 32768, 97)
    assert_bars(y[sel], no.rms_norm_f64(x[sel].cpu(), w.cpu(), 1e-6), what="prefill 32768 x 4096")
    # the rows the sample skipped equal a call on them alone
    y2 = torch.empty_like(x[:300])
    ext.rms_norm(x[:300].contiguous(), w, y2, 1e-6, 0.0, 1.0, False, False)
    assert torch.equal(y[:300], y2)


# ---- invariance, graphs, sentinels, edge inputs -----------------------------------------------------------------------------

@pytest.mark.parametrize("dim", [128, 2880, 4096, 8192])
def test_invariance(ext, cuda, dim):
    x = _rand((257, dim), torch.half, dim, 2.0).to(cuda)
    w = _rand(dim, torch.half, 41, 0.1).add(1).to(cuda)
    y = torch.empty_like(x)
    ext.rms_norm(x, w, y, 1e-6, 0.0, 1.0, False, False)
    for _ in range(3):
        y2 = torch.empty_like(x)
        ext.rms_norm(x, w, y2, 1e-6, 0.0, 1.0, False, False)
        assert torch.equal(y, y2)
    for i in (0, 1, 128, 256):
        y1 = torch.empty(1, dim, dtype=torch.half, device=cuda)
        ext.rms_norm(x[i:i + 1].clone(), w, y1, 1e-6, 0.0, 1.0, False, False)
        assert torch.equal(y1[0], y[i]), f"row {i}"
    xi = x.clone()
    ext.rms_norm(xi, w, xi, 1e-6, 0.0, 1.0, False, False)
    assert torch.equal(xi, y)
    xg = _rand((257, dim), torch.bfloat16, 42).to(cuda)
    g = _rand((257, dim), torch.float, 43).to(cuda)
    wg = _rand(dim, torch.bfloat16, 44).to(cuda)
    ya = torch.empty(257, dim, dtype=torch.half, device=cuda)
    ext.gated_rms_norm(xg, wg, ya, g, 1e-5, 0.0, 1, False)
    yb = torch.empty(1, dim, dtype=torch.half, device=cuda)
    ext.gated_rms_norm(xg[200:201].clone(), wg, yb, g[200:201].clone(), 1e-5, 0.0, 1, False)
    assert torch.equal(ya[200], yb[0])


def test_graph_capture(ext, cuda):
    rows, dim = 4, 8192
    x = _rand((rows, dim), torch.half, 51).to(cuda)
    w = _rand(dim, torch.bfloat16, 52, 0.1).add(1).to(cuda)
    r = _rand((rows, dim), torch.half, 53).to(cuda)
    y, y2 = torch.empty_like(x), torch.empty(rows, dim, dtype=torch.float, device=cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ext.rms_norm_res_in(x, w, y, r.clone(), 1e-6, 0.0, 1.0)          # first call outside the capture
        torch.cuda.synchronize()
        gph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gph, stream=s):
            ext.rms_norm_res_in(x, w, y, r, 1e-6, 0.0, 1.0)
            ext.rms_norm(y, w, y2, 1e-6, 0.0, 0.5, False, True)
    for seed in (54, 55):
        x.copy_(_rand((rows, dim), torch.half, seed).to(cuda))
        r0 = _rand((rows, dim), torch.half, seed + 10).to(cuda)
        r.copy_(r0)
        y2.fill_(0.25)
        gph.replay()
        torch.cuda.synchronize()
        re, ye, y2e = r0.clone(), torch.empty_like(x), torch.full_like(y2, 0.25)
        ext.rms_norm_res_in(x, w, ye, re, 1e-6, 0.0, 1.0)
        ext.rms_norm(ye, w, y2e, 1e-6, 0.0, 0.5, False, True)
        torch.cuda.synchronize()
        assert torch.equal(r, re) and torch.equal(y, ye) and torch.equal(y2, y2e)


def test_sentinels(ext, cuda):
    rows, dim = 5, 4096
    for ydt, rdt in ((torch.half, torch.half), (torch.half, torch.float)):
        ybuf = torch.full((rows + 2, dim), -7.5, dtype=ydt, device=cuda)
        rbuf = torch.full((rows + 2, dim), 3.25, dtype=rdt, device=cuda)
        rbuf[1:-1] = _rand((rows, dim), rdt, 61).to(cuda)
        x = _rand((rows, dim), torch.half, 62).to(cuda)
        ext.rms_norm_res_in(x, None, ybuf[1:-1], rbuf[1:-1], 1e-6, 0.0, 1.0)
        torch.cuda.synchronize()
        for b, val in ((ybuf, -7.5), (rbuf, 3.25)):
            assert (b[0] == val).all() and (b[-1] == val).all()
    yb = torch.full((3, 130), 9.0, dtype=torch.float, device=cuda)
    y = yb.view(-1)[132:260].view(1, 128)                           # 16-byte aligned; the elements around it keep their bits
    ext.gated_rms_norm(_rand((1, 128), torch.bfloat16, 63).to(cuda), _rand(128, torch.float, 64).to(cuda), y,
                       _rand((1, 128), torch.float, 65).to(cuda), 1e-5, 0.0, 1, True)
    torch.cuda.synchronize()
    flat = yb.view(-1)
    assert (flat[:132] == 9.0).all() and (flat[260:] == 9.0).all() and not (y == 9.0).any()


def test_edge_inputs(ext, cuda):
    dim = 4096
    x = _rand((4, dim), torch.half, 71).to(cuda)
    x[0, 5], x[0, 77], x[2, 0] = float("inf"), -float("inf"), float("inf")
    x[1].zero_()
    w = _rand(dim, torch.half, 72, 0.1).add(1).to(cuda)
    for ydt in (torch.half, torch.float):
        y = torch.empty(4, dim, dtype=ydt, device=cuda)
        ext.rms_norm(x, w, y, 1e-6, 0.0, 1.0, False, False)
        assert torch.isfinite(y.float()).all()
        assert_bars(y, no.rms_norm_f64(x.cpu(), w.cpu(), 1e-6), what=f"inf / zero rows, y {ydt}")
        assert (y[1] == 0).all()
    # an all-zero row has rmf = rsqrt(eps): a zero row of r in RES_IN stays zero and y is zero
    r = torch.zeros(2, dim, dtype=torch.float, device=cuda)
    y = torch.empty(2, dim, dtype=torch.half, device=cuda)
    ext.rms_norm_res_in(torch.zeros(2, dim, dtype=torch.half, device=cuda), w, y, r, 1e-6, 0.0, 1.0)
    assert (y == 0).all() and (r == 0).all()
    # a tiny row: the eps term dominates, so y = x * w * rsqrt(eps)
    xt = torch.full((1, dim), 1e-4, dtype=torch.float, device=cuda)
    yt = torch.empty_like(xt)
    ext.rms_norm(xt, None, yt, 1e-2, 0.0, 1.0, False, False)
    assert_bars(yt, no.rms_norm_f64(xt.cpu(), None, 1e-2), what="eps-dominated row")


def test_odd_dims_and_alignment(ext, cuda):
    # dim % 8 != 0 and views that are 8- but not 16-byte aligned take the 8-byte load path
    for dim in (4, 12, 2884):
        x = _rand((3, dim), torch.half, dim, 2.0).to(cuda)
        w = _rand(dim, torch.half, 81, 0.1).add(1).to(cuda)
        y = torch.empty_like(x)
        ext.rms_norm(x, w, y, 1e-6, 0.0, 1.0, False, False)
        assert_bars(y, no.rms_norm_f64(x.cpu(), w.cpu(), 1e-6), what=f"dim {dim}")
    buf = _rand(4 + 2 * 64, torch.half, 82).to(cuda)
    x = buf[4:].view(2, 64)                                        # 8-byte aligned
    y = torch.empty(2, 64, dtype=torch.float, device=cuda)
    ext.rms_norm(x, None, y, 1e-6, 0.0, 2.0, False, False)
    assert_bars(y, no.rms_norm_f64(x.cpu(), None, 1e-6, 0.0, 2.0), what="8-byte aligned view")
