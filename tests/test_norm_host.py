"""
The RMSNorm operators without a GPU: properties of the fp64 model (oracle/norm_oracle.py) the GPU tests hold the kernels to,
the reference's recorded call sites (tests/golden/ref_norm_callsites.json.gz) bound against the shim's signatures, and a catalog
of invalid calls with the exception and message each raises, in the shim or in the C ABI, before any device access.
"""
import contextlib, ctypes, gzip, inspect, json, os
import pytest
import torch

from oracle import norm_oracle as no

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ERR_SHAPE, ERR_ARG, ERR_UNSUP = -1, -2, -4


# ---- the fp64 model -------------------------------------------------------------------------------------------------------

def _x(rows=3, dim=64, dtype=torch.float, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(rows, dim, generator=g, dtype=torch.float64).to(dtype)


def test_model_scale_invariant():
    x, w = _x(), _x(1, 64, seed=1)[0]
    a = no.rms_norm_f64(x, w, 0.0)
    for s in (2.0 ** -6, 2.0 ** 5):
        assert torch.allclose(no.rms_norm_f64(x * s, w, 0.0), a, rtol=1e-12, atol=0)


def test_model_no_weight_is_unit_weight():
    x = _x()
    assert torch.equal(no.rms_norm_f64(x, None, 1e-6, 0.0, 0.75), no.rms_norm_f64(x, torch.ones(64), 1e-6, 0.0, 0.75))
    # constant_bias applies to a present w only, as in the reference
    assert torch.equal(no.rms_norm_f64(x, None, 1e-6, 1.0), no.rms_norm_f64(x, None, 1e-6, 0.0))
    assert torch.equal(no.rms_norm_f64(x, torch.zeros(64), 1e-6, 1.0), no.rms_norm_f64(x, torch.ones(64), 1e-6, 0.0))


def test_model_post_is_old_y_plus_none():
    x, w, y0 = _x(), _x(1, 64, seed=1)[0], _x(seed=2)
    v = no.rms_norm_f64(x, w, 1e-6)
    assert torch.equal(y0.double() + v, y0.double() + no.rms_norm_f64(x, w, 1e-6))


def test_model_in_is_rounded_add_then_none():
    x, r = _x(dtype=torch.half) * 300, _x(seed=3, dtype=torch.half)
    x[0, 0] = float("inf")
    r2 = no.res_in_sum(x, r)
    assert r2.dtype == torch.half
    assert torch.equal(r2, (x.float().clamp(-65504, 65504) + r.float()).half())
    assert torch.equal(no.res_in_sum(x, r.float()), x.float().clamp(-65504, 65504) + r.float())
    assert torch.equal(no.rms_norm_f64(r2, None, 1e-6), no.rms_norm_f64(r2.float(), None, 1e-6))


def test_model_clamps_fp16_input():
    x = torch.zeros(1, 8, dtype=torch.half)
    x[0, 0], x[0, 1] = float("inf"), -float("inf")
    v = no.rms_norm_f64(x, None, 0.0)
    assert torch.isfinite(v).all() and v[0, 0] == -v[0, 1] == 2.0
    assert no.rms_norm_f64(torch.zeros(2, 8), None, 1e-6).abs().max() == 0


def test_model_gated():
    x, g = _x(4, 8, torch.bfloat16), _x(4, 8, seed=5)
    w = _x(2, 8, seed=6).flatten()
    y = no.gated_rms_norm_f64(x, w, g, 1e-5, 0.0, 2, False)
    s = no.silu_f64(g)
    assert torch.allclose(y[1], no.rms_norm_f64(x[1:2], w[8:], 1e-5)[0] * s[1], rtol=1e-12)
    yf = no.gated_rms_norm_f64(x, w, g, 1e-5, 0.0, 2, True)
    assert torch.allclose(yf[2], no.rms_norm_f64((x.double() * s)[2:3], w[:8], 1e-5)[0], rtol=1e-12)


def test_ulp16():
    assert no.ulp16(torch.tensor([1.0, 1.5, 2.0, -3.0, 0.0, 1e-6])).tolist() == [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -9,
                                                                                2.0 ** -24, 2.0 ** -24]


# ---- the reference's call sites --------------------------------------------------------------------------------------------

def test_reference_call_sites_bind():
    from exllamav3_b200 import ext
    with gzip.open(os.path.join(GOLDEN, "ref_norm_callsites.json.gz")) as f:
        rec = json.loads(f.read())
    assert {s["name"] for s in rec["sites"]} == {"rms_norm", "rms_norm_res_in", "gated_rms_norm"}
    for s in rec["sites"]:
        sig = inspect.signature(getattr(ext, s["name"]))
        sig.bind(*([None] * s["positional"]), **{k: None for k in s["keywords"]})


# ---- invalid calls -----------------------------------------------------------------------------------------------------------

@pytest.fixture()
def host_shim(monkeypatch):
    """The shim with its CUDA plumbing stubbed: CPU tensors reach the argument checks and the C ABI's own checks, which come
    before any device access."""
    from exllamav3_b200 import ext
    monkeypatch.setattr(ext, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(ext, "_stream", lambda t: None)
    monkeypatch.setattr(ext.torch.cuda, "device", lambda d: contextlib.nullcontext())
    yield ext


def _t(*shape, dtype=torch.half):
    return torch.zeros(shape, dtype=dtype)


def rms(ext, x=None, w="default", y=None, add_residual=False, span_heads=False):
    x = _t(2, 64) if x is None else x
    w = _t(x.shape[-1]) if isinstance(w, str) else w
    y = torch.zeros_like(x) if y is None else y
    return ext.rms_norm(x, w, y, 1e-6, 0.0, 1.0, span_heads, add_residual)


def res_in(ext, x=None, w="default", y=None, r="default"):
    x = _t(2, 64) if x is None else x
    w = _t(x.shape[-1]) if isinstance(w, str) else w
    y = torch.zeros_like(x) if y is None else y
    r = torch.zeros_like(x) if isinstance(r, str) else r
    return ext.rms_norm_res_in(x, w, y, r, 1e-6, 0.0, 1.0)


def gated(ext, x=None, w=None, y=None, g=None, w_groups=1):
    x = _t(2, 64, dtype=torch.bfloat16) if x is None else x
    w = _t(x.shape[-1] * w_groups, dtype=torch.float) if w is None else w
    y = _t(*x.shape) if y is None else y
    g = _t(*x.shape, dtype=torch.bfloat16) if g is None else g
    return ext.gated_rms_norm(x, w, y, g, 1e-5, 0.0, w_groups, False)


def _noncontig(x):
    return x.transpose(-1, -2).contiguous().transpose(-1, -2)


INVALID = [
    ("dim % 4", lambda e: rms(e, x=_t(2, 6)), "x dimension -1 must be divisible by 4"),
    ("dim % 4, span_heads", lambda e: rms(e, x=_t(2, 3, 2), w=None, span_heads=True), "x dimension -1 must be divisible by 4"),
    ("dim % 4, res_in", lambda e: res_in(e, x=_t(2, 10)), "x dimension -1 must be divisible by 4"),
    ("dim % 4, gated", lambda e: gated(e, x=_t(2, 6, dtype=torch.bfloat16)), "x dimension -1 must be divisible by 4"),
    ("x / y shapes", lambda e: rms(e, y=_t(2, 128)), "x and y have incompatible shapes"),
    ("x / y rows", lambda e: rms(e, y=_t(3, 64)), "x and y have incompatible shapes"),
    ("x / r shapes", lambda e: res_in(e, r=_t(3, 64)), "x and r have incompatible shapes"),
    ("x / g shapes", lambda e: gated(e, g=_t(2, 128, dtype=torch.bfloat16)), "x and g have incompatible shapes"),
    ("w length", lambda e: rms(e, w=_t(32)), "x and w have incompatible shapes"),
    ("w 2-D", lambda e: rms(e, w=_t(64, 2)), "x and w have incompatible shapes"),
    ("w length, res_in", lambda e: res_in(e, w=_t(128)), "x and w have incompatible shapes"),
    ("w length, gated", lambda e: gated(e, w=_t(32, dtype=torch.float)), "x and w have incompatible shapes"),
    ("w_groups * dim", lambda e: gated(e, w=_t(64 * 3, dtype=torch.float), w_groups=2), "w must have w_groups * dim elements"),
    ("w_groups 0", lambda e: gated(e, w_groups=0), "w_groups must be positive"),
    ("missing r", lambda e: res_in(e, r=None), "rms_norm: res_mode RES_IN requires residual tensor"),
    ("x bf16", lambda e: rms(e, x=_t(2, 64, dtype=torch.bfloat16)), "rms_norm: Invalid datatypes for input/output"),
    ("w fp32", lambda e: rms(e, w=_t(64, dtype=torch.float)), "rms_norm: Invalid datatypes for input/output"),
    ("y bf16", lambda e: rms(e, y=_t(2, 64, dtype=torch.bfloat16)), "rms_norm: Invalid datatypes for input/output"),
    ("y bf16, post", lambda e: rms(e, y=_t(2, 64, dtype=torch.bfloat16), add_residual=True), "rms_norm: Invalid datatypes for input/output"),
    ("res_in y fp32", lambda e: res_in(e, y=_t(2, 64, dtype=torch.float)), "rms_norm: Invalid datatypes for input/output"),
    ("res_in r bf16", lambda e: res_in(e, r=_t(2, 64, dtype=torch.bfloat16)), "rms_norm: Invalid datatypes for input/output"),
    ("x int", lambda e: rms(e, x=_t(2, 64, dtype=torch.int16)), "rms_norm: Invalid datatypes for input/output"),
    ("gated x fp16", lambda e: gated(e, x=_t(2, 64)), "gated_rms_norm: Invalid datatypes for input/output"),
    ("gated w fp16", lambda e: gated(e, w=_t(64)), "gated_rms_norm: Invalid datatypes for input/output"),
    ("gated g fp16", lambda e: gated(e, g=_t(2, 64)), "gated_rms_norm: Invalid datatypes for input/output"),
    ("gated y bf16", lambda e: gated(e, y=_t(2, 64, dtype=torch.bfloat16)), "gated_rms_norm: Invalid datatypes for input/output"),
    ("x non-contiguous", lambda e: rms(e, x=_noncontig(_t(64, 64)), w=None), "must be contiguous"),
    ("y non-contiguous", lambda e: rms(e, x=_t(64, 64), y=_noncontig(_t(64, 64)), w=None), "must be contiguous"),
    ("r non-contiguous", lambda e: res_in(e, x=_t(64, 64), r=_noncontig(_t(64, 64)), w=None), "must be contiguous"),
    ("g non-contiguous", lambda e: gated(e, x=_t(64, 64, dtype=torch.bfloat16), g=_noncontig(_t(64, 64, dtype=torch.bfloat16))),
     "must be contiguous"),
    ("dim > 16384", lambda e: rms(e, x=_t(1, 16388), w=None), "exceeds the 16384 elements"),
    ("dim > 16384, gated", lambda e: gated(e, x=_t(1, 16388, dtype=torch.bfloat16)), "exceeds the 16384 elements"),
    ("x misaligned", lambda e: rms(e, x=_t(129, dtype=torch.float)[1:].view(2, 64), w=None), "must be aligned to 4 of their elements"),
]


@pytest.mark.parametrize("what,call,msg", INVALID, ids=[c[0] for c in INVALID])
def test_invalid_call(host_shim, what, call, msg):
    n = host_shim.launch_count()
    with pytest.raises(RuntimeError, match=msg.replace("*", r"\*").replace("(", r"\(")):
        call(host_shim)
    assert host_shim.launch_count() == n


def test_non_cuda_tensor_refused():
    from exllamav3_b200 import ext
    with pytest.raises(RuntimeError, match="not on a CUDA device"):
        rms(ext)
    with pytest.raises(RuntimeError, match="not on a CUDA device"):
        gated(ext)


def test_empty_calls_launch_nothing(host_shim):
    n = host_shim.launch_count()
    rms(host_shim, x=_t(0, 64))
    res_in(host_shim, x=_t(0, 4096))
    gated(host_shim, x=_t(0, 128, dtype=torch.bfloat16))
    rms(host_shim, x=_t(3, 0), w=None)
    assert host_shim.launch_count() == n


def test_c_abi_checks():
    from exllamav3_b200 import ext
    lib = ext.lib
    buf = torch.zeros(4096, dtype=torch.half)
    p = buf.data_ptr()
    err = lambda: lib.exl3b_last_error().decode()
    assert lib.exl3b_rms_norm(None, p, None, p, None, 2, 64, 0, 0, 0, 0, 3, 1e-6, 0.0, 1.0) == ERR_ARG
    assert "res_mode must be" in err()
    assert lib.exl3b_rms_norm(None, p, None, p, None, 2, 62, 0, 0, 0, 0, 0, 1e-6, 0.0, 1.0) == ERR_SHAPE
    assert lib.exl3b_rms_norm(None, p, None, p, None, -1, 64, 0, 0, 0, 0, 0, 1e-6, 0.0, 1.0) == ERR_SHAPE
    assert lib.exl3b_rms_norm(None, p, None, p, None, 2, 64, 0, 0, 0, 0, 2, 1e-6, 0.0, 1.0) == ERR_ARG
    assert "RES_IN requires residual tensor" in err()
    assert lib.exl3b_rms_norm(None, p, p, p, p, 2, 64, 0, 0, 1, 1, 2, 1e-6, 0.0, 1.0) == ERR_ARG       # RES_IN, y fp32
    assert err() == "rms_norm: Invalid datatypes for input/output"
    assert lib.exl3b_rms_norm(None, p, None, None, None, 2, 64, 0, 0, 0, 0, 0, 1e-6, 0.0, 1.0) == ERR_ARG
    assert "null tensor" in err()
    assert lib.exl3b_rms_norm(None, p, None, p, None, 1, 32768, 0, 0, 0, 0, 0, 1e-6, 0.0, 1.0) == ERR_UNSUP
    assert lib.exl3b_rms_norm(None, p + 2, None, p, None, 2, 64, 0, 0, 0, 0, 0, 1e-6, 0.0, 1.0) == ERR_ARG
    assert "aligned" in err()
    assert lib.exl3b_gated_rms_norm(None, p, p, p, p, 2, 64, 0, 1, 0, 2, 1, 0, 1e-5, 0.0) == ERR_ARG     # x fp16
    assert err() == "gated_rms_norm: Invalid datatypes for input/output"
    assert lib.exl3b_gated_rms_norm(None, p, p, p, p, 2, 64, 2, 1, 0, 2, 0, 0, 1e-5, 0.0) == ERR_ARG
    assert "w_groups must be positive" in err()
    # a valid call with no rows returns before any device access
    assert lib.exl3b_rms_norm(None, p, None, p, None, 0, 64, 0, 0, 0, 0, 0, 1e-6, 0.0, 1.0) == 0
    assert lib.exl3b_gated_rms_norm(None, p, p, p, p, 0, 64, 2, 1, 0, 2, 1, 0, 1e-5, 0.0) == 0
