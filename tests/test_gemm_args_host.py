"""
Argument checks of the decode-GEMM entry points, without a GPU: a catalog of invalid calls to exl3_gemm, exl3_gemm_allreduce,
exl3_gemv, exl3_gemm_gated, GemmChain and exl3_mgemm with the exception each raises and a substring of its message, and the
C ABI's own checks (exl3b_gemm, exl3b_gemm_gated, exl3b_gemm_allreduce, exl3b_gemm_plan) with their status codes and
exl3b_last_error text.  Every call here is refused before any device access, in the shim or in the library.
"""
import contextlib, ctypes
import pytest
import torch

ERR_SHAPE, ERR_ARG, ERR_UNSUP = -1, -2, -4
TAG_NOP = 0


@pytest.fixture()
def host_shim(monkeypatch):
    """The shim with its CUDA plumbing stubbed: CPU tensors reach the argument checks and the C ABI's own checks, which come
    before any device access."""
    from exllamav3_b200 import ext
    monkeypatch.setattr(ext, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(ext, "_stream", lambda t: None)
    monkeypatch.setattr(ext.torch.cuda, "device", lambda d: contextlib.nullcontext())
    yield ext
    ext.set_gemm_path(0)


def _h(*shape):
    return torch.zeros(shape, dtype=torch.half)


def _trellis(k=256, n=128, K=4):
    return torch.zeros((k // 16, n // 16, 16 * K), dtype=torch.int16)


def _t(x):
    """A non-contiguous view with x's shape and values."""
    return x.transpose(-1, -2).contiguous().transpose(-1, -2) if x.dim() >= 2 else x


def gemm(ext, A=None, B=None, C=None, mcg=False, mul1=True):
    A = _h(2, 256) if A is None else A
    B = _trellis() if B is None else B
    C = _h(2, 128) if C is None else C
    return ext.exl3_gemm(A, B, C, None, None, None, -1, mcg, mul1, 0)


def allreduce(ext, A=None, B=None, C=None, mcg=False, mul1=True):
    A = _h(2, 256) if A is None else A
    B = _trellis() if B is None else B
    C = _h(2, 128) if C is None else C
    return ext.exl3_gemm_allreduce(A, B, C, None, None, None, mcg, mul1)


def gemv(ext, A=None, B=None, C=None, mcg=False, mul1=True):
    A = _h(2, 256) if A is None else A
    B = _trellis() if B is None else B
    C = _h(2, 128) if C is None else C
    return ext.exl3_gemv(A, B, C, _h(256), _h(2, 256), _h(128), mcg, mul1)


def gated(ext, G=None, U=None, B=None, C=None, mcg=False, mul1=True):
    G = _h(2, 256) if G is None else G
    U = torch.zeros_like(G) if U is None else U
    B = _trellis() if B is None else B
    C = _h(2, 128) if C is None else C
    return ext.exl3_gemm_gated(G, U, B, C, None, None, ext.ACT_SILU, 0.0, mcg, mul1)


def chain(ext, **op):
    o = {"x": _h(2, 256), "trellis": _trellis(), "y": _h(2, 128), "mul1": True}
    o.update(op)
    return ext.GemmChain([o])


def mgemm(ext, A=None, B=None, C=None, suh=None, K=4, mcg=False, mul1=True, idx=None):
    A = _h(1, 2, 256) if A is None else A
    B = torch.tensor([16, 32], dtype=torch.long) if B is None else B
    C = _h(2, 2, 128) if C is None else C
    suh = torch.tensor([16, 32], dtype=torch.long) if suh is None else suh
    svh = torch.tensor([16, 32], dtype=torch.long)
    Ah = _h(2, 2, 256)
    return ext.exl3_mgemm(A, B, C, suh, Ah, svh, idx, None, K, -1, mcg, mul1, -1, -1, 0)


# (id, call, exception, message substring)
CATALOG = [
    # exl3_gemm
    ("gemm-A-dtype", lambda e: gemm(e, A=torch.zeros(2, 256)), RuntimeError, "A is incorrect datatype"),
    ("gemm-B-dtype", lambda e: gemm(e, B=_trellis().int()), RuntimeError, "B is incorrect datatype"),
    ("gemm-C-dtype", lambda e: gemm(e, C=torch.zeros(2, 128, dtype=torch.bfloat16)), RuntimeError, "C is incorrect datatype"),
    ("gemm-B-rank", lambda e: gemm(e, B=_trellis()[0]), RuntimeError, "B: incorrect number of dimensions"),
    ("gemm-k-mismatch", lambda e: gemm(e, A=_h(2, 384)), RuntimeError, "A and B incompatible shapes"),
    ("gemm-n-mismatch", lambda e: gemm(e, C=_h(2, 256)), RuntimeError, "C and B incompatible shapes"),
    ("gemm-k-128", lambda e: gemm(e, A=_h(2, 144), B=_trellis(k=144)), RuntimeError, "exl3_gemm: k (144) must be divisible by 128"),
    ("gemm-n-128", lambda e: gemm(e, B=_trellis(n=144), C=_h(2, 144)), RuntimeError, "exl3_gemm: n (144) must be divisible by 128"),
    ("gemm-K-9", lambda e: gemm(e, B=_trellis(K=9)), RuntimeError, "K must be 1..8"),
    ("gemm-K-0", lambda e: gemm(e, B=_trellis(K=0)), RuntimeError, "K must be 1..8"),
    ("gemm-mcg-mul1", lambda e: gemm(e, mcg=True, mul1=True), RuntimeError, "Specified both mcg and mul1"),
    ("gemm-A-strided", lambda e: gemm(e, A=_t(_h(2, 256))), RuntimeError, "exl3_gemm"),
    ("gemm-C-strided", lambda e: gemm(e, C=_t(_h(2, 128))), RuntimeError, "exl3_gemm"),
    ("gemm-B-strided", lambda e: gemm(e, B=_t(_trellis())), RuntimeError, "exl3_gemm"),
    # exl3_gemm_allreduce
    ("allreduce-A-dtype", lambda e: allreduce(e, A=torch.zeros(2, 256)), RuntimeError, "A is incorrect datatype"),
    ("allreduce-B-rank", lambda e: allreduce(e, B=_trellis()[0]), RuntimeError, "B: incorrect number of dimensions"),
    ("allreduce-k-mismatch", lambda e: allreduce(e, A=_h(2, 384)), RuntimeError, "A and B incompatible shapes"),
    ("allreduce-n-mismatch", lambda e: allreduce(e, C=_h(2, 256)), RuntimeError, "C and B incompatible shapes"),
    ("allreduce-k-128", lambda e: allreduce(e, A=_h(2, 144), B=_trellis(k=144)), RuntimeError,
     "exl3_gemm_allreduce: k (144) must be divisible by 128"),
    ("allreduce-n-128", lambda e: allreduce(e, B=_trellis(n=144), C=_h(2, 144)), RuntimeError,
     "exl3_gemm_allreduce: n (144) must be divisible by 128"),
    ("allreduce-no-rows", lambda e: allreduce(e, A=_h(0, 256), C=_h(0, 128)), RuntimeError, "exl3_gemm_allreduce: bad size"),
    ("allreduce-K-9", lambda e: allreduce(e, B=_trellis(K=9)), RuntimeError, "K must be 1..8"),
    ("allreduce-mcg-mul1", lambda e: allreduce(e, mcg=True, mul1=True), RuntimeError, "Specified both mcg and mul1"),
    ("allreduce-A-strided", lambda e: allreduce(e, A=_t(_h(2, 256))), RuntimeError, "exl3_gemm_allreduce"),
    ("allreduce-C-strided", lambda e: allreduce(e, C=_t(_h(2, 128))), RuntimeError, "exl3_gemm_allreduce"),
    # exl3_gemv (eligibility, then exl3_gemm)
    ("gemv-A-dtype", lambda e: gemv(e, A=torch.zeros(2, 256)), RuntimeError, "A is incorrect datatype"),
    ("gemv-B-rank", lambda e: gemv(e, B=_trellis()[0]), RuntimeError, "B: incorrect number of dimensions"),
    ("gemv-k-mismatch", lambda e: gemv(e, A=_h(2, 384)), RuntimeError, "A and B incompatible shapes"),
    ("gemv-n-mismatch", lambda e: gemv(e, C=_h(2, 256)), RuntimeError, "C and B incompatible shapes"),
    ("gemv-k-128", lambda e: gemv(e, A=_h(2, 144), B=_trellis(k=144)), RuntimeError, "exl3_gemv: call not eligible"),
    ("gemv-K-5", lambda e: gemv(e, B=_trellis(K=5)), RuntimeError, "exl3_gemv: call not eligible"),
    ("gemv-rows", lambda e: gemv(e, A=_h(9, 256), C=_h(9, 128)), RuntimeError, "exl3_gemv: call not eligible"),
    ("gemv-mcg-mul1", lambda e: gemv(e, mcg=True, mul1=True), RuntimeError, "Specified both mcg and mul1"),
    ("gemv-A-strided", lambda e: gemv(e, A=_t(_h(2, 256))), RuntimeError, "exl3_gemv"),
    # exl3_gemm_gated
    ("gated-G-dtype", lambda e: gated(e, G=torch.zeros(2, 256, dtype=torch.bfloat16), U=torch.zeros(2, 256, dtype=torch.bfloat16)),
     RuntimeError, "G is incorrect datatype"),
    ("gated-U-dtype", lambda e: gated(e, U=torch.zeros(2, 256)), RuntimeError, "U is incorrect datatype"),
    ("gated-B-dtype", lambda e: gated(e, B=_trellis().int()), RuntimeError, "B is incorrect datatype"),
    ("gated-C-dtype", lambda e: gated(e, C=torch.zeros(2, 128, dtype=torch.bfloat16)), RuntimeError, "C is incorrect datatype"),
    ("gated-B-rank", lambda e: gated(e, B=_trellis()[0]), RuntimeError, "B: incorrect number of dimensions"),
    ("gated-GU-mismatch", lambda e: gated(e, U=_h(1, 256)), RuntimeError, "G and U incompatible shapes"),
    ("gated-k-mismatch", lambda e: gated(e, G=_h(2, 384)), RuntimeError, "G and B incompatible shapes"),
    ("gated-n-mismatch", lambda e: gated(e, C=_h(2, 256)), RuntimeError, "C and B incompatible shapes"),
    ("gated-C-rows", lambda e: gated(e, C=_h(3, 128)), RuntimeError, "C and B incompatible shapes"),
    ("gated-k-128", lambda e: gated(e, G=_h(2, 144), B=_trellis(k=144)), RuntimeError, "exl3_gemm_gated: k (144) must be divisible by 128"),
    ("gated-n-128", lambda e: gated(e, B=_trellis(n=144), C=_h(2, 144)), RuntimeError, "exl3_gemm_gated: n (144) must be divisible by 128"),
    ("gated-K-9", lambda e: gated(e, B=_trellis(K=9)), RuntimeError, "K must be 1..8"),
    ("gated-mcg-mul1", lambda e: gated(e, mcg=True, mul1=True), RuntimeError, "Specified both mcg and mul1"),
    ("gated-G-strided", lambda e: gated(e, G=_t(_h(2, 256))), RuntimeError, "exl3_gemm_gated: tensors must be contiguous"),
    ("gated-U-strided", lambda e: gated(e, U=_t(_h(2, 256))), RuntimeError, "exl3_gemm_gated: tensors must be contiguous"),
    # GemmChain (one op)
    ("chain-empty", lambda e: e.GemmChain([]), RuntimeError, "GemmChain: empty op list"),
    ("chain-x-dtype", lambda e: chain(e, x=torch.zeros(2, 256)), RuntimeError, "A is incorrect datatype"),
    ("chain-B-dtype", lambda e: chain(e, trellis=_trellis().int()), RuntimeError, "B is incorrect datatype"),
    ("chain-C-dtype", lambda e: chain(e, y=torch.zeros(2, 128, dtype=torch.bfloat16)), RuntimeError, "C is incorrect datatype"),
    ("chain-B-rank", lambda e: chain(e, trellis=_trellis()[0]), RuntimeError, "B: incorrect number of dimensions"),
    ("chain-k-mismatch", lambda e: chain(e, x=_h(2, 384)), RuntimeError, "A and B incompatible shapes"),
    ("chain-n-mismatch", lambda e: chain(e, y=_h(2, 256)), RuntimeError, "C and B incompatible shapes"),
    ("chain-C-rows", lambda e: chain(e, y=_h(3, 128)), RuntimeError, "C and B incompatible shapes"),
    ("chain-gate-up", lambda e: chain(e, gate=torch.zeros(2, 256), up=_h(2, 256)), RuntimeError,
     "gate / up must be fp32 or fp16 tensors of one shape"),
    ("chain-mcg-mul1", lambda e: chain(e, mcg=True), RuntimeError, "Specified both mcg and mul1"),
    ("chain-x-strided", lambda e: chain(e, x=_t(_h(2, 256))), RuntimeError, "GemmChain"),
    ("chain-up-strided", lambda e: chain(e, gate=torch.zeros(2, 256), up=_t(torch.zeros(2, 256))), RuntimeError, "GemmChain"),
    # exl3_mgemm (2 rows, mul1: the calls the shim hands to exl3b_mgemm as they are)
    ("mgemm-A-dtype", lambda e: mgemm(e, A=torch.zeros(1, 2, 256)), RuntimeError, "A is incorrect datatype"),
    ("mgemm-B-dtype", lambda e: mgemm(e, B=torch.tensor([16, 32], dtype=torch.int)), RuntimeError, "B is incorrect datatype"),
    ("mgemm-C-dtype", lambda e: mgemm(e, C=torch.zeros(2, 2, 128, dtype=torch.bfloat16)), RuntimeError, "C is incorrect datatype"),
    ("mgemm-A-rank", lambda e: mgemm(e, A=_h(2, 256)), RuntimeError, "exl3_mgemm: incorrect number of dimensions"),
    ("mgemm-AC-rows", lambda e: mgemm(e, C=_h(2, 3, 128)), RuntimeError, "A and C incompatible shapes"),
    ("mgemm-tables", lambda e: mgemm(e, suh=torch.tensor([16], dtype=torch.long)), RuntimeError,
     "B, suh and svh tables must have the same length"),
    ("mgemm-k-128", lambda e: mgemm(e, A=_h(1, 2, 144)), RuntimeError, "exl3_mgemm: k (144) must be divisible by 128"),
    ("mgemm-n-128", lambda e: mgemm(e, C=_h(2, 2, 144)), RuntimeError, "exl3_mgemm: n (144) must be divisible by 128"),
    ("mgemm-K-9", lambda e: mgemm(e, K=9), RuntimeError, "K must be 1..8"),
    ("mgemm-mcg-mul1", lambda e: mgemm(e, mcg=True, mul1=True), RuntimeError, "Specified both mcg and mul1"),
    ("mgemm-indices-rank", lambda e: mgemm(e, idx=torch.zeros(2, dtype=torch.long)), RuntimeError,
     "indices: incorrect number of dimensions"),
    # the other operators on strided memory
    ("reconstruct-strided", lambda e: e.reconstruct_slice(_t(_h(256, 128)), _trellis(), 4, False, True, 0), RuntimeError,
     "reconstruct"),
    ("reconstruct-had-strided", lambda e: e.reconstruct_had_slice(_t(_h(256, 128)), _trellis(), _h(256), _h(128), 4, False, True, 0),
     RuntimeError, "reconstruct_had"),
    ("had-strided", lambda e: e.had_r_128(_t(_h(2, 128)), _h(2, 128), None, None, 1.0), RuntimeError, "had_r_128"),
    ("hgemm-strided", lambda e: e.hgemm(_t(_h(2, 128)), _h(128, 128), _h(2, 128)), RuntimeError, "hgemm"),
]


@pytest.mark.parametrize("call,exc,msg", [c[1:] for c in CATALOG], ids=[c[0] for c in CATALOG])
def test_invalid_gemm_calls_are_refused(host_shim, call, exc, msg):
    with pytest.raises(exc) as info:
        call(host_shim)
    assert type(info.value) is exc
    assert msg in str(info.value)


@pytest.fixture(scope="module")
def abi():
    """A private handle on the library (own ctypes prototypes), and its last error message."""
    from exllamav3_b200 import ext
    L = ctypes.CDLL(ext.lib_path)
    vp, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.exl3b_gemm.argtypes = [vp] * 7 + [i] * 8
    L.exl3b_gemm_gated.argtypes = [vp] * 7 + [i] * 8 + [f, i]
    L.exl3b_gemm_allreduce.argtypes = [vp] * 7 + [i] * 6
    L.exl3b_gemm_plan.argtypes = [i] * 7 + [vp]
    L.exl3b_last_error.restype = ctypes.c_char_p
    return L, (lambda: L.exl3b_last_error().decode())


P = ctypes.c_void_p(4096)                 # never dereferenced: every call below is refused before any device access


def _gemm(L, m=2, k=256, n=128, K=4, cb=2, A=P, B=P, C=P, fsi=-1):
    return L.exl3b_gemm(None, A, B, C, None, None, None, m, k, n, K, cb, 0, fsi, 0)


def _gated(L, m=2, k=256, n=128, K=4, cb=2, G=P, U=P, B=P, C=P, act=0):
    return L.exl3b_gemm_gated(None, G, U, B, C, None, None, m, k, n, K, cb, 0, 0, act, 0.0, 0)


def _allreduce(L, m=2, k=256, n=128, K=4, cb=2, A=P, B=P, C=P):
    return L.exl3b_gemm_allreduce(None, A, B, C, None, None, None, m, k, n, K, cb, 0)


def _plan(L, m=2, k=256, n=128, K=4, cb=2, sms=132, out=True):
    buf = ctypes.create_string_buffer(64)
    return L.exl3b_gemm_plan(m, k, n, K, cb, sms, 0, buf if out else None)


# (id, entry, arguments, status, message substring)
ABI_CASES = [
    ("gemm-K", _gemm, dict(K=9), ERR_ARG, "K must be 1..8"),
    ("gemm-cb", _gemm, dict(cb=3), ERR_ARG, "cb must be 0 (3inst), 1 (mcg) or 2 (mul1)"),
    ("gemm-fsi", _gemm, dict(fsi=3), ERR_ARG, "exl3_gemm: force_shape_idx 3 out of range"),
    ("gemm-neg", _gemm, dict(m=-1), ERR_SHAPE, "exl3_gemm: negative size"),
    ("gemm-neg-k", _gemm, dict(k=-128), ERR_SHAPE, "exl3_gemm: negative size"),
    ("gemm-k", _gemm, dict(k=200), ERR_SHAPE, "exl3_gemm: k (200) must be divisible by 128"),
    ("gemm-n", _gemm, dict(n=200), ERR_SHAPE, "exl3_gemm: n (200) must be divisible by 128"),
    ("gemm-null-A", _gemm, dict(A=None), ERR_ARG, "exl3_gemm: null tensor"),
    ("gemm-null-C", _gemm, dict(C=None), ERR_ARG, "exl3_gemm: null tensor"),
    ("gemm-empty-m", _gemm, dict(m=0, A=None, B=None, C=None), TAG_NOP, None),
    ("gemm-empty-n", _gemm, dict(n=0, A=None, B=None, C=None), TAG_NOP, None),
    ("gated-K", _gated, dict(K=0), ERR_ARG, "K must be 1..8"),
    ("gated-act", _gated, dict(act=3), ERR_ARG, "exl3_gemm_gated: act must be 0 (SiLU), 1 (GELU) or 2 (ReLU^2)"),
    ("gated-neg", _gated, dict(n=-128), ERR_SHAPE, "exl3_gemm_gated: negative size"),
    ("gated-k", _gated, dict(k=200), ERR_SHAPE, "exl3_gemm_gated: k (200) must be divisible by 128"),
    ("gated-n", _gated, dict(n=200), ERR_SHAPE, "exl3_gemm_gated: n (200) must be divisible by 128"),
    ("gated-rows", _gated, dict(m=9), ERR_UNSUP, "exl3_gemm_gated: gated input is implemented for 1..8 rows, got 9"),
    ("gated-null-U", _gated, dict(U=None), ERR_ARG, "exl3_gemm_gated: null tensor"),
    ("gated-null-B", _gated, dict(B=None), ERR_ARG, "exl3_gemm_gated: null tensor"),
    ("gated-empty", _gated, dict(m=0, G=None, U=None, B=None, C=None), TAG_NOP, None),
    ("allreduce-K", _allreduce, dict(K=9), ERR_ARG, "K must be 1..8"),
    ("allreduce-rows", _allreduce, dict(m=0), ERR_SHAPE, "exl3_gemm_allreduce: bad size"),
    ("allreduce-neg", _allreduce, dict(n=-128), ERR_SHAPE, "exl3_gemm_allreduce: bad size"),
    ("allreduce-k", _allreduce, dict(k=200), ERR_SHAPE, "exl3_gemm_allreduce: k (200) must be divisible by 128"),
    ("allreduce-n", _allreduce, dict(n=200), ERR_SHAPE, "exl3_gemm_allreduce: n (200) must be divisible by 128"),
    ("allreduce-null-A", _allreduce, dict(A=None), ERR_ARG, "exl3_gemm_allreduce: null tensor"),
    ("allreduce-null-B", _allreduce, dict(B=None), ERR_ARG, "exl3_gemm_allreduce: null tensor"),
    ("plan-K", _plan, dict(K=9), ERR_ARG, "K must be 1..8"),
    ("plan-cb", _plan, dict(cb=-1), ERR_ARG, "cb must be"),
    ("plan-null", _plan, dict(out=False), ERR_ARG, "exl3_gemm_plan: null output"),
    ("plan-rows", _plan, dict(m=0), ERR_SHAPE, "exl3_gemm_plan: empty problem"),
    ("plan-small-k", _plan, dict(k=0), ERR_SHAPE, "exl3_gemm_plan: empty problem"),
    ("plan-k", _plan, dict(k=200), ERR_SHAPE, "exl3_gemm: k (200) must be divisible by 128"),
    ("plan-n", _plan, dict(n=200), ERR_SHAPE, "exl3_gemm: n (200) must be divisible by 128"),
    ("plan-sms", _plan, dict(sms=0), ERR_ARG, "exl3_gemm_plan: num_sms must be positive"),
]


@pytest.mark.parametrize("entry,kw,status,msg", [c[1:] for c in ABI_CASES], ids=[c[0] for c in ABI_CASES])
def test_c_abi_gemm_argument_checks(abi, entry, kw, status, msg):
    L, err = abi
    assert entry(L, **kw) == status, err()
    if msg is not None:
        assert msg in err()


def test_c_abi_check_order(abi):
    """Where a call breaks several rules, the entry's first check decides."""
    L, err = abi
    assert _gemm(L, K=9, fsi=3) == ERR_ARG and "K must be" in err()
    assert _gemm(L, fsi=3, m=-1) == ERR_ARG and "force_shape_idx" in err()
    assert _gemm(L, m=0, k=200) == ERR_SHAPE                   # divisibility before the empty-problem exit
    assert _gated(L, act=3, k=200) == ERR_ARG and "act must be" in err()
    assert _gated(L, m=9, G=None) == ERR_UNSUP                 # row limit before the null check
    assert _allreduce(L, m=0, k=200) == ERR_SHAPE and "bad size" in err()
    assert _plan(L, K=9, out=False) == ERR_ARG and "K must be" in err()
    assert _plan(L, out=False, m=0) == ERR_ARG and "null output" in err()
    assert _plan(L, m=0, k=200) == ERR_SHAPE and "empty problem" in err()
