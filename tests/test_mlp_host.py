"""
Host side of the MLP block surface (no GPU needed): the reference's modules/mlp.py must bind against the shim's BC_GatedMLP,
BC_MLP and gated activation operators exactly as it calls them (call sites recorded by oracle/gen_golden_mlp_callsites.py into
tests/golden/ref_mlp_callsites.json.gz), and the argument checks of silu_mul / gelu_mul / relu2_mul, exl3_gemm_gated and the
blocks raise RuntimeError before anything is launched -- in the shim and in the C ABI alike.
"""
import contextlib, ctypes, gzip, inspect, json, os
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_mlp_callsites.json.gz")
TAG_SIMT, TAG_TC, TAG_I8, TAG_CHAIN = 100, 200, 210, 220


@pytest.fixture(scope="module")
def gold():
    with gzip.open(GOLDEN, "rt") as f:
        return json.load(f)


def _bind(fn, positional, keywords):
    inspect.signature(fn).bind(*([None] * positional), **{k: None for k in keywords})


def test_reference_mlp_call_sites_bind_against_the_shim(gold):
    from exllamav3_b200 import ext
    assert gold["MAX_BSZN"] == ext.MAX_BSZN == 8
    names = sorted(s["name"] for s in gold["sites"])
    assert names == ["BC_GatedMLP", "BC_MLP"]
    for s in gold["sites"]:
        _bind(getattr(ext, s["name"]), s["positional"], s["keywords"])
    # GatedMLP binds ext.silu_mul / relu2_mul / gelu_mul as activation_fn_call and calls it as (g, u, a, act_limit)
    assert sorted(r["name"] for r in gold["act_refs"]) == ["gelu_mul", "relu2_mul", "silu_mul"]
    assert gold["act_calls"]
    for r in gold["act_refs"]:
        for c in gold["act_calls"]:
            _bind(getattr(ext, r["name"]), c["positional"], c["keywords"])


def test_block_constructors_take_the_reference_parameter_order():
    from exllamav3_b200 import ext
    assert list(inspect.signature(ext.BC_GatedMLP).parameters) == [
        "guh", "gu", "a", "down_xh", "gu_ptrs_trellis", "gu_ptrs_suh", "gu_ptrs_svh", "gu_K", "gu_mcg", "gu_mul1",
        "act_silu", "act_gelu", "act_relu2", "gate", "up", "down", "act_limit"]
    assert list(inspect.signature(ext.BC_MLP).parameters) == [
        "xp", "u", "ones", "yp", "act_silu", "act_gelu", "act_relu2", "up", "down", "act_limit", "hidden_size", "out_size"]
    for name in ("silu_mul", "gelu_mul", "relu2_mul"):
        assert list(inspect.signature(getattr(ext, name)).parameters) == ["x", "y", "z", "act_limit"]


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


def _gated_args(m=2, k=256, n=128, dt=torch.half, K=4):
    G = torch.zeros((m, k), dtype=dt)
    U = torch.zeros((m, k), dtype=dt)
    B = torch.zeros((k // 16, n // 16, 16 * K), dtype=torch.int16)
    C = torch.zeros((m, n), dtype=torch.half)
    return G, U, B, C


def test_act_mul_argument_checks(host_shim):
    ext = host_shim
    h, f = torch.zeros(8, dtype=torch.half), torch.zeros(8, dtype=torch.float)
    with pytest.raises(RuntimeError, match="datatype"):
        ext.silu_mul(h, f, h, 0.0)                    # fp16 x with fp32 y
    with pytest.raises(RuntimeError, match="datatype"):
        ext.gelu_mul(f, h, h, 0.0)                    # fp32 x with fp16 y
    with pytest.raises(RuntimeError, match="datatype"):
        ext.relu2_mul(h, h, f, 0.0)                   # z must be fp16
    with pytest.raises(RuntimeError, match="datatype"):
        ext.silu_mul(torch.zeros(8, dtype=torch.bfloat16), torch.zeros(8, dtype=torch.bfloat16), h, 0.0)
    with pytest.raises(RuntimeError, match="number of elements"):
        ext.silu_mul(h, torch.zeros(6, dtype=torch.half), h, 0.0)
    with pytest.raises(RuntimeError, match="contiguous"):
        ext.silu_mul(torch.zeros((4, 4), dtype=torch.half).t(), torch.zeros((4, 4), dtype=torch.half),
                     torch.zeros((4, 4), dtype=torch.half), 0.0)


def test_gemm_gated_argument_checks_in_the_shim(host_shim):
    ext = host_shim
    G, U, B, C = _gated_args()
    with pytest.raises(RuntimeError, match="datatype"):
        ext.exl3_gemm_gated(G, U.float(), B, C, None, None, ext.ACT_SILU, 0.0, False, True)
    with pytest.raises(RuntimeError, match="datatype"):
        ext.exl3_gemm_gated(G.float(), U, B, C, None, None, ext.ACT_SILU, 0.0, False, True)
    with pytest.raises(RuntimeError, match="datatype"):
        ext.exl3_gemm_gated(G, U, B, C.to(torch.bfloat16), None, None, ext.ACT_SILU, 0.0, False, True)
    with pytest.raises(RuntimeError, match="incompatible"):
        ext.exl3_gemm_gated(G, U[:1], B, C, None, None, ext.ACT_SILU, 0.0, False, True)
    with pytest.raises(RuntimeError, match="incompatible"):
        ext.exl3_gemm_gated(G[:, :128].contiguous(), U[:, :128].contiguous(), B, C, None, None, ext.ACT_SILU, 0.0, False, True)
    # rows beyond 8, a forced path without a gated input stage, and a bad activation: refused by the library
    G9, U9, B9, C9 = _gated_args(m=9)
    with pytest.raises(RuntimeError, match="1..8 rows"):
        ext.exl3_gemm_gated(G9, U9, B9, C9, None, None, ext.ACT_SILU, 0.0, False, True)
    with pytest.raises(RuntimeError, match="act must be"):
        ext.exl3_gemm_gated(G, U, B, C, None, None, 3, 0.0, False, True)
    for tag, m, mul1 in ((TAG_SIMT, 2, True), (TAG_CHAIN, 2, True), (TAG_I8, 6, True), (TAG_I8, 2, False)):
        ext.set_gemm_path(tag)
        Gm, Um, Bm, Cm = _gated_args(m=m)
        with pytest.raises(RuntimeError, match="path|forced"):
            ext.exl3_gemm_gated(Gm, Um, Bm, Cm, None, None, ext.ACT_SILU, 0.0, False, mul1)


def _abi():
    from exllamav3_b200 import ext
    return ext.lib, (lambda: ext.lib.exl3b_last_error().decode())


def test_c_abi_checks_without_a_device():
    from exllamav3_b200 import ext
    L, err = _abi()
    p = ctypes.c_void_p(4096)                         # never dereferenced: every case is refused before any device access
    ERR_SHAPE, ERR_ARG, ERR_UNSUP = -1, -2, -4

    def gated(m=2, k=256, n=128, K=4, cb=2, gu_fp32=0, act=0, G=p, U=p, force=0):
        return L.exl3b_gemm_gated(None, G, U, p, p, None, None, m, k, n, K, cb, 0, gu_fp32, act, 0.0, force)

    assert gated(m=9) == ERR_UNSUP and "1..8 rows" in err()
    assert gated(k=200) == ERR_SHAPE
    assert gated(act=5) == ERR_ARG
    assert gated(K=9) == ERR_ARG
    assert gated(G=None) == ERR_ARG
    assert gated(gu_fp32=1, G=ctypes.c_void_p(4096 + 8)) == ERR_ARG and "aligned" in err()
    assert gated(m=0) == 0                                     # empty problem: nothing to do
    try:
        for tag, m, cb in ((TAG_SIMT, 2, 2), (TAG_CHAIN, 2, 2), (TAG_I8, 5, 2), (TAG_I8, 8, 2), (TAG_I8, 2, 0)):
            ext.set_gemm_path(tag)
            assert gated(m=m, cb=cb) in (ERR_UNSUP,), (tag, m, cb, err())
    finally:
        ext.set_gemm_path(0)
    assert L.exl3b_act_mul(None, p, p, p, 16, 0, 3, 0.0) == ERR_ARG
    assert L.exl3b_act_mul(None, p, p, p, -1, 0, 0, 0.0) == ERR_SHAPE
    assert L.exl3b_act_mul(None, None, p, p, 16, 0, 0, 0.0) == ERR_ARG
    assert L.exl3b_act_mul(None, p, p, p, 0, 0, 0, 0.0) == 0


def test_blocks_refuse_bad_token_counts_and_missing_activation():
    from exllamav3_b200 import ext
    z = torch.zeros((2, 8, 128), dtype=torch.half)
    with pytest.raises(RuntimeError, match="act_silu"):
        ext.BC_GatedMLP(z, z, z, z, None, None, None, 4, False, True, False, False, False, object(), object(), object(), 0.0)
    with pytest.raises(RuntimeError, match="act_silu"):
        ext.BC_MLP(None, z, z, None, False, False, False, object(), object(), 0.0, 128, 128)
    bc = ext.BC_GatedMLP(z, z, z, z, None, None, None, 4, False, True, True, False, False, object(), object(), object(), 0.0)
    for tokens in (0, 9):
        with pytest.raises(RuntimeError, match="bsz out of supported range"):
            bc.run_bszN(torch.zeros((1, tokens, 128), dtype=torch.half), torch.zeros((1, tokens, 128), dtype=torch.half))
