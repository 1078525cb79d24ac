"""
The MLP blocks on the H100: the gated activation operators (silu_mul / gelu_mul / relu2_mul), the down projection with the
activation in its input stage (exl3_gemm_gated) and the blocks built on them (BC_GatedMLP.run_bszN, BC_MLP.run_bsz1).

Bars: the operators are within 1 fp16 ulp of fp16(fp64 model) and exact where the model is (g = 0, relu2 at g <= 0);
exl3_gemm_gated and the blocks are bit-identical to the reference's launch sequence composed from this library's operators
(act_mul into a buffer, then exl3_gemm), on the same path; the gated block also meets the fp64-oracle bars of
tests/test_gpu_parity.py.  Every exl3_gemm_gated output is written between sentinel rows that must keep their bits; on tags 100 and
200 it is also held to the exact model of the fp16 path on the activation's output (test_edges_host.check_f16_gemm).
"""
import contextlib
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc
from test_edges_host import check_f16_gemm

pytestmark = pytest.mark.gpu

TAG_TC, TAG_I8 = 200, 210
ACTS = (0, 1, 2)
ACT_OPS = ("silu_mul", "gelu_mul", "relu2_mul")
SENTINEL = {torch.half: (torch.int16, 0x7E5A), torch.float: (torch.int32, 0x7FA5A5A5)}
LLAMA_HIDDEN, LLAMA_INTER = 4096, 14336


def _ext():
    from exllamav3_b200 import ext
    return ext


@contextlib.contextmanager
def gemm_path(tag):
    ext = _ext()
    prev = ext.set_gemm_path(tag)
    try:
        yield
    finally:
        ext.set_gemm_path(prev)


def act_model(g, u, act, limit):
    """fp16(act(g) * u) in fp64, with the limit rule"""
    g = g.astype(np.float64); u = u.astype(np.float64)
    if act == 0:
        a = g / (1.0 + np.exp(-g))
    elif act == 1:
        a = 0.5 * g * (1.0 + np.tanh(0.797884560803 * (g + 0.044715 * g ** 3)))
    else:
        a = np.maximum(g, 0.0) ** 2
    if limit != 0.0:
        u = np.clip(u, -limit, limit)
        a = np.minimum(a, limit)
    return (a * u).astype(np.float16)


def ulp_distance(a, b):
    """distance in representable fp16 steps (sign-aware)"""
    def ordered(x):
        i = x.view(np.int16).astype(np.int32)
        return np.where(i < 0, -(i & 0x7FFF), i)
    return np.abs(ordered(a) - ordered(b))


def rand_gu(shape, dt, dev, seed, scale=3.0):
    gen = torch.Generator(device=dev).manual_seed(seed)
    g = torch.randn(shape, generator=gen, device=dev) * scale
    u = torch.randn(shape, generator=gen, device=dev)
    g.view(-1)[::17] = 0.0                                     # exact zeros of the gate
    return g.to(dt).contiguous(), u.to(dt).contiguous()


# ---- standalone operators ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("dt", (torch.half, torch.float))
@pytest.mark.parametrize("limit", (0.0, 2.5))
@pytest.mark.parametrize("inplace", (None, "x", "y"))
def test_act_mul_operators_match_the_fp64_model(cuda, act, dt, limit, inplace):
    ext = _ext()
    op = getattr(ext, ACT_OPS[act])
    for size in (2, 3, 7, 128, 1001, LLAMA_INTER * 8):
        g, u = rand_gu((size,), dt, cuda, seed=size + 10 * act)
        ref = act_model(g.float().cpu().numpy(), u.float().cpu().numpy(), act, limit)
        if inplace is None:
            z = torch.empty(size, dtype=torch.half, device=cuda)
            op(g, u, z, limit)
        elif dt != torch.half:
            continue                                            # z is fp16: only fp16 inputs can alias it
        else:
            z = g if inplace == "x" else u
            op(g, u, z, limit)
        got = z.cpu().numpy()
        assert np.isfinite(got).all()
        d = ulp_distance(got, ref)
        assert d.max() <= 1, (size, int(d.max()))
        gh = (g.float().cpu().numpy() if inplace != "x" else None)
        if gh is not None:
            exact = gh == 0.0
            if act == 2:
                exact |= gh <= 0.0
            assert (got[exact] == ref[exact]).all()


def test_act_mul_in_a_cuda_graph(cuda):
    ext = _ext()
    g, u = rand_gu((4096,), torch.half, cuda, seed=3)
    z = torch.empty_like(g)
    ext.silu_mul(g, u, z, 0.0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ext.silu_mul(g, u, z, 0.0)
    g2, u2 = rand_gu((4096,), torch.half, cuda, seed=4)
    g.copy_(g2); u.copy_(u2)
    graph.replay()
    ref = torch.empty_like(z)
    ext.silu_mul(g2, u2, ref, 0.0)
    torch.cuda.synchronize()
    assert torch.equal(z.view(torch.int16), ref.view(torch.int16))


# ---- exl3_gemm_gated ------------------------------------------------------------------------------------------------------

class Mat:
    def __init__(self, dev, k, n, K, cb, seed):
        gen = torch.Generator(device=dev).manual_seed(seed)
        self.k, self.n, self.K, self.cb = k, n, K, cb
        self.tr = torch.randint(-32768, 32768, (k // 16, n // 16, 16 * K), generator=gen, device=dev, dtype=torch.int32).to(torch.int16)
        sg = torch.where(torch.rand(k, generator=gen, device=dev) < 0.5, -1.0, 1.0)
        self.suh = (sg * (0.5 + 1.5 * torch.rand(k, generator=gen, device=dev)) / k ** 0.5).half()
        sg = torch.where(torch.rand(n, generator=gen, device=dev) < 0.5, -1.0, 1.0)
        self.svh = (sg * (0.5 + 1.5 * torch.rand(n, generator=gen, device=dev))).half()

    @property
    def mcg(self):
        return self.cb == 1

    @property
    def mul1(self):
        return self.cb == 2


def framed(m, n, dt, dev):
    """C between two sentinel rows"""
    it, bits = SENTINEL[dt]
    full = torch.full((m + 2, n), bits, dtype=it, device=dev).view(dt)
    return full, full[1:m + 1]


def assert_frame(full, dt):
    it, bits = SENTINEL[dt]
    raw = full.view(it)
    assert (raw[0] == bits).all() and (raw[-1] == bits).all(), "rows around C were written"


def gated_vs_composed(dev, mt, m, act, limit, gu_dt, c_dt, force=0, seed=0):
    ext = _ext()
    GU = torch.stack(rand_gu((m, mt.k), gu_dt, dev, seed=seed, scale=2.0))          # (2, m, k), as an mgemm output
    G, U = GU[0], GU[1]
    a = torch.empty((m, mt.k), dtype=torch.half, device=dev)
    getattr(ext, ACT_OPS[act])(G, U, a, limit)
    full1, C1 = framed(m, mt.n, c_dt, dev)
    ah = torch.empty_like(a)
    tag1 = ext.exl3_gemm(a, mt.tr, C1, mt.suh, ah, mt.svh, -1, mt.mcg, mt.mul1, force)
    full2, C2 = framed(m, mt.n, c_dt, dev)
    tag2 = ext.exl3_gemm_gated(G, U, mt.tr, C2, mt.suh, mt.svh, act, limit, mt.mcg, mt.mul1, force)
    torch.cuda.synchronize()
    assert tag2 == tag1, (tag1, tag2)
    assert_frame(full2, c_dt)
    it = SENTINEL[c_dt][0]
    assert torch.equal(C1.view(it), C2.view(it)), ("not bit-identical", m, mt.k, mt.n, mt.K, mt.cb, act, limit, gu_dt, c_dt, force)
    assert torch.isfinite(C2).all()
    if tag2 in (100, 200):
        np_ = lambda t: t.cpu().numpy()
        check_f16_gemm(np_(C2), np_(a), np_(mt.tr), np_(mt.suh), np_(mt.svh), mt.K, mt.cb, c_dt == torch.float,
                       ("gated", m, mt.k, mt.n, mt.K, mt.cb, act, limit, force))
    return tag2


def test_gemm_gated_every_K_and_row_count_at_mul1(cuda):
    tags = set()
    for K in range(1, 9):
        mt = Mat(cuda, 512, 256, K, 2, seed=K)
        for m in range(1, 9):
            tags.add(gated_vs_composed(cuda, mt, m, act=(K + m) % 3, limit=0.0, gu_dt=torch.half, c_dt=torch.half, seed=m))
    assert tags == {TAG_I8, TAG_TC}


@pytest.mark.parametrize("cb", (0, 1))
def test_gemm_gated_mcg_and_3inst(cuda, cb):
    for K in (2, 4):
        mt = Mat(cuda, 384, 256, K, cb, seed=20 + K)
        for m in (1, 3, 8):
            assert gated_vs_composed(cuda, mt, m, act=m % 3, limit=0.0, gu_dt=torch.half, c_dt=torch.half) == TAG_TC


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("limit", (0.0, 1.5))
@pytest.mark.parametrize("gu_dt", (torch.half, torch.float))
@pytest.mark.parametrize("c_dt", (torch.half, torch.float))
def test_gemm_gated_activations_dtypes_limits(cuda, act, limit, gu_dt, c_dt):
    mt = Mat(cuda, 1024, 384, 4, 2, seed=31)
    for m in (1, 4, 5, 8):
        gated_vs_composed(cuda, mt, m, act, limit, gu_dt, c_dt, seed=m)


def test_gemm_gated_forced_grids_and_paths(cuda):
    mt = Mat(cuda, 1152, 1152, 3, 2, seed=41)
    for force in (2, 7, 10):
        for m in (1, 4, 8):
            gated_vs_composed(cuda, mt, m, act=0, limit=0.0, gu_dt=torch.half, c_dt=torch.float, force=force)
    with gemm_path(TAG_TC):
        for m in (1, 3):
            assert gated_vs_composed(cuda, mt, m, act=1, limit=0.0, gu_dt=torch.half, c_dt=torch.half, force=7) == TAG_TC
    with gemm_path(TAG_I8):
        assert gated_vs_composed(cuda, mt, 2, act=2, limit=0.0, gu_dt=torch.float, c_dt=torch.half, force=10) == TAG_I8


def test_gemm_gated_both_sides_of_the_activation_cache(cuda):
    for m, k, cached in ((4, 8192, True), (4, 8320, False), (2, 16384, True), (3, 11008, False)):
        assert (m * k * 2 <= 64 * 1024) == cached
        mt = Mat(cuda, k, 256, 4, 2, seed=k)
        for gu_dt in (torch.half, torch.float):
            assert gated_vs_composed(cuda, mt, m, act=0, limit=0.0, gu_dt=gu_dt, c_dt=torch.half) == TAG_I8


def test_gemm_gated_llama_down_full_size(cuda):
    mt = Mat(cuda, LLAMA_INTER, LLAMA_HIDDEN, 4, 2, seed=77)
    for m in (1, 2, 3, 4, 8):
        gated_vs_composed(cuda, mt, m, act=0, limit=0.0, gu_dt=torch.half, c_dt=torch.half, seed=m)
    gated_vs_composed(cuda, mt, 4, act=0, limit=0.0, gu_dt=torch.float, c_dt=torch.float)


def test_gemm_gated_cuda_graph_replay(cuda):
    ext = _ext()
    mt = Mat(cuda, 2048, 512, 4, 2, seed=5)
    for m in (2, 6):
        G, U = rand_gu((m, mt.k), torch.half, cuda, seed=1)
        C = torch.empty((m, mt.n), dtype=torch.half, device=cuda)
        ext.exl3_gemm_gated(G, U, mt.tr, C, mt.suh, mt.svh, 0, 0.0, False, True)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ext.exl3_gemm_gated(G, U, mt.tr, C, mt.suh, mt.svh, 0, 0.0, False, True)
        G2, U2 = rand_gu((m, mt.k), torch.half, cuda, seed=2)
        G.copy_(G2); U.copy_(U2)
        graph.replay()
        a = torch.empty_like(G2)
        ext.silu_mul(G2, U2, a, 0.0)
        ref = torch.empty_like(C)
        ext.exl3_gemm(a, mt.tr, ref, mt.suh, torch.empty_like(a), mt.svh, -1, False, True, 0)
        torch.cuda.synchronize()
        assert torch.equal(C.view(torch.int16), ref.view(torch.int16))


# ---- blocks ---------------------------------------------------------------------------------------------------------------

HID, INTER = 512, 1024


def linear(ext, dev, k, n, K, seed, bias):
    mt = Mat(dev, k, n, K, 2, seed)
    b = (torch.randn(n, generator=torch.Generator(device=dev).manual_seed(seed), device=dev) * 0.1).half() if bias else None
    bc = ext.BC_LinearEXL3(mt.tr, mt.suh, mt.svh, K, b, False, True, torch.empty((1, k), dtype=torch.half, device=dev))
    return mt, bc


def f64_linear(x, mt, bias):
    y = orc.exl3_gemm_f64(x.astype(np.float16), mt.tr.cpu().numpy(), mt.suh.cpu().numpy(), mt.svh.cpu().numpy(), mt.K, 2)
    return y + (bias.double().cpu().numpy() if bias is not None else 0.0)


class GatedBlock:
    def __init__(self, ext, dev, fused, bias, interm_dt, act=0, limit=0.0):
        self.gate_mt, self.gate = linear(ext, dev, HID, INTER, 4, 101, bias and not fused)
        self.up_mt, self.up = linear(ext, dev, HID, INTER, 4, 102, bias and not fused)
        self.down_mt, self.down = linear(ext, dev, INTER, HID, 3, 103, bias)
        self.fused, self.act, self.limit = fused, act, limit
        if fused:
            mk = lambda a: torch.tensor([getattr(self.gate_mt, a).data_ptr(), getattr(self.up_mt, a).data_ptr()], dtype=torch.long, device=dev)
            self.tabs = (mk("tr"), mk("suh"), mk("svh"))
        else:
            self.tabs = (None, None, None)
        self.guh = torch.empty((2, 8, HID), dtype=interm_dt, device=dev)
        self.gu = torch.empty((2, 8, INTER), dtype=interm_dt, device=dev)
        self.a = torch.full((1, 8, INTER), 7.0, dtype=torch.half, device=dev)
        self.down_xh = torch.full((1, 8, INTER), 7.0, dtype=torch.half, device=dev)
        self.bc = ext.BC_GatedMLP(self.guh, self.gu, self.a, self.down_xh, *self.tabs, 4, False, fused,
                                  act == 0, act == 1, act == 2, None if fused else self.gate, None if fused else self.up,
                                  self.down, limit)

    def composed(self, ext, x, d):
        """the reference's launch sequence (libtorch/mlp.cpp:14-91) on this library's operators"""
        n = x.numel() // x.shape[-1]
        gu = torch.empty((2, n, INTER), dtype=self.gu.dtype, device=x.device)
        guh = torch.empty((2, n, HID), dtype=self.gu.dtype, device=x.device)
        x3 = x.view(1, n, HID)
        if self.fused:
            ext.exl3_mgemm(x3, self.tabs[0], gu, self.tabs[1], guh, self.tabs[2], None, None, 4, -1, False, True, -1, -1, 0)
        else:
            for j, lin in enumerate((self.gate, self.up)):
                ext.exl3_gemm(x3, lin.trellis, gu[j], lin.suh, guh[j], lin.svh, -1, False, True, 0)
                if lin.bias is not None:
                    gu[j] += lin.bias
        a = torch.empty((1, n, INTER), dtype=torch.half, device=x.device)
        getattr(ext, ACT_OPS[self.act])(gu[0].unsqueeze(0), gu[1].unsqueeze(0), a, self.limit)
        ext.exl3_gemm(a, self.down.trellis, d, self.down.suh, torch.empty_like(a), self.down.svh, -1, False, True, 0)
        if self.down.bias is not None:
            d += self.down.bias

    def f64(self, x):
        g = f64_linear(x, self.gate_mt, self.gate.bias)
        u = f64_linear(x, self.up_mt, self.up.bias)
        a = g / (1.0 + np.exp(-g))
        return f64_linear(a * u, self.down_mt, self.down.bias)


@pytest.mark.parametrize("fused", (True, False))
@pytest.mark.parametrize("bias", (False, True))
def test_gated_mlp_run_bszN_matches_the_reference_sequence(cuda, fused, bias):
    ext = _ext()
    blk = GatedBlock(ext, cuda, fused, bias, torch.half)
    for n in range(1, 9):
        x = (torch.randn((1, n, HID), generator=torch.Generator(device=cuda).manual_seed(n), device=cuda)).half()
        d = torch.empty((1, n, HID), dtype=torch.half, device=cuda)
        ref = torch.empty_like(d)
        blk.composed(ext, x, ref)
        l0 = ext.launch_count()
        blk.bc.run_bszN(x, d)
        launches = ext.launch_count() - l0
        torch.cuda.synchronize()
        assert torch.equal(d.view(torch.int16), ref.view(torch.int16)), (n, fused, bias)
        if fused and not bias and n <= 4:
            assert launches == 2, launches
        y = blk.f64(x.view(n, HID).cpu().numpy().astype(np.float64))
        err = np.abs(d.view(n, HID).double().cpu().numpy() - y)
        mx, rms = err.max() / np.abs(y).max(), np.sqrt((err ** 2).mean() / (y ** 2).mean())
        assert mx <= 2e-3 + 2.0 ** -10 and rms <= 1e-3, (n, mx, rms)
    assert (blk.a == 7.0).all() and (blk.down_xh == 7.0).all()


@pytest.mark.parametrize("act", ACTS)
def test_gated_mlp_activations_fp32_intermediate_and_limit(cuda, act):
    ext = _ext()
    blk = GatedBlock(ext, cuda, True, False, torch.float, act=act, limit=4.0)
    for n in (1, 4, 8):
        x = torch.randn((1, n, HID), generator=torch.Generator(device=cuda).manual_seed(n), device=cuda).half()
        d = torch.empty((1, n, HID), dtype=torch.half, device=cuda)
        ref = torch.empty_like(d)
        blk.composed(ext, x, ref)
        blk.bc.run_bszN(x, d)
        torch.cuda.synchronize()
        assert torch.equal(d.view(torch.int16), ref.view(torch.int16)), (n, act)


def test_gated_mlp_under_graph_capture(cuda):
    ext = _ext()
    blk = GatedBlock(ext, cuda, True, False, torch.half)
    for n in (1, 4, 7):
        x = torch.randn((1, n, HID), generator=torch.Generator(device=cuda).manual_seed(n), device=cuda).half()
        d = torch.empty((1, n, HID), dtype=torch.half, device=cuda)
        blk.bc.run_bszN(x, d)                                   # eager first: buffers and pointer tables are set up outside capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            blk.bc.run_bszN(x, d)
        x2 = torch.randn((1, n, HID), generator=torch.Generator(device=cuda).manual_seed(100 + n), device=cuda).half()
        x.copy_(x2)
        graph.replay()
        ref = torch.empty_like(d)
        blk.composed(ext, x2, ref)
        torch.cuda.synchronize()
        assert torch.equal(d.view(torch.int16), ref.view(torch.int16)), n


@pytest.mark.parametrize("padded", (False, True))
@pytest.mark.parametrize("act", ACTS)
def test_mlp_run_bsz1_matches_the_reference_sequence(cuda, padded, act):
    ext = _ext()
    hidden = 448 if padded else 512                              # not a multiple of 128: zero-padded staging
    up_mt, up = linear(ext, cuda, 512, INTER, 4, 201, True)
    dn_mt, dn = linear(ext, cuda, INTER, 512, 4, 202, True)
    u = torch.empty((1, 1, INTER), dtype=torch.half, device=cuda)
    ones = torch.ones((1, 1, INTER), dtype=torch.half, device=cuda)
    xp = torch.zeros((1, 512), dtype=torch.half, device=cuda) if padded else None
    yp = torch.empty((1, 512), dtype=torch.half, device=cuda) if padded else None
    bc = ext.BC_MLP(xp=xp, u=u, ones=ones, yp=yp, act_silu=act == 0, act_gelu=act == 1, act_relu2=act == 2, up=up, down=dn,
                    act_limit=0.0, hidden_size=hidden, out_size=hidden)
    x = torch.randn((1, 1, hidden), generator=torch.Generator(device=cuda).manual_seed(act), device=cuda).half()
    d = torch.empty((1, 1, hidden), dtype=torch.half, device=cuda)
    bc.run_bsz1(x, d)
    # the reference's sequence (libtorch/mlp.cpp:93-128): staging copy, up, in-place act_mul(u, ones, u), down, copy out
    xr = torch.zeros((1, 512), dtype=torch.half, device=cuda)
    xr[:, :hidden] = x.view(1, hidden)
    ur = torch.empty((1, INTER), dtype=torch.half, device=cuda)
    up.run(xr, ur)
    getattr(ext, ACT_OPS[act])(ur, ones.view(1, INTER), ur, 0.0)
    yr = torch.empty((1, 512), dtype=torch.half, device=cuda)
    dn.run(ur, yr)
    torch.cuda.synchronize()
    assert torch.equal(d.view(1, hidden).view(torch.int16), yr[:, :hidden].view(torch.int16)), (padded, act)
