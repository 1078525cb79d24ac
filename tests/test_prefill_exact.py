"""
The prefill sibling (QLinear.forward_dense: had_r_128 -> reconstruct -> hgemm -> had_r_128, or reconstruct_had_slice -> hgemm
from 1024 rows on, in weight windows of <= 32768 columns) held to exact models at the benchmark's prefill shapes (H100).

  1. hgemm, both kernels (hgemm_tc_kernel on wgmma, hgemm_simt_kernel on CUDA cores), on operands whose product is exact in any
     fp32 summation order (small integers times a power of two per row of A and column of B, sum |a b| < 2^23 quanta): fp32 C
     bit for bit equal to the fp64 product, fp16 C equal to its round-to-nearest.  At the geometry edges, the four ways to the
     CUDA-core kernel, both bench.py prefill_tensor shapes and the Llama-3.1-8B / -70B down projections in every element, a
     strided C inside a NaN-filled wider buffer, and one CUDA-graph replay.  torch.profiler names the kernel each case ran.
  2. reconstruct / reconstruct_slice (bit for bit against oracle.exl3_oracle_torch.decode_weights), had_r_128 (bit for bit) and
     reconstruct_had_slice on both kernels (the fp32-sum model's element bar and shares of bit-identical elements over the whole
     output and in every 128 x 128 block) at q, gate, down and lm_head's four windows, on bench.Token's own tensors.
  3. A replica of forward_dense keeps every intermediate; each stage is held to its model fed with the kernel's own input, hgemm
     per 128 x 128 tile against an fp64 product of its operands; lin.forward must equal the replica bit for bit and meet the fp64
     oracle in every 128-column strip.  Folded: bench.py's two prefill shapes on its seeded x, down at 2049 rows, lm_head at
     1024 rows; unfolded: q at 145, down at 1023, lm_head at 145 rows.

A failure names the stage, the window and the worst tile or block.  Bars and shapes: tests/test_prefill_host.py, which also runs
the fault catalog.  On one H100 80 GB HBM3 (700 W power limit) the file takes 13 s and peaks at 4.2 GiB of device memory.
"""
import sys
import pytest
import torch
from conftest import ROOT
from oracle import exl3_oracle_torch as ot
from test_prefill_host import (EDGE_K, EDGE_M, EDGE_N, FULL_SHAPES, LLAMA, RECON_SAME, WAVE_SHAPE, exact_product, f64_oracle,
                               hg_tiles, hgemm_excess, int_operands, recon_stats, strip_excess, strip_stats, windows)

sys.path.insert(0, ROOT)
import bench

pytestmark = pytest.mark.gpu

TC, SIMT = "hgemm_tc_kernel", "hgemm_simt_kernel"
ROWS, COLS = 8192, 4096              # device-side checks in blocks of this many rows / columns (whole 128 x 128 tiles)


def same_bits(a, b):
    return torch.equal(a.view(torch.int16 if a.dtype == torch.half else torch.int32),
                       b.view(torch.int16 if b.dtype == torch.half else torch.int32))


def hgemm_kernels(calls):
    """Run each call once under torch.profiler; the hgemm kernel name of each, in launch order."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)          # the session's first kernel: its activity record can arrive late
        torch.cuda.synchronize()
        for c in calls:
            c()
        torch.cuda.synchronize()
    evs = sorted((e for e in prof.events() if "hgemm" in e.name and e.device_type.name == "CUDA"),
                 key=lambda e: e.time_range.start)
    return [TC if TC in e.name else SIMT if SIMT in e.name else e.name for e in evs]


def int_case(m, k, n, gen, dev, c_dtype, a_off=0, c_pitch=None):
    """Integer operands (A at element offset a_off into its buffer), a NaN-filled C of pitch c_pitch, the exact product."""
    from exllamav3_b200 import ext
    buf, b = int_operands(m, k, n, gen, dev, a_rows=m + 1)
    a = buf.view(-1)[a_off:a_off + m * k].view(m, k)
    cbuf = torch.full((m, c_pitch or n), float("nan"), dtype=c_dtype, device=dev)
    c = cbuf[:, :n]
    ref = exact_product(a, b)
    return (lambda: ext.hgemm(a, b, c)), c, cbuf, ref


def check_exact(c, ref, what):
    want = ref if c.dtype == torch.float32 else ref.half()
    if not same_bits(c, want):
        bad = (c.float() != want.float()) | c.isnan()
        r, col = [int(v) for v in bad.nonzero()[0]]
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ, first ({r}, {col}): {float(c[r, col])} != "
                             f"{float(want[r, col])} (tile {r // 128}, {col // 128})")


# ---- 1. hgemm on the integer fixture --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c_dtype", [torch.float32, torch.half], ids=["f32", "f16"])
def test_hgemm_integer_geometry_edges_both_kernels(cuda, c_dtype):
    g = torch.Generator(device=cuda).manual_seed(11)
    shapes = [(m, k, n) for m in EDGE_M for n in EDGE_N for k in EDGE_K] + [WAVE_SHAPE]
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    m, k, n = WAVE_SHAPE
    assert hg_tiles(m, n) > 2 * sms and hg_tiles(m, n) % sms, "every CTA takes several tiles, the last wave is partial"
    cases = []
    for shape in shapes:
        for kern, off in ((TC, 0), (SIMT, 1)):         # A one element off 16-byte alignment: the CUDA-core kernel
            cases.append((shape, kern) + int_case(*shape, g, cuda, c_dtype, a_off=off))
    ran = hgemm_kernels([cs[2] for cs in cases])
    assert ran == [cs[1] for cs in cases], "a case ran another kernel than the one it is meant to reach"
    for shape, kern, _, c, _, ref in cases:
        check_exact(c, ref, f"{kern} m, k, n = {shape}")


@pytest.mark.parametrize("c_dtype", [torch.float32, torch.half], ids=["f32", "f16"])
def test_hgemm_integer_cuda_core_fallback_four_ways(cuda, c_dtype):
    g = torch.Generator(device=cuda).manual_seed(12)
    cases = {"k % 8 != 0": int_case(257, 4101, 136, g, cuda, c_dtype),
             "n % 8 != 0": int_case(257, 4104, 133, g, cuda, c_dtype),
             "C pitch % 8 != 0": int_case(257, 4104, 136, g, cuda, c_dtype, c_pitch=141),
             "A base off alignment": int_case(257, 4104, 136, g, cuda, c_dtype, a_off=1)}
    assert hgemm_kernels([cs[0] for cs in cases.values()]) == [SIMT] * 4
    for what, (_, c, cbuf, ref) in cases.items():
        check_exact(c, ref, what)
        assert cbuf[:, c.shape[1]:].isnan().all(), f"{what}: C written beyond its n columns"


def test_hgemm_empty_leaves_c_untouched(cuda):
    from exllamav3_b200 import ext
    for m, n in ((0, 64), (64, 0)):
        a = torch.ones((m, 64), dtype=torch.half, device=cuda)
        b = torch.ones((64, n), dtype=torch.half, device=cuda)
        cbuf = torch.full((max(m, 1) * max(n, 1) + 64,), float("nan"), dtype=torch.half, device=cuda)
        ext.hgemm(a, b, cbuf[:m * n].view(m, n))
        torch.cuda.synchronize()
        assert cbuf.isnan().all()


@pytest.mark.parametrize("shape", FULL_SHAPES, ids=[f"{m}x{k}x{n}" for m, k, n in FULL_SHAPES])
def test_hgemm_integer_full_size(cuda, shape):
    m, k, n = shape
    g = torch.Generator(device=cuda).manual_seed(13)
    for c_dtype in (torch.half, torch.float32):
        run, c, _, ref = int_case(m, k, n, g, cuda, c_dtype)
        assert hgemm_kernels([run]) == [TC]
        check_exact(c, ref, f"hgemm {shape} {c_dtype}")
        del run, c, ref
        torch.cuda.empty_cache()


@pytest.mark.parametrize("c_dtype", [torch.float32, torch.half], ids=["f32", "f16"])
def test_hgemm_integer_strided_window_of_lm_head_pitch(cuda, c_dtype):
    from exllamav3_b200 import ext
    g = torch.Generator(device=cuda).manual_seed(14)
    m, k, n = 129, LLAMA["hidden"], LLAMA["vocab"]
    for c0, c1 in windows(n)[2:]:
        a, b = int_operands(m, k, c1 - c0, g, cuda)
        c = torch.empty((m, n), dtype=c_dtype, device=cuda)
        c.view(torch.int16 if c_dtype == torch.half else torch.int32).copy_(
            torch.randint(-2 ** 15, 2 ** 15, c.shape, generator=g, device=cuda) | (0x7e00 if c_dtype == torch.half else 0x7fc00000))
        before = c.clone()
        assert hgemm_kernels([lambda: ext.hgemm(a, b, c[:, c0:c1])]) == [TC]
        check_exact(c[:, c0:c1], exact_product(a, b), f"window [{c0}, {c1})")
        outside = torch.ones_like(c, dtype=torch.bool); outside[:, c0:c1] = False
        assert same_bits(c[outside], before[outside]), f"window [{c0}, {c1}): C changed outside the window"


def test_hgemm_integer_cuda_graph_replay(cuda):
    from exllamav3_b200 import ext
    g = torch.Generator(device=cuda).manual_seed(15)
    m, k, n = 257, 4104, 264
    a, b = int_operands(m, k, n, g, cuda)
    c = torch.empty((m, n), dtype=torch.float32, device=cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ext.hgemm(a, b, c)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ext.hgemm(a, b, c)
    a2, b2 = int_operands(m, k, n, g, cuda)
    a.copy_(a2); b.copy_(b2); c.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    check_exact(c, exact_product(a2, b2), "graph replay")


# ---- 2. weights and Hadamards at full size --------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def token(cuda):
    """bench.py's Llama-3.1-8B tensors: layer 0 is what bench.Token(cfg) builds (same generator, same order); lm_head follows."""
    cfg = dict(bench.MODELS["llama-3.1-8b"], layers=1)
    tok = bench.Token(cfg, 1, 0, cuda)
    mats = {mt["name"] if mt["layer"] >= 0 else "lm_head": mt for mt in tok.mats}
    yield mats
    del tok, mats
    torch.cuda.empty_cache()


def _w_cases(mt, name):
    return [(c0, c1) for c0, c1 in windows(mt["n"])] if name == "lm_head" else [(0, mt["n"])]


@pytest.mark.parametrize("name", ["q", "gate", "down", "lm_head"])
def test_reconstruct_bit_exact_full_size(cuda, token, name):
    from exllamav3_b200 import ext
    mt = token[name]
    cbs = (2, 0, 1) if name == "q" else (2,)
    for cb in cbs:
        for c0, c1 in _w_cases(mt, name):
            w = torch.full((mt["k"], c1 - c0), float("nan"), dtype=torch.half, device=cuda)
            if c1 - c0 == mt["n"]:
                ext.reconstruct(w, mt["tr"], mt["K"], cb == 1, cb == 2)
            else:
                ext.reconstruct_slice(w, mt["tr"], mt["K"], cb == 1, cb == 2, c0)
            ref = ot.decode_weights(mt["tr"][:, c0 // 16:c1 // 16], mt["K"], cb)
            bad = w.view(torch.int16) != ref.view(torch.int16)
            assert not bad.any(), f"{name} cb {cb} window [{c0}, {c1}): {int(bad.sum())} weights differ, first at " \
                                  f"{[int(v) for v in bad.nonzero()[0]]}"
            del w, ref


@pytest.mark.parametrize("case", ["f16_pre_1023x14336", "f16_post_145x128256", "f32_post_145x128256"])
def test_had_r_128_bit_exact_full_size(cuda, token, case):
    from exllamav3_b200 import ext
    g = torch.Generator(device=cuda).manual_seed(16)
    if case.startswith("f16_pre"):
        s = token["down"]["suh"]
        x = torch.randn((1023, s.numel()), generator=g, device=cuda).half()
        y = torch.empty_like(x)
        ext.had_r_128(x, y, s, None, 1.0)
        ref = ot.had_r_128(x, s, None)
    else:
        s = token["lm_head"]["svh"]
        x = (torch.randn((145, s.numel()), generator=g, device=cuda) * 8).to(torch.half if case.startswith("f16") else torch.float)
        ref = ot.had_r_128(x, None, s)
        y = x
        ext.had_r_128(y, y, None, s, 1.0)                 # in place, as forward_dense's output transform
    assert same_bits(y, ref), f"{case}: {int((y != ref).sum())} elements differ"


def recon_check(w, mt, c0, mode, what):
    """reconstruct_had output w of window [c0, c0 + n) against the fp32-sum model: element bar and bit-identical shares."""
    over, same, worst, blk = 0.0, 0.0, 1.0, None
    for s0 in range(0, w.shape[1], COLS):
        ws = w[:, s0:s0 + COLS]
        model, pre, ts = ot.reconstruct_had_model(mt["tr"], mt["suh"], mt["svh"], mt["K"], 2, n_offset=c0 + s0, n=ws.shape[1])
        o, sh, wb, b = recon_stats(ws, model, pre, ts, mt["suh"], mt["svh"][c0 + s0:c0 + s0 + ws.shape[1]])
        over, same = max(over, o), same + sh * ws.numel()
        if wb < worst:
            worst, blk = wb, (b[0], b[1] + s0 // 128)
        del model, pre, ts
    share = same / w.numel()
    whole, block = RECON_SAME[mode]
    print(f"reconstruct_had mode {mode} {what}: worst/bar {over:.3f}, identical {share:.5f}, worst block {worst:.5f} at {blk}")
    assert over <= 1, f"{what} mode {mode}: an element {over:.2f}x outside the fp32-sum model's bar"
    assert share >= whole, f"{what} mode {mode}: {share:.4f} of the elements bit-identical to the model (floor {whole})"
    assert worst >= block, f"{what} mode {mode}: block {blk} only {worst:.4f} bit-identical (floor {block})"


@pytest.mark.parametrize("name", ["q", "gate", "down", "lm_head"])
def test_reconstruct_had_both_kernels_per_block(cuda, token, name):
    from exllamav3_b200 import ext
    mt = token[name]
    try:
        for mode in (2, 1):                              # tensor cores, CUDA cores
            ext.lib.exl3b_debug_reconstruct_had(mode)
            for c0, c1 in _w_cases(mt, name):
                w = torch.full((mt["k"], c1 - c0), float("nan"), dtype=torch.half, device=cuda)
                ext.reconstruct_had_slice(w, mt["tr"], mt["suh"], mt["svh"][c0:], mt["K"], False, True, c0)
                recon_check(w, mt, c0, mode, f"{name} window [{c0}, {c1})")
                del w
    finally:
        ext.lib.exl3b_debug_reconstruct_had(0)


# ---- 3. forward_dense stage by stage ------------------------------------------------------------------------------------------

def replica(lin, x, dt):
    """QLinear.forward_dense with every intermediate kept: (y, stages)."""
    from exllamav3_b200 import ext, qlinear
    k, n = lin.in_features, lin.out_features
    rows = x.shape[0]
    folded = rows >= qlinear.FOLDED_MIN_ROWS
    y = torch.empty((rows, n), dtype=dt, device=x.device)
    st = {"folded": folded, "windows": []}
    a = x
    if not folded:
        a = torch.empty_like(x)
        ext.had_r_128(x, a, lin.suh, None, 1.0)
        st["a"] = a
    for c0, c1 in windows(n):
        w = lin._window(c0, c1, folded)
        ext.hgemm(a, w, y[:, c0:c1])
        st["windows"].append((c0, c1, w))
    st["y_gemm"] = y.clone()
    if not folded:
        ext.had_r_128(y, y, None, lin.svh, 1.0)
    if lin.bias is not None:
        y += lin.bias
    return y, st


def check_forward(cuda, mt, x, dt, bias=None):
    from exllamav3_b200 import QLinear
    lin = QLinear(mt["tr"], mt["suh"], mt["svh"], mul1=True, bias=bias)
    what = f"{mt['name'] if mt['layer'] >= 0 else 'lm_head'} rows {x.shape[0]} {dt}"
    y_rep, st = replica(lin, x, dt)
    if not st["folded"]:
        assert same_bits(st["a"], ot.had_r_128(x, lin.suh, None)), f"{what}: input had_r_128 differs from its model"
    a = x if st["folded"] else st["a"]
    worst_tile = 0.0
    for c0, c1, w in st["windows"]:
        if st["folded"]:
            recon_check(w, mt, c0, 2, f"{what} window [{c0}, {c1})")
        else:
            assert same_bits(w, ot.decode_weights(mt["tr"][:, c0 // 16:c1 // 16], mt["K"], 2)), f"{what} [{c0}, {c1}): W_hat"
        for s0 in range(0, c1 - c0, COLS):
            wd = w[:, s0:s0 + COLS].double()
            for r0 in range(0, a.shape[0], ROWS):
                ex, tile = hgemm_excess(st["y_gemm"][r0:r0 + ROWS, c0 + s0:c0 + s0 + COLS], a[r0:r0 + ROWS].double() @ wd)
                worst_tile = max(worst_tile, ex)
                assert ex <= 1, f"{what} hgemm window [{c0}, {c1}): tile {r0 // 128 + tile[0]}, {(c0 + s0) // 128 + tile[1]} " \
                                f"at {ex:.2f}x the bar"
            del wd
    if not st["folded"]:
        y_had = ot.had_r_128(st["y_gemm"], None, lin.svh)
        if bias is not None:
            y_had += bias
        assert same_bits(y_rep, y_had), f"{what}: output had_r_128 differs from its model"
    del st
    y = lin.forward(x, None, dt)
    assert same_bits(y, y_rep), f"{what}: forward differs from the stage-by-stage replica"
    del y_rep
    worst = (0.0, None)
    for s0 in range(0, mt["n"], COLS):
        W = ot.decode_weights(mt["tr"][:, s0 // 16:(s0 + COLS) // 16], mt["K"], 2)
        sv = lin.svh[s0:s0 + COLS]
        acc = None
        for r0 in range(0, x.shape[0], ROWS):
            ref = f64_oracle(x[r0:r0 + ROWS], W, lin.suh, sv)
            if bias is not None:
                ref += bias[s0:s0 + COLS].double()
            st_ = strip_stats(y[r0:r0 + ROWS, s0:s0 + COLS], ref)
            acc = st_ if acc is None else torch.stack([torch.maximum(acc[0], st_[0]), torch.maximum(acc[1], st_[1]),
                                                       acc[2] + st_[2], acc[3] + st_[3]])
            del ref
        ex, strip = strip_excess(stats=acc)
        worst = max(worst, (ex, s0 // 128 + strip), key=lambda t: t[0])
    print(f"{what}: worst hgemm tile at {worst_tile:.3f}x its bar, worst strip at {worst[0]:.3f}x the fp64-oracle bar")
    assert worst[0] <= 1, f"{what}: strip {worst[1]} at {worst[0]:.2f}x the fp64-oracle bar"


@pytest.mark.parametrize("which", ["q_m65536", "gate_m16384"])
def test_forward_dense_bench_prefill(cuda, token, which):
    # bench.py qgemm_section: generator seeded 7, x for q (32 x 2048 rows) then for gate (8 x 2048 rows)
    gen = torch.Generator(device=cuda).manual_seed(7)
    xq = torch.randn((32 * 2048, LLAMA["hidden"]), generator=gen, device=cuda).half()
    if which.startswith("q"):
        check_forward(cuda, token["q"], xq, torch.half)
    else:
        del xq
        xg = torch.randn((8 * 2048, LLAMA["hidden"]), generator=gen, device=cuda).half()
        check_forward(cuda, token["gate"], xg, torch.half)


@pytest.mark.parametrize("name,rows,dt,bias", [("down", 2049, torch.float32, True), ("lm_head", 1024, torch.float32, False),
                                               ("q", 145, torch.half, True), ("down", 1023, torch.float32, False),
                                               ("lm_head", 145, torch.float32, False)])
def test_forward_dense_stages(cuda, token, name, rows, dt, bias):
    g = torch.Generator(device=cuda).manual_seed(rows)
    mt = token[name]
    x = torch.randn((rows, mt["k"]), generator=g, device=cuda).half()
    b = torch.randn((mt["n"],), generator=g, device=cuda).half() if bias else None
    check_forward(cuda, mt, x, dt, b)
