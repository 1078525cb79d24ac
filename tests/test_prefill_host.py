"""
The prefill sibling's exact models and bars on the CPU: what tests/test_prefill_exact.py runs on the GPU, planned and checked here.

  * the torch restatements in oracle.exl3_oracle_torch (W_hat of every codebook, had_r_128, reconstruct_had's fp32-sum model) equal
    their numpy originals in exl3_oracle bit for bit on the CPU device;
  * the integer hgemm fixture keeps every fp32 partial sum exact (sum |a b| < 2^23 quanta) at every planned shape, and its partial
    sums outgrow fp16 (> 2^11 quanta);
  * the planned shapes reach the kernels' edges: several tiles per CTA with a partial last wave, lm_head's four weight windows;
  * the fault catalog: each fault a kernel could plausibly make, applied to the models at the GPU tests' geometry (reduced in k
    and n where the CPU is too slow), misses the bar the GPU test holds it to by at least MARGIN.
"""
import math
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc
from oracle import exl3_oracle_torch as ot

MARGIN = 3.0
SMS = 132                                    # H100 SXM
HG_TILE, HG_BK = 128, 64                     # csrc/hgemm_tc.cu: output tile, k per ring stage
WINDOW = 32768                               # QLinear.DENSE_WINDOW_COLS
QUANTA = 2 ** 23                             # fp32 significand: integer partial sums below this are exact in any order
F16_PARTIAL = 2 ** 11                        # fp16 significand: a partial sum above this kept in fp16 would round
SCALE_EXP = (-8, -4)                         # power-of-two scales per row of A / column of B: |y| < 2^23 * 2^-8 < 65504

EDGE_M = (1, 127, 128, 129, 257)
EDGE_N = (8, 56, 64, 120, 136, 264)
EDGE_K = (8, 40, 64, 72, 4104)
WAVE_SHAPE = (1032, 72, 4104)                # (m, k, n): 9 x 33 = 297 tiles = 2 waves of 132 + 33
# m, k, n of the full-size integer checks: bench.py's prefill_tensor shapes, Llama-3.1-8B's and -70B's down projections
FULL_SHAPES = ((65536, 4096, 4096), (16384, 4096, 14336), (2048, 14336, 4096), (1024, 28672, 8192))
LLAMA = dict(hidden=4096, inter=14336, vocab=128256)

# tile bars of hgemm on real operands against an fp64 product of its own operands (per 128 x 128 tile)
# The decode-GEMM's 2e-5 / 1e-5 do not hold: hgemm keeps one fp32 accumulator chain over all of k, and on an H100 its
# max-abs reached 1.7x 2e-5 of max|tile| at k = 14336 (README, Parity).
HG_F32_BAR = (1e-4, 5e-5)                    # max-abs / max|tile|, rel-RMS
HG_F16_REL = HG_F32_BAR[0]                   # fp16 C: one fp16 step of fp16(ref) + the fp32 term
F64_BAR = (2e-3, 1e-3)                       # end to end against the fp64 oracle, per 128-column strip (+1 fp16 step)
# reconstruct_had against its fp32-sum model: every element within recon_tol, and at least these shares of elements
# bit-identical over the output and in every 128 x 128 block (tests/test_prefill_exact.py prints the measured worst)
RECON_SAME = {1: (0.9999, 0.999), 2: (0.9999, 0.999)}     # debug mode (1 CUDA cores, 2 tensor cores): (whole, per block)


def int_range(k: int) -> int:
    """Largest r (<= 1024) with k r^2 < 2^23: integers in [-r, r] on both sides keep every partial sum below 2^23 quanta."""
    return min(1024, math.isqrt((QUANTA - 1) // max(k, 1)))


def int_operands(m, k, n, gen, device, a_rows=None):
    """fp16 A (m, k), B (k, n): integers in [-r, r] times 2^e per row of A / column of B, e in SCALE_EXP."""
    r = int_range(k)
    lo, hi = SCALE_EXP
    ia = torch.randint(-r, r + 1, (a_rows or m, k), generator=gen, device=device).float()
    ib = torch.randint(-r, r + 1, (k, n), generator=gen, device=device).float()
    ea = torch.randint(lo, hi + 1, (a_rows or m, 1), generator=gen, device=device).float()
    eb = torch.randint(lo, hi + 1, (1, n), generator=gen, device=device).float()
    return (ia * torch.exp2(ea)).half(), (ib * torch.exp2(eb)).half()


def exact_product(a, b, rows=8192):
    """A @ B in fp64 in row chunks, as fp32: exact for the integer fixture (every value below 2^23 quanta)."""
    out = torch.empty((a.shape[0], b.shape[1]), dtype=torch.float32, device=a.device)
    bd = b.double()
    for r0 in range(0, a.shape[0], rows):
        out[r0:r0 + rows] = (a[r0:r0 + rows].double() @ bd).float()
    return out


def hg_tiles(m, n):
    return -(-m // HG_TILE) * -(-n // HG_TILE)


def windows(n):
    return [(c, min(c + WINDOW, n)) for c in range(0, n, WINDOW)]


def f16_ulp(v: torch.Tensor) -> torch.Tensor:
    """np.spacing of fp16 values, in fp64 (2^-24 at zero and below the normal range)."""
    _, e = torch.frexp(v.float().abs())
    return torch.exp2((e - 11).clamp(min=-24).double())


def _tiles(d: torch.Tensor, t=HG_TILE):
    m, n = d.shape
    pm, pn = -m % t, -n % t
    d = torch.nn.functional.pad(d, (0, pn, 0, pm))
    return d.view((m + pm) // t, t, (n + pn) // t, t).permute(0, 2, 1, 3).reshape((m + pm) // t, (n + pn) // t, t * t)


def hgemm_excess(y: torch.Tensor, ref: torch.Tensor):
    """Worst ratio of error to bar over the 128 x 128 tiles of hgemm's C against ref (fp64), and that tile (row, col)."""
    ref = ref.double()
    yd = y.double()
    mx = _tiles(ref.abs()).amax(-1)
    if y.dtype == torch.float32:
        d = _tiles((yd - ref).abs())
        e_max = d.amax(-1) / (HG_F32_BAR[0] * mx)
        e_rms = (d ** 2).sum(-1).sqrt() / ((_tiles(ref) ** 2).sum(-1).sqrt() * HG_F32_BAR[1])
        ex = torch.maximum(e_max, e_rms)
    else:
        r16 = ref.float().half().double()              # fp16(fp64) through fp32: one rounding for every value a test passes
        tol = _tiles(f16_ulp(r16)) + HG_F16_REL * mx[..., None]
        ex = (_tiles((yd - r16).abs()) / tol).amax(-1)
    ex = torch.nan_to_num(ex, nan=float("inf"))
    i = int(ex.argmax())
    return float(ex.flatten()[i]), divmod(i, ex.shape[1])


def recon_tol(w, pre, t_step, suh, svh):
    """
    oracle.f16_model_tol for reconstruct_had: one fp16 step of the pre-scale value, plus what one flipped rounding of the fp16
    tile between the two Hadamards moves it by (t_step, from ot.reconstruct_had_model), times |suh svh|; one step of pre * suh
    times |svh|; plus one step of w.  With one step of pre and of w alone the bar fails on an H100 (measured 1.98x at 14336 x
    4096): an accumulation-order change in the first Hadamard flips a rounding of the tile, the second Hadamard carries it into
    128 outputs at the tile's step, and either fp16 multiply after it may then round the other way.
    """
    step = f16_ulp(pre) + t_step.double().repeat_interleave(128, 1)
    mid = f16_ulp(ot.hmul(pre, suh[:, None])) * svh.double().abs()[None, :]      # the suh multiply's own rounding
    return step * (suh.double().abs()[:, None] * svh.double().abs()[None, :]) + mid + f16_ulp(w)


def recon_stats(w, model, pre, t_step, suh, svh):
    """(worst |w - model| / recon_tol, share bit-identical overall, worst share per 128 x 128 block, that block)."""
    tol = recon_tol(model, pre, t_step, suh, svh)
    over = float(torch.nan_to_num((w.double() - model.double()).abs() / tol, nan=float("inf")).max())
    same = (w.view(torch.int16) == model.view(torch.int16))
    blk = _tiles(same.float()).mean(-1)
    i = int(blk.argmin())
    return over, float(same.float().mean()), float(blk.flatten()[i]), divmod(i, blk.shape[1])


def recon_excess(w, model, pre, t_step, suh, svh, mode):
    """Worst ratio of error to bar: the element bar, and the non-identical share against 1 - floor (overall and per block)."""
    over, share, worst, _ = recon_stats(w, model, pre, t_step, suh, svh)
    whole, block = RECON_SAME[mode]
    return max(over, (1 - share) / (1 - whole), (1 - worst) / (1 - block))


def f64_oracle(x, w_hat, suh, svh):
    """exl3_gemm_f64 in fp64 throughout, from x (not its fp16 transform): y = ((x suh) H) W_hat H svh, H orthonormal."""
    H = torch.from_numpy(orc.hadamard_matrix_128() / math.sqrt(128.0)).to(x.device)
    m, k = x.shape
    n = w_hat.shape[1]
    xh = ((x.double() * suh.double()).view(m, k // 128, 128) @ H).view(m, k)
    acc = xh @ w_hat.double()
    return (acc.view(m, n // 128, 128) @ H).view(m, n) * svh.double()


def strip_stats(y, ref):
    """Per 128-column strip: max |y - ref|, max |ref|, sum (y - ref)^2, sum ref^2 (add the sums and take the maxima of row chunks)."""
    y, ref = y.double(), ref.double()
    n = y.shape[1]
    d = (y - ref).abs().view(-1, n // 128, 128)
    r = ref.view(-1, n // 128, 128)
    return torch.stack([d.amax(dim=(0, 2)), r.abs().amax(dim=(0, 2)), (d ** 2).sum(dim=(0, 2)), (r ** 2).sum(dim=(0, 2))])


def strip_excess(y=None, ref=None, stats=None):
    """Worst ratio of error to the fp64-oracle bar over 128-column strips (max-abs <= 2e-3 max|ref| + 1 fp16 step, rel-RMS
    <= 1e-3), and that strip."""
    dmax, rmax, d2, r2 = strip_stats(y, ref) if stats is None else stats
    e_max = dmax / (F64_BAR[0] * rmax + f16_ulp(rmax))
    e_rms = d2.sqrt() / (r2.sqrt() * F64_BAR[1])
    ex = torch.nan_to_num(torch.maximum(e_max, e_rms), nan=float("inf"))
    return float(ex.max()), int(ex.argmax())


def small_linear(k, n, K, seed, cb=2):
    g = torch.Generator().manual_seed(seed)
    tr = torch.randint(-32768, 32768, (k // 16, n // 16, 16 * K), generator=g, dtype=torch.int32).to(torch.int16)
    sgn = lambda sz: torch.randint(0, 2, (sz,), generator=g).float() * 2 - 1
    suh = (sgn(k) * (0.5 + 1.5 * torch.rand(k, generator=g)) / k ** 0.5).half()
    svh = (sgn(n) * (0.5 + 1.5 * torch.rand(n, generator=g))).half()
    return tr, suh, svh


# ---- the restatements equal their numpy originals ------------------------------------------------------------------------------

@pytest.mark.parametrize("cb", range(3))
@pytest.mark.parametrize("K", (2, 4, 6))
def test_decode_weights_is_reconstruct(K, cb):
    tr, _, _ = small_linear(256, 384, K, 10 + K)
    ref = orc.reconstruct(tr.numpy(), K, cb)
    got = ot.decode_weights(tr, K, cb, elems=256 * 128).numpy()
    assert (got.view(np.uint16) == ref.view(np.uint16)).all()
    if cb == 2:
        assert (ot.mul1_weights(tr, K).view(np.uint16) == ref.view(np.uint16)).all()


@pytest.mark.parametrize("case", ["f16_pre", "f16_post", "f32_post", "f16_none", "f32_none"])
def test_had_r_128_restatement(case):
    rng = np.random.default_rng(5)
    dt = np.float16 if case.startswith("f16") else np.float32
    x = (rng.standard_normal((37, 512)) * rng.choice([1e-3, 1.0, 30.0], (37, 1))).astype(dt)
    s = (rng.choice([-1, 1], 512) * rng.uniform(0.5, 2.0, 512)).astype(np.float16)
    pre, post = (s, None) if case.endswith("pre") else ((None, s) if case.endswith("post") else (None, None))
    ref = orc.had_r_128(x, pre_scale=pre, post_scale=post)
    T = lambda a: None if a is None else torch.from_numpy(a)
    got = ot.had_r_128(T(x), T(pre), T(post), rows=16).numpy()
    assert got.dtype == ref.dtype and (got.view(np.uint8) == ref.view(np.uint8)).all()


@pytest.mark.parametrize("cb", range(3))
def test_reconstruct_had_model_restatement(cb):
    k, n, K = 256, 640, 3
    tr, suh, svh = small_linear(k, n, K, 20 + cb)
    ref = orc.reconstruct_had_fp32_model(tr.numpy(), suh.numpy(), svh.numpy(), K, cb)
    got, _, _ = ot.reconstruct_had_model(tr, suh, svh, K, cb, elems=k * 256)
    assert (got.numpy().view(np.uint16) == ref.view(np.uint16)).all()
    # a window at n_offset (svh indexed from the offset) is the same columns of the whole
    win, _, _ = ot.reconstruct_had_model(tr, suh, svh, K, cb, n_offset=256, n=384, elems=k * 128)
    assert (win.numpy().view(np.uint16) == ref[:, 256:].view(np.uint16)).all()


# ---- the integer fixture and the planned shapes ----------------------------------------------------------------------------------

def planned_gemm_shapes():
    shapes = [(m, k, n) for m in EDGE_M for n in EDGE_N for k in EDGE_K] + [WAVE_SHAPE] + list(FULL_SHAPES)
    shapes += [(m, LLAMA["hidden"], n) for m in (129, 1024) for n in (WINDOW, LLAMA["vocab"] - 3 * WINDOW)]
    return shapes


def test_integer_fixture_range_holds_at_every_planned_shape():
    for m, k, n in planned_gemm_shapes():
        r = int_range(k)
        assert k * r * r < QUANTA, (m, k, n)
        assert k * r * r * 2.0 ** (2 * SCALE_EXP[1]) < 65504, (m, k, n)       # |y| below fp16's largest finite value
    assert int_range(28672) >= 16                                              # 70B down: the largest k the project runs


@pytest.mark.parametrize("k", EDGE_K)
def test_integer_fixture_partial_sums_outgrow_fp16(k):
    g = torch.Generator().manual_seed(k)
    a, b = int_operands(64, k, 64, g, "cpu")
    y = exact_product(a, b).double()
    quanta = y.abs() / (2.0 ** (2 * SCALE_EXP[1]))                 # a lower bound: the largest quantum an element can have
    assert quanta.max() > F16_PARTIAL, f"k = {k}: largest |y| {quanta.max():.0f} quanta"
    assert (exact_product(a, b) == (a.float() @ b.float())).all()  # fp32 sums are exact in this order too


def test_planned_shapes_reach_the_edges():
    m, k, n = WAVE_SHAPE
    t = hg_tiles(m, n)
    assert t > 2 * SMS and t % SMS, "every CTA takes at least two tiles and the last wave is partial"
    assert m % HG_TILE and n % HG_TILE and k % HG_BK, "ragged m, n and k"
    assert {nn % HG_TILE for nn in EDGE_N} >= {8, 56, 64, 120}, "n tails of 8 .. 120 columns"
    assert min(EDGE_N) < 64 and min(EDGE_K) < HG_BK, "a TMA box wider than the tensor"
    for mm, kk, nn in FULL_SHAPES:
        assert hg_tiles(mm, nn) > SMS
    assert windows(LLAMA["vocab"]) == [(0, 32768), (32768, 65536), (65536, 98304), (98304, 128256)]
    assert windows(LLAMA["vocab"])[-1][1] - windows(LLAMA["vocab"])[-1][0] == 29952
    assert len(windows(LLAMA["inter"])) == 1


# ---- fault catalog -------------------------------------------------------------------------------------------------------------

def _real_operands(m, k, n, seed=3):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((m, k), generator=g).half(), (torch.randn((k, n), generator=g) / k ** 0.5).half()


def _gemm_fault(name, a, b):
    """C of hgemm with one fault, fp32 unless noted; the faults act on tile (0, 0) or the tail."""
    m, k = a.shape
    n = b.shape[1]
    A, B = a.double(), b.double()
    y = A @ B
    t = HG_TILE
    if name == "dropped_k16_slice":                  # stage 1's third k16 slice never reaches the MMA
        s = HG_BK + 32
        y[:t, :t] -= A[:t, s:s + 16] @ B[s:s + 16, :t]
    elif name == "swapped_k16_slices_in_a":          # A's swizzle puts slices 0 and 1 of a stage in each other's place
        a2 = A[:t].clone()
        a2[:, 0:16], a2[:, 16:32] = A[:t, 16:32], A[:t, 0:16]
        y[:t, :t] = a2 @ B[:, :t]
    elif name == "k_tail_garbage":                   # the zero-filled k tail holds other values
        kp = -k % HG_BK
        g = torch.Generator().manual_seed(9)
        y = y + torch.randn((m, kp), generator=g).double() @ torch.randn((kp, n), generator=g).double()
    elif name == "c_tile_one_over":                  # tile (0, 0) is stored at tile (0, 1)
        y[:t, t:2 * t] = y[:t, :t]
    elif name == "n_tail_last_pair_dropped":         # the tail's last column pair is never stored: C keeps its NaN fill
        y[:, n - 2:] = float("nan")
    elif name == "fp16_partial_sums":                # the accumulator is rounded to fp16 after every k16 slice
        acc = torch.zeros((m, n), dtype=torch.float64)
        for s in range(0, k, 16):
            acc = (acc + A[:, s:s + 16] @ B[s:s + 16]).float().half().double()
        y = acc
    return y.float()


GEMM_FAULTS = ["dropped_k16_slice", "swapped_k16_slices_in_a", "k_tail_garbage", "c_tile_one_over",
               "n_tail_last_pair_dropped", "fp16_partial_sums"]


@pytest.mark.parametrize("fault", GEMM_FAULTS)
def test_hgemm_faults_miss_the_tile_bar(fault):
    # geometry of the GPU's real-operand hgemm (ragged k and n), reduced in m, k and n
    a, b = _real_operands(256, 1000, 264)
    ref = a.double() @ b.double()
    ex0, _ = hgemm_excess((ref).float(), ref)
    assert ex0 < 1
    ex, tile = hgemm_excess(_gemm_fault(fault, a, b), ref)
    assert ex >= MARGIN, f"{fault}: {ex:.2f}x the bar at tile {tile}"


def test_hgemm_fp16_c_truncated_misses_the_integer_check():
    # truncation stays within one fp16 step, inside the real-operand fp16 bar: the integer fixture's bit-for-bit check sees it
    g = torch.Generator().manual_seed(1)
    a, b = int_operands(129, 4104, 136, g, "cpu")
    y = exact_product(a, b)
    rn = y.half()
    tr = torch.where((rn.float() - y).abs() > 0, torch.where(rn.float().abs() > y.abs(),
                     torch.nextafter(rn, torch.zeros_like(rn)), rn), rn)
    assert ((tr.float() - y).abs() <= (rn.float() - y).abs() + f16_ulp(rn).float()).all()
    assert (tr.view(torch.int16) != rn.view(torch.int16)).float().mean() > 0.2
    assert hgemm_excess(tr, y.double())[0] < 1, "the fp16 tile bar alone does not see a truncation"


def _recon_fault(name, tr, suh, svh, K, c0, n):
    w, pre, _ = ot.reconstruct_had_model(tr, suh, svh, K, 2, n_offset=c0, n=n)
    sv = svh[c0:c0 + n]
    if name == "fp16_tile_skipped":                  # the tile between the two Hadamards stays fp32
        H = torch.from_numpy(orc.hadamard_matrix_128())
        k = tr.shape[0] * 16
        wh = ot.decode_weights(tr[:, c0 // 16:(c0 + n) // 16], K, 2).double()
        t = ((H @ wh.view(k // 128, 128, n)).reshape(k, n).float() * float(orc.R_SCALE_F32)).double()
        p = ((t.view(k, n // 128, 128) @ H).reshape(k, n).float() * float(orc.R_SCALE_F32)).half()
        return ot.hmul(ot.hmul(p, suh[:, None]), sv[None, :])
    if name == "suh_neighbour_k_block":              # k-block 1 multiplied by k-block 2's suh
        f = ot.hmul(ot.hmul(pre[128:256], suh[256:384, None]), sv[None, :])
        w = w.clone(); w[128:256] = f
    elif name == "svh_neighbour_column_block":       # column block 1 multiplied by column block 2's svh
        f = ot.hmul(ot.hmul(pre[:, 128:256], suh[:, None]), sv[None, 256:384])
        w = w.clone(); w[:, 128:256] = f
    elif name == "stale_block":                      # block (1, 2) keeps the previous persistent iteration's block (1, 1)
        w = w.clone(); w[128:256, 256:384] = w[128:256, 128:256]
    elif name == "window_svh_not_offset":            # the window reads svh instead of svh[c0:]
        w = ot.hmul(ot.hmul(pre, suh[:, None]), svh[None, :n])
    return w


RECON_FAULTS = ["fp16_tile_skipped", "suh_neighbour_k_block", "svh_neighbour_column_block", "stale_block",
                "window_svh_not_offset"]


@pytest.mark.parametrize("fault", RECON_FAULTS)
def test_reconstruct_had_faults_miss_the_bars(fault):
    # lm_head's last window geometry (n_offset a multiple of 32768 in the real one) reduced to k = 512, 3 column blocks at 256
    k, n_all, K, c0, n = 512, 640, 6, 256, 384
    tr, suh, svh = small_linear(k, n_all, K, 31)
    model, pre, ts = ot.reconstruct_had_model(tr, suh, svh, K, 2, n_offset=c0, n=n)
    sv = svh[c0:c0 + n]
    for mode in (1, 2):
        assert recon_excess(model, model, pre, ts, suh, sv, mode) == 0
        ex = recon_excess(_recon_fault(fault, tr, suh, svh, K, c0, n), model, pre, ts, suh, sv, mode)
        assert ex >= MARGIN, f"{fault} mode {mode}: {ex:.2f}x the bars"


@pytest.mark.parametrize("fault", ["window_n_offset_off_by_128", "window_buffer_overwritten"])
def test_forward_dense_faults_miss_the_f64_bar(fault):
    # forward_dense's folded window walk at reduced width: windows of 256 over n = 640 (the real: 32768 over 128256)
    k, n, K, win = 256, 640, 4, 256
    tr, suh, svh = small_linear(k, n, K, 41)
    x = torch.randn((16, k), generator=torch.Generator().manual_seed(2)).half()
    wins = [(c, min(c + win, n)) for c in range(0, n, win)]
    full, _, _ = ot.reconstruct_had_model(tr, suh, svh, K, 2)
    ref = f64_oracle(x, ot.decode_weights(tr, K, 2), suh, svh)
    W = []
    for j, (c0, c1) in enumerate(wins):
        off = c0 + (128 if fault == "window_n_offset_off_by_128" and j == len(wins) - 1 else 0)
        if off + (c1 - c0) > n:
            off = c0 - 128
        w, _, _ = ot.reconstruct_had_model(tr, suh, svh, K, 2, n_offset=off, n=c1 - c0)
        if fault == "window_buffer_overwritten" and j == 1:
            w = W[0][:, :c1 - c0]                    # the GEMM of window 1 reads window 0's weights
        W.append(w)
    good = (x.double() @ full.double()).float()
    assert strip_excess(good, ref)[0] < 1
    y = torch.cat([(x.double() @ w.double()).float() for w in W], 1)
    ex, strip = strip_excess(y, ref)
    assert ex >= MARGIN, f"{fault}: {ex:.2f}x the bar at strip {strip}"
