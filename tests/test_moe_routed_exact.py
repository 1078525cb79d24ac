"""
Routed / weighted exl3_mgemm on the int8 path (csrc/gemm_tc_i8_routed.cu, tag 212) held to the exact model of its arithmetic:
the MoE decode calls of the reference (modules/block_sparse_mlp.py) at bsz 1 and batched (num_tokens > 1, the reference's
BC_BlockSparseMLP::run_bszN_gr), expert-parallel shards, every CTA-group size, cached and uncached activations, the reduce
bit for bit, the CUDA-core fallbacks and CUDA-graph replay with the routing rewritten between replays.

Every call is checked against two references, slot by slot:
  * oracle.exl3_mgemm_i8_model: w_j * exl3_gemm_i8_model(A[j or 0], expert) per active slot, then the reduce;
    max-abs <= 2e-5 max|y|, rel-RMS <= 1e-5 (fp32 C), 1.5e-3 / 5e-4 (fp16 C), as tags 210 and 220;
  * the fp64 oracle (exl3_gemm_f64 per slot with the same slot table and reduce) at max-abs <= 2e-3 max|y| (+2^-9 for
    fp16 C), rel-RMS <= 1e-3.
Unweighted slots must also equal the single-matrix tag-210 exl3_gemm on the same input and expert bit for bit, at the grid
of the slot's CTA group.  The weighted reduce is checked bit for bit against the host sum of the per-slot outputs, which the
same call returns with num_tokens = slots (stride 1: the reduce is the identity).

C lives in the middle of a larger allocation whose outer slots hold a NaN sentinel; A is a view whose trailing slot is NaN.

The CPU tests at the end hold the oracle's exl3_mgemm and the new model's reduce to a direct restatement of the reference's
reduction loop (exllamav3_ext/quant/exl3_gemm_kernel.cuh:238-291).
"""
import itertools
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc
from test_edges_host import CACHE_PAIRS, check_f16_model, gemm_plan

gpu = pytest.mark.gpu

TAG_SIMT, TAG_I8, TAG_ROUTED = 100, 210, 212
SENTINEL = {torch.half: (torch.int16, 0x7E5A), torch.float: (torch.int32, 0x7FA5A5A5)}     # NaN payloads nobody writes
QWEN3 = dict(E=128, topk=8, hidden=2048, inter=768)            # Qwen3-30B-A3B experts
MIXTRAL = dict(E=8, topk=2, hidden=4096, inter=14336)          # Mixtral 8x7B experts


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def rel_err(y, ref):
    y = np.asarray(y, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(y - ref)
    return err.max() / max(np.abs(ref).max(), 1e-30), np.sqrt((err ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Experts:
    """
    E experts of one projection (k -> n): `uniq` distinct trellis tensors shared cyclically (expert e uses tensor e % uniq), so
    the host decodes few matrices, and every expert its own suh and svh, so that a slot that reads another expert's pointer
    table entry gives another result.
    """

    def __init__(self, dev, E, k, n, K, uniq=8, cb=2, seed=0):
        rng = np.random.default_rng(seed)
        self.E, self.k, self.n, self.K, self.cb, self.uniq = E, k, n, K, cb, min(uniq, E)
        self.tr = [rng.integers(0, 65536, size=(k // 16, n // 16, 16 * K), dtype=np.uint16).view(np.int16) for _ in range(self.uniq)]
        self.suh = [(np.sign(rng.standard_normal(k)) * rng.uniform(0.5, 2.0, k) / np.sqrt(k)).astype(np.float16) for _ in range(E)]
        self.svh = [(np.sign(rng.standard_normal(n)) * rng.uniform(0.5, 2.0, n)).astype(np.float16) for _ in range(E)]
        self.d_tr = [T(t, dev) for t in self.tr]
        self.d_suh = [T(s, dev) for s in self.suh]
        self.d_svh = [T(s, dev) for s in self.svh]
        ptr = lambda ts: torch.tensor([t.data_ptr() for t in ts], dtype=torch.long, device=dev)
        self.pt = ptr([self.d_tr[e % self.uniq] for e in range(E)])
        self.ps, self.pv = ptr(self.d_suh), ptr(self.d_svh)
        self._bsum, self._w, self._memo = {}, {}, {}

    def tables(self, lo=0, hi=None):
        hi = self.E if hi is None else hi
        return tuple(t[lo:hi].contiguous() for t in (self.pt, self.ps, self.pv))

    def _cached(self, kind, e, a):
        key = (kind, e, a.tobytes())
        if key not in self._memo:
            u = e % self.uniq
            if kind == "model":                                         # before the svh multiply (i8_model_output)
                if u not in self._bsum:
                    self._bsum[u] = orc.mul1_bytesum(self.tr[u], self.K)
                y = orc.exl3_gemm_i8_model(a, self.tr[u], self.suh[e], None, self.K, bsum=self._bsum[u])
            else:
                if u not in self._w:
                    self._w[u] = orc.reconstruct(self.tr[u], self.K, self.cb)
                y = orc.exl3_gemm_f64(a, self.tr[u], self.suh[e], self.svh[e], self.K, self.cb, w=self._w[u])
            self._memo[key] = y
        return self._memo[key]

    def reference(self, kind, A, c_b, fp32, off=0, **kw):
        """Whole-call reference of `kind` "model" (exact int8 model) or "f64"; expert numbers are local + off (shards)."""
        dt = np.float32 if fp32 else np.float16

        def slot(a, q, scale):
            y = self._cached(kind, q + off, np.ascontiguousarray(a))
            return orc.i8_model_output(y, self.svh[q + off], dt, scale) if kind == "model" else scale * y

        return orc.mgemm_compose(A, slot, c_b, self.n, dt, **kw)


class Call:
    """One exl3_mgemm call: C inside a sentinel frame, A followed by a NaN slot."""

    def __init__(self, dev, ex, A, idx, w=None, fp32=True, num_tokens=1, lo=-1, hi=-1, c_b=None, C_init=None):
        self.ex, self.A, self.idx, self.w, self.fp32, self.num_tokens, self.lo, self.hi = ex, A, idx, w, fp32, num_tokens, lo, hi
        a_b, m, k = A.shape
        self.c_b = c_b if c_b is not None else len(idx)
        self.slots = min(max(a_b, self.c_b), len(idx))                 # the kernels' slot count (exl3_gemm.cu:476-489)
        self.C_init = C_init
        dt = torch.float if fp32 else torch.half
        Af = torch.full((a_b + 1, m, k), float("nan"), dtype=torch.half, device=dev)
        Af[:a_b] = T(A, dev)
        self.Cf = torch.empty((self.c_b + 2, m, ex.n), dtype=dt, device=dev)
        self.Cf.view(SENTINEL[dt][0]).fill_(SENTINEL[dt][1])
        self.Cf[1:-1] = 0 if C_init is None else T(C_init, dev).to(dt)
        it = torch.tensor([list(idx)], dtype=torch.long, device=dev)
        wt = None if w is None else T(np.asarray(w, dtype=np.float16), dev).view(1, -1)
        tables = ex.tables(lo, hi) if lo >= 0 else ex.tables()
        from exllamav3_b200 import ext
        self.tag = ext.exl3_mgemm(Af[:a_b], tables[0], self.Cf[1:-1], tables[1],
                                  torch.empty((self.slots, m, k), dtype=torch.half, device=dev), tables[2], it, wt, ex.K, -1,
                                  ex.cb == 1, ex.cb == 2, lo, hi, 0, num_tokens)

    def result(self):
        """C as numpy in its own dtype, after checking the sentinel frame and finiteness."""
        torch.cuda.synchronize()
        itype, bits = SENTINEL[self.Cf.dtype]
        raw = self.Cf.view(itype).cpu().numpy()
        assert (raw[0] == bits).all() and (raw[-1] == bits).all(), "slots outside C written"
        y = self.Cf[1:-1].cpu().numpy()
        assert np.isfinite(y).all(), "non-finite output"
        return y

    def kw(self):
        return dict(indices=self.idx, weights=self.w, min_index=self.lo, max_index=self.hi, num_tokens=self.num_tokens,
                    C_init=self.C_init)

    def check(self, y, what, model=True):
        """Each slot of C against the f64 oracle and (mul1) the exact model; where a reference is exactly zero, so must C be."""
        off = max(self.lo, 0)
        refs = [("f64", self.ex.reference("f64", self.A, self.c_b, self.fp32, off, **self.kw()))]
        if model:
            refs.append(("model", self.ex.reference("model", self.A, self.c_b, self.fp32, off, **self.kw())))
        for kind, ref in refs:
            for j in range(self.c_b):
                r = ref[j].astype(np.float64)
                if not r.any():
                    assert not y[j].any(), (what, kind, j, "expected exact zeros")
                    continue
                mx, rms = rel_err(y[j], r)
                if kind == "model":
                    bar = (2e-5, 1e-5) if self.fp32 else (1.5e-3, 5e-4)
                else:
                    bar = (2e-3 + (0 if self.fp32 else 2.0 ** -9), 1e-3)
                assert mx <= bar[0] and rms <= bar[1], (what, kind, j, self.fp32, mx, rms)
        return refs


def run(dev, ex, A, idx, w=None, fp32=True, tag=TAG_ROUTED, what=None, model=True, **kw):
    c = Call(dev, ex, A, idx, w, fp32, **kw)
    assert c.tag == tag, (what, c.tag)
    y = c.result()
    c.check(y, what, model=model and ex.cb == 2)
    return c, y


def check_single_slots(dev, ex, c, y, what):
    """Unweighted call: every active slot equals the single-matrix tag-210 exl3_gemm on its input and expert at its group's grid."""
    from exllamav3_b200 import ext
    a_b, m, k = c.A.shape
    units = (ex.k // 128) * (ex.n // 128)
    G = min(num_sms() // c.slots, units)
    p = gemm_plan(m, ex.k, ex.n, ex.K, 2, force=G, sms=num_sms())
    assert (p.path, p.grid) == (TAG_I8, G), (what, p.path, p.grid, G)
    off = max(c.lo, 0)
    for j, (q, _) in enumerate(orc.mgemm_slots(c.slots, c.idx, None, c.lo, c.hi)):
        if q < 0:
            continue
        e = q + off
        a = T(c.A[0] if a_b == 1 else c.A[j], dev)
        out = torch.empty((m, ex.n), dtype=c.Cf.dtype, device=dev)
        tag = ext.exl3_gemm(a, ex.d_tr[e % ex.uniq], out, ex.d_suh[e], torch.empty_like(a), ex.d_svh[e], -1, False, True, G)
        assert tag == TAG_I8
        assert np.array_equal(out.cpu().numpy().view(np.uint8), y[j].view(np.uint8)), (what, j, e, G)


def check_reduce(dev, ex, A, idx, w, fp32, num_tokens, tag=TAG_ROUTED, what=None, C_init=None):
    """
    The weighted call with num_tokens = T against the same call with num_tokens = slots (stride 1: the reduce is the identity,
    C holds the weighted per-slot outputs): row t is their host sum in slot order, in C's dtype, bit for bit; rows T.. are the
    identity call's rows.  Returns (first call, its C).
    """
    c1 = Call(dev, ex, A, idx, w, fp32, num_tokens=num_tokens, C_init=C_init)
    c2 = Call(dev, ex, A, idx, w, fp32, num_tokens=len(idx), C_init=C_init)
    assert c1.tag == tag and c2.tag == tag, (what, c1.tag, c2.tag)
    y1, y2 = c1.result(), c2.result()
    host = orc.mgemm_reduce(y2, len(idx), num_tokens)
    assert np.array_equal(y1[:num_tokens].view(np.uint8), host[:num_tokens].view(np.uint8)), (what, "reduced rows")
    assert np.array_equal(y1[num_tokens:].view(np.uint8), y2[num_tokens:].view(np.uint8)), (what, "rows past the tokens")
    return c1, y1


def route(rng, E, T_, topk, shared=()):
    """topk distinct experts per token, token-major; experts in `shared` are forced into every token's selection."""
    idx = []
    for _ in range(T_):
        rest = rng.permutation([e for e in range(E) if e not in shared])[:topk - len(shared)]
        sel = list(shared) + [int(e) for e in rest]
        idx += [int(e) for e in rng.permutation(sel)]
    return idx


def routing_weights(rng, n):
    return rng.uniform(0.05, 1.0, n).astype(np.float16)


# ---- 1. bsz-1 decode -------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("shape", ["qwen3", "mixtral"])
def test_bsz1_decode(cuda, shape):
    """gate / up with one input, down with per-slot inputs and weights: 8 (Qwen3) or 2 (Mixtral) slots at real widths."""
    s = QWEN3 if shape == "qwen3" else MIXTRAL
    uniq = 8 if shape == "qwen3" else 2
    gate = Experts(cuda, s["E"], s["hidden"], s["inter"], 4, uniq=uniq, seed=1)
    down = Experts(cuda, s["E"], s["inter"], s["hidden"], 4, uniq=uniq, seed=2)
    rng = np.random.default_rng(3)
    idx = route(rng, s["E"], 1, s["topk"])
    x = rng.standard_normal((1, 1, s["hidden"])).astype(np.float16)
    h = rng.standard_normal((s["topk"], 1, s["inter"])).astype(np.float16)
    w = routing_weights(rng, s["topk"])
    for fp32 in (True, False):
        c, y = run(cuda, gate, x, idx, fp32=fp32, what=(shape, "gate", fp32))
        check_single_slots(cuda, gate, c, y, (shape, "gate", fp32))
        run(cuda, down, h, idx, w, fp32=fp32, what=(shape, "down", fp32))
        check_reduce(cuda, down, h, idx, w, fp32, 1, what=(shape, "down reduce", fp32))


# ---- 2. expert-parallel shard ----------------------------------------------------------------------------------------------

@gpu
def test_expert_parallel_shard(cuda):
    """Experts [32, 64) with local tables: selections off the shard are compacted away with their inputs and weights."""
    s = QWEN3
    lo, hi = 32, 64
    gate = Experts(cuda, s["E"], s["hidden"], s["inter"], 4, seed=11)
    down = Experts(cuda, s["E"], s["inter"], s["hidden"], 4, seed=12)
    rng = np.random.default_rng(13)
    x = rng.standard_normal((1, 1, s["hidden"])).astype(np.float16)
    h = rng.standard_normal((8, 1, s["inter"])).astype(np.float16)
    w = routing_weights(rng, 8)
    # on-shard selections at positions 1, 2, 4, 7: a resolve that keeps the weight of the compacted position instead of the
    # selection's own, or reads the input of the original position, gives other numbers
    cases = [[5, 40, 33, 100, 63, 0, 127, 32],
             [lo, 70, 71, 72, 73, 74, 75, 76]]
    for idx in cases:
        for fp32 in (True, False):
            c, y = run(cuda, gate, x, idx, fp32=fp32, lo=lo, hi=hi, what=(idx, "gate", fp32))
            check_single_slots(cuda, gate, c, y, (idx, "gate", fp32))
            run(cuda, down, h, idx, w, fp32=fp32, lo=lo, hi=hi, what=(idx, "down", fp32))
    # nothing on this shard: no active slot, C[0] is the empty sum and every other slot keeps its bits
    init = rng.standard_normal((8, 1, s["hidden"])).astype(np.float16)
    for fp32 in (True, False):
        c = Call(cuda, down, h, [0, 1, 2, 3, 64, 65, 100, 127], w, fp32, lo=lo, hi=hi, C_init=init)
        assert c.tag == TAG_ROUTED
        y = c.result()
        assert not y[0].any()
        assert np.array_equal(y[1:], init[1:].astype(y.dtype))


# ---- 3. batched decode -----------------------------------------------------------------------------------------------------

BATCHED = list(itertools.product((2, 3, 8), (2, 8, 16)))


@gpu
@pytest.mark.parametrize("T_,topk", BATCHED)
def test_batched_decode(cuda, T_, topk):
    """
    num_tokens = T: gate / up on per-slot inputs gathered per token (each token's rows identical), down with weights reduced into
    C[t]; two experts are in every token's selection, so slots repeat experts.  4 .. 128 slots.
    """
    s = QWEN3 if topk == 8 else dict(E=64, hidden=1024, inter=512)
    gate = Experts(cuda, s["E"], s["hidden"], s["inter"], 4, seed=20 + topk)
    down = Experts(cuda, s["E"], s["inter"], s["hidden"], 4, seed=30 + topk)
    rng = np.random.default_rng(100 * T_ + topk)
    idx = route(rng, s["E"], T_, topk, shared=(5, 17))
    slots = T_ * topk
    x = rng.standard_normal((T_, 1, s["hidden"])).astype(np.float16)
    xg = np.repeat(x, topk, axis=0)                                     # the per-slot gather of each token's row
    h = rng.standard_normal((slots, 1, s["inter"])).astype(np.float16)
    w = routing_weights(rng, slots)
    for fp32 in (True, False):
        what = (T_, topk, fp32)
        c, y = run(cuda, gate, xg, idx, fp32=fp32, num_tokens=T_, what=what + ("gate",))
        check_single_slots(cuda, gate, c, y, what + ("gate",))
        c1 = Call(cuda, gate, xg, idx, None, fp32)                       # no weights: num_tokens changes nothing
        assert c1.tag == TAG_ROUTED and np.array_equal(c1.result().view(np.uint8), y.view(np.uint8)), what
        c, y = check_reduce(cuda, down, h, idx, w, fp32, T_, what=what + ("down",))
        c.check(y, what + ("down",))


# ---- 4. slot-count sweep ---------------------------------------------------------------------------------------------------

def sweep_slots(S):
    return sorted({1, 2, 3, 8, 16, S // 4, S // 2 - 2, S // 2, S // 2 + 1, min(128, S)})


@gpu
def test_slot_count_sweep(cuda):
    """Slot counts at which a slot's CTA group (num_sms // slots CTAs) takes every size down to one CTA."""
    S = num_sms()
    E, k, n = 128, 1024, 512
    gate = Experts(cuda, E, k, n, 4, seed=40)
    down = Experts(cuda, E, n, k, 4, seed=41)
    rng = np.random.default_rng(42)
    groups = set()
    for slots in sweep_slots(S):
        idx = [int(e) for e in rng.permutation(E)[:slots]]
        groups.add(min(S // slots, (k // 128) * (n // 128)))
        x = rng.standard_normal((1, 1, k)).astype(np.float16)
        h = rng.standard_normal((slots, 1, n)).astype(np.float16)
        w = routing_weights(rng, slots)
        for fp32 in (True, False):
            c, y = run(cuda, gate, x, idx, fp32=fp32, what=(slots, "gate", fp32))
            check_single_slots(cuda, gate, c, y, (slots, "gate", fp32))
        c, y = check_reduce(cuda, down, h, idx, w, True, 1, what=(slots, "down"))
        c.check(y, (slots, "down"))
    assert 1 in groups and 2 in groups


# ---- 5. rows per slot, and the activation cache ----------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("K", (2, 3, 4, 6))
def test_rows_per_slot(cuda, K):
    """m = 1, 2, 4 rows per slot (the MR = 4 tile) at num_tokens = 1: gate on one input, down with weights."""
    E, k, n = 8, 512, 384
    gate = Experts(cuda, E, k, n, K, seed=50 + K)
    down = Experts(cuda, E, n, k, K, seed=60 + K)
    rng = np.random.default_rng(K)
    idx = [6, 1, 3, 6]
    for m in (1, 2, 4):
        x = rng.standard_normal((1, m, k)).astype(np.float16)
        h = rng.standard_normal((4, m, n)).astype(np.float16)
        w = routing_weights(rng, 4)
        for fp32 in (True, False):
            c, y = run(cuda, gate, x, idx, fp32=fp32, what=(K, m, "gate", fp32))
            check_single_slots(cuda, gate, c, y, (K, m, "gate", fp32))
            c, y = check_reduce(cuda, down, h, idx, w, fp32, 1, what=(K, m, "down", fp32))
            c.check(y, (K, m, "down", fp32))


@gpu
def test_activation_cache_pairs(cuda):
    """Per-slot inputs just inside and just outside the 64 KiB activation cache, one routed call each."""
    rng = np.random.default_rng(70)
    for (m, k, cached) in CACHE_PAIRS:
        ex = Experts(cuda, 4, k, 256, 4, uniq=2, seed=k)
        idx = [3, 0, 2]
        A = rng.standard_normal((3, m, k)).astype(np.float16)
        for fp32 in (True, False):
            c, y = run(cuda, ex, A, idx, fp32=fp32, what=(m, k, cached, fp32))
            check_single_slots(cuda, ex, c, y, (m, k, cached, fp32))


# ---- 6. a skipped slot inside a weighted batched call ----------------------------------------------------------------------

@gpu
def test_skipped_slot_in_weighted_batch(cuda):
    """Index -1: the GEMM leaves the slot's rows as they were and the reduce adds them, as the reference kernel does."""
    E, k, n = 16, 1024, 512
    down = Experts(cuda, E, k, n, 4, seed=80)
    rng = np.random.default_rng(81)
    idx = [3, 9, 12, 0, 7, -1, 3, 15]                                   # 2 tokens x top-4, one selection skipped
    A = rng.standard_normal((8, 1, k)).astype(np.float16)
    w = routing_weights(rng, 8)
    init = (rng.standard_normal((8, 1, n)) * 4).astype(np.float16)
    for fp32 in (True, False):
        c, y = check_reduce(cuda, down, A, idx, w, fp32, 2, what=("skip", fp32), C_init=init)
        c.check(y, ("skip", fp32))
        c2 = Call(cuda, down, A, idx, w, fp32, num_tokens=8, C_init=init)
        assert np.array_equal(c2.result()[5], init[5].astype(y.dtype))


# ---- 7. path selection and fallbacks ---------------------------------------------------------------------------------------

def check_f16_slots(ex, c, y, what):
    """A tag-100 call against the exact model of the fp16 paths (oracle.exl3_mgemm_f16_model), slot by slot."""
    trl = [ex.tr[e % ex.uniq] for e in range(ex.E)]
    ref, tol = orc.exl3_mgemm_f16_model(c.A, trl, ex.suh, ex.svh, ex.K, ex.cb, np.float32 if c.fp32 else np.float16, bszm_out=c.c_b,
                                        **c.kw())
    for j in range(c.c_b):
        check_f16_model(y[j], ref[j], None if tol is None else tol[j], (what, j))


@gpu
def test_cuda_core_fallbacks(cuda):
    """m = 5, the mcg and 3inst codebooks and a forced EXL3B_TAG_SIMT go to tag 100: oracle bar and the reduce bit for bit."""
    from exllamav3_b200 import ext
    rng = np.random.default_rng(90)
    k, n, E = 1024, 512, 16
    idx = [2, 11, 5, 2, 14, 0, 9, 5]                                    # 2 tokens x top-4, expert 2 and 5 in both
    w = routing_weights(rng, 8)
    for (cb, m, force) in ((2, 5, 0), (1, 1, 0), (0, 1, 0), (2, 1, TAG_SIMT)):
        ex = Experts(cuda, E, k, n, 4, cb=cb, seed=91 + cb)
        x = rng.standard_normal((1, m, k)).astype(np.float16)
        A = rng.standard_normal((8, m, k)).astype(np.float16)
        prev = ext.set_gemm_path(force)
        try:
            for fp32 in (True, False):
                what = (cb, m, force, fp32)
                c, y = run(cuda, ex, x, idx, fp32=fp32, tag=TAG_SIMT, what=what, model=False)
                check_f16_slots(ex, c, y, what)
                c, y = check_reduce(cuda, ex, A, idx, w, fp32, 2, tag=TAG_SIMT, what=what)
                c.check(y, what, model=False)
                check_f16_slots(ex, c, y, what)
        finally:
            ext.set_gemm_path(prev)


@gpu
def test_more_than_128_slots_is_refused(cuda):
    from exllamav3_b200 import ext
    ex = Experts(cuda, 8, 512, 256, 4, seed=95)
    A = torch.zeros((1, 1, 512), dtype=torch.half, device=cuda)
    C = torch.empty((131, 1, 256), dtype=torch.float, device=cuda)
    C.view(torch.int32).fill_(SENTINEL[torch.float][1])
    idx = torch.tensor([[j % 8 for j in range(129)]], dtype=torch.long, device=cuda)
    w = torch.full((1, 129), 0.5, dtype=torch.half, device=cuda)
    with pytest.raises(RuntimeError, match="more than 128 slots"):
        ext.exl3_mgemm(A, ex.pt, C[1:130], ex.ps, torch.empty((129, 1, 512), dtype=torch.half, device=cuda), ex.pv, idx, w, 4, -1,
                       False, True, -1, -1, 0)
    torch.cuda.synchronize()
    assert (C.view(torch.int32) == SENTINEL[torch.float][1]).all()


# ---- 8. CUDA-graph replay --------------------------------------------------------------------------------------------------

@gpu
def test_graph_replay_with_new_routing(cuda):
    """
    The bsz-1 decode step gate -> up -> silu(g) * u -> weighted down, all with the expert filter of a shard, captured on a side
    stream and replayed with new routing copied into the captured indices / weights; eager routed calls of other shapes in
    between go around the 8 scratch slots.  Every replay equals the eager step on the same routing bit for bit.
    """
    from exllamav3_b200 import ext
    s = QWEN3
    lo, hi = 32, 96
    gate = Experts(cuda, s["E"], s["hidden"], s["inter"], 4, seed=101)
    up = Experts(cuda, s["E"], s["hidden"], s["inter"], 4, seed=102)
    down = Experts(cuda, s["E"], s["inter"], s["hidden"], 4, seed=103)
    tg, tu, td = gate.tables(lo, hi), up.tables(lo, hi), down.tables(lo, hi)
    rng = np.random.default_rng(104)
    x = T(rng.standard_normal((1, 1, s["hidden"])).astype(np.float16), cuda)
    idx = torch.zeros((1, 8), dtype=torch.long, device=cuda)
    wt = torch.zeros((1, 8), dtype=torch.half, device=cuda)
    g = torch.empty((8, 1, s["inter"]), dtype=torch.half, device=cuda)
    u, hbuf = torch.empty_like(g), torch.empty_like(g)
    y = torch.empty((8, 1, s["hidden"]), dtype=torch.float, device=cuda)
    Ah_g = torch.empty((8, 1, s["hidden"]), dtype=torch.half, device=cuda)
    Ah_d = torch.empty((8, 1, s["inter"]), dtype=torch.half, device=cuda)

    def step():
        g.zero_(); u.zero_(); y.zero_()
        tags = [ext.exl3_mgemm(x, tg[0], g, tg[1], Ah_g, tg[2], idx, None, 4, -1, False, True, lo, hi, 0),
                ext.exl3_mgemm(x, tu[0], u, tu[1], Ah_g, tu[2], idx, None, 4, -1, False, True, lo, hi, 0)]
        hbuf.copy_(torch.nn.functional.silu(g) * u)
        tags.append(ext.exl3_mgemm(hbuf, td[0], y, td[1], Ah_d, td[2], idx, wt, 4, -1, False, True, lo, hi, 0))
        return tags

    routings = [(route(rng, s["E"], 1, 8), routing_weights(rng, 8)) for _ in range(4)]

    def set_routing(r):
        idx.copy_(torch.tensor([r[0]], dtype=torch.long))
        wt.copy_(T(r[1], "cpu").view(1, 8))

    def eager(r):
        set_routing(r)
        assert step() == [TAG_ROUTED] * 3
        torch.cuda.synchronize()
        return y.clone(), hbuf.clone()

    set_routing(routings[3])
    assert step() == [TAG_ROUTED] * 3                                   # eager first: tensor maps and kernel attributes
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        with torch.cuda.graph(gr, stream=st):
            assert step() == [TAG_ROUTED] * 3
    others = []
    for j, (k, n, slots) in enumerate(((1024, 512, 3), (512, 1024, 16), (2048, 256, 66))):
        ex = Experts(cuda, 16, k, n, 4, uniq=2, seed=110 + j)
        A = rng.standard_normal((slots, 1, k)).astype(np.float16)
        others.append((ex, A, [int(e) for e in rng.integers(0, 16, slots)], routing_weights(rng, slots)))
    for rnd in range(3):
        set_routing(routings[rnd])
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            gr.replay()
        st.synchronize()
        got_y, got_h = y.clone(), hbuf.clone()
        for _ in range(3):                                              # 3 x 3 launch slots: around the ring of 8
            for (ex, A, oi, ow) in others:
                assert Call(cuda, ex, A, oi, ow, True).tag == TAG_ROUTED
        e_y, e_h = eager(routings[rnd])
        e_y2, _ = eager(routings[rnd])
        assert torch.equal(e_y.view(torch.int32), e_y2.view(torch.int32)), rnd
        assert torch.equal(got_h.view(torch.int16), e_h.view(torch.int16)), rnd
        assert torch.equal(got_y.view(torch.int32), e_y.view(torch.int32)), rnd
        assert got_y[0].abs().max() > 0 or not any(lo <= e < hi for e in routings[rnd][0])


# ---- 9. CPU: the references' reduce against the reference kernel's loop ----------------------------------------------------

def reduce_restated(C, bszm, num_tokens):
    """exl3_gemm_kernel.cuh:238-291 as written: per column, groups t = 0, 1, ... in increasing order, in place in C."""
    C = np.array(C, copy=True)
    b, m, n = C.shape
    flat = C.reshape(b, m * n)
    stride = bszm // num_tokens
    for col in range(m * n):
        for t in range(num_tokens):
            if C.dtype == np.float32:
                s = np.float32(0.0)
                for j in range(stride):
                    s = np.float32(s + flat[t * stride + j, col])
            else:
                s = np.float16(0.0)
                for j in range(stride):
                    s = np.float16(float(s) + float(flat[t * stride + j, col]))      # __hadd: exact sum, one rounding
            flat[t, col] = s
    return C


@pytest.mark.parametrize("dt", (np.float32, np.float16))
@pytest.mark.parametrize("T_,topk", ((1, 3), (2, 3), (3, 2), (4, 1), (2, 5)))
def test_oracle_mgemm_reduce_matches_reference_loop(dt, T_, topk):
    """oracle.exl3_mgemm(num_tokens = T) is its own per-slot outputs (num_tokens = slots) put through the reference's loop."""
    k, n, K, E = 256, 128, 3, 4
    mats = [orc.make_synthetic(k, n, K, seed=7 + e) for e in range(E)]
    trl, sul, svl = [m[0] for m in mats], [m[1] for m in mats], [m[2] for m in mats]
    rng = np.random.default_rng(T_ * 10 + topk)
    slots = T_ * topk
    A = rng.standard_normal((slots, 2, k)).astype(np.float16)
    idx = [int(e) for e in rng.integers(0, E, slots)]
    w = routing_weights(rng, slots)
    per_slot = orc.exl3_mgemm(A, trl, sul, svl, K, 0, dt, indices=idx, weights=w, num_tokens=slots)
    got = orc.exl3_mgemm(A, trl, sul, svl, K, 0, dt, indices=idx, weights=w, num_tokens=T_)
    assert np.array_equal(got.view(np.uint8), reduce_restated(per_slot, slots, T_).view(np.uint8))


@pytest.mark.parametrize("dt", (np.float32, np.float16))
@pytest.mark.parametrize("T_,topk", ((1, 4), (2, 3), (3, 2), (2, 1)))
def test_model_reduce_matches_reference_loop(dt, T_, topk):
    """oracle.exl3_mgemm_i8_model: the same restatement, in C's dtype, and each slot is w_j times the single-matrix model."""
    k, n, K, E = 256, 128, 4, 4
    mats = [orc.make_synthetic(k, n, K, seed=70 + e) for e in range(E)]
    trl, sul, svl = [m[0] for m in mats], [m[1] for m in mats], [m[2] for m in mats]
    rng = np.random.default_rng(T_ * 10 + topk + 1)
    slots = T_ * topk
    A = rng.standard_normal((slots, 1, k)).astype(np.float16)
    idx = [int(e) for e in rng.integers(0, E, slots)]
    w = routing_weights(rng, slots)
    per_slot = orc.exl3_mgemm_i8_model(A, trl, sul, svl, K, dt, indices=idx, weights=w, num_tokens=slots)
    for j in range(slots):
        pre = orc.exl3_gemm_i8_model(A[j], trl[idx[j]], sul[idx[j]], None, K)
        y = float(w[j]) * pre * svl[idx[j]].astype(np.float64)
        if dt == np.float16:                                # rounded before the fp16 svh multiply, as the epilogue does
            y = (orc._hmul((float(w[j]) * pre).astype(np.float16), svl[idx[j]][None, :]))
        assert np.array_equal(per_slot[j], y.astype(per_slot.dtype))
    got = orc.exl3_mgemm_i8_model(A, trl, sul, svl, K, dt, indices=idx, weights=w, num_tokens=T_)
    ref_dt = np.float32 if dt == np.float32 else np.float16
    expect = reduce_restated(per_slot.astype(ref_dt), slots, T_)
    if dt == np.float16:
        assert np.array_equal(got.view(np.uint8), expect.view(np.uint8))
    else:                                                   # the fp32-C model sums in fp64
        assert np.abs(got - expect).max() <= 1e-6 * np.abs(expect).max()
    # the fp32 host sum the GPU tests use for fp32 C is the restated loop bit for bit
    per32 = per_slot.astype(np.float32)
    assert np.array_equal(orc.mgemm_reduce(per32, slots, T_).view(np.uint8), reduce_restated(per32, slots, T_).view(np.uint8))


def test_model_slot_table_under_the_expert_filter():
    """Compaction: on-shard selections keep their own weight (weights[s]) and take the compacted position's input and output."""
    k, n, K, E = 256, 128, 4, 6
    mats = [orc.make_synthetic(k, n, K, seed=90 + e) for e in range(E)]
    trl, sul, svl = [m[0] for m in mats], [m[1] for m in mats], [m[2] for m in mats]
    lo, hi = 2, 5
    idx = [0, 4, 5, 2, 1, 3]
    w = np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6], dtype=np.float16)
    assert orc.mgemm_slots(6, idx, w, lo, hi) == [(2, np.float16(0.2)), (0, np.float16(0.4)), (1, np.float16(0.6))]
    A = np.random.default_rng(3).standard_normal((6, 1, k)).astype(np.float16)
    got = orc.exl3_mgemm_i8_model(A, trl[lo:hi], sul[lo:hi], svl[lo:hi], K, np.float32, indices=idx, weights=w,
                                  min_index=lo, max_index=hi)
    ys = [float(np.float16(wj)) * orc.exl3_gemm_i8_model(A[j], trl[e], sul[e], None, K) * svl[e].astype(np.float64)
          for j, (e, wj) in enumerate(((4, 0.2), (2, 0.4), (3, 0.6)))]
    assert np.array_equal(got[0], (ys[0] + ys[1]) + ys[2])               # the reduce of the three active slots into C[0]
    assert np.array_equal(got[1], ys[1]) and np.array_equal(got[2], ys[2])
    assert not got[3:].any()
    # the oracle's mgemm has the same slot table
    ref = orc.exl3_mgemm(A, trl[lo:hi], sul[lo:hi], svl[lo:hi], K, 2, np.float32, indices=idx, weights=w, min_index=lo,
                         max_index=hi)
    for j in range(3):
        assert rel_err(got[j], ref[j])[0] < 2e-3, j
