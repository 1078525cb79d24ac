"""
exl3_moe, the fused routed-expert MLP (csrc/moe_tc.cu, tag 230), against two references on the same synthetic experts
(oracle.exl3_oracle.make_synthetic):
  * the fp64 oracle: per expert exl3_gemm_f64 for gate / up / down, fp16 rounding of g, u and h (the fp16 buffers between
    the GEMMs), the activation in fp64;
  * a composition of verified operators: per expert ext.exl3_gemm on the exact tensor-core path (tag 200) for gate and up,
    the activation in torch, ext.exl3_gemm for down, a weighted index_add.
Bars (README "parity"): max-abs <= 4e-3 * max|y|, rel-RMS <= 2e-3.  Rows of tokens with no processed position keep their bits.
Every case is also held to the exact model of the operator's arithmetic, oracle.exl3_moe_model (test_edges_host.check_moe_model).
"""
import zlib
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc
from test_edges_host import check_moe_model

pytestmark = pytest.mark.gpu

SENTINEL_BITS = 0x7FA5A5A5          # a NaN payload: any write to a row that must stay untouched shows


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def bars(y, ref):
    y = np.asarray(y, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
    err = np.abs(y - ref)
    mx = max(np.abs(ref).max(), 1e-30)
    return err.max() / mx, np.sqrt((err ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


class Experts:
    """E experts of gate / up / down; `uniq` distinct tensors per projection, expert e uses tensor e % uniq."""

    def __init__(self, dev, E, hidden, inter, Kg, Ku, Kd, cb, uniq=None, seed=0):
        self.E, self.hidden, self.inter, self.cb = E, hidden, inter, cb
        self.K = {"gate": Kg, "up": Ku, "down": Kd}
        self.uniq = min(E, uniq or E)
        self.np, self.dev, self.w = {}, {}, {}
        for i, (name, k, n) in enumerate((("gate", hidden, inter), ("up", hidden, inter), ("down", inter, hidden))):
            mats = [orc.make_synthetic(k, n, self.K[name], seed=seed + 7919 * i + 31 * u) for u in range(self.uniq)]
            self.np[name] = [m[:3] for m in mats]
            self.dev[name] = [tuple(T(a, dev) for a in m[:3]) for m in mats]
        self.tables = {}
        for name in ("gate", "up", "down"):
            for j, part in enumerate(("trellis", "suh", "svh")):
                self.tables[f"{name}_{part}"] = torch.tensor(
                    [self.dev[name][e % self.uniq][j].data_ptr() for e in range(E)], dtype=torch.long, device=dev)

    def W(self, name, u):
        key = (name, u)
        if key not in self.w:
            self.w[key] = orc.reconstruct(self.np[name][u][0], self.K[name], self.cb)
        return self.w[key]

    def gemm64(self, name, e, x):
        tr, suh, svh = self.np[name][e % self.uniq]
        return orc.exl3_gemm_f64(x, tr, suh, svh, self.K[name], self.cb, w=self.W(name, e % self.uniq))

    def gemm_tc(self, name, e, x, out_dtype):
        tr, suh, svh = self.dev[name][e % self.uniq]
        y = torch.empty((x.shape[0], tr.shape[1] * 16), dtype=out_dtype, device=x.device)
        tag = ext().exl3_gemm(x, tr, y, suh, torch.empty_like(x), svh, 2, self.cb == 1, self.cb == 2, 0)
        assert tag == ext().EXL3B_TAG_TC
        return y


def ext():
    from exllamav3_b200 import ext as e
    return e


def route(rng, bsz, E, topk, sentinel_frac=0.0, hot=None):
    """Top-k routing sorted by expert, as the reference's BlockSparseMLP builds it; a share of the choices goes to the
    sentinel bucket (expert index E: experts of another device in expert-parallel mode).  hot: force these experts into
    the choices of the first tokens, to give them large counts."""
    ex = np.stack([rng.choice(E, topk, replace=False) for _ in range(bsz)])
    if hot:
        for i, (e, n) in enumerate(hot.items()):
            for t in range(min(n, bsz)):
                if e not in ex[t]:
                    ex[t, i % topk] = e
    if sentinel_frac:
        ex[rng.random(ex.shape) < sentinel_frac] = E
    wt = rng.uniform(0.05, 1.0, ex.shape).astype(np.float16)
    fe, ft, fw = ex.reshape(-1), np.repeat(np.arange(bsz), topk), wt.reshape(-1)
    order = np.argsort(fe, kind="stable")
    count = np.bincount(fe, minlength=E + 1).astype(np.int64)
    return count, ft[order].astype(np.int64), fw[order]


def act64(g, u, act, limit):
    g = g.astype(np.float64); u = u.astype(np.float64)
    if act == 0:
        a = g / (1.0 + np.exp(-g))
    elif act == 1:
        a = 0.5 * g * (1.0 + np.tanh(0.797884560803 * (g + 0.044715 * g ** 3)))
    else:
        a = np.maximum(u, 0.0)
    if limit:
        u = np.clip(u, -limit, limit); a = np.minimum(a, limit)
    return a * u


def act_torch(g, u, act, limit):
    g = g.float(); u = u.float()
    if act == 0:
        a = torch.nn.functional.silu(g)
    elif act == 1:
        a = torch.nn.functional.gelu(g, approximate="tanh")
    else:
        a = torch.relu(u)
    if limit:
        u = u.clamp(-limit, limit); a = a.clamp(max=limit)
    return (a * u).half()


def processed(count, T_, N):
    s, lo, out = 0, 0, []
    for e, c in enumerate(count[:-1]):
        if 0 < c <= T_ and s >= lo and s + c <= N:
            out.append((e, s, int(c)))
            lo = s + c
        s += int(c)
    return out


def references(ex, x, out0, count, tok, wts, T_, act, limit, dev, fp64=True):
    procs = processed(count, T_, len(tok))
    ref64 = out0.astype(np.float64).copy() if fp64 else None
    comp = torch.from_numpy(out0.copy()).to(dev)
    xd = T(x, dev)
    for e, s, c in procs:
        J = np.arange(s, s + c)
        X = x[tok[J]]
        if fp64:
            u = ex.gemm64("up", e, X).astype(np.float16)
            g = u if act == 2 else ex.gemm64("gate", e, X).astype(np.float16)
            h = act64(g, u, act, limit).astype(np.float16)
            y = ex.gemm64("down", e, h)
            np.add.at(ref64, tok[J], wts[J].astype(np.float64)[:, None] * y)
        Xd = xd[torch.from_numpy(tok[J]).to(dev)].contiguous()
        ud = ex.gemm_tc("up", e, Xd, torch.half)
        gd = ud if act == 2 else ex.gemm_tc("gate", e, Xd, torch.half)
        yd = ex.gemm_tc("down", e, act_torch(gd, ud, act, limit), torch.float)
        comp.index_add_(0, torch.from_numpy(tok[J]).to(dev), torch.from_numpy(wts[J].astype(np.float32)).to(dev)[:, None] * yd)
    touched = np.zeros(len(out0), dtype=bool)
    for e, s, c in procs:
        touched[tok[s:s + c]] = True
    return ref64, comp.cpu().numpy(), touched, procs


def call(ex, dev, x, out, count, tok, wts, T_, act, limit, num_active=-1, conc=None, poison=True):
    e = ext()
    conc = conc or e.exl3_moe_max_concurrency(dev.index or 0)
    fill = float("nan") if poison else 0.0
    tsg = torch.full((conc, T_, ex.hidden), fill, dtype=torch.half, device=dev)
    tig = torch.full((conc, T_, ex.inter), fill, dtype=torch.half, device=dev)
    t = ex.tables
    gate = "up" if act == 2 else "gate"              # ReLU^2 without a gate: the caller passes the up tables as gate tables
    e.exl3_moe(x, out, count, tok, wts, tsg, tsg.clone(), tig, tig.clone(), act, ex.K[gate], ex.K["up"], ex.K["down"],
               t[f"{gate}_trellis"], t[f"{gate}_suh"], t[f"{gate}_svh"], t["up_trellis"], t["up_suh"], t["up_svh"],
               t["down_trellis"], t["down_suh"], t["down_svh"],
               ex.cb == 1, ex.cb == 2, ex.cb == 1, ex.cb == 2, ex.cb == 1, ex.cb == 2, limit, num_active)


def run_case(dev, E, topk, bsz, hidden, inter, Ks, cb, act, limit, T_, seed, sentinel_frac=0.0, hot=None, uniq=None,
             fp64=True, expect=()):
    rng = np.random.default_rng(seed)
    ex = Experts(dev, E, hidden, inter, *Ks, cb, uniq=uniq, seed=seed)
    count, tok, wts = route(rng, bsz, E, topk, sentinel_frac, hot)
    if T_ == "auto":                                 # the second-largest distinct count: some experts at exactly T, some above
        T_ = int(np.unique(count[:-1][count[:-1] > 0])[-2])
    elif isinstance(T_, tuple):                      # ("of", e): expert e's count
        T_ = int(count[T_[1]])
    x = rng.standard_normal((bsz, hidden)).astype(np.float16)
    out0 = (rng.standard_normal((bsz, hidden)) * 0.5).astype(np.float32)
    ref64, comp, touched, procs = references(ex, x, out0, count, tok, wts, T_, act, limit, dev, fp64)
    out0.view(np.uint32)[~touched] = SENTINEL_BITS
    if "zero" in expect:
        assert (count[:-1] == 0).any()
    if "exact" in expect:
        assert (count[:-1] == T_).any()
    if "over" in expect:
        assert (count[:-1] > T_).any()
    if "sentinel" in expect:
        assert count[-1] > 0
    out = T(out0, dev)
    call(ex, dev, T(x, dev), out, T(count, dev), T(tok, dev), T(wts, dev), T_, act, limit)
    y = out.cpu().numpy()
    assert (y.view(np.uint32)[~touched] == SENTINEL_BITS).all(), "a row with no processed position was written"
    assert np.isfinite(y[touched]).all()
    mx, rms = bars(y[touched], comp[touched])
    assert mx <= 4e-3 and rms <= 2e-3, f"vs composition: max {mx:.2e} rms {rms:.2e}"
    mats = {name: [ex.np[name][e % ex.uniq] + (ex.K[name], ex.W(name, e % ex.uniq)) for e in range(E)] for name in ex.np}
    model = orc.exl3_moe_model(x, out0, count, tok, wts, T_, act, limit, mats, cb)
    check_moe_model(y[touched], model[touched], "vs exact model")
    if fp64:
        mx, rms = bars(y[touched], ref64[touched])
        assert mx <= 4e-3 and rms <= 2e-3, f"vs fp64 oracle: max {mx:.2e} rms {rms:.2e}"
    return ex, procs


# E, topk, bsz, hidden, inter, (Kg, Ku, Kd), cb, act, limit, T, sentinel share, hot experts, expected edges
CASES = {
    "e8-top1-bsz1": (8, 1, 1, 256, 384, (4, 4, 4), 2, 0, 0.0, 16, 0.0, None, ()),
    "e8-top2-bsz5-mixedK": (8, 2, 5, 384, 640, (2, 5, 3), 2, 0, 0.0, "auto", 0.0, None, ("exact", "over")),
    "e64-top8-bsz64-mcg-gelu": (64, 8, 64, 384, 256, (3, 4, 6), 1, 1, 0.0, "auto", 0.1, None, ("exact", "over", "sentinel")),
    "e128-top2-bsz300-relu2-pass2": (128, 2, 300, 256, 384, (4, 4, 2), 2, 2, 0.0, ("of", 7), 0.05, {3: 150, 5: 250, 7: 200},
                                     ("zero", "exact", "over", "sentinel")),
    "e8-top8-bsz300-silu-limit-pass3": (8, 8, 300, 640, 384, (1, 8, 7), 1, 0, 0.75, 300, 0.0, None, ("exact",)),
    "e64-top2-bsz64-gelu-limit": (64, 2, 64, 256, 640, (5, 6, 8), 2, 1, 0.5, "auto", 0.0, None, ("zero", "exact", "over")),
    "e8-top2-bsz64-relu2-limit": (8, 2, 64, 384, 256, (3, 3, 3), 1, 2, 0.6, "auto", 0.0, None, ("exact", "over")),
}


@pytest.mark.parametrize("name", list(CASES))
def test_moe_matches_oracle_and_composition(cuda, name):
    E, topk, bsz, hidden, inter, Ks, cb, act, limit, T_, sf, hot, expect = CASES[name]
    run_case(cuda, E, topk, bsz, hidden, inter, Ks, cb, act, limit, T_, seed=zlib.crc32(name.encode()) % 10000, sentinel_frac=sf, hot=hot,
             expect=expect)


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("limit", [0.0, 0.4])
def test_moe_activations(cuda, act, limit):
    run_case(cuda, 8, 2, 24, 256, 384, (4, 3, 5), 2, act, limit, 16, seed=40 + 3 * act + int(limit * 10))


@pytest.mark.parametrize("bsz", [64, 300])
def test_moe_qwen3_30b_a3b_shape(cuda, bsz):
    # Qwen3-30B-A3B: hidden 2048, moe_intermediate 768, 128 experts, top-8 (8 distinct tensors per projection, shared cyclically)
    run_case(cuda, 128, 8, bsz, 2048, 768, (4, 4, 4), 2, 0, 0.0, 128, seed=77 + bsz, uniq=8, fp64=bsz == 64)


def test_moe_multiple_chunks(cuda):
    # Mixtral-8x7B widths: 3200 positions do not fit the fixed work area at once, so the call runs in several chunks
    E, topk, bsz, hidden, inter = 8, 2, 1600, 4096, 14336
    rng = np.random.default_rng(123)
    count, _, _ = route(rng, bsz, E, topk)
    plan = ext().exl3_moe_plan(count, bsz, bsz * topk, hidden, inter)[0]
    assert plan.chunks >= 2
    run_case(cuda, E, topk, bsz, hidden, inter, (2, 3, 2), 2, 0, 0.0, bsz, seed=123, uniq=2, fp64=False)


def _setup_small(dev, seed=5, E=8, topk=2, bsz=40, T_=16, act=0):
    rng = np.random.default_rng(seed)
    ex = Experts(dev, E, 256, 384, 4, 3, 5, 2, seed=seed)
    count, tok, wts = route(rng, bsz, E, topk, 0.1)
    x = T(rng.standard_normal((bsz, 256)).astype(np.float16), dev)
    out0 = T((rng.standard_normal((bsz, 256))).astype(np.float32), dev)
    return ex, x, out0, T(count, dev), T(tok, dev), T(wts, dev), count


def test_moe_num_active(cuda):
    ex, x, out0, count, tok, wts, c = _setup_small(cuda)
    n_act = int(((c[:-1] > 0) & (c[:-1] <= 16)).sum())
    outs = []
    for na in (-1, n_act):
        out = out0.clone()
        call(ex, cuda, x, out, count, tok, wts, 16, 0, 0.0, num_active=na)
        outs.append(out)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    out = out0.clone()
    call(ex, cuda, x, out, count, tok, wts, 16, 0, 0.0, num_active=0)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int32), out0.view(torch.int32))


def test_moe_deterministic_and_graph_replay(cuda):
    ex, x, out0, count, tok, wts, _ = _setup_small(cuda, seed=9, E=64, topk=8, bsz=96, T_=24)
    a, b = out0.clone(), out0.clone()
    call(ex, cuda, x, a, count, tok, wts, 24, 0, 0.0)
    call(ex, cuda, x, b, count, tok, wts, 24, 0, 0.0)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two identical calls differ"
    conc = ext().exl3_moe_max_concurrency(0)
    tsg = torch.zeros((conc, 24, 256), dtype=torch.half, device=cuda)
    tig = torch.zeros((conc, 24, 384), dtype=torch.half, device=cuda)
    g_out = torch.empty_like(out0)
    t = ex.tables
    args = lambda: (x, g_out, count, tok, wts, tsg, tsg, tig, tig, 0, 4, 3, 5,
                    t["gate_trellis"], t["gate_suh"], t["gate_svh"], t["up_trellis"], t["up_suh"], t["up_svh"],
                    t["down_trellis"], t["down_suh"], t["down_svh"], False, True, False, True, False, True, 0.0, -1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g_out.copy_(out0); ext().exl3_moe(*args())
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out.copy_(out0)
        ext().exl3_moe(*args())
    for _ in range(2):
        g_out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(g_out.view(torch.int32), a.view(torch.int32)), "graph replay differs from the eager call"


def test_moe_graph_capture_larger_than_any_eager_call(cuda):
    # the work area is fixed: a capture with more positions than any earlier call needs no allocation
    ex, x, out0, count, tok, wts, _ = _setup_small(cuda, seed=3, bsz=4)
    o = out0.clone()
    call(ex, cuda, x, o, count, tok, wts, 16, 0, 0.0)
    ex, x, out0, count, tok, wts, c = _setup_small(cuda, seed=4, E=64, topk=8, bsz=1000)
    T_ = int(c[:-1].max())
    conc = ext().exl3_moe_max_concurrency(0)
    tsg = torch.zeros((conc, T_, 256), dtype=torch.half, device=cuda)
    tig = torch.zeros((conc, T_, 384), dtype=torch.half, device=cuda)
    t = ex.tables
    g_out = torch.empty_like(out0)
    args = (x, g_out, count, tok, wts, tsg, tsg, tig, tig, 0, 4, 3, 5,
            t["gate_trellis"], t["gate_suh"], t["gate_svh"], t["up_trellis"], t["up_suh"], t["up_svh"],
            t["down_trellis"], t["down_suh"], t["down_svh"], False, True, False, True, False, True, 0.0, -1)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out.copy_(out0)
        ext().exl3_moe(*args)
    graph.replay()
    torch.cuda.synchronize()
    eager = out0.clone()
    call(ex, cuda, x, eager, count, tok, wts, T_, 0, 0.0)
    assert torch.equal(g_out.view(torch.int32), eager.view(torch.int32))


def test_moe_surface(cuda):
    e = ext()
    assert hasattr(e, "exl3_moe") and hasattr(e, "exl3_moe_max_concurrency")
    assert e.exl3_moe_max_concurrency(0) == torch.cuda.get_device_properties(0).multi_processor_count // 8


def test_moe_validation_errors(cuda):
    e = ext()
    ex, x, out0, count, tok, wts, _ = _setup_small(cuda)
    conc = e.exl3_moe_max_concurrency(0)
    tsg = torch.zeros((conc, 16, 256), dtype=torch.half, device=cuda)
    tig = torch.zeros((conc, 16, 384), dtype=torch.half, device=cuda)
    t = ex.tables
    base = dict(hidden_state=x, output_state=out0.clone(), expert_count=count, token_sorted=tok, weight_sorted=wts,
                temp_state_g=tsg, temp_state_u=tsg, temp_intermediate_g=tig, temp_intermediate_u=tig, act_function=0,
                K_gate=4, K_up=3, K_down=5,
                gate_ptrs_trellis=t["gate_trellis"], gate_ptrs_suh=t["gate_suh"], gate_ptrs_svh=t["gate_svh"],
                up_ptrs_trellis=t["up_trellis"], up_ptrs_suh=t["up_suh"], up_ptrs_svh=t["up_svh"],
                down_ptrs_trellis=t["down_trellis"], down_ptrs_suh=t["down_suh"], down_ptrs_svh=t["down_svh"],
                gate_mcg=False, gate_mul1=True, up_mcg=False, up_mul1=True, down_mcg=False, down_mul1=True,
                act_limit=0.0, num_active=-1)
    bad = {
        "hidden dtype": dict(hidden_state=x.float()),
        "hidden dims": dict(hidden_state=x[None]),
        "output dtype": dict(output_state=out0.half()),
        "output shape": dict(output_state=out0[:-1].clone()),
        "count dtype": dict(expert_count=count.int()),
        "token dtype": dict(token_sorted=tok.int()),
        "weight dtype": dict(weight_sorted=wts.float()),
        "weight shape": dict(weight_sorted=wts[:-1]),
        "temp dtype": dict(temp_state_g=tsg.float()),
        "temp dims": dict(temp_state_g=tsg[0]),
        "temp hidden": dict(temp_state_g=tsg[..., :128], temp_state_u=tsg[..., :128]),
        "intermediate shape": dict(temp_intermediate_u=tig[:, :8]),
        "table length": dict(up_ptrs_svh=t["up_svh"][:-1]),
        "mixed codebook": dict(down_mcg=True, down_mul1=False),
        "no codebook": dict(gate_mul1=False, up_mul1=False, down_mul1=False),
        "both codebooks": dict(gate_mcg=True, up_mcg=True, down_mcg=True),
        "concurrency": dict(temp_state_g=torch.zeros((conc + 1, 16, 256), dtype=torch.half, device=cuda),
                            temp_state_u=torch.zeros((conc + 1, 16, 256), dtype=torch.half, device=cuda)),
        "K": dict(K_down=9),
        "act": dict(act_function=3),
        "hidden % 128": dict(hidden_state=x[:, :192].contiguous(), output_state=out0[:, :192].contiguous(),
                             temp_state_g=tsg[..., :192], temp_state_u=tsg[..., :192]),
        "intermediate % 128": dict(temp_intermediate_g=tig[..., :320], temp_intermediate_u=tig[..., :320]),
        "cpu tensor": dict(expert_count=count.cpu()),
        "misaligned hidden_state": dict(hidden_state=torch.zeros(x.numel() + 2, dtype=torch.half, device=cuda)[2:].view_as(x)),
        "misaligned output_state": dict(output_state=torch.zeros(out0.numel() + 1, device=cuda)[1:].view_as(out0)),
    }
    for what, change in bad.items():
        kw = dict(base, **change)
        o = kw["output_state"]
        before = o.clone()
        with pytest.raises(RuntimeError):
            e.exl3_moe(**kw)
        torch.cuda.synchronize()
        assert torch.equal(o.view(torch.int32), before.view(torch.int32)), f"{what}: output written"
