"""
Every output of bench.py's decode token held to the int8 path's exact model, in every column (H100).

bench.py times 129 launches per Llama-3.1-8B token, all on the int8 decode-GEMM (tag 210).  Here the same bench.Token is built
and run, eagerly with each of its three launch lists and as the CUDA graph bench.py times, and every element of its 225 outputs
is compared with oracle.exl3_gemm_i8_model.  The model's integer contraction runs exactly on the GPU
(oracle.exl3_oracle_torch.i8_contract: an fp64 matmul of integers below 2^39), everything else is the numpy model, so the GPU
and the host model share every rounding point.  Inputs that share a weight are contracted in one pass over it.

Bars, per output:
  fp32 C (o, gate, up, down, lm_head): max-abs <= 2e-5 max|y|, rel-RMS <= 1e-5 against the model;
  fp16 C (q, k, v): every element within oracle.f16_model_tol of the model (one fp16 step of the pre-svh value times |svh|, plus
      one step of C) plus 2e-5 max|y| (the fp32 bar, for elements far below max|y|), at least TOKEN_F16_SAME of the elements of
      a launch list's fp16 outputs bit-identical to it, and 1.5e-3 / 5e-4 against the model before C's rounding;
  all: the fp64 oracle (exl3_gemm_f64, W_hat from the byte-sum table) max-abs <= 2e-3 max|y| (+1 fp16 step), rel-RMS <= 1e-3.
A failure names the output, its worst 128-column strip and the CTAs and units that wrote that strip (from the planner).

The rank-0 shard tokens `bench.py --tp-shapes N` runs, and the qgemm section's batch and codebook legs, are held the same way.
The fault catalog shows what the bars see at these shapes that a sample of strips does not (tests/test_bench_token_host.py
builds the faults and asserts the shapes reach the unit walk's schedules).
"""
import sys, time
import numpy as np
import pytest
import torch
from conftest import ROOT
from oracle import exl3_oracle as orc
from oracle import exl3_oracle_torch as ot
from test_bench_token_host import TOKENS, fault_unit, launch_kind, matrix_grids, strip_writers, unit_faults
from test_edges_host import check_f16_gemm, gemm_plan

sys.path.insert(0, ROOT)
import bench

pytestmark = pytest.mark.gpu

TAG_TC, TAG_I8 = 200, 210
I8_BAR = (2e-5, 1e-5)
I8_F16_BAR = (1.5e-3, 5e-4)
F64_BAR = (2e-3, 1e-3)
TOKEN_F16_SAME = 0.99                # fp16 C elements bit-identical to the model, at least (measured on an H100: 99.6 %)
MARGIN = 3.0                         # a catalog fault misses the bars by at least this factor
# faults the bars do not see by MARGIN at the catalog's units (README.md, Parity): none.  (f) is caught there, but its size is
# C1 (sum of q over the neighbouring k-block - over the unit's), C1 = 1534 k_inv + k_bias ~ -0.0018, and a k-block sum of q is
# sqrt(128) times one transformed input: at other units or inputs it can fall inside the bars.
NOT_CAUGHT = set()


def key(mt):
    return "lm_head" if mt["layer"] < 0 else f"L{mt['layer']:02d}_{mt['name']}"


def by_layer(tok):
    d = {}
    for mt in tok.mats:
        d.setdefault(mt["layer"], {})[mt["name"]] = mt
    return d


def share_inputs(tok, xs):
    """k and v read q's input, up reads gate's: what the fused launches do, so that every launch list computes the same."""
    idx = {id(mt): i for i, mt in enumerate(tok.mats)}
    for d in by_layer(tok).values():
        if "q" in d:
            for a, b in (("q", "k"), ("q", "v"), ("gate", "up")):
                xs[idx[id(d[b])]] = xs[idx[id(d[a])]]
    return xs


def list_outputs(tok, launches):
    """Every output of a launch list, by matrix, gathered as bench.Token.outputs() gathers the default list's."""
    out = {}
    for ln in launches:
        for j, mt in enumerate(ln["mats"]):
            out[key(mt)] = ln["y"][j].view(1, -1) if ln["kind"] == "mgemm" and ln["cp"] is None else mt["y"]
    return out


def list_geometry(launches, sms):
    """(U, G, KB) of every matrix of a launch list, by matrix."""
    geo = {}
    for ln in launches:
        mats = tuple((mt["name"], mt["k"], mt["n"], mt["K"]) for mt in ln["mats"])
        for mt, g in zip(ln["mats"], matrix_grids(launch_kind(ln), mats, sms=sms)):
            geo[key(mt)] = g
    return geo


def poison(tok, launches):
    for mt in tok.mats:
        mt["y"].fill_(float("nan"))
    for ln in launches:
        if ln["kind"] == "mgemm":
            ln["y"].fill_(float("nan"))
    torch.cuda.synchronize()


class Model:
    """The int8 model of one matrix for rows x (r, k): pre (r, n) before svh, f64 (r, n) the fp64 oracle."""

    def __init__(self, mt, x):
        suh, self.svh = mt["suh"].cpu().numpy(), mt["svh"].cpu().numpy()
        q, _ = orc.i8_activation_q(x, suh)
        qb, acc = ot.i8_contract(mt["tr"], mt["K"], q, orc.had_r_128(x, pre_scale=suh))
        self.x, self.suh, self.K = x, suh, mt["K"]
        self.pre = orc.exl3_gemm_i8_model(x, None, suh, None, mt["K"], qb=qb)
        self.f64 = orc.exl3_gemm_f64(None, None, None, self.svh, mt["K"], 2, acc=acc)


def token_models(tok, xs_new):
    """Model per matrix key for two inputs per matrix: its current x (row 0) and xs_new (row 1), contracted in one pass."""
    return {key(mt): Model(mt, np.concatenate([mt["x"].cpu().numpy(), xn.cpu().numpy()]))
            for mt, xn in zip(tok.mats, xs_new)}


def rel(y, ref):
    y = np.asarray(y, np.float64); ref = np.asarray(ref, np.float64)
    d = np.abs(y - ref)
    return d.max() / max(np.abs(ref).max(), 1e-30), np.sqrt((d ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def ratios(y, pre, f64, svh, fp32):
    """How far C is from each bar (<= 1: within).  y, pre, f64: (r, n)."""
    y = np.asarray(y)
    r = {}
    if fp32:
        mx, rms = rel(y, pre * svh.astype(np.float64)[None, :])
        r["model"] = max(mx / I8_BAR[0], rms / I8_BAR[1])
        ulp = 0.0
    else:
        model = orc.i8_model_output(pre, svh, np.float16)
        # one fp16 step of the pre-svh value and of C (oracle.f16_model_tol), plus the fp32 bar of the accumulation itself: where
        # |C| is far below max|C| the kernel's fp32 round-off, which scales with max|C|, is more than a step of that element
        tol = orc.f16_model_tol(model, pre.astype(np.float16), svh) + I8_BAR[0] * np.abs(model.astype(np.float64)).max()
        d = np.abs(y.astype(np.float64) - model.astype(np.float64))
        r["f16_tol"] = float(np.max(np.where(d > 0, d / np.maximum(tol, 1e-300), 0.0)))
        r["changed"] = float((y.astype(np.float16).view(np.uint16) != model.view(np.uint16)).mean()) / (1 - TOKEN_F16_SAME)
        mx, rms = rel(y, pre * svh.astype(np.float64)[None, :])
        r["model"] = max(mx / I8_F16_BAR[0], rms / I8_F16_BAR[1])
        ulp = 2.0 ** -10
    mx, rms = rel(y, f64)
    r["f64"] = max(mx / (F64_BAR[0] + ulp), rms / F64_BAR[1])
    return r


def worst_strip(y, ref):
    d = np.abs(np.asarray(y, np.float64) - np.asarray(ref, np.float64))
    d = np.where(np.isnan(d), np.inf, d)
    return int(d.reshape(d.shape[0], -1, 128).max(axis=(0, 2)).argmax())


STATS = {}


def check(y, model, row, fp32, what, geo):
    """C (1, n) against row `row` of the model; on failure the worst strip and the CTAs / units that wrote it."""
    y = y.float().cpu().numpy() if fp32 else y.cpu().numpy()
    pre, f64 = model.pre[row:row + 1], model.f64[row:row + 1]
    r = ratios(y, pre, f64, model.svh, fp32)
    kind = "fp32" if fp32 else "fp16"
    for k_, v in r.items():
        STATS[(kind, k_)] = max(STATS.get((kind, k_), 0.0), v)
    if not fp32:
        STATS[("fp16", "changed_frac")] = max(STATS.get(("fp16", "changed_frac"), 0.0), r["changed"] * (1 - TOKEN_F16_SAME))
    if max(v for k_, v in r.items() if k_ != "changed") > 1.0 or not np.isfinite(y).all():
        s = worst_strip(y, pre * model.svh.astype(np.float64)[None, :])
        U, G, KB = geo
        raise AssertionError(f"{what}: {r}; worst strip {s} of {U // KB}, written by (cta, first unit, last unit) "
                             f"{strip_writers(U, G, KB, s)} of {G} CTAs, {KB} k-blocks per strip")
    return 0.0 if fp32 else r["changed"] * (1 - TOKEN_F16_SAME) * y.size, 0 if fp32 else y.size


def check_list(tok, launches, models, row, what, sms):
    outs, geo = list_outputs(tok, launches), list_geometry(launches, sms)
    assert len(outs) == len(tok.mats)
    fp32 = {key(mt): mt["c_fp32"] for mt in tok.mats}
    changed = total = 0
    for k_, y in outs.items():
        c, t = check(y, models[k_], row, fp32[k_], f"{what} {k_}", geo[k_])
        changed, total = changed + c, total + t
    # the bit-identical share is taken over all fp16 outputs of the list: a 128-column output alone is too coarse for it
    assert changed <= (1 - TOKEN_F16_SAME) * total, (what, "fp16 C elements not bit-identical to the model", changed / total)
    STATS[("fp16", "changed_frac_of_list")] = max(STATS.get(("fp16", "changed_frac_of_list"), 0.0), changed / total)
    return outs


def run(tok, launches, stream):
    with torch.cuda.stream(stream):
        tok.run(launches)
    stream.synchronize()


def capture(tok, stream):
    """bench.py's CUDA graph of the token: eager warm-up on a side stream, then the capture."""
    with torch.cuda.stream(stream):
        for _ in range(2):
            tok.run()
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        tok.run()
    return graph


def new_inputs(tok, seed):
    g = torch.Generator(device=tok.dev); g.manual_seed(seed)
    return share_inputs(tok, [torch.randn(tuple(mt["x"].shape), generator=g, device=tok.dev).half() for mt in tok.mats])


def graph_checks(tok, models, xs_new, stream, what, sms):
    """Replay of the captured token: bit-identical to the eager run, then with new inputs written in place, held to the model."""
    poison(tok, tok.launches)
    run(tok, tok.launches, stream)
    eager = {k_: y.clone() for k_, y in list_outputs(tok, tok.launches).items()}
    graph = capture(tok, stream)
    poison(tok, tok.launches)
    with torch.cuda.stream(stream):
        graph.replay()
    stream.synchronize()
    for k_, y in list_outputs(tok, tok.launches).items():
        assert torch.equal(y.view(torch.uint8), eager[k_].view(torch.uint8)), (what, "graph replay differs from the eager run", k_)
    old = [mt["x"].clone() for mt in tok.mats]
    for mt, xn in zip(tok.mats, xs_new):
        mt["x"].copy_(xn)
    poison(tok, tok.launches)
    with torch.cuda.stream(stream):
        graph.replay()
    stream.synchronize()
    check_list(tok, tok.launches, models, 1, f"{what} graph replay, new inputs", sms)
    for mt, xo in zip(tok.mats, old):
        mt["x"].copy_(xo)
    del graph
    torch.cuda.synchronize()


def prepare(cfg, tp, dev, seed):
    tok = bench.Token(cfg, tp, 0, dev)
    tok.skip_reduce = True                             # one rank's shard alone, as bench.py --tp-shapes
    xs = share_inputs(tok, [mt["x"] for mt in tok.mats])
    for mt, x in zip(tok.mats, xs):
        if mt["x"] is not x:
            mt["x"].copy_(x)
    xs_new = new_inputs(tok, seed)
    t0 = time.time()
    models = token_models(tok, xs_new)
    print(f"# models of {len(models)} matrices ({cfg['layers']} layers, tp {tp}): {time.time() - t0:.1f} s")
    return tok, xs_new, models


def device_used(dev):
    """The most device memory this process has held (GiB, torch's caching allocator: tensors, graph pools, workspaces)."""
    return torch.cuda.max_memory_reserved(dev) / 2 ** 30


def sms_of(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


# ---- bench.py's token (Llama-3.1-8B, one GPU) --------------------------------------------------------------------------------

class TestToken8B:
    @pytest.fixture(scope="class")
    def token(self, cuda):
        tok, xs_new, models = prepare(bench.MODELS["llama-3.1-8b"], 1, cuda, 99)
        yield tok, xs_new, models, torch.cuda.Stream(device=cuda)
        print(f"# 8B: device memory in use at most {device_used(cuda):.2f} GiB; worst ratios {STATS}")
        del tok, models
        torch.cuda.empty_cache()

    @pytest.mark.parametrize("which", ("fanout", "reference", "one_per_projection"))
    def test_launch_list_every_output(self, token, cuda, which):
        tok, _, models, stream = token
        launches = {"fanout": tok.launches, "reference": tok.launches_ref,
                    "one_per_projection": tok._launch_list(False, False)}[which]
        assert len(launches) == {"fanout": 129, "reference": 161, "one_per_projection": 225}[which]
        poison(tok, launches)
        run(tok, launches, stream)
        outs = check_list(tok, launches, models, 0, which, sms_of(cuda))
        if which == "fanout":
            assert outs.keys() == tok.outputs().keys() and len(outs) == 225

    def test_graph_replay_new_inputs(self, token, cuda):
        tok, xs_new, models, stream = token
        graph_checks(tok, models, xs_new, stream, "8B", sms_of(cuda))

    @pytest.mark.parametrize("name", ("q", "gate", "down"))
    def test_decode_batch(self, token, cuda, name):
        """bench.py's decode_batch leg at m = 8 and 32, one matrix: the tag the planner names, every element against its model."""
        from exllamav3_b200 import ext
        tok, _, _, _ = token
        mt = by_layer(tok)[0][name]
        k, n, K, fp32 = mt["k"], mt["n"], mt["K"], mt["c_fp32"]
        suh, svh = mt["suh"].cpu().numpy(), mt["svh"].cpu().numpy()
        g = torch.Generator(device=cuda); g.manual_seed(8 + k + n)
        w = None
        for m in (8, 32):
            xb = torch.randn((m, k), generator=g, device=cuda).half()
            yb = torch.empty((m, n), dtype=torch.float if fp32 else torch.half, device=cuda)
            tag = ext.exl3_gemm(xb, mt["tr"], yb, mt["suh"], torch.empty_like(xb), mt["svh"], -1, False, True, 0)
            torch.cuda.synchronize()
            assert tag == gemm_plan(m, k, n, K, 2, sms=sms_of(cuda)).path, (name, m, tag)
            x = xb.cpu().numpy()
            y = yb.float().cpu().numpy() if fp32 else yb.cpu().numpy()
            if tag == TAG_I8:
                model = Model(mt, x)
                r = ratios(y, model.pre, model.f64, svh, fp32)
                assert max(r.values()) <= 1.0, (name, m, r)
            else:
                assert tag == TAG_TC, (name, m, tag)
                w = ot.mul1_weights(mt["tr"], K) if w is None else w
                check_f16_gemm(y, x, None, suh, svh, K, 2, fp32, (name, m), w=w)

    @pytest.mark.parametrize("name,cb", (("q", 0), ("q", 1), ("gate", 0)))
    def test_decode_codebooks(self, token, cuda, name, cb):
        """bench.py's decode_codebooks leg (3INST, MCG) at m = 1 on tag 200, every element against the fp16 path's model."""
        from exllamav3_b200 import ext
        tok, _, _, _ = token
        mt = by_layer(tok)[0][name]
        k, n, K, fp32 = mt["k"], mt["n"], mt["K"], mt["c_fp32"]
        y = torch.empty((1, n), dtype=torch.float if fp32 else torch.half, device=cuda)
        tag = ext.exl3_gemm(mt["x"], mt["tr"], y, mt["suh"], torch.empty_like(mt["x"]), mt["svh"], -1, cb == 1, False, 0)
        torch.cuda.synchronize()
        assert tag == TAG_TC
        tr = mt["tr"].cpu().numpy()
        w = np.concatenate([orc.reconstruct(tr[:, c0 // 16:c1 // 16], K, cb) for c0, c1 in ot.column_chunks(k, n, 1 << 22)], axis=1)
        check_f16_gemm(y.float().cpu().numpy() if fp32 else y.cpu().numpy(), mt["x"].cpu().numpy(), None,
                       mt["suh"].cpu().numpy(), mt["svh"].cpu().numpy(), K, cb, fp32, (name, cb), w=w)

    def test_fault_catalog(self, token, cuda):
        """
        Faults of the unit walk at one 128 x 128 unit of lm_head (the last sub-segment of its CTA with the most units) and of
        L00 down, and svh before the rounding over all of L00 q: each misses the bars by MARGIN unless it is in NOT_CAUGHT.  Below every
        bar and not in the table: a row's activation scale off by one fp32 ulp (~1e-7 relative), held bit for bit by
        tests/test_i8_div_host.py.
        """
        tok, _, models, _ = token
        d = by_layer(tok)
        table, missed = [], []
        for mt in (d[-1]["lm_head"], d[0]["down"], d[0]["q"]):
            md = models[key(mt)]
            x, pre, f64 = md.x[:1], md.pre[:1], md.f64[:1]
            strip, kb, cta, units, _ = fault_unit(mt["k"], mt["n"], mt["K"], sms=sms_of(cuda))
            for name, y in unit_faults(x, mt["tr"], md.suh, md.svh, mt["K"], pre, strip, kb, mt["c_fp32"]).items():
                if mt["name"] == "q" and not name.startswith("(h)"):
                    continue
                r = ratios(y, pre, f64, md.svh, mt["c_fp32"])
                caught = max(v for k_, v in r.items() if k_ != "f64")
                table.append((key(mt), strip, kb, cta, units, name, round(caught, 1), round(r["f64"], 3)))
                if caught < MARGIN and name not in NOT_CAUGHT:
                    missed.append(table[-1])
        for row in table:
            print("# fault", row)
        assert not missed, missed


# ---- the rank-0 shard tokens of bench.py --tp-shapes --------------------------------------------------------------------------

@pytest.mark.parametrize("model,tp", TOKENS[1:])
def test_shard_token_every_output(cuda, model, tp):
    tok, xs_new, models = prepare(bench.MODELS[model], tp, cuda, 100 + tp)
    stream = torch.cuda.Stream(device=cuda)
    try:
        poison(tok, tok.launches)
        run(tok, tok.launches, stream)
        check_list(tok, tok.launches, models, 0, f"{model} tp{tp}", sms_of(cuda))
        graph_checks(tok, models, xs_new, stream, f"{model} tp{tp}", sms_of(cuda))
    finally:
        print(f"# {model} tp{tp}: device memory in use at most {device_used(cuda):.2f} GiB")
        del tok, models
        torch.cuda.empty_cache()
