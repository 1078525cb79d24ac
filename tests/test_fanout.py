"""
Fan-out launches: exl3_mgemm with per-matrix output widths (size_n_list / c_ptrs; exllamav3_ext/quant/exl3_gemm.cu:402-447,
exl3_gemm_kernel.cuh:172-181; used by the reference for same-input projections, libtorch/dsv4_attn.cpp:88-99) as ONE launch of the
wgmma int8 kernel.  CPU: the CTA-group partition and the width registry.  GPU: parity of the fused call with the separate calls
and with the oracle on the Llama q + k + v shapes (8B, and a 70B TP-8 shard), shared and per-matrix inputs, graph replay, fall-backs.
"""
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc


def test_fanout_partition_properties():
    from exllamav3_b200 import ext
    for k, widths, sms in ((4096, [4096, 1024, 1024], 148), (8192, [1024, 128, 128], 148), (4096, [14336, 14336], 148),
                           (128, [128, 128, 128], 148), (4096, [128, 14336], 148), (256, [128] * 8, 16), (4096, [4096, 1024, 1024], 7)):
        b = ext.plan_fanout(k, widths, sms)
        assert b is not None and b[0] == 0 and len(b) == len(widths) + 1
        units = [(k // 128) * (w // 128) for w in widths]
        assert b[-1] == min(sms, sum(units))
        for j, u in enumerate(units):
            g = b[j + 1] - b[j]
            assert 1 <= g <= u, (widths, b)
        # proportional up to rounding and the one-CTA minimum: no group is more than one CTA + 25 % away from its share
        for j, u in enumerate(units):
            share = b[-1] * u / sum(units)
            assert abs((b[j + 1] - b[j]) - share) <= 1 + 0.25 * share + len(widths), (widths, b)
    assert ext.plan_fanout(4096, [4096, 1024, 1024], 148) == [0, 99, 124, 148]
    # not eligible: width not a multiple of 128, too many matrices, more matrices than CTAs
    assert ext.plan_fanout(4096, [4096, 576], 148) is None
    assert ext.plan_fanout(4096, [128] * 9, 148) is None
    assert ext.plan_fanout(4096, [128, 128, 128], 2) is None
    assert ext.plan_fanout(4096, [0, 128], 148) is None


def test_fanout_covers_every_tp_shard_of_the_bench_models():
    """The q + k + v call of bench.py's token at every tensor-parallel degree the driver runs (1, 2, 4, 8), both models: eligible
    for the one-launch path, every matrix served, no CTA group larger than its unit count."""
    import sys
    from conftest import ROOT
    sys.path.insert(0, ROOT)
    import bench
    from exllamav3_b200 import ext
    for name, cfg in bench.MODELS.items():
        for tp in (1, 2, 4, 8):
            layer, _ = bench.token_plan(cfg, tp)
            spec = {nm: (k, n, K) for (nm, k, n, K, _, _) in layer}
            (kq, nq, Kq), (kk, nk, Kk), (kv, nv, Kv) = spec["q"], spec["k"], spec["v"]
            assert kq == kk == kv and Kq == Kk == Kv
            b = ext.plan_fanout(kq, [nq, nk, nv], 148)
            assert b is not None, (name, tp)
            units = [(kq // 128) * (w // 128) for w in (nq, nk, nv)]
            assert b[-1] == min(148, sum(units)) and all(1 <= b[j + 1] - b[j] <= units[j] for j in range(3)), (name, tp, b)


def test_width_cache_is_tied_to_the_tensor_object(monkeypatch):
    """The shim's host copy of a size_n_list is trusted only for the tensor object it was read from, at the same version: a new
    tensor at a recycled address, or an in-place write, re-reads; a dead tensor's entry is withdrawn from the library."""
    import gc
    from exllamav3_b200 import ext
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    seen = []
    real = ext._lib.exl3b_register_widths
    class Spy:
        def __call__(self, key, arr, count):
            seen.append((key.value, count, [arr[i] for i in range(count)] if count else None))
            return real(key, arr, count)
    monkeypatch.setattr(ext._lib, "exl3b_register_widths", Spy())
    ext._widths_known.clear()
    t = torch.tensor([256, 128, 128], dtype=torch.int)
    key = t.data_ptr()
    ext._register_widths(t); ext._register_widths(t)
    assert seen == [(key, 3, [256, 128, 128])]                       # second call: cache hit
    t.mul_(2)
    ext._register_widths(t)
    assert seen[-1] == (key, 3, [512, 256, 256]) and seen[-2] == (key, 0, None)      # withdrawn, then re-read
    alias = t.view(-1)                                               # same address and version, ANOTHER object: not trusted
    ext._register_widths(alias)
    assert seen[-1] == (key, 3, [512, 256, 256]) and seen[-2] == (key, 0, None)
    n = len(seen)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    ext._register_widths(t)                                          # during capture: the stale entry goes, nothing is read
    assert seen[n:] == [(key, 0, None)] and key not in ext._widths_known
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    ext._register_widths(t)
    del alias, t; gc.collect()
    assert seen[-1] == (key, 0, None) and key not in ext._widths_known


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def synth(k, n, K, dev, seed):
    g = torch.Generator(device=dev); g.manual_seed(seed)
    tr = torch.randint(0, 65536, (k // 16, n // 16, 16 * K), generator=g, device=dev, dtype=torch.int32).to(torch.int16)
    sgn = lambda sz: (torch.randint(0, 2, (sz,), generator=g, device=dev) * 2 - 1).float()
    suh = (sgn(k) * (0.5 + 1.5 * torch.rand(k, generator=g, device=dev)) / k ** 0.5).half()
    svh = (sgn(n) * (0.5 + 1.5 * torch.rand(n, generator=g, device=dev))).half()
    return tr, suh, svh


def rel(got, ref):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    d = got - ref
    return np.abs(d).max() / max(np.abs(ref).max(), 1e-30), np.sqrt((d ** 2).mean()) / max(np.sqrt((ref ** 2).mean()), 1e-30)


def fan_call(ext, x3, ts, outs, K, snl=None):
    dev = x3.device
    ptr = lambda j: torch.tensor([t[j].data_ptr() for t in ts], dtype=torch.long, device=dev)
    widths = [o.shape[-1] for o in outs]
    m, k = x3.shape[1], x3.shape[2]
    C = torch.zeros((len(ts), m, max(widths)), dtype=outs[0].dtype, device=dev)
    Ah = torch.empty((len(ts), m, k), dtype=torch.half, device=dev)
    snl = torch.tensor(widths, dtype=torch.int, device=dev) if snl is None else snl
    cp = torch.tensor([o.data_ptr() for o in outs], dtype=torch.long, device=dev)
    keep = (ptr(0), ptr(1), ptr(2), C, Ah, snl, cp)
    tag = ext.exl3_mgemm(x3, keep[0], C, keep[1], Ah, keep[2], None, None, K, -1, False, True, -1, -1, 0, 1, snl, cp)
    return tag, keep


@pytest.mark.gpu
@pytest.mark.parametrize("k,widths,K", [(4096, [4096, 1024, 1024], 4), (8192, [1024, 128, 128], 4), (4096, [2048, 512, 512], 6),
                                        (512, [256, 128, 640, 128], 3), (4096, [1024, 256, 256], 4), (4096, [512, 128, 128], 4)])
@pytest.mark.parametrize("m", [1, 4])
def test_fanout_equals_separate_calls_and_oracle(cuda, k, widths, K, m):
    from exllamav3_b200 import ext
    ts = [synth(k, n, K, cuda, 900 + 7 * j + n) for j, n in enumerate(widths)]
    rng = np.random.default_rng(k + m)
    x = T(rng.standard_normal((1, m, k)).astype(np.float16), cuda)
    for fp32 in (False, True):
        dt = torch.float if fp32 else torch.half
        outs = [torch.full((m, n), float("nan"), dtype=dt, device=cuda) for n in widths]
        tag, keep = fan_call(ext, x, ts, outs, K)
        torch.cuda.synchronize()
        assert tag == ext.EXL3B_TAG_TC_I8, "a registered fan-out of mul1 matrices at <= 4 rows is one tensor-core launch"
        for (tr, suh, svh), o, n in zip(ts, outs, widths):
            y = torch.zeros((m, n), dtype=dt, device=cuda)
            t1 = ext.exl3_gemm(x[0], tr, y, suh, torch.empty((m, k), dtype=torch.half, device=cuda), svh, -1, False, True, 0)
            torch.cuda.synchronize()
            assert t1 == ext.EXL3B_TAG_TC_I8
            assert torch.isfinite(o).all()
            # same kernel, same arithmetic; only the split of a column strip over CTAs (fp32 summation order of the partial sums) differs
            mx, rms = rel(o.float().cpu().numpy(), y.float().cpu().numpy())
            assert mx <= 2e-3 and rms <= 2e-4, (n, fp32, mx, rms)
            blk = int(rng.integers(0, n // 128))
            sl = slice(blk * 128, blk * 128 + 128)
            ref = orc.exl3_gemm_f64(x[0].cpu().numpy(), tr[:, blk * 8: blk * 8 + 8].contiguous().cpu().numpy(), suh.cpu().numpy(),
                                    svh[sl].cpu().numpy(), K, 2)
            mx, rms = rel(o[:, sl].float().cpu().numpy(), ref)
            assert mx <= 4e-3 + (2.0 ** -10 if not fp32 else 0) and rms <= 2e-3, ("oracle", n, fp32, mx, rms)


@pytest.mark.gpu
def test_fanout_per_matrix_inputs_and_graph_replay(cuda):
    from exllamav3_b200 import ext
    k, widths, K, m = 1024, [512, 128, 256], 4, 2
    ts = [synth(k, n, K, cuda, 1300 + n) for n in widths]
    g = torch.Generator(device=cuda); g.manual_seed(5)
    x = torch.randn((3, m, k), generator=g, device=cuda).half()                  # one input per matrix
    outs = [torch.zeros((m, n), dtype=torch.half, device=cuda) for n in widths]
    tag, keep = fan_call(ext, x, ts, outs, K)                                  # eager first: registers the widths
    torch.cuda.synchronize()
    assert tag == ext.EXL3B_TAG_TC_I8
    first = [o.clone() for o in outs]
    for j, ((tr, suh, svh), n) in enumerate(zip(ts, widths)):
        y = torch.zeros((m, n), dtype=torch.half, device=cuda)
        ext.exl3_gemm(x[j], tr, y, suh, torch.empty((m, k), dtype=torch.half, device=cuda), svh, -1, False, True, 0)
        mx, rms = rel(first[j].float().cpu().numpy(), y.float().cpu().numpy())
        assert mx <= 2e-3 and rms <= 3e-4, (j, mx, rms)
    # captured and replayed with new inputs: same pointers, same registered widths
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            tag2 = ext.exl3_mgemm(x, keep[0], keep[3], keep[1], keep[4], keep[2], None, None, K, -1, False, True, -1, -1, 0, 1, keep[5], keep[6])
        assert tag2 == ext.EXL3B_TAG_TC_I8
        for o in outs: o.zero_()
        gr.replay(); gr.replay()
    st.synchronize()
    for o, f in zip(outs, first):
        assert torch.equal(o, f)                                               # bit-reproducible across launches


@pytest.mark.gpu
def test_fanout_fallbacks_and_rewritten_width_list(cuda):
    """A fan-out the tensor-core path does not take (more than eight matrices) and a width list rewritten in place: correct results
    through the generic path / after re-registration (the shim keys the host copy on torch's version counter)."""
    from exllamav3_b200 import ext
    k, K, m = 512, 4, 1
    g = torch.Generator(device=cuda); g.manual_seed(6)
    x = torch.randn((1, m, k), generator=g, device=cuda).half()

    def check(widths, snl=None, expect_tc=None):
        ts = [synth(k, n, K, cuda, 1700 + n) for n in widths]
        outs = [torch.zeros((m, n), dtype=torch.half, device=cuda) for n in widths]
        tag, keep = fan_call(ext, x, ts, outs, K, snl)
        torch.cuda.synchronize()
        if expect_tc is not None:
            assert (tag == ext.EXL3B_TAG_TC_I8) == expect_tc, tag
        for (tr, suh, svh), o in zip(ts, outs):
            ref = orc.exl3_gemm_f64(x[0].cpu().numpy(), tr.cpu().numpy(), suh.cpu().numpy(), svh.cpu().numpy(), K, 2)
            mx, rms = rel(o.float().cpu().numpy(), ref)
            assert mx <= 4e-3 + 2.0 ** -10 and rms <= 2e-3, (widths, mx, rms)
        return keep

    check([128, 256] * 4 + [128], expect_tc=False)       # nine matrices: generic path
    snl = torch.tensor([256, 128, 384], dtype=torch.int, device=cuda)
    check([256, 128, 384], snl, expect_tc=True)
    snl.copy_(torch.tensor([128, 384, 256], dtype=torch.int))         # same device address, new contents
    check([128, 384, 256], snl, expect_tc=True)
