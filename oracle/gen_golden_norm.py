"""
TEST INFRASTRUCTURE (oracle).  Runs the reference's RMSNorm operators (oracle/_ref/exl3_ref_norm.so, built by
oracle/build_ref_norm.py) on seeded inputs on the GPU and writes the inputs and the reference's outputs to
tests/golden/ref_norm.npz, for tests/test_norm_gpu.py.

Cases: every one of rms_norm's 24 dtype combinations (x, w, y, residual mode, r) with w present and constant_bias 0, w present
and constant_bias 1, and w absent; constant_scale 1 or 0.75 alternating; dim in {4, 128, 2880, 4096, 5120, 8192} and rows in
{1, 3, 8, 257}: dims 2880 to 8192 with one row once each, the other cases dim 4 at up to 257 rows and dim 128 at up to 3, so the
file stays small.  Then every gated_rms_norm dtype
combination (w, y, g) with gate_first off and on, constant_bias 0 or 1, w_groups 1 or 2.
Per case i the archive holds i_x, i_w (absent when w is None), i_y0 (RES_POST: y before the call, else y starts zeroed), i_r0 (RES_IN),
i_g (gated), and the reference's i_y and i_r (RES_IN's written-back residual); bf16 arrays are stored as their uint16 bits.  The
key `meta` is a JSON list of the cases' parameters.

    python oracle/gen_golden_norm.py [out.npz]      (on a GPU machine, after build(); default tests/golden/ref_norm.npz)
"""
import io, itertools, json, os, sys
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "ref_norm.npz")

DT = {"fp16": torch.half, "fp32": torch.float, "bf16": torch.bfloat16}
DIMS = (4, 128, 2880, 4096, 5120, 8192)
ROWS = (1, 3, 8, 257)


def rms_cases():
    """(x, w, y, mode, r) of the reference's table (exllamav3_ext/norm.cu:380-404), r = x's dtype outside RES_IN"""
    out = []
    for mode in ("none", "post", "in"):
        for tx, tw in itertools.product(("fp16", "fp32"), ("fp16", "bf16")):
            if mode == "in":
                out += [(tx, tw, "fp16", mode, tr) for tr in ("fp16", "fp32")]
            else:
                out += [(tx, tw, ty, mode, tx) for ty in ("fp16", "fp32")]
    return out


def gated_cases():
    return list(itertools.product(("fp32", "bf16"), ("fp16", "fp32"), ("bf16", "fp32")))


def _shape(k):
    """(dim, rows) of case k: the model widths (dim >= 2880, one row) once each, at cases spread over the table; the other cases
    cycle through the short rows"""
    big = [(d, 1) for d in DIMS if d > 128]
    if k % 22 == 5 and k // 22 < len(big):
        return big[k // 22]
    small = [(d, r) for d in DIMS if d <= 128 for r in ROWS if d * r <= 1028 and (d, r) != (128, 8)]
    return small[k % len(small)]


def case_list():
    cases = []
    k = 0
    for combo in rms_cases():
        for wkind in ("w", "w+1", "none"):
            dim, rows = _shape(k)
            tx, tw, ty, mode, tr = combo
            cases.append({"op": "rms_norm", "x": tx, "w": None if wkind == "none" else tw, "y": ty, "mode": mode, "r": tr,
                          "bias": 1.0 if wkind == "w+1" else 0.0, "scale": 0.75 if k % 2 else 1.0, "eps": 1e-6,
                          "dim": dim, "rows": rows, "seed": 1000 + k})
            k += 1
    for j, (tw, ty, tg) in enumerate(gated_cases()):
        for gate_first in (False, True):
            dim, rows = _shape(k)
            groups = 2 if j % 2 else 1
            cases.append({"op": "gated_rms_norm", "x": "bf16", "w": tw, "y": ty, "g": tg, "gate_first": gate_first,
                          "bias": float(j % 2 == 0 and gate_first), "eps": 1e-5, "w_groups": groups,
                          "dim": dim, "rows": rows, "seed": 1000 + k})
            k += 1
    return cases


def make_inputs(c):
    """The case's input tensors (CPU), from its seed: x with rows of different scales, w around 1 (around 0 when a bias of 1 is
    added, as the models that use one store it), the old y / r / g as randn"""
    gen = torch.Generator().manual_seed(c["seed"])
    rows, dim = c["rows"], c["dim"]
    rs = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    t = {"x": (rs(rows, dim) * torch.exp2(rs(rows, 1).mul(2).round())).to(DT[c["x"]])}
    if c["w"] is not None:
        groups = c.get("w_groups", 1)
        w = rs(groups * dim) * 0.1 + (0.0 if c["bias"] else 1.0)
        t["w"] = w.to(DT[c["w"]])
    if c["op"] == "rms_norm":
        if c["mode"] == "post":
            t["y0"] = rs(rows, dim).to(DT[c["y"]])
        if c["mode"] == "in":
            t["r0"] = (rs(rows, dim) * 4).to(DT[c["r"]])
    else:
        t["g"] = (rs(rows, dim) * 3).to(DT[c["g"]])
    return t


def to_np(t: torch.Tensor) -> np.ndarray:
    return t.view(torch.int16).numpy().view(np.uint16) if t.dtype == torch.bfloat16 else t.numpy()


def from_np(a: np.ndarray, dtype: str) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.view(torch.bfloat16) if dtype == "bf16" else t


def run(mod, c, t, dev):
    """One call of `mod` (the reference's extension or exllamav3_b200.ext) on the case; returns (y, r) on the CPU"""
    d = {k: v.clone().to(dev) for k, v in t.items()}
    y = d["y0"] if "y0" in d else torch.zeros(c["rows"], c["dim"], dtype=DT[c["y"]], device=dev)
    r, w = d.get("r0"), d.get("w")
    if c["op"] == "rms_norm":
        if c["mode"] == "in":
            mod.rms_norm_res_in(d["x"], w, y, r, c["eps"], c["bias"], c["scale"])
        else:
            mod.rms_norm(d["x"], w, y, c["eps"], c["bias"], c["scale"], False, c["mode"] == "post")
    else:
        mod.gated_rms_norm(d["x"], w, y, d["g"], c["eps"], c["bias"], c["w_groups"], c["gate_first"])
    torch.cuda.synchronize()
    return y.cpu(), None if r is None else r.cpu()


def main(out=OUT):
    sys.path.insert(0, os.path.join(HERE, "_ref"))
    import exl3_ref_norm as ref
    dev = torch.device("cuda:0")
    cases = case_list()
    arrays = {"meta": np.frombuffer(json.dumps(cases).encode(), dtype=np.uint8)}
    for i, c in enumerate(cases):
        t = make_inputs(c)
        y, r = run(ref, c, t, dev)
        for k, v in t.items():
            arrays[f"{i}_{k}"] = to_np(v)
        arrays[f"{i}_y"] = to_np(y)
        if r is not None:
            arrays[f"{i}_r"] = to_np(r)
    buf = io.BytesIO()
    np.savez_compressed(buf, **arrays)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "wb") as f:
        f.write(buf.getvalue())
    print(f"{out}: {len(cases)} cases, {len(buf.getvalue()) / 1e6:.2f} MB")


if __name__ == "__main__":
    main(*sys.argv[1:])
