"""
TEST INFRASTRUCTURE (oracle).  Runs the reference's OWN Python modules (exllamav3/modules/quant/exl3.py, modules/multilinear.py,
model/config.py; loaded unmodified from the checkout of oracle/build_ref.py's reference_root(), never copied) with their `ext`
bound to this repo's shim, and records what tests/test_reference_callsites.py compares this repo's mirror against:

  * linear      the extension calls (op name, argument shapes / values, keyword names) LinearEXL3.forward issues per input
                shape and parameter set, its output shape / dtype, and its dispatch constants
  * slicing     the same for wide outputs with MAX_RECONSTRUCT_SLICE_N = 256
  * multilinear MultiLinear's pointer tables, as (matrix index, tensor name) per entry, and its fields
  * audit       every `ext.<op>(...)` call site of the qgemm surface in the reference's Python tree (file, line, positional count,
                keyword names)
  * use_mgemm   InferParams.use_mgemm (model/config.py:48-64) for K 1..8, narrow / wide outputs, mul1 or not, with the int8
                GEMV bound the extension reports set to 0 (this shim) and 6 (the reference's extension on Hopper)
  * tp          LinearEXL3.tp_import_split shards (sha256 of trellis / suh / svh / bias, fields) for every split of world 3

    python oracle/gen_golden_callsites.py          -> tests/golden/ref_callsites.json.gz (gzip-compressed JSON)
"""
import ast, gzip, importlib.util, inspect, json, os, sys, types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, HERE)
import torch
import refstubs
from build_ref import reference_root

PKG = os.path.join(reference_root(), "exllamav3")
OUT = os.path.join(ROOT, "tests", "golden", "ref_callsites.json.gz")


def stub(name, **attrs):
    m = types.ModuleType(name)
    m.__path__ = []
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(PKG, *rel.split("/")))
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


def load_exl3(ext, calls):
    def wrap(name):
        real = getattr(ext, name)
        sig = inspect.signature(real)

        def f(*a, **kw):
            sig.bind(*a, **kw)                                    # the reference's argument list fits the shim's signature
            calls.append([name, [refstubs.encode(t) for t in a], sorted(kw)])
            return 210
        return f

    for name in refstubs.RECORDED_OPS:
        setattr(ext, name, wrap(name))

    class Config: pass
    stub("exllamav3"); stub("exllamav3.model")
    stub("exllamav3.model.config", Config=Config, NullConfig=refstubs.NullConfig)
    stub("exllamav3.ext", exllamav3_ext=ext)
    stub("exllamav3.util", profile_opt=lambda f: f)
    stub("exllamav3.util.tensor", g_tensor_cache=refstubs.g_tensor_cache)
    stub("exllamav3.modules"); stub("exllamav3.modules.quant"); stub("exllamav3.modules.quant.exl3_lib")
    stub("exllamav3.modules.quant.exl3_lib.quantize", preapply_had_l=refstubs.preapply_had_l, preapply_had_r=refstubs.preapply_had_r,
         had_k=128, had_n=128)
    return load("exllamav3.modules.quant.exl3", "modules/quant/exl3.py")


def main():
    from exllamav3_b200 import ext
    out = {}
    calls = []
    ref = load_exl3(ext, calls)
    k, n = 256, 384
    lin = ref.LinearEXL3(None, k, n, key="q", **refstubs.tensors(k, n))
    out["linear"] = {"AUTO_RECONSTRUCT_THRESHOLD": ref.AUTO_RECONSTRUCT_THRESHOLD, "MAX_RECONSTRUCT_SLICE_N": ref.MAX_RECONSTRUCT_SLICE_N,
                     "bc_type": type(lin.bc).__name__, "K": lin.K, "mcg": bool(lin.mcg), "mul1": bool(lin.mul1), "cases": []}
    for shape, params, odt in refstubs.LINEAR_CASES:
        calls.clear()
        y = lin.forward(torch.zeros(shape, dtype=torch.half), params, getattr(torch, odt) if odt else None)
        out["linear"]["cases"].append({"calls": list(calls), "y_shape": list(y.shape), "y_dtype": str(y.dtype)})

    ref.MAX_RECONSTRUCT_SLICE_N = 256
    k2, n2 = 128, 640
    lin2 = ref.LinearEXL3(None, k2, n2, **refstubs.tensors(k2, n2))
    out["slicing"] = []
    for rows in refstubs.SLICING_ROWS:
        calls.clear(); lin2.forward(torch.zeros((rows, k2), dtype=torch.half), {})
        out["slicing"].append(list(calls))
    ref.MAX_RECONSTRUCT_SLICE_N = out["linear"]["MAX_RECONSTRUCT_SLICE_N"]

    # multilinear tables over three LinearEXL3 objects of the reference
    src = open(os.path.join(PKG, "modules", "multilinear.py")).read()
    ns = {}
    exec(compile(src.replace("from . import Linear", "Linear = object"), "multilinear_ref", "exec"), ns)     # executed in memory
    km, nm = 128, 256
    inners = [ref.LinearEXL3(None, km, nm, **refstubs.tensors(km, nm)) for _ in range(3)]
    for i in inners:
        i.quant_type = "exl3"

    class Lin:
        def __init__(self, inner):
            self.inner, self.quant_type, self.softcap, self.post_scale = inner, "exl3", 0.0, 1.0
            self.in_features, self.out_features = inner.in_features, inner.out_features
    ml = ns["MultiLinear"]("cpu", [Lin(i) for i in inners])
    where = {}
    for j, i in enumerate(inners):
        for a in ("trellis", "suh", "svh"):
            where[getattr(i, a).data_ptr()] = [j, a]
    out["multilinear"] = {"tables": {a: [where[int(p)] for p in getattr(ml, a).tolist()] for a in ("ptrs_trellis", "ptrs_suh", "ptrs_svh")},
                          "dtype": str(ml.ptrs_trellis.dtype), "fields": [ml.K, bool(ml.mcg), bool(ml.mul1), ml.in_features, ml.out_features]}

    # static audit of the reference's call sites of the qgemm surface
    sites = []
    for root, _, names in os.walk(os.path.dirname(PKG)):
        if "exllamav3_ext" in root:
            continue
        for nmf in sorted(names):
            if not nmf.endswith(".py"):
                continue
            path = os.path.join(root, nmf)
            try:
                tree = ast.parse(open(path).read())
            except SyntaxError:
                continue
            for node in ast.walk(tree):
                if (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr in refstubs.AUDIT_OPS
                        and isinstance(node.func.value, ast.Name) and node.func.value.id == "ext"):
                    if any(isinstance(a, ast.Starred) for a in node.args) or any(kw.arg is None for kw in node.keywords):
                        continue
                    sites.append([os.path.relpath(path, os.path.dirname(PKG)), node.lineno, node.func.attr, len(node.args),
                                  sorted(kw.arg for kw in node.keywords)])
    out["audit"] = sorted(sites)

    # the reference's own use_mgemm policy
    stub("exllamav3"); stub("exllamav3.model"); stub("exllamav3.util")
    stub("exllamav3.util.rope", RopeSettings=object, RopeStyle=object)
    stub("exllamav3.loader", SafetensorsCollection=object)
    stub("exllamav3.util.file", read_dict=None, no_value=None, no_default=None)
    fake = types.SimpleNamespace()
    stub("exllamav3.ext", exllamav3_ext=fake)
    for v in ("EXL3_INT8_GEMV", "EXL3_MGEMM_K_THRESHOLD", "EXL3_MGEMM_N_THRESHOLD"):
        os.environ.pop(v, None)
    cfg = load("exllamav3.model.config", "model/config.py")
    ip = cfg.InferParams()
    out["use_mgemm"] = []
    for max_k in (0, 6):
        fake.exl3_gemv_int8_max_k = lambda dev, mk=max_k: mk
        for K in range(1, 9):
            for nn in (1024, 14336):
                for mul1 in (True, False):
                    out["use_mgemm"].append([max_k, K, nn, mul1, bool(ip.use_mgemm(K, nn, mul1=mul1, device="cuda:0"))])

    # tensor-parallel shards of the reference's tp_export / tp_import_split
    calls2 = []
    ref = load_exl3(ext, calls2)

    class Producer:
        def send(self, t): return t

    class Consumer:
        def recv(self, t, cuda=False, slice_dim=None, first=None, last=None):
            if t is None:
                return None
            return t if slice_dim is None else t.narrow(slice_dim, first, last - first).contiguous()

    from exllamav3_b200 import tp
    kt, nt = 512, 768
    tens, bias = refstubs.tp_tensors(kt, nt)
    full = ref.LinearEXL3(None, kt, nt, bias=bias, out_dtype=torch.float, **tens)
    exported = full.tp_export(None, Producer())
    ctx = {"consumer": Consumer(), "device": "cpu"}
    world = 3
    splits = [[True, a, b] for (a, b) in tp.split_ranges(nt, world)] + [[False, a, b] for (a, b) in tp.split_ranges(kt, world)] + [None]
    out["tp"] = {"inputs": {a: refstubs.digest(tens[a]) for a in ("trellis", "suh", "svh")} | {"bias": refstubs.digest(bias)}, "shards": []}
    for split in splits:
        r = ref.LinearEXL3.tp_import_split(ctx, exported, None, tuple(split) if split else None)
        out["tp"]["shards"].append({"split": split, "fields": [r.in_features, r.out_features, r.K, bool(r.mcg), bool(r.mul1), str(r.out_dtype)],
                                    "trellis": refstubs.digest(r.trellis), "suh": refstubs.digest(r.suh), "svh": refstubs.digest(r.svh),
                                    "bias": refstubs.digest(r.bias)})

    with open(OUT, "wb") as f:
        f.write(gzip.compress(json.dumps(out, sort_keys=True, separators=(",", ":")).encode(), mtime=0))
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
