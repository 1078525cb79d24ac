"""
TEST INFRASTRUCTURE (oracle).  Static audit of the reference's modules/mlp.py (read from the checkout of oracle/build_ref.py's
reference_root(), parsed, never executed or copied): every place where the MLP modules reach the extension's block and activation
surface, recorded for tests/test_mlp_callsites_host.py, which binds each one against this repo's shim.

  * sites         every `ext.BC_GatedMLP(...)`, `ext.BC_MLP(...)`, `ext.silu_mul(...)` / `gelu_mul` / `relu2_mul` call: class,
                  line, positional argument count (a starred generator over a list literal counts its elements) and keyword names
  * act_refs      every `ext.silu_mul` / `gelu_mul` / `relu2_mul` referenced without a call (bound as GatedMLP.activation_fn_call)
  * act_calls     every `self.activation_fn_call(...)` call inside GatedMLP: line, positional count, keyword names
  * MAX_BSZN      the module constant (tokens per BC_GatedMLP.run_bszN call)

    python oracle/gen_golden_mlp_callsites.py      -> tests/golden/ref_mlp_callsites.json.gz (gzip-compressed JSON)
"""
import ast, gzip, json, os, sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from build_ref import reference_root

OUT = os.path.join(ROOT, "tests", "golden", "ref_mlp_callsites.json.gz")
BLOCKS = ("BC_GatedMLP", "BC_MLP")
ACTS = ("silu_mul", "gelu_mul", "relu2_mul")


def _ext_attr(node):
    return isinstance(node, ast.Attribute) and isinstance(node.value, ast.Name) and node.value.id == "ext" and node.attr


def _list_lengths(func):
    """target source -> element count of the list literals assigned to it inside `func`"""
    out = {}
    for n in ast.walk(func):
        if isinstance(n, ast.Assign) and isinstance(n.value, ast.List):
            for t in n.targets:
                out[ast.unparse(t)] = len(n.value.elts)
    return out


def _positional(call, lengths):
    count = 0
    for a in call.args:
        if isinstance(a, ast.Starred):
            v = a.value
            src = ast.unparse(v.generators[0].iter) if isinstance(v, ast.GeneratorExp) else ast.unparse(v)
            if src not in lengths:
                raise RuntimeError(f"line {call.lineno}: cannot count starred argument {ast.unparse(a)}")
            count += lengths[src]
        else:
            count += 1
    return count


def audit(src):
    tree = ast.parse(src)
    out = {"sites": [], "act_refs": [], "act_calls": [], "MAX_BSZN": None}
    for n in tree.body:
        if isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "MAX_BSZN" for t in n.targets):
            out["MAX_BSZN"] = ast.literal_eval(n.value)
    called = set()
    for cls in (n for n in tree.body if isinstance(n, ast.ClassDef)):
        for func in (n for n in cls.body if isinstance(n, ast.FunctionDef)):
            lengths = _list_lengths(func)
            for n in ast.walk(func):
                if isinstance(n, ast.Call):
                    name = _ext_attr(n.func)
                    if name in BLOCKS + ACTS:
                        called.add(id(n.func))
                        out["sites"].append({"class": cls.name, "line": n.lineno, "name": name, "positional": _positional(n, lengths),
                                             "keywords": sorted(k.arg for k in n.keywords)})
                    f = n.func
                    if (cls.name == "GatedMLP" and isinstance(f, ast.Attribute) and f.attr == "activation_fn_call"
                            and isinstance(f.value, ast.Name) and f.value.id == "self"):
                        out["act_calls"].append({"line": n.lineno, "positional": _positional(n, lengths),
                                                 "keywords": sorted(k.arg for k in n.keywords)})
            for n in ast.walk(func):
                name = _ext_attr(n)
                if name in ACTS and id(n) not in called:
                    out["act_refs"].append({"class": cls.name, "line": n.lineno, "name": name})
    return out


def main():
    path = os.path.join(reference_root(), "exllamav3", "modules", "mlp.py")
    with open(path) as f:
        out = audit(f.read())
    assert out["MAX_BSZN"] is not None and out["sites"] and out["act_calls"], "audit found nothing: not the expected mlp.py"
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with gzip.GzipFile(OUT, "wb", mtime=0) as f:
        f.write(json.dumps(out, indent=1, sort_keys=True).encode())
    print(f"{OUT}: {len(out['sites'])} call sites, {len(out['act_refs'])} activation references, "
          f"{len(out['act_calls'])} activation calls, MAX_BSZN = {out['MAX_BSZN']}")


if __name__ == "__main__":
    main()
