"""
TEST INFRASTRUCTURE (oracle).  Static audit of the reference's modules/rmsnorm.py, modules/gated_rmsnorm.py and
modules/transformer.py (read from the checkout of oracle/build_ref.py's reference_root(), parsed, never executed or copied):
every call of `ext.rms_norm(...)`, `ext.rms_norm_res_in(...)` and `ext.gated_rms_norm(...)` with its file, class, line,
positional argument count and keyword names, recorded for tests/test_norm_host.py, which binds each one against this repo's shim.

    python oracle/gen_golden_norm_callsites.py      -> tests/golden/ref_norm_callsites.json.gz (gzip-compressed JSON)
"""
import ast, gzip, json, os, sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from build_ref import reference_root

OUT = os.path.join(ROOT, "tests", "golden", "ref_norm_callsites.json.gz")
FILES = ("rmsnorm.py", "gated_rmsnorm.py", "transformer.py")
OPS = ("rms_norm", "rms_norm_res_in", "gated_rms_norm")


def audit(src, fname):
    tree = ast.parse(src)
    sites = []
    for cls in (n for n in tree.body if isinstance(n, ast.ClassDef)):
        for n in ast.walk(cls):
            if (isinstance(n, ast.Call) and isinstance(n.func, ast.Attribute) and isinstance(n.func.value, ast.Name)
                    and n.func.value.id == "ext" and n.func.attr in OPS):
                if any(isinstance(a, ast.Starred) for a in n.args) or any(k.arg is None for k in n.keywords):
                    raise RuntimeError(f"{fname}:{n.lineno}: starred arguments are not counted")
                sites.append({"file": fname, "class": cls.name, "line": n.lineno, "name": n.func.attr,
                              "positional": len(n.args), "keywords": sorted(k.arg for k in n.keywords)})
    return sites


def main():
    sites = []
    for f in FILES:
        with open(os.path.join(reference_root(), "exllamav3", "modules", f)) as fh:
            sites += audit(fh.read(), f)
    names = {s["name"] for s in sites}
    assert names == set(OPS), f"audit found {sorted(names)}: not the expected modules"
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with gzip.GzipFile(OUT, "wb", mtime=0) as f:
        f.write(json.dumps({"files": list(FILES), "sites": sites}, indent=1, sort_keys=True).encode())
    print(f"{OUT}: {len(sites)} call sites")


if __name__ == "__main__":
    main()
