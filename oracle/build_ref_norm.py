"""
TEST INFRASTRUCTURE (oracle) -- builds oracle/_ref/exl3_ref_norm.so, the reference's RMSNorm operators (rms_norm,
rms_norm_res_in, gated_rms_norm), from the UNMODIFIED norm.cu of the exllamav3 checkout that oracle/build_ref.py uses
($EXLLAMAV3_SOURCE, by default BASELINE.json's reference_path) and the stub oracle/ref_norm_bindings.cpp.  Same compiler flags
as oracle/build_ref.py; nothing is copied into the repo, outputs go only to oracle/_ref/ (git-ignored).  Used by
oracle/gen_golden_norm.py and tools/norm_bench.py.

usage: python oracle/build_ref_norm.py [-j N]
"""
from __future__ import annotations
import os, sys, subprocess, hashlib
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_ref   # noqa: E402  (reference location and compiler flags)

NAME = "exl3_ref_norm"
OBJ = os.path.join(build_ref.OUT, "obj_norm")
SO = os.path.join(build_ref.OUT, NAME + ".so")


def sources():
    cu = [os.path.join(build_ref.REF, f) for f in ("norm.cu", "graph.cu", os.path.join("quant", "exl3_devctx.cu"))]
    cpp = [os.path.join(build_ref.REF, "cuda_drv.cpp"), os.path.join(HERE, "ref_norm_bindings.cpp")]
    return cu, cpp


def obj_name(src):
    h = hashlib.md5((src + " sm_90a").encode()).hexdigest()[:6]
    return os.path.join(OBJ, os.path.basename(src).rsplit(".", 1)[0] + "_" + h + ".o")


def build(jobs=8, verbose=True):
    if not build_ref.REF or not os.path.isdir(build_ref.REF):
        if os.path.exists(SO):
            return SO
        raise RuntimeError("reference sources not present and no prebuilt " + SO)
    os.makedirs(OBJ, exist_ok=True)
    name = lambda flags: [f.replace("exl3_ref_ext", NAME) if f.startswith("-DTORCH_EXTENSION_NAME") else f for f in flags]
    nvcc, gxx, link = build_ref.flags()
    nvcc, gxx = name(nvcc), name(gxx)
    link = [SO if f == build_ref.SO else f for f in link]
    cu, cpp = sources()
    tasks = [(s, nvcc + [s, "-o", obj_name(s)]) for s in cu] + [(s, gxx + [s, "-o", obj_name(s)]) for s in cpp]

    def run(t):
        src, cmd = t
        o = cmd[-1]
        if os.path.exists(o) and os.path.getmtime(o) > os.path.getmtime(src):
            return src, 0, ""
        p = subprocess.run(cmd, capture_output=True, text=True)
        return src, p.returncode, p.stderr[-4000:]

    with ThreadPoolExecutor(jobs) as ex:
        for src, rc, err in ex.map(run, tasks):
            if verbose:
                print(("ok  " if rc == 0 else "FAIL"), os.path.basename(src), flush=True)
            if rc != 0:
                print(err)
                raise RuntimeError("compile failed: " + src)
    stub = "/usr/local/cuda/lib64/stubs"
    cmd = link[:4] + [obj_name(s) for s in cu + cpp] + link[4:] + ([f"-L{stub}"] if os.path.isdir(stub) else [])
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode != 0:
        print(p.stderr[-6000:])
        raise RuntimeError("link failed")
    return SO


if __name__ == "__main__":
    j = 8
    if "-j" in sys.argv:
        j = int(sys.argv[sys.argv.index("-j") + 1])
    print(build(j))
