"""
TEST INFRASTRUCTURE (oracle) -- builds oracle/_ref/exl3_ref_ext.so from the UNMODIFIED reference sources of the
exllamav3 checkout at $EXLLAMAV3_SOURCE, by default BASELINE.json's reference_path (nothing is copied into the repo; outputs go only to oracle/_ref/,
which is git-ignored).

This is our own short recipe (nvcc/g++ on the reference's own source files + oracle/ref_bindings.cpp); the
reference's build system (setup.py / torch JIT over ~150 TUs) is not run.  Only the EXL3 qgemm-path TUs are
compiled.  Used for: golden-vector generation on the GPU box (oracle/gen_golden_gpu.py) and the
the "reference kernel on the same GPU" timing of bench.py's qgemm section.

usage: python oracle/build_ref.py [-j N]
"""
from __future__ import annotations
import os, sys, subprocess, sysconfig, glob, hashlib
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))


def reference_root():
    """The exllamav3 checkout the oracle is built from: $EXLLAMAV3_SOURCE, else the reference_path recorded in BASELINE.json."""
    p = os.environ.get("EXLLAMAV3_SOURCE", "")
    if not p:
        try:
            import json
            p = json.load(open(os.path.join(HERE, "..", "BASELINE.json")))["reference_path"]
        except (OSError, ValueError, KeyError):
            p = ""
    return p


REF = os.path.join(reference_root(), "exllamav3", "exllamav3_ext") if reference_root() else ""
OUT = os.path.join(HERE, "_ref")
OBJ = os.path.join(OUT, "obj")
SO = os.path.join(OUT, "exl3_ref_ext.so")


def sources():
    q = os.path.join(REF, "quant")
    cu = [os.path.join(q, f) for f in (
        "exl3_gemm.cu", "exl3_gemv.cu", "exl3_gemv_int8.cu", "exl3_kernel_map.cu", "exl3_devctx.cu",
        "coop_autotune.cu", "reconstruct.cu", "hadamard.cu")]
    cu += sorted(glob.glob(os.path.join(q, "comp_units", "exl3_comp_unit_*_cb*.cu")))
    cu += sorted(glob.glob(os.path.join(q, "comp_units", "exl3_gemv_int8_inst_*.cu")))
    cu += [os.path.join(REF, f) for f in ("hgemm.cu", "graph.cu", "add.cu")]
    cpp = [os.path.join(REF, "cuda_drv.cpp"), os.path.join(HERE, "ref_bindings.cpp")]
    return cu, cpp


def flags():
    import torch
    from torch.utils import cpp_extension as ce
    inc = [REF] + ce.include_paths("cuda") + [sysconfig.get_paths()["include"]]
    incf = [f"-I{p}" for p in inc]
    common = ["-DTORCH_EXTENSION_NAME=exl3_ref_ext", "-DTORCH_API_INCLUDE_EXTENSION_H",
              "-D_GLIBCXX_USE_CXX11_ABI=" + str(int(torch._C._GLIBCXX_USE_CXX11_ABI)), "-std=c++17"]
    # flags as in the reference's ext.py:92-96 (-lineinfo -O3 --use_fast_math), arch = this box
    nvcc = ["nvcc", "-c", "-O3", "--use_fast_math", "-lineinfo",
            "-gencode", "arch=compute_90a,code=sm_90a",
            "-Xcudafe", "--diag_suppress=177", "-Xcudafe", "--diag_suppress=20012",
            "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
            "-D__CUDA_NO_HALF_OPERATORS__", "-D__CUDA_NO_HALF_CONVERSIONS__",
            "-D__CUDA_NO_BFLOAT16_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__"] + common + incf
    gxx = ["g++", "-c", "-O2", "-fPIC"] + common + incf
    lib = ce.library_paths("cuda")
    link = ["g++", "-shared", "-o", SO] + [f"-L{p}" for p in lib] + \
           [f"-Wl,-rpath,{p}" for p in lib] + \
           ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
            "-lcudart", "-lcublas", "-lcuda"]
    return nvcc, gxx, link


def obj_name(src):
    h = hashlib.md5((src + " sm_90a").encode()).hexdigest()[:6]        # the target is part of the object's identity
    return os.path.join(OBJ, os.path.basename(src).rsplit(".", 1)[0] + "_" + h + ".o")


def build(jobs=8, verbose=True):
    if not REF or not os.path.isdir(REF):
        if os.path.exists(SO):
            return SO
        raise RuntimeError("reference sources not present and no prebuilt oracle/_ref")
    os.makedirs(OBJ, exist_ok=True)
    cu, cpp = sources()
    nvcc, gxx, link = flags()
    tasks = []
    for s in cu:
        tasks.append((s, nvcc + [s, "-o", obj_name(s)]))
    for s in cpp:
        tasks.append((s, gxx + [s, "-o", obj_name(s)]))

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
                print(("ok  " if rc == 0 else "FAIL"), os.path.relpath(src, REF) if src.startswith(REF) else src, flush=True)
            if rc != 0:
                print(err)
                raise RuntimeError("compile failed: " + src)
    objs = [obj_name(s) for s in cu + cpp]
    # libcuda stub for linking without a driver
    stub = "/usr/local/cuda/lib64/stubs"
    cmd = link[:4] + objs + link[4:] + ([f"-L{stub}"] if os.path.isdir(stub) else [])
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
