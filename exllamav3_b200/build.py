"""
In-tree build of libexl3b200.so (hand-written sm_90a kernels + C ABI) with nvcc.  No torch headers are involved:
the library is plain CUDA C++ behind the C ABI in include/exl3b200.h.

    python -m exllamav3_b200.build [-f] [-v]
"""
from __future__ import annotations
import os, sys, subprocess, shutil
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# EXL3B_LIB_SUFFIX=_dbg builds a second library (own object directory) next to the production one, e.g. the bring-up build
# with in-kernel timeline stamps: EXL3B_LIB_SUFFIX=_dbg EXL3B_TC_DEBUG=1 python -m exllamav3_b200.build; ext.py loads it when
# EXL3B_LIBRARY points at it.
_SUFFIX = os.environ.get("EXL3B_LIB_SUFFIX", "")
OBJ = os.path.join(HERE, "build" + _SUFFIX)
LIB = os.path.join(HERE, f"libexl3b200{_SUFFIX}.so")

SOURCES = ["api.cu", "kernels_basic.cu", "reconstruct_tc.cu", "gemm_simt.cu", "gemm_tc.cu", "gemm_tc_i8.cu", "gemm_tc_i8_ar.cu", "gemm_tc_i8_routed.cu", "chain_i8.cu", "hgemm.cu", "hgemm_tc.cu"]
HEADERS = ["common.cuh", "decode.cuh", "epilogue.cuh", "ptx.cuh", "tc_common.cuh", "gemm_tc_i8_body.cuh", "i8_math.cuh", os.path.join("..", "..", "include", "exl3b200.h")]

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]
if os.environ.get("EXL3B_TC_DEBUG", "0") != "0":       # bring-up build: in-kernel timeline stamps + experiment knobs
    NVCC_FLAGS.append("-DEXL3B_TC_DEBUG")


if os.environ.get("EXL3B_NVCC_EXTRA"):                   # extra nvcc flags, e.g. EXL3B_NVCC_EXTRA="-Xptxas -warn-spills" (+ -f)
    NVCC_FLAGS += os.environ["EXL3B_NVCC_EXTRA"].split()


def _nvcc():
    nv = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nv) and shutil.which("nvcc") is None:
        raise RuntimeError("nvcc not found")
    return nv


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    nv = _nvcc()
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + hdrs):
            jobs.append((src, obj))

    def run(job):
        src, obj = job
        cmd = [nv, "-c"] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [src, "-o", obj]
        p = subprocess.run(cmd, capture_output=True, text=True)
        return src, p.returncode, p.stdout + p.stderr

    if jobs:
        with ThreadPoolExecutor(min(8, len(jobs))) as ex:
            for src, rc, out in ex.map(run, jobs):
                if verbose or rc != 0:
                    print(out)
                if rc != 0:
                    raise RuntimeError(f"nvcc failed on {src}")
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if jobs or force or _stale(LIB, objs):
        cmd = [nv, "-shared", "-o", LIB] + objs + ["-lcudart_static", "-ldl", "-lrt", "-lpthread"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        if p.returncode != 0:
            print(p.stdout + p.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="-f" in sys.argv, verbose="-v" in sys.argv))
