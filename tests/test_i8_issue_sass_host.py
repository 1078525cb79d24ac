"""
SASS guard for the wgmma issue sequence of the int8 decode-GEMM (no GPU needed).

The decode warps issue their 8 wgmma of a k-half back to back.  When ptxas cannot tell that the warp index is warp-uniform,
it builds every wgmma descriptor in per-thread registers (64-bit add) and moves it to uniform registers with R2UR right
before the IGMMA: three to six extra instructions and an R2UR latency per wgmma, about a third of the decode warps'
instructions.  For every gemm_tc_i8 / AR / routed kernel this file asserts that no R2UR sits inside a batch of IGMMA
(between the WARPGROUP.ARRIVE that opens it and the IGMMA that commits it, `gsb0`).
"""
import os, re, subprocess, sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_wgmma_sass_host import _cuobjdump  # noqa: E402

_I8_KERNEL = re.compile(r"gemm_tc_i8_(kernel|ar_kernel|routed_kernel)I")


def batch_r2ur(sass: str):
    """{kernel: (batches, R2UR inside batches)} for the int8 decode-GEMM kernels of one object's SASS."""
    out, name = {}, None
    in_batch = False
    for ln in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            name = m.group(1) if _I8_KERNEL.search(m.group(1)) else None
            if name:
                out[name] = [0, 0]
            in_batch = False
            continue
        if name is None:
            continue
        if "WARPGROUP.ARRIVE" in ln:
            in_batch = True
            out[name][0] += 1
        elif in_batch and re.search(r"\bR2UR\b", ln):
            out[name][1] += 1
        elif in_batch and re.search(r"\bIGMMA\..*gsb0", ln):
            in_batch = False
    return {k: tuple(v) for k, v in out.items()}


@pytest.fixture(scope="module")
def objects():
    import importlib.util
    spec = importlib.util.spec_from_file_location("exl3b_build", os.path.join(ROOT, "exllamav3_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    b.build()
    return [os.path.join(b.OBJ, s + ".o") for s in ("gemm_tc_i8", "gemm_tc_i8_ar", "gemm_tc_i8_routed")]


def test_i8_wgmma_descriptors_stay_uniform(objects):
    exe = _cuobjdump()
    seen, bad = 0, []
    for o in objects:
        sass = subprocess.run([exe, "-sass", o], capture_output=True, text=True, check=True).stdout
        for name, (batches, r2ur) in batch_r2ur(sass).items():
            if batches == 0:
                continue
            seen += 1
            if r2ur:
                bad.append(f"{os.path.basename(o)} {name}: {r2ur} R2UR inside {batches} wgmma batches")
    # 16 plain <K, MR> instantiations, 8 AR, 8 routed
    assert seen >= 32, f"only {seen} int8 decode-GEMM kernels found"
    assert not bad, "\n".join(bad)


def test_parser_counts_r2ur_inside_batches_only():
    sass = """
        Function : _ZN5exl3b17gemm_tc_i8_kernelILi4ELi4EEEvNS_8TcParamsE14CUtensorMap_st
        /*0010*/  R2UR UR6, R4 ;
        /*0020*/  WARPGROUP.ARRIVE ;
        /*0030*/  IGMMA.64x8x32.U8.S8 R24, R28, gdesc[UR4], R24 ;
        /*0040*/  R2UR UR6, R16 ;
        /*0050*/  IGMMA.64x8x32.U8.S8 R24, R36, gdesc[UR4], R24, gsb0 ;
        /*0060*/  R2UR UR6, R16 ;
        Function : _ZN5exl3b24gemm_tc_i8_routed_kernelILi4EEEvNS_8TcParamsE14CUtensorMap_stNS_9RouteArgsE
        /*0010*/  WARPGROUP.ARRIVE ;
        /*0020*/  IGMMA.64x8x32.U8.S8 R24, R28, gdesc[UR4], R24 ;
        /*0030*/  IGMMA.64x8x32.U8.S8 R24, R36, gdesc[UR12], R24, gsb0 ;
        Function : _Z5otherv
        /*0010*/  WARPGROUP.ARRIVE ;
        /*0020*/  R2UR UR6, R16 ;
    """
    st = batch_r2ur(sass)
    assert st == {"_ZN5exl3b17gemm_tc_i8_kernelILi4ELi4EEEvNS_8TcParamsE14CUtensorMap_st": (1, 1),
                  "_ZN5exl3b24gemm_tc_i8_routed_kernelILi4EEEvNS_8TcParamsE14CUtensorMap_stNS_9RouteArgsE": (1, 0)}
