"""
SASS guard for the wgmma kernels (no GPU needed): builds the library and reads every object with `cuobjdump -sass`.

ptxas waits for each wgmma on its own (`WARPGROUP.DEPBAR.LE gsb0, 0x0` after every IGMMA/HGMMA, compile message C7510)
when a kernel that issues wgmma contains a function call: printf, a 64-bit integer division subroutine or the slow path of
the fp32 division or sqrtf.  The MMAs then run one at a time with their full latency.  For every kernel with IGMMA/HGMMA this
file asserts that it has no CALL and that no wgmma waits alone: every full wait follows a batch of at least two wgmma.
"""
import os, re, shutil, subprocess, sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

_GMMA = re.compile(r"\b[IHQ]GMMA\.")
_FULL_WAIT = re.compile(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x0\b")
_CALL = re.compile(r"\bCALL\.")


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    assert os.path.exists(exe), "cuobjdump not found"
    return exe


def kernel_stats(sass: str):
    """{kernel: (wgmma, wgmma that wait alone, calls)} of one object's SASS.  A wgmma waits alone when a full wait follows it
    and no other wgmma was issued since the previous full wait."""
    out, name, body = {}, None, []

    def close():
        if name is None:
            return
        n_mma = alone = calls = 0
        run = 0                                          # wgmma issued since the last full wait
        for ln in body:
            if _GMMA.search(ln):
                n_mma += 1
                run += 1
            elif _FULL_WAIT.search(ln):
                if run == 1:
                    alone += 1
                run = 0
            if _CALL.search(ln):
                calls += 1
        out[name] = (n_mma, alone, calls)

    for ln in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            close()
            name, body = m.group(1), []
        elif name is not None:
            body.append(ln)
    close()
    return out


@pytest.fixture(scope="module")
def objects():
    import importlib.util
    spec = importlib.util.spec_from_file_location("exl3b_build", os.path.join(ROOT, "exllamav3_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    b.build()
    return [os.path.join(b.OBJ, s.replace(".cu", ".o")) for s in b.SOURCES]


def test_wgmma_kernels_have_no_calls_and_no_per_mma_waits(objects):
    exe = _cuobjdump()
    seen = 0
    bad = []
    for o in objects:
        sass = subprocess.run([exe, "-sass", o], capture_output=True, text=True, check=True).stdout
        for name, (n_mma, alone, calls) in kernel_stats(sass).items():
            if n_mma == 0:
                continue
            seen += 1
            if calls:
                bad.append(f"{os.path.basename(o)} {name}: {calls} CALL")
            if alone:
                bad.append(f"{os.path.basename(o)} {name}: {alone} of {n_mma} wgmma wait alone")
    # the int8 decode-GEMM (16 <K, MR> instantiations), AR, routed and chain kernels, the exact path, reconstruct, hgemm
    assert seen >= 40, f"only {seen} wgmma kernels found"
    assert not bad, "\n".join(bad)


def test_parser_flags_a_serialized_kernel():
    sass = """
        Function : serialized
        /*0010*/  WARPGROUP.ARRIVE ;
        /*0020*/  IGMMA.64x8x32.U8.S8 R24, R40, gdesc[UR4], R24, gsb0 ;
        /*0030*/  WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
        /*0040*/  IGMMA.64x8x32.U8.S8 R24, R44, gdesc[UR4], R24, gsb0 ;
        /*0050*/  WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
        /*0060*/  CALL.REL.NOINC 0x2b0 ;
        Function : half_serialized
        /*0010*/  IGMMA.64x8x32.U8.S8 R24, R40, gdesc[UR4], R24 ;
        /*0020*/  IGMMA.64x8x32.U8.S8 R24, R44, gdesc[UR4], R24, gsb0 ;
        /*0030*/  WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
        /*0040*/  IGMMA.64x8x32.U8.S8 R24, R48, gdesc[UR4], R24, gsb0 ;
        /*0050*/  WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
        Function : pipelined
        /*0010*/  IGMMA.64x8x32.U8.S8 R24, R40, gdesc[UR4], R24 ;
        /*0020*/  IGMMA.64x8x32.U8.S8 R24, R44, gdesc[UR4], R24, gsb0 ;
        /*0030*/  WARPGROUP.DEPBAR.LE gsb0, 0x1 ;
        /*0040*/  HGMMA.64x128x16.F32 R24, gdesc[UR4], R24, gsb0 ;
        /*0050*/  WARPGROUP.DEPBAR.LE gsb0, 0x0 ;
    """
    st = kernel_stats(sass)
    assert st["serialized"] == (2, 2, 1)
    assert st["half_serialized"] == (3, 1, 0)
    assert st["pipelined"] == (3, 0, 0)


def test_timeline_build_keeps_wgmma_unserialized(tmp_path):
    """The bring-up build with timeline stamps (EXL3B_TC_DEBUG=1) is the one the phase profiles time, so its int8 decode-GEMM
    and chain kernels must issue the same unserialized wgmma as the production build: no CALL (a timeout printf) in them."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("exl3b_build", os.path.join(ROOT, "exllamav3_b200", "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    flags = [f for f in b.NVCC_FLAGS if not f.startswith("-DEXL3B_TC_DEBUG")] + ["-DEXL3B_TC_DEBUG=1"]
    exe = _cuobjdump()
    seen, bad = 0, []
    for s in ("gemm_tc_i8.cu", "chain_i8.cu"):
        obj = str(tmp_path / s.replace(".cu", ".o"))
        subprocess.run([b._nvcc(), "-c"] + flags + [os.path.join(b.CSRC, s), "-o", obj], check=True, capture_output=True)
        sass = subprocess.run([exe, "-sass", obj], capture_output=True, text=True, check=True).stdout
        for name, (n_mma, alone, calls) in kernel_stats(sass).items():
            if n_mma == 0:
                continue
            seen += 1
            if calls or alone:
                bad.append(f"{s} {name}: {calls} CALL, {alone} of {n_mma} wgmma wait alone")
    # 16 <K, MR> instantiations of the decode-GEMM, 9 of the chain
    assert seen >= 25, f"only {seen} wgmma kernels found"
    assert not bad, "\n".join(bad)
