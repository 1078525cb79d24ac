"""
The int8 path's scale divisions without the compiler's division subroutine (i8_qmax_over / i8_over_qmax in
exllamav3_b200/csrc/i8_math.cuh, used by the decode-GEMM's digit warps and epilogue and by the chain kernel) must round
exactly like IEEE division, and the chain kernel's square root (i8_sqrt_rn) like IEEE sqrt.  Built for the host with g++
from the library header (tests/emu/i8_div_emu.cpp) and compared bit for bit with the host's IEEE operations: the divisions
over every float in [2^-24, 2^20) (all positive fp16 magnitudes, the row maxima, and the chain's block-norm bounds), the
square root over every float in [2^-48, 2^40] (the chain's nonzero sums of squares).
"""
import ctypes, os, shutil, subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "emu", "i8_div_emu.cpp")


def _build(src, so):
    gxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else shutil.which("g++")
    assert gxx, "g++ not found"
    subprocess.check_call([gxx, "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, src])
    lib = ctypes.CDLL(so)
    for fn in (lib.emu_check_divisions, lib.emu_check_sqrt):
        fn.restype = ctypes.c_longlong
        fn.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32)]
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _build(SRC, str(tmp_path_factory.mktemp("divemu") / "libi8_div_emu.so"))


def _bits(x):
    return int(np.float32(x).view(np.uint32))


def _check(emu, lo, hi, step=1, fn="emu_check_divisions"):
    first = ctypes.c_uint32()
    bad = getattr(emu, fn)(lo, hi, step, ctypes.byref(first))
    return bad, first.value


def _every_float(emu, lo, hi, fn):
    # one binade per task: ctypes releases the GIL, so the binades run in parallel
    edges = list(range(_bits(lo), _bits(hi), 1 << 23)) + [_bits(hi)]
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        res = list(ex.map(lambda ab: _check(emu, ab[0], ab[1], fn=fn), zip(edges[:-1], edges[1:])))
    return [(hex(first), n) for (n, first) in res if n]


def test_every_fp16_magnitude(emu):
    mags = np.arange(1, 0x7c00, dtype=np.uint16).view(np.float16).astype(np.float32)   # positive finite fp16
    for b in mags.view(np.uint32):
        assert _check(emu, int(b), int(b) + 1) == (0, 0), f"mismatch at {float(np.uint32(b).view(np.float32))!r}"


def test_every_float_of_the_range(emu):
    bad = _every_float(emu, 2.0 ** -24, 2.0 ** 20, "emu_check_divisions")
    assert not bad, f"mismatches (first bit pattern, count per binade): {bad}"


def test_sqrt_every_float_of_the_range(emu):
    # the chain kernel's block norms: nonzero sums of squares of fp16 values lie in [2^-48, 2^40]
    bad = _every_float(emu, 2.0 ** -48, 2.0 ** 40, "emu_check_sqrt")
    assert not bad, f"mismatches (first bit pattern, count per binade): {bad}"


def test_checker_detects_a_wrong_rounding(emu, tmp_path):
    # the same check with i8_over_qmax off by one ulp must fail: the comparison really looks at the bits
    src = open(SRC).read().replace("i8_f32_to_bits(i8_over_qmax(x))", "(i8_f32_to_bits(i8_over_qmax(x)) + 1u)")
    p = tmp_path / "broken.cpp"
    p.write_text(src.replace('"../../exllamav3_b200', '"' + os.path.join(ROOT, "exllamav3_b200").replace("\\", "/")))
    lib = _build(str(p), str(tmp_path / "broken.so"))
    first = ctypes.c_uint32()
    assert lib.emu_check_divisions(_bits(1.0), _bits(1.0) + 16, 1, ctypes.byref(first)) == 16
