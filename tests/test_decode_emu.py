"""
The library's per-thread trellis decode (exllamav3_b200/csrc/decode.cuh: compile-time bit-window extraction + codebooks, the
code every CUDA kernel here runs per weight) built for the HOST with g++ (tests/emu/decode_emu.cpp restates the few PTX
instructions) and checked against the oracle without a GPU:

  * decode16<K, cb, half>   -- 16 k-rows of one tile column as fp16 pairs: must equal the oracle's decoded tile bit for bit
    (= reconstruct(), pinned to the reference's own kernels by tests/golden/ref_gpu.npz), for every K, codebook, chunk, half;
  * decode16_i8<K, half>    -- the same column as raw products state * 0x83DCD12D (operand of the int8 tensor-core path):
    must equal unpack_states() * multiplier mod 2^32, and its byte sums must reproduce the mul1 codebook values;
  * strip_col               -- thread -> column mapping of a 128-column strip is a permutation.

This pins the device header's arithmetic on the CPU (so a change to the extraction can be vetted before it reaches a GPU);
the GPU tests remain the proof that the compiled kernels do the same.
"""
import ctypes, os, subprocess, shutil
import numpy as np
import pytest
from conftest import ROOT
from oracle import exl3_oracle as orc

SRC = os.path.join(ROOT, "tests", "emu", "decode_emu.cpp")
HDR = os.path.join(ROOT, "exllamav3_b200", "csrc", "decode.cuh")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    gxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else shutil.which("g++")
    assert gxx, "g++ not found"
    so = str(tmp_path_factory.mktemp("emu") / "libdecode_emu.so")
    subprocess.check_call([gxx, "-O1", "-std=c++17", "-fPIC", "-shared", "-o", so, SRC])
    lib = ctypes.CDLL(so)
    u32p = ctypes.POINTER(ctypes.c_uint32)
    lib.emu_load_chunk.argtypes = [ctypes.c_int, u32p, ctypes.c_int, u32p]
    lib.emu_decode16.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, u32p, u32p]
    lib.emu_decode16_i8.argtypes = [ctypes.c_int, ctypes.c_int, u32p, u32p]
    lib.emu_strip_col.argtypes = [ctypes.c_int, ctypes.c_int]
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32))


def _tiles(K, count, seed):
    rng = np.random.default_rng(seed)
    tr = rng.integers(0, 65536, size=(count, 16 * K), dtype=np.uint16)
    tr[0] = 0; tr[1] = 0xffff                                  # all-zero / all-one streams
    if count > 2:
        tr[2] = np.arange(16 * K, dtype=np.uint16) * 4099       # a ramp: every window differs
    return tr


@pytest.mark.parametrize("K", range(1, 9))
def test_decode16_matches_oracle_tile_bit_exactly(emu, K):
    tr = _tiles(K, 6, seed=100 + K)
    for cb in range(3):
        ref = orc.decode_tiles(tr, K, cb).view(np.uint16)                    # (tiles, 16 k, 16 n)
        for t in range(tr.shape[0]):
            words = np.ascontiguousarray(tr[t]).view(np.uint32).copy()
            for chunk in range(8):
                w = np.zeros(K + 1, dtype=np.uint32)
                assert emu.emu_load_chunk(K, _p(words), chunk, _p(w)) == 0
                assert w[0] == words[(chunk * K - 1) % (8 * K)] and (w[1:] == words[chunk * K:(chunk + 1) * K]).all()
                for half in range(2):
                    out = np.zeros(8, dtype=np.uint32)
                    assert emu.emu_decode16(K, cb, half, _p(w), _p(out)) == 0
                    col = out.view(np.uint16)                                # k = 0..15 in order (pair j = k 2j, 2j+1)
                    assert (col == ref[t, :, chunk + 8 * half]).all(), (K, cb, t, chunk, half)


@pytest.mark.parametrize("K", range(1, 9))
def test_decode16_i8_products_and_byte_sums(emu, K):
    tr = _tiles(K, 6, seed=200 + K)
    states = orc.unpack_states(tr, K).astype(np.uint64)                      # (tiles, 256) in stream order
    perm = orc.tensor_core_perm()                                            # position -> k * 16 + n
    st_kn = np.zeros((tr.shape[0], 256), dtype=np.uint64)
    st_kn[:, perm] = states
    st_kn = st_kn.reshape(-1, 16, 16)
    prod_ref = (st_kn * np.uint64(0x83DCD12D)) & np.uint64(0xffffffff)
    vals_ref = orc.decode_tiles(tr, K, 2).astype(np.float64)                 # mul1 codebook values (fp16-rounded)
    k_inv = float(np.uint16(0x1eee).view(np.float16)); k_bias = float(np.uint16(0xc931).view(np.float16))
    for t in range(tr.shape[0]):
        words = np.ascontiguousarray(tr[t]).view(np.uint32).copy()
        for chunk in range(8):
            w = np.zeros(K + 1, dtype=np.uint32)
            emu.emu_load_chunk(K, _p(words), chunk, _p(w))
            for half in range(2):
                out = np.zeros(16, dtype=np.uint32)
                assert emu.emu_decode16_i8(K, half, _p(w), _p(out)) == 0
                n = chunk + 8 * half
                assert (out.astype(np.uint64) == prod_ref[t, :, n]).all(), (K, t, chunk, half)
                # the tensor core sums the four bytes: k_inv * (1024 + bytesum) + k_bias is the codebook value before its
                # fp16 rounding (codebook.cuh:77-89) -> within half an fp16 ulp of the oracle's rounded value
                bs = sum(((out >> (8 * i)) & 0xff).astype(np.float64) for i in range(4))
                full = k_inv * (1024.0 + bs) + k_bias
                assert (np.abs(full - vals_ref[t, :, n]) <= 2.0 ** -11 * np.maximum(np.abs(full), 2.0 ** -14) + 1e-12).all()


def test_branch_free_k4_decode_equals_the_templated_one(emu):
    """decode16_i8_k4_rt (half as a run-time span shift, one funnel shift per four weights) == decode16_i8<4, half>."""
    emu.emu_decode16_i8_k4_rt.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32)]
    rng = np.random.default_rng(7)
    for it in range(2000):
        w = rng.integers(0, 2 ** 32, size=5, dtype=np.uint64).astype(np.uint32)
        if it == 0: w[:] = 0
        if it == 1: w[:] = 0xffffffff
        for half in range(2):
            a = np.zeros(16, dtype=np.uint32); b = np.zeros(16, dtype=np.uint32)
            emu.emu_decode16_i8(4, half, _p(w), _p(a))
            emu.emu_decode16_i8_k4_rt(half, _p(w), _p(b))
            assert (a == b).all()


def test_strip_column_mapping_is_a_permutation(emu):
    cols = sorted(emu.emu_strip_col(q, lane) for q in range(4) for lane in range(32))
    assert cols == list(range(128))
    # lane quarter q: half = q & 1, tiles 4 * (q >> 1) ..; chunk = lane & 7
    assert emu.emu_strip_col(0, 0) == 0 and emu.emu_strip_col(1, 0) == 8 and emu.emu_strip_col(2, 0) == 64 and emu.emu_strip_col(3, 31) == 127


def test_emulation_builds_from_the_library_header():
    # the emulation must compile the product header itself, not a copy
    src = open(SRC).read()
    assert '#include "../../exllamav3_b200/csrc/decode.cuh"' in src
    assert "EXL3B_HOST_EMU" in open(HDR).read()


@pytest.mark.parametrize("K", [2, 4, 6])
def test_i8_path_arithmetic_from_device_headers_matches_oracle_model(emu, K):
    """
    The int8 tensor-core path's arithmetic, run on the host FROM THE DEVICE HEADERS (csrc/i8_math.cuh digits + reassembly,
    csrc/decode.cuh product words, byte sums standing in for the u8 x s8 wgmma), against the oracle's independent fp64
    model of the path (oracle.exl3_gemm_i8_model): same result to fp32 round-off.  Also asserts what the kernel relies on:
    digits replicated over four bytes, hi in [-127, 127], s32 accumulators never overflow at these sizes.
    """
    emu.emu_i8_row.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.c_int,
                               ctypes.POINTER(ctypes.c_float)]
    k, n = 512, 256
    tr, suh, svh, x = orc.make_synthetic(k, n, K, seed=11 * K, m=3)
    xh = orc.had_r_128(x, pre_scale=suh).astype(np.float32)                  # bit-exact fp16 transformed activations
    tiles = np.ascontiguousarray(tr).view(np.uint16).reshape(k // 16, n // 16, 16 * K).copy().view(np.uint32)
    want = orc.exl3_gemm_i8_model(x, tr, suh, svh, K)                        # (m, n) fp64, after output Hadamard and svh
    H = orc.hadamard_matrix_128() * float(np.float32(0.088388347648))
    for r in range(x.shape[0]):
        acc = np.zeros(n, dtype=np.float32)
        row = np.ascontiguousarray(xh[r])
        rc = emu.emu_i8_row(K, tiles.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), row.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                            k, n, acc.ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
        assert rc == 0, rc
        y = (acc.astype(np.float64).reshape(n // 128, 128) @ H).reshape(n) * svh.astype(np.float64)
        err = np.abs(y - want[r]).max() / np.abs(want[r]).max()
        assert err < 2e-6, (K, r, err)
    # an all-zero row quantises to zero digits and a zero output
    z = np.zeros(k, dtype=np.float32); acc = np.ones(n, dtype=np.float32)
    assert emu.emu_i8_row(K, tiles.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), z.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), k, n,
                          acc.ctypes.data_as(ctypes.POINTER(ctypes.c_float))) == 0 and (acc == 0).all()
