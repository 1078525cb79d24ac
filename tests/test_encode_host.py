"""
Trellis encoder, host side: the fp64 dynamic program oracle.encode_oracle.viterbi_anchored against brute force on reduced trellises,
the oracle's pack_states / unpack_states on valid tail-biting sequences, and the argument checks of the C ABI and of
ext.quantize_tiles / ext.pack_trellis, which all fire before anything touches a device.
"""
import itertools
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc
from oracle import encode_oracle as enc
from exllamav3_b200 import ext


def brute_force(x, K, values, bits, e):
    """min over all tail-biting sequences with wrap overlap e (s[0] >> K == e == s[L-1] & mask), fp64."""
    L, Kr = len(x), bits - K
    mask = (1 << Kr) - 1
    best, arg = np.inf, None
    for low in range(1 << K):
        s0 = (e << K) | low
        for syms in itertools.product(range(1 << K), repeat=L - 1):
            seq = [s0]
            for q in syms:
                seq.append(((seq[-1] << K) | q) & ((1 << bits) - 1))
            if seq[-1] & mask != e:
                continue
            c = float(((np.asarray(x, np.float64) - values[seq]) ** 2).sum())
            if c < best:
                best, arg = c, seq
    return best, arg


@pytest.mark.parametrize("K,L", [(1, 6), (1, 8), (2, 6), (2, 7)])
def test_viterbi_anchored_matches_brute_force(K, L):
    bits = 6
    rng = np.random.default_rng(100 * K + L)
    for trial in range(3):
        values = rng.standard_normal(1 << bits)
        x = rng.standard_normal(L)
        for e in rng.choice(1 << (bits - K), 4, replace=False):
            ref, seq = brute_force(x, K, values, bits, int(e))
            cost, states = enc.viterbi_anchored(x, K, values, int(e), bits=bits)
            assert cost == pytest.approx(ref, rel=1e-12, abs=1e-12)
            assert ((x - values[states.astype(np.int64)]) ** 2).sum() == pytest.approx(ref, rel=1e-12, abs=1e-12)
            mask = (1 << (bits - K)) - 1
            st = states.astype(np.int64)
            assert (st[1:] >> K == st[:-1] & mask).all() and st[0] >> K == e and st[-1] & mask == e


def test_viterbi_anchored_full_width_is_tail_biting():
    x = enc.encode_inputs(1, 2, 5)[0]
    for K in (3, 8):
        e = 17
        cost, s = enc.viterbi_anchored(x, K, 2, e)
        st = s.astype(np.int64)
        mask = (1 << (16 - K)) - 1
        assert (st[1:] >> K == st[:-1] & mask).all() and st[0] >> K == e and st[-1] & mask == e
        assert enc.tile_sq_error(x, s, 2) == pytest.approx(cost, rel=1e-12)


@pytest.mark.parametrize("K", range(1, 9))
def test_pack_unpack_round_trip(K):
    rng = np.random.default_rng(K)
    trellis = rng.integers(0, 65536, size=(3, 5, 16 * K), dtype=np.uint16)      # every bitstream is a valid tile
    states = orc.unpack_states(trellis, K)
    st = states.astype(np.int64)
    mask = (1 << (16 - K)) - 1
    assert (st[..., 1:] >> K == st[..., :-1] & mask).all()
    assert (st[..., 0] >> K == st[..., -1] & mask).all()
    assert (orc.pack_states(states, K) == trellis).all()
    assert (orc.unpack_states(orc.pack_states(states, K), K) == states).all()


# ---- argument checks: no device needed ---------------------------------------------------------------------------------

def test_abi_rejects_bad_arguments():
    lib = ext.lib
    assert lib.exl3b_quantize_tiles(None, None, None, None, 4, 0, 2) == -2
    assert lib.exl3b_quantize_tiles(None, None, None, None, 4, 9, 2) == -2
    assert lib.exl3b_quantize_tiles(None, None, None, None, 4, 4, 3) == -2
    assert lib.exl3b_quantize_tiles(None, None, None, None, -1, 4, 2) == -1
    assert lib.exl3b_quantize_tiles(None, None, None, None, 4, 4, 2) == -2                  # null tensors
    assert b"null" in lib.exl3b_last_error()
    assert lib.exl3b_quantize_tiles(None, None, None, None, 0, 4, 2) == 0                   # no tiles: nothing to do
    assert lib.exl3b_pack_trellis(None, None, None, 4, 9) == -2
    assert lib.exl3b_pack_trellis(None, None, None, -1, 4) == -1
    assert lib.exl3b_pack_trellis(None, None, None, 4, 4) == -2
    assert lib.exl3b_pack_trellis(None, None, None, 0, 4) == 0


def qt_args(n=2, K=4, **over):
    a = dict(input_tiles=torch.zeros((n, 256)), output_tiles=torch.zeros((n, 256)),
             output_indices=torch.zeros((n, 256), dtype=torch.int16),
             temp_costs=torch.zeros((1, 2, 65536 >> K), dtype=torch.half),
             temp_edges=torch.zeros((1, 256, 65536 >> K), dtype=torch.int16), K=K, mcg=False, mul1=True)
    a.update(over)
    return a


@pytest.mark.parametrize("over,msg", [
    (dict(K=0), "K must be in range"),
    (dict(K=9), "K must be in range"),
    (dict(input_tiles=torch.zeros((2, 128))), "dimension 1"),
    (dict(input_tiles=torch.zeros((2, 256, 1))), "number of dimensions"),
    (dict(output_tiles=torch.zeros((3, 256))), "same shape"),
    (dict(output_indices=torch.zeros((2, 256), dtype=torch.int32)), "output_indices is incorrect datatype"),
    (dict(input_tiles=torch.zeros((2, 256), dtype=torch.half)), "input_tiles is incorrect datatype"),
    (dict(output_tiles=torch.zeros((2, 256), dtype=torch.half)), "output_tiles is incorrect datatype"),
    (dict(temp_costs=torch.zeros((1, 2, 4096), dtype=torch.float)), "temp_costs is incorrect datatype"),
    (dict(temp_costs=torch.zeros((1, 2, 2048), dtype=torch.half)), "temp_costs must have shape"),
    (dict(temp_edges=torch.zeros((1, 128, 4096), dtype=torch.int16)), "temp_edges must have shape"),
    (dict(mcg=True, mul1=True), "both mcg and mul1"),
    ({}, "not on a CUDA device"),
])
def test_quantize_tiles_shim_validation(over, msg):
    with pytest.raises(RuntimeError, match=msg):
        ext.quantize_tiles(**qt_args(**over))


def test_quantize_tiles_empty_is_noop():
    ext.quantize_tiles(**qt_args(n=0))               # CPU tensors, but nothing to do: returns before any device check


@pytest.mark.parametrize("packed,unpacked,K,msg", [
    (torch.zeros((2, 3, 64), dtype=torch.int16), torch.zeros((2, 3, 256), dtype=torch.int16), 9, "K must be in range"),
    (torch.zeros((2, 3, 48), dtype=torch.int16), torch.zeros((2, 3, 256), dtype=torch.int16), 4, "dimension 2, must be 64"),
    (torch.zeros((2, 4, 64), dtype=torch.int16), torch.zeros((2, 3, 256), dtype=torch.int16), 4, "incompatible shapes"),
    (torch.zeros((2, 3, 64), dtype=torch.int16), torch.zeros((2, 3, 128), dtype=torch.int16), 4, "must be 256"),
    (torch.zeros((2, 3, 64), dtype=torch.int32), torch.zeros((2, 3, 256), dtype=torch.int16), 4, "packed is incorrect datatype"),
    (torch.zeros((2, 3, 64), dtype=torch.int16), torch.zeros((2, 3, 256), dtype=torch.int16), 4, "not on a CUDA device"),
])
def test_pack_trellis_shim_validation(packed, unpacked, K, msg):
    with pytest.raises(RuntimeError, match=msg):
        ext.pack_trellis(packed, unpacked, K)
