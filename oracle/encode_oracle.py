"""
CPU oracle for the trellis encoder (quantize_tiles)  --  TEST INFRASTRUCTURE, NOT PRODUCT.

The fp64 dynamic program that gives the exact minimum-error tail-biting state sequence for a given wrap overlap, the
per-tile error measure, and the seeded synthetic tiles shared by tests/test_encode_*.py, oracle/gen_golden_encode.py and
tools/encode_bench.py.  Codebook values come from oracle.exl3_oracle.decode_values (bit-exact with the reference's decode).
"""
from __future__ import annotations
import numpy as np
from oracle.exl3_oracle import decode_values

ENCODE_SCALE = {0: 1.24371, 1: 1.24371, 2: 1.0}        # input scale of the encoder's synthetic tiles per codebook


def encode_seed(K: int, cb: int) -> int:
    """Seed of the 512 fixed tiles of (K, cb) that tests/golden/ref_encode.npz records the reference encoder on."""
    return 1000 + 8 * cb + K


def encode_inputs(n: int, cb: int, seed: int) -> np.ndarray:
    """Seeded synthetic tiles for the encoder: randn(n, 256) fp32 x 1.24371 for 3inst / mcg, x 1.0 for mul1."""
    return (np.random.default_rng(seed).standard_normal((n, 256)) * ENCODE_SCALE[cb]).astype(np.float32)


def tile_sq_error(x: np.ndarray, states: np.ndarray, cb: int) -> np.ndarray:
    """Per-tile squared error sum_t (x_t - v(s_t))^2 in fp64, from the unrounded input."""
    v = decode_values(np.asarray(states).view(np.uint16), cb).astype(np.float64)
    return ((np.asarray(x, dtype=np.float64) - v) ** 2).sum(-1)


def viterbi_anchored(x, K: int, cb, e: int, bits: int = 16):
    """
    Exact minimum of sum_t (x_t - v(s_t))^2 over tail-biting state sequences s[0 .. L-1] of `bits`-bit states with
    s[t] >> K == s[t-1] & (2^(bits-K) - 1) (t = 1 .. L-1), the same from s[L-1] to s[0], and the wrap overlap
    s[0] >> K == e.  fp64 dynamic program over the 2^(bits-K) overlaps, vectorised over the 2^bits states.
    `cb` is a codebook index (bits = 16) or an explicit table of 2^bits values.  Returns (cost, states (L,) uint16).
    """
    x = np.asarray(x, dtype=np.float64)
    if np.isscalar(cb) or np.ndim(cb) == 0:
        assert bits == 16
        v = decode_values(np.arange(65536, dtype=np.uint32).astype(np.uint16), int(cb)).astype(np.float64)
    else:
        v = np.asarray(cb, dtype=np.float64)
    assert v.shape == (1 << bits,) and 1 <= K < bits
    Kr = bits - K
    E = 1 << Kr
    s = np.arange(1 << bits)
    pred = s >> K                                          # the overlap state s continues; s = (k << Kr) | out_edge
    cost = np.full(E, np.inf)
    cost[e] = 0.0
    back = np.empty((len(x), E), dtype=np.uint8 if K <= 8 else np.uint16)
    for t in range(len(x)):
        cand = (cost[pred] + (v - x[t]) ** 2).reshape(1 << K, E)
        back[t] = cand.argmin(0)
        cost = cand[back[t], np.arange(E)]
    out = np.empty(len(x), dtype=np.uint16)
    edge = e                                               # s[L-1] passes on the overlap e
    for t in range(len(x) - 1, -1, -1):
        st = (int(back[t, edge]) << Kr) | edge
        out[t] = st
        edge = st >> K
    assert edge == e
    return float(cost[e]), out
