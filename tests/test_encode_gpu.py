"""
Trellis encoder on the GPU (ext.quantize_tiles, ext.pack_trellis), every (K, codebook) pair.  The contract (README.md,
Parity): the states form a valid tail-biting sequence whose packed form decodes back to them; the values are the fp32 of
the GEMMs' codebook decode, bit for bit; the error is the exact minimum for the sequence's own wrap overlap (against
oracle.encode_oracle.viterbi_anchored); the summed error over 512 fixed tiles is no larger than the reference encoder's
(tests/golden/ref_encode.npz); results are deterministic and independent of the other tiles of a call.
"""
import os
import zlib
import numpy as np
import pytest
import torch
from oracle import exl3_oracle as orc
from oracle import encode_oracle as enc
from exllamav3_b200 import ext

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_encode.npz")
PAIRS = [(K, cb) for cb in range(3) for K in range(1, 9)]
IDS = [f"K{K}-cb{cb}" for K, cb in PAIRS]
SENT_F32 = 0x7FA5A5A5                                   # NaN payload nobody writes
SENT_I16 = 0x5A5A


def temps(K, dev):
    return (torch.zeros((1, 2, 65536 >> K), dtype=torch.half, device=dev),
            torch.zeros((1, 256, 65536 >> K), dtype=torch.int16, device=dev))


def quantize(x, K, cb, dev):
    xt = torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    vals = torch.empty_like(xt)
    idx = torch.empty(xt.shape, dtype=torch.int16, device=dev)
    ext.quantize_tiles(xt, vals, idx, *temps(K, dev), K, cb == 1, cb == 2)
    return vals.cpu().numpy(), idx.cpu().numpy().view(np.uint16)


def check_tail_biting(states, K):
    st = states.astype(np.int64)
    mask = (1 << (16 - K)) - 1
    assert (st[:, 1:] >> K == st[:, :-1] & mask).all(), "not a trellis path"
    assert (st[:, 0] >> K == st[:, -1] & mask).all(), "does not wrap"


_cache = {}


def fixed_tiles(K, cb, dev):
    """The 512 seeded tiles of the golden file, quantized once per module."""
    if (K, cb) not in _cache:
        x = enc.encode_inputs(512, cb, enc.encode_seed(K, cb))
        _cache[(K, cb)] = (x,) + quantize(x, K, cb, dev)
    return _cache[(K, cb)]


@pytest.mark.parametrize("K,cb", PAIRS, ids=IDS)
def test_lossless_reencode(K, cb, cuda):
    rng = np.random.default_rng(77 + 8 * cb + K)
    trellis = rng.integers(0, 65536, size=(64, 16 * K), dtype=np.uint16)        # every bitstream is a valid tile
    x = orc.decode_values(orc.unpack_states(trellis, K), cb).astype(np.float32)
    vals, idx = quantize(x, K, cb, cuda)
    assert (vals.view(np.uint32) == x.view(np.uint32)).all()
    assert enc.tile_sq_error(x, idx, cb).max() == 0.0
    check_tail_biting(idx, K)


@pytest.mark.parametrize("K,cb", PAIRS, ids=IDS)
def test_valid_values_and_optimal(K, cb, cuda):
    x, vals, idx = fixed_tiles(K, cb, cuda)
    check_tail_biting(idx, K)
    ref_vals = orc.decode_values(idx, cb).astype(np.float32)
    assert (vals.view(np.uint32) == ref_vals.view(np.uint32)).all()
    # packed by this library, decoded by the oracle's unpacker: the same states
    packed = torch.empty((1, 512, 16 * K), dtype=torch.int16, device=cuda)
    ext.pack_trellis(packed, torch.from_numpy(idx.view(np.int16)).to(cuda).view(1, 512, 256), K)
    assert (orc.unpack_states(packed.cpu().numpy()[0], K) == idx).all()
    err = enc.tile_sq_error(x, idx, cb)
    for t in (0, 1, 255, 511):
        e = int(idx[t, 0]) >> K
        best, _ = enc.viterbi_anchored(x[t], K, cb, e)
        assert err[t] <= (1 + 1e-4) * best + 1e-6, f"tile {t}: {err[t]} vs optimum {best} at overlap {e}"


@pytest.mark.parametrize("K,cb", PAIRS, ids=IDS)
def test_not_worse_than_reference(K, cb, cuda):
    g = np.load(GOLDEN)
    x, _, idx = fixed_tiles(K, cb, cuda)
    assert np.uint32(zlib.crc32(x.tobytes())) == g[f"incrc_K{K}_cb{cb}"], "inputs differ from the golden run's"
    ours, ref = enc.tile_sq_error(x, idx, cb).sum(), g[f"err_K{K}_cb{cb}"].sum()
    print(f"K={K} cb={cb}: summed squared error ours / reference = {ours / ref:.6f}")
    assert ours <= ref


@pytest.mark.parametrize("K,cb", PAIRS, ids=IDS)
def test_deterministic_and_batch_independent(K, cb, cuda):
    rng = np.random.default_rng(500 + 8 * cb + K)
    x = (rng.standard_normal((4097, 256)) * enc.ENCODE_SCALE[cb]).astype(np.float32)
    v1, i1 = quantize(x, K, cb, cuda)
    v2, i2 = quantize(x, K, cb, cuda)
    assert (v1.view(np.uint32) == v2.view(np.uint32)).all() and (i1 == i2).all()
    probe = x[:3]
    alone = [quantize(probe[j:j + 1], K, cb, cuda)[1][0] for j in range(3)]
    for n in (1, 17, 4097):
        for pos in (p for p in (0, 1, 4096) if p < n):
            for j in range(3 if n < 4097 else 1):                # one probe is enough in the big call
                xb = x[:n].copy()
                xb[pos] = probe[j]
                assert (quantize(xb, K, cb, cuda)[1][pos] == alone[j]).all(), f"n={n} pos={pos}"


@pytest.mark.parametrize("K,cb", [(1, 2), (4, 2), (8, 0)])
def test_outputs_stay_inside_their_rows(K, cb, cuda):
    n = 37
    x = enc.encode_inputs(n, cb, 9)
    xt = torch.from_numpy(x).to(cuda)
    big_v = torch.full((n + 2, 256), SENT_F32, dtype=torch.int32, device=cuda)
    big_i = torch.full((n + 2, 256), SENT_I16, dtype=torch.int16, device=cuda)
    ext.quantize_tiles(xt, big_v.view(torch.float)[1:-1], big_i[1:-1], *temps(K, cuda), K, cb == 1, cb == 2)
    bv, bi = big_v.cpu().numpy(), big_i.cpu().numpy()
    assert (bv[0] == SENT_F32).all() and (bv[-1] == SENT_F32).all()
    assert (bi[0] == SENT_I16).all() and (bi[-1] == SENT_I16).all()
    vals, idx = quantize(x, K, cb, cuda)
    assert (bv[1:-1].view(np.float32).view(np.uint32) == vals.view(np.uint32)).all()
    assert (bi[1:-1].view(np.uint16) == idx).all()
    # packer: the rows around the packed view keep their bits
    big_p = torch.full((n + 2, 16 * K), SENT_I16, dtype=torch.int16, device=cuda)
    ext.pack_trellis(big_p[1:-1].view(1, n, 16 * K), torch.from_numpy(idx.view(np.int16)).to(cuda).view(1, n, 256), K)
    bp = big_p.cpu().numpy()
    assert (bp[0] == SENT_I16).all() and (bp[-1] == SENT_I16).all()
    assert (bp[1:-1].view(np.uint16) == orc.pack_states(idx, K)).all()


@pytest.mark.parametrize("K", range(1, 9))
def test_pack_trellis_matches_oracle(K, cuda):
    rng = np.random.default_rng(40 + K)
    states = rng.integers(0, 65536, size=(3, 7, 256), dtype=np.uint16)       # any states: only the low K bits are packed
    packed = torch.empty((3, 7, 16 * K), dtype=torch.int16, device=cuda)
    ext.pack_trellis(packed, torch.from_numpy(states.view(np.int16)).to(cuda), K)
    assert (packed.cpu().numpy().view(np.uint16) == orc.pack_states(states, K)).all()


@pytest.mark.parametrize("K,cb", PAIRS, ids=IDS)
def test_encode_pack_reconstruct(K, cb, cuda):
    """A 128 x 256 weight block through quantize_tiles, pack_trellis and this library's reconstruct."""
    rng = np.random.default_rng(900 + 8 * cb + K)
    W = (rng.standard_normal((128, 256)) * enc.ENCODE_SCALE[cb]).astype(np.float32)
    perm = orc.tensor_core_perm()
    tiles = W.reshape(8, 16, 16, 16).transpose(0, 2, 1, 3).reshape(8, 16, 256)     # (k tile, n tile, row * 16 + col)
    x = np.ascontiguousarray(tiles[..., perm]).reshape(-1, 256)                     # trellis position order
    vals, idx = quantize(x, K, cb, cuda)
    packed = torch.empty((8, 16, 16 * K), dtype=torch.int16, device=cuda)
    ext.pack_trellis(packed, torch.from_numpy(idx.view(np.int16)).to(cuda).view(8, 16, 256), K)
    W_hat = torch.empty((128, 256), dtype=torch.half, device=cuda)
    ext.reconstruct(W_hat, packed, K, cb == 1, cb == 2)
    un = np.empty((8 * 16, 256), dtype=np.float32)
    un[:, perm] = vals
    expect = un.reshape(8, 16, 16, 16).transpose(0, 2, 1, 3).reshape(128, 256)
    assert (W_hat.cpu().numpy().astype(np.float32).view(np.uint32) == expect.view(np.uint32)).all()
