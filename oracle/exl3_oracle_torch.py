"""
The part of the int8 path's exact model that scales with the weights, in plain torch  --  TEST INFRASTRUCTURE, NOT PRODUCT.

oracle.exl3_gemm_i8_model contracts the activation integers q with the centred byte sums of the mul1 codebook on the host.  At
the benchmark's shapes (7.5 G weights per Llama-3.1-8B token) numpy needs minutes and tens of GB for that; here the same integer
contraction runs on whatever device holds the trellis, in column chunks, and the rest of the model (q and the row scales, the
k_inv / k_bias terms, the output Hadamard, svh, the fp16 rounding of C) stays the numpy code of exl3_oracle, which takes the
contraction through exl3_gemm_i8_model(..., qb=...).  unpack_states / mul1_bytesum restate exl3_oracle's functions of the same
name operation for operation; tests/test_bench_token_host.py holds them equal on the CPU device.

Also the mul1 weights W_hat for the fp64 oracle (exl3_gemm_f64) at the same sizes: W_hat depends on the byte sum alone, so a
1021-entry fp16 table built on the host (exl3_oracle.mul1_values) indexed by the byte sums gives it bit for bit on the device.
"""
from __future__ import annotations
import numpy as np
import torch
from oracle import exl3_oracle as orc

CHUNK_ELEMS = 1 << 24            # weights per column chunk: ~134 MB per int64 intermediate, about 1 GB at the peak

MUL1_W_TABLE = orc.mul1_values(np.arange(1021))                     # fp16 W_hat of byte sums 0 .. 1020


def _window(K: int):
    """Word indices and shift of each tile position's 16-bit window (exl3_oracle.unpack_states)."""
    nw = 8 * K
    t = np.arange(256, dtype=np.int64)
    b0 = t * K + K - 16 + 256 * K
    b1 = b0 + 16
    i0 = (b0 // 32) % nw
    i1 = ((b1 - 1) // 32) % nw
    shift = (((b1 - 1) // 32) + 1) * 32 - b1
    return i0, i1, shift


def unpack_states(trellis: torch.Tensor, K: int) -> torch.Tensor:
    """trellis (..., 16K) int16  ->  states (..., 256) int64, as exl3_oracle.unpack_states."""
    assert trellis.dtype == torch.int16 and trellis.shape[-1] == 16 * K
    dev = trellis.device
    words = trellis.contiguous().view(torch.int32).to(torch.int64) & 0xffffffff          # little-endian u32 words, (..., 8K)
    i0, i1, shift = (torch.from_numpy(a).to(dev) for a in _window(K))
    # (a << 32) may set bit 63; the shift is at most 31 and only bits shift .. shift + 15 are kept, so the sign never shows
    merged = (words[..., i0] << 32) | words[..., i1]
    return (merged >> shift) & 0xffff


def mul1_bytesum(trellis: torch.Tensor, K: int) -> torch.Tensor:
    """(k, n) int64 byte sums of state * 0x83DCD12D of trellis (k/16, n/16, 16K), as exl3_oracle.mul1_bytesum."""
    x = (unpack_states(trellis, K) * orc.CB_MUL1_MUL) & 0xffffffff                     # state < 2^16: the product fits in 48 bits
    bs = (x & 0xff) + ((x >> 8) & 0xff) + ((x >> 16) & 0xff) + (x >> 24)
    tk, tn, _ = bs.shape
    tiles = torch.empty_like(bs)
    tiles[..., torch.from_numpy(orc._PERM).to(bs.device)] = bs
    return tiles.view(tk, tn, 16, 16).permute(0, 2, 1, 3).reshape(tk * 16, tn * 16)


def column_chunks(k: int, n: int, elems: int = CHUNK_ELEMS):
    """[(c0, c1)] column ranges of whole 128-column strips with at most `elems` weights each (one strip at least)."""
    step = max(128, elems // k // 128 * 128)
    return [(c0, min(n, c0 + step)) for c0 in range(0, n, step)]


def centred_contract(q_t: torch.Tensor, bsum: torch.Tensor) -> torch.Tensor:
    """q (m, k) fp64 holding integers @ (bsum - 510) (k, c) in fp64: exact, see i8_contract."""
    return q_t @ (bsum - 510).to(torch.float64)


def i8_contract(trellis: torch.Tensor, K: int, q, xh=None, elems: int = CHUNK_ELEMS):
    """
    qb = q @ (mul1_bytesum(trellis) - 510) for the rows q (m, k) of integers, |q| <= 32512, as (m, n) float64 numpy, exactly; with
    xh (m, k) fp16 also acc = xh @ W_hat in fp64 (exl3_gemm_f64's contraction), W_hat from MUL1_W_TABLE.  The trellis is read
    once for every row, in column chunks of `elems` weights.

    Why the fp64 matmul is exact: |q| <= 32512 < 2^15, |bytesum - 510| <= 510 < 2^9 and k <= 28672 < 2^15 in every model this
    project runs, so every product and every partial sum, in whatever order the matmul adds them, is an integer of magnitude
    below 2^39 < 2^53: each fp64 operation is exact and the result is the integer itself.  (No int64 matmul is needed.)
    """
    dev = trellis.device
    k, n = trellis.shape[0] * 16, trellis.shape[1] * 16
    q = np.asarray(q)
    assert q.shape[1] == k and np.abs(q).max(initial=0) <= orc.I8_QMAX and k < 2 ** 15
    q_t = torch.from_numpy(q.astype(np.float64)).to(dev)
    xh_t = None if xh is None else torch.from_numpy(np.asarray(xh, dtype=np.float16).astype(np.float64)).to(dev)
    table = torch.from_numpy(MUL1_W_TABLE.astype(np.float64)).to(dev)            # fp16 -> fp64 is exact
    qb = torch.empty((q.shape[0], n), dtype=torch.float64, device=dev)
    acc = None if xh is None else torch.empty_like(qb)
    for c0, c1 in column_chunks(k, n, elems):
        bs = mul1_bytesum(trellis[:, c0 // 16:c1 // 16], K)
        qb[:, c0:c1] = centred_contract(q_t, bs)
        if acc is not None:
            acc[:, c0:c1] = xh_t @ table[bs]
        del bs
    qb = qb.cpu().numpy()
    return qb if acc is None else (qb, acc.cpu().numpy())


def mul1_weights(trellis: torch.Tensor, K: int, elems: int = CHUNK_ELEMS) -> np.ndarray:
    """W_hat (k, n) fp16 numpy of a mul1 trellis, bit for bit reconstruct(trellis, K, 2): the byte sums on the device, then the table."""
    k, n = trellis.shape[0] * 16, trellis.shape[1] * 16
    out = np.empty((k, n), dtype=np.float16)
    for c0, c1 in column_chunks(k, n, elems):
        out[:, c0:c1] = MUL1_W_TABLE[mul1_bytesum(trellis[:, c0 // 16:c1 // 16], K).cpu().numpy()]
    return out


# ---- the prefill sibling's models: W_hat of every codebook, had_r_128, reconstruct_had's fp32-sum model -----------------------
# Restated from exl3_oracle at its rounding points; tests/test_prefill_host.py holds each equal to its numpy original on the CPU
# device.  torch rounds fp64 -> fp16 through fp32 (two roundings), so every fp16 result below is formed from an fp32 value that
# is exact or is the numpy model's own fp32 intermediate: an fp16 x fp16 product and a decode's two-half sum fit in 24 bits.

DECODE_TABLES = {cb: orc.decode_values(np.arange(65536, dtype=np.uint16), cb) for cb in range(3)}    # state -> fp16 W_hat


def decode_weights(trellis: torch.Tensor, K: int, cb: int, elems: int = CHUNK_ELEMS) -> torch.Tensor:
    """W_hat (k, n) fp16 on trellis's device, bit for bit exl3_oracle.reconstruct(trellis, K, cb) (any codebook)."""
    dev = trellis.device
    k, n = trellis.shape[0] * 16, trellis.shape[1] * 16
    table = torch.from_numpy(DECODE_TABLES[cb]).to(dev)
    perm = torch.from_numpy(orc._PERM).to(dev)
    out = torch.empty((k, n), dtype=torch.half, device=dev)
    for c0, c1 in column_chunks(k, n, elems):
        v = table[unpack_states(trellis[:, c0 // 16:c1 // 16], K)]
        tiles = torch.empty_like(v)
        tiles[..., perm] = v
        tk, tn, _ = tiles.shape
        out[:, c0:c1] = tiles.view(tk, tn, 16, 16).permute(0, 2, 1, 3).reshape(tk * 16, tn * 16)
        del v, tiles
    return out


def hmul(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """fp16 * fp16 -> fp16 with one rounding (exl3_oracle._hmul): the product is exact in fp32."""
    return (a.float() * b.float()).half()


def fwht128_f32(x: torch.Tensor) -> torch.Tensor:
    """exl3_oracle.fwht128_f32 on fp32 (..., 128): the same butterflies, width 1, 2, 4 ... 64."""
    assert x.dtype == torch.float32 and x.shape[-1] == 128
    lead, v, w = x.shape[:-1], x, 1
    while w < 128:
        v = v.reshape(*lead, 128 // (2 * w), 2, w)
        v = torch.stack((v[..., 0, :] + v[..., 1, :], v[..., 0, :] - v[..., 1, :]), dim=-2)
        w *= 2
    return v.reshape(*lead, 128)


def had_r_128(x: torch.Tensor, pre_scale=None, post_scale=None, rows: int = 4096) -> torch.Tensor:
    """exl3_oracle.had_r_128 at scale 1 for fp16 x (pre- or post-scale) and fp32 x (post-scale only), in row chunks."""
    r_scale = float(orc.R_SCALE_F32)
    if x.dtype == torch.float32:
        assert pre_scale is None, "the fp32 pre-scale path (fma contraction) is exl3_oracle.had_r_128's alone"
    out = torch.empty_like(x)
    m, c = x.shape
    for r0 in range(0, m, rows):
        v = x[r0:r0 + rows]
        if pre_scale is not None:
            v = hmul(v, pre_scale[None, :])
        h = fwht128_f32(v.float().reshape(-1, c // 128, 128)).reshape(-1, c) * r_scale
        if x.dtype == torch.float16:
            o = h.half()
            out[r0:r0 + rows] = hmul(o, post_scale[None, :]) if post_scale is not None and pre_scale is None else o
        else:
            out[r0:r0 + rows] = h * post_scale.float()[None, :] if post_scale is not None else h
    return out


def reconstruct_had_model(trellis: torch.Tensor, suh: torch.Tensor, svh: torch.Tensor, K: int, cb: int, n_offset: int = 0,
                          n: int | None = None, elems: int = CHUNK_ELEMS // 4):
    """
    exl3_oracle.reconstruct_had_fp32_model of output columns [n_offset, n_offset + n), on the device in column chunks: returns
    (w, pre, t_step): the fp16 weights, their value before the suh / svh multiplies, and per row and 128-column block the largest
    fp16 step of the intermediate tile times fp32(1/sqrt(128)), in fp32 (k, n / 128): what one flipped rounding of that tile
    moves pre by.  svh is the full vector (indexed by column).
    Each 128-point sum of fp16 values is exact in fp64 in any order (47 significant bits at most), so the fp64 matmuls give
    numpy's sums bit for bit.
    """
    dev = trellis.device
    k = trellis.shape[0] * 16
    n = trellis.shape[1] * 16 - n_offset if n is None else n
    H = torch.from_numpy(orc.hadamard_matrix_128()).to(dev)
    r_scale = float(orc.R_SCALE_F32)
    w_out = torch.empty((k, n), dtype=torch.half, device=dev)
    pre = torch.empty_like(w_out)
    t_step = torch.empty((k, n // 128), dtype=torch.float32, device=dev)
    for c0, c1 in column_chunks(k, n, elems):
        w = decode_weights(trellis[:, (n_offset + c0) // 16:(n_offset + c1) // 16], K, cb).double()
        c = c1 - c0
        t = ((H @ w.view(k // 128, 128, c)).reshape(k, c).float() * r_scale).half()
        p = ((t.double().view(k, c // 128, 128) @ H).reshape(k, c).float() * r_scale).half()
        pre[:, c0:c1] = p
        _, e = torch.frexp(t.float().abs().view(k, c // 128, 128).amax(-1))
        t_step[:, c0 // 128:c1 // 128] = torch.exp2((e - 11).clamp(min=-24).float()) * r_scale
        w_out[:, c0:c1] = hmul(hmul(p, suh[:, None]), svh[None, n_offset + c0:n_offset + c1])
        del w, t, p
    return w_out, pre, t_step
