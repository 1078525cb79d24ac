"""
TEST INFRASTRUCTURE (oracle).  Runs the UNMODIFIED reference trellis encoder (quantize_tiles in oracle/_ref/exl3_ref_encode.so,
built by oracle/build_ref_encode.py) on a GPU and records, for every (K, codebook), its per-tile squared error (fp64, against the
unrounded fp32 input) and a CRC of its indices over the 512 seeded tiles of oracle.encode_oracle.encode_inputs /
encode_seed.  Inputs are not stored: tests regenerate them from the seed (a CRC of each input is stored to prove identity).

    python oracle/gen_golden_encode.py [out.npz]        (default tests/golden/ref_encode.npz)
"""
import os, sys, zlib
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "_ref"))
from oracle import encode_oracle as enc   # noqa: E402

N_TILES = 512


def ref_temp_buffers(K, dev):
    """Sized as the reference converter's get_temp_buffers (modules/quant/exl3_lib/quantize.py:53-63)."""
    B = 256
    if K >= 4:
        B = max(256, 2 * torch.cuda.get_device_properties(dev).multi_processor_count)
    return (torch.zeros((B, 2, 65536 >> K), dtype=torch.half, device=dev),
            torch.zeros((B, 256, 65536 >> K), dtype=torch.short, device=dev))


def ref_quantize(ref, x, K, cb, temps):
    xt = torch.from_numpy(x).cuda()
    vals = torch.empty_like(xt)
    idx = torch.empty(xt.shape, dtype=torch.short, device=xt.device)
    ref.quantize_tiles(xt, vals, idx, temps[0], temps[1], K, cb == 1, cb == 2)
    torch.cuda.synchronize()
    return vals.cpu().numpy(), idx.cpu().numpy()


def main():
    import exl3_ref_encode as ref
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_encode.npz")
    dev = torch.device("cuda:0")
    rec = {}
    for K in range(1, 9):
        temps = ref_temp_buffers(K, dev)
        for cb in range(3):
            x = enc.encode_inputs(N_TILES, cb, enc.encode_seed(K, cb))
            _, idx = ref_quantize(ref, x, K, cb, temps)
            err = enc.tile_sq_error(x, idx, cb)
            rec[f"err_K{K}_cb{cb}"] = err
            rec[f"crc_K{K}_cb{cb}"] = np.uint32(zlib.crc32(idx.tobytes()))
            rec[f"incrc_K{K}_cb{cb}"] = np.uint32(zlib.crc32(x.tobytes()))
            print(f"K={K} cb={cb} mean sq err per tile {err.mean():.6f}", flush=True)
        del temps
        torch.cuda.empty_cache()
    np.savez_compressed(out, **rec)
    print("wrote", out)


if __name__ == "__main__":
    main()
