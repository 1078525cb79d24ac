"""
exllamav3_b200 -- Hopper-native (sm_90a) EXL3 quantized-GEMM path.

    ext           reference-named operator surface (exl3_gemm, exl3_mgemm, reconstruct*, had_r_128, hgemm,
                  BC_LinearEXL3) over the C ABI of libexl3b200.so -- the drop-in boundary
    QLinear       minimal caller of that surface (kernel path / dense sibling dispatch) for bench, smoke and tests; the
                  reference's own LinearEXL3 runs on `ext` unchanged (INTEGRATION.md)
    tp            column/row tensor-parallel shards + the row-parallel sum (NCCL, or fused into the GEMM epilogue)
"""
import sys as _sys

# `python -m exllamav3_b200.build` imports this package before the library exists: only then skip the operator surface
# (everything else fails loudly in ext.py when libexl3b200.so is missing -- there is no fallback implementation)
if "exllamav3_b200.build" not in getattr(_sys, "orig_argv", ()):
    from . import ext
    from .qlinear import QLinear, pointer_tables, KERNEL_MAX_ROWS

__all__ = ["ext", "QLinear", "pointer_tables", "KERNEL_MAX_ROWS"]
