"""
Test harness only: the few names the REFERENCE'S OWN modules import from the rest of its package (config defaults, the
process-global scratch cache, the Hadamard helpers of its quantizer), provided as minimal stand-ins so that the
reference's exllamav3/modules/quant/exl3.py can be loaded unmodified with its `ext` bound to exllamav3_b200.ext
(oracle/gen_golden_callsites.py), and the inputs / encodings that fixture generator and tests/test_reference_callsites.py
share.  Nothing in the product imports this file.
"""
import numpy as np
import torch


class InferParams:
    no_reconstruct = False


class NullConfig:
    def __init__(self):
        self.infer_params = InferParams()


class TensorCache:
    def __init__(self):
        self.d = {}

    def get(self, device, shape, dtype):
        return self.d.setdefault((str(device), tuple(shape), dtype), torch.empty(shape, dtype=torch.half, device=device))


g_tensor_cache = TensorCache()


def _h(n, ref):
    from oracle import exl3_oracle as orc
    assert n == 128
    return torch.from_numpy(orc.hadamard_matrix_128() / np.sqrt(128.0)).to(ref.device, ref.dtype)


def preapply_had_l(x, had_dim):
    k, n = x.shape
    return (_h(had_dim, x) @ x.view(k // had_dim, had_dim, n)).view(k, n)


def preapply_had_r(x, had_dim):
    k, n = x.shape
    return (x.view(k, n // had_dim, had_dim) @ _h(had_dim, x)).view(k, n)


# ---- shared by oracle/gen_golden_callsites.py (reference side) and tests/test_reference_callsites.py (mirror side) ----
LINEAR_CASES = [((1, 256), {}, None), ((144, 256), {}, "float"), ((3, 7, 256), {}, None), ((145, 256), {}, None),
                ((1, 256), {"reconstruct": True}, None), ((1024, 256), {}, "float"), ((2, 256), {}, None)]
SLICING_ROWS = (200, 2048)
RECORDED_OPS = ("exl3_gemm", "had_r_128", "reconstruct", "reconstruct_slice", "reconstruct_had_slice", "hgemm")
AUDIT_OPS = ["exl3_gemm", "exl3_mgemm", "reconstruct", "reconstruct_slice", "reconstruct_had_slice", "had_r_128", "hgemm",
             "exl3_gemv", "g_get_cc", "g_get_num_sms", "exl3_gemv_int8_max_k", "exl3_gemm_num_kernel_shapes", "exl3_gemm_shape_compat"]


def encode(v):
    """One extension-call argument as JSON: tensors by shape (the data of these recorded calls is all zeros), dtypes by name."""
    if isinstance(v, torch.Tensor):
        return {"shape": list(v.shape)}
    if isinstance(v, torch.dtype):
        return {"dtype": str(v)}
    if isinstance(v, (bool, int, float, str)) or v is None:
        return v
    return {"repr": type(v).__name__}


def tensors(k, n, K=4):
    g = torch.Generator().manual_seed(1)
    tr = torch.randint(0, 32767, (k // 16, n // 16, 16 * K), generator=g, dtype=torch.int32).to(torch.int16)
    return dict(suh=torch.ones(k, dtype=torch.half), svh=torch.ones(n, dtype=torch.half), trellis=tr, mul1=torch.zeros((), dtype=torch.int))


def tp_tensors(k=512, n=768):
    t = tensors(k, n)
    g = torch.Generator().manual_seed(5)
    t["suh"] = torch.randn(k, generator=g).half(); t["svh"] = torch.randn(n, generator=g).half()
    bias = torch.randn(n, generator=g).half()
    return t, bias


def digest(t):
    import hashlib
    if t is None:
        return None
    t = t.contiguous().cpu()
    return {"shape": list(t.shape), "dtype": str(t.dtype), "sha256": hashlib.sha256(t.view(torch.uint8).numpy().tobytes()).hexdigest()}
