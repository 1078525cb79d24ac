"""
TEST INFRASTRUCTURE (oracle).  fp64 model of the RMSNorm operators (exllamav3_b200 rms_norm / rms_norm_res_in / gated_rms_norm,
the reference's exllamav3_ext/norm.cu), on CPU torch tensors.  The model takes its inputs as the kernel reads them: fp16 x
clamped to +-65504, w + constant_bias formed in fp32; everything after that is fp64.  Also the exact rule of RES_IN's residual:
r' = (x_clamped + r) added in fp32 and rounded to r's dtype.

    rms_norm_f64(x, w, eps, bias, scale)          v, the normalized term (fp64, x's shape)
    res_in_sum(x, r)                              r' (r's dtype)
    gated_rms_norm_f64(x, w, g, eps, bias, w_groups, gate_first)     the gated operator's result (fp64)
    ulp16(a)                                      spacing of fp16 at |a| (fp64 array), the unit of the fp16 bars
"""
from __future__ import annotations
import torch

F16_MAX = 65504.0


def read_x(x: torch.Tensor) -> torch.Tensor:
    """x as the kernel reads it, in fp64: fp16 clamped to +-65504, fp32 / bf16 as they are"""
    return x.double().clamp(-F16_MAX, F16_MAX) if x.dtype == torch.half else x.double()


def read_w(w: torch.Tensor | None, bias: float) -> torch.Tensor | None:
    """w + constant_bias formed in fp32 (a bias of 0 leaves w as it is), in fp64"""
    if w is None:
        return None
    w32 = w.float()
    if bias != 0.0:
        w32 = w32 + torch.tensor(bias, dtype=torch.float)
    return w32.double()


def _rmf(v: torch.Tensor, eps: float) -> torch.Tensor:
    eps32 = float(torch.tensor(eps, dtype=torch.float))
    return 1.0 / torch.sqrt((v * v).mean(dim=-1, keepdim=True) + eps32)


def rms_norm_f64(x: torch.Tensor, w: torch.Tensor | None, eps: float, bias: float = 0.0, scale: float = 1.0) -> torch.Tensor:
    """v = (x * (w + bias)) * rsqrt(mean(x^2) + eps) * scale over the last dimension, x as read (fp16 clamped)"""
    xv = read_x(x)
    wv = read_w(w, bias)
    scale32 = float(torch.tensor(scale, dtype=torch.float))
    v = xv if wv is None else xv * wv
    return v * (_rmf(xv, eps) * scale32)


def res_in_sum(x: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """RES_IN's new residual: x (fp16 clamped) + r added in fp32, rounded once to r's dtype"""
    xc = read_x(x).float()
    return (xc + r.float()).to(r.dtype)


def silu_f64(g: torch.Tensor) -> torch.Tensor:
    g = g.double()
    return g / (1.0 + torch.exp(-g))


def gated_rms_norm_f64(x: torch.Tensor, w: torch.Tensor, g: torch.Tensor, eps: float, bias: float = 0.0, w_groups: int = 1,
                       gate_first: bool = False) -> torch.Tensor:
    """gate_first: norm(x * silu(g)) * (w + bias); else norm(x) * (w + bias) * silu(g).  Row i uses w row i % w_groups."""
    dim = x.shape[-1]
    xv = x.double().reshape(-1, dim)
    s = silu_f64(g).reshape(-1, dim)
    wv = read_w(w, bias).reshape(w_groups, dim)
    wr = wv[torch.arange(xv.shape[0]) % w_groups]
    if gate_first:
        xv = xv * s
    y = xv * wr * _rmf(xv, eps)
    if not gate_first:
        y = y * s
    return y.reshape(x.shape)


def ulp16(a: torch.Tensor) -> torch.Tensor:
    """fp16 spacing at |a| (a rounded to fp16 first): 2^(e - 10) for normal values, 2^-24 below the normal range"""
    m = a.double().abs().half().double().clamp(min=2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(m)) - 10)
