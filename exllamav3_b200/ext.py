"""
Host-side mirror of the reference's `exllamav3_ext` operator surface for the EXL3 qgemm path, implemented over the
C ABI of libexl3b200.so (include/exl3b200.h) with ctypes.  Same names, argument order, argument meaning and error
behaviour (RuntimeError for shape/dtype violations) as the pybind11 bindings they replace:

    exl3_gemm, exl3_mgemm                      exllamav3_ext/bindings.cpp:126,146
    reconstruct, reconstruct_slice, reconstruct_had_slice      bindings.cpp:122-124
    had_r_128, hgemm                           bindings.cpp:125,147
    BC_LinearEXL3                              exllamav3_ext/libtorch/linear_bc.h:13-35, linear.cpp:34-71
    exl3_gemv, g_get_cc, g_get_num_sms, exl3_gemm_num_kernel_shapes, exl3_gemm_shape_compat     bindings.cpp:127-131
    exl3_moe, exl3_moe_max_concurrency         bindings.cpp:209-210
    quantize_tiles, pack_trellis               bindings.cpp:116,119 (the converter's trellis encoder)
    silu_mul, gelu_mul, relu2_mul              exllamav3_ext/activation.cu (gated activations)
    rms_norm, rms_norm_res_in, gated_rms_norm  exllamav3_ext/bindings.cpp:84-86, norm.cu (RMSNorm)
    BC_GatedMLP, BC_MLP                        exllamav3_ext/libtorch/mlp_bc.h, mlp.cpp (MLP decode blocks)
    exl3_gemm_gated                            this library's own: the down projection with the activation in its input stage

PyTorch is plumbing only here: device memory, the current CUDA stream and the device guard.
There is no CPU or torch fallback: if the shared library is missing this module fails to import, and every op
raises RuntimeError when given a non-CUDA tensor.
"""
from __future__ import annotations
import ctypes, os, weakref
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# EXL3B_LIBRARY selects another build of the SAME library (e.g. the bring-up build with in-kernel timeline stamps); never a
# different implementation
_LIB_PATH = os.environ.get("EXL3B_LIBRARY") or os.path.join(_HERE, "libexl3b200.so")

if not os.path.exists(_LIB_PATH):
    raise ImportError(
        f"{_LIB_PATH} not found: build it with `python -m exllamav3_b200.build` (or `python __graft_entry__.py`) "
        "(the EXL3 path has no fallback implementation)")

_lib = ctypes.CDLL(_LIB_PATH)

_vp, _i, _i64, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float

_lib.exl3b_abi_version.restype = _i
_lib.exl3b_last_error.restype = ctypes.c_char_p
_lib.exl3b_launch_count.restype = _i64
_lib.exl3b_num_sms.argtypes = [_i]; _lib.exl3b_num_sms.restype = _i
_lib.exl3b_cc.argtypes = [_i]; _lib.exl3b_cc.restype = _i
_lib.exl3b_set_gemm_path.argtypes = [_i]; _lib.exl3b_set_gemm_path.restype = _i
_lib.exl3b_gemm.argtypes = [_vp] * 7 + [_i] * 8
_lib.exl3b_gemm.restype = _i
_lib.exl3b_mgemm.argtypes = [_vp] * 8 + [_i, _vp] + [_i] * 11 + [_vp, _vp] + [_i] * 3
_lib.exl3b_mgemm.restype = _i
_lib.exl3b_reconstruct.argtypes = [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i64]
_lib.exl3b_reconstruct.restype = _i
_lib.exl3b_reconstruct_had.argtypes = [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i64]
_lib.exl3b_reconstruct_had.restype = _i
_lib.exl3b_had_r_128.argtypes = [_vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i]
_lib.exl3b_had_r_128.restype = _i
_lib.exl3b_hgemm.argtypes = [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i64]
_lib.exl3b_hgemm.restype = _i
_lib.exl3b_gemm_host.argtypes = [_vp] * 9 + [_i] * 6
_lib.exl3b_gemm_host.restype = _i

_lib.exl3b_gemm_allreduce.argtypes = [_vp] * 7 + [_i] * 6
_lib.exl3b_gemm_allreduce.restype = _i
_lib.exl3b_gemm_allreduce_check.argtypes = [_i] * 6 + [_i64]
_lib.exl3b_gemm_allreduce_check.restype = _i
_lib.exl3b_tp_alloc.argtypes = [_i, _i, _i64, _vp]; _lib.exl3b_tp_alloc.restype = _i
_lib.exl3b_tp_attach.argtypes = [_vp, _i]; _lib.exl3b_tp_attach.restype = _i
_lib.exl3b_tp_attach_loopback.restype = _i
_lib.exl3b_tp_info.argtypes = [_vp] * 4; _lib.exl3b_tp_info.restype = _i
_lib.exl3b_tp_free.restype = _i
_lib.exl3b_tp_debug_inject.argtypes = [_vp, _i, _vp, _i64]; _lib.exl3b_tp_debug_inject.restype = _i
_lib.exl3b_tp_debug_peek.argtypes = [_i, _i, _i, _vp, _i64]; _lib.exl3b_tp_debug_peek.restype = _i
_lib.exl3b_tp_debug_epoch.restype = _i64



class _ChainOp(ctypes.Structure):
    _fields_ = [("A", _vp), ("A2", _vp), ("B", _vp), ("suh", _vp), ("svh", _vp), ("C", _vp),
                ("m", _i), ("k", _i), ("n", _i), ("K", _i), ("cb", _i), ("c_fp32", _i), ("in_mode", _i), ("new_stage", _i)]


class _ChainPlan(ctypes.Structure):
    _fields_ = [("stages", _i), ("grid", _i), ("ring_stages", _i), ("smem_bytes", _i), ("cache_bytes", _i), ("units", _i64)]


_lib.exl3b_register_widths.argtypes = [_vp, _vp, _i]; _lib.exl3b_register_widths.restype = _i
_lib.exl3b_plan_fanout.argtypes = [_i, _vp, _i, _i, _vp]; _lib.exl3b_plan_fanout.restype = _i
_lib.exl3b_chain_plan.argtypes = [ctypes.POINTER(_ChainOp), _i, _i, ctypes.POINTER(_ChainPlan)]; _lib.exl3b_chain_plan.restype = _i
_lib.exl3b_chain_walk.argtypes = [ctypes.POINTER(_ChainOp), _i, _i, _i, _vp, _i]; _lib.exl3b_chain_walk.restype = _i
_lib.exl3b_chain_create.argtypes = [ctypes.POINTER(_ChainOp), _i, ctypes.POINTER(_vp)]; _lib.exl3b_chain_create.restype = _i
_lib.exl3b_chain_run.argtypes = [_vp, _vp]; _lib.exl3b_chain_run.restype = _i
_lib.exl3b_chain_destroy.argtypes = [_vp]; _lib.exl3b_chain_destroy.restype = _i


class MoePlan(ctypes.Structure):
    _fields_ = [("passes", ctypes.c_int32), ("chunks", ctypes.c_int32), ("rows", ctypes.c_int32), ("chunk_rows", ctypes.c_int32),
                ("max_passes", ctypes.c_int32), ("max_chunks", ctypes.c_int32), ("units_gate_up", _i64), ("units_down", _i64)]


_lib.exl3b_moe.argtypes = [_vp] * 6 + [_i] * 11 + [_vp] * 9 + [_i] * 6 + [_f, _i]
_lib.exl3b_moe.restype = _i
_lib.exl3b_moe_max_concurrency.argtypes = [_i]; _lib.exl3b_moe_max_concurrency.restype = _i
_lib.exl3b_moe_plan.argtypes = [_vp, _i, _i, _i, _i, _i, ctypes.POINTER(MoePlan), _vp, _vp]; _lib.exl3b_moe_plan.restype = _i
_lib.exl3b_act_mul.argtypes = [_vp] * 4 + [_i64, _i, _i, _f]; _lib.exl3b_act_mul.restype = _i
_lib.exl3b_gemm_gated.argtypes = [_vp] * 7 + [_i] * 8 + [_f, _i]; _lib.exl3b_gemm_gated.restype = _i
_lib.exl3b_rms_norm.argtypes = [_vp] * 5 + [_i64] + [_i] * 6 + [_f] * 3; _lib.exl3b_rms_norm.restype = _i
_lib.exl3b_gated_rms_norm.argtypes = [_vp] * 5 + [_i64] + [_i] * 7 + [_f] * 2; _lib.exl3b_gated_rms_norm.restype = _i
_lib.exl3b_quantize_tiles.argtypes = [_vp] * 4 + [_i64, _i, _i]; _lib.exl3b_quantize_tiles.restype = _i
_lib.exl3b_pack_trellis.argtypes = [_vp] * 3 + [_i64, _i]; _lib.exl3b_pack_trellis.restype = _i

assert _lib.exl3b_abi_version() == 1

EXL3B_TAG_SIMT = 100
EXL3B_TAG_TC = 200
EXL3B_TAG_TC_I8 = 210
EXL3B_TAG_TC_I8_CHAIN = 220
EXL3B_TAG_TC_I8_AR = 211
EXL3B_TAG_TC_I8_ROUTED = 212
EXL3B_TAG_TC_MOE = 230
TP_HANDLE_BYTES = 64
ACT_SILU, ACT_GELU, ACT_RELU2 = 0, 1, 2
MAX_BSZN = 8        # rows of BC_GatedMLP.run_bszN, as the reference's modules/mlp.py MAX_BSZN

lib = _lib      # raw handle for bench.py / tests (symbol export checks)
lib_path = _LIB_PATH


def _check(rc: int) -> int:
    if rc < 0:
        raise RuntimeError(_lib.exl3b_last_error().decode())
    return rc


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream(t: torch.Tensor):
    return torch.cuda.current_stream(t.device).cuda_stream


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("exllamav3_b200: tensor is not on a CUDA device (no CPU path exists)")


def _cb(mcg, mul1) -> int:
    mcg, mul1 = bool(mcg), bool(mul1)
    if mcg and mul1:
        raise RuntimeError("Specified both mcg and mul1")
    return 1 if mcg else (2 if mul1 else 0)


def _dtype(t, dt, name):
    if t.dtype != dt:
        raise RuntimeError(f"{name} is incorrect datatype, must be {dt}")


def _contiguous(op: str, *ts):
    for t in ts:
        if t is not None and not t.is_contiguous():
            raise RuntimeError(f"{op}: tensors must be contiguous")


def _gemm_operands(op: str, A, B, C, *more, c_numel=False, a_name="A"):
    """
    Checks of a GEMM entry's (input A, trellis B, output C); the input's dtype is the caller's to check.  `more`: further inputs
    that must be contiguous.  c_numel: C must also hold exactly m * n elements, not only n columns.  Returns (m, k, n, K, c_fp32).
    """
    if B.dim() != 3:
        raise RuntimeError("B: incorrect number of dimensions, must be 3")
    _dtype(B, torch.int16, "B")
    c_fp32 = C.dtype == torch.float
    if not c_fp32:
        _dtype(C, torch.half, "C")
    k = A.shape[-1]
    m = A.numel() // k if k else 0
    n, K = B.shape[1] * 16, B.shape[2] // 16
    if k != B.shape[0] * 16:
        raise RuntimeError(f"{a_name} and B incompatible shapes")
    if C.shape[-1] != n or (c_numel and C.numel() != m * n):
        raise RuntimeError("C and B incompatible shapes")
    _contiguous(op, A, B, C, *more)
    return m, k, n, K, c_fp32


def launch_count() -> int:
    return int(_lib.exl3b_launch_count())


def set_gemm_path(tag: int) -> int:
    """0 = auto, EXL3B_TAG_SIMT, EXL3B_TAG_TC, EXL3B_TAG_TC_I8, EXL3B_TAG_TC_I8_CHAIN.  Returns the previous setting."""
    global _forced_path
    _forced_path = int(tag)
    return int(_lib.exl3b_set_gemm_path(int(tag)))


_forced_path = 0


# ---------------------------------------------------------------------------------------------------------------
# ops
# ---------------------------------------------------------------------------------------------------------------

def exl3_gemm(A, B, C, suh, A_had, svh, force_shape_idx: int, mcg, mul1, force_num_sms: int) -> int:
    """A @ B -> C with EXL3-quantized B.  exllamav3_ext/quant/exl3_gemm.cu:110-339."""
    _need_cuda(A, B, C, suh, A_had, svh)
    _dtype(A, torch.half, "A")
    m, k, n, K, c_fp32 = _gemm_operands("exl3_gemm", A, B, C)
    with torch.cuda.device(A.device):
        return _check(_lib.exl3b_gemm(
            _stream(A), _ptr(A), _ptr(B), _ptr(C), _ptr(suh), _ptr(A_had) if suh is not None else None, _ptr(svh),
            m, k, n, K, _cb(mcg, mul1), int(c_fp32), int(force_shape_idx), int(force_num_sms)))


# ---- GEMM chains: the quantized linears of a decode block as ONE persistent launch (include/exl3b200.h) --------------------

class GemmChain:
    """
    The launch sequences of the reference's C++ block modules as one kernel: BC_GatedMLP's exl3_mgemm(gate, up) -> silu_mul ->
    exl3_gemm(down) (exllamav3_ext/libtorch/mlp.cpp:14-91) and BC_Attention's q / k / v projections
    (libtorch/attention.cpp:286-365).  `ops` is a list of dicts, executed in order:
        x        (m, k) fp16 input rows,          or   gate=, up=   (m, k) fp32|fp16 outputs of earlier ops: input = silu(gate) * up
        trellis, suh, svh, y                       as exl3_gemm's B, suh, svh, C (y fp16 or fp32, (m, n))
        mcg / mul1                                 codebook flags (only mul1 is eligible)
        new_stage                                  True: this op (and the following ones) may read outputs of earlier ops
    Construction validates like exl3_gemm and copies the table to the device (do it once, outside graph capture); run() is one
    asynchronous launch on the current stream.  Holds references to every tensor.
    """

    def __init__(self, ops: list):
        if not ops:
            raise RuntimeError("GemmChain: empty op list")
        arr = (_ChainOp * len(ops))()
        self._keep = []
        dev = None
        for i, o in enumerate(ops):
            tr, y = o["trellis"], o["y"]
            gated = "gate" in o
            x = o["gate"] if gated else o["x"]
            x2 = o["up"] if gated else None
            _need_cuda(x, x2, tr, y, o.get("suh"), o.get("svh"))
            if gated:
                if x.dtype not in (torch.float, torch.half) or x2.dtype != x.dtype or x2.shape != x.shape:
                    raise RuntimeError("gate / up must be fp32 or fp16 tensors of one shape")
                in_mode = 1 if x.dtype == torch.float else 2
            else:
                _dtype(x, torch.half, "A")
                in_mode = 0
            m, k, n, K, c_fp32 = _gemm_operands("GemmChain", x, tr, y, x2, c_numel=True)
            if dev is None:
                dev = tr.device
            elif tr.device != dev:
                raise RuntimeError("GemmChain: all tensors must live on one device")
            a = arr[i]
            a.A, a.A2, a.B, a.suh, a.svh, a.C = _ptr(x), _ptr(x2), _ptr(tr), _ptr(o.get("suh")), _ptr(o.get("svh")), _ptr(y)
            a.m, a.k, a.n, a.K, a.cb, a.c_fp32 = m, k, n, K, _cb(o.get("mcg", False), o.get("mul1", False)), int(c_fp32)
            a.in_mode, a.new_stage = in_mode, int(bool(o.get("new_stage", False)))
            self._keep.append((x, x2, tr, o.get("suh"), o.get("svh"), y))
        self.device, self.n_ops = dev, len(ops)
        self._h = _vp()
        with torch.cuda.device(dev):
            _check(_lib.exl3b_chain_create(arr, len(ops), ctypes.byref(self._h)))

    def run(self) -> int:
        with torch.cuda.device(self.device):
            return _check(_lib.exl3b_chain_run(torch.cuda.current_stream(self.device).cuda_stream, self._h))

    def close(self) -> None:
        if getattr(self, "_h", None):
            _lib.exl3b_chain_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- tensor-parallel row-parallel output: GEMM + sum over ranks in one kernel (include/exl3b200.h) --------------------

def tp_alloc(rank: int, world: int, max_elems: int) -> bytes:
    """Allocate this rank's receive buffer on the current CUDA device; returns its 64-byte CUDA IPC handle."""
    buf = ctypes.create_string_buffer(TP_HANDLE_BYTES)
    _check(_lib.exl3b_tp_alloc(int(rank), int(world), int(max_elems), ctypes.cast(buf, _vp)))
    return buf.raw


def tp_attach(handles: bytes, world: int) -> None:
    """Map the peers' receive buffers; `handles` = the world handles concatenated in rank order."""
    if len(handles) != world * TP_HANDLE_BYTES:
        raise RuntimeError(f"tp_attach: expected {world * TP_HANDLE_BYTES} handle bytes, got {len(handles)}")
    buf = ctypes.create_string_buffer(bytes(handles), len(handles))
    _check(_lib.exl3b_tp_attach(ctypes.cast(buf, _vp), int(world)))


def tp_attach_loopback() -> None:
    _check(_lib.exl3b_tp_attach_loopback())


def tp_info():
    """(rank, world, max_elems, attached) of the current device's group; rank = -1 if none."""
    r, w, a, me = ctypes.c_int(-1), ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int64(0)
    _check(_lib.exl3b_tp_info(ctypes.addressof(r), ctypes.addressof(w), ctypes.addressof(me), ctypes.addressof(a)))
    return r.value, w.value, me.value, bool(a.value)


def tp_free() -> None:
    _check(_lib.exl3b_tp_free())


def exl3_gemm_allreduce_supported(m: int, k: int, n: int, K: int, mcg, mul1, world: int, max_elems: int) -> bool:
    return _lib.exl3b_gemm_allreduce_check(int(m), int(k), int(n), int(K), _cb(mcg, mul1), int(world), int(max_elems)) == 0


def exl3_gemm_allreduce(A, B, C, suh, A_had, svh, mcg, mul1) -> int:
    """
    Row-parallel exl3_gemm whose epilogue sums the output over the tensor-parallel ranks through NVLink peer memory:
    one kernel instead of exl3_gemm + all_reduce (modules/mlp.py:769-770, modules/attn.py:546-547,
    model/model_tp_backend.py:119-126).  Same tensor arguments as exl3_gemm.  Raises RuntimeError when the call is not
    eligible (mul1, rows <= 4, group attached, rows * n within the exchange slot); the caller then uses exl3_gemm + NCCL.
    """
    _need_cuda(A, B, C, suh, A_had, svh)
    _dtype(A, torch.half, "A")
    m, k, n, K, c_fp32 = _gemm_operands("exl3_gemm_allreduce", A, B, C)
    with torch.cuda.device(A.device):
        return _check(_lib.exl3b_gemm_allreduce(
            _stream(A), _ptr(A), _ptr(B), _ptr(C), _ptr(suh), None, _ptr(svh), m, k, n, K, _cb(mcg, mul1), int(c_fp32)))


# Dense exl3_mgemm calls the int8 tensor-core kernel cannot take (other codebooks, or 5..32 rows: the reference's model code
# fuses k+v and gate+up up to 32 rows, modules/attn.py:603, modules/mlp.py:726) are issued as one exact tensor-core exl3_gemm per
# matrix (tag 200; same results as separate calls, checked against the fused CUDA-core kernels by the tests).  That needs the
# pointer tables' VALUES on the host, so each table tensor is copied back once (_host_copy, keyed on the tensor object).  A
# table first seen during CUDA-graph capture cannot be copied: such a call runs on the CUDA-core multi-matrix kernels
# (tag 100), as does everything with EXL3B_MGEMM_SPLIT=0.
_MGEMM_SPLIT = os.environ.get("EXL3B_MGEMM_SPLIT", "1") != "0"


def _capturing() -> bool:
    """Whether the current CUDA stream is capturing a graph; a process without a usable CUDA driver captures nothing."""
    try:
        return torch.cuda.is_current_stream_capturing()
    except RuntimeError:
        return False


def _host_copy(cache: dict, key, t: torch.Tensor, mirror=None):
    """
    The values of integer tensor `t` as a host list, copied once and kept in `cache` under `key` for as long as that tensor object
    lives and is not modified.  An entry is trusted only for the very object it was made from (a freed tensor's address is reused
    by the caching allocator, found the hard way) at the same version (in-place writes bump it).  The copy synchronises, so
    during stream capture nothing is copied and None is returned.  mirror(key, values) is told of each new copy, and
    mirror(key, None) when the entry is withdrawn: the object died, or another object or version replaced it.
    """
    hit = cache.get(key)
    if hit is not None:
        if hit[0]() is t and hit[1] == t._version:
            return hit[2]
        _forget_copy(cache, key, hit[0])
    if _capturing():
        return None
    vals = [int(v) for v in t.detach().cpu().tolist()]
    if mirror is not None:
        mirror(key, vals)
    cache[key] = (weakref.ref(t, lambda r, key=key, forget=_forget_copy: forget(cache, key, r)), t._version, vals, mirror)
    return vals


def _forget_copy(cache: dict, key, ref) -> None:
    hit = cache.get(key)
    if hit is not None and hit[0] is ref:
        del cache[key]
        if hit[3] is not None:
            try:
                hit[3](key, None)
            except Exception:                      # interpreter shutdown
                pass


_table_cache: dict = {}                            # id(table tensor) -> host copy


def _mgemm_split(A, B, C, suh, A_had, svh, K, cb, c_fp32, bszm_in, bszm_out, m, k, n, force_num_sms):
    """One exl3b_gemm per matrix for a dense multi-matrix call; returns the path tag or None if the tables are unavailable."""
    tb, ts, tv = (_host_copy(_table_cache, id(t), t) for t in (B, suh, svh))
    if tb is None or ts is None or tv is None or len(tb) < bszm_out:
        return None
    a0, c0, h0 = A.data_ptr(), C.data_ptr(), A_had.data_ptr()
    a_stride = 0 if bszm_in == 1 else m * k * 2
    c_stride = m * n * (4 if c_fp32 else 2)
    tag = 0
    with torch.cuda.device(A.device):
        stream = _stream(A)
        for j in range(bszm_out):
            tag = _check(_lib.exl3b_gemm(stream, a0 + j * a_stride, tb[j], c0 + j * c_stride, ts[j], h0 + j * m * k * 2, tv[j],
                                         m, k, n, int(K), cb, int(c_fp32), -1, int(force_num_sms)))
    return tag


# size_n_list tensors whose host copy the library knows (exl3b_register_widths, keyed by device address), mirrored by a host copy
# here.  An unknown list (first seen during stream capture) simply takes the generic path.
_widths_known: dict = {}


def _library_widths(key: int, widths) -> None:
    n = 0 if widths is None else len(widths)
    _check(_lib.exl3b_register_widths(ctypes.c_void_p(key), (ctypes.c_int32 * n)(*widths) if n else None, n))


def _register_widths(size_n_list) -> None:
    _host_copy(_widths_known, size_n_list.data_ptr(), size_n_list, _library_widths)


def plan_fanout(k: int, widths, num_sms: int):
    """CTA-group boundaries of a fan-out launch (host logic, no GPU needed); None if the shapes are not eligible."""
    arr = (ctypes.c_int32 * len(widths))(*[int(w) for w in widths])
    out = (ctypes.c_int32 * (len(widths) + 1))()
    g = _lib.exl3b_plan_fanout(int(k), arr, len(widths), int(num_sms), out)
    return list(out) if g > 0 else None


def exl3_mgemm(A, B, C, suh, A_had, svh, indices, weights, K: int, force_shape_idx: int, mcg, mul1,
               min_index: int, max_index: int, force_num_sms: int, num_tokens: int = 1,
               size_n_list=None, c_ptrs=None) -> int:
    """Multi-matrix EXL3 GEMM over pointer tables.  exllamav3_ext/quant/exl3_gemm.cu:341-680."""
    _need_cuda(A, B, C, suh, A_had, svh, indices, weights, size_n_list, c_ptrs)
    _dtype(A, torch.half, "A")
    _dtype(B, torch.long, "B"); _dtype(suh, torch.long, "suh"); _dtype(svh, torch.long, "svh")
    c_fp32 = C.dtype == torch.float
    if not c_fp32:
        _dtype(C, torch.half, "C")
    if A.dim() != 3 or C.dim() != 3 or B.dim() != 1 or suh.dim() != 1 or svh.dim() != 1:
        raise RuntimeError("exl3_mgemm: incorrect number of dimensions")
    if A.shape[1] != C.shape[1]:
        raise RuntimeError("A and C incompatible shapes")
    if B.shape[0] != suh.shape[0] or B.shape[0] != svh.shape[0]:
        raise RuntimeError("B, suh and svh tables must have the same length")
    bszm_in, m, k = A.shape
    bszm_out, _, n = C.shape
    num_c_ptrs = 0
    if size_n_list is not None:
        if c_ptrs is None:
            raise RuntimeError("exl3_mgemm: size_n_list requires c_ptrs")
        _dtype(size_n_list, torch.int, "size_n_list"); _dtype(c_ptrs, torch.long, "c_ptrs")
        num_c_ptrs = c_ptrs.shape[0]
    bszm = max(bszm_in, num_c_ptrs if size_n_list is not None else bszm_out)
    if A_had.numel() < bszm * m * k:
        raise RuntimeError("exl3_mgemm: A_had must hold bszm * m * k elements")
    num_indices = 0
    if indices is not None:
        if indices.dim() != 2:
            raise RuntimeError("indices: incorrect number of dimensions, must be 2")
        _dtype(indices, torch.long, "indices")
        num_indices = indices.shape[1]
    if weights is not None:
        if weights.dim() != 2:
            raise RuntimeError("weights: incorrect number of dimensions, must be 2")
        _dtype(weights, torch.half, "weights")
    cb = _cb(mcg, mul1)
    if (_MGEMM_SPLIT and _forced_path in (0, EXL3B_TAG_TC) and indices is None and weights is None and size_n_list is None and min_index < 0 and num_tokens == 1
            and not (cb == 2 and m <= 4) and bszm_in in (1, bszm_out) and m >= 1 and bszm_out >= 1 and k % 128 == 0 and n % 128 == 0):
        tag = _mgemm_split(A, B, C, suh, A_had, svh, K, cb, c_fp32, bszm_in, bszm_out, m, k, n, force_num_sms)
        if tag is not None:
            return tag
    if size_n_list is not None:
        _register_widths(size_n_list)
    with torch.cuda.device(A.device):
        return _check(_lib.exl3b_mgemm(
            _stream(A), _ptr(A), _ptr(B), _ptr(C), _ptr(suh), _ptr(A_had), _ptr(svh),
            _ptr(indices), num_indices, _ptr(weights),
            bszm_in, bszm_out, m, k, n, int(K), cb, int(c_fp32),
            int(min_index), int(max_index), int(num_tokens),
            _ptr(size_n_list), _ptr(c_ptrs), num_c_ptrs, int(force_shape_idx), int(force_num_sms)))


def exl3_moe_max_concurrency(device: int) -> int:
    """Expert groups the reference's fused MoE kernel runs at once: num_sms // 8 (exllamav3_ext/quant/exl3_moe.cu:14-18)."""
    return _check(_lib.exl3b_moe_max_concurrency(int(device)))


def exl3_moe_plan(expert_count, max_tokens: int, num_positions: int, hidden: int, intermediate: int):
    """Host-only view of the work list the device derives from these counts (include/exl3b200.h): (MoePlan,
    [(expert, pos0, rows, row0, chunk) per pass], numpy int32 code per position: 128 * pass + row, -1 = not processed)."""
    import numpy as np
    c = np.ascontiguousarray(np.asarray(expert_count, dtype=np.int64))
    E = c.shape[0] - 1
    args = (c.ctypes.data, E, int(max_tokens), int(num_positions), int(hidden), int(intermediate))
    out = MoePlan()
    _check(_lib.exl3b_moe_plan(*args, ctypes.byref(out), None, None))
    buf = np.zeros(5 * max(out.max_passes, 1), dtype=np.int32)
    codes = np.zeros(max(int(num_positions), 1), dtype=np.int32)
    _check(_lib.exl3b_moe_plan(*args, ctypes.byref(out), buf.ctypes.data, codes.ctypes.data))
    return out, [tuple(int(v) for v in buf[5 * i:5 * i + 5]) for i in range(out.passes)], codes[:int(num_positions)]


def exl3_moe(hidden_state, output_state, expert_count, token_sorted, weight_sorted,
             temp_state_g, temp_state_u, temp_intermediate_g, temp_intermediate_u,
             act_function: int, K_gate: int, K_up: int, K_down: int,
             gate_ptrs_trellis, gate_ptrs_suh, gate_ptrs_svh,
             up_ptrs_trellis, up_ptrs_suh, up_ptrs_svh,
             down_ptrs_trellis, down_ptrs_suh, down_ptrs_svh,
             gate_mcg, gate_mul1, up_mcg, up_mul1, down_mcg, down_mul1,
             act_limit: float, num_active: int) -> None:
    """
    Fused routed-expert MLP, exllamav3_ext/quant/exl3_moe.cu:36-200: for every expert with 0 < count <= temp_state_g.size(1)
    tokens, output_state[t] += w * down(act(gate(x_t)) * up(x_t)) over its positions.  Experts with more tokens, and tokens
    routed nowhere, are left to the caller: their rows of output_state keep their bits.  Unlike the reference, each token's
    contributions are added in ascending position order, so the result is deterministic.  The temp buffers are validated as
    the reference does but not used (the library keeps its own scratch).  num_active = 0 launches nothing.
    """
    if num_active == 0:
        return
    tabs = (gate_ptrs_trellis, gate_ptrs_suh, gate_ptrs_svh, up_ptrs_trellis, up_ptrs_suh, up_ptrs_svh,
            down_ptrs_trellis, down_ptrs_suh, down_ptrs_svh)
    _need_cuda(hidden_state, output_state, expert_count, token_sorted, weight_sorted,
               temp_state_g, temp_state_u, temp_intermediate_g, temp_intermediate_u, *tabs)
    _dtype(hidden_state, torch.half, "hidden_state")
    if hidden_state.dim() != 2:
        raise RuntimeError("hidden_state: incorrect number of dimensions, must be 2")
    bsz, hidden = hidden_state.shape
    _dtype(output_state, torch.float, "output_state")
    if output_state.shape != hidden_state.shape:
        raise RuntimeError("output_state and hidden_state have incompatible shapes")
    _dtype(expert_count, torch.long, "expert_count")
    if expert_count.dim() != 1:
        raise RuntimeError("expert_count: incorrect number of dimensions, must be 1")
    num_experts = expert_count.shape[0] - 1
    _dtype(token_sorted, torch.long, "token_sorted")
    if token_sorted.dim() != 1:
        raise RuntimeError("token_sorted: incorrect number of dimensions, must be 1")
    _dtype(weight_sorted, torch.half, "weight_sorted")
    if weight_sorted.shape != token_sorted.shape:
        raise RuntimeError("token_sorted and weight_sorted have incompatible shapes")
    for t, name in ((temp_state_g, "temp_state_g"), (temp_state_u, "temp_state_u"),
                    (temp_intermediate_g, "temp_intermediate_g"), (temp_intermediate_u, "temp_intermediate_u")):
        _dtype(t, torch.half, name)
        if t.dim() != 3:
            raise RuntimeError(f"{name}: incorrect number of dimensions, must be 3")
    if temp_state_g.shape[2] != hidden or temp_state_u.shape != temp_state_g.shape:
        raise RuntimeError("temp_state_g / temp_state_u incompatible shapes")
    if temp_intermediate_u.shape != temp_intermediate_g.shape or temp_intermediate_g.shape[1] != temp_state_g.shape[1]:
        raise RuntimeError("temp_intermediate_g / temp_intermediate_u incompatible shapes")
    concurrency, max_tokens, _ = temp_state_g.shape
    intermediate = temp_intermediate_g.shape[2]
    for t in tabs:
        _dtype(t, torch.long, "pointer table")
        if t.dim() != 1:
            raise RuntimeError("pointer table: incorrect number of dimensions, must be 1")
    if gate_ptrs_trellis.shape[0] != num_experts:
        raise RuntimeError("Number of gate tensors doesn't match num_experts")
    if any(t.shape != gate_ptrs_trellis.shape for t in tabs):
        raise RuntimeError("pointer tables have incompatible shapes")
    for t in (hidden_state, output_state, expert_count, token_sorted, weight_sorted, *tabs):
        if not t.is_contiguous():
            raise RuntimeError("exl3_moe: tensors must be contiguous")
    with torch.cuda.device(hidden_state.device):
        _check(_lib.exl3b_moe(
            _stream(hidden_state), _ptr(hidden_state), _ptr(output_state), _ptr(expert_count), _ptr(token_sorted),
            _ptr(weight_sorted), bsz, hidden, intermediate, num_experts, token_sorted.shape[0], max_tokens, concurrency,
            int(act_function), int(K_gate), int(K_up), int(K_down), *[_ptr(t) for t in tabs],
            int(bool(gate_mcg)), int(bool(gate_mul1)), int(bool(up_mcg)), int(bool(up_mul1)),
            int(bool(down_mcg)), int(bool(down_mul1)), float(act_limit), int(num_active)))


def reconstruct_slice(unpacked, packed, K: int, mcg, mul1, n_offset: int) -> None:
    """exllamav3_ext/quant/reconstruct.cu:98-144."""
    _need_cuda(unpacked, packed)
    if unpacked.shape[0] != packed.shape[0] * 16:
        raise RuntimeError("unpacked and packed incompatible shapes")
    if packed.shape[2] != 256 * K // 16:
        raise RuntimeError("packed: incorrect size in dimension 2")
    _dtype(unpacked, torch.half, "unpacked")
    _contiguous("reconstruct", unpacked, packed)
    with torch.cuda.device(unpacked.device):
        _check(_lib.exl3b_reconstruct(_stream(unpacked), _ptr(unpacked), _ptr(packed), unpacked.shape[0],
                                      unpacked.shape[1], packed.shape[1], int(K), _cb(mcg, mul1), int(n_offset)))


def reconstruct(unpacked, packed, K: int, mcg, mul1) -> None:
    """exllamav3_ext/quant/reconstruct.cu:375-386."""
    if unpacked.shape[1] != packed.shape[1] * 16:
        raise RuntimeError("unpacked and packed incompatible shapes")
    reconstruct_slice(unpacked, packed, K, mcg, mul1, 0)


def reconstruct_had_slice(unpacked, packed, suh, svh, K: int, mcg, mul1, n_offset: int) -> None:
    """exllamav3_ext/quant/reconstruct.cu:324-373."""
    _need_cuda(unpacked, packed, suh, svh)
    if unpacked.shape[0] != packed.shape[0] * 16:
        raise RuntimeError("unpacked and packed incompatible shapes")
    if packed.shape[2] != 256 * K // 16:
        raise RuntimeError("packed: incorrect size in dimension 2")
    _dtype(unpacked, torch.half, "unpacked"); _dtype(suh, torch.half, "suh"); _dtype(svh, torch.half, "svh")
    if suh.numel() < unpacked.shape[0]:
        raise RuntimeError("reconstruct_had: suh size")
    if svh.numel() < unpacked.shape[1]:
        raise RuntimeError("reconstruct_had: svh size")
    _contiguous("reconstruct_had", unpacked, packed)
    with torch.cuda.device(unpacked.device):
        _check(_lib.exl3b_reconstruct_had(_stream(unpacked), _ptr(unpacked), _ptr(packed), _ptr(suh), _ptr(svh),
                                          unpacked.shape[0], unpacked.shape[1], packed.shape[1], int(K),
                                          _cb(mcg, mul1), int(n_offset)))


def had_r_128(input, output, pre_scale, post_scale, scale: float) -> None:
    """exllamav3_ext/quant/hadamard.cu:88-173."""
    _need_cuda(input, output, pre_scale, post_scale)
    if input.shape != output.shape:
        raise RuntimeError("input and output incompatible shapes")
    if input.dim() != 2:
        raise RuntimeError("input: incorrect number of dimensions, must be 2")
    if input.dtype == torch.half:
        _dtype(output, torch.half, "output"); fp32 = 0
    elif input.dtype == torch.float:
        _dtype(output, torch.float, "output"); fp32 = 1
    else:
        raise RuntimeError("unsupported datatype")
    _contiguous("had_r_128", input, output)
    with torch.cuda.device(input.device):
        _check(_lib.exl3b_had_r_128(_stream(input), _ptr(input), _ptr(output), _ptr(pre_scale), _ptr(post_scale),
                                    float(scale), input.shape[0], input.shape[1], fp32))


def hgemm(a, b, c) -> None:
    """Row-major fp16 a @ b -> c (fp16 or fp32), fp32 accumulate.  exllamav3_ext/hgemm.cu:19-102."""
    _need_cuda(a, b, c)
    if c.dtype not in (torch.half, torch.float):
        raise RuntimeError("c must be float32 or float16")
    _dtype(a, torch.half, "a"); _dtype(b, torch.half, "b")
    if b.dim() != 2 or c.dim() < 2:
        raise RuntimeError("hgemm: incorrect number of dimensions")
    k = a.shape[-1]
    m = a.numel() // k if k else 0
    n = b.shape[-1]
    if k != b.shape[0] or c.shape[-1] != n:
        raise RuntimeError("a, b and c incompatible shapes")
    if c.stride(-1) != 1:
        raise RuntimeError("c must have contiguous columns")
    _contiguous("hgemm", a, b)
    with torch.cuda.device(a.device):
        _check(_lib.exl3b_hgemm(_stream(a), _ptr(a), _ptr(b), _ptr(c), m, k, n, int(c.dtype == torch.float),
                                c.stride(-2)))


def exl3_gemv(A, B, C, suh, A_had, svh, mcg, mul1) -> None:
    """
    Direct entry of the reference's small-m GEMV kernel, exposed for testing (exllamav3_ext/quant/exl3_gemv.cu:171-243,
    bindings.cpp:127): errors if the call is not hard-eligible for that kernel (suh/A_had/svh given, m <= 8, K in 2..4,
    k % 128 == 0, n % 128 == 0; exl3_gemv.cu:36-47,198).  Here small-m calls have no separate kernel family -- the
    tensor-core decode-GEMM is the small-m kernel -- so the same eligibility rules are enforced and the call is exl3_gemm.
    """
    _need_cuda(A, B, C, suh, A_had, svh)
    _dtype(A, torch.half, "A")
    m, k, n, K, _ = _gemm_operands("exl3_gemv", A, B, C)
    if suh is None or A_had is None or svh is None:
        raise RuntimeError("exl3_gemv requires suh, A_had and svh")
    if not (1 <= m <= 8 and 2 <= K <= 4 and k % 128 == 0 and n % 128 == 0):
        raise RuntimeError("exl3_gemv: call not eligible (needs m <= 8, K in 2..4, k % 128 == 0, n % 128 == 0)")
    exl3_gemm(A, B, C, suh, A_had, svh, -1, mcg, mul1, 0)


def g_get_cc(device: int) -> int:
    return _check(_lib.exl3b_cc(int(device)))


def g_get_num_sms(device: int) -> int:
    return _check(_lib.exl3b_num_sms(int(device)))


def exl3_gemv_int8_max_k(device: int) -> int:
    """
    The reference's model code asks this to decide whether same-input projections (k+v, gate+up) go out as ONE fused
    exl3_mgemm or as separate calls: it unfuses mul1 tensors with K <= this value because its separate int8 GEMVs beat its
    fused kernel there (model/config.py:48-64 use_mgemm, exllamav3_ext/quant/exl3_gemv_int8.cu:46-52: 6 on Hopper).
    Here the fused call is one launch of the same tensor-core kernel with one CTA group per matrix, so the answer is 0:
    use_mgemm() then returns True for every K.
    """
    _check(_lib.exl3b_num_sms(int(device)))          # same failure mode as the reference on a bad device index
    return 0


def exl3_gemm_num_kernel_shapes() -> int:
    """The reference enumerates 4 mma.sync tile shapes (exl3_kernel_map.cuh:53-60) that force_shape_idx selects; here the
    selectable kernels are 1 = CUDA-core twin, 2 = exact tensor-core kernel (exl3_gemm honours force_shape_idx 1 / 2 per call);
    the int8 tensor-core path is what automatic selection (-1) adds for mul1 at <= 4 rows."""
    return 2


def exl3_gemm_shape_compat(shape_idx: int, size_m: int, size_k: int, size_n: int, K: int) -> bool:
    return size_k % 128 == 0 and size_n % 128 == 0 and 1 <= K <= 8 and shape_idx in (1, 2)


class BC_LinearEXL3:
    """
    Holder of one quantized linear's tensors with run / run_alloc, as exllamav3_ext/libtorch/linear_bc.h:13-35 and
    linear.cpp:34-71.  `xh` is the caller's shared (1, k) scratch used for single-row inputs.
    """

    def __init__(self, trellis, suh, svh, K: int, bias, mcg: bool, mul1: bool, xh):
        self.trellis, self.suh, self.svh, self.K = trellis, suh, svh, int(K)
        self.bias, self.mcg, self.mul1, self.xh = bias, bool(mcg), bool(mul1), xh

    def run(self, x: torch.Tensor, y: torch.Tensor) -> None:
        if x.numel() == x.shape[-1] and self.xh is not None:
            exl3_gemm(x, self.trellis, y, self.suh, self.xh, self.svh, -1, self.mcg, self.mul1, 0)
        else:
            xh_ = torch.empty_like(x)
            exl3_gemm(x, self.trellis, y, self.suh, xh_, self.svh, -1, self.mcg, self.mul1, 0)
        if self.bias is not None:
            y += self.bias

    def run_alloc(self, x: torch.Tensor, out_features: int, output_fp32: bool) -> torch.Tensor:
        out_shape = list(x.shape)
        out_shape[-1] = out_features
        y = torch.empty(out_shape, dtype=torch.float if output_fp32 else torch.half, device=x.device)
        if out_features == 0:
            return y
        self.run(x.view(-1, x.shape[-1]), y.view(-1, out_features))
        return y


# ---- gated activations and the MLP blocks (exllamav3_ext/activation.cu, libtorch/mlp.cpp) ------------------------------------

def _act_mul(act: int, name: str, x, y, z, act_limit: float) -> None:
    _need_cuda(x, y, z)
    if x.dtype == torch.float:
        _dtype(y, torch.float, "y")
    else:
        _dtype(x, torch.half, "x")
        _dtype(y, torch.half, "y")
    _dtype(z, torch.half, "z")
    if y.numel() != x.numel() or z.numel() != x.numel():
        raise RuntimeError(f"{name}: x, y and z must have the same number of elements")
    if not (x.is_contiguous() and y.is_contiguous() and z.is_contiguous()):
        raise RuntimeError(f"{name}: x, y and z must be contiguous")
    if y.device != x.device or z.device != x.device:
        raise RuntimeError(f"{name}: x, y and z must be on one device")
    with torch.cuda.device(x.device):
        _check(_lib.exl3b_act_mul(_stream(x), _ptr(x), _ptr(y), _ptr(z), x.numel(), int(x.dtype == torch.float), act,
                                  float(act_limit)))


def silu_mul(x, y, z, act_limit: float) -> None:
    """
    z = silu(x) * y, with the limit rule of the reference (act_limit != 0: y clamped to [-act_limit, act_limit], silu(x) from above
    at act_limit).  x, y fp16 or both fp32, z fp16, equal element counts, contiguous; z may be x or y.  exllamav3_ext/activation.cu.
    Computed in fp32 and rounded to fp16 once; the reference's fp16-input kernel computes in half arithmetic (h2exp, h2rcp), so
    results can differ from it in the last bit.
    """
    _act_mul(ACT_SILU, "silu_mul", x, y, z, act_limit)


def gelu_mul(x, y, z, act_limit: float) -> None:
    """z = gelu(x) * y, gelu in the tanh form; otherwise as silu_mul (fp32 arithmetic, one rounding)."""
    _act_mul(ACT_GELU, "gelu_mul", x, y, z, act_limit)


def relu2_mul(x, y, z, act_limit: float) -> None:
    """z = max(x, 0)^2 * y; otherwise as silu_mul (fp32 arithmetic, one rounding)."""
    _act_mul(ACT_RELU2, "relu2_mul", x, y, z, act_limit)


def exl3_gemm_gated(G, U, B, C, suh, svh, act: int, act_limit: float, mcg, mul1, force_num_sms: int = 0) -> int:
    """
    exl3_gemm(act_mul(G, U), B, C, suh, svh) without the intermediate: the kernel forms fp16(act(G) * U) where it reads its input
    rows.  G, U (m, k) fp16 or both fp32, contiguous, m <= 8 (e.g. the two halves of a (2, m, k) exl3_mgemm output); act is
    ACT_SILU, ACT_GELU or ACT_RELU2.  Bit-identical to silu_mul / gelu_mul / relu2_mul into a buffer followed by exl3_gemm on it,
    on the same path and grid: tag 210 for mul1 at m <= 4, tag 200 otherwise (include/exl3b200.h).  Returns the path tag.
    """
    _need_cuda(G, U, B, C, suh, svh)
    if G.dtype == torch.float:
        _dtype(U, torch.float, "U")
    else:
        _dtype(G, torch.half, "G")
        _dtype(U, torch.half, "U")
    if U.shape != G.shape:
        raise RuntimeError("G and U incompatible shapes")
    m, k, n, K, c_fp32 = _gemm_operands("exl3_gemm_gated", G, B, C, U, c_numel=True, a_name="G")
    with torch.cuda.device(G.device):
        return _check(_lib.exl3b_gemm_gated(
            _stream(G), _ptr(G), _ptr(U), _ptr(B), _ptr(C), _ptr(suh), _ptr(svh), m, k, n, K, _cb(mcg, mul1),
            int(c_fp32), int(G.dtype == torch.float), int(act), float(act_limit), int(force_num_sms)))


def _act_kind(act_silu: bool, act_gelu: bool, act_relu2: bool, name: str) -> int:
    if act_silu:
        return ACT_SILU
    if act_gelu:
        return ACT_GELU
    if act_relu2:
        return ACT_RELU2
    raise RuntimeError(f"{name}: one of act_silu, act_gelu, act_relu2 must be set")


class BC_GatedMLP:
    """
    Gated MLP decode block, exllamav3_ext/libtorch/mlp_bc.h and mlp.cpp (same constructor arguments, so modules/mlp.py binds it
    unchanged).  run_bszN(x, d) for 1..MAX_BSZN tokens is two launches where the reference issues three: gate and up (one
    exl3_mgemm over the pointer tables, or two exl3_gemm on the `gate` / `up` BC_LinearEXL3 plus their biases), then
    exl3_gemm_gated for down, which applies the activation in its input stage, then down's bias.  Results are bit-identical to
    exl3_mgemm -> silu_mul / gelu_mul / relu2_mul -> exl3_gemm on this library.
    `a` and `down_xh` are accepted and left untouched: the activated intermediate is never written (as A_had elsewhere, the
    library keeps its own scratch).  `guh` / `gu` give width and dtype; the gate/up outputs go to exactly shaped (2, tokens, width)
    buffers kept per token count (the mgemm slot stride is tokens * width, libtorch/mlp.cpp:22-26).
    Runs eagerly on the current stream; a caller may capture it in a CUDA graph after one eager call per token count.
    """

    def __init__(self, guh, gu, a, down_xh, gu_ptrs_trellis, gu_ptrs_suh, gu_ptrs_svh, gu_K: int, gu_mcg: bool, gu_mul1: bool,
                 act_silu: bool, act_gelu: bool, act_relu2: bool, gate, up, down, act_limit: float):
        self.act = _act_kind(act_silu, act_gelu, act_relu2, "BC_GatedMLP")
        if gu_ptrs_trellis is None and (gate is None or up is None):
            raise RuntimeError("BC_GatedMLP: needs the gate/up pointer tables or the gate and up linears")
        self.guh, self.gu, self.a, self.down_xh = guh, gu, a, down_xh
        self.gu_ptrs_trellis, self.gu_ptrs_suh, self.gu_ptrs_svh = gu_ptrs_trellis, gu_ptrs_suh, gu_ptrs_svh
        self.gu_K, self.gu_mcg, self.gu_mul1 = int(gu_K), bool(gu_mcg), bool(gu_mul1)
        self.gate, self.up, self.down, self.act_limit = gate, up, down, float(act_limit)
        self._bufs = {}

    def _buffers(self, num_tokens: int):
        b = self._bufs.get(num_tokens)
        if b is None:
            b = (torch.empty((2, num_tokens, self.guh.shape[2]), dtype=self.guh.dtype, device=self.guh.device),
                 torch.empty((2, num_tokens, self.gu.shape[2]), dtype=self.gu.dtype, device=self.gu.device))
            self._bufs[num_tokens] = b
        return b

    def run_bszN(self, x, d) -> None:
        num_tokens = x.numel() // x.shape[-1] if x.shape[-1] else 0
        if not 1 <= num_tokens <= MAX_BSZN:
            raise RuntimeError("run_bszN: bsz out of supported range")
        guh_n, gu_n = self._buffers(num_tokens)
        x3 = x.view(1, num_tokens, x.shape[-1])
        g, u = gu_n[0], gu_n[1]
        if self.gu_ptrs_trellis is not None:
            exl3_mgemm(x3, self.gu_ptrs_trellis, gu_n, self.gu_ptrs_suh, guh_n, self.gu_ptrs_svh, None, None, self.gu_K, -1,
                       self.gu_mcg, self.gu_mul1, -1, -1, 0)
        else:
            gt, up = self.gate, self.up
            exl3_gemm(x3, gt.trellis, g, gt.suh, guh_n[0], gt.svh, -1, gt.mcg, gt.mul1, 0)
            exl3_gemm(x3, up.trellis, u, up.suh, guh_n[1], up.svh, -1, up.mcg, up.mul1, 0)
            if gt.bias is not None:
                g += gt.bias
            if up.bias is not None:
                u += up.bias
        dn = self.down
        exl3_gemm_gated(g, u, dn.trellis, d, dn.suh, dn.svh, self.act, self.act_limit, dn.mcg, dn.mul1)
        if dn.bias is not None:
            d += dn.bias


class BC_MLP:
    """
    Ungated MLP decode block for one token, exllamav3_ext/libtorch/mlp_bc.h and mlp.cpp (same constructor arguments, so
    modules/mlp.py binds it unchanged).  run_bsz1(x, d): the optional zero-padded staging copy into `xp`, up (with its bias)
    into `u`, then down as exl3_gemm_gated(G = u, U = ones) -- the reference's in-place act_mul(u, ones, u) applied in down's input
    stage, so `u` keeps up's output -- then down's bias, and the optional copy out of the padded `yp`.  Runs eagerly.
    """

    def __init__(self, xp, u, ones, yp, act_silu: bool, act_gelu: bool, act_relu2: bool, up, down, act_limit: float,
                 hidden_size: int, out_size: int):
        self.act = _act_kind(act_silu, act_gelu, act_relu2, "BC_MLP")
        self.xp, self.u, self.ones, self.yp = xp, u, ones, yp
        self.up, self.down, self.act_limit = up, down, float(act_limit)
        self.hidden_size, self.out_size = int(hidden_size), int(out_size)

    def run_bsz1(self, x, d) -> None:
        x_in = x
        if self.xp is not None:
            self.xp[:, :self.hidden_size].copy_(x.view(1, self.hidden_size))
            x_in = self.xp.view(1, 1, -1)
        self.up.run(x_in.view(1, -1), self.u.view(1, -1))
        dn = self.down
        y = self.yp.view(1, 1, -1) if self.yp is not None else d
        exl3_gemm_gated(self.u, self.ones, dn.trellis, y, dn.suh, dn.svh, self.act, self.act_limit, dn.mcg, dn.mul1)
        if dn.bias is not None:
            y += dn.bias
        if self.yp is not None:
            d.view(1, self.out_size).copy_(self.yp[:, :self.out_size])


# ---- RMSNorm (exllamav3_ext/norm.cu) ---------------------------------------------------------------------------------------

RES_NONE, RES_POST, RES_IN = 0, 1, 2
_NORM_DTYPES = {torch.half: 0, torch.float: 1, torch.bfloat16: 2}


def _norm_operands(name: str, x, y, *more):
    """Device, contiguity and dtype checks of a norm call; returns (rows, dim, dtype code of each of x, y, *more; None -> 0)."""
    _need_cuda(x, y, *more)
    ts = [t for t in (x, y) + more if t is not None]
    if any(t.device != x.device for t in ts):
        raise RuntimeError(f"{name}: all tensors must be on one device")
    if not all(t.is_contiguous() for t in ts):
        raise RuntimeError(f"{name}: all tensors must be contiguous")
    if any(t.dtype not in _NORM_DTYPES for t in ts):
        raise RuntimeError(f"{name}: Invalid datatypes for input/output")
    dim = x.shape[-1] if x.dim() else 1
    if dim % 4:
        raise RuntimeError("x dimension -1 must be divisible by 4")
    if y.shape != x.shape:
        raise RuntimeError("x and y have incompatible shapes")
    rows = x.numel() // dim if dim else 0
    return (rows, dim) + tuple(0 if t is None else _NORM_DTYPES[t.dtype] for t in (x, y) + more)


def _rms_norm(x, w, y, r, epsilon: float, constant_bias: float, constant_scale: float, res_mode: int) -> None:
    rows, dim, tx, ty, tw, tr = _norm_operands("rms_norm", x, y, w, r)
    if w is not None and (w.dim() == 0 or w.shape[0] != dim or w.numel() != dim):
        raise RuntimeError("x and w have incompatible shapes")
    if res_mode == RES_IN:
        if r is None:
            raise RuntimeError("rms_norm: res_mode RES_IN requires residual tensor")
        if r.shape != x.shape:
            raise RuntimeError("x and r have incompatible shapes")
    with torch.cuda.device(x.device):
        _check(_lib.exl3b_rms_norm(_stream(x), _ptr(x), _ptr(w), _ptr(y), _ptr(r), rows, dim, tx, tw, ty, tr, res_mode,
                                   float(epsilon), float(constant_bias), float(constant_scale)))


def rms_norm(x, w, y, epsilon: float, constant_bias: float, constant_scale: float, span_heads: bool, add_residual: bool) -> None:
    """
    y = (x * (w + constant_bias)) * rsqrt(mean(x^2) + epsilon) * constant_scale over the last dimension (over the last two with
    span_heads), or y += that with add_residual.  x fp16 (clamped to +-65504 where read) or fp32, w fp16 / bf16 / None, y fp16 or
    fp32 of x's shape and may be x; contiguous, last dimension a multiple of 4 and at most 16384.  exllamav3_ext/norm.cu:429-443.
    Computed in fp32 with one rounding of the result; a row's result is the same in any call that contains it.
    """
    if span_heads:
        x, y = x.flatten(-2), y.flatten(-2)
    _rms_norm(x, w, y, None, epsilon, constant_bias, constant_scale, RES_POST if add_residual else RES_NONE)


def rms_norm_res_in(x, w, y, r, epsilon: float, constant_bias: float, constant_scale: float) -> None:
    """
    The residual add folded into the next norm: r = r + x (rounded to r's dtype, written back), then y = rms_norm(r) as
    rms_norm.  r fp16 or fp32 of x's shape, y fp16.  exllamav3_ext/norm.cu:461-474.
    """
    _rms_norm(x, w, y, r, epsilon, constant_bias, constant_scale, RES_IN)


def gated_rms_norm(x, w, y, g, epsilon: float, constant_bias: float, w_groups: int = 1, gate_first: bool = False) -> None:
    """
    y = rms_norm(x) * (w + constant_bias) * silu(g), or with gate_first y = rms_norm(x * silu(g)) * (w + constant_bias).  x bf16,
    w fp32 or bf16 holding w_groups rows of dim (row i of x uses w row i % w_groups), g bf16 or fp32 and y fp16 or fp32 of x's
    shape; contiguous.  exllamav3_ext/norm.cu:582-678.  silu is computed with expf (the reference uses __expf).
    """
    rows, dim, tx, ty, tw, tg = _norm_operands("gated_rms_norm", x, y, w, g)
    w_groups = int(w_groups)
    if w_groups < 1:
        raise RuntimeError("gated_rms_norm: w_groups must be positive")
    if w_groups == 1:
        if w.dim() == 0 or w.shape[0] != dim or w.numel() != dim:
            raise RuntimeError("x and w have incompatible shapes")
    elif w.numel() != w_groups * dim:
        raise RuntimeError("gated_rms_norm: w must have w_groups * dim elements")
    if g.shape != x.shape:
        raise RuntimeError("x and g have incompatible shapes")
    with torch.cuda.device(x.device):
        _check(_lib.exl3b_gated_rms_norm(_stream(x), _ptr(x), _ptr(w), _ptr(y), _ptr(g), rows, dim, tx, tw, ty, tg, w_groups,
                                         int(bool(gate_first)), float(epsilon), float(constant_bias)))


# ---- trellis encoder (the converter's two GPU bindings, modules/quant/exl3_lib/quantize.py) ---------------------------------

def _same_cuda_contiguous(op: str, *ts):
    _need_cuda(*ts)
    dev = ts[0].device
    for t in ts:
        if t.device != dev:
            raise RuntimeError(f"{op}: all tensors must be on the same device")
        if not t.is_contiguous():
            raise RuntimeError(f"{op}: all tensors must be contiguous")


def quantize_tiles(input_tiles, output_tiles, output_indices, temp_costs, temp_edges, K: int, mcg, mul1) -> None:
    """
    Trellis-quantize tiles: row i of input_tiles (N, 256) fp32 holds one tile in trellis position order; output_indices
    (int16) receives the tail-biting state sequence of least squared error and output_tiles (fp32) its codebook values.
    exllamav3_ext/quant/quantize.cu:23-92.  The temp buffers are validated as the reference does and otherwise unused:
    the kernel keeps its backpointers as K-bit choices in a fixed per-device scratch (include/exl3b200.h).
    """
    if input_tiles.dim() != 2:
        raise RuntimeError("input_tiles: incorrect number of dimensions, must be 2")
    if input_tiles.shape[1] != 256:
        raise RuntimeError("input_tiles: incorrect size of dimension 1, must be 256")
    if tuple(output_indices.shape) != tuple(input_tiles.shape) or tuple(output_tiles.shape) != tuple(input_tiles.shape):
        raise RuntimeError("input_tiles, output_tiles and output_indices must have the same shape")
    _dtype(input_tiles, torch.float, "input_tiles")
    _dtype(output_tiles, torch.float, "output_tiles")
    _dtype(output_indices, torch.int16, "output_indices")
    K = int(K)
    if not 1 <= K <= 8:
        raise RuntimeError("quantize_tiles K must be in range 1..8")
    cb = _cb(mcg, mul1)
    num_tiles = input_tiles.shape[0]
    if num_tiles == 0:
        return
    edges = 65536 >> K
    _dtype(temp_costs, torch.half, "temp_costs")
    if temp_costs.dim() != 3 or temp_costs.shape[1] != 2 or temp_costs.shape[2] != edges:
        raise RuntimeError(f"temp_costs must have shape (B, 2, {edges})")
    _dtype(temp_edges, torch.int16, "temp_edges")
    if temp_edges.dim() != 3 or temp_edges.shape[1] != 256 or temp_edges.shape[2] != edges:
        raise RuntimeError(f"temp_edges must have shape (B, 256, {edges})")
    _same_cuda_contiguous("quantize_tiles", input_tiles, output_tiles, output_indices, temp_costs, temp_edges)
    with torch.cuda.device(input_tiles.device):
        _check(_lib.exl3b_quantize_tiles(_stream(input_tiles), _ptr(input_tiles), _ptr(output_tiles), _ptr(output_indices),
                                         num_tiles, K, cb))


def pack_trellis(packed, unpacked, K: int) -> None:
    """unpacked (a, b, 256) int16 states -> packed (a, b, 16K) int16 trellis.  exllamav3_ext/quant/pack.cu:61-86."""
    K = int(K)
    if not 1 <= K <= 8:
        raise RuntimeError("pack_trellis K must be in range 1..8")
    if packed.dim() != 3 or unpacked.dim() != 3:
        raise RuntimeError("packed and unpacked: incorrect number of dimensions, must be 3")
    if packed.shape[0] != unpacked.shape[0] or packed.shape[1] != unpacked.shape[1]:
        raise RuntimeError("packed and unpacked have incompatible shapes")
    if unpacked.shape[2] != 256:
        raise RuntimeError("unpacked: incorrect size of dimension 2, must be 256")
    if packed.shape[2] != 16 * K:
        raise RuntimeError(f"packed: incorrect size of dimension 2, must be {16 * K}")
    _dtype(packed, torch.int16, "packed")
    _dtype(unpacked, torch.int16, "unpacked")
    num_tiles = unpacked.shape[0] * unpacked.shape[1]
    if num_tiles == 0:
        return
    _same_cuda_contiguous("pack_trellis", packed, unpacked)
    with torch.cuda.device(unpacked.device):
        _check(_lib.exl3b_pack_trellis(_stream(unpacked), _ptr(packed), _ptr(unpacked), num_tiles, K))
