"""
Host-side mirror of the reference's `exllamav3_ext` operator surface for the EXL3 qgemm path, implemented over the
C ABI of libexl3b200.so (include/exl3b200.h) with ctypes.  Same names, argument order, argument meaning and error
behaviour (RuntimeError for shape/dtype violations) as the pybind11 bindings they replace:

    exl3_gemm, exl3_mgemm                      exllamav3_ext/bindings.cpp:126,146
    reconstruct, reconstruct_slice, reconstruct_had_slice      bindings.cpp:122-124
    had_r_128, hgemm                           bindings.cpp:125,147
    BC_LinearEXL3                              exllamav3_ext/libtorch/linear_bc.h:13-35, linear.cpp:34-71
    exl3_gemv, g_get_cc, g_get_num_sms, exl3_gemm_num_kernel_shapes, exl3_gemm_shape_compat     bindings.cpp:127-131

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

assert _lib.exl3b_abi_version() == 1

EXL3B_TAG_SIMT = 100
EXL3B_TAG_TC = 200
EXL3B_TAG_TC_I8 = 210
EXL3B_TAG_TC_I8_CHAIN = 220
EXL3B_TAG_TC_I8_AR = 211
EXL3B_TAG_TC_I8_ROUTED = 212
TP_HANDLE_BYTES = 64

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
    if B.dim() != 3:
        raise RuntimeError("B: incorrect number of dimensions, must be 3")
    _dtype(A, torch.half, "A")
    _dtype(B, torch.int16, "B")
    c_fp32 = C.dtype == torch.float
    if not c_fp32:
        _dtype(C, torch.half, "C")
    size_k = A.shape[-1]
    size_m = A.numel() // size_k if size_k else 0
    size_n = B.shape[1] * 16
    if size_k != B.shape[0] * 16:
        raise RuntimeError("A and B incompatible shapes")
    if C.shape[-1] != size_n:
        raise RuntimeError("C and B incompatible shapes")
    K = B.shape[2] // 16
    assert A.is_contiguous() and B.is_contiguous() and C.is_contiguous()
    with torch.cuda.device(A.device):
        return _check(_lib.exl3b_gemm(
            _stream(A), _ptr(A), _ptr(B), _ptr(C), _ptr(suh), _ptr(A_had) if suh is not None else None, _ptr(svh),
            size_m, size_k, size_n, K, _cb(mcg, mul1), int(c_fp32), int(force_shape_idx), int(force_num_sms)))


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
            if tr.dim() != 3:
                raise RuntimeError("B: incorrect number of dimensions, must be 3")
            _dtype(tr, torch.int16, "B")
            if gated:
                if x.dtype not in (torch.float, torch.half) or x2.dtype != x.dtype or x2.shape != x.shape:
                    raise RuntimeError("gate / up must be fp32 or fp16 tensors of one shape")
                in_mode = 1 if x.dtype == torch.float else 2
            else:
                _dtype(x, torch.half, "A")
                in_mode = 0
            c_fp32 = y.dtype == torch.float
            if not c_fp32:
                _dtype(y, torch.half, "C")
            k = x.shape[-1]
            m = x.numel() // k if k else 0
            n, K = tr.shape[1] * 16, tr.shape[2] // 16
            if k != tr.shape[0] * 16:
                raise RuntimeError("A and B incompatible shapes")
            if y.shape[-1] != n or y.numel() != m * n:
                raise RuntimeError("C and B incompatible shapes")
            assert x.is_contiguous() and tr.is_contiguous() and y.is_contiguous() and (x2 is None or x2.is_contiguous())
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
    if B.dim() != 3:
        raise RuntimeError("B: incorrect number of dimensions, must be 3")
    _dtype(A, torch.half, "A")
    _dtype(B, torch.int16, "B")
    c_fp32 = C.dtype == torch.float
    if not c_fp32:
        _dtype(C, torch.half, "C")
    size_k = A.shape[-1]
    size_m = A.numel() // size_k if size_k else 0
    size_n = B.shape[1] * 16
    if size_k != B.shape[0] * 16:
        raise RuntimeError("A and B incompatible shapes")
    if C.shape[-1] != size_n:
        raise RuntimeError("C and B incompatible shapes")
    K = B.shape[2] // 16
    assert A.is_contiguous() and B.is_contiguous() and C.is_contiguous()
    with torch.cuda.device(A.device):
        return _check(_lib.exl3b_gemm_allreduce(
            _stream(A), _ptr(A), _ptr(B), _ptr(C), _ptr(suh), None, _ptr(svh),
            size_m, size_k, size_n, K, _cb(mcg, mul1), int(c_fp32)))


# Dense exl3_mgemm calls the int8 tensor-core kernel cannot take (other codebooks, or 5..32 rows: the reference's model code
# fuses k+v and gate+up up to 32 rows, modules/attn.py:603, modules/mlp.py:726) are issued as one exact tensor-core exl3_gemm per
# matrix (tag 200; same results as separate calls, checked against the fused CUDA-core kernels by the tests).  That needs the
# pointer tables' VALUES on the host, so each table tensor is copied back once and remembered for as long as that tensor
# object lives and is not modified (weak reference + version counter; never keyed on an address, which the caching allocator
# reuses).  A table first seen during CUDA-graph capture cannot be copied: such a call runs on the CUDA-core multi-matrix
# kernels (tag 100), as does everything with EXL3B_MGEMM_SPLIT=0.
_MGEMM_SPLIT = os.environ.get("EXL3B_MGEMM_SPLIT", "1") != "0"
_table_cache: dict = {}


def _host_table(t: torch.Tensor):
    key = id(t)
    ent = _table_cache.get(key)
    if ent is not None and ent[0]() is t and ent[1] == t._version:
        return ent[2]
    if t.is_cuda and torch.cuda.is_current_stream_capturing():
        return None
    vals = [int(v) for v in t.detach().cpu().tolist()]
    _table_cache[key] = (weakref.ref(t, lambda _r, key=key: _table_cache.pop(key, None)), t._version, vals)
    return vals


def _mgemm_split(A, B, C, suh, A_had, svh, K, cb, c_fp32, bszm_in, bszm_out, m, k, n, force_num_sms):
    """One exl3b_gemm per matrix for a dense multi-matrix call; returns the path tag or None if the tables are unavailable."""
    tb, ts, tv = _host_table(B), _host_table(suh), _host_table(svh)
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


# size_n_list tensors whose host copy the library knows: device address -> (weak reference to THE tensor object, torch version
# counter, widths).  An entry is trusted only for the very tensor object it was made from (a freed tensor's address is reused by
# the caching allocator, found the hard way) at the same version (in-place writes bump it); when that object dies the entry is
# withdrawn from the library.  The copy to the host synchronises, so it happens on the first call with a tensor object -- never
# during stream capture: an unknown list simply takes the generic path there.
_widths_known: dict = {}


def _forget_widths(key: int, ref) -> None:
    hit = _widths_known.get(key)
    if hit is not None and hit[0] is ref:
        del _widths_known[key]
        try:
            _lib.exl3b_register_widths(ctypes.c_void_p(key), None, 0)
        except Exception:                          # interpreter shutdown
            pass


def _register_widths(size_n_list) -> None:
    import weakref
    key = size_n_list.data_ptr()
    ver = size_n_list._version
    hit = _widths_known.get(key)
    if hit is not None and hit[0]() is size_n_list and hit[1] == ver:
        return
    if hit is not None:                            # another tensor at this address, or rewritten: the library must not trust it
        del _widths_known[key]
        _lib.exl3b_register_widths(ctypes.c_void_p(key), None, 0)
    if torch.cuda.is_current_stream_capturing():
        return
    widths = [int(v) for v in size_n_list.detach().cpu().tolist()]
    arr = (ctypes.c_int32 * len(widths))(*widths)
    _check(_lib.exl3b_register_widths(ctypes.c_void_p(key), arr, len(widths)))
    ref = weakref.ref(size_n_list, lambda r, key=key: _forget_widths(key, r))
    _widths_known[key] = (ref, ver, widths)


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
            bszm_in, bszm_out, m, k, n, int(K), _cb(mcg, mul1), int(c_fp32),
            int(min_index), int(max_index), int(num_tokens),
            _ptr(size_n_list), _ptr(c_ptrs), num_c_ptrs, int(force_shape_idx), int(force_num_sms)))


def reconstruct_slice(unpacked, packed, K: int, mcg, mul1, n_offset: int) -> None:
    """exllamav3_ext/quant/reconstruct.cu:98-144."""
    _need_cuda(unpacked, packed)
    if unpacked.shape[0] != packed.shape[0] * 16:
        raise RuntimeError("unpacked and packed incompatible shapes")
    if packed.shape[2] != 256 * K // 16:
        raise RuntimeError("packed: incorrect size in dimension 2")
    _dtype(unpacked, torch.half, "unpacked")
    assert unpacked.is_contiguous() and packed.is_contiguous()
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
    assert unpacked.is_contiguous() and packed.is_contiguous()
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
    assert input.is_contiguous() and output.is_contiguous()
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
    assert a.is_contiguous() and b.is_contiguous()
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
    if B.dim() != 3:
        raise RuntimeError("B: incorrect number of dimensions, must be 3")
    if suh is None or A_had is None or svh is None:
        raise RuntimeError("exl3_gemv requires suh, A_had and svh")
    size_k = A.shape[-1]
    size_m = A.numel() // size_k if size_k else 0
    size_n, K = B.shape[1] * 16, B.shape[2] // 16
    if not (1 <= size_m <= 8 and 2 <= K <= 4 and size_k % 128 == 0 and size_n % 128 == 0):
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
