"""
Tensor-parallel shard + collective plumbing around the EXL3 linear -- the part of the reference's TP machinery that
touches the qgemm path (SURVEY.md 8e):

  * shard construction: LinearEXL3.tp_import_split slicing rules (modules/quant/exl3.py:284-330) as the free function tp_slice
  * partition: q/k/v/gate/up column-parallel, o/down row-parallel, 128-channel granularity (modules/linear.py:645-656)
  * one all-reduce (sum) per row-parallel output, called by the CALLER of the linear (modules/mlp.py:769-770,
    modules/attn.py:546-547) -- here `row_parallel_forward`.

One process per GPU, torch.distributed for the plumbing (backend "nccl" over NVLink on multi-GPU boxes; "gloo" in the CPU
tests).  The reference's NCCL backend casts fp32 payloads to bf16 on the wire (model/model_tp_backend.py:119-126);
we reduce in the tensor's own dtype.

Two ways to produce a row-parallel output:
  * default: the shard's exl3_gemm, then ONE NCCL all-reduce (what the reference does);
  * `enable_fused_allreduce()`: ONE kernel -- the decode-GEMM's epilogue exchanges every finished 128-column segment with
    the peers over NVLink peer memory and adds the partials in rank order (csrc/gemm_tc_i8_ar.cu).  Eligible calls
    (mul1, <= 4 rows, no bias) take it, everything else falls back to the default.  Opt-in until verified on hardware.
"""
from __future__ import annotations
import torch
import torch.distributed as dist

GRANULARITY = 128


def split_ranges(total: int, parts: int, granularity: int = GRANULARITY):
    """Contiguous [first, last) per rank in units of `granularity` channels, as even as possible (earlier ranks get
    the remainder), every rank non-empty when total >= parts * granularity."""
    units = total // granularity
    assert units * granularity == total, f"{total} is not a multiple of {granularity}"
    assert units >= parts, f"cannot split {total} channels over {parts} ranks at granularity {granularity}"
    base, rem = divmod(units, parts)
    out, first = [], 0
    for r in range(parts):
        n = (base + (1 if r < rem else 0)) * granularity
        out.append((first, first + n))
        first += n
    return out


def tp_slice(lin, split, device=None):
    """
    Shard [first, last) of a QLinear, channels in multiples of 128 (both Hadamards are block-diagonal over 128 channels and
    suh / svh are per channel, so a shard is again a complete EXL3 linear).  split = (split_out, first, last):
      column shard (split_out = True)   trellis[:, first/16:last/16], svh[first:last], bias[first:last]; suh whole
      row shard    (split_out = False)  trellis[first/16:last/16], suh[first:last]; svh whole; the bias goes to the shard
                                        that starts at 0 only (it must be added once to the summed output)
    -- the slicing of the reference's tp_import_split (modules/quant/exl3.py:284-330), without its shared-memory transport.
    Every shard records whether ANY shard of the linear carries a bias (`bias_in_group`), so that all ranks pick the same
    collective in row_parallel_forward.
    """
    from .qlinear import QLinear
    split_out, first, last = split if split is not None else (True, 0, lin.out_features)
    if first % GRANULARITY or last % GRANULARITY:
        raise ValueError("tensor-parallel split granularity is 128 channels")
    dev = device or lin.trellis.device
    put = lambda t: None if t is None else t.to(dev).contiguous()
    t0, t1 = first // 16, last // 16
    if split_out:
        tr, suh, svh = lin.trellis[:, t0:t1, :], lin.suh, lin.svh[first:last]
        bias = None if lin.bias is None else lin.bias[first:last]
    else:
        tr, suh, svh = lin.trellis[t0:t1], lin.suh[first:last], lin.svh
        bias = lin.bias if first == 0 else None
    return QLinear(put(tr), put(suh), put(svh), mcg=lin.mcg, mul1=lin.mul1, bias=put(bias), out_dtype=lin.out_dtype,
                   bias_in_group=lin.bias is not None)


def column_shard(lin, rank: int, world: int, device=None):
    first, last = split_ranges(lin.out_features, world)[rank]
    return tp_slice(lin, (True, first, last), device)


def row_shard(lin, rank: int, world: int, device=None):
    first, last = split_ranges(lin.in_features, world)[rank]
    return tp_slice(lin, (False, first, last), device)


def all_reduce(t: torch.Tensor, group=None) -> torch.Tensor:
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


_fused = {"on": False, "world": 1, "max_elems": 0}


def enable_fused_allreduce(max_elems: int = 4 * 16384, group=None) -> None:
    """
    Set up the peer-memory exchange for the fused row-parallel GEMM on the current CUDA device: allocate the receive
    buffer, trade the CUDA IPC handles over the (already initialised) process group, map the peers.  `max_elems` bounds
    rows * out_features of a fused call.  Collective: every rank of the group must call it.
    """
    from . import ext
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    handle = ext.tp_alloc(rank, world, max_elems)
    handles = [None] * world
    dist.all_gather_object(handles, handle, group=group)
    ext.tp_attach(b"".join(handles), world)
    dist.barrier(group)                     # nobody sends before everybody has mapped
    _fused.update(on=True, world=world, max_elems=max_elems)


def disable_fused_allreduce(group=None) -> None:
    from . import ext
    if _fused["on"]:
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        if dist.is_initialized():
            dist.barrier(group)             # nobody unmaps while a peer may still write
        ext.tp_free()
    _fused.update(on=False, world=1, max_elems=0)


def fused_allreduce_eligible(shard, rows: int, any_bias: bool = False) -> bool:
    """Pure host logic (no device): would row_parallel_forward take the one-kernel path for this call?  The answer must be
    the same on every rank (a rank on the NCCL path while its peers wait in the fused kernel is a hang), so it depends only
    on rank-invariant facts: the shard's shape / codebook, the group, and `bias_in_group` -- never on whether THIS shard
    happens to hold the bias (only the first row shard does)."""
    from . import ext
    if not _fused["on"] or any_bias or getattr(shard, "bias_in_group", shard.bias is not None):
        return False
    return ext.exl3_gemm_allreduce_supported(rows, shard.in_features, shard.out_features, shard.K, shard.mcg, shard.mul1,
                                             _fused["world"], _fused["max_elems"])


def row_parallel_forward(shard, x_local: torch.Tensor, params: dict, out_dtype=None, group=None,
                         any_bias: bool = False) -> torch.Tensor:
    """
    y = sum over ranks of shard(x[:, first:last]): each rank applies its own full epilogue to its partial, one sum.
    A bias anywhere in the group (shard.bias_in_group, recorded by tp_slice on every rank; `any_bias` forces it) keeps the
    call on the NCCL path on ALL ranks.
    """
    rows = x_local.numel() // x_local.shape[-1]
    if not params.get("reconstruct") and fused_allreduce_eligible(shard, rows, any_bias):
        from . import ext
        dtype = out_dtype or shard.out_dtype
        y = torch.empty(tuple(x_local.shape[:-1]) + (shard.out_features,), dtype=dtype, device=x_local.device)
        ext.exl3_gemm_allreduce(x_local.view(-1, x_local.shape[-1]), shard.trellis, y.view(-1, shard.out_features),
                                shard.suh, None, shard.svh, shard.mcg, shard.mul1)
        return y
    y = shard.forward(x_local, params, out_dtype)
    return all_reduce(y, group)


def column_parallel_forward(shard, x: torch.Tensor, params: dict, out_dtype=None) -> torch.Tensor:
    """No communication: every rank keeps its slice of the output channels."""
    return shard.forward(x, params, out_dtype)


def gather_columns(y_local: torch.Tensor, total: int, group=None) -> torch.Tensor:
    """
    Full-width output of a column-parallel linear on every rank (the lm_head case, SURVEY.md 8e: col-split + gather).
    Shards may differ in width (split_ranges gives earlier ranks the remainder), so the gather is padded to the widest.
    """
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return y_local
    world = dist.get_world_size(group)
    ranges = split_ranges(total, world)
    widest = max(b - a for a, b in ranges)
    pad = torch.zeros(tuple(y_local.shape[:-1]) + (widest,), dtype=y_local.dtype, device=y_local.device)
    pad[..., :y_local.shape[-1]] = y_local
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=group)
    return torch.cat([p[..., :b - a] for p, (a, b) in zip(parts, ranges)], dim=-1)
