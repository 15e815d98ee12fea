"""Python face of the C ABI: argument validation, stream plumbing, autograd glue.

Mirrors the reference's op wrapper
(projects/mmdet3d_plugin/bevformer/modules/multi_scale_deformable_attn_function.py): same class
names, same ``apply`` signature, same 6-tuple of gradients.  PyTorch is used for device memory and
the current stream only; all arithmetic happens in ``libbevformer_b200.so``.
"""
from __future__ import annotations

import math
import os
import warnings

import torch
from torch.autograd.function import Function, once_differentiable

from . import _lib

F32, BF16, F16 = _lib.ENUMS["BEVF_DTYPE_F32"], _lib.ENUMS["BEVF_DTYPE_BF16"], _lib.ENUMS["BEVF_DTYPE_F16"]
_DT = {torch.float32: F32, torch.bfloat16: BF16, torch.float16: F16}
# operand types of the tensor-core projections (fp32 accumulation for both)
TC_DTYPES = (torch.bfloat16, torch.float16)


def deterministic() -> bool:
    """``torch.use_deterministic_algorithms(True)`` is in effect: every backward of this package that would sum
    through atomics (sampler grad_value, LayerNorm dgamma / dbeta, bias column sums, weight gradients) takes its
    fixed-order kernel instead, and results repeat bit for bit from run to run on one GPU model."""
    return torch.are_deterministic_algorithms_enabled()


def alert_not_deterministic(name: str) -> None:
    """PyTorch's contract for an op without a deterministic implementation: raise under
    ``torch.use_deterministic_algorithms(True)``, warn under ``warn_only=True``."""
    if not torch.are_deterministic_algorithms_enabled():
        return
    msg = (f"{name} does not have a deterministic implementation, but you set "
           "'torch.use_deterministic_algorithms(True)'.")
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(msg)
    else:
        raise RuntimeError(msg)

# bench.py's roofline needs the duration of individual launches inside the timed region: when a name
# is present in KERNEL_TIMERS, the wrapper brackets that launch with CUDA events on the launching
# stream and appends (start, end, tag) -- elapsed times are read after the region's final synchronize;
# tag = (rows, levels) of the launch, which tells the SCA launches (4 levels) from the TSA ones (1).
KERNEL_TIMERS: dict = {}


class _timed:
    def __init__(self, name, device, tag=None):
        self.rec = KERNEL_TIMERS.get(name)
        self.device = device
        self.tag = tag

    def __enter__(self):
        if self.rec is not None:
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record(torch.cuda.current_stream(self.device))

    def __exit__(self, *a):
        if self.rec is not None:
            self.e.record(torch.cuda.current_stream(self.device))
            self.rec.append((self.s, self.e, self.tag))


def _stream_ptr(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _need_cuda(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (bevformer_b200 has no CPU path)")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} tensor has to be contiguous")


def _level_tensors(value, spatial_shapes, level_start_index):
    ss = torch.as_tensor(spatial_shapes)
    ls = torch.as_tensor(level_start_index)
    if ss.dim() != 2 or ss.shape[1] != 2 or ls.dim() != 1 or ls.shape[0] != ss.shape[0]:
        raise RuntimeError("spatial_shapes must be (num_levels, 2) and level_start_index (num_levels,)")
    ss = ss.to(device=value.device, dtype=torch.int64).contiguous()
    ls = ls.to(device=value.device, dtype=torch.int64).contiguous()
    return ss, ls


def _dims(value, loc, attn):
    if value.dim() != 4 or loc.dim() != 6 or attn.dim() != 5 or loc.shape[-1] != 2:
        raise RuntimeError("expected value (B,S,M,D), sampling_locations (B,Q,M,L,P,2), "
                           "attention_weights (B,Q,M,L,P)")
    B, S, M, D = value.shape
    B2, Q, M2, L, P, _ = loc.shape
    if (B2, M2) != (B, M) or tuple(attn.shape) != (B, Q, M, L, P):
        raise RuntimeError("value / sampling_locations / attention_weights shapes disagree")
    return B, S, M, D, Q, L, P


def msda_forward(value, spatial_shapes, level_start_index, sampling_locations, attention_weights,
                 out_dtype=None):
    """ms_deform_attn_forward: returns (B, Q, M*D) in ``out_dtype`` (default: value's dtype)."""
    if value.dtype not in _DT:
        raise RuntimeError(f"value dtype {value.dtype} not supported (float32, bfloat16 or float16)")
    for t, n in ((value, "value"), (sampling_locations, "sampling_loc"),
                 (attention_weights, "attn_weight")):
        _need_cuda(t, n)
    loc = sampling_locations if sampling_locations.dtype == torch.float32 else sampling_locations.float()
    attn = attention_weights if attention_weights.dtype == torch.float32 else attention_weights.float()
    B, S, M, D, Q, L, P = _dims(value, loc, attn)
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    if ss.shape[0] != L:
        raise RuntimeError("spatial_shapes and sampling_locations disagree on num_levels")
    out_dtype = out_dtype or value.dtype
    out = torch.empty((B, Q, M * D), device=value.device, dtype=out_dtype)
    lib = _lib.load()
    with torch.cuda.device(value.device), _timed("msda_forward", value.device):
        st = lib.bevf_msda_forward(value.data_ptr(), _DT[value.dtype], ss.data_ptr(), ls.data_ptr(),
                                   loc.data_ptr(), attn.data_ptr(), out.data_ptr(), _DT[out_dtype],
                                   B, S, M, D, Q, L, P, _stream_ptr(value))
    _lib.check(st, lib)
    return out


def msda_backward(value, spatial_shapes, level_start_index, sampling_locations, attention_weights,
                  grad_output, grad_value=None):
    """ms_deform_attn_backward. ``grad_value`` (fp32, zero-filled) is accumulated into when given,
    otherwise allocated here. Returns (grad_value f32, grad_loc f32, grad_attn f32)."""
    for t, n in ((value, "value"), (sampling_locations, "sampling_loc"),
                 (attention_weights, "attn_weight"), (grad_output, "grad_output")):
        _need_cuda(t, n)
    if value.dtype not in _DT or grad_output.dtype not in _DT:
        raise RuntimeError("value / grad_output must be float32, bfloat16 or float16")
    loc = sampling_locations if sampling_locations.dtype == torch.float32 else sampling_locations.float()
    attn = attention_weights if attention_weights.dtype == torch.float32 else attention_weights.float()
    B, S, M, D, Q, L, P = _dims(value, loc, attn)
    if tuple(grad_output.shape) != (B, Q, M * D):
        raise RuntimeError("grad_output must be (B, Q, M*D)")
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    if grad_value is None:
        grad_value = torch.zeros(value.shape, device=value.device, dtype=torch.float32)
    elif grad_value.dtype != torch.float32 or tuple(grad_value.shape) != tuple(value.shape):
        raise RuntimeError("grad_value must be float32 with value's shape")
    if deterministic():
        gv, grad_loc, grad_attn = msda_backward_fx(value, ss, ls, loc, attn, grad_output)
        gv.add_into(grad_value)
        return grad_value, grad_loc, grad_attn
    grad_loc = torch.empty(loc.shape, device=value.device, dtype=torch.float32)
    grad_attn = torch.empty(attn.shape, device=value.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(value.device), _timed("msda_backward", value.device):
        st = lib.bevf_msda_backward(value.data_ptr(), _DT[value.dtype], ss.data_ptr(), ls.data_ptr(),
                                    loc.data_ptr(), attn.data_ptr(), grad_output.data_ptr(),
                                    _DT[grad_output.dtype], grad_value.data_ptr(),
                                    grad_loc.data_ptr(), grad_attn.data_ptr(),
                                    B, S, M, D, Q, L, P, _stream_ptr(value))
    _lib.check(st, lib)
    return grad_value, grad_loc, grad_attn


def _check_im2col(batch: int, im2col_step) -> None:
    # mmcv asserts batch % min(batch, im2col_step) == 0; the step itself is not needed here
    step = min(batch, int(im2col_step)) if batch > 0 else 1
    if step <= 0 or batch % step != 0:
        raise RuntimeError(f"batch({batch}) must divide im2col_step({step})")


class _MSDAFunction(Function):
    """Shared body of the two reference-named classes below."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations,
                attention_weights, im2col_step):
        _check_im2col(value.shape[0], im2col_step)
        ctx.im2col_step = im2col_step
        out = msda_forward(value, value_spatial_shapes, value_level_start_index,
                           sampling_locations, attention_weights)
        ctx.save_for_backward(value, torch.as_tensor(value_spatial_shapes),
                              torch.as_tensor(value_level_start_index), sampling_locations,
                              attention_weights)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, ss, ls, loc, attn = ctx.saved_tensors
        gv, gl, ga = msda_backward(value, ss, ls, loc, attn, grad_output.contiguous())
        return (gv.to(value.dtype), None, None, gl.to(loc.dtype), ga.to(attn.dtype), None)


def _cast_args(args, dtype):
    return tuple(a.to(dtype) if torch.is_tensor(a) and a.is_floating_point() else a for a in args)


class MultiScaleDeformableAttnFunction_fp32(_MSDAFunction):
    """Same contract as the reference class of this name
    (multi_scale_deformable_attn_function.py:90-163): under autocast every floating input is cast
    to fp32 first (``custom_fwd(cast_inputs=torch.float32)``, :93). Outside autocast a bf16 or fp16 ``value``
    is consumed natively (16-bit storage, fp32 accumulation) -- an extension the reference lacks."""

    @staticmethod
    def forward(ctx, *args):
        if torch.is_autocast_enabled():
            with torch.autocast(device_type="cuda", enabled=False):
                return _MSDAFunction.forward(ctx, *_cast_args(args, torch.float32))
        return _MSDAFunction.forward(ctx, *args)


class MultiScaleDeformableAttnFunction_fp16(_MSDAFunction):
    """Name kept for import compatibility (spatial_cross_attention.py:24-25, decoder.py:27-28).
    The reference never selects it; as its ``custom_fwd(cast_inputs=torch.float32)`` does, every floating input
    is widened to fp32 (this class keeps the reference contract; fp16 storage is reached through the _fp32 class
    outside autocast or the plugin modules)."""

    @staticmethod
    def forward(ctx, *args):
        with torch.autocast(device_type="cuda", enabled=False):
            return _MSDAFunction.forward(ctx, *_cast_args(args, torch.float32))


# =================================================================================================
# Row-list sampler + fused encoder-layer pieces (see include/bevformer_b200.h for what each replaces)
# =================================================================================================
def _i32(t, device):
    return torch.as_tensor(t).to(device=device, dtype=torch.int32).contiguous()


def msda_rows_forward(value, spatial_shapes, level_start_index, loc, attn, row_map, out_dtype=None):
    """value (NB,S,M,D); loc (R,M,L,P,2) f32; attn (R,M,L,P) f32; row_map (R,) int32 -> (R, M*D)."""
    for t, n in ((value, "value"), (loc, "sampling_loc"), (attn, "attn_weight"), (row_map, "row_map")):
        _need_cuda(t, n)
    if value.dtype not in _DT or loc.dtype != torch.float32 or attn.dtype != torch.float32:
        raise RuntimeError("value must be float32/bfloat16/float16, sampling_loc and attn_weight float32")
    if row_map.dtype != torch.int32:
        raise RuntimeError("row_map must be int32")
    NB, S, M, D = value.shape
    R, M2, L, P, _ = loc.shape
    if M2 != M or tuple(attn.shape) != (R, M, L, P) or row_map.numel() != R:
        raise RuntimeError("value / sampling_loc / attn_weight / row_map shapes disagree")
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    out_dtype = out_dtype or value.dtype
    out = torch.empty((R, M * D), device=value.device, dtype=out_dtype)
    lib = _lib.load()
    with torch.cuda.device(value.device), _timed("msda_rows_forward", value.device, (R, L)):
        st = lib.bevf_msda_rows_forward(value.data_ptr(), _DT[value.dtype], ss.data_ptr(),
                                        ls.data_ptr(), loc.data_ptr(), attn.data_ptr(),
                                        out.data_ptr(), _DT[out_dtype], row_map.data_ptr(),
                                        NB, S, M, D, R, L, P, _stream_ptr(value))
    _lib.check(st, lib)
    return out


_DENSE_INIT = [False]


def _dense_mode_init(lib) -> None:
    """BEVF_MSDA_DENSE=2: the dense kernel on the library's second stream (created here, i.e. at the first eager
    backward -- never inside a stream capture); 0 / 1 are read by the library itself."""
    if not _DENSE_INIT[0]:
        _DENSE_INIT[0] = True
        if os.environ.get("BEVF_MSDA_DENSE", "") == "2" and not torch.cuda.is_current_stream_capturing():
            _lib.check(lib.bevf_msda_set_dense_backward(2), lib)


def msda_rows_backward(value, spatial_shapes, level_start_index, loc, attn, row_map, grad_output,
                       grad_value=None, group_order=None, dense=None):
    """``group_order`` (R,) int32: optional permutation of the rows in which runs of 64 entries are
    spatial neighbours on one value map (see bevf_msda_rows_backward_ordered).
    ``dense`` = (level_hw_host, map_range) for row lists grouped by value map: grad_value of the coarse levels
    through the tensor-core kernel (bevf_msda_rows_backward_dense)."""
    for t, n in ((value, "value"), (loc, "sampling_loc"), (attn, "attn_weight"),
                 (row_map, "row_map"), (grad_output, "grad_output")):
        _need_cuda(t, n)
    NB, S, M, D = value.shape
    R, _, L, P, _ = loc.shape
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    if grad_value is None:
        grad_value = torch.zeros(value.shape, device=value.device, dtype=torch.float32)
    if deterministic():
        # fixed point sums in any order: group_order has nothing to merge, and the dense kernel sums in fp32
        gv, grad_loc, grad_attn = msda_backward_fx(value, ss, ls, loc, attn, grad_output, row_map)
        gv.add_into(grad_value)
        return grad_value, grad_loc, grad_attn
    grad_loc = torch.empty(loc.shape, device=value.device, dtype=torch.float32)
    grad_attn = torch.empty(attn.shape, device=value.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(value.device), _timed("msda_rows_backward", value.device, (R, L)):
        if group_order is not None and (group_order.dtype != torch.int32 or group_order.numel() != R
                                        or not group_order.is_cuda):
            raise RuntimeError("group_order must be a CUDA int32 tensor with one entry per row")
        if dense is not None and group_order is None:
            import ctypes
            _dense_mode_init(lib)
            level_hw_host, map_range = dense
            _need_cuda(map_range, "map_range")
            if len(level_hw_host) != L or map_range.numel() != 2 * NB or map_range.dtype != torch.int32:
                raise RuntimeError("dense backward: level_hw_host / map_range do not match value and sampling_loc")
            hw = (ctypes.c_int32 * (2 * L))(*[int(v) for hw_ in level_hw_host for v in hw_])
            st = lib.bevf_msda_rows_backward_dense(value.data_ptr(), _DT[value.dtype], ss.data_ptr(), ls.data_ptr(),
                                                   ctypes.addressof(hw), loc.data_ptr(), attn.data_ptr(),
                                                   grad_output.data_ptr(), _DT[grad_output.dtype],
                                                   grad_value.data_ptr(), grad_loc.data_ptr(),
                                                   grad_attn.data_ptr(), row_map.data_ptr(), map_range.data_ptr(),
                                                   NB, S, M, D, R, L, P, _stream_ptr(value))
            _lib.check(st, lib)
            return grad_value, grad_loc, grad_attn
        st = lib.bevf_msda_rows_backward_ordered(value.data_ptr(), _DT[value.dtype], ss.data_ptr(),
                                                 ls.data_ptr(), loc.data_ptr(), attn.data_ptr(),
                                                 grad_output.data_ptr(), _DT[grad_output.dtype],
                                                 grad_value.data_ptr(), grad_loc.data_ptr(),
                                                 grad_attn.data_ptr(), row_map.data_ptr(), _ptr(group_order),
                                                 NB, S, M, D, R, L, P, _stream_ptr(value))
    _lib.check(st, lib)
    return grad_value, grad_loc, grad_attn


def gv_mode_for(rows_per_map: float, num_points: int, level_hw_host):
    """How SamplerRows' backward accumulates grad_value for a bf16 value tensor (``gv_mode``):
    levels on which a (pixel, head) collects on average at most BEVF_GV_MAXCONTRIB (default 64) contributions
    -- rows_per_map * num_points * 4 / (H * W) -- accumulate in scaled fp16 (half the L2 reduction sectors), the
    others in fp32.  Measured on the base launches against Oracle-S (tests/test_msda_gpu.py): TSA (16 per pixel)
    3.0e-3, SCA level 0 (10) 5.2e-3, level 1 (41) 6.1e-3, level 2 (164) 9.6e-3, level 3 (630) 1.3e-2 of max|grad| --
    hence the cut at 64.  BEVF_GV_ACC=fp32 switches it off.  Returns None, "f16" or ("mixed", shapes, n_fine);
    only a PREFIX of the pyramid can be fp16 (the fine levels come first in every BEVFormer config)."""
    if os.environ.get("BEVF_GV_ACC", "f16") != "f16" or not level_hw_host:
        return None
    cap = float(os.environ.get("BEVF_GV_MAXCONTRIB", "64"))
    shapes = [(int(h), int(w)) for h, w in level_hw_host]
    nfine = 0
    for h, w in shapes:
        if rows_per_map * num_points * 4.0 / (h * w) > cap:
            break
        nfine += 1
    if nfine == 0:
        return None
    return "f16" if nfine == len(shapes) else ("mixed", shapes, nfine)


def dense_levels_for(rows_per_map: float, num_points: int, level_hw_host):
    """First level of the suffix of the pyramid whose grad_value the mixed backward hands to the dense tensor-core
    kernel (bevf_msda_rows_backward_mixed_dense), or None: the levels on which a (pixel, head) collects on average
    more than 256 contributions (rows_per_map * num_points * 4 / (H * W), as in gv_mode_for).  Every level costs the
    reduction path the same number of sectors, but the dense kernel's cost grows with the pixels of its levels.
    Measured on the base SCA launch (H100 SXM, 400 W; tools/bench_sca_backward.py): level 3 alone (630 per pixel)
    1.48 ms against 1.67 ms for the fp32 reductions, levels 2-3 (from 164) 1.74 ms, levels 1-3 (from 41) 3.07 ms."""
    shapes = [(int(h), int(w)) for h, w in level_hw_host]
    first = None
    for l in range(len(shapes) - 1, -1, -1):
        h, w = shapes[l]
        if rows_per_map * num_points * 4.0 / (h * w) <= 256:
            break
        first = l
    return first


def gv_replicas_for(rows_per_map: float, num_points: int, level_hw_host):
    """{level: k} for the mixed backward's REPLICATED fp16 levels: those that gv_mode_for leaves in fp32 and
    dense_levels_for does not take (at base: level 2, 164 contributions per pixel) accumulate in scaled fp16 into
    k = ceil(contributions / BEVF_GV_MAXCONTRIB) copies, pair row r into copy r % k, so that each copy sums about as
    many contributions as a fine level; the merge adds the copies in fp32.  Half the L2 reduction sectors of fp32 and
    the colliding rows spread over k addresses.  Empty where gv_mode_for picks no mixed mode (BEVF_GV_ACC=fp32, TSA)."""
    mode = gv_mode_for(rows_per_map, num_points, level_hw_host)
    if not isinstance(mode, tuple):
        return {}
    _, shapes, nfine = mode
    cap = float(os.environ.get("BEVF_GV_MAXCONTRIB", "64"))
    kd = dense_levels_for(rows_per_map, num_points, shapes)
    out = {}
    for l in range(nfine, len(shapes) if kd is None else kd):
        h, w = shapes[l]
        out[l] = int(math.ceil(rows_per_map * num_points * 4.0 / (h * w) / cap))
    return out


def replica_plan(replicas, num_f16_levels):
    """(num_rep_levels, k) the replicated backward takes from a gv_replicas_for result: its levels directly follow
    the ``num_f16_levels`` fine ones and share one copy count, the largest; (0, 1) for none."""
    if not replicas:
        return 0, 1
    levels = sorted(replicas)
    if levels != list(range(num_f16_levels, num_f16_levels + len(levels))):
        raise RuntimeError("replicated grad_value levels must directly follow the fp16 ones")
    return len(levels), max(replicas.values())


class LazyGradValue:
    """grad_value of a sampler backward still in accumulator form (scaled fp16 [+ fp32 side buffer]): ``materialize()``
    runs the one conversion pass (bevf_gv16_unscale / bevf_gv_merge[_replicated]) on the CURRENT stream and returns
    the bf16 gradient.  Lets the consumer (plugin/linear.py's shared projections) do that pass off the critical path,
    exactly where it converts an fp32 grad_value.  ``rep`` = (S_fine, S_rep, k): ``fine`` holds k copies of the
    S_rep replicated pixels after its S_fine fine ones."""

    def __init__(self, shape, fine, side, amax, rep=None):
        self.shape, self.fine, self.side, self.amax, self.rep = tuple(shape), fine, side, amax, rep
        self.tensors = tuple(t for t in (fine, side, amax) if t is not None)
        self.device = fine.device

    def materialize(self) -> torch.Tensor:
        nb, s, m, d = self.shape
        gv = torch.empty(self.shape, device=self.device, dtype=torch.bfloat16)
        lib = _lib.load()
        with torch.cuda.device(self.device):
            if self.rep is not None:
                s_fine, s_rep, k = self.rep
                st = lib.bevf_gv_merge_replicated(self.fine.data_ptr(), _ptr(self.side), self.amax.data_ptr(),
                                                  gv.data_ptr(), nb, s, s_fine, s_rep, k, m * d, _stream_ptr(gv))
            elif self.side is None:
                st = lib.bevf_gv16_unscale(self.fine.data_ptr(), self.amax.data_ptr(), gv.data_ptr(), gv.numel(),
                                           _stream_ptr(gv))
            else:
                st = lib.bevf_gv_merge(self.fine.data_ptr(), self.side.data_ptr(), self.amax.data_ptr(), gv.data_ptr(),
                                       nb, s, self.fine.shape[1], m * d, _stream_ptr(gv))
        _lib.check(st, lib)
        return gv


class FixedPointGradValue(LazyGradValue):
    """grad_value of the deterministic sampler backward, still as int64 fixed-point sums (bevf_msda_backward_fx):
    ``materialize()`` converts it into a new tensor of ``dtype`` (the value's), ``add_into(t)`` adds it into an fp32
    buffer; both on the CURRENT stream, so the conversion can run off the critical path like LazyGradValue's."""

    def __init__(self, fx, bounds, frac_bits, dtype):
        self.shape, self.fx, self.bounds, self.frac_bits, self.dtype = tuple(fx.shape), fx, bounds, frac_bits, dtype
        self.tensors = (fx, bounds)
        self.device = fx.device

    def _convert(self, out, accumulate):
        lib = _lib.load()
        with torch.cuda.device(self.device):
            st = lib.bevf_msda_fx_convert(self.fx.data_ptr(), self.bounds.data_ptr(), self.frac_bits, out.data_ptr(),
                                          _DT[out.dtype], int(accumulate), out.numel(), _stream_ptr(out))
        _lib.check(st, lib)
        return out

    def materialize(self) -> torch.Tensor:
        return self._convert(torch.empty(self.shape, device=self.device, dtype=self.dtype), False)

    def add_into(self, out: torch.Tensor) -> torch.Tensor:
        if out.dtype not in _DT or tuple(out.shape) != self.shape or not out.is_contiguous():
            raise RuntimeError("add_into: a contiguous float32 / bfloat16 / float16 tensor of grad_value's shape is required")
        return self._convert(out, True)


def msda_backward_fx(value, spatial_shapes, level_start_index, loc, attn, grad_output, row_map=None):
    """Deterministic sampler backward (bevf_msda_backward_fx / bevf_msda_rows_backward_fx): grad_value summed in
    64-bit fixed point, whatever the order of the rows.  Plain form: loc (B, Q, M, L, P, 2), grad_output (B, Q, M*D);
    row-list form (``row_map`` (R,) int32): loc (R, M, L, P, 2), grad_output (R, M*D).  Returns (FixedPointGradValue,
    grad_loc f32, grad_attn f32); grad_loc / grad_attn equal those of msda_backward / msda_rows_backward bit for bit."""
    for t, n in ((value, "value"), (loc, "sampling_loc"), (attn, "attn_weight"), (grad_output, "grad_output")):
        _need_cuda(t, n)
    if value.dtype not in _DT or grad_output.dtype not in _DT:
        raise RuntimeError("value / grad_output must be float32, bfloat16 or float16")
    loc = loc if loc.dtype == torch.float32 else loc.float()
    attn = attn if attn.dtype == torch.float32 else attn.float()
    NB, S, M, D = value.shape
    if row_map is None:
        B, S, M, D, Q, L, P = _dims(value, loc, attn)
        if grad_output.numel() != B * Q * M * D:
            raise RuntimeError("grad_output must be (B, Q, M*D)")
    else:
        _need_cuda(row_map, "row_map")
        Q, _, L, P, _ = loc.shape
        if (row_map.dtype != torch.int32 or row_map.numel() != Q or tuple(attn.shape) != (Q, M, L, P)
                or grad_output.numel() != Q * M * D):
            raise RuntimeError("value / sampling_loc / attn_weight / row_map / grad_output shapes disagree")
    rows_per_map = Q
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    lib = _lib.load()
    k = int(lib.bevf_msda_fx_frac_bits(rows_per_map, L, P))
    fx = torch.zeros(value.shape, device=value.device, dtype=torch.int64)
    bounds = torch.empty(2, device=value.device, dtype=torch.int32)
    grad_loc = torch.empty(loc.shape, device=value.device, dtype=torch.float32)
    grad_attn = torch.empty(attn.shape, device=value.device, dtype=torch.float32)
    name = "msda_backward" if row_map is None else "msda_rows_backward"
    with torch.cuda.device(value.device), _timed(name, value.device, None if row_map is None else (Q, L)):
        args = (value.data_ptr(), _DT[value.dtype], ss.data_ptr(), ls.data_ptr(), loc.data_ptr(), attn.data_ptr(),
                grad_output.data_ptr(), _DT[grad_output.dtype], fx.data_ptr(), bounds.data_ptr(), k,
                grad_loc.data_ptr(), grad_attn.data_ptr())
        if row_map is None:
            st = lib.bevf_msda_backward_fx(*args, NB, S, M, D, Q, L, P, _stream_ptr(value))
        else:
            st = lib.bevf_msda_rows_backward_fx(*args, row_map.data_ptr(), NB, S, M, D, Q, L, P, _stream_ptr(value))
    _lib.check(st, lib)
    return FixedPointGradValue(fx, bounds, k, value.dtype), grad_loc, grad_attn


def abs_max_bits(x: torch.Tensor) -> torch.Tensor:
    """(1,) int32 device word holding the float bits of max|x| (bevf_abs_max): the scale source of the fp16-accumulated
    sampler backward."""
    _need_cuda(x, "x")
    x = x.contiguous()
    out = torch.empty(1, device=x.device, dtype=torch.int32)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        st = lib.bevf_abs_max(x.data_ptr(), _DT[x.dtype], x.numel(), out.data_ptr(), _stream_ptr(x))
    _lib.check(st, lib)
    return out


def msda_rows_backward_f16acc(value, spatial_shapes, level_start_index, loc, attn, row_map, grad_output,
                              group_order=None, lazy=False):
    """Row-list backward with grad_value accumulated in scaled fp16 (bevf_msda_rows_backward_f16acc): half the L2
    reduction sectors of the fp32 path.  Returns (grad_value as bf16 -- or, with ``lazy``, a LazyGradValue --,
    grad_loc, grad_attn)."""
    for t, n in ((value, "value"), (loc, "sampling_loc"), (attn, "attn_weight"), (row_map, "row_map"),
                 (grad_output, "grad_output")):
        _need_cuda(t, n)
    alert_not_deterministic("msda_rows_backward_f16acc (grad_value summed with fp16 atomics)")
    if value.dtype != torch.bfloat16 or value.shape[-1] != 32:
        raise RuntimeError("fp16-accumulated backward: value must be bfloat16 with head_dim 32")
    NB, S, M, D = value.shape
    R, _, L, P, _ = loc.shape
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    grad_output = grad_output.contiguous()
    grad_loc = torch.empty(loc.shape, device=value.device, dtype=torch.float32)
    grad_attn = torch.empty(attn.shape, device=value.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(value.device), _timed("msda_rows_backward", value.device, (R, L)):
        # (the scale source and the zero-fill belong to the op: they are inside the bracket bench.py times)
        amax = abs_max_bits(grad_output)
        gv16 = torch.zeros(value.shape, device=value.device, dtype=torch.float16)
        st = lib.bevf_msda_rows_backward_f16acc(value.data_ptr(), _DT[value.dtype], ss.data_ptr(), ls.data_ptr(),
                                                loc.data_ptr(), attn.data_ptr(), grad_output.data_ptr(),
                                                _DT[grad_output.dtype], gv16.data_ptr(), amax.data_ptr(),
                                                grad_loc.data_ptr(), grad_attn.data_ptr(), row_map.data_ptr(),
                                                _ptr(group_order), NB, S, M, D, R, L, P, _stream_ptr(value))
        _lib.check(st, lib)
    gv = LazyGradValue(value.shape, gv16, None, amax)
    return (gv if lazy else gv.materialize()), grad_loc, grad_attn


def msda_rows_backward_mixed(value, spatial_shapes, level_start_index, level_hw_host, num_f16_levels, loc, attn,
                             row_map, grad_output, group_order=None, lazy=False, map_range=None,
                             first_dense_level=None, replicas=None):
    """Row-list backward with MIXED accumulation (bevf_msda_rows_backward_mixed): the first ``num_f16_levels`` levels
    in scaled fp16, the others in fp32 into a side buffer that only spans their pixels; one merge pass produces the
    bf16 gradient.  ``level_hw_host``: [(h, w), ...] python ints that MUST equal the device spatial_shapes.
    ``map_range`` (B, 2) int32 for row lists grouped by value map (instead of ``group_order``): the levels
    [first_dense_level, L) (default: every side level) come from the dense tensor-core kernel where its plan covers
    them (bevf_msda_rows_backward_mixed_dense).  ``replicas`` (gv_replicas_for): the levels after the fine ones that
    accumulate in scaled fp16 copies instead of fp32 (bevf_msda_rows_backward_replicated)."""
    import ctypes
    for t, n in ((value, "value"), (loc, "sampling_loc"), (attn, "attn_weight"), (row_map, "row_map"),
                 (grad_output, "grad_output")):
        _need_cuda(t, n)
    alert_not_deterministic("msda_rows_backward_mixed (grad_value summed with fp16 / fp32 atomics)")
    if value.dtype != torch.bfloat16 or value.shape[-1] != 32:
        raise RuntimeError("mixed-accumulation backward: value must be bfloat16 with head_dim 32")
    NB, S, M, D = value.shape
    R, _, L, P, _ = loc.shape
    if len(level_hw_host) != L or not (1 <= num_f16_levels < L):
        raise RuntimeError("mixed-accumulation backward: level_hw_host / num_f16_levels do not fit the pyramid")
    if map_range is not None:
        _need_cuda(map_range, "map_range")
        if group_order is not None or map_range.numel() != 2 * NB or map_range.dtype != torch.int32:
            raise RuntimeError("mixed-accumulation backward: map_range must be (B, 2) int32, without group_order")
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    nrep, k = replica_plan(replicas, num_f16_levels)
    s_fine = sum(int(h) * int(w) for h, w in level_hw_host[:num_f16_levels])
    s_rep = sum(int(h) * int(w) for h, w in level_hw_host[num_f16_levels:num_f16_levels + nrep])
    grad_output = grad_output.contiguous()
    grad_loc = torch.empty(loc.shape, device=value.device, dtype=torch.float32)
    grad_attn = torch.empty(attn.shape, device=value.device, dtype=torch.float32)
    hw = (ctypes.c_int32 * (2 * L))(*[int(v) for hw_ in level_hw_host for v in hw_])
    lib = _lib.load()
    with torch.cuda.device(value.device), _timed("msda_rows_backward", value.device, (R, L)):
        amax = abs_max_bits(grad_output)
        fine = torch.zeros((NB, s_fine + k * s_rep, M, D), device=value.device, dtype=torch.float16)
        side = torch.zeros((NB, S - s_fine - s_rep, M, D), device=value.device, dtype=torch.float32)
        args = (value.data_ptr(), _DT[value.dtype], ss.data_ptr(), ls.data_ptr(), ctypes.addressof(hw), loc.data_ptr(),
                attn.data_ptr(), grad_output.data_ptr(), _DT[grad_output.dtype], fine.data_ptr(), _ptr(side),
                amax.data_ptr(), int(num_f16_levels))
        tail = (grad_loc.data_ptr(), grad_attn.data_ptr(), row_map.data_ptr())
        if nrep:
            kd = num_f16_levels + nrep if first_dense_level is None else int(first_dense_level)
            st = lib.bevf_msda_rows_backward_replicated(*args, nrep, k, kd, *tail, _ptr(group_order), _ptr(map_range),
                                                        NB, S, M, D, R, L, P, _stream_ptr(value))
        elif map_range is None:
            st = lib.bevf_msda_rows_backward_mixed(*args, *tail, _ptr(group_order), NB, S, M, D, R, L, P,
                                                   _stream_ptr(value))
        else:
            kd = num_f16_levels if first_dense_level is None else int(first_dense_level)
            st = lib.bevf_msda_rows_backward_mixed_dense(*args, kd, *tail, map_range.data_ptr(), NB, S, M, D, R, L, P,
                                                         _stream_ptr(value))
        _lib.check(st, lib)
    gv = LazyGradValue(value.shape, fine, side if side.numel() else None, amax,
                       (s_fine, s_rep, k) if nrep else None)
    return (gv if lazy else gv.materialize()), grad_loc, grad_attn


# Second stream for work that is off the critical path (weight gradients, zero-fills and projections that
# are needed later): set by BEVFormerEncoder.enable_grad_arena(overlap=True); None = everything in order.
AUX_STREAM: dict = {}


def aux_stream(device):
    return AUX_STREAM.get(torch.device(device))


class SamplerRows(Function):
    """Sampler over a compact list of query rows (SCA's in-view (camera, query) pairs)."""

    @staticmethod
    def forward(ctx, value, loc, attn, row_map, spatial_shapes, level_start_index, group_order=None,
                dense=None, gv_mode=None):
        """``dense`` = (level_hw_host, map_range) for rows grouped by value map: the backward may hand the coarse
        levels' grad_value to the dense tensor-core kernel.  An fp16 ``value`` is read natively (no widened copy);
        the dense and fp16-accumulating variants take bf16 / fp32 only and are skipped for it."""
        half = value.dtype == torch.float16
        out = msda_rows_forward(value, spatial_shapes, level_start_index, loc, attn, row_map)
        ctx.save_for_backward(value, loc, attn, row_map, spatial_shapes, level_start_index)
        ctx.group_order = group_order
        # grad_value accumulated in scaled fp16 -- "f16": every level, ("mixed", level_hw_host, n[, replicas]): the
        # first n levels [and the replicated ones of gv_replicas_for] -- (half the L2 reduction sectors of those
        # levels): only where the caller asks for it
        ctx.gv_mode = gv_mode if (gv_mode is not None and value.dtype == torch.bfloat16 and value.shape[-1] == 32) else None
        ctx.dense = dense if (dense is not None and not half and value.shape[-1] == 32) else None
        ctx.value_early = getattr(value, "_bevf_early", None)     # see plugin/linear.py::shared_input_projections
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        value, loc, attn, row_map, ss, ls = ctx.saved_tensors
        if deterministic():
            # fixed-point grad_value; gv_mode and the dense / split kernels sum in floating point and are bypassed
            gv, gl, ga = msda_backward_fx(value, ss, ls, loc, attn, grad_out.contiguous(), row_map)
            if ctx.value_early is not None and ctx.value_early(gv):
                return None, gl, ga, None, None, None, None, None, None      # converted off the critical path
            return gv.materialize(), gl, ga, None, None, None, None, None, None
        if ctx.gv_mode is not None and grad_out.dtype == torch.bfloat16:
            if ctx.gv_mode == "f16":
                gv, gl, ga = msda_rows_backward_f16acc(value, ss, ls, loc, attn, row_map, grad_out, ctx.group_order,
                                                       lazy=True)
            else:
                hw_host, nfine = ctx.gv_mode[1:3]
                reps = ctx.gv_mode[3] if len(ctx.gv_mode) > 3 else None     # gv_replicas_for, where the caller planned it
                if sum(h * w for h, w in hw_host) != value.shape[1]:
                    # a stale host copy of the pyramid (it no longer adds up to S): plain fp32 accumulation instead
                    gv, gl, ga = msda_rows_backward(value, ss, ls, loc, attn, row_map, grad_out.contiguous(), None,
                                                    group_order=ctx.group_order)
                    if ctx.value_early is not None and ctx.value_early(gv):
                        return None, gl, ga, None, None, None, None, None, None
                    return gv.to(value.dtype), gl, ga, None, None, None, None, None, None
                kd = None
                if ctx.dense is not None and ctx.group_order is None and _lib.load().bevf_msda_get_dense_backward():
                    kd = dense_levels_for(row_map.numel() / max(1, value.shape[0]), loc.shape[3], hw_host)
                if kd is not None:
                    # levels [nfine, kd) fp32 reductions, [kd, L) on the tensor cores, both into the side buffer
                    gv, gl, ga = msda_rows_backward_mixed(value, ss, ls, hw_host, nfine, loc, attn, row_map, grad_out,
                                                          lazy=True, map_range=ctx.dense[1],
                                                          first_dense_level=max(kd, nfine), replicas=reps)
                else:
                    gv, gl, ga = msda_rows_backward_mixed(value, ss, ls, hw_host, nfine, loc, attn, row_map, grad_out,
                                                          ctx.group_order, lazy=True, replicas=reps)
            if ctx.value_early is not None and ctx.value_early(gv):
                return None, gl, ga, None, None, None, None, None, None      # the producer converts it off the critical path
            return gv.materialize(), gl, ga, None, None, None, None, None, None
        # (the coarse levels of an fp32-accumulated pyramid go to the dense kernel only where the caller opted in:
        # bevf_msda_rows_backward_dense is off under the library default)
        gv, gl, ga = msda_rows_backward(value, ss, ls, loc, attn, row_map, grad_out.contiguous(),
                                        group_order=ctx.group_order, dense=ctx.dense)
        if ctx.value_early is not None and ctx.value_early(gv):
            # the producer of `value` took the gradient (conversion + its GEMMs run off the critical path)
            return None, gl, ga, None, None, None, None, None, None
        return gv.to(value.dtype), gl, ga, None, None, None, None, None, None


def sca_prep_forward(raw, ref_cam, pair_q, pair_cam, level_hw, B, Nq, M, L, P):
    _need_cuda(raw, "raw")
    R, D, ncam = pair_q.numel(), ref_cam.shape[3], ref_cam.shape[0]
    loc = torch.empty((B * R, M, L, P, 2), device=raw.device, dtype=torch.float32)
    attn = torch.empty((B * R, M, L, P), device=raw.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(raw.device):
        st = lib.bevf_sca_prep_forward(raw.data_ptr(), ref_cam.data_ptr(), pair_q.data_ptr(),
                                       pair_cam.data_ptr(), level_hw.data_ptr(), loc.data_ptr(),
                                       attn.data_ptr(), B, Nq, R, M, L, P, D, ncam, _stream_ptr(raw))
    _lib.check(st, lib)
    return loc, attn


def sca_prep_backward(raw, grad_loc, grad_attn, pair_of, level_hw, B, Nq, R, M, L, P,
                      out_dtype=torch.float32):
    """d_raw of the SCA sampling-point prep; out_dtype=bfloat16 / float16 rounds in the kernel (the result then
    feeds the 16-bit GEMMs of the head without a cast pass)."""
    ncam = pair_of.shape[0]
    d_raw = torch.empty(raw.shape, device=raw.device, dtype=out_dtype)
    lib = _lib.load()
    with torch.cuda.device(raw.device):
        st = lib.bevf_sca_prep_backward(raw.data_ptr(), grad_loc.data_ptr(), grad_attn.data_ptr(),
                                        pair_of.data_ptr(), level_hw.data_ptr(), d_raw.data_ptr(),
                                        _DT[out_dtype], B, Nq, R, M, L, P, ncam, _stream_ptr(raw))
    _lib.check(st, lib)
    return d_raw


class ScaPrep(Function):
    @staticmethod
    def forward(ctx, raw, ref_cam, pair_q, pair_cam, pair_of, level_hw, B, Nq, M, L, P):
        loc, attn = sca_prep_forward(raw, ref_cam, pair_q, pair_cam, level_hw, B, Nq, M, L, P)
        ctx.save_for_backward(raw, pair_of, level_hw)
        ctx.dims = (B, Nq, pair_q.numel(), M, L, P)
        return loc, attn

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loc, grad_attn):
        raw, pair_of, level_hw = ctx.saved_tensors
        d_raw = sca_prep_backward(raw, grad_loc.contiguous(), grad_attn.contiguous(), pair_of,
                                  level_hw, *ctx.dims)
        return (d_raw,) + (None,) * 10


def sca_rows_forward_fused(value, spatial_shapes, level_start_index, raw, ref_cam, pair_q, pair_cam, row_map, bs, nq,
                           coarse_from=None):
    """SCA's row-list sampler reading the head's raw offsets|logits instead of loc / attn
    (bevf_sca_rows_forward_fused): value (bs*ncam, S, 8, 32) bf16, raw (bs*Nq, 768) f32, ref_cam (ncam, bs, Nq, Dz, 2)
    f32, pair_q / pair_cam (pairs,) int32, row_map (bs*pairs,) int32.  Returns (out (bs*pairs, 256) bf16, stats
    (bs*pairs*8, 2) f32 -- the softmax statistics the backward recomputes the samples from --, coarse) where coarse is
    None or, with ``coarse_from``, the samples of the levels [coarse_from, L) as (loc, attn, coarse_from): what the
    backward's dense tensor-core kernel reads."""
    for t, n in ((value, "value"), (raw, "raw"), (ref_cam, "ref_cam"), (pair_q, "pair_q"), (pair_cam, "pair_cam"),
                 (row_map, "row_map")):
        _need_cuda(t, n)
    NB, S, M, D = value.shape
    L = int(torch.as_tensor(spatial_shapes).shape[0])
    P = raw.shape[1] // (3 * M * L)
    R = row_map.numel()
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    out = torch.empty((R, M * D), device=value.device, dtype=value.dtype)
    stats = torch.empty((R * M, 2), device=value.device, dtype=torch.float32)
    coarse = None
    if coarse_from is not None and 0 <= coarse_from < L:
        nl = L - coarse_from
        coarse = (torch.empty((R, M, nl, P, 2), device=value.device, dtype=torch.float32),
                  torch.empty((R, M, nl, P), device=value.device, dtype=torch.float32), int(coarse_from))
    lib = _lib.load()
    with torch.cuda.device(value.device), _timed("msda_rows_forward", value.device, (R, L)):
        st = lib.bevf_sca_rows_forward_fused(value.data_ptr(), _DT[value.dtype], ss.data_ptr(), ls.data_ptr(),
                                             raw.data_ptr(), ref_cam.data_ptr(), pair_q.data_ptr(), pair_cam.data_ptr(),
                                             stats.data_ptr(), _ptr(coarse and coarse[0]), _ptr(coarse and coarse[1]),
                                             L if coarse is None else coarse[2], out.data_ptr(), _DT[value.dtype],
                                             row_map.data_ptr(), NB, S, M, D, R, L, P, bs, nq, pair_q.numel(),
                                             ref_cam.shape[3], ref_cam.shape[0], _stream_ptr(value))
    _lib.check(st, lib)
    return out, stats, coarse


def sca_rows_backward_fused(value, spatial_shapes, level_start_index, level_hw_host, num_f16_levels, raw, stats,
                            ref_cam, pair_q, pair_cam, pair_of, row_map, grad_output, bs, nq, map_range=None,
                            first_dense_level=None, coarse=None, replicas=None):
    """Backward of sca_rows_forward_fused with msda_rows_backward_mixed's grad_value accumulation (``map_range``: the
    coarse levels from ``first_dense_level`` on through the dense tensor-core kernel, which reads the forward's
    ``coarse`` samples; without them those levels stay on the reduction path).  Returns (grad_value as a
    LazyGradValue, d_raw (bs*Nq, 768) bf16): the sampler finishes the d_raw rows of queries seen by one camera, the
    finish kernel (bevf_sca_prep_backward_multi) the others from the sampler's grad_loc / grad_attn.  ``replicas``: as
    for msda_rows_backward_mixed (bevf_sca_rows_backward_fused_replicated)."""
    import ctypes
    for t, n in ((value, "value"), (raw, "raw"), (stats, "stats"), (ref_cam, "ref_cam"), (pair_of, "pair_of"),
                 (row_map, "row_map"), (grad_output, "grad_output")):
        _need_cuda(t, n)
    alert_not_deterministic("sca_rows_backward_fused (grad_value summed with fp16 / fp32 atomics)")
    NB, S, M, D = value.shape
    L = len(level_hw_host)
    P = raw.shape[1] // (3 * M * L)
    R = row_map.numel()
    if not (1 <= num_f16_levels < L):
        raise RuntimeError("fused SCA backward: num_f16_levels does not fit the pyramid")
    ss, ls = _level_tensors(value, spatial_shapes, level_start_index)
    nrep, k = replica_plan(replicas, num_f16_levels)
    s_fine = sum(int(h) * int(w) for h, w in level_hw_host[:num_f16_levels])
    s_rep = sum(int(h) * int(w) for h, w in level_hw_host[num_f16_levels:num_f16_levels + nrep])
    grad_output = grad_output.contiguous()
    # scratch of the pair rows whose query more than one camera sees (only those rows are written)
    grad_loc = torch.empty((R, M, L, P, 2), device=value.device, dtype=torch.float32)
    grad_attn = torch.empty((R, M, L, P), device=value.device, dtype=torch.float32)
    d_raw = torch.empty(raw.shape, device=value.device, dtype=torch.bfloat16)
    hw = (ctypes.c_int32 * (2 * L))(*[int(v) for hw_ in level_hw_host for v in hw_])
    lib = _lib.load()
    with torch.cuda.device(value.device), _timed("msda_rows_backward", value.device, (R, L)):
        amax = abs_max_bits(grad_output)
        fine = torch.zeros((NB, s_fine + k * s_rep, M, D), device=value.device, dtype=torch.float16)
        side = torch.zeros((NB, S - s_fine - s_rep, M, D), device=value.device, dtype=torch.float32)
        kd = num_f16_levels + nrep if first_dense_level is None else int(first_dense_level)
        head = (value.data_ptr(), _DT[value.dtype], ss.data_ptr(), ls.data_ptr(), ctypes.addressof(hw), raw.data_ptr(),
                stats.data_ptr(), _ptr(coarse and coarse[0]), _ptr(coarse and coarse[1]),
                L if coarse is None else coarse[2], ref_cam.data_ptr(), pair_q.data_ptr(), pair_cam.data_ptr(),
                pair_of.data_ptr(), grad_output.data_ptr(), _DT[grad_output.dtype], fine.data_ptr(), _ptr(side),
                amax.data_ptr(), int(num_f16_levels))
        tail = (kd, grad_loc.data_ptr(), grad_attn.data_ptr(), d_raw.data_ptr(), row_map.data_ptr(), _ptr(map_range),
                NB, S, M, D, R, L, P, bs, nq, pair_q.numel(), ref_cam.shape[3], ref_cam.shape[0], _stream_ptr(value))
        if nrep:
            st = lib.bevf_sca_rows_backward_fused_replicated(*head, nrep, k, *tail)
        else:
            st = lib.bevf_sca_rows_backward_fused(*head, *tail)
        _lib.check(st, lib)
    st = lib.bevf_sca_prep_backward_multi(raw.data_ptr(), grad_loc.data_ptr(), grad_attn.data_ptr(), pair_of.data_ptr(),
                                          ss.data_ptr(), d_raw.data_ptr(), BF16, bs, nq, pair_q.numel(), M, L, P,
                                          pair_of.shape[0], _stream_ptr(value))
    _lib.check(st, lib)
    return LazyGradValue(value.shape, fine, side if side.numel() else None, amax,
                         (s_fine, s_rep, k) if nrep else None), d_raw


def tsa_prep_forward(raw, ref2d, level_hw, B, Nq, M, L, P, interleave=False):
    _need_cuda(raw, "raw")
    shape = (B * Nq * 2, M, L, P) if interleave else (B * 2, Nq, M, L, P)
    loc = torch.empty(shape + (2,), device=raw.device, dtype=torch.float32)
    attn = torch.empty(shape, device=raw.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(raw.device):
        st = lib.bevf_tsa_prep_forward(raw.data_ptr(), ref2d.data_ptr(), level_hw.data_ptr(),
                                       loc.data_ptr(), attn.data_ptr(), B, Nq, M, L, P,
                                       int(interleave), _stream_ptr(raw))
    _lib.check(st, lib)
    return loc, attn


def tsa_prep_backward(raw, grad_loc, grad_attn, level_hw, B, Nq, M, L, P, interleave=0,
                      out_dtype=torch.float32):
    d_raw = torch.empty(raw.shape, device=raw.device, dtype=out_dtype)
    lib = _lib.load()
    with torch.cuda.device(raw.device):
        st = lib.bevf_tsa_prep_backward(raw.data_ptr(), grad_loc.contiguous().data_ptr(),
                                        grad_attn.contiguous().data_ptr(), level_hw.data_ptr(),
                                        d_raw.data_ptr(), _DT[out_dtype], B, Nq, M, L, P,
                                        int(interleave), _stream_ptr(raw))
    _lib.check(st, lib)
    return d_raw


class TsaPrep(Function):
    @staticmethod
    def forward(ctx, raw, ref2d, level_hw, B, Nq, M, L, P, interleave=False):
        loc, attn = tsa_prep_forward(raw, ref2d, level_hw, B, Nq, M, L, P, interleave)
        ctx.save_for_backward(raw, level_hw)
        ctx.dims = (B, Nq, M, L, P, int(interleave))
        return loc, attn

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loc, grad_attn):
        raw, level_hw = ctx.saved_tensors
        d_raw = tsa_prep_backward(raw, grad_loc, grad_attn, level_hw, *ctx.dims)
        return (d_raw,) + (None,) * 8


def query_prep_forward(raw, ref2d, level_hw, B, Nq, M, L, P, F, interleave=False):
    """(loc, attn) of the query-side sampling points for F frames (bevf_query_prep_forward); F = 2 is TSA's
    tsa_prep_forward, F = 1 the decoder's CustomMSDeformableAttention."""
    _need_cuda(raw, "raw")
    shape = (B * Nq * F, M, L, P) if interleave else (B * F, Nq, M, L, P)
    loc = torch.empty(shape + (2,), device=raw.device, dtype=torch.float32)
    attn = torch.empty(shape, device=raw.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(raw.device):
        st = lib.bevf_query_prep_forward(raw.data_ptr(), ref2d.data_ptr(), level_hw.data_ptr(), loc.data_ptr(),
                                         attn.data_ptr(), B, Nq, M, L, P, F, int(interleave), _stream_ptr(raw))
    _lib.check(st, lib)
    return loc, attn


def query_prep_backward(raw, grad_loc, grad_attn, level_hw, B, Nq, M, L, P, F, interleave=0,
                        out_dtype=torch.float32):
    d_raw = torch.empty(raw.shape, device=raw.device, dtype=out_dtype)
    lib = _lib.load()
    with torch.cuda.device(raw.device):
        st = lib.bevf_query_prep_backward(raw.data_ptr(), grad_loc.contiguous().data_ptr(),
                                          grad_attn.contiguous().data_ptr(), level_hw.data_ptr(), d_raw.data_ptr(),
                                          _DT[out_dtype], B, Nq, M, L, P, F, int(interleave), _stream_ptr(raw))
    _lib.check(st, lib)
    return d_raw


class QueryPrep(Function):
    """query_prep_forward as an autograd node on an fp32 ``raw`` (the 16-bit path fuses it with the head GEMM,
    plugin.linear)."""

    @staticmethod
    def forward(ctx, raw, ref2d, level_hw, B, Nq, M, L, P, F):
        loc, attn = query_prep_forward(raw, ref2d, level_hw, B, Nq, M, L, P, F)
        ctx.save_for_backward(raw, level_hw)
        ctx.dims = (B, Nq, M, L, P, F)
        return loc, attn

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loc, grad_attn):
        raw, level_hw = ctx.saved_tensors
        d_raw = query_prep_backward(raw, grad_loc, grad_attn, level_hw, *ctx.dims)
        return (d_raw,) + (None,) * 8


def refine_points(tmp, ref, with_ref2d=True):
    """DetectionTransformerDecoder's reference-point refinement (decoder.py:106-118) in one kernel:
    sigmoid(tmp[..., (0, 1, 4)] + inverse_sigmoid(ref)) for ref (..., 3) and the regression output tmp (..., >= 5),
    both in one dtype; tmp is read in place (its last dim must be contiguous).  Returns (new ref (..., 3) in that
    dtype, its x, y as a contiguous (..., 1, 2) fp32 tensor -- the next layer's prep input -- or None).  No autograd:
    the result is detached, as in the reference."""
    _need_cuda(ref, "ref")
    if tmp.dtype != ref.dtype:
        raise RuntimeError(f"refine_points: tmp ({tmp.dtype}) and ref ({ref.dtype}) must share one dtype")
    if ref.shape[-1] != 3 or tmp.shape[:-1] != ref.shape[:-1] or tmp.shape[-1] < 5:
        raise RuntimeError(f"refine_points: shapes {tuple(tmp.shape)} / {tuple(ref.shape)}: need (..., >=5) / (..., 3)")
    rows = ref.numel() // 3
    tmp2 = tmp.reshape(rows, tmp.shape[-1])
    if tmp2.stride(1) != 1:
        tmp2 = tmp2.contiguous()
    ref = ref.contiguous()
    out = torch.empty_like(ref)
    ref2d = torch.empty(ref.shape[:-1] + (1, 2), device=ref.device, dtype=torch.float32) if with_ref2d else None
    lib = _lib.load()
    with torch.cuda.device(ref.device):
        st = lib.bevf_refine_points(tmp2.data_ptr(), tmp2.stride(0), ref.data_ptr(), out.data_ptr(), _ptr(ref2d),
                                    _DT[ref.dtype], rows, _stream_ptr(ref))
    _lib.check(st, lib)
    return out, ref2d


def _ptr(t):
    return 0 if t is None else t.data_ptr()


_seed_counter = [0]
_seed_state: dict = {}        # device -> int64[1] step counter living on the device
_seed_snap: dict = {}         # device -> int64[1] copy of the counter taken by the last advance_seed()


def seed_state(device) -> torch.Tensor:
    """The dropout step key the kernels of the CURRENT forward read: the snapshot taken by the last
    ``advance_seed`` (the persistent counter itself before the first one).  Autograd nodes keep the
    tensor they were given, so a backward always regenerates the masks of its own forward even when
    other training-mode forwards ran in between."""
    key = torch.device(device)
    if key in _seed_snap:
        return _seed_snap[key]
    if key not in _seed_state:
        _seed_state[key] = torch.zeros(1, dtype=torch.int64, device=key)
    return _seed_state[key]


def advance_seed(device) -> None:
    """Bump the device-side dropout step counter and snapshot it (two tiny kernels; capturable in a
    CUDA graph: the in-place add lives on a persistent tensor, so every replay of a captured training
    step draws new masks, and the snapshot is recomputed by the replay)."""
    key = torch.device(device)
    if key not in _seed_state:
        _seed_state[key] = torch.zeros(1, dtype=torch.int64, device=key)
    _seed_state[key].add_(0x9E3779B97F4A7C1)
    _seed_snap[key] = _seed_state[key].clone()


def _next_seed() -> int:
    """A fresh 63-bit Philox key per dropout site, derived from torch's global seed (so
    torch.manual_seed makes runs repeatable) without touching the device."""
    _seed_counter[0] += 1
    return (torch.initial_seed() * 6364136223846793005 + _seed_counter[0] * 1442695040888963407) & ((1 << 63) - 1)


def _param_ptr(p, act_dtype):
    """Parameters are read in their own dtype when the kernel supports the combination."""
    if p.dtype == act_dtype or p.dtype == torch.float32:
        q = p.detach().contiguous()
    else:
        q = p.detach().float().contiguous()
    return q, _DT[q.dtype]


class LayerNormResidual(Function):
    """y = LayerNorm(dropout_p(x) + residual) * gamma + beta (fp32 statistics); residual may be None.
    The dropout keep-mask is regenerated from a Philox seed in backward (nothing stored).
    With ``pos`` the kernel also writes y + pos (the next block's positional-encoded query) and the
    call returns (y, y + pos); their two gradients are summed inside the backward kernel.
    With ``twin`` the call returns (y, y') where y' aliases y: the caller feeds y to the next block and y'
    to that block's residual connection, so their two gradients arrive separately and are summed inside
    the backward kernel too (autograd would otherwise add them with a three-pass elementwise kernel)."""

    @staticmethod
    def forward(ctx, x, residual, gamma, beta, eps, drop_p=0.0, pos=None, twin=False):
        _need_cuda(x, "x")
        if x.dtype not in _DT:
            raise RuntimeError("layernorm: float32, bfloat16 or float16 only")
        C = x.shape[-1]
        rows = x.numel() // C
        rc = None if residual is None else residual.contiguous()
        g, pd = _param_ptr(gamma, x.dtype)
        b, pd2 = _param_ptr(beta, x.dtype)
        if pd != pd2:
            g, b, pd = g.float(), b.float(), F32
        y = torch.empty_like(x)
        y2 = None
        if pos is not None:
            if pos.dtype != x.dtype or pos.numel() != x.numel():
                raise RuntimeError("layernorm: pos must match x in dtype and size")
            pos = pos.contiguous()
            y2 = torch.empty_like(x)
        mean = torch.empty(rows, device=x.device, dtype=torch.float32)
        rstd = torch.empty(rows, device=x.device, dtype=torch.float32)
        seed = _next_seed() if drop_p > 0.0 else 0
        sbase = seed_state(x.device) if drop_p > 0.0 else None
        lib = _lib.load()
        with torch.cuda.device(x.device):
            st = lib.bevf_layernorm_forward(x.data_ptr(), _ptr(rc), g.data_ptr(), b.data_ptr(), pd,
                                            _ptr(pos), y.data_ptr(), _ptr(y2), mean.data_ptr(),
                                            rstd.data_ptr(), rows, C, float(eps), float(drop_p), seed,
                                            _ptr(sbase), _DT[x.dtype], _stream_ptr(x))
        _lib.check(st, lib)
        ctx.save_for_backward(x, rc, g, mean, rstd)
        from .arena import arena_of
        ctx.arena, ctx.arena_accs = arena_of(gamma, beta)            # flat gradient arena, when enabled
        ctx.arena_params = (gamma, beta) if ctx.arena is not None else None
        ctx.sbase = sbase                 # the step key of THIS forward (see seed_state)
        ctx.pos_shape = None if pos is None else tuple(pos.shape)
        ctx.meta = (residual is not None, gamma.dtype, beta.dtype, pd, float(drop_p), seed, pos is not None)
        if pos is None and twin:
            return y, y.view(y.shape)
        return y if pos is None else (y, y2)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy, dy2=None):
        x, res, g, mean, rstd = ctx.saved_tensors
        has_res, gdt, bdt, pd, drop_p, seed, has_pos = ctx.meta
        C = x.shape[-1]
        rows = x.numel() // C
        # d(y + pos)/d pos = 1: pos (the learned BEV positional encoding) receives the gradient of y2
        d_pos = None
        if has_pos and ctx.needs_input_grad[6] and dy2 is not None:
            d_pos = dy2.reshape(ctx.pos_shape)
        if dy is None:                                   # only y + pos was used downstream
            dy, dy2 = dy2, None
        dy = dy.contiguous()
        ld2 = 0
        if dy2 is not None:
            # usually a column slice of the gradient of cat([prev_bev, query + pos]): rows at a
            # uniform stride are read in place
            r2 = dy2.reshape(-1, C) if dy2.is_contiguous() else dy2
            uniform = (r2.stride(-1) == 1 and r2.dim() >= 2 and r2.stride(-2) >= C
                       and all(r2.stride(i) == r2.stride(i + 1) * r2.shape[i + 1] for i in range(r2.dim() - 2))
                       and r2.stride(-2) % 8 == 0 and r2.data_ptr() % 16 == 0)
            if uniform:
                ld2 = int(r2.stride(-2))
                dy2 = r2
            else:
                dy2 = dy2.contiguous()
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if (has_res and drop_p > 0.0) else None
        if ctx.arena is not None:
            ctx.arena.touch(*ctx.arena_params)
            dgb = ctx.arena_accs                                    # accumulate straight into the arena
        else:
            dgb = torch.zeros(2, C, device=x.device, dtype=torch.float32)
        lib = _lib.load()
        with torch.cuda.device(x.device):
            args = (x.data_ptr(), _ptr(res), g.data_ptr(), pd, mean.data_ptr(), rstd.data_ptr(), dy.data_ptr(),
                    _ptr(dy2), ld2, dx.data_ptr(), _ptr(dres), dgb[0].data_ptr(), dgb[1].data_ptr())
            tail = (rows, C, drop_p, seed, _ptr(ctx.sbase) if drop_p > 0.0 else 0, _DT[x.dtype], _stream_ptr(x))
            if deterministic():
                need = int(lib.bevf_layernorm_backward_workspace_bytes(rows, C))
                ws = torch.empty(max(need, 16), device=x.device, dtype=torch.uint8)
                st = lib.bevf_layernorm_backward_det(*args, ws.data_ptr(), need, *tail)
            else:
                st = lib.bevf_layernorm_backward(*args, *tail)
        _lib.check(st, lib)
        d_res = None if not has_res else (dres if dres is not None else dx)
        if ctx.arena is not None:
            return dx, d_res, None, None, None, None, d_pos, None
        return dx, d_res, dgb[0].to(gdt), dgb[1].to(bdt), None, None, d_pos, None


class ScaCombine(Function):
    """Per-query mean over the cameras that see it (spatial_cross_attention.py:165-172)."""

    @staticmethod
    def forward(ctx, out, pair_of, pair_q, inv_count, B, Nq):
        _need_cuda(out, "out")
        C = out.shape[-1]
        R = pair_q.numel()
        ncam = pair_of.shape[0]
        slots = torch.empty((B, Nq, C), device=out.device, dtype=out.dtype)
        lib = _lib.load()
        with torch.cuda.device(out.device):
            st = lib.bevf_sca_combine_forward(out.data_ptr(), pair_of.data_ptr(),
                                              inv_count.data_ptr(), slots.data_ptr(), B, Nq, R, C,
                                              ncam, _DT[out.dtype], _stream_ptr(out))
        _lib.check(st, lib)
        ctx.save_for_backward(pair_q, inv_count)
        ctx.dims = (B, Nq, R, C)
        return slots

    @staticmethod
    @once_differentiable
    def backward(ctx, g_slots):
        pair_q, inv_count = ctx.saved_tensors
        B, Nq, R, C = ctx.dims
        g_slots = g_slots.contiguous()
        g_out = torch.empty((B * R, C), device=g_slots.device, dtype=g_slots.dtype)
        lib = _lib.load()
        with torch.cuda.device(g_slots.device):
            st = lib.bevf_sca_combine_backward(g_slots.data_ptr(), pair_q.data_ptr(),
                                               inv_count.data_ptr(), g_out.data_ptr(), B, Nq, R, C,
                                               _DT[g_slots.dtype], _stream_ptr(g_slots))
        _lib.check(st, lib)
        return g_out, None, None, None, None, None


def sca_plan_build(mask_u8, qorder, capacity):
    """Device-side pair list (bevf_sca_plan_build): mask_u8 (ncam, B, Nq, D) uint8, qorder (Nq,) int32 or
    None -> dict of the plan tensors; no host synchronisation."""
    _need_cuda(mask_u8, "bev_mask")
    if mask_u8.dtype != torch.uint8:
        raise RuntimeError("bev_mask must be uint8")
    ncam, B, Nq, D = mask_u8.shape
    dev = mask_u8.device
    lib = _lib.load()
    i32 = dict(device=dev, dtype=torch.int32)
    out = dict(pair_q=torch.empty(capacity, **i32), pair_cam=torch.empty(capacity, **i32),
               pair_of=torch.empty((ncam, Nq), **i32), row_map=torch.empty(B * capacity, **i32),
               inv_count=torch.empty((B, Nq), device=dev, dtype=torch.float32),
               map_range=torch.empty((B * ncam, 2), **i32), counters=torch.empty(2, **i32))
    ws = torch.empty(int(lib.bevf_sca_plan_workspace_ints(ncam, Nq)), **i32)
    with torch.cuda.device(dev):
        st = lib.bevf_sca_plan_build(mask_u8.data_ptr(), _ptr(qorder), out["pair_q"].data_ptr(),
                                     out["pair_cam"].data_ptr(), out["pair_of"].data_ptr(),
                                     out["row_map"].data_ptr(), out["inv_count"].data_ptr(),
                                     out["map_range"].data_ptr(), out["counters"].data_ptr(), ws.data_ptr(),
                                     B, ncam, Nq, D,
                                     int(capacity), _stream_ptr(mask_u8))
    _lib.check(st, lib)
    return out


def point_sampling(lidar2img, pc_range, z_norm, img_h, img_w, bev_h, bev_w, raw_mask=False):
    """lidar2img (B, ncam, 4, 4) f32 CUDA -> ref_cam (ncam,B,Nq,D,2) f32, bev_mask (ncam,B,Nq,D) bool
    (uint8 with ``raw_mask``: what the device-side plan builder reads)."""
    _need_cuda(lidar2img, "lidar2img")
    import ctypes
    B, ncam = lidar2img.shape[:2]
    D = len(z_norm)
    Nq = bev_h * bev_w
    ref_cam = torch.empty((ncam, B, Nq, D, 2), device=lidar2img.device, dtype=torch.float32)
    mask = torch.empty((ncam, B, Nq, D), device=lidar2img.device, dtype=torch.uint8)
    pc = (ctypes.c_float * 6)(*[float(v) for v in pc_range])
    zs = (ctypes.c_float * D)(*[float(v) for v in z_norm])
    lib = _lib.load()
    with torch.cuda.device(lidar2img.device):
        st = lib.bevf_point_sampling(lidar2img.data_ptr(), ctypes.addressof(pc), ctypes.addressof(zs),
                                     float(img_h), float(img_w), ref_cam.data_ptr(),
                                     mask.data_ptr(), B, ncam, bev_h, bev_w, D,
                                     _stream_ptr(lidar2img))
    _lib.check(st, lib)
    return ref_cam, (mask if raw_mask else mask.bool())


def linear_tc(x, weight, bias=None, residual=None, relu=False, out_dtype=None):
    """y = act(x @ weight.T + bias) (+ residual) on the wgmma GEMM.  x (..., K) and weight (N, K) both bf16 or
    both fp16, bias (N) any float dtype, residual (..., N) in x's dtype; returns (..., N) in x's dtype (default)
    or fp32.  Strided operands are copied to contiguous ones first."""
    x = x.contiguous()
    _need_cuda(x, "x")
    if x.dtype not in TC_DTYPES or weight.dtype != x.dtype:
        raise RuntimeError("linear_tc: x and weight must be both bfloat16 or both float16")
    K = x.shape[-1]
    if weight.dim() != 2 or weight.shape[1] != K:
        raise RuntimeError(f"linear_tc: weight must be (N, {K}) for x (..., {K}), got {tuple(weight.shape)}")
    N = weight.shape[0]
    M = x.numel() // K
    out_shape = x.shape[:-1] + (N,)
    if bias is not None and (bias.dim() != 1 or bias.shape[0] != N):
        raise RuntimeError(f"linear_tc: bias must be ({N},), got {tuple(bias.shape)}")
    if residual is not None and (residual.dtype != x.dtype or residual.shape != out_shape):
        raise RuntimeError(f"linear_tc: residual must be {tuple(out_shape)} in {x.dtype}, got "
                           f"{tuple(residual.shape)} in {residual.dtype}")
    w = weight.contiguous()
    bq, bdt = (None, F32) if bias is None else _param_ptr(bias, x.dtype)
    res = None if residual is None else residual.contiguous()
    out_dtype = out_dtype or x.dtype
    y = torch.empty(out_shape, device=x.device, dtype=out_dtype)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        st = lib.bevf_linear_forward_dt(x.data_ptr(), w.data_ptr(), _ptr(bq), bdt, _ptr(res), y.data_ptr(),
                                        _DT[out_dtype], M, N, K, int(bool(relu)), _DT[x.dtype], _stream_ptr(x))
    _lib.check(st, lib)
    return y


def linear_dgrad_tc(dy, weight, addend=None):
    """dx = dy @ weight (+ addend) on the wgmma GEMM, the weight (N, K) read in place (no transposed
    copy).  dy (M, N) bf16 / fp16 -> (M, K) of the same dtype; ``addend`` (M, K) of that dtype is summed in the
    epilogue.  N or K not a multiple of 64: falls back to the transposed-copy form."""
    _need_cuda(dy, "dy")
    if dy.dtype not in TC_DTYPES or weight.dtype != dy.dtype or dy.shape[-1] != weight.shape[0]:
        raise RuntimeError("linear_dgrad_tc: dy (M,N) and weight (N,K) must be both bfloat16 or both float16")
    N, K = weight.shape
    if N % 64 or K % 64 or os.environ.get("BEVF_DGRAD", "mn") == "copy":
        dx = linear_tc(dy, weight.t().contiguous())
        return dx if addend is None else dx + addend.view(dx.shape)
    dy = dy.contiguous()
    w = weight.contiguous()
    M = dy.numel() // N
    dx = torch.empty(dy.shape[:-1] + (K,), device=dy.device, dtype=dy.dtype)
    lib = _lib.load()
    with torch.cuda.device(dy.device):
        if addend is None:
            st = lib.bevf_linear_dgrad_dt(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), M, N, K, _DT[dy.dtype],
                                          _stream_ptr(dy))
        else:
            if addend.dtype != dy.dtype or addend.numel() != M * K or not addend.is_contiguous():
                raise RuntimeError("linear_dgrad_tc: addend must be a contiguous (M, K) tensor of dy's dtype")
            st = lib.bevf_linear_dgrad_acc_dt(dy.data_ptr(), w.data_ptr(), addend.data_ptr(), dx.data_ptr(), M, N, K,
                                              _DT[dy.dtype], _stream_ptr(dy))
    _lib.check(st, lib)
    return dx


def _wgrad_operands(dy, x, who):
    """dy (M, N) and x (M, K) as contiguous CUDA tensors of one tensor-core dtype: (dy, x, M, N, K)."""
    if dy.dim() != 2 or x.dim() != 2:
        raise RuntimeError(f"{who}: dy (M,N) and x (M,K) must be 2-D, got {tuple(dy.shape)} and {tuple(x.shape)}")
    dy, x = dy.contiguous(), x.contiguous()
    _need_cuda(dy, "dy")
    _need_cuda(x, "x")
    if dy.dtype not in TC_DTYPES or x.dtype != dy.dtype or dy.shape[0] != x.shape[0]:
        raise RuntimeError(f"{who}: dy (M,N) and x (M,K) must be both bfloat16 or both float16 with equal M")
    return dy, x, dy.shape[0], dy.shape[1], x.shape[1]


def linear_wgrad_tc(dy, x, with_bias=False, out_dtype=None):
    """dW = dy^T @ x on the wgmma split-M kernel (and db = column sums of dy from the same pass).
    dy (M, N), x (M, K) both bf16 or both fp16 -> (N, K) fp32 [, (N,) fp32].  The kernel accumulates in one fp32
    buffer holding [dW | db]; ``out_dtype`` converts that buffer once (dW and db are views of it)."""
    dy, x, M, N, K = _wgrad_operands(dy, x, "linear_wgrad_tc")
    npad = (N + 3) // 4 * 4
    buf = torch.zeros(N * K + (npad if with_bias else 0), device=x.device, dtype=torch.float32)
    dw = buf[: N * K].view(N, K)
    db = buf[N * K: N * K + N] if with_bias else None
    _wgrad_acc(dy, x, dw, db)
    if out_dtype is not None and out_dtype != torch.float32:
        buf = buf.to(out_dtype)
        dw = buf[: N * K].view(N, K)
        db = buf[N * K: N * K + N] if with_bias else None
    return (dw, db) if with_bias else dw


def linear_wgrad_into(dy, x, dw_acc, db_acc=None):
    """dW += dy^T @ x (and db += column sums of dy) accumulated into caller-provided fp32 buffers (the
    gradient arena): no allocation, no zero-fill, no conversion here."""
    dy, x, M, N, K = _wgrad_operands(dy, x, "linear_wgrad_into")
    if dw_acc.dtype != torch.float32 or dw_acc.numel() != N * K or not dw_acc.is_contiguous():
        raise RuntimeError("linear_wgrad_into: dw_acc must be a contiguous fp32 (N, K) buffer")
    if db_acc is not None and (db_acc.dtype != torch.float32 or db_acc.numel() != N or not db_acc.is_contiguous()):
        raise RuntimeError("linear_wgrad_into: db_acc must be a contiguous fp32 (N,) buffer")
    _wgrad_acc(dy, x, dw_acc, db_acc)


def _wgrad_acc(dy, x, dw, db):
    """dw += dy^T x (db += column sums of dy): split-M partial tiles reduced into dw with fp32 atomics, or -- in
    deterministic mode -- stored into per-split slabs and summed in split order (bevf_linear_wgrad_into)."""
    M, N = dy.shape
    K = x.shape[1]
    lib = _lib.load()
    with torch.cuda.device(x.device):
        if deterministic() and M > 0:
            need = int(lib.bevf_linear_wgrad_workspace_bytes(M, N, K))
            ws = torch.empty(need, device=x.device, dtype=torch.uint8)
            st = lib.bevf_linear_wgrad_into_dt(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), _ptr(db), ws.data_ptr(),
                                               need, M, N, K, _DT[x.dtype], _stream_ptr(x))
        else:
            st = lib.bevf_linear_wgrad_dt(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), _ptr(db), M, N, K, _DT[x.dtype],
                                          _stream_ptr(x))
    _lib.check(st, lib)


def linear_wgrad_out(dy, x, grad_dtype, with_bias):
    """Two-pass weight (+ bias) gradient written directly in ``grad_dtype``: returns (dW, db|None)."""
    dy, x, M, N, K = _wgrad_operands(dy, x, "linear_wgrad_out")
    if M == 0:
        return (torch.zeros((N, K), device=x.device, dtype=grad_dtype),
                torch.zeros((N,), device=x.device, dtype=grad_dtype) if with_bias else None)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        need = int(lib.bevf_linear_wgrad_workspace_bytes(M, N, K))
        ws = torch.empty(need, device=x.device, dtype=torch.uint8)
        dw = torch.empty((N, K), device=x.device, dtype=grad_dtype)
        db = torch.empty((N,), device=x.device, dtype=grad_dtype) if with_bias else None
        st = lib.bevf_linear_wgrad_out_dt(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), _ptr(db),
                                          _DT[grad_dtype], ws.data_ptr(), need, M, N, K, _DT[x.dtype], _stream_ptr(x))
    _lib.check(st, lib)
    return dw, db


def sum_tensors(ts):
    """Sum of up to 8 equally-shaped contiguous bf16 / f32 CUDA tensors in one pass (fp32 accumulation)."""
    import ctypes
    ts = [t.contiguous() for t in ts]
    if len(ts) == 1:
        return ts[0]
    t0 = ts[0]
    _need_cuda(t0, "tensors[0]")
    if len(ts) > 8 or any(t.shape != t0.shape or t.dtype != t0.dtype for t in ts) or t0.dtype not in _DT:
        raise RuntimeError("sum_tensors: 1..8 tensors of one shape, float32, bfloat16 or float16")
    out = torch.empty_like(t0)
    arr = (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
    lib = _lib.load()
    with torch.cuda.device(t0.device):
        st = lib.bevf_sum_tensors(ctypes.addressof(arr), len(ts), out.data_ptr(), t0.numel(), _DT[t0.dtype],
                                  _stream_ptr(t0))
    _lib.check(st, lib)
    return out


def colsum(x):
    """fp32 column sums of a (rows, C) tensor (bias gradients)."""
    _need_cuda(x, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    out = torch.zeros(C, device=x.device, dtype=torch.float32)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        if deterministic() and rows > 0:
            need = int(lib.bevf_colsum_workspace_bytes(rows, C))
            ws = torch.empty(need, device=x.device, dtype=torch.uint8)
            st = lib.bevf_colsum_det(x.data_ptr(), out.data_ptr(), ws.data_ptr(), need, rows, C, _DT[x.dtype],
                                     _stream_ptr(x))
        else:
            st = lib.bevf_colsum(x.data_ptr(), out.data_ptr(), rows, C, _DT[x.dtype], _stream_ptr(x))
    _lib.check(st, lib)
    return out


def dropout_inplace_(x, p):
    """x *= keep / (1 - p) in place with Philox bits keyed by the device-side step counter."""
    _need_cuda(x, "x")
    if p <= 0.0:
        return x
    lib = _lib.load()
    with torch.cuda.device(x.device):
        st = lib.bevf_dropout_inplace(x.data_ptr(), x.numel(), float(p), _next_seed(),
                                      seed_state(x.device).data_ptr(), _DT[x.dtype], _stream_ptr(x))
    _lib.check(st, lib)
    return x


def relu_dropout_backward(dy, h, p):
    """Gradient w.r.t. z of h = dropout_p(relu(z)), from the saved h alone."""
    _need_cuda(dy, "dy")
    _need_cuda(h, "h")
    if h.dtype != dy.dtype or h.numel() != dy.numel():
        raise RuntimeError("relu_dropout_backward: h must match dy in dtype and size")
    out = torch.empty_like(dy)
    lib = _lib.load()
    with torch.cuda.device(dy.device):
        st = lib.bevf_relu_dropout_backward(dy.data_ptr(), h.data_ptr(), out.data_ptr(), dy.numel(),
                                            1.0 / (1.0 - p), _DT[dy.dtype], _stream_ptr(dy))
    _lib.check(st, lib)
    return out


# ---------------------------------------------------------------------------------------------------
# Device-resident ego-motion (csrc/ego_motion.cu): the per-frame shift / rotation / CAN-bus block of
# PerceptionTransformer.get_bev_features without host arithmetic.
# ---------------------------------------------------------------------------------------------------
EGO_DELTAS, EGO_CONTINUE, EGO_NEW_SCENE = (_lib.ENUMS["BEVF_EGO_DELTAS"], _lib.ENUMS["BEVF_EGO_CONTINUE"],
                                          _lib.ENUMS["BEVF_EGO_NEW_SCENE"])


def ego_state(device) -> torch.Tensor:
    """An empty stream-state block for ``ego_motion`` (previous position (3 doubles), previous angle, has-history
    word): int64[5] zeros; ``state.view(torch.float64)[:4]`` reads the doubles."""
    return torch.zeros(5, device=device, dtype=torch.int64)


def ego_motion(can_bus, bev_h, bev_w, grid_length, rotate_center, use_shift, out_dtype, state=None,
               mode=EGO_DELTAS):
    """can_bus (bs, 18) float64 CUDA -> (shift (bs, 2) f32, rot (bs, 6) f32, can_bus_mlp_in (bs, 18) out_dtype);
    see bevf_ego_motion in the header.  ``out_dtype`` is the dtype the host path's ``bev_queries.new_tensor`` would
    round to.  With ``state`` (``ego_state``) and a stream mode, sample 0's absolute position / angle are turned
    into deltas on the device and the state is advanced.  No host synchronisation."""
    _need_cuda(can_bus, "can_bus")
    if can_bus.dtype != torch.float64 or can_bus.dim() != 2 or can_bus.shape[1] != 18:
        raise RuntimeError("can_bus must be a (bs, 18) float64 tensor")
    if out_dtype not in _DT:
        raise RuntimeError("ego_motion: float32, bfloat16 or float16 only")
    if mode != EGO_DELTAS:
        if state is None:
            raise RuntimeError("ego_motion: a stream mode needs the state block")
        _need_cuda(state, "state")
        if state.dtype != torch.int64 or state.numel() != 5:
            raise RuntimeError("ego_motion: state must come from ops.ego_state()")
    bs, dev = can_bus.shape[0], can_bus.device
    shift = torch.empty((bs, 2), device=dev, dtype=torch.float32)
    rot = torch.empty((bs, 6), device=dev, dtype=torch.float32)
    mlp_in = torch.empty((bs, 18), device=dev, dtype=out_dtype)
    lib = _lib.load()
    with torch.cuda.device(dev):
        st = lib.bevf_ego_motion(can_bus.data_ptr(), _ptr(state) if mode != EGO_DELTAS else 0, int(mode),
                                 shift.data_ptr(), rot.data_ptr(), mlp_in.data_ptr(), _DT[out_dtype], bs,
                                 int(bev_h), int(bev_w), float(grid_length[0]), float(grid_length[1]),
                                 float(rotate_center[0]), float(rotate_center[1]), int(bool(use_shift)),
                                 _stream_ptr(can_bus))
    _lib.check(st, lib)
    return shift, rot, mlp_in


def rotate_bev(prev_bev, rot, bev_h, bev_w, out_dtype=None):
    """prev_bev (bs, Nq, C) or (Nq, bs, C) (any strides with contiguous channels; a second dimension of Nq means
    batch-first, as in get_bev_features) rotated through the grid rows ``rot`` (bs, 6) of ``ego_motion``:
    (Nq, bs, C) in ``out_dtype`` (default: prev_bev's), one gather pass (bevf_rotate_bev).  No gradient."""
    if not prev_bev.is_cuda:
        raise RuntimeError("prev_bev must be a CUDA tensor (bevformer_b200 has no CPU path)")
    out_dtype = out_dtype or prev_bev.dtype
    if prev_bev.dtype not in _DT or out_dtype not in _DT:
        raise RuntimeError("rotate_bev: float32, bfloat16 or float16 only")
    if prev_bev.requires_grad and torch.is_grad_enabled():
        raise RuntimeError("rotate_bev has no backward: pass prev_bev without gradient")
    nq = bev_h * bev_w
    if prev_bev.dim() != 3 or nq not in prev_bev.shape[:2]:
        raise RuntimeError("prev_bev must be (bs, bev_h*bev_w, C) or (bev_h*bev_w, bs, C)")
    if prev_bev.shape[1] == nq:
        prev_bev = prev_bev.permute(1, 0, 2)
    C = prev_bev.shape[2]
    if prev_bev.stride(2) != 1 or prev_bev.stride(0) % 8 or prev_bev.stride(1) % 8 or prev_bev.data_ptr() % 16:
        prev_bev = prev_bev.contiguous()
    bs = prev_bev.shape[1]
    _need_cuda(rot, "rot")
    if rot.dtype != torch.float32 or tuple(rot.shape) != (bs, 6):
        raise RuntimeError("rot must be the (bs, 6) float32 tensor of ego_motion")
    out = torch.empty((nq, bs, C), device=prev_bev.device, dtype=out_dtype)
    lib = _lib.load()
    with torch.cuda.device(prev_bev.device):
        st = lib.bevf_rotate_bev(prev_bev.data_ptr(), _DT[prev_bev.dtype], prev_bev.stride(0), prev_bev.stride(1),
                                 rot.data_ptr(), out.data_ptr(), _DT[out_dtype], bs, int(bev_h), int(bev_w), C,
                                 _stream_ptr(prev_bev))
    _lib.check(st, lib)
    return out


class FlattenFeats(Function):
    """Multi-level camera features [(bs, ncam, C, h, w)] -> (ncam, S, bs, C) with cams_embeds and
    level_embeds added (PerceptionTransformer.get_bev_features, transformer.py:161-181): one kernel
    per level instead of flatten / permute / add / add / cat / permute.  Call as
    ``FlattenFeats.apply(cams_embeds_or_None, level_embeds, *mlvl_feats)``."""

    @staticmethod
    def forward(ctx, cams_embeds, level_embeds, *feats):
        f0 = feats[0]
        _need_cuda(f0, "mlvl_feats[0]")
        if f0.dtype not in _DT:
            raise RuntimeError("flatten_feats: float32, bfloat16 or float16 only")
        bs, ncam, C = f0.shape[:3]
        hws = [int(f.shape[3] * f.shape[4]) for f in feats]
        S = sum(hws)
        out = torch.empty((ncam, S, bs, C), device=f0.device, dtype=f0.dtype)
        ce = None if cams_embeds is None else cams_embeds.detach().float().contiguous()
        le = level_embeds.detach().float().contiguous()
        lib = _lib.load()
        start = 0
        with torch.cuda.device(f0.device):
            for lvl, f in enumerate(feats):
                if f.dtype != f0.dtype or tuple(f.shape[:3]) != (bs, ncam, C):
                    raise RuntimeError("flatten_feats: levels disagree in dtype / (bs, ncam, C)")
                fc = f.contiguous()
                st = lib.bevf_flatten_feats(fc.data_ptr(), _ptr(ce), le[lvl].data_ptr(), out.data_ptr(),
                                            bs, ncam, C, hws[lvl], S, start, _DT[f0.dtype],
                                            _stream_ptr(f0))
                _lib.check(st, lib)
                start += hws[lvl]
        ctx.shapes = [tuple(f.shape) for f in feats]
        ctx.meta = (None if cams_embeds is None else cams_embeds.dtype, level_embeds.dtype)
        ctx.level_shape = tuple(level_embeds.shape)       # may hold more rows than there are levels
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        # data movement only (the transposes back to NCHW and three small reductions): torch ops
        cdt, ldt = ctx.meta
        need = ctx.needs_input_grad
        d_cams = dy.sum((1, 2), dtype=torch.float32).to(cdt) if (cdt is not None and need[0]) else None
        # the reference slices level_embeds[lvl:lvl+1] (transformer.py:172): rows beyond the pyramid's
        # levels (tiny / small: 1 level, num_feature_levels = 4) simply get a zero gradient
        d_level = torch.zeros(ctx.level_shape, device=dy.device, dtype=torch.float32) if need[1] else None
        d_feats, start = [], 0
        for i, (bs, ncam, C, h, w) in enumerate(ctx.shapes):
            sl = dy[:, start:start + h * w]                          # (ncam, hw, bs, C)
            if need[1]:
                d_level[i] = sl.sum((0, 1, 2), dtype=torch.float32)
            d_feats.append(sl.permute(2, 0, 3, 1).reshape(bs, ncam, C, h, w) if need[2 + i] else None)
            start += h * w
        if need[1]:
            d_level = d_level.to(ldt)
        return (d_cams, d_level, *d_feats)


# ---------------------------------------------------------------------------------------------------
# Grouped multi-head attention (csrc/attention.cu): the self-attention of Group DETR's decoder.
# ---------------------------------------------------------------------------------------------------

def _seq_operand(t: torch.Tensor):
    """(tensor, row stride) of a sequence-first (N, bs, W) operand read in place: unit channel stride, rows at one
    uniform stride (a column slice of a projection output qualifies).  Anything else is copied contiguous."""
    if (t.dim() == 3 and t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
            and t.stride(1) % 8 == 0 and t.data_ptr() % 16 == 0):
        return t, int(t.stride(1))
    t = t.contiguous()
    return t, int(t.shape[2])


def attention_dropout_mask(nq, nk, bs, heads, groups, drop_p, seed, seed_base, device):
    """Keep-mask (bs, groups, heads, nq / groups, nk / groups), uint8, that the attention kernels apply for this
    (seed, seed_base): a test and debugging aid (the kernels regenerate it and never store it)."""
    mask = torch.empty(bs, groups, heads, nq // groups, nk // groups, device=device, dtype=torch.uint8)
    lib = _lib.load()
    with torch.cuda.device(mask.device):
        st = lib.bevf_attn_dropout_mask(mask.data_ptr(), nq, nk, bs, heads, groups, float(drop_p), seed,
                                        _ptr(seed_base), torch.cuda.current_stream(mask.device).cuda_stream)
    _lib.check(st, lib)
    return mask


class GroupAttention(Function):
    """Block-diagonal softmax attention over sequence-first projections, head_dim 32, bf16 / fp16.

    ``apply(q, k, v, heads, groups, scale, drop_p)``: q (Nq, bs, H*32), k / v (Nk, bs, H*32); query group g
    (tokens [g*Nq/G, (g+1)*Nq/G)) attends to key group g.  With ``k`` None, ``q`` is the stacked in-projection
    [Q | K] (Nq, bs, 2*H*32) of a self-attention and its gradient comes back as one (Nq, bs, 2*H*32) tensor, ready
    for a single dX GEMM against the stacked weight rows.  Returns (Nq, bs, H*32) in the operands' dtype.
    ``drop_p`` > 0 drops attention probabilities with masks regenerated in backward (``attention_dropout_mask``
    gives them).  The backward has no atomics: its result repeats bit for bit."""

    @staticmethod
    def forward(ctx, q, k, v, heads, groups, scale, drop_p=0.0):
        stacked = k is None
        C = heads * 32
        for t, name in ((q, "q"), (v, "v")) + (() if stacked else ((k, "k"),)):
            if not t.is_cuda:
                raise RuntimeError(f"{name} must be a CUDA tensor (bevformer_b200 has no CPU path)")
            if t.dtype not in TC_DTYPES or t.dtype != q.dtype:
                raise RuntimeError("group attention: q, k and v must be all bfloat16 or all float16")
        qs, ldq = _seq_operand(q)
        if stacked:
            if qs.shape[2] != 2 * C:
                raise RuntimeError("group attention: stacked [Q | K] must have 2 * heads * 32 channels")
            ks, ldk, k_off = qs, ldq, C
        else:
            ks, ldk = _seq_operand(k)
            k_off = 0
        vs, ldv = _seq_operand(v)
        nq, bs = qs.shape[0], qs.shape[1]
        nk = vs.shape[0]
        if vs.shape[2] != C or (not stacked and (ks.shape[2] != C or ks.shape[0] != nk)) or vs.shape[1] != bs:
            raise RuntimeError("group attention: q, k, v shapes do not match (N, bs, heads * 32)")
        out = torch.empty(nq, bs, C, device=q.device, dtype=q.dtype)
        lse = torch.empty(bs, groups, heads, nq // max(groups, 1), device=q.device, dtype=torch.float32)
        seed = _next_seed() if drop_p > 0.0 else 0
        # a copy: before the first advance_seed the step key is the live counter, which a later advance changes in
        # place; the backward must regenerate this forward's masks
        sbase = seed_state(q.device).clone() if drop_p > 0.0 else None
        esz = qs.element_size()
        lib = _lib.load()
        with torch.cuda.device(q.device):
            st = lib.bevf_attn_forward(qs.data_ptr(), ldq, ks.data_ptr() + k_off * esz, ldk, vs.data_ptr(), ldv,
                                       out.data_ptr(), C, lse.data_ptr(), nq, nk, bs, heads, 32, groups, float(scale),
                                       float(drop_p), seed, _ptr(sbase), _DT[q.dtype], _stream_ptr(q))
        _lib.check(st, lib)
        ctx.save_for_backward(qs, None if stacked else ks, vs, out, lse)
        ctx.meta = (stacked, ldq, ldk, k_off, ldv, heads, groups, float(scale), float(drop_p), seed)
        ctx.sbase = sbase
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        qs, ks, vs, out, lse = ctx.saved_tensors
        stacked, ldq, ldk, k_off, ldv, heads, groups, scale, drop_p, seed = ctx.meta
        if stacked:
            ks = qs
        C = heads * 32
        nq, bs, nk = qs.shape[0], qs.shape[1], vs.shape[0]
        dout = dout.to(out.dtype)
        dos, ldgo = _seq_operand(dout)
        esz = qs.element_size()
        if stacked:
            dqk = torch.empty(nq, bs, 2 * C, device=qs.device, dtype=qs.dtype)
            dq_ptr, lddq, dk_ptr, lddk = dqk.data_ptr(), 2 * C, dqk.data_ptr() + C * esz, 2 * C
        else:
            dq = torch.empty(nq, bs, C, device=qs.device, dtype=qs.dtype)
            dk = torch.empty(nk, bs, C, device=qs.device, dtype=qs.dtype)
            dq_ptr, lddq, dk_ptr, lddk = dq.data_ptr(), C, dk.data_ptr(), C
        dv = torch.empty(nk, bs, C, device=qs.device, dtype=qs.dtype)
        delta = torch.empty_like(lse)
        lib = _lib.load()
        with torch.cuda.device(qs.device):
            st = lib.bevf_attn_backward(qs.data_ptr(), ldq, ks.data_ptr() + k_off * esz, ldk, vs.data_ptr(), ldv,
                                        out.data_ptr(), C, dos.data_ptr(), ldgo, lse.data_ptr(), delta.data_ptr(),
                                        dq_ptr, lddq, dk_ptr, lddk, dv.data_ptr(), C, nq, nk, bs, heads, 32, groups,
                                        scale, drop_p, seed, _ptr(ctx.sbase), _DT[qs.dtype], _stream_ptr(qs))
        _lib.check(st, lib)
        if stacked:
            return dqk, None, dv, None, None, None, None
        return dq, dk, dv, None, None, None, None


# ---------------------------------------------------------------------------------------------------
# Detection head (csrc/det_head.cu): BEVFormerHead's branch MLPs for every decoder level in one launch, and
# NMSFreeCoder's decode without host synchronisation.
# ---------------------------------------------------------------------------------------------------
def det_branch_params(cls_branch, reg_branch):
    """The 16 parameter tensors of one level's (cls, reg) branch pair, in the order bevf_det_branches_forward reads
    them.  The branches must have BEVFormerHead's layout with num_reg_fcs = 2: cls = Linear-LayerNorm-ReLU x 2 +
    Linear, reg = Linear-ReLU x 2 + Linear."""
    import torch.nn as nn
    c, r = list(cls_branch), list(reg_branch)
    kinds_c = [nn.Linear, nn.LayerNorm, nn.ReLU] * 2 + [nn.Linear]
    kinds_r = [nn.Linear, nn.ReLU] * 2 + [nn.Linear]
    if len(c) != 7 or len(r) != 5 or not all(isinstance(m, k) for m, k in zip(c + r, kinds_c + kinds_r)):
        raise NotImplementedError("det_branches_forward: the fused branches need BEVFormerHead's layout with "
                                  "num_reg_fcs=2 (Linear-LayerNorm-ReLU x 2 + Linear / Linear-ReLU x 2 + Linear)")
    if any(m.bias is None for m in (c[0], c[3], c[6], r[0], r[2], r[4])) or not (c[1].elementwise_affine
                                                                               and c[4].elementwise_affine):
        raise NotImplementedError("det_branches_forward: Linear layers need a bias and LayerNorms an affine transform")
    return [c[0].weight, c[0].bias, c[1].weight, c[1].bias, c[3].weight, c[3].bias, c[4].weight, c[4].bias,
            c[6].weight, c[6].bias, r[0].weight, r[0].bias, r[2].weight, r[2].bias, r[4].weight, r[4].bias]


def det_branches_forward(states, init_reference, inter_references, level_params, pc_range, ln_eps=1e-5):
    """BEVFormerHead.forward after the transformer (bevformer_head.py:171-203) for every level in one launch.

    states            (L, nq, bs, 256) bf16 / fp16 decoder states, read through their strides (channels contiguous)
    init_reference    (bs, nq, 3), inter_references (L, bs, nq, 3): fp32 or the states' dtype
    level_params      L lists of ``det_branch_params``; all in the states' dtype or all fp32 (autocast: fp32 weights
                      and Linear biases are rounded to the states' dtype inside the kernel, as autocast's Linear
                      rounds them; LayerNorm parameters are read in fp32)
    pc_range          6 numbers
    Returns (all_cls_scores (L, bs, nq, ncls), all_bbox_preds (L, bs, nq, 10)) in the states' dtype.  No autograd."""
    if not states.is_cuda:
        raise RuntimeError("states must be a CUDA tensor (bevformer_b200 has no CPU path)")
    if states.dtype not in TC_DTYPES:
        raise RuntimeError(f"det_branches_forward: bf16 or fp16 states only (got {states.dtype})")
    if states.dim() != 4 or states.shape[3] != 256 or states.stride(3) != 1:
        raise RuntimeError(f"det_branches_forward: states must be (L, nq, bs, 256) with contiguous channels, got "
                           f"{tuple(states.shape)}")
    L, nq, bs, C = states.shape
    if any(s % 8 for s in states.stride()[:3]) or states.data_ptr() % 16:
        states = states.contiguous()
    if len(level_params) != L or not 1 <= L <= 8:
        raise RuntimeError(f"det_branches_forward: {len(level_params)} parameter sets for {L} levels (1 to 8)")
    pdt = level_params[0][0].dtype
    if pdt not in (states.dtype, torch.float32):
        raise RuntimeError(f"det_branches_forward: parameters in {pdt}; need {states.dtype} or float32")
    ncls = level_params[0][8].shape[0]
    shapes = [(C, C), (C,), (C,), (C,), (C, C), (C,), (C,), (C,), (ncls, C), (ncls,),
              (C, C), (C,), (C, C), (C,), (10, C), (10,)]
    if not 1 <= ncls <= 16:
        raise RuntimeError(f"det_branches_forward: {ncls} classes; the kernel takes 1 to 16")
    ptrs = []
    for ps in level_params:
        if len(ps) != 16:
            raise RuntimeError("det_branches_forward: 16 parameter tensors per level (ops.det_branch_params)")
        for t, shp in zip(ps, shapes):
            if tuple(t.shape) != shp:
                raise RuntimeError(f"det_branches_forward: parameter of shape {tuple(t.shape)}, expected {shp} "
                                   "(embed_dims 256, code_size 10)")
            if t.dtype != pdt or t.device != states.device or not t.is_contiguous():
                raise RuntimeError("det_branches_forward: parameters must be contiguous, on the states' device and "
                                   "all of one dtype")
            ptrs.append(t.data_ptr())
    refs = []
    for name, r, shp in (("init_reference", init_reference, (bs, nq, 3)),
                         ("inter_references", inter_references, (L, bs, nq, 3))):
        if tuple(r.shape) != shp:
            raise RuntimeError(f"det_branches_forward: {name} of shape {tuple(r.shape)}, expected {shp}")
        if r.dtype not in _DT:
            raise RuntimeError(f"det_branches_forward: {name} must be float32, bfloat16 or float16")
        if r.device != states.device:
            raise RuntimeError(f"det_branches_forward: {name} must be on the states' device ({states.device})")
        refs.append(r.to(init_reference.dtype).contiguous())
    if len(pc_range) != 6:
        raise RuntimeError("det_branches_forward: pc_range needs 6 numbers")
    cls = torch.empty((L, bs, nq, ncls), device=states.device, dtype=states.dtype)
    box = torch.empty((L, bs, nq, 10), device=states.device, dtype=states.dtype)
    import ctypes
    table = (ctypes.c_void_p * len(ptrs))(*ptrs)
    pc = (ctypes.c_double * 6)(*[float(v) for v in pc_range])
    lib = _lib.load()
    with torch.cuda.device(states.device):
        st = lib.bevf_det_branches_forward(states.data_ptr(), states.stride(0), states.stride(1), states.stride(2),
                                           _DT[states.dtype], refs[0].data_ptr(), refs[1].data_ptr(),
                                           _DT[refs[0].dtype], ctypes.cast(table, ctypes.c_void_p), _DT[pdt],
                                           cls.data_ptr(), box.data_ptr(), L, bs, nq, C, ncls, 10, float(ln_eps),
                                           ctypes.cast(pc, ctypes.c_void_p), _stream_ptr(states))
    _lib.check(st, lib)
    return cls, box


def nms_free_decode(cls_scores, bbox_preds, max_num, post_center_range, score_threshold=None, z_shift=False):
    """NMSFreeCoder.decode (nms_free_coder.py:40-121) for a batch in one launch, no host synchronisation.

    cls_scores (bs, nq, ncls) logits, bbox_preds (bs, nq, 10) normalised boxes: fp32 / bf16 / fp16, widened to fp32.
    Returns fixed-capacity tensors (bboxes (bs, max_num, 9) f32, scores (bs, max_num) f32, labels (bs, max_num) i64,
    num (bs,) i32): sample i's detections are the first num[i] rows, in the order (score descending, flat index
    ascending) -- torch.topk leaves the order of equal scores unspecified; this kernel takes the lower flat index
    first.  Rows past num are zero.  ``score_threshold`` follows the reference's loop, including its quirks (0.0
    applies no mask); ``z_shift`` applies BEVFormerHead.get_bboxes' z -= h / 2."""
    if post_center_range is None:
        raise NotImplementedError("Need to reorganize output as a batch, only support post_center_range is not None "
                                  "for now!")
    for name, t in (("cls_scores", cls_scores), ("bbox_preds", bbox_preds)):
        _need_cuda(t, name)
        if t.dtype not in _DT:
            raise RuntimeError(f"nms_free_decode: {name} must be float32, bfloat16 or float16")
    if cls_scores.dim() != 3 or bbox_preds.dim() != 3 or bbox_preds.shape[:2] != cls_scores.shape[:2]:
        raise RuntimeError(f"nms_free_decode: shapes {tuple(cls_scores.shape)} / {tuple(bbox_preds.shape)}; need "
                           "(bs, nq, ncls) / (bs, nq, 10)")
    bs, nq, ncls = cls_scores.shape
    if bbox_preds.shape[2] != 10:
        raise RuntimeError("nms_free_decode: code_size must be 10")
    max_num = int(max_num)
    if not 1 <= max_num <= nq * ncls:
        raise RuntimeError(f"nms_free_decode: max_num {max_num} must lie in [1, nq * ncls = {nq * ncls}]")
    lib = _lib.load()
    if lib.bevf_nms_free_decode_smem_bytes(nq, ncls, max_num) > 200 * 1024:
        raise RuntimeError(f"nms_free_decode: nq * ncls = {nq * ncls} is too large for the shared-memory top-k")
    import ctypes
    import numpy as np
    pcr = (ctypes.c_float * 6)(*np.asarray(post_center_range, dtype=np.float32).reshape(6).tolist())
    dev = cls_scores.device
    bboxes = torch.empty((bs, max_num, 9), device=dev, dtype=torch.float32)
    scores = torch.empty((bs, max_num), device=dev, dtype=torch.float32)
    labels = torch.empty((bs, max_num), device=dev, dtype=torch.int64)
    num = torch.empty((bs,), device=dev, dtype=torch.int32)
    has_thr = score_threshold is not None and bool(score_threshold)
    with torch.cuda.device(dev):
        st = lib.bevf_nms_free_decode(cls_scores.data_ptr(), _DT[cls_scores.dtype], bbox_preds.data_ptr(),
                                      _DT[bbox_preds.dtype], bs, nq, ncls, 10, max_num, ctypes.cast(pcr, ctypes.c_void_p),
                                      int(has_thr), float(score_threshold) if has_thr else 0.0, int(bool(z_shift)),
                                      bboxes.data_ptr(), scores.data_ptr(), labels.data_ptr(), num.data_ptr(),
                                      _stream_ptr(cls_scores))
    _lib.check(st, lib)
    return bboxes, scores, labels, num


# ---------------------------------------------------------------------------------------------------
# Detection loss (csrc/det_loss.cu): the matching cost of every (layer, sample) in one launch, and the focal /
# L1 / smooth-L1 losses of every (layer, group) slot with their gradient.  The assignment between them is the host's.
# ---------------------------------------------------------------------------------------------------
DET_REG = {"l1": _lib.ENUMS["BEVF_DET_REG_L1"], "smooth_l1": _lib.ENUMS["BEVF_DET_REG_SMOOTH_L1"]}


def _det_preds(cls_scores, bbox_preds, who):
    for name, t in (("cls_scores", cls_scores), ("bbox_preds", bbox_preds)):
        _need_cuda(t, name)
        if t.dtype not in _DT:
            raise RuntimeError(f"{who}: {name} must be float32, bfloat16 or float16")
    if (cls_scores.dim() != 4 or bbox_preds.dim() != 4 or bbox_preds.shape[:3] != cls_scores.shape[:3]
            or bbox_preds.shape[3] != 10):
        raise RuntimeError(f"{who}: shapes {tuple(cls_scores.shape)} / {tuple(bbox_preds.shape)}; need "
                           "(L, bs, nq, ncls) / (L, bs, nq, 10)")
    return cls_scores.shape


def _det_gt(gt, gt_labels, n_gt, bs, device, who):
    G = gt.shape[1]
    if (gt.dtype != torch.float32 or tuple(gt.shape) != (bs, G, 9) or gt_labels.dtype != torch.int64
            or tuple(gt_labels.shape) != (bs, G) or n_gt.dtype != torch.int32 or tuple(n_gt.shape) != (bs,)):
        raise RuntimeError(f"{who}: ground truth must be gt (bs, G, 9) float32, gt_labels (bs, G) int64 and "
                           f"n_gt (bs,) int32; got {tuple(gt.shape)} {gt.dtype}, {tuple(gt_labels.shape)} "
                           f"{gt_labels.dtype}, {tuple(n_gt.shape)} {n_gt.dtype}")
    for name, t in (("gt", gt), ("gt_labels", gt_labels), ("n_gt", n_gt)):
        _need_cuda(t, name)
        if t.device != device:
            raise RuntimeError(f"{who}: {name} must be on the predictions' device ({device})")
    return G


def det_match_cost(cls_scores, bbox_preds, gt, gt_labels, n_gt, reg_kind, cls_weight, reg_weight, alpha=0.25,
                   gamma=2.0, eps=1e-12):
    """HungarianAssigner3D's cost (hungarian_assigner_3d.py:106-116) for every decoder layer and sample in one launch.

    cls_scores (L, bs, nq, ncls) / bbox_preds (L, bs, nq, 10): fp32, bf16 or fp16.  gt (bs, G, 9) f32 gravity-centred
    boxes, gt_labels (bs, G) i64, n_gt (bs,) i32, all on the device; reg_kind 'l1' (BBox3DL1Cost) or 'smooth_l1'
    (SmoothL1Cost).  Returns the fp32 cost (L * bs, nq, G): row l * bs + b; columns past n_gt[b] are zero."""
    L, bs, nq, ncls = _det_preds(cls_scores, bbox_preds, "det_match_cost")
    G = _det_gt(gt, gt_labels, n_gt, bs, cls_scores.device, "det_match_cost")
    if reg_kind not in DET_REG:
        raise RuntimeError(f"det_match_cost: reg_kind must be one of {sorted(DET_REG)}")
    if G == 0:
        raise RuntimeError("det_match_cost: no ground-truth column (G = 0)")
    if not 1 <= ncls <= 64:
        raise RuntimeError(f"det_match_cost: {ncls} classes; the kernel takes 1 to 64")
    lib = _lib.load()
    if lib.bevf_det_match_cost_smem_bytes(ncls, G) > 200 * 1024:
        raise RuntimeError(f"det_match_cost: {G} ground-truth boxes per sample is more than the kernel's tile holds")
    cost = torch.empty((L * bs, nq, G), device=cls_scores.device, dtype=torch.float32)
    with torch.cuda.device(cls_scores.device):
        st = lib.bevf_det_match_cost(cls_scores.data_ptr(), _DT[cls_scores.dtype], bbox_preds.data_ptr(),
                                     _DT[bbox_preds.dtype], gt.data_ptr(), gt_labels.data_ptr(), n_gt.data_ptr(),
                                     cost.data_ptr(), L * bs, bs, nq, ncls, G, DET_REG[reg_kind], float(cls_weight),
                                     float(reg_weight), float(alpha), float(gamma), float(eps),
                                     _stream_ptr(cls_scores))
    _lib.check(st, lib)
    return cost


class DetLoss(Function):
    """BEVFormerHead.loss_single after the assignment, for every (layer, group) slot in one launch each way.

    apply(cls_scores, bbox_preds, assign, gt, gt_labels, n_gt, code_weights, avg, cfg) -> (L * groups, 2) fp32
    [loss_cls, loss_bbox] per slot s = l * groups + group, nan_to_num applied.
      cls_scores / bbox_preds  (L, bs, nq, ncls) / (L, bs, nq, 10), fp32 / bf16 / fp16; their gradients come back in
                               their own dtype
      assign                   (L * bs, nq) int32 ground-truth index or -1
      gt / gt_labels / n_gt    as det_match_cost; code_weights (10,) f32; avg (L * groups, 2) f32 avg factors
                               (cls, regression) before max(., 1), in device memory
      cfg                      dict(groups, reg_kind, cls_loss_weight, bbox_loss_weight, alpha, gamma, beta)
    Both directions are sums in a fixed order: the results repeat bit for bit."""

    @staticmethod
    def _args(cls_scores, bbox_preds, assign, gt, gt_labels, n_gt, code_weights, avg, cfg):
        L, bs, nq, ncls = _det_preds(cls_scores, bbox_preds, "DetLoss")
        G = _det_gt(gt, gt_labels, n_gt, bs, cls_scores.device, "DetLoss")
        groups = int(cfg["groups"])
        if groups < 1 or nq % groups:
            raise RuntimeError(f"DetLoss: {nq} queries do not split into {groups} groups")
        for name, t, dt, shp in (("assign", assign, torch.int32, (L * bs, nq)),
                                 ("code_weights", code_weights, torch.float32, (10,)),
                                 ("avg", avg, torch.float32, (L * groups, 2))):
            _need_cuda(t, name)
            if t.dtype != dt or tuple(t.shape) != shp or t.device != cls_scores.device:
                raise RuntimeError(f"DetLoss: {name} must be {dt} of shape {shp} on {cls_scores.device}, got "
                                   f"{t.dtype} {tuple(t.shape)} on {t.device}")
        if cfg["reg_kind"] not in DET_REG:
            raise RuntimeError(f"DetLoss: reg_kind must be one of {sorted(DET_REG)}")
        head = [cls_scores.data_ptr(), _DT[cls_scores.dtype], bbox_preds.data_ptr(), _DT[bbox_preds.dtype],
                assign.data_ptr(), gt.data_ptr(), gt_labels.data_ptr(), n_gt.data_ptr(), code_weights.data_ptr(),
                avg.data_ptr()]
        tail = [L, bs, nq, groups, ncls, G, DET_REG[cfg["reg_kind"]], float(cfg["cls_loss_weight"]),
                float(cfg["bbox_loss_weight"]), float(cfg["alpha"]), float(cfg["gamma"]), float(cfg.get("beta", 1.0)),
                _stream_ptr(cls_scores)]
        return head, tail, L * groups

    @staticmethod
    def forward(ctx, cls_scores, bbox_preds, assign, gt, gt_labels, n_gt, code_weights, avg, cfg):
        cls_scores, bbox_preds = cls_scores.contiguous(), bbox_preds.contiguous()
        head, tail, S = DetLoss._args(cls_scores, bbox_preds, assign, gt, gt_labels, n_gt, code_weights, avg, cfg)
        out = torch.empty((2, S, 2), device=cls_scores.device, dtype=torch.float32)
        lib = _lib.load()
        with torch.cuda.device(cls_scores.device):
            st = lib.bevf_det_loss_forward(*head, out[0].data_ptr(), out[1].data_ptr(), *tail)
        _lib.check(st, lib)
        ctx.save_for_backward(cls_scores, bbox_preds, assign, gt, gt_labels, n_gt, code_weights, avg, out[1])
        ctx.cfg = cfg
        return out[0]

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loss):
        cls_scores, bbox_preds, assign, gt, gt_labels, n_gt, code_weights, avg, loss_raw = ctx.saved_tensors
        head, tail, S = DetLoss._args(cls_scores, bbox_preds, assign, gt, gt_labels, n_gt, code_weights, avg,
                                      ctx.cfg)
        grad_loss = grad_loss.to(torch.float32).contiguous()
        grad_cls = torch.empty_like(cls_scores)
        grad_box = torch.empty_like(bbox_preds)
        lib = _lib.load()
        with torch.cuda.device(cls_scores.device):
            st = lib.bevf_det_loss_backward(*head, loss_raw.data_ptr(), grad_loss.data_ptr(), grad_cls.data_ptr(),
                                            grad_box.data_ptr(), *tail)
        _lib.check(st, lib)
        return grad_cls, grad_box, None, None, None, None, None, None, None


# ---- modulated deformable convolution (DCNv2) ---------------------------------------------------------------------
def _dcn_geom(input, offset, mask, weight, stride, padding, dilation, groups, deform_groups):
    """(N, H, W, C, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, dg) of a modulated_deform_conv2d call, after mmcv's
    argument checks and the kernels' alignment constraints."""
    def pair(v):
        return (int(v), int(v)) if isinstance(v, int) else tuple(int(x) for x in v)
    if groups != 1:
        raise NotImplementedError("modulated_deform_conv2d: groups != 1 is not implemented")
    if input.dim() != 4 or weight.dim() != 4 or offset.dim() != 4 or mask.dim() != 4:
        raise RuntimeError("modulated_deform_conv2d: input, offset, mask and weight must be 4-D")
    if input.dtype not in _DT:
        raise RuntimeError("modulated_deform_conv2d: input must be float32, bfloat16 or float16")
    N, C, H, W = input.shape
    Cout, Cw, kh, kw = weight.shape
    (sh, sw), (ph, pw), (dh, dw) = pair(stride), pair(padding), pair(dilation)
    dg, kk = int(deform_groups), kh * kw
    if Cw != C:
        raise RuntimeError(f"modulated_deform_conv2d: weight has {Cw} input channels, input has {C}")
    if min(sh, sw, dh, dw, dg) <= 0 or min(ph, pw) < 0:
        raise RuntimeError("modulated_deform_conv2d: stride, dilation and deform_groups must be positive, padding >= 0")
    if C % dg:
        raise RuntimeError(f"modulated_deform_conv2d: in_channels {C} is not divisible by deform_groups {dg}")
    Ho = (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1
    Wo = (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1
    Ho, Wo = max(Ho, 0), max(Wo, 0)
    if offset.shape[1] != 2 * dg * kk or mask.shape[1] != dg * kk:
        raise RuntimeError(f"modulated_deform_conv2d: offset must have {2 * dg * kk} channels and mask {dg * kk} "
                           f"(deform_groups * 2 * kh * kw, deform_groups * kh * kw), got {offset.shape[1]} and "
                           f"{mask.shape[1]}")
    if (offset.shape[0], mask.shape[0]) != (N, N) or tuple(offset.shape[2:]) != (Ho, Wo) or \
            tuple(mask.shape[2:]) != (Ho, Wo):
        raise RuntimeError(f"modulated_deform_conv2d: offset and mask must be ({N}, *, {Ho}, {Wo}) for this "
                           f"convolution, got {tuple(offset.shape)} and {tuple(mask.shape)}")
    vec = 16 // input.element_size()
    if (C // dg) % vec:
        raise RuntimeError(f"modulated_deform_conv2d: in_channels / deform_groups = {C // dg} must be a multiple of "
                           f"{vec} in {input.dtype} (16-byte vector loads)")
    if input.dtype in TC_DTYPES and ((kk * C) % 64 or Cout % 64):
        raise RuntimeError(f"modulated_deform_conv2d: 16-bit storage needs kh * kw * in_channels ({kk * C}) and "
                           f"out_channels ({Cout}) to be multiples of 64 (the wgmma GEMM's K and N)")
    for t, n in ((input, "input"), (offset, "offset"), (mask, "mask"), (weight, "weight")):
        if not t.is_cuda:
            raise RuntimeError(f"modulated_deform_conv2d: {n} must be a CUDA tensor (bevformer_b200 has no CPU path)")
    return N, H, W, C, Ho, Wo, kh, kw, sh, sw, ph, pw, dh, dw, dg


def _channels_last(x: torch.Tensor) -> torch.Tensor:
    """(N, C, H, W) -> contiguous (N, H, W, C): a view of a channels_last tensor, one transpose otherwise."""
    return x.permute(0, 2, 3, 1).contiguous()


def dcn_sampling_forward(x_nhwc, offset, mask, geom):
    """Deformable im2col (bevf_dcn_sampling_forward): x (N, H, W, C), offset / mask in mmcv's layout, all of x's dtype
    -> cols (N*Ho*Wo, kh*kw*C), column tap*C + c."""
    N, H, W, C, Ho, Wo, kh, kw = geom[:8]
    cols = torch.empty((N * Ho * Wo, kh * kw * C), device=x_nhwc.device, dtype=x_nhwc.dtype)
    if cols.numel() == 0:
        return cols
    lib = _lib.load()
    with torch.cuda.device(x_nhwc.device):
        st = lib.bevf_dcn_sampling_forward(x_nhwc.data_ptr(), offset.data_ptr(), mask.data_ptr(), _DT[x_nhwc.dtype],
                                           cols.data_ptr(), *geom, _stream_ptr(x_nhwc))
    _lib.check(st, lib)
    return cols


def dcn_sampling_backward(x_nhwc, offset, mask, dcols, geom):
    """Backward of the deformable im2col: (grad_input (N, H, W, C), grad_offset, grad_mask), all in x's dtype.
    grad_input is summed with fp32 vector reductions, or -- under torch.use_deterministic_algorithms(True) -- in 64-bit
    fixed point (bevf_dcn_sampling_backward_fx), which repeats bit for bit."""
    N, H, W, C, Ho, Wo, kh, kw = geom[:8]
    dev, dt = x_nhwc.device, x_nhwc.dtype
    goff = torch.empty(offset.shape, device=dev, dtype=dt)
    gmask = torch.empty(mask.shape, device=dev, dtype=dt)
    if N * Ho * Wo == 0:
        return torch.zeros(x_nhwc.shape, device=dev, dtype=dt), goff, gmask
    lib = _lib.load()
    common = (x_nhwc.data_ptr(), offset.data_ptr(), mask.data_ptr(), dcols.data_ptr(), _DT[dt])
    with torch.cuda.device(dev):
        if deterministic():
            k = int(lib.bevf_msda_fx_frac_bits(Ho * Wo, 1, kh * kw))
            fx = torch.zeros(x_nhwc.shape, device=dev, dtype=torch.int64)
            bounds = torch.empty(2, device=dev, dtype=torch.int32)
            st = lib.bevf_dcn_sampling_backward_fx(*common, fx.data_ptr(), bounds.data_ptr(), k, goff.data_ptr(),
                                                   gmask.data_ptr(), *geom, _stream_ptr(x_nhwc))
            _lib.check(st, lib)
            gin = FixedPointGradValue(fx, bounds, k, dt).materialize()
        else:
            acc = torch.zeros(x_nhwc.shape, device=dev, dtype=torch.float32)
            st = lib.bevf_dcn_sampling_backward(*common, acc.data_ptr(), goff.data_ptr(), gmask.data_ptr(), *geom,
                                                _stream_ptr(x_nhwc))
            _lib.check(st, lib)
            gin = acc if dt == torch.float32 else acc.to(dt)
    return gin, goff, gmask


class ModulatedDeformConv2dFunction(Function):
    """mmcv's ModulatedDeformConv2dFunction (mmcv/ops/modulated_deform_conv.py) on the library: the sampling kernels of
    csrc/dcn.cu around the library's GEMMs -- y = cols . Wp^T (+ bias), Wp = weight.permute(0, 2, 3, 1) as
    (Cout, kh*kw*Cin), on the wgmma kernel for bf16 / fp16 storage and on torch for fp32 (the parity configuration).
    The backward recomputes the columns instead of saving them.  Input, offset, mask and weight share one dtype
    (``modulated_deform_conv2d`` casts); the output is a channels_last (N, Cout, Ho, Wo) view of the GEMM's rows."""

    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                deform_groups=1):
        geom = _dcn_geom(input, offset, mask, weight, stride, padding, dilation, groups, deform_groups)
        N, H, W, C, Ho, Wo, kh, kw = geom[:8]
        Cout = weight.shape[0]
        x = _channels_last(input)
        offset, mask = offset.contiguous(), mask.contiguous()
        wp = weight.permute(0, 2, 3, 1).reshape(Cout, kh * kw * C).contiguous()
        ctx.geom, ctx.has_bias = geom, bias is not None
        ctx.dtypes = (weight.dtype, None if bias is None else bias.dtype)
        ctx.save_for_backward(x, offset, mask, wp)
        if N * Ho * Wo == 0:
            return torch.empty((N, Cout, Ho, Wo), device=input.device, dtype=input.dtype)
        cols = dcn_sampling_forward(x, offset, mask, geom)
        if input.dtype in TC_DTYPES:
            y = linear_tc(cols, wp, bias)
        else:
            y = cols @ wp.t()
            if bias is not None:
                y += bias
        return y.view(N, Ho, Wo, Cout).permute(0, 3, 1, 2)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        x, offset, mask, wp = ctx.saved_tensors
        geom = ctx.geom
        N, H, W, C, Ho, Wo, kh, kw = geom[:8]
        Cout = wp.shape[0]
        dt = x.dtype
        if N * Ho * Wo == 0:
            return (torch.zeros((N, C, H, W), device=x.device, dtype=dt), torch.zeros_like(offset),
                    torch.zeros_like(mask), torch.zeros((Cout, C, kh, kw), device=x.device, dtype=ctx.dtypes[0]),
                    None if not ctx.has_bias else torch.zeros(Cout, device=x.device, dtype=ctx.dtypes[1]),
                    None, None, None, None, None)
        dy = grad_output.permute(0, 2, 3, 1).reshape(N * Ho * Wo, Cout).to(dt).contiguous()
        cols = dcn_sampling_forward(x, offset, mask, geom)
        if dt in TC_DTYPES:
            dcols = linear_dgrad_tc(dy, wp)
            if ctx.has_bias:
                dwp, db = linear_wgrad_tc(dy, cols, with_bias=True)
            else:
                dwp, db = linear_wgrad_tc(dy, cols), None
        else:
            dcols = dy @ wp
            dwp = dy.t() @ cols
            db = colsum(dy) if ctx.has_bias else None
        gin, goff, gmask = dcn_sampling_backward(x, offset, mask, dcols, geom)
        grad_input = gin.permute(0, 3, 1, 2)
        grad_weight = dwp.view(Cout, kh, kw, C).permute(0, 3, 1, 2).to(ctx.dtypes[0]).contiguous()
        grad_bias = None if db is None else db.to(ctx.dtypes[1])
        return grad_input, goff, gmask, grad_weight, grad_bias, None, None, None, None, None


def modulated_deform_conv2d(input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                            deform_groups=1):
    """mmcv.ops.modulated_deform_conv2d with mmcv's argument order: out[n, co, ho, wo] = bias[co] +
    sum_{c, i, j} weight[co, c, i, j] * mask[n, g*kk + i*kw + j, ho, wo] * bilinear(input[n, c], h, w)
    (SURVEY.md Appendix B).  Computes in input's dtype: offset, mask and weight are cast to it (autograd returns
    their gradients in their own dtypes); the bias may be any float dtype.  Returns (N, Cout, Ho, Wo) in
    channels_last memory format."""
    if input.is_floating_point() and input.dtype in _DT:
        offset, mask, weight = (t.to(input.dtype) for t in (offset, mask, weight))
    return ModulatedDeformConv2dFunction.apply(input, offset, mask, weight, bias, stride, padding, dilation, groups,
                                               deform_groups)


# ---- GridMask -----------------------------------------------------------------------------------------------------
def grid_mask_apply(x, d, l, st_h, st_w, use_h, use_w, mode):
    """x (planes, H, W) times GridMask's mask for the drawn integers (bevf_grid_mask): a new contiguous tensor in x's
    dtype, bit for bit torch's ``x * mask.to(x.dtype)``.  No autograd."""
    _need_cuda(x, "grid_mask input")
    if x.dtype not in _DT:
        raise RuntimeError(f"grid_mask: dtype {x.dtype} not supported (float32, bfloat16 or float16)")
    if x.dim() != 3:
        raise RuntimeError(f"grid_mask: expected (planes, H, W), got {tuple(x.shape)}")
    planes, H, W = x.shape
    out = torch.empty_like(x)
    lib = _lib.load()
    with torch.cuda.device(x.device):
        st = lib.bevf_grid_mask(x.data_ptr(), out.data_ptr(), _DT[x.dtype], planes, H, W, int(d), int(l), int(st_h),
                                int(st_w), int(bool(use_h)), int(bool(use_w)), int(mode), _stream_ptr(x))
    _lib.check(st, lib)
    return out


class GridMaskFunction(Function):
    """out = x * m for GridMask's mask m (grid_mask.py:90-122 with rotate = 1, offset = False); the backward is the
    same kernel on grad_out.  Saves only the drawn integers."""

    @staticmethod
    def forward(ctx, x, d, l, st_h, st_w, use_h, use_w, mode):
        ctx.args = (d, l, st_h, st_w, use_h, use_w, mode)
        return grid_mask_apply(x.contiguous(), *ctx.args)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        return (grid_mask_apply(grad_out.contiguous(), *ctx.args),) + (None,) * 7


def grid_mask(x, d, l, st_h, st_w, use_h=True, use_w=True, mode=0):
    """GridMask's multiply for x (planes, H, W) in float32, bfloat16 or float16 on a CUDA device: row / column stripes
    of period d and width l starting at st_h / st_w in the (1.5 H, 1.5 W) frame whose centre crop is the image, zeroed
    (mode 0) or kept (mode 1).  Differentiable in x."""
    return GridMaskFunction.apply(x, d, l, st_h, st_w, use_h, use_w, mode)
