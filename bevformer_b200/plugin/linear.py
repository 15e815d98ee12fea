"""The dense projections of the encoder layer (value_proj / output_proj / the stacked
sampling_offsets|attention_weights head / FFN) behind one function.

bf16 / fp16 CUDA inputs run on the hand-written wgmma kernel of ``csrc/gemm.cu`` (bias, ReLU and the fp32
result of the offsets|logits head fused into its epilogue); its backward uses the same kernel for
dX = dY . W and the split-M wgmma kernel for dW = dY^T . X (``BEVF_WGRAD=cublas`` switches that one
back to the library); bias gradients come from the column-sum kernel.
fp32 inputs (the fp32 parity configuration) use the library GEMM.  ``BEVF_GEMM=cublas`` forces the
library path everywhere (A/B measurement).
"""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F
from torch.autograd.function import Function, once_differentiable

from .. import ops
from ..arena import arena_of


def _use_tc(x: torch.Tensor, weight: torch.Tensor) -> bool:
    return (x.is_cuda and x.dtype in ops.TC_DTYPES and weight.shape[1] % 64 == 0
            and weight.shape[0] % 16 == 0 and os.environ.get("BEVF_GEMM", "tc") != "cublas")


def stacked_head(weights, biases, x):
    """(W, b) of several Linear layers applied as one projection (sampling_offsets | attention_weights).
    On the wgmma path with a gradient arena the stack is a view of the arena's parameter buffer."""
    from ..arena import stacked
    n, k = sum(w.shape[0] for w in weights), weights[0].shape[1]
    direct = (x.is_cuda and x.dtype in ops.TC_DTYPES and k % 64 == 0 and n % 16 == 0
              and os.environ.get("BEVF_GEMM", "tc") != "cublas")
    return stacked(weights, direct), stacked(biases, direct)


def _arena_ctx(weight, bias):
    """(arena, accumulators, params) when weight (and bias) accumulate in a gradient arena, else None."""
    ar, accs = arena_of(weight, bias) if bias is not None else arena_of(weight)
    return None if ar is None else (ar, accs, (weight, bias))


class _LinearTC(Function):
    @staticmethod
    def forward(ctx, x, weight, bias, relu, fp32_out):
        w = weight.to(x.dtype)           # weights run in the activation dtype (a cast per call for fp32 masters)
        xc = x.contiguous()
        y = ops.linear_tc(xc, w, bias, None, relu, torch.float32 if fp32_out else x.dtype)
        ctx.save_for_backward(xc, w, y if relu else None)
        ctx.has_bias = bias is not None
        ctx.dtypes = (weight.dtype, None if bias is None else bias.dtype)
        ctx.arena = _arena_ctx(weight, bias)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        k, n = w.shape[1], w.shape[0]
        dy2 = dy.reshape(-1, n)
        if y is not None:                                  # ReLU: gradient only where the output is > 0
            dy2 = dy2 * (y.reshape(-1, n) > 0)
        dy2 = dy2.to(w.dtype).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = ops.linear_dgrad_tc(dy2, w).view(x.shape)
        if ctx.needs_input_grad[1]:
            dw, db = _wgrad(dy2, x.reshape(-1, k), n, k, ctx.dtypes[0],
                            ctx.dtypes[1] if ctx.has_bias else None, ctx.arena)
        elif ctx.has_bias and ctx.needs_input_grad[2]:
            db = ops.colsum(dy2).to(ctx.dtypes[1])
        return dx, dw, db, None, None


def _wgrad(dy2, x2, n, k, wdtype, bdtype=None, arena=None):
    """(dW, db) of a projection; db comes out of the same kernel pass as dW when requested.
    ``arena`` = (GradArena, [dW accumulator, db accumulator | None], params): accumulate into the flat
    gradient arena instead and return (None, None) -- the arena hands the gradients over at the end of the
    backward pass."""
    if arena is not None and n % 8 == 0:
        ar, accs, params = arena
        ar.touch(*[p for p in params if p is not None])
        dw_acc, db_acc = accs[0].view(n, k), (accs[1] if len(accs) > 1 else None)
        ar.run_off_critical_path(lambda: ops.linear_wgrad_into(dy2, x2, dw_acc, db_acc), dy2, x2)
        return None, None
    mode = os.environ.get("BEVF_WGRAD", "tc")     # "tc2": two-pass variant (opt-in)
    if mode == "tc2" and n % 8 == 0 and wdtype in (torch.bfloat16, torch.float16, torch.float32) and bdtype in (None, wdtype):
        return ops.linear_wgrad_out(dy2, x2, wdtype, bdtype is not None)
    if mode != "cublas" and n % 8 == 0:
        if bdtype is None:
            return ops.linear_wgrad_tc(dy2, x2, out_dtype=wdtype), None
        if bdtype == wdtype:                               # one conversion pass for [dW | db]
            return ops.linear_wgrad_tc(dy2, x2, with_bias=True, out_dtype=wdtype)
        dw, db = ops.linear_wgrad_tc(dy2, x2, with_bias=True)
        return dw.to(wdtype), db.to(bdtype)
    dw = torch.mm(dy2.t(), x2).to(wdtype)
    return dw, (None if bdtype is None else ops.colsum(dy2).to(bdtype))


class _LinearReluDropoutTC(Function):
    """h = dropout_p(relu(x W^T + b)): ReLU in the GEMM epilogue, dropout in place with Philox bits;
    the backward needs only h (h != 0 <=> pre-activation > 0 and kept)."""

    @staticmethod
    def forward(ctx, x, weight, bias, p):
        w = weight.to(x.dtype)
        xc = x.contiguous()
        h = ops.linear_tc(xc, w, bias, None, True, x.dtype)
        ops.dropout_inplace_(h, p)
        ctx.save_for_backward(xc, w, h)
        ctx.meta = (bias is not None, weight.dtype, None if bias is None else bias.dtype, float(p))
        ctx.arena = _arena_ctx(weight, bias)
        return h

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, w, h = ctx.saved_tensors
        has_bias, wdt, bdt, p = ctx.meta
        k, n = w.shape[1], w.shape[0]
        dz = ops.relu_dropout_backward(dy.reshape(-1, n), h.reshape(-1, n), p)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = ops.linear_dgrad_tc(dz, w).view(x.shape)
        if ctx.needs_input_grad[1]:
            dw, db = _wgrad(dz, x.reshape(-1, k), n, k, wdt, bdt if has_bias else None, ctx.arena)
        elif has_bias and ctx.needs_input_grad[2]:
            db = ops.colsum(dz).to(bdt)
        return dx, dw, db, None


class _SharedInputProjections(Function):
    """V_l = x W_l^T + b_l for several layers that read the SAME input x (every encoder layer projects the
    same camera features with its own SCA value_proj, and the same BEV queue with its own TSA value_proj:
    spatial_cross_attention.py:334, temporal_self_attention.py:198; encoder.py:214-232 never updates
    either between layers).  One autograd node instead of one per layer: its backward sums the per-layer
    input gradients in ONE pass (bevf_sum_tensors: n reads + 1 write) instead of autograd's n-1 pairwise
    add kernels (3 tensor passes each).  (Chaining them through the GEMM epilogue -- bevf_linear_dgrad_acc
    -- adds per-row addend loads to the epilogue of every layer's GEMM.)"""

    @staticmethod
    def forward(ctx, state, x, *wb):
        xc = x.contiguous()
        ws, outs, meta = [], [], []
        # layer l needs its projection only when layer l runs: with a second stream they are all issued there
        # now and each consumer waits for its own (state["ready"][l]) -- the projections of the later layers
        # run under the earlier layers' forward.  Opt-in (BEVF_AUX_PROJ=1)
        aux = ops.aux_stream(xc.device) if os.environ.get("BEVF_AUX_PROJ", "0") == "1" else None
        main = torch.cuda.current_stream(xc.device) if aux is not None else None
        ready = []
        if aux is not None:
            ev = torch.cuda.Event()
            ev.record(main)
            aux.wait_event(ev)
        for i in range(0, len(wb), 2):
            w = wb[i].to(xc.dtype)
            ws.append(w)
            if aux is None:
                outs.append(ops.linear_tc(xc, w, wb[i + 1], None, False, xc.dtype))
            else:
                with torch.cuda.stream(aux):
                    o = ops.linear_tc(xc, w, wb[i + 1], None, False, xc.dtype)
                    e = torch.cuda.Event()
                    e.record(aux)
                o.record_stream(main)
                outs.append(o)
                ready.append(e)
            meta.append((wb[i].dtype, None if wb[i + 1] is None else wb[i + 1].dtype))
        if aux is not None:
            xc.record_stream(aux)
        state["ready"] = ready
        ctx.save_for_backward(xc, *ws)
        # an output whose gradient was handed over through the early path arrives as None: keep it None
        # (the default would materialise a zero tensor the size of the value maps for each of them)
        ctx.set_materialize_grads(False)
        ctx.meta = meta
        ctx.arenas = [_arena_ctx(wb[i], wb[i + 1]) for i in range(0, len(wb), 2)]
        ctx.state = state
        # what the early (gradient-hook) path needs, kept outside autograd's saved tensors
        state.update(x2=xc.reshape(-1, xc.shape[-1]), ws=ws, meta=meta, arenas=ctx.arenas,
                     early=[None] * len(ws), need_dx=x.requires_grad)
        return tuple(outs)

    @staticmethod
    def early(state, l, dy):
        """Gradient hook of output l: with an overlap-enabled arena, this layer's dX and dW / db are issued
        on the side stream the moment its output gradient exists (right after that layer's sampler backward)
        instead of when the whole node runs at the end of the pass -- they then execute under the following
        layers' backward.  Returns nothing: the node's backward picks the results up."""
        ar = state["arenas"][l]
        if ar is None or ar[0].side_stream is None or state["early"][l] is not None:
            return False
        arena = ar[0]
        w = state["ws"][l]
        n, k = w.shape
        wdt, bdt = state["meta"][l]
        box = {}

        def work():
            # (the fp32 -> bf16 / fp16 conversion of a sampler's grad_value happens here too, off the critical path)
            dyt = dy.materialize() if isinstance(dy, ops.LazyGradValue) else dy    # fp16 accumulators -> bf16 here
            dy2 = dyt.reshape(-1, n).to(w.dtype).contiguous()
            if state["need_dx"]:
                box["dx"] = ops.linear_dgrad_tc(dy2, w)
            dw_acc, db_acc = ar[1][0].view(n, k), (ar[1][1] if len(ar[1]) > 1 else None)
            ops.linear_wgrad_into(dy2, state["x2"], dw_acc, db_acc)

        arena.touch(*[p for p in ar[2] if p is not None])
        arena.run_off_critical_path(work, *(dy.tensors if isinstance(dy, ops.LazyGradValue) else (dy,)), state["x2"], w)
        state["early"][l] = box
        return True

    @staticmethod
    @once_differentiable
    def backward(ctx, *dys):
        xc, *ws = ctx.saved_tensors
        state = ctx.state
        k = xc.shape[-1]
        x2 = xc.reshape(-1, k)
        dxs = []
        grads = []
        joined = False
        for l, (w, dy, (wdt, bdt)) in enumerate(zip(ws, dys, ctx.meta)):
            n = w.shape[0]
            box = state["early"][l]
            if box is None and dy is None:
                grads += [None, None]
                continue
            if box is not None:                                  # done ahead of time on the side stream
                if "dx" in box:
                    if not joined:
                        side = ctx.arenas[l][0].side_stream
                        torch.cuda.current_stream(xc.device).wait_stream(side)
                        joined = True
                    dxs.append(box["dx"])
                grads += [None, None]
                continue
            dy2 = dy.reshape(-1, n).to(w.dtype).contiguous()
            if ctx.needs_input_grad[1]:
                dxs.append(ops.linear_dgrad_tc(dy2, w))
            dw = db = None
            if ctx.needs_input_grad[2 + 2 * l]:
                dw, db = _wgrad(dy2, x2, n, k, wdt, bdt, ctx.arenas[l])
            elif bdt is not None and ctx.needs_input_grad[3 + 2 * l]:
                db = ops.colsum(dy2).to(bdt)
            grads += [dw, db]
        dx = ops.sum_tensors(dxs).view(xc.shape) if dxs else None
        for t in dxs:
            t.record_stream(torch.cuda.current_stream(xc.device))
        state["early"] = [None] * len(ws)
        return (None, dx, *grads)


def shared_input_projections(x, weights_and_biases):
    """[x W_l^T + b_l for l] for [(W_l, b_l), ...]; one autograd node on the wgmma path (see
    _SharedInputProjections), plain per-layer projections otherwise."""
    if all(_use_tc(x, w) for w, _ in weights_and_biases):
        flat = [t for wb in weights_and_biases for t in wb]
        state = {}
        outs = list(_SharedInputProjections.apply(state, x, *flat))
        if torch.is_grad_enabled() and any(o.requires_grad for o in outs):
            for l, o in enumerate(outs):
                o.register_hook(lambda g, l=l: (_SharedInputProjections.early(state, l, g), None)[1])
                # consumers that produce this output's gradient themselves (the sampler: fp32 grad_value) may
                # hand it over directly and skip autograd's dtype conversion on the critical path
                o._bevf_early = (lambda g, l=l: _SharedInputProjections.early(state, l, g))
        for l, o in enumerate(outs):
            if state.get("ready"):
                o._bevf_ready = state["ready"][l]
        return outs
    return [linear(x, w, b) for w, b in weights_and_biases]


def linear_relu_dropout(x, weight, bias, p: float):
    """FFN hidden layer: Linear -> ReLU -> Dropout(p) (p = 0 outside training)."""
    if _use_tc(x, weight):
        return _LinearReluDropoutTC.apply(x, weight, bias, p)
    y = F.relu(F.linear(x, weight.to(x.dtype), None if bias is None else bias.to(x.dtype)), inplace=True)
    return F.dropout(y, p, training=p > 0.0)


def linear(x: torch.Tensor, weight: torch.Tensor, bias, relu: bool = False) -> torch.Tensor:
    if _use_tc(x, weight):
        return _LinearTC.apply(x, weight, bias, relu, False)
    y = F.linear(x, weight.to(x.dtype), None if bias is None else bias.to(x.dtype))
    return F.relu(y, inplace=True) if relu else y


def linear_fp32_out(x: torch.Tensor, weight: torch.Tensor, bias) -> torch.Tensor:
    """Projection whose result is consumed in fp32 (sampling offsets / attention logits): taken
    straight from the fp32 accumulator on the wgmma path."""
    if _use_tc(x, weight):
        return _LinearTC.apply(x, weight, bias, False, True)
    y = F.linear(x, weight.to(x.dtype), None if bias is None else bias.to(x.dtype))
    return y.float()


# ---------------------------------------------------------------------------------------------------
# offsets|logits head + sampling-point preparation as ONE autograd node.  Between the two sits the
# (rows, M*L*P*3) fp32 tensor of raw offsets and logits; as separate nodes its gradient has to be
# fp32 (autograd casts a gradient to the dtype of the forward output) and is then cast to bf16 for the
# dX / dW GEMMs -- a read+write of 180 MB per layer at base.  Fused, the prep backward rounds to bf16
# itself.
# ---------------------------------------------------------------------------------------------------
class _HeadTC(Function):
    @staticmethod
    def forward(ctx, x, weight, bias, kind, prep_args):
        w = weight.to(x.dtype)
        xc = x.contiguous()
        raw = ops.linear_tc(xc, w, bias, None, False, torch.float32).reshape(-1, w.shape[0])
        if kind == "sca":
            ref_cam, pair_q, pair_cam, pair_of, ss, bs, nq, m, l, p = prep_args
            loc, attn = ops.sca_prep_forward(raw, ref_cam, pair_q, pair_cam, ss, bs, nq, m, l, p)
        elif kind == "query":
            ref, ss, bs, nq, m, l, p = prep_args
            loc, attn = ops.query_prep_forward(raw, ref, ss, bs, nq, m, l, p, 1)
        else:
            ref, ss, bs, nq, m, l, p, interleave = prep_args
            loc, attn = ops.tsa_prep_forward(raw, ref, ss, bs, nq, m, l, p, interleave)
        ctx.save_for_backward(xc, w, raw)
        ctx.kind, ctx.prep_args = kind, prep_args
        ctx.meta = (bias is not None, weight.dtype, None if bias is None else bias.dtype)
        ctx.arena = _arena_ctx(weight, bias)
        return loc, attn

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_loc, grad_attn):
        x, w, raw = ctx.saved_tensors
        grad_loc, grad_attn = grad_loc.contiguous(), grad_attn.contiguous()
        if ctx.kind == "sca":
            _ref_cam, pair_q, _pair_cam, pair_of, ss, bs, nq, m, l, p = ctx.prep_args
            d_raw = ops.sca_prep_backward(raw, grad_loc, grad_attn, pair_of, ss, bs, nq,
                                          pair_q.numel(), m, l, p, out_dtype=w.dtype)
        elif ctx.kind == "query":
            _ref, ss, bs, nq, m, l, p = ctx.prep_args
            d_raw = ops.query_prep_backward(raw, grad_loc, grad_attn, ss, bs, nq, m, l, p, 1, out_dtype=w.dtype)
        else:
            _ref, ss, bs, nq, m, l, p, interleave = ctx.prep_args
            d_raw = ops.tsa_prep_backward(raw, grad_loc, grad_attn, ss, bs, nq, m, l, p, interleave,
                                          out_dtype=w.dtype)
        return (*_head_grads(ctx, d_raw, x, w), None, None)


def _head_grads(ctx, d_raw, x, w):
    """(dX, dW, db) of the offsets|logits head from its 16-bit d_raw."""
    has_bias, wdt, bdt = ctx.meta
    k, n = w.shape[1], w.shape[0]
    dx = dw = db = None
    if ctx.needs_input_grad[0]:
        dx = ops.linear_dgrad_tc(d_raw, w).view(x.shape)
    if ctx.needs_input_grad[1]:
        dw, db = _wgrad(d_raw, x.reshape(-1, k), n, k, wdt, bdt if has_bias else None, ctx.arena)
    elif has_bias and ctx.needs_input_grad[2]:
        db = ops.colsum(d_raw).to(bdt)
    return dx, dw, db


class _ScaHeadSamplerTC(Function):
    """SpatialCrossAttention's offsets|logits head and its row-list sampler with the sampling-point prep inside the
    sampler kernels (ops.sca_rows_forward_fused): loc / attn are not stored, the backward recomputes them from
    ``raw`` and the forward's softmax statistics -- except the samples of the coarse levels that the dense tensor-core
    kernel takes in the backward (a quarter of them at base), which the forward writes as it computes them: that
    kernel handles one sample per thread and would otherwise wait on the pair-list and raw loads of every
    coefficient.  One autograd node, because the sampler backward produces d_raw in
    bf16: as a separate consumer of the fp32 ``raw`` it would be cast back to fp32 by autograd (and then to bf16
    again for the head's GEMMs).  ``fuse`` = (ref_cam, pair_q, pair_cam, pair_of, row_map, ss, lsi, bs, nq,
    level_hw_host, num_f16_levels, map_range, replicas) -- replicas: ops.gv_replicas_for."""

    @staticmethod
    def forward(ctx, x, weight, bias, value, fuse):
        ref_cam, pair_q, pair_cam, _pair_of, row_map, ss, lsi, bs, nq, hw_host, nfine, map_range, _reps = fuse
        w = weight.to(x.dtype)
        xc = x.contiguous()
        raw = ops.linear_tc(xc, w, bias, None, False, torch.float32).reshape(-1, w.shape[0])
        # the levels the dense kernel takes in the backward: as SamplerRows' backward hands them to it
        kd = None
        if any(ctx.needs_input_grad) and map_range is not None and ops._lib.load().bevf_msda_get_dense_backward():
            kd = ops.dense_levels_for(row_map.numel() / max(1, value.shape[0]), raw.shape[1] // (3 * 8 * len(hw_host)),
                                      hw_host)
            kd = None if kd is None else max(kd, nfine)
        out, stats, coarse = ops.sca_rows_forward_fused(value, ss, lsi, raw, ref_cam, pair_q, pair_cam, row_map, bs,
                                                        nq, coarse_from=kd)
        ctx.save_for_backward(xc, w, raw, stats, value)
        ctx.fuse, ctx.coarse = fuse, coarse
        ctx.meta = (bias is not None, weight.dtype, None if bias is None else bias.dtype)
        ctx.arena = _arena_ctx(weight, bias)
        ctx.value_early = getattr(value, "_bevf_early", None)     # see shared_input_projections
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        x, w, raw, stats, value = ctx.saved_tensors
        ref_cam, pair_q, pair_cam, pair_of, row_map, ss, lsi, bs, nq, hw_host, nfine, map_range, reps = ctx.fuse
        coarse = ctx.coarse
        dense = coarse is not None and ops._lib.load().bevf_msda_get_dense_backward()
        gv, d_raw = ops.sca_rows_backward_fused(value, ss, lsi, hw_host, nfine, raw, stats, ref_cam, pair_q, pair_cam,
                                                pair_of, row_map, grad_out, bs, nq,
                                                map_range=map_range if dense else None,
                                                first_dense_level=coarse[2] if dense else None, coarse=coarse,
                                                replicas=reps)
        ctx.coarse = None
        gvalue = None
        if ctx.needs_input_grad[3] and not (ctx.value_early is not None and ctx.value_early(gv)):
            gvalue = gv.materialize()
        return (*_head_grads(ctx, d_raw, x, w), gvalue, None)


def sca_sampling_head(x, weight, bias, ref_cam, pair_q, pair_cam, pair_of, ss, bs, nq, m, l, p):
    """(loc, attn) of SpatialCrossAttention for the in-view (camera, query) pairs: the stacked
    sampling_offsets|attention_weights projection followed by softmax / normalisation / anchor
    broadcast (spatial_cross_attention.py:338-372)."""
    if _use_tc(x, weight):
        return _HeadTC.apply(x, weight, bias, "sca", (ref_cam, pair_q, pair_cam, pair_of, ss, bs, nq, m, l, p))
    raw = linear_fp32_out(x, weight, bias).reshape(bs * nq, -1)
    return ops.ScaPrep.apply(raw, ref_cam, pair_q, pair_cam, pair_of, ss, bs, nq, m, l, p)


def sca_head_sampler(x, weight, bias, value, fuse):
    """Sampler output (bs*pairs, C) of SpatialCrossAttention straight from the query: the offsets|logits head and the
    row-list sampler with the sampling-point prep fused in (_ScaHeadSamplerTC; the caller checks that it applies)."""
    return _ScaHeadSamplerTC.apply(x, weight, bias, value, fuse)


def query_sampling_head(x, weight, bias, ref, ss, bs, nq, m, l, p):
    """(loc, attn) of the decoder's CustomMSDeformableAttention for 2-d reference points (decoder.py:300-330): the
    TSA prep with one frame.  16-bit x: one node with the head GEMM, d_raw in 16 bits; fp32: GEMM + QueryPrep."""
    if _use_tc(x, weight):
        return _HeadTC.apply(x, weight, bias, "query", (ref, ss, bs, nq, m, l, p))
    raw = linear_fp32_out(x, weight, bias).reshape(bs * nq, -1)
    return ops.QueryPrep.apply(raw, ref, ss, bs, nq, m, l, p, 1)


def tsa_sampling_head(x, weight, bias, ref, ss, bs, nq, m, l, p, interleave=False):
    """(loc, attn) of TemporalSelfAttention (temporal_self_attention.py:199-229)."""
    if _use_tc(x, weight):
        return _HeadTC.apply(x, weight, bias, "tsa", (ref, ss, bs, nq, m, l, p, bool(interleave)))
    raw = linear_fp32_out(x, weight, bias).reshape(bs * nq, -1)
    return ops.TsaPrep.apply(raw, ref, ss, bs, nq, m, l, p, interleave)
