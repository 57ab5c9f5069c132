"""torch.autograd.Function wrappers: the training-mode forward/backward of the hot path on the sm_90a kernels.

The reference gets its backward from autograd over F.conv2d / BatchNorm2d / ReLU / F.interpolate / torch.cat and the
`result + op(x) * w` python arithmetic (search/operations.py, search/model_search.py:60-78,318-333).  Here each fused unit
is one autograd node whose backward calls the kernels in csrc/train.cu, so `loss.backward()`, `torch.autograd.grad`,
`clip_grad_norm_` and the stock optimizers work unchanged on the fp32 master parameters.

Gradient precision: activation gradients are fp16 NHWC; to keep small mean-reduced-loss gradients out of the fp16
subnormal range they carry a static loss scale GRAD_SCALE, applied where fp32 NCHW logits gradients enter
(`UpsampleLogitsFn`, `ToNCHWFn`) and divided out of every fp32 parameter / scalar gradient by the kernels.
"""
from __future__ import annotations

import torch

from . import engine
from . import functional as F_

GRAD_SCALE = 1024.0
# Weight gradients are accumulated by the wgrad kernel straight into `param.grad` (created zero-filled on first use) instead
# of being returned to autograd as freshly allocated full-size tensors: the supernet's slimmable weights are max-width
# masters of which a forward touches one corner, and it runs 4 forwards per backward.  `loss.backward()` users (the
# reference drivers, architect.py's first-order step) see exactly the same `.grad`; code that needs
# `torch.autograd.grad(loss, weights)` can switch this off.
import os as _os
FUSED_WGRAD_ACCUMULATION = _os.environ.get("FSB_FUSED_WGRAD", "1") != "0"


def set_grad_scale(v: float):
    global GRAD_SCALE
    GRAD_SCALE = float(v)


# ----------------------------------------------------------------------------------------------
# EXPERIMENTAL (FSB_TAPE=1, default off): one torch.autograd node per network forward.
#
# The supernet step is bound by Python time per unit (DESIGN.md section 3), and a large share of that is
# torch.autograd.Function.apply itself (ctx construction, functorch bookkeeping, engine dispatch: ~30 us forward + ~30 us
# backward per node, ~5 400 nodes per step).  With the tape enabled a whole forward pass runs inside ONE autograd node:
# every unit below is executed through `call()`, which runs `Fn.forward` on a minimal context object and appends it to a
# list; the node's backward replays the list in reverse, accumulating activation gradients with our add kernel.  The
# scalar plumbing on the architecture parameters (softmax, gumbel sampling, weight * width-score products) stays ordinary
# torch autograd: it runs under enable_grad inside the node and is differentiated at the end of the replay.
# The Function classes are unchanged -- the tape only replaces who calls their forward / backward.
# ----------------------------------------------------------------------------------------------
TAPE_ENABLED = _os.environ.get("FSB_TAPE", "0") == "1"
_TAPE = None


class _NodeCtx:
    """what our Function.forward / backward use of autograd's ctx: save_for_backward, saved_tensors, needs_input_grad and
    free-form attributes"""
    saved_tensors = ()

    def save_for_backward(self, *tensors):
        self.saved_tensors = tensors


class Tape:
    def __init__(self, streams=False):
        self.nodes = []        # (Function class, ctx, args, output, stream) in execution order
        self.tracked = set()   # ids of tape-produced tensors that need a gradient
        self.keep = []         # every tape-produced tensor stays alive until backward, so ids are unique
        # streams=True (captured passes, graphed.py): every node remembers the CUDA stream it ran on; the backward replay runs
        # each node's backward on that stream and orders streams with events along the gradient data flow, so the independent
        # ops of a MixedOp / Cell overlap in both directions
        self.streams = streams

    def needs(self, t):
        return isinstance(t, torch.Tensor) and (t.requires_grad or id(t) in self.tracked)

    def record(self, fn, args):
        ctx = _NodeCtx()
        tracked, tensor = self.tracked, torch.Tensor
        ctx.needs_input_grad = tuple(isinstance(a, tensor) and (a.requires_grad or id(a) in tracked) for a in args)
        prev = torch.is_grad_enabled()
        torch._C._set_grad_enabled(False)          # like Function.forward
        try:
            out = fn.forward(ctx, *args)
        finally:
            torch._C._set_grad_enabled(prev)
        if any(ctx.needs_input_grad):
            self.tracked.add(id(out))
            self.nodes.append((fn, ctx, args, out, torch.cuda.current_stream() if self.streams else None))
        self.keep.append(out)
        return out

    def _backward_streams(self, out_grads):
        """`backward` with every node on the stream of its forward.  A gradient tensor becomes visible to other streams through
        the event recorded after the node that (last) wrote it; gradients are kept alive until the end so that the caching
        allocator never hands a block to one stream while another still reads it."""
        main = torch.cuda.current_stream()
        start = torch.cuda.Event()
        start.record(main)
        ready, keep, used = {}, [], {}
        grads = dict(out_grads)
        leaves = {}
        for fn, ctx, args, out, s in reversed(self.nodes):
            g = grads.pop(id(out), None)
            if g is None:
                continue
            s.wait_event(ready.get(id(g), start))
            used[id(s)] = s
            with torch.cuda.stream(s):
                res = fn.backward(ctx, g)
                if not isinstance(res, tuple):
                    res = (res,)
                wrote = []
                for a, need, ga in zip(args, ctx.needs_input_grad, res):
                    if ga is None or not need:
                        continue
                    key = id(a)
                    if key in self.tracked:
                        have = grads.get(key)
                        if have is None:
                            grads[key] = ga
                        else:
                            s.wait_event(ready.get(id(have), start))
                            F_.add_inplace(ga, have)
                        wrote.append(grads[key])
                    else:
                        have = leaves.get(key)
                        if have is None:
                            leaves[key] = (a, ga)
                        else:
                            s.wait_event(ready.get(id(have[1]), start))
                            leaves[key] = (a, have[1] + ga)
                        wrote.append(leaves[key][1])
                done = torch.cuda.Event()
                done.record(s)
            for t in wrote:
                ready[id(t)] = done
            keep.append(g)
            keep.extend(r for r in res if r is not None)
        for s in used.values():      # join: everything (incl. gradients accumulated in place by the kernels) is done
            e = torch.cuda.Event()
            e.record(s)
            main.wait_event(e)
        self._bwd_keep = keep
        return leaves

    def backward(self, out_grads):
        """out_grads: {id(output tensor): gradient}.  Returns {id: (leaf tensor, gradient)} for everything that is not a
        tape intermediate: parameters and tensors of the surrounding torch autograd graph (the scalar plumbing)."""
        if self.streams:
            return self._backward_streams(out_grads)
        grads = dict(out_grads)
        leaves = {}
        for fn, ctx, args, out, _ in reversed(self.nodes):
            g = grads.pop(id(out), None)
            if g is None:
                continue
            res = fn.backward(ctx, g)
            if not isinstance(res, tuple):
                res = (res,)
            for a, need, ga in zip(args, ctx.needs_input_grad, res):
                if ga is None or not need:
                    continue
                key = id(a)
                if key in self.tracked:
                    have = grads.get(key)
                    grads[key] = ga if have is None else F_.add_inplace(ga, have)   # have += ga on our kernel
                else:
                    have = leaves.get(key)
                    leaves[key] = (a, ga) if have is None else (a, have[1] + ga)
        return leaves


def call(fn, *args):
    """Execute one unit: as its own torch.autograd node (default) or on the active tape."""
    if _TAPE is None:
        return fn.apply(*args)
    return _TAPE.record(fn, args)


class TapedForwardFn(torch.autograd.Function):
    """forward(body, n_inputs, *inputs, *parameters): runs `body(*inputs)` with a tape active and returns its tuple of
    output tensors; backward replays the tape and hands every parameter its gradient."""

    @staticmethod
    def forward(ctx, body, n_inputs, *tensors):
        global _TAPE
        assert _TAPE is None, "nested taped forwards are not supported"
        tape = Tape()
        _TAPE = tape
        try:
            with torch.enable_grad():      # scalar plumbing on the architecture parameters builds a normal torch graph
                outs = body(*tensors[:n_inputs])
        finally:
            _TAPE = None
        outs = tuple(outs) if isinstance(outs, (tuple, list)) else (outs,)
        ctx.tape = tape
        ctx.out_ids = [id(o) for o in outs]
        ctx.params = tensors[n_inputs:]
        ctx.n_inputs = n_inputs
        ctx.mark_non_differentiable(*[o for o in outs if id(o) not in tape.tracked])
        return outs

    @staticmethod
    def backward(ctx, *gouts):
        leaves = ctx.tape.backward({oid: g for oid, g in zip(ctx.out_ids, gouts) if g is not None})
        result = {}
        plumbing, plumbing_grads = [], []
        for t, g in leaves.values():
            if t.grad_fn is not None:          # produced by torch ops from the architecture parameters
                plumbing.append(t)
                plumbing_grads.append(g.to(t.dtype).reshape(t.shape))
            else:
                result[id(t)] = g
        if plumbing:
            # differentiate the scalar plumbing: accumulates straight into the .grad of the architecture parameters, which is
            # what the outer engine would do with returned gradients (re-entrant autograd is allowed inside a backward)
            torch.autograd.backward(plumbing, plumbing_grads)
        ctx.tape = None
        return (None, None) + (None,) * ctx.n_inputs + tuple(result.get(id(p)) for p in ctx.params)


def run_taped(module, body, *inputs):
    """One autograd node for `body(*inputs)`; all parameters of `module` that require a gradient are its inputs."""
    # walking 3 700 parameters through nn.Module.parameters() costs ~40 ms; Parameter objects are stable for the life of a
    # model (optimizers rely on that too), so the list is taken once -- delete `module._fsb_params` after surgery on a model
    params = module.__dict__.get("_fsb_params")
    if params is None:
        params = [p for p in module.parameters() if p.requires_grad]
        module.__dict__["_fsb_params"] = params
    return TapedForwardFn.apply(body, len(inputs), *inputs, *params)


def _dy(t):
    """Incoming gradient as an NHWC fp16 view (autograd may hand us a differently-strided tensor after accumulation)."""
    if F_.is_nhwc_half(t):
        return t
    return t.contiguous(memory_format=torch.channels_last) if t.dtype == torch.float16 else F_.to_nhwc_half(t)


def grad_slot(param):
    """fp32 tensor the kernels accumulate this parameter's gradient into: `param.grad` (created zero-filled on first use), or
    the staging view of the graph context that is capturing a pass (graphed.py)."""
    ctx = engine.graph_ctx()
    if ctx is not None:
        return ctx.stage(param)
    if param.grad is None:
        param.grad = torch.zeros_like(param, memory_format=torch.contiguous_format)
    return param.grad


def _dgrad_pack(conv, ci, co):
    if engine.graph_ctx() is not None:
        return engine.graph_ctx().packed(conv, ci, co, True)
    cache = conv.__dict__.setdefault("_fsb_wtcache", {})
    ver = engine._versions(conv.weight)
    hit = cache.get((ci, co))
    if hit is not None and hit[0] == ver:
        return hit[1]
    packed = F_.pack_conv_weight_dgrad(conv.weight.detach(), ci, co, conv.kernel_size[0])
    cache[(ci, co)] = (ver, packed)
    return packed


def _conv_backward(ctx_conv, x, draw, ci, co, off, need_dx, need_dw):
    k, s, p = ctx_conv.kernel_size[0], ctx_conv.stride[0], ctx_conv.padding[0]
    w = ctx_conv.weight.detach()
    dx = dw = None
    if need_dx:
        wt = _dgrad_pack(ctx_conv, ci, co)  # stride 1: one launch; stride 2: one launch per input parity plane
        dx = F_.conv_dgrad(draw, w, tuple(x.shape), ci, co, k, s, p, off=off, wpacked_t=wt)
    if need_dw:
        if FUSED_WGRAD_ACCUMULATION:
            F_.conv_wgrad(x, draw, w, ci, co, k, s, p, GRAD_SCALE, off=off, accumulate_into=grad_slot(ctx_conv.weight))
        else:
            dw = F_.conv_wgrad(x, draw, w, ci, co, k, s, p, GRAD_SCALE, off=off)
    return dx, dw


class ConvBnActFn(torch.autograd.Function):
    """act(BN_train(conv(x))): conv with fused per-channel statistics -> finalize (running-stat update) -> apply.
    One fused C-ABI call per direction (csrc/train_fused.cu) for a single process and for data parallelism with the
    library's own communicator (csrc/dp.cu: the statistics are all-reduced on the stream inside the call); with SyncBN over
    torch.distributed the statistics are all-reduced between the stages from here, so the separate entry points are used."""

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, conv, bn, relu, ci, co, off):
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        wp = engine.packed_weight(conv, ci, co)
        momentum = bn.momentum if bn.momentum is not None else 0.1
        ctx.conv, ctx.relu, ctx.ci, ctx.co, ctx.off = conv, relu, ci, co, off
        if engine.dp_world_size() == 1 or engine.dp_native():
            track = bn.track_running_stats
            y, raw, vec, d = F_.conv_bn_act_train_fwd(x, wp, co, k, s, p, off, gamma, beta, bn.eps, momentum,
                                                      bn.running_mean if track else None, bn.running_var if track else None,
                                                      bn.num_batches_tracked if track else None, relu)
            ctx.fused, ctx.desc = True, d
            ctx.save_for_backward(x, raw, y, vec, gamma)
            return y
        stats = F_.conv_stats_buffer(x, co, k, s, p, off=off)
        raw = F_.conv_fwd(x, wp, co, k, s, p, relu=False, off=off, stats=stats, out_f32=True)
        N, _, Ho, Wo = raw.shape
        stats = engine.dp_allreduce_stats(stats)
        count = N * Ho * Wo * engine.dp_world_size()
        scale, shift, mean, invstd = F_.bn_finalize(stats, count, gamma, beta, bn.eps, momentum,
                                                    bn.running_mean if bn.track_running_stats else None,
                                                    bn.running_var if bn.track_running_stats else None, want_save=True)
        if bn.track_running_stats and bn.num_batches_tracked is not None:
            bn.num_batches_tracked += 1
        y = F_.affine_act(raw, scale, shift, relu=relu)
        ctx.fused, ctx.count = False, count
        ctx.save_for_backward(x, raw, y, mean, invstd, gamma)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = _dy(dy)
        need = ctx.needs_input_grad
        if ctx.fused:
            x, raw, y, vec, gamma = ctx.saved_tensors
            conv = ctx.conv
            dw_acc = None
            if need[1]:
                if not FUSED_WGRAD_ACCUMULATION:
                    raise RuntimeError("the fused training unit accumulates weight gradients into param.grad; set "
                                       "FSB_FUSED_WGRAD=1 or enable SyncBN mode for the unfused path")
                dw_acc = grad_slot(conv.weight)
            wt = _dgrad_pack(conv, ctx.ci, ctx.co) if need[0] else None
            dx, dgamma, dbeta = F_.conv_bn_act_train_bwd(ctx.desc, x, dy, y, raw, vec, gamma, ctx.relu, wt, conv.weight.detach(),
                                                         bool(need[0]), dw_acc, GRAD_SCALE)
            return dx, None, dgamma if need[2] else None, dbeta if need[3] else None, None, None, None, None, None, None
        x, raw, y, mean, invstd, gamma = ctx.saved_tensors
        sync = engine.dp_allreduce_stats if engine.dp_world_size() > 1 else None
        draw, dgamma, dbeta = F_.bn_bwd(dy, y, raw, mean, invstd, gamma, ctx.count, ctx.relu, GRAD_SCALE,
                                        want_param_grads=bool(need[2] or need[3]), allreduce=sync)
        dx, dw = _conv_backward(ctx.conv, x, draw, ctx.ci, ctx.co, ctx.off, need[0], need[1])
        return dx, dw, dgamma if need[2] else None, dbeta if need[3] else None, None, None, None, None, None, None


class ConvBnActSelFn(torch.autograd.Function):
    """act(BN_train(conv(x))) of a slimmable unit whose width is chosen ON THE DEVICE (engine.SelBN): the unit runs at its maximum
    width, the BatchNorm kernels pick the parameter set from the width index of the pass and force the inactive channel tail to
    zero, which reproduces USConv2d / USBatchNorm2d slicing exactly (zero activations meet the unused weight columns downstream;
    zero gradients meet the unused weight rows).  gamma / beta / weight gradients are accumulated by the kernels."""

    @staticmethod
    def forward(ctx, x, weight, conv, sel, relu, ci, co):
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        wp = engine.packed_weight(conv, ci, co)
        y, raw, vec, d = F_.conv_bn_act_train_fwd_sel(x, wp, co, k, s, p, (0, 0), sel, relu)
        ctx.conv, ctx.sel, ctx.relu, ctx.ci, ctx.co, ctx.desc = conv, sel, relu, ci, co, d
        ctx.save_for_backward(x, raw, y, vec)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, raw, y, vec = ctx.saved_tensors
        need = ctx.needs_input_grad
        conv = ctx.conv
        wt = _dgrad_pack(conv, ctx.ci, ctx.co) if need[0] else None
        dx = F_.conv_bn_act_train_bwd_sel(ctx.desc, x, _dy(dy), y, raw, vec, ctx.sel, ctx.relu, wt, conv.weight.detach(), bool(need[0]),
                                          grad_slot(conv.weight) if need[1] else None, GRAD_SCALE)
        return dx, None, None, None, None, None, None


class FactorizedReduceSelFn(torch.autograd.Function):
    """FactorizedReduceFn with a device-selected width: both 1x1 stride-2 convs run at their maximum half-width hmax and write
    raw channels [0, hmax) / [hmax, 2 hmax); the BatchNorm kernels map that to the compact order [conv1[:h] | conv2[:h] | 0...]
    the parameter set and every consumer expect (h = active half-width, read on the device)."""

    @staticmethod
    def forward(ctx, x, w1, w2, op, sel, ci, hmax):
        co = 2 * hmax
        N, _, H, W = x.shape
        p1 = engine.packed_weight(op.conv1, ci, hmax)
        p2 = engine.packed_weight(op.conv2, ci, hmax)
        raw = F_.empty_nhwc(N, co, H // 2, W // 2, x.device, dtype=torch.float32)
        stats = F_.conv_stats_buffer(x, hmax, 1, 2, 0, total_C=co)
        F_.conv_fwd(x, p1, hmax, 1, 2, 0, out=raw[:, :hmax], stats=stats, out_f32=True)
        F_.conv_fwd(x, p2, hmax, 1, 2, 0, out=raw[:, hmax:], off=(1, 1), stats=stats, stats_off=hmax, out_f32=True)
        world = engine.dp_world_size()
        if world > 1:      # SyncBN: totals of all ranks (exchanged by the library, on the stream)
            stats = F_.dp_allreduce(F_.rowsum(stats))
        count = N * (H // 2) * (W // 2) * world
        scale, shift, mean, invstd = F_.bn_finalize_sel(stats, count, sel, hmax=hmax)
        y = F_.affine_act_sel(raw, scale, shift, sel, hmax, relu=True)
        ctx.op, ctx.sel, ctx.ci, ctx.hmax, ctx.count, ctx.world = op, sel, ci, hmax, count, world
        ctx.save_for_backward(x, raw, y, mean, invstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, raw, y, mean, invstd = ctx.saved_tensors
        need = ctx.needs_input_grad
        h = ctx.hmax
        draw = F_.bn_bwd_sel(_dy(dy), y, raw, mean, invstd, ctx.count, True, GRAD_SCALE, ctx.sel, hmax=h, world=ctx.world)
        dx1, _ = _conv_backward(ctx.op.conv1, x, draw[:, :h], ctx.ci, h, (0, 0), need[0], need[1])
        dx2, _ = _conv_backward(ctx.op.conv2, x, draw[:, h:], ctx.ci, h, (1, 1), need[0], need[2])
        dx = F_.add_inplace(dx2, dx1) if need[0] else None
        return dx, None, None, None, None, None, None


class ConvBiasFn(torch.autograd.Function):
    """conv(x) + bias, optional ReLU, no BN (Head.conv_1x1, seg_oprs.py:246,273)."""

    @staticmethod
    def forward(ctx, x, weight, bias, conv, relu, ci, co):
        k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        wp = engine.packed_weight(conv, ci, co)
        shift = None if bias is None else bias.detach()[:co].float().contiguous()
        y = F_.conv_fwd(x, wp, co, k, s, p, None, shift, relu=relu)
        ctx.conv, ctx.relu, ctx.ci, ctx.co = conv, relu, ci, co
        ctx.save_for_backward(x, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y = ctx.saved_tensors
        dy = _dy(dy)
        if ctx.relu:
            dy = F_.relu_bwd(dy, y)
        need = ctx.needs_input_grad
        dx, dw = _conv_backward(ctx.conv, x, dy, ctx.ci, ctx.co, (0, 0), need[0], need[1])
        db = None
        if need[2]:
            # bias gradient = per-channel sum of dy: reuse the statistics kernel (first half of its output)
            full = torch.zeros(ctx.conv.bias.shape, device=dy.device, dtype=torch.float32)
            full[:ctx.co] = F_.bn_stats(dy)[:ctx.co] / GRAD_SCALE
            db = full
        return dx, dw, db, None, None, None, None


class FactorizedReduceFn(torch.autograd.Function):
    """cat[conv1(x), conv2(x[:, :, 1:, 1:])] -> BN(train) -> ReLU (operations.py:521-526) as one node."""

    @staticmethod
    def forward(ctx, x, w1, w2, gamma, beta, op, bn, ci, co_half):
        co = 2 * co_half
        N, _, H, W = x.shape
        p1 = engine.packed_weight(op.conv1, ci, co_half)
        p2 = engine.packed_weight(op.conv2, ci, co_half)
        raw = F_.empty_nhwc(N, co, H // 2, W // 2, x.device, dtype=torch.float32)
        # both halves write their columns of ONE statistics buffer (rows are per spatial tile, identical for the two convs)
        stats = F_.conv_stats_buffer(x, co_half, 1, 2, 0, total_C=co)
        F_.conv_fwd(x, p1, co_half, 1, 2, 0, out=raw[:, :co_half], stats=stats, out_f32=True)
        F_.conv_fwd(x, p2, co_half, 1, 2, 0, out=raw[:, co_half:], off=(1, 1), stats=stats, stats_off=co_half, out_f32=True)
        stats = engine.dp_allreduce_stats(stats)
        count = N * (H // 2) * (W // 2) * engine.dp_world_size()
        scale, shift, mean, invstd = F_.bn_finalize(stats, count, gamma, beta, bn.eps, 0.1 if bn.momentum is None else bn.momentum,
                                                    bn.running_mean, bn.running_var, want_save=True)
        if bn.num_batches_tracked is not None:
            bn.num_batches_tracked += 1
        y = F_.affine_act(raw, scale, shift, relu=True)
        ctx.op, ctx.ci, ctx.co_half, ctx.count = op, ci, co_half, count
        ctx.save_for_backward(x, raw, y, mean, invstd, gamma)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, raw, y, mean, invstd, gamma = ctx.saved_tensors
        dy = _dy(dy)
        need = ctx.needs_input_grad
        sync = engine.dp_allreduce_stats if engine.dp_world_size() > 1 else None
        draw, dgamma, dbeta = F_.bn_bwd(dy, y, raw, mean, invstd, gamma, ctx.count, True, GRAD_SCALE,
                                        want_param_grads=bool(need[3] or need[4]), allreduce=sync)
        ch = ctx.co_half
        dx1, dw1 = _conv_backward(ctx.op.conv1, x, draw[:, :ch], ctx.ci, ch, (0, 0), need[0], need[1])
        dx2, dw2 = _conv_backward(ctx.op.conv2, x, draw[:, ch:], ctx.ci, ch, (1, 1), need[0], need[2])
        dx = None
        if need[0]:
            dx = F_.add_inplace(dx2, dx1)
        return dx, dw1, dw2, dgamma if need[3] else None, dbeta if need[4] else None, None, None, None, None


class BilinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, size, relu):
        y = F_.bilinear(x, size, relu=relu)
        ctx.in_hw, ctx.relu = (x.shape[2], x.shape[3]), relu
        if relu:
            ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        mask = ctx.saved_tensors[0] if ctx.relu else None
        return F_.bilinear_bwd(_dy(dy), ctx.in_hw, relu_mask_y=mask), None, None


class UpsampleLogitsFn(torch.autograd.Function):
    """NHWC fp16 logits -> upsampled NCHW logits (model_seg.py:359-361); backward re-enters the fp16 domain (x GRAD_SCALE)."""

    @staticmethod
    def forward(ctx, x, size, dtype):
        ctx.in_hw = (x.shape[2], x.shape[3])
        return F_.upsample_logits(x, size, dtype=dtype)

    @staticmethod
    def backward(ctx, dy):
        return F_.upsample_logits_bwd(dy, ctx.in_hw, GRAD_SCALE), None, None


class ToNCHWFn(torch.autograd.Function):
    """NHWC fp16 -> NCHW fp32 (logits handed to the caller's criterion at 1/8 resolution, model_search.py:346-358)."""

    @staticmethod
    def forward(ctx, x, dtype):
        return F_.to_nchw(x, dtype)

    @staticmethod
    def backward(ctx, dy):
        return F_.nchw_grad_to_nhwc(dy, GRAD_SCALE), None


class WsumFn(torch.autograd.Function):
    """out = sum_k wts[k] * xs[k] (MixedOp / beta aggregation, model_search.py:75-78,330-333) in one kernel."""

    @staticmethod
    def forward(ctx, wts, *xs):
        wts32 = wts.detach().float().contiguous()
        out = F_.wsum_fwd(list(xs), wts32)
        ctx.save_for_backward(wts32, *xs)
        return out

    @staticmethod
    def backward(ctx, dout):
        wts32, *xs = ctx.saved_tensors
        need = ctx.needs_input_grad
        dxs, dw = F_.wsum_bwd(_dy(dout), list(xs), wts32, [bool(n) for n in need[1:]], bool(need[0]), GRAD_SCALE)
        return (dw, *dxs)


class CatFn(torch.autograd.Function):
    """torch.cat(dim=1) (operations.py:523, model_search.py:340-350, model_seg.py:307-331): strided copies forward,
    channel-slice views backward."""

    @staticmethod
    def forward(ctx, *xs):
        N, _, H, W = xs[0].shape
        ctx.sizes = [t.shape[1] for t in xs]
        out = F_.empty_nhwc(N, sum(ctx.sizes), H, W, xs[0].device)
        at = 0
        for t in xs:
            F_.copy_channels(t, out[:, at:at + t.shape[1]])
            at += t.shape[1]
        return out

    @staticmethod
    def backward(ctx, dy):
        dy = _dy(dy)
        outs, at = [], 0
        for c in ctx.sizes:
            outs.append(dy[:, at:at + c])
            at += c
        return tuple(outs)


# ----------------------------------------------------------------------------------------------
# entry points used by engine / operations / models
# ----------------------------------------------------------------------------------------------
def conv_bn_act_train(x, conv, bn, relu, ci, co, out=None, off=(0, 0)):
    assert conv.bias is None, "conv bias followed by train-mode BN is not on the hot path"
    y = call(ConvBnActFn, x, conv.weight, bn.weight, bn.bias, conv, bn, relu, ci, co, off)
    if out is not None:  # autograd-visible copy into a caller-provided slot (training path does not use zero-copy concat)
        raise RuntimeError("out= is an inference-only fast path")
    return y


def conv_bn_act_train_sel(x, conv, sel, relu, ci, co):
    assert conv.bias is None
    assert FUSED_WGRAD_ACCUMULATION, "device-selected units accumulate weight gradients in the kernels"
    return call(ConvBnActSelFn, x, conv.weight, conv, sel, relu, ci, co)


def factorized_reduce_sel(op, x, sel, ci, hmax):
    assert FUSED_WGRAD_ACCUMULATION
    return call(FactorizedReduceSelFn, x, op.conv1.weight, op.conv2.weight, op, sel, ci, hmax)


def conv_bias_act(x, conv, relu, ci, co):
    return call(ConvBiasFn, x, conv.weight, conv.bias, conv, relu, ci, co)


def factorized_reduce_train(op, x, bn, ci, co_half, out=None):
    if out is not None:
        raise RuntimeError("out= is an inference-only fast path")
    return call(FactorizedReduceFn, x, op.conv1.weight, op.conv2.weight, bn.weight, bn.bias, op, bn, ci, co_half)


def bilinear(x, size, relu=False):
    return call(BilinearFn, x, (int(size[0]), int(size[1])), relu)


def upsample_logits(x, size, dtype=torch.float32):
    return call(UpsampleLogitsFn, x, (int(size[0]), int(size[1])), dtype)


def to_nchw(x, dtype=torch.float32):
    return call(ToNCHWFn, x, dtype)


class SupernetLatencyFn(torch.autograd.Function):
    """Network_Multi_Path.forward_latency (model_search.py:361-475) as K14: one launch forward, one backward.  Inputs the plan does
    not differentiate arrive detached and get None, like the walk, which never puts them in the graph (Adam then skips them)."""

    @staticmethod
    def forward(ctx, plan, noise, diff, *params):
        dev = noise.device
        ws = torch.empty(F_.supernet_latency_workspace_bytes(plan.host) // 4, dtype=torch.float32, device=dev)
        out = torch.empty((), dtype=torch.float32, device=dev)
        F_.supernet_latency_fwd(plan.host, plan.on(dev), params, noise, ws, out)
        ctx.plan, ctx.diff, ctx.ws = plan, diff, ws
        ctx.shapes = [p.shape for p in params]
        return out

    @staticmethod
    def backward(ctx, gout):
        dev = gout.device
        grads = [torch.empty(s, dtype=torch.float32, device=dev) if d else None for s, d in zip(ctx.shapes, ctx.diff)]
        F_.supernet_latency_bwd(ctx.plan.host, ctx.plan.on(dev), gout.float().contiguous(), ctx.ws, grads)
        return (None, None, None, *grads)


def supernet_latency(plan, noise, params, diff):
    return SupernetLatencyFn.apply(plan, noise, tuple(diff), *params)


def weighted_sum(wts, xs):
    return call(WsumFn, wts, *xs)


def cat_channels(xs):
    xs = [F_.to_nhwc_half(t) for t in xs]
    return xs[0] if len(xs) == 1 else call(CatFn, *xs)


def grad_mode(*tensors):
    """True when an autograd graph must be recorded for these inputs."""
    if _TAPE is not None:
        return any(_TAPE.needs(t) for t in tensors)
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


class FusedOhemCEFn(torch.autograd.Function):
    """ProbOhemCrossEntropy2d(F.interpolate(x, size, bilinear, align_corners=True), target) (tools/seg_opr/loss_opr.py:63-93 on
    train/model_seg.py:357-362's upsampled logits) from the LOW-RESOLUTION NHWC fp16 logits x: csrc/loss.cu.  No tensor of label
    resolution with a class axis exists in either direction; the OHEM threshold is an exact order statistic (no sort, no sync)."""

    @staticmethod
    def forward(ctx, x, target, size, ignore_label, thresh, min_kept):
        import math
        target = target.contiguous()
        Cc = x.shape[1]
        logp, lse = F_.loss_logp_fwd(x, target, size, ignore_label)
        valid = (target != ignore_label) & (target >= 0) & (target < Cc)
        num_valid = valid.sum()
        thr = None
        if min_kept > 0:
            n = logp.numel()
            kth = F_.kth_smallest(logp.view(-1), min(n, int(min_kept)))
            thr = torch.clamp(kth, min=math.log(thresh))                         # max(k-th smallest prob, thresh), in log space
            mining = (num_valid >= min_kept) & (num_valid > 0)                    # loss_opr.py:68-71: no mining with fewer valid pixels
            thr = torch.where(mining, thr, torch.full_like(thr, float("inf"))).contiguous()
        sums = F_.ohem_reduce(logp, target, ignore_label, Cc, thr)
        loss = sums[0] / sums[1]
        ctx.save_for_backward(x, target, lse, logp, thr if thr is not None else torch.empty(0, device=x.device), sums)
        ctx.cfg = (tuple(int(v) for v in size), int(ignore_label), thr is not None)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        x, target, lse, logp, thr, sums = ctx.saved_tensors
        size, ignore_label, has_thr = ctx.cfg
        coef = (dloss.float() / sums[1]).reshape(1).contiguous()
        dx = F_.loss_ce_bwd(x, target, size, ignore_label, lse, logp, thr if has_thr else None, coef, GRAD_SCALE)
        return dx, None, None, None, None, None


class FusedKLFn(torch.autograd.Function):
    """nn.KLDivLoss(reduction='mean')(log_softmax(up(xs)), softmax(up(xt))) (train/train.py:254-260) from the two low-resolution
    NHWC fp16 logit maps; gradient w.r.t. the student only (the teacher runs under no_grad in the reference)."""

    @staticmethod
    def forward(ctx, xs, xt, size):
        total, lse_s, lse_t = F_.loss_kl_fwd(xs, xt, size)
        numel = float(xs.shape[0] * xs.shape[1] * int(size[0]) * int(size[1]))
        ctx.save_for_backward(xs, xt, lse_s, lse_t)
        ctx.cfg = (tuple(int(v) for v in size), numel)
        return total / numel

    @staticmethod
    def backward(ctx, dloss):
        xs, xt, lse_s, lse_t = ctx.saved_tensors
        size, numel = ctx.cfg
        coef = (dloss.float() / numel).reshape(1).contiguous()
        return F_.loss_kl_bwd(xs, xt, size, lse_s, lse_t, coef, GRAD_SCALE), None, None


def fused_ohem_ce(x, target, size, ignore_label, thresh, min_kept):
    return call(FusedOhemCEFn, x, target, (int(size[0]), int(size[1])), int(ignore_label), float(thresh), int(min_kept))


def fused_kl(xs, xt, size):
    return call(FusedKLFn, xs, xt, (int(size[0]), int(size[1])))
