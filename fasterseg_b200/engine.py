"""Fused conv -> BatchNorm -> activation unit used by every operator class of the boundary.

What the reference executes as three framework calls and three HBM round trips
(nn.Conv2d / USConv2d -> nn.BatchNorm2d / USBatchNorm2d -> nn.ReLU, e.g. search/operations.py:72-83,196-200)
runs here as ONE kernel in eval mode (BN folded into the conv epilogue) and as conv(+fused statistics) ->
finalize -> apply in training mode.  Master parameters stay fp32 in the nn.Module (checkpoint format);
packed fp16 weights and folded BN vectors are cached per module and invalidated through tensor version counters.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import functional as F_


# ----------------------------------------------------------------------------------------------
# Device-selected widths (captured training graphs, graphed.py).  A SymRatio stands for "the width whose index sits in slot
# `slot` of the pass's width-index vector on the device"; a slimmable conv given a SymRatio runs at its MAXIMUM width and its
# USBatchNorm2d hands out a SelBN (all per-width parameter sets as a device table) instead of one nn.BatchNorm2d.
# ----------------------------------------------------------------------------------------------
class SymRatio:
    __slots__ = ("slot",)

    def __init__(self, slot):
        self.slot = int(slot)

    def __repr__(self):
        return "SymRatio(%d)" % self.slot


class SelBN:
    """The per-width nn.BatchNorm2d sets of one USBatchNorm2d, selected on the device by the width index in slot `slot`."""
    training = True

    def __init__(self, usbn, slot, ctx):
        self.usbn, self.slot, self.ctx = usbn, int(slot), ctx
        self.bns = list(usbn.bn)
        self.eps = self.bns[0].eps
        self.momentum = 0.1 if self.bns[0].momentum is None else self.bns[0].momentum
        assert all(b.eps == self.eps and (0.1 if b.momentum is None else b.momentum) == self.momentum and b.track_running_stats
                   for b in self.bns), "the per-width BatchNorm sets of a slimmable unit must share eps / momentum"
        self.C_max = usbn.num_features_max

    @property
    def table_ptr(self):
        return self.ctx.sel_table_ptr(self)

    @property
    def idx_ptr(self):
        return self.ctx.width_idx_ptr(self.slot)


_GRAPH_CTX = None   # the graphed.PassContext that is currently building / capturing a pass (None: ordinary execution)


def graph_ctx():
    return _GRAPH_CTX


WEIGHTS_EPOCH = 0      # bumped by optimizers that write parameters through raw pointers (optim.FlatSGD)


def bump_weights_epoch():
    global WEIGHTS_EPOCH
    WEIGHTS_EPOCH += 1


def _versions(*tensors):
    return (WEIGHTS_EPOCH,) + tuple(-1 if t is None else (t._version, t.data_ptr()) for t in tensors)


def packed_weight(conv: nn.Conv2d, ci: int, co: int) -> torch.Tensor:
    """fp16 packed copy of conv.weight[:co, :ci] (USConv2d slice, slimmable_ops.py:42), cached."""
    if _GRAPH_CTX is not None:
        return _GRAPH_CTX.packed(conv, ci, co, False)
    cache = conv.__dict__.setdefault("_fsb_wcache", {})
    key = (ci, co)
    weight = conv.weight
    ver = (weight._version, weight.data_ptr(), WEIGHTS_EPOCH)
    hit = cache.get(key)
    if hit is not None and hit[0] == ver:
        return hit[1]
    w = weight.detach()
    if w.dtype != torch.float32:
        w = w.float()
    packed = F_.pack_conv_weight(w, ci, co, conv.kernel_size[0])
    cache[key] = (ver, packed)
    return packed


def folded_bn(bn: Optional[nn.BatchNorm2d], co: int, conv_bias: Optional[torch.Tensor]):
    """(scale, shift) fp32[co] of eval-mode BN (+ conv bias), cached; (None, bias) when there is no BN."""
    if bn is None:
        if conv_bias is None:
            return None, None
        return None, conv_bias.detach()[:co].float().contiguous()
    cache = bn.__dict__.setdefault("_fsb_bncache", {})
    ver = _versions(bn.weight, bn.bias, bn.running_mean, bn.running_var, conv_bias) + (bn.eps,)
    hit = cache.get(co)
    if hit is not None and hit[0] == ver:
        return hit[1], hit[2]
    assert bn.running_mean is not None and bn.running_mean.numel() == co, \
        "BatchNorm has %s features, conv produces %d" % (None if bn.running_mean is None else bn.running_mean.numel(), co)
    scale, shift = F_.bn_fold(bn.weight.detach() if bn.weight is not None else None,
                              bn.bias.detach() if bn.bias is not None else None,
                              bn.running_mean, bn.running_var, bn.eps,
                              None if conv_bias is None else conv_bias.detach()[:co].contiguous())
    cache[co] = (ver, scale, shift)
    return scale, shift


def active_channels(conv: nn.Conv2d):
    """(ci, co) the conv runs with: USConv2d resolves them from its ratio (slimmable_ops.py:36-40)."""
    resolve = getattr(conv, "_resolve_channels", None)
    if resolve is not None:
        return resolve()
    return conv.in_channels, conv.out_channels


def active_bn(bn):
    """USBatchNorm2d dispatches to the per-width nn.BatchNorm2d (slimmable_ops.py:66-69)."""
    pick = getattr(bn, "_active_bn", None)
    return pick() if pick is not None else bn


def conv_bn_act(x: torch.Tensor, conv: nn.Conv2d, bn: Optional[nn.BatchNorm2d], relu: bool,
                out: Optional[torch.Tensor] = None, off=(0, 0), out_half: Optional[torch.Tensor] = None) -> torch.Tensor:
    """act(BN(conv(x))) on NHWC fp16 views.  `off` = input origin shift (FactorizedReduce, operations.py:523).  out_half: also
    write bilinear(y, (Ho // 2, Wo // 2)) there -- from the conv's own epilogue with eval-mode BN (F_.conv_fwd), else by a
    separate resize."""
    x = F_.to_nhwc_half(x)
    ci, co = active_channels(conv)
    assert x.shape[1] == ci, "input has %d channels, conv expects %d" % (x.shape[1], ci)
    k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
    assert conv.dilation[0] == 1 and conv.groups == 1, "only dense dilation-1 convs are on the hot path (SURVEY section 0)"
    wp = packed_weight(conv, ci, co)
    bn = active_bn(bn) if bn is not None else None
    from . import autograd as AG
    if out_half is not None and ((bn is not None and (bn.training or bn.running_mean is None)) or AG.grad_mode(x, conv.weight)):
        y = conv_bn_act(x, conv, bn, relu, out=out, off=off)   # batch statistics (SelBN included) or autograd: a separate /2
        F_.bilinear(y, (y.shape[2] // 2, y.shape[3] // 2), out=out_half)
        return y
    if isinstance(bn, SelBN):
        from .autograd import conv_bn_act_train_sel
        assert out is None and off == (0, 0)
        return conv_bn_act_train_sel(x, conv, bn, relu, ci, co)
    training = bn is not None and (bn.training or bn.running_mean is None)
    want_grad = AG.grad_mode(x, conv.weight)
    if not training:
        if want_grad and bn is None:
            from .autograd import conv_bias_act  # conv (+bias) with backward, e.g. Head.conv_1x1
            assert out is None and off == (0, 0)
            return conv_bias_act(x, conv, relu, ci, co)
        # eval-mode BN: inference only (the teacher runs under no_grad, train/train.py:249-252)
        scale, shift = folded_bn(bn, co, conv.bias)
        half = {} if out_half is None else {"out_half": out_half}   # only where given: wrappers' stand-ins need not know it
        return F_.conv_fwd(x, wp, co, k, s, p, scale, shift, relu=relu, out=out, off=off, **half)
    if want_grad:
        from .autograd import conv_bn_act_train  # training path with backward
        return conv_bn_act_train(x, conv, bn, relu, ci, co, out=out, off=off)
    return conv_bn_act_train_nograd(x, conv, bn, relu, ci, co, out=out, off=off)


def conv_bn_act_train_nograd(x, conv, bn, relu, ci, co, out=None, off=(0, 0)):
    """Training-mode forward without autograd: batch statistics + running-stat update (K2/K3)."""
    assert conv.bias is None, "conv bias followed by train-mode BN is not on the hot path"
    k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
    wp = packed_weight(conv, ci, co)
    stats = F_.conv_stats_buffer(x, co, k, s, p, off=off)
    raw = F_.conv_fwd(x, wp, co, k, s, p, relu=False, off=off, stats=stats, out_f32=True)
    N, _, Ho, Wo = raw.shape
    stats = dp_allreduce_stats(stats)
    count = N * Ho * Wo * dp_world_size()
    momentum = bn.momentum if bn.momentum is not None else 0.1
    scale, shift, _, _ = F_.bn_finalize(stats, count, bn.weight, bn.bias, bn.eps, momentum,
                                        bn.running_mean if bn.track_running_stats else None,
                                        bn.running_var if bn.track_running_stats else None)
    if bn.track_running_stats and bn.num_batches_tracked is not None:
        bn.num_batches_tracked += 1
    return F_.affine_act(raw, scale, shift, relu=relu, out=out)


# ----------------------------------------------------------------------------------------------
# data-parallel hooks (SyncBN statistics); identity when torch.distributed is not initialised
# ----------------------------------------------------------------------------------------------
_SYNC_BN = {"enabled": False, "group": None, "native": False}


def enable_sync_bn(enabled=True, group=None):
    _SYNC_BN["enabled"] = enabled
    _SYNC_BN["group"] = group
    if _SYNC_BN["native"]:   # the library's own communicator follows the switch (a rank-0-only reference run must not all-reduce)
        from . import _lib
        _lib.check(_lib.lib().fsb_dp_enable(1 if enabled else 0), "fsb_dp_enable")
        _lib.check(_lib.lib().fsb_peer_enable(1 if enabled else 0), "fsb_peer_enable")


def dp_world_size():
    if _SYNC_BN["enabled"] and torch.distributed.is_available() and torch.distributed.is_initialized():
        return torch.distributed.get_world_size(_SYNC_BN["group"])
    return 1


def dp_native():
    """True when the library owns a NCCL communicator (parallel.init_native_dp): the fused training units then exchange
    their BatchNorm statistics themselves, on the stream, and stay on the one-call-per-unit path under data parallelism."""
    return _SYNC_BN["native"] and _SYNC_BN["enabled"]


def dp_allreduce_stats(stats):
    """SyncBN exchange.  `stats` = partial rows [R, L] (or totals [L]); with more than one rank the rows are first added in
    index order (deterministic), then summed over the ranks; single process: returned untouched (bn_finalize adds the rows)."""
    if dp_world_size() > 1:
        if stats.dim() == 2 and stats.shape[0] > 1:
            stats = F_.rowsum(stats)
        torch.distributed.all_reduce(stats, group=_SYNC_BN["group"])
    return stats
