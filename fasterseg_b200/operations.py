"""The five search-space primitives + ConvNorm -- drop-in for the reference's operations.py.

API kept from search/operations.py:42-552: class names, constructor signatures, `forward`, `set_ratio`,
`forward_latency` (same lookup-table key strings), static `_latency` / `_flops`, attributes
(`C_in, C_out, stride, ratio, slimmable, width_mult_list`), registries `OPS / OPS_name / OPS_Class`
and the parameter names that make up the checkpoint format (`conv1.weight`, `bn1.bn.{i}.*`, `conv.0.weight` ...).

Execution differs completely: activations are NHWC fp16, each conv+BN(+ReLU) is one fused wgmma
implicit-GEMM kernel (`engine.conv_bn_act`), the "zoomed" ops run bilinear down / up as vectorised resize
kernels with the trailing ReLU fused into the upsample, and `out=` lets a caller have the result written
straight into a channel slice of a concat buffer.
"""
__all__ = ['ConvNorm', 'BasicResidual1x', 'BasicResidual_downup_1x', 'BasicResidual2x', 'BasicResidual_downup_2x',
           'FactorizedReduce', 'OPS', 'OPS_name', 'OPS_Class']

import os.path as osp
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import engine
from . import functional as F_
from .slimmable_ops import USBatchNorm2d, USConv2d

BatchNorm2d = nn.BatchNorm2d

# per-op latency table (ms) consulted by forward_latency; the reference loads it from cwd at import time
# (search/operations.py:33-36) and so do we -- same file name, same keys.
latency_lookup_table = {}
table_file_name = "latency_lookup_table.npy"
if osp.isfile(table_file_name):
    latency_lookup_table = np.load(table_file_name, allow_pickle=True).item()


def compute_latency(layer, input_size, iterations=None):
    from .latency import compute_latency_ms
    return compute_latency_ms(layer, input_size, iterations=iterations)


def _table_latency(name, measure):
    """Lookup-or-measure-and-persist, as every forward_latency in the reference does (e.g. operations.py:116-122)."""
    if name in latency_lookup_table:
        return latency_lookup_table[name]
    print("not found in latency_lookup_table:", name)
    latency = measure()
    latency_lookup_table[name] = latency
    np.save(table_file_name, latency_lookup_table)
    return latency


def _conv(slimmable, c_in, c_out, k, stride, padding, dilation, groups, bias, width_mult_list):
    if slimmable:
        return USConv2d(c_in, c_out, k, stride, padding=padding, dilation=dilation, groups=groups, bias=bias,
                        width_mult_list=width_mult_list)
    return nn.Conv2d(c_in, c_out, k, stride, padding=padding, dilation=dilation, groups=groups, bias=bias)


def _norm(slimmable, c, width_mult_list):
    return USBatchNorm2d(c, width_mult_list) if slimmable else BatchNorm2d(c)


def _conv_macs(h, w, c_in, c_out, k, stride):
    return (h // stride) * (w // stride) * c_in * c_out * k * k


class _Primitive(nn.Module):
    """Shared bookkeeping of the primitives: ratio plumbing, output-size rule and latency-table access."""
    _table_prefix = None  # key prefix in latency_lookup_table

    def _init_common(self, C_in, C_out, kernel_size, stride, dilation, groups, slimmable, width_mult_list):
        assert stride in [1, 2]
        self.C_in, self.C_out = C_in, C_out
        self.kernel_size = kernel_size
        self.stride = stride
        self.dilation = 1 if stride == 2 else dilation
        self.groups = groups
        self.slimmable = slimmable
        self.width_mult_list = width_mult_list
        self.ratio = (1., 1.)
        self.relu = nn.ReLU(inplace=True)  # parameter-free; kept for module-tree parity (fused into the kernels)

    def _active_io(self, c_in):
        """Checks `c_in` against the configured width and returns the active output channels (int(C*ratio), like
        the reference's forward_latency -- NOT make_divisible)."""
        if self.slimmable:
            assert c_in == int(self.C_in * self.ratio[0]), "c_in %d, int(self.C_in * self.ratio[0]) %d" % (
                c_in, int(self.C_in * self.ratio[0]))
            return int(self.C_out * self.ratio[1])
        assert c_in == self.C_in, "c_in %d, self.C_in %d" % (c_in, self.C_in)
        return self.C_out

    def _out_hw(self, h, w):
        return (h, w) if self.stride == 1 else (h // 2, w // 2)

    def _set_pairs(self, ratio, convs_bns):
        assert len(ratio) == 2
        self.__dict__["ratio"] = ratio   # plain attribute on the per-step hot path: bypass nn.Module.__setattr__
        first = True
        for conv, bn in convs_bns:
            conv.set_ratio(ratio if first else (ratio[1], ratio[1]))
            bn.set_ratio(ratio[1])
            first = False


class ConvNorm(_Primitive):
    '''conv => norm => activation (reference: search/operations.py:42-128).'''

    def __init__(self, C_in, C_out, kernel_size=3, stride=1, padding=None, dilation=1, groups=1, bias=False,
                 slimmable=True, width_mult_list=[1.]):
        super(ConvNorm, self).__init__()
        assert type(groups) == int
        self._init_common(C_in, C_out, kernel_size, stride, dilation, 1 if kernel_size == 1 else groups, slimmable,
                          width_mult_list)
        self.dilation = dilation
        # "assume h_out = h_in / s"
        self.padding = int(np.ceil((dilation * (kernel_size - 1) + 1 - stride) / 2.)) if padding is None else padding
        self.bias = bias
        del self.relu
        self.conv = nn.Sequential(
            _conv(slimmable, C_in, C_out, kernel_size, stride, self.padding, dilation, self.groups, bias, width_mult_list),
            _norm(slimmable, C_out, width_mult_list),
            nn.ReLU(inplace=True),
        )

    def set_ratio(self, ratio):
        assert self.slimmable
        assert len(ratio) == 2
        self.__dict__["ratio"] = ratio
        self.conv[0].set_ratio(ratio)
        self.conv[1].set_ratio(ratio[1])

    @staticmethod
    def _flops(h, w, C_in, C_out, kernel_size=3, stride=1, padding=None, dilation=1, groups=1, bias=False):
        return _conv_macs(h, w, C_in, C_out, kernel_size, stride) + 2 * (h // stride) * (w // stride) * C_out

    @staticmethod
    def _latency(h, w, C_in, C_out, kernel_size=3, stride=1, padding=None, dilation=1, groups=1, bias=False):
        layer = ConvNorm(C_in, C_out, kernel_size, stride, padding, dilation, groups, bias, slimmable=False)
        return compute_latency(layer, (1, C_in, h, w))

    def latency_key(self, size):
        """(latency-table key, output size) of this op at the configured ratio for an input of `size` = (C, H, W)"""
        c_in, h_in, w_in = size
        if self.slimmable:
            assert c_in == int(self.C_in * self.ratio[0]), "c_in %d, self.C_in * self.ratio[0] %d" % (c_in, self.C_in * self.ratio[0])
            c_out = int(self.C_out * self.ratio[1])
        else:
            assert c_in == self.C_in, "c_in %d, self.C_in %d" % (c_in, self.C_in)
            c_out = self.C_out
        h_out, w_out = self._out_hw(h_in, w_in)
        name = "ConvNorm_H%d_W%d_Cin%d_Cout%d_kernel%d_stride%d" % (h_in, w_in, c_in, c_out, self.kernel_size, self.stride)
        return name, (c_out, h_out, w_out)

    def forward_latency(self, size):
        name, size_out = self.latency_key(size)
        c_in, h_in, w_in = size
        latency = _table_latency(name, lambda: ConvNorm._latency(h_in, w_in, c_in, size_out[0], self.kernel_size, self.stride,
                                                                 self.padding, self.dilation, self.groups, self.bias))
        return latency, size_out

    def forward(self, x, out=None):
        assert x.size()[1] == self.C_in, "{} {}".format(x.size()[1], self.C_in)
        conv, bn = self.conv[0], self.conv[1]
        if x.dtype == torch.uint8:
            # the image itself (uint8 HWC behind a logical NCHW view): normalisation folded into the stem's gather (evaluator path)
            lut = self.__dict__.get("_fsb_norm_lut")
            assert lut is not None, "uint8 input needs set_input_normalization(mean, std) on the network"
            assert self.C_in == 3 and self.kernel_size == 3 and self.stride == 2 and self.padding == 1 and not bn.training
            scale, shift = engine.folded_bn(bn, self.C_out, None)
            w = conv.weight.detach()
            return F_.stem_conv_u8hwc(x, lut, w if w.dtype == torch.float32 else w.float(), scale, shift, relu=True, out=out)
        if (self.C_in == 3 and self.kernel_size == 3 and self.stride == 2 and self.padding == 1 and not self.slimmable
                and not F_.is_nhwc_half(x) and not bn.training and conv.bias is None and x.is_contiguous()):
            # RGB stem straight from the caller's NCHW tensor (model_seg.py:193, model_search.py:148)
            scale, shift = engine.folded_bn(bn, self.C_out, None)
            w = conv.weight.detach()
            return F_.stem_conv_nchw(x if x.dtype in (torch.float32, torch.float16) else x.float(),
                                     w if w.dtype == torch.float32 else w.float(), scale, shift, relu=True, out=out)
        return engine.conv_bn_act(x, conv, bn, relu=True, out=out)


class _Residual(_Primitive):
    """Common body of the four residual-style primitives: `n_convs` 3x3 conv+BN stages, optionally wrapped in a
    bilinear /2 ... x2 "zoom" (reference: search/operations.py:131-446)."""
    _n_convs = 1
    _zoom = False

    def __init__(self, C_in, C_out, kernel_size=3, stride=1, dilation=1, groups=1, slimmable=True, width_mult_list=[1.]):
        super(_Residual, self).__init__()
        self._init_common(C_in, C_out, kernel_size, stride, dilation, groups, slimmable, width_mult_list)
        conv_stride = 1 if self._zoom else stride  # zoomed ops get their stride from the resize
        self.conv1 = _conv(slimmable, C_in, C_out, 3, conv_stride, dilation, dilation, groups, False, width_mult_list)
        self.bn1 = _norm(slimmable, C_out, width_mult_list)
        if self._n_convs == 2:
            self.conv2 = _conv(slimmable, C_out, C_out, 3, 1, dilation, dilation, groups, False, width_mult_list)
            self.bn2 = _norm(slimmable, C_out, width_mult_list)

    def _stages(self):
        stages = [(self.conv1, self.bn1)]
        if self._n_convs == 2:
            stages.append((self.conv2, self.bn2))
        return stages

    def set_ratio(self, ratio):
        self._set_pairs(ratio, self._stages())

    @classmethod
    def _flops(cls, h, w, C_in, C_out, kernel_size=3, stride=1, dilation=1, groups=1):
        assert stride in [1, 2]
        if cls._zoom:
            hh, ww, s = h // 2, w // 2, 1
        else:
            hh, ww, s = h, w, stride
        total = _conv_macs(hh, ww, C_in, C_out, 3, s) + 2 * (hh // s) * (ww // s) * C_out
        if cls._n_convs == 2:
            total += _conv_macs(hh // s, ww // s, C_out, C_out, 3, 1) + 2 * (hh // s) * (ww // s) * C_out
        return total

    @classmethod
    def _latency(cls, h, w, C_in, C_out, kernel_size=3, stride=1, dilation=1, groups=1):
        assert stride in [1, 2]
        layer = cls(C_in, C_out, kernel_size, stride, dilation, groups, slimmable=False)
        return compute_latency(layer, (1, C_in, h, w))

    def latency_key(self, size):
        """(latency-table key, output size) of this op at the configured ratio for an input of `size` = (C, H, W)"""
        c_in, h_in, w_in = size
        c_out = self._active_io(c_in)
        h_out, w_out = self._out_hw(h_in, w_in)
        name = "%s_H%d_W%d_Cin%d_Cout%d_stride%d_dilation%d" % (self._table_prefix, h_in, w_in, c_in, c_out, self.stride,
                                                               self.dilation)
        return name, (c_out, h_out, w_out)

    def forward_latency(self, size):
        name, size_out = self.latency_key(size)
        c_in, h_in, w_in = size
        measure_cls = self._measure_classes[self._table_prefix]
        latency = _table_latency(name, lambda: measure_cls._latency(h_in, w_in, c_in, size_out[0], self.kernel_size, self.stride,
                                                                    self.dilation, self.groups))
        return latency, size_out

    def forward(self, x, out=None, out_half=None, x_half=None):
        """out_half (inference): a (N, C_out, Ho // 2, Wo // 2) buffer that also receives bilinear(y, (Ho // 2, Wo // 2)), from the
        kernel that writes y.  x_half (zoomed ops): bilinear(x, (H // 2, W // 2)) already computed, e.g. by x's producer."""
        stages = self._stages()
        if not self._zoom:
            for i, (conv, bn) in enumerate(stages):
                last = i == len(stages) - 1
                x = engine.conv_bn_act(x, conv, bn, relu=True, out=out if last else None, out_half=out_half if last else None)
            return x
        x = F_.to_nhwc_half(x)
        H, W = int(x.size(2)), int(x.size(3))
        from . import autograd as AG
        if AG.grad_mode(x, self.conv1.weight):
            assert out_half is None and x_half is None, "out_half / x_half are inference-only"
            y = AG.bilinear(x, (H // 2, W // 2))
            for i, (conv, bn) in enumerate(stages):
                last = i == len(stages) - 1
                y = engine.conv_bn_act(y, conv, bn, relu=(not last) or self.stride == 2)
            return AG.bilinear(y, (H, W), relu=True) if self.stride == 1 else y
        if x_half is not None:
            assert tuple(x_half.shape) == (x.shape[0], x.shape[1], H // 2, W // 2), (tuple(x_half.shape), tuple(x.shape))
            y = x_half
        else:
            y = F_.bilinear(x, (H // 2, W // 2))
        for i, (conv, bn) in enumerate(stages):
            last = i == len(stages) - 1
            # the final ReLU comes AFTER the upsample when stride == 1 (operations.py:273-276, 442-445)
            y = engine.conv_bn_act(y, conv, bn, relu=(not last) or self.stride == 2,
                                   out=out if (last and self.stride == 2) else None,
                                   out_half=out_half if (last and self.stride == 2) else None)
        if self.stride == 1:
            half = {} if out_half is None else {"out_half": out_half}
            y = F_.bilinear(y, (H, W), relu=True, out=out, **half)
        return y


class BasicResidual1x(_Residual):
    """conv3x3(stride) -> BN -> ReLU (reference: search/operations.py:131-200)."""
    _n_convs, _zoom, _table_prefix = 1, False, "BasicResidual1x"


class BasicResidual_downup_1x(_Residual):
    """bilinear /2 -> conv3x3 -> BN -> [bilinear back if stride 1] -> ReLU (reference: operations.py:203-277)."""
    _n_convs, _zoom, _table_prefix = 1, True, "BasicResidual_downup_1x"


class BasicResidual2x(_Residual):
    """two conv3x3 -> BN -> ReLU stages, first one strided (reference: operations.py:280-359)."""
    _n_convs, _zoom, _table_prefix = 2, False, "BasicResidual2x"


class BasicResidual_downup_2x(_Residual):
    """bilinear /2 -> (conv -> BN -> ReLU) -> conv -> BN -> [bilinear back] -> ReLU (reference: operations.py:362-446).
    NOTE: its latency-table keys use the "BasicResidual2x_" prefix, exactly like the reference (:426-431)."""
    _n_convs, _zoom, _table_prefix = 2, True, "BasicResidual2x"


class FactorizedReduce(_Primitive):
    """'skip': identity (stride 1, non-slimmable), 1x1 conv-BN-ReLU (stride 1, slimmable) or the two-phase stride-2
    reduction cat[conv1(x), conv2(x[:, :, 1:, 1:])] -> BN -> ReLU (reference: search/operations.py:449-534)."""

    def __init__(self, C_in, C_out, stride=1, slimmable=True, width_mult_list=[1.]):
        super(FactorizedReduce, self).__init__()
        assert stride in [1, 2]
        assert C_out % 2 == 0
        self.C_in, self.C_out, self.stride = C_in, C_out, stride
        self.slimmable, self.width_mult_list = slimmable, width_mult_list
        self.ratio = (1., 1.)
        if stride == 1 and slimmable:
            self.conv1 = USConv2d(C_in, C_out, 1, stride=1, padding=0, bias=False, width_mult_list=width_mult_list)
            self.bn = USBatchNorm2d(C_out, width_mult_list)
            self.relu = nn.ReLU(inplace=True)
        elif stride == 2:
            self.relu = nn.ReLU(inplace=True)
            self.conv1 = _conv(slimmable, C_in, C_out // 2, 1, 2, 0, 1, 1, False, width_mult_list)
            self.conv2 = _conv(slimmable, C_in, C_out // 2, 1, 2, 0, 1, 1, False, width_mult_list)
            self.bn = _norm(slimmable, C_out, width_mult_list)

    def set_ratio(self, ratio):
        assert len(ratio) == 2
        self.__dict__["ratio"] = ratio
        if self.stride == 1:
            self.conv1.set_ratio(ratio)
            self.bn.set_ratio(ratio[1])
        else:
            self.conv1.set_ratio(ratio)
            self.conv2.set_ratio(ratio)
            self.bn.set_ratio(ratio[1])

    @staticmethod
    def _flops(h, w, C_in, C_out, stride=1):
        if stride == 1:
            return 0
        return 2 * _conv_macs(h, w, C_in, C_out // 2, 1, 2) + 2 * (h // 2) * (w // 2) * C_out

    @staticmethod
    def _latency(h, w, C_in, C_out, stride=1):
        layer = FactorizedReduce(C_in, C_out, stride, slimmable=False)
        return compute_latency(layer, (1, C_in, h, w))

    def latency_key(self, size):
        """(latency-table key, output size) of this op at the configured ratio for an input of `size` = (C, H, W)"""
        c_in, h_in, w_in = size
        if self.slimmable:
            assert c_in == int(self.C_in * self.ratio[0])
            c_out = int(self.C_out * self.ratio[1])
        else:
            assert c_in == self.C_in
            c_out = self.C_out
        h_out, w_out = self._out_hw(h_in, w_in)
        name = "FactorizedReduce_H%d_W%d_Cin%d_Cout%d_stride%d" % (h_in, w_in, c_in, c_out, self.stride)
        return name, (c_out, h_out, w_out)

    def forward_latency(self, size):
        name, size_out = self.latency_key(size)
        c_in, h_in, w_in = size
        latency = _table_latency(name, lambda: FactorizedReduce._latency(h_in, w_in, c_in, size_out[0], self.stride))
        return latency, size_out

    def forward(self, x, out=None):
        if self.stride == 2:
            return _factorized_reduce_s2(self, x, out)
        if self.slimmable:
            return engine.conv_bn_act(x, self.conv1, self.bn, relu=True, out=out)
        if out is not None:
            return F_.copy_channels(F_.to_nhwc_half(x), out)
        return x


def _factorized_reduce_s2(op, x, out):
    """Both 1x1 stride-2 convs write their half of the channels of ONE buffer (the torch.cat at operations.py:523
    disappears); BN + ReLU run per half in the conv epilogues in eval mode, or over the joint buffer in train mode."""
    x = F_.to_nhwc_half(x)
    bn = engine.active_bn(op.bn)
    ci, co_half = engine.active_channels(op.conv1)
    engine.active_channels(op.conv2)
    N, _, H, W = x.shape
    assert H % 2 == 0 and W % 2 == 0, "FactorizedReduce needs even H, W (the reference's cat fails otherwise)"
    co = 2 * co_half
    from .autograd import grad_mode
    if isinstance(bn, engine.SelBN):   # width chosen on the device: both halves at their maximum width (autograd.FactorizedReduceSelFn)
        from .autograd import factorized_reduce_sel
        assert out is None
        return factorized_reduce_sel(op, x, bn, ci, co_half)
    if bn.training and grad_mode(x, op.conv1.weight):
        from .autograd import factorized_reduce_train
        return factorized_reduce_train(op, x, bn, ci, co_half, out)
    if out is None:
        out = F_.empty_nhwc(N, co, H // 2, W // 2, x.device)
    w1 = engine.packed_weight(op.conv1, ci, co_half)
    w2 = engine.packed_weight(op.conv2, ci, co_half)
    if not bn.training:
        scale, shift = engine.folded_bn(bn, co, None)
        F_.conv_fwd(x, w1, co_half, 1, 2, 0, scale[:co_half], shift[:co_half], relu=True, out=out[:, :co_half])
        F_.conv_fwd(x, w2, co_half, 1, 2, 0, scale[co_half:], shift[co_half:], relu=True, out=out[:, co_half:], off=(1, 1))
        return out
    # both halves write their columns of one statistics buffer ([rows, sum(co) | sumsq(co)], one row per spatial tile)
    stats = F_.conv_stats_buffer(x, co_half, 1, 2, 0, total_C=co)
    raw = F_.empty_nhwc(N, co, H // 2, W // 2, x.device, dtype=torch.float32)
    F_.conv_fwd(x, w1, co_half, 1, 2, 0, out=raw[:, :co_half], stats=stats, out_f32=True)
    F_.conv_fwd(x, w2, co_half, 1, 2, 0, out=raw[:, co_half:], off=(1, 1), stats=stats, stats_off=co_half, out_f32=True)
    stats = engine.dp_allreduce_stats(stats)
    count = N * (H // 2) * (W // 2) * engine.dp_world_size()
    scale, shift, _, _ = F_.bn_finalize(stats, count, bn.weight, bn.bias, bn.eps, 0.1 if bn.momentum is None else bn.momentum,
                                        bn.running_mean, bn.running_var)
    if bn.num_batches_tracked is not None:
        bn.num_batches_tracked += 1
    return F_.affine_act(raw, scale, shift, relu=True, out=out)


OPS = {
    'skip': lambda C_in, C_out, stride, slimmable, width_mult_list: FactorizedReduce(C_in, C_out, stride, slimmable, width_mult_list),
    'conv': lambda C_in, C_out, stride, slimmable, width_mult_list: BasicResidual1x(C_in, C_out, kernel_size=3, stride=stride, dilation=1, slimmable=slimmable, width_mult_list=width_mult_list),
    'conv_downup': lambda C_in, C_out, stride, slimmable, width_mult_list: BasicResidual_downup_1x(C_in, C_out, kernel_size=3, stride=stride, dilation=1, slimmable=slimmable, width_mult_list=width_mult_list),
    'conv_2x': lambda C_in, C_out, stride, slimmable, width_mult_list: BasicResidual2x(C_in, C_out, kernel_size=3, stride=stride, dilation=1, slimmable=slimmable, width_mult_list=width_mult_list),
    'conv_2x_downup': lambda C_in, C_out, stride, slimmable, width_mult_list: BasicResidual_downup_2x(C_in, C_out, kernel_size=3, stride=stride, dilation=1, slimmable=slimmable, width_mult_list=width_mult_list),
}
OPS_name = ["FactorizedReduce", "BasicResidual1x", "BasicResidual_downup_1x", "BasicResidual2x", "BasicResidual_downup_2x"]
OPS_Class = OrderedDict()
OPS_Class['skip'] = FactorizedReduce
OPS_Class['conv'] = BasicResidual1x
OPS_Class['conv_downup'] = BasicResidual_downup_1x
OPS_Class['conv_2x'] = BasicResidual2x
OPS_Class['conv_2x_downup'] = BasicResidual_downup_2x
# the reference measures a missing downup_2x table entry with BasicResidual2x._latency (operations.py:430)
OPS_Class_by_prefix = {"BasicResidual1x": BasicResidual1x, "BasicResidual_downup_1x": BasicResidual_downup_1x,
                       "BasicResidual2x": BasicResidual2x}
_Residual._measure_classes = OPS_Class_by_prefix   # a network variant with other operator classes measures with its own
