"""The primitives of the reference's latency/ deployment network -- drop-in for latency/operations.py.

Same class names, constructor signatures, `__all__`, `OPS / OPS_name / OPS_Class`, `forward_latency` keys and parameter names
as the train/ primitives (fasterseg_b200/operations.py), with the two differences of latency/operations.py:
  - the zoomed primitives resize with mode='nearest' (:265,269,427,434) instead of bilinear align_corners=True;
  - a non-slimmable stride-2 FactorizedReduce is ONE 1x1 stride-2 conv C_in -> C_out (:461-463,513-514): state_dict
    `conv1.weight [C_out, C_in, 1, 1]`, `bn.*`, no `conv2`.
On even maps the nearest /2 and x2 are no kernels at all: the conv reads the even pixels of the full map through its input
tensor map (FSB_CONV_X_DOWN2) and stores every output pixel to its 2x2 block through four lattice output maps
(FSB_CONV_Y_UP2).  `resize_fold` decides from the shapes; other sizes run the standalone nearest kernel.

Inference only: the reference's latency/ tree has no training driver.  A training-mode or grad-mode forward raises.
"""
__all__ = ['ConvNorm', 'BasicResidual1x', 'BasicResidual_downup_1x', 'BasicResidual2x', 'BasicResidual_downup_2x',
           'FactorizedReduce', 'OPS', 'OPS_name', 'OPS_Class']

from collections import OrderedDict

import torch.nn as nn

from .. import engine
from .. import functional as F_
from .. import operations as _train
from ..operations import (BasicResidual1x, BasicResidual2x, BatchNorm2d, ConvNorm, compute_latency,  # noqa: F401
                          latency_lookup_table, table_file_name)


def resize_fold(src_hw, dst_hw):
    """How a nearest resize src_hw -> dst_hw runs: "down2" (exactly half: folded into the consumer conv's input map), "up2"
    (exactly twice: folded into the producer conv's output maps) or None (the standalone fsb_nearest_fwd kernel)."""
    (hs, ws), (hd, wd) = (int(v) for v in src_hw), (int(v) for v in dst_hw)
    if 2 * hd == hs and 2 * wd == ws:
        return "down2"
    if hd == 2 * hs and wd == 2 * ws:
        return "up2"
    return None


def inference_only(what, training, *tensors):
    """raise unless this is an eval-mode forward without autograd recording"""
    from .. import autograd as AG
    if training or AG.grad_mode(*tensors):
        raise NotImplementedError(
            "%s: the latency/ network variant is inference only (eval mode, under torch.no_grad()); the reference's latency/ "
            "tree has no training driver -- train the train/ variant" % what)


def conv_bn_act_nearest(x, conv, bn, relu, out=None, down2=False, up2=False):
    """eval-mode act(BN(conv(x))) with the nearest /2 of its input and / or the nearest x2 of its output folded in"""
    ci, co = engine.active_channels(conv)
    k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
    scale, shift = engine.folded_bn(engine.active_bn(bn), co, conv.bias)
    return F_.conv_fwd(x, engine.packed_weight(conv, ci, co), co, k, s, p, scale, shift, relu=relu, out=out, down2=down2, up2=up2)


class _NearestZoom:
    """forward of the zoomed primitives: nearest /2 -> conv stages -> [nearest back if stride 1] -> ReLU.  The ReLU after the
    upsample runs in the last conv's epilogue (a copy commutes with it)."""

    def forward(self, x, out=None):
        stages = self._stages()
        inference_only(type(self).__name__, any(bn.training for _, bn in stages), x, self.conv1.weight)
        x = F_.to_nhwc_half(x)
        H, W = int(x.size(2)), int(x.size(3))
        half = (H // 2, W // 2)
        down2 = resize_fold((H, W), half) == "down2"
        y = x if down2 else F_.nearest(x, half)
        for i, (conv, bn) in enumerate(stages):
            last = i == len(stages) - 1
            if not last:
                y = conv_bn_act_nearest(y, conv, bn, True, down2=down2 and i == 0)
                continue
            if self.stride == 2:
                return conv_bn_act_nearest(y, conv, bn, True, out=out, down2=down2 and i == 0)
            up2 = resize_fold(half, (H, W)) == "up2"
            if up2:
                return conv_bn_act_nearest(y, conv, bn, True, out=out, down2=down2 and i == 0, up2=True)
            y = conv_bn_act_nearest(y, conv, bn, True, down2=down2 and i == 0)
            return F_.nearest(y, (H, W), out=out)


class BasicResidual_downup_1x(_NearestZoom, _train.BasicResidual_downup_1x):
    """nearest /2 -> conv3x3 -> BN -> [nearest back if stride 1] -> ReLU (reference: latency/operations.py:203-271)."""


class BasicResidual_downup_2x(_NearestZoom, _train.BasicResidual_downup_2x):
    """nearest /2 -> (conv -> BN -> ReLU) -> conv -> BN -> [nearest back] -> ReLU (reference: latency/operations.py:362-436).
    Its latency-table keys use the "BasicResidual2x_" prefix, like the reference."""


class FactorizedReduce(_train.FactorizedReduce):
    """'skip' of the latency/ network: identity / 1x1 conv-BN-ReLU at stride 1 as in train/; at stride 2 the non-slimmable op is
    a single 1x1 stride-2 conv -> BN -> ReLU (reference: latency/operations.py:449-520; TensorRT rejected the x[:, :, 1:, 1:]
    slice of the two-conv form)."""

    def __init__(self, C_in, C_out, stride=1, slimmable=True, width_mult_list=[1.]):
        if stride != 2 or slimmable:
            super(FactorizedReduce, self).__init__(C_in, C_out, stride, slimmable, width_mult_list)
            return
        nn.Module.__init__(self)
        assert C_out % 2 == 0
        self.C_in, self.C_out, self.stride = C_in, C_out, stride
        self.slimmable, self.width_mult_list = slimmable, width_mult_list
        self.ratio = (1., 1.)
        self.relu = nn.ReLU(inplace=True)
        self.conv1 = nn.Conv2d(C_in, C_out, 1, stride=2, padding=0, bias=False)
        self.bn = nn.BatchNorm2d(C_out)

    @staticmethod
    def _latency(h, w, C_in, C_out, stride=1):
        layer = FactorizedReduce(C_in, C_out, stride, slimmable=False)
        return compute_latency(layer, (1, C_in, h, w))

    def forward(self, x, out=None):
        if self.stride == 2 and not self.slimmable:
            inference_only("FactorizedReduce", self.bn.training, x, self.conv1.weight)
            return conv_bn_act_nearest(F_.to_nhwc_half(x), self.conv1, self.bn, True, out=out)
        return super(FactorizedReduce, self).forward(x, out=out)


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
# a missing table entry is measured with this module's operators (downup_2x with BasicResidual2x, like the reference)
OPS_Class_by_prefix = {"BasicResidual1x": BasicResidual1x, "BasicResidual_downup_1x": BasicResidual_downup_1x,
                       "BasicResidual2x": BasicResidual2x}
BasicResidual_downup_1x._measure_classes = OPS_Class_by_prefix
BasicResidual_downup_2x._measure_classes = OPS_Class_by_prefix
