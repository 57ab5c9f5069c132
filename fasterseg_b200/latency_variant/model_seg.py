"""The derived network of the reference's latency/ tree -- drop-in for latency/model_seg.py (what latency/run_latency.py builds and
times, and what the paper's FPS was measured on).

Same public surface and state_dict as fasterseg_b200/model_seg.py, built from this package's operators
(latency_variant/operations.py), with the resizes of latency/model_seg.py:
  - the x2 of the arm / refine tails is sized as twice the coarse map (:305,309,315); the arm conv stores straight into its
    channel slice of the concat buffer at twice its size (FSB_CONV_Y_UP2), so no resize kernel runs;
  - the final x8 is nearest (:362): `forward` returns nearest logits, `predict_labels` the fused nearest upsample + argmax.
Inference only (eval mode under torch.no_grad()); everything else -- streams, CUDA graphs (runtime.GraphedInference,
InferencePipeline), the uint8 stem of `set_input_normalization`, `forward_latency` -- is the train/ network's.
"""
import torch
import torch.nn as nn

from .. import functional as F_
from .. import model_seg as _train
from ..decode import (alphas2ops_path_width, betas2path, downs2path, network_metas, path2downs, path2widths,  # noqa: F401
                      softmax)
from ..genotypes import PRIMITIVES
from .operations import *  # noqa: F401,F403  (the reference does `from operations import *`)
from .operations import OPS, conv_bn_act_nearest, inference_only, resize_fold

BatchNorm2d = nn.BatchNorm2d


class MixedOp(_train.MixedOp):
    """Single selected primitive (non-slimmable, fixed channels) of the latency/ operator set."""

    def __init__(self, C_in, C_out, op_idx, stride=1):
        nn.Module.__init__(self)
        self._op = OPS[PRIMITIVES[op_idx]](C_in, C_out, stride, slimmable=False, width_mult_list=[1.])


class Cell(_train.Cell):
    def __init__(self, op_idx, C_in, C_out, down):
        nn.Module.__init__(self)
        self._C_in, self._C_out, self._down = C_in, C_out, down
        self._op = MixedOp(C_in, C_out, op_idx, stride=2 if down else 1)


class Network_Multi_Path_Infer(_train.Network_Multi_Path_Infer):
    _cell_cls = Cell
    fuse_resizes = False   # nearest resizes, folded into the convs' tensor maps instead

    def _inference_only(self, input):
        inference_only("Network_Multi_Path_Infer", self.training, input, next(self.parameters(), None))

    def _arm_refine(self, arm, refine, coarse, skip, out=None):
        """arm 1x1 -> nearest x2 -> cat([up, skip]) -> refine 3x3 (latency/model_seg.py:304-319); the arm conv writes its x2
        output into the first channels of the concat buffer."""
        coarse = F_.to_nhwc_half(coarse)
        N, Hc, Wc = coarse.shape[0], coarse.shape[2], coarse.shape[3]
        c_skip, Hs, Ws = skip.shape[1], skip.shape[2], skip.shape[3]
        assert (Hs, Ws) == (2 * Hc, 2 * Wc), (
            "latency/ network: the skip feature is %dx%d but the upsampled arm output is %dx%d -- the reference's torch.cat fails "
            "here (latency/model_seg.py:305-319); use input sizes divisible by 32" % (Hs, Ws, 2 * Hc, 2 * Wc))
        conv, bn = arm.conv[0], arm.conv[1]
        c_up = conv.out_channels
        cat = F_.empty_nhwc(N, c_up + c_skip, Hs, Ws, coarse.device)
        if resize_fold((Hc, Wc), (Hs, Ws)) == "up2":
            conv_bn_act_nearest(coarse, conv, bn, True, out=cat[:, :c_up], up2=True)
        else:
            F_.nearest(arm(coarse), (Hs, Ws), out=cat[:, :c_up])
        F_.copy_channels(F_.to_nhwc_half(skip), cat[:, c_up:])
        return refine(cat, out=out)

    def forward(self, input):
        self._inference_only(input)
        if self.__dict__.get("lazy_logits", False):
            raise NotImplementedError("latency/ network variant: lazy_logits serves the training criteria (bilinear); not available")
        pred8 = self._features(input)
        size = (int(pred8.size(2)) * 8, int(pred8.size(3)) * 8)
        return F_.upsample_logits_nearest(pred8, size, dtype=self.logits_dtype)

    @torch.no_grad()
    def predict_labels(self, input, out=None):
        """argmax(forward(input), dim=1) as uint8 from the fused nearest upsample + argmax"""
        self._inference_only(input)
        pred8 = self._features(input)
        return F_.upsample_argmax_nearest(pred8, (int(pred8.size(2)) * 8, int(pred8.size(3)) * 8), out=out)

    @torch.no_grad()
    def accumulate_confusion(self, input, gt, cm):
        """hist_info of predict_labels(input) against `gt` into `cm` (metric.ConfusionMatrix); the fused kernel of the train/
        network is bilinear, so the nearest labels go through the label map"""
        cm.update(self.predict_labels(input), gt)
