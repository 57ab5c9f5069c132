"""Evaluator metrics on the device ("next" row N4; tools/seg_opr/metric.py:7-24, tools/engine/evaluator.py:206-225).

The reference pulls the full-resolution score map to the host for every image (19 x H x W fp32 = 159 MB at 1024 x 2048), takes
the argmax there and builds the confusion matrix with numpy.  Here the label map never leaves the GPU: the fused upsample+argmax
kernel produces uint8 labels, `ConfusionMatrix.update` accumulates hist_info with integer atomics (exact, order-independent), and
only the n_cl x n_cl matrix crosses PCIe once at the end."""
import numpy as np
import torch

from . import functional as F_


class ConfusionMatrix:
    def __init__(self, n_cl, device="cuda"):
        self.n_cl = int(n_cl)
        self.acc = torch.zeros(self.n_cl * self.n_cl + 2, device=device, dtype=torch.int64)

    def update(self, pred_u8, gt):
        """pred_u8: uint8 label map(s); gt: same number of elements, uint8 / int32 / int64 (255 or negative = ignore)"""
        F_.confusion_matrix(pred_u8.contiguous(), gt.contiguous(), self.n_cl, out=self.acc)

    def update_from_logits(self, logits, size, gt):
        """accumulate hist_info of argmax(upsample(logits, size)) vs gt in one kernel, without a label map: `logits` are the
        low-resolution NHWC fp16 class scores (n_cl channels), bilinear align_corners=True to `size` = gt's (H, W)"""
        F_.upsample_argmax_confusion(logits, size, gt.contiguous(), self.n_cl, self.acc)

    def result(self):
        """-> (hist [n_cl, n_cl] int64, labeled, correct) like metric.hist_info summed over the images seen"""
        a = self.acc.cpu().numpy()
        n = self.n_cl * self.n_cl
        return a[:n].reshape(self.n_cl, self.n_cl).copy(), int(a[n]), int(a[n + 1])


def hist_info(n_cl, pred, gt):
    """drop-in for tools/seg_opr/metric.py:7-15 on device tensors (returns numpy like the reference)"""
    cm = ConfusionMatrix(n_cl, device=pred.device)
    cm.update(pred.to(torch.uint8), gt)
    return cm.result()


def compute_score(hist, correct, labeled):
    """tools/seg_opr/metric.py:18-27"""
    with np.errstate(divide="ignore", invalid="ignore"):
        hist = hist.astype(np.float64)
        iu = np.diag(hist) / (hist.sum(1) + hist.sum(0) - np.diag(hist))
        return iu, np.nanmean(iu), np.nanmean(iu[1:]), correct / labeled
