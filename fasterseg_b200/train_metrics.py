"""The drivers' per-step training mIoU on the device (train/seg_metrics.py:11-14 `Seg_Metrics.update`, train/train.py:262-263).

The reference's `batch_intersection_union` (train/seg_metrics.py:43-69) takes `torch.max` over the label-resolution logits, copies
the argmax and the target (two int64 maps) to the host and builds three numpy histograms.  For LazyLogits on the target's CUDA
device, `install` replaces that with one upsample + argmax + confusion-matrix launch (K9c, `ConfusionMatrix.update_from_logits`)
and a copy of its n_cl^2 + 2 counters; the caller's `get_scores()` needs the value on the host anyway.

Why the counters give the reference's numbers exactly: `np.histogram(v, bins=n, range=(1, n))` puts the integer k + 1 into bin k
for every 0 <= k < n and drops 0 and everything above n; the reference's target mask 1 <= target + 1 <= n is K9c's 0 <= gt < n_cl.
So area_inter, area_pred and area_lab are the diagonal, the column sums and the row sums of K9c's matrix (row = ground truth),
and area_union = area_pred + area_lab - area_inter.  tests/golden/seg_metrics.json pins this against the reference's code."""
import numpy as np
import torch

from .losses import LazyLogits
from .metric import ConfusionMatrix


def inter_union(hist):
    """(area_inter, area_union) of batch_intersection_union from an n_cl x n_cl confusion matrix (row = ground truth)"""
    hist = np.asarray(hist, dtype=np.int64)
    inter = np.diag(hist).copy()
    return inter, hist.sum(0) + hist.sum(1) - inter


def eligible(metrics, pred, target):
    """the device path: lazy logits of n_classes channels and a label-resolution integer target on the logits' CUDA device"""
    if not isinstance(pred, LazyLogits) or not isinstance(target, torch.Tensor):
        return False
    x = pred.lowres
    return (_on_device(x, target) and target.dtype in (torch.uint8, torch.int32, torch.int64)
            and int(x.shape[1]) == int(metrics.n_classes) and tuple(target.shape) == (int(x.shape[0]),) + pred.size)


def _on_device(x, target):
    return x.is_cuda and target.device == x.device


def install(seg_metrics):
    """Patch the driver's Seg_Metrics.update in place (get_scores and reset stay the reference's).  Idempotent; returns the
    class."""
    cls = seg_metrics.Seg_Metrics
    if getattr(cls.update, "_fsb_original", None) is not None:
        return cls
    original = cls.update

    def update(self, pred, target):
        if not eligible(self, pred, target):
            return original(self, pred, target)
        cm = ConfusionMatrix(self.n_classes, device=target.device)
        cm.update_from_logits(pred.lowres, pred.size, target)
        inter, union = inter_union(cm.result()[0])
        self.total_inter += inter
        self.total_union += union

    update._fsb_original = original
    update.__name__ = "update"
    cls.update = update
    return cls
