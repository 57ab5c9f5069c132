"""Validation on the device behind the reference's `Evaluator` (tools/engine/evaluator.py), for the drivers that run it unmodified
(train/train.py:274-281, search/train_search.py:259-271).

The reference normalises every validation image on the host, copies the fp32 frame to the GPU, copies the full-resolution score map
(19 x 1024 x 2048 fp32 = 159 MB) back, takes the argmax and builds the confusion matrix with numpy, in 3 spawned processes that
each receive a pickled copy of the CUDA model.  `install(module)` patches `Evaluator.run_online` and `run_online_multiprocess` in
place; for the evaluations the device path covers (`eligible`) they instead

  * read `dataset[idx]` through a DataLoader with host workers (the uint8 HWC image and uint8 label, copied into pinned memory),
  * run the network on the uint8 image with the normalisation folded into the stem (`set_input_normalization`), and add each
    image's hist_info on the device (`accumulate_confusion`: one kernel after the forward, no label map),
  * copy the n_cl^2 + 2 counters to the host once and hand them to the driver's own `compute_metric`, which prints and returns
    the result line and mIoU as before.

Everything runs in the driver's process.  The forwards of a supernet in 'arch_ratio' mode draw widths from torch's generator
('random' from numpy's); in the reference those draws happen in the spawned children, so the driver's own RNG streams -- which the
training that follows consumes -- do not move.  The device path therefore runs under `torch.random.fork_rng` with numpy's state
saved and restored.  Any other evaluation (several scales, flipping, saving or showing predictions, a tensorboard logger, a network
that is not ours or not on CUDA) calls the reference's method unchanged."""
import numpy as np
import torch

from . import metric
from .model_search import Network_Multi_Path
from .model_seg import Network_Multi_Path_Infer

PATCHED = ("run_online", "run_online_multiprocess")


def _on_cuda(net):
    p = next(iter(net.parameters()), None)
    return p is not None and p.is_cuda


def eligible(ev):
    """True when `ev` (an Evaluator) evaluates what the device path computes: one of our networks on CUDA, a single scale without
    flipping, and nothing saved, shown or logged per image"""
    net = getattr(ev, "network", None)
    return (isinstance(net, (Network_Multi_Path_Infer, Network_Multi_Path)) and _on_cuda(net)
            and len(ev.multi_scales) == 1 and not ev.is_flip
            and ev.save_path is None and not ev.show_image and not ev.show_prediction and ev.logger is None)


def image(d):
    """a dataset item's uint8 image as a contiguous H x W x 3 tensor (the dataset hands out a BGR->RGB flipped view)"""
    img = d["data"]
    if img.shape[2] < 3:                      # gray images, as process_image (tools/engine/evaluator.py:319-326) treats them
        img = np.concatenate((img, img, img), axis=2)
    if img.dtype != np.uint8:
        raise TypeError("device evaluation expects the dataset's uint8 image, got %s" % img.dtype)
    return torch.from_numpy(np.ascontiguousarray(img))


def _collate(batch):
    """dataset items -> (uint8 image N x H x W x 3, label N x H x W), contiguous"""
    imgs, labels = [], []
    for d in batch:
        lab = np.asarray(d["label"])
        if lab.dtype not in (np.uint8, np.int32, np.int64):
            lab = lab.astype(np.int64)
        imgs.append(image(d))
        labels.append(torch.from_numpy(np.ascontiguousarray(lab)))
    return torch.stack(imgs), torch.stack(labels)


def loader(ev, collate_fn=_collate):
    """DataLoader over the evaluator's dataset in index order, images decoded by `ev.threds` host workers into pinned memory"""
    n = ev.ndata
    workers = max(0, min(int(ev.threds or 0), n))
    return torch.utils.data.DataLoader(ev.dataset, batch_size=1, sampler=list(range(n)), num_workers=workers, collate_fn=collate_fn,
                                       pin_memory=True)


def evaluate(ev):
    """The device path: -> ev.compute_metric([{'hist', 'labeled', 'correct'}]) = (result_line, mIoU)"""
    net = ev.network
    dev = next(net.parameters()).device
    dev_index = dev.index if dev.index is not None else torch.cuda.current_device()
    supernet = isinstance(net, Network_Multi_Path)
    modes = [(m, m.training) for m in net.modules()]
    np_state = np.random.get_state()
    try:
        with torch.cuda.device(dev), torch.random.fork_rng(devices=[dev_index]), torch.no_grad():
            net.eval()
            net.set_input_normalization(ev.image_mean, ev.image_std)
            cm = metric.ConfusionMatrix(ev.class_num, device=dev)
            for img, label in loader(ev):
                x = img.to(dev, non_blocking=True).permute(0, 3, 1, 2)
                gt = label.to(dev, non_blocking=True)
                if supernet:
                    net.accumulate_confusion(x, gt, cm, head=ev.out_idx)
                else:
                    net.accumulate_confusion(x, gt, cm)
            hist, labeled, correct = cm.result()
    finally:
        np.random.set_state(np_state)
        for m, training in modes:
            m.training = training
    return ev.compute_metric([{"hist": hist, "labeled": labeled, "correct": correct}])


def _device_or(name, orig):
    def method(self):
        if eligible(self):
            self.val_func = self.network
            return evaluate(self)
        return orig(self)
    method.__name__ = name
    method.__doc__ = orig.__doc__
    method._fsb_original = orig
    return method


def install(module):
    """Patch `module.Evaluator` (tools/engine/evaluator.py) in place; idempotent"""
    cls = module.Evaluator
    for name in PATCHED:
        orig = getattr(cls, name)
        if getattr(orig, "_fsb_original", None) is None:
            setattr(cls, name, _device_or(name, orig))
    return cls
