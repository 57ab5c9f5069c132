"""The drivers' training augmentation on the device, behind the reference's own DataLoader (train/dataloader.py:8-31,
search/dataloader.py: `TrainPre` and `get_train_loader`).

The reference's DataLoader workers decode each PNG and then run `TrainPre` on the host: random mirror, a cv2.resize of the
whole image by the random scale, normalisation of the whole scaled image in float64, crop / pad, the label's nearest resizes,
and the conversion to fp32 / int64 tensors.  `install(module)` wraps the module's `get_train_loader`; for a loader that
`eligible` accepts:

  * worker side: the dataset's `TrainPre` is replaced by `DeviceTrainPre`, which makes the reference's random draws in the
    reference's order (`draw`) and hands back the uint8 source, the uint8 label and the drawn geometry.  Those travel in the
    dataset's `extra_dict` under keys that contain neither 'img' nor 'label', so `BaseDataset.__getitem__`
    (tools/datasets/BaseDataset.py:47-56) passes them through unconverted; `collate` packs a batch's sources back to back and
    the DataLoader pins them;
  * main-process side: each batch the driver takes (`next()` / `.next()`) copies the pinned sources to the current device and
    runs `fsb_train_pre` (csrc/trainpre.cu) on the current stream.  `data` and `label` become the device tensors, bit-identical
    to the reference's; `fn` and `n` are untouched, and the driver's `.cuda(non_blocking=True)` is then a no-op.

Python's `random` is consumed exactly as the reference consumes it, so every later draw of a worker matches too.  Any other loader
(another preprocess, a custom collate, a dataset whose `__getitem__` is not the one of the reference's tools/datasets/BaseDataset.py)
and any host without CUDA keep the reference path."""
import os
import random
import sys

import numpy as np
import torch
from torch.utils.data import default_collate

from . import functional

SRC_KEY, GT_KEY, GEOM_KEY = "tp_src", "tp_gt", "tp_geom"   # extra_dict keys: no 'img' / 'label' in them (BaseDataset.py:50-56)
BATCH_KEY = "_fsb_trainpre"
RECORD = 11   # worker record: H, W, mirror, sh, sw, pos_h, pos_w, crop_h, crop_w, label_h, label_w


def draw(h, w, config):
    """The random draws of TrainPre.__call__ for an h x w source, in the reference's order: random_mirror's `random.random()`
    (tools/utils/img_utils.py:126), random_scale's `random.choice` (:106) and generate_random_crop_pos's `random.randint`s
    (:42-57).  -> (mirror, sh, sw, pos_h, pos_w)"""
    mirror = int(random.random() >= 0.5)
    sh, sw = h, w
    if config.train_scale_array is not None:
        scale = random.choice(config.train_scale_array)
        sh, sw = int(h * scale), int(w * scale)
    crop_h, crop_w = int(config.image_height), int(config.image_width)
    pos_h = random.randint(0, sh - crop_h + 1) if sh > crop_h else 0
    pos_w = random.randint(0, sw - crop_w + 1) if sw > crop_w else 0
    return mirror, sh, sw, pos_h, pos_w


def label_size(config):
    """(h, w) of the label map: the crop resized by gt_down_sampling (train/dataloader.py:25)"""
    g = config.gt_down_sampling
    return int(config.image_height) // g, int(config.image_width) // g


def normalization_lut(mean, std):
    """float32 [3, 256]: normalize (tools/utils/img_utils.py:179-184) of every uint8 value -- float32(v) / 255.0 in float32, then
    `- mean` and `/ std` in float64 -- rounded to float32 like the dataset's `.float()`; the same expression elementwise, so exact"""
    v = np.arange(256, dtype=np.uint8).astype(np.float32) / 255.0
    t = (v[:, None] - np.asarray(mean)) / np.asarray(std)
    return torch.from_numpy(np.ascontiguousarray(t.T)).float()


class DeviceTrainPre:
    """Worker-side drop-in for the reference's TrainPre: the draws only; the pixels are left to the device"""

    def __init__(self, pre):
        self.config, self.img_mean, self.img_std = pre.config, pre.img_mean, pre.img_std

    def __call__(self, img, gt):
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3 or gt.dtype != np.uint8 or gt.shape != img.shape[:2]:
            raise TypeError("device training augmentation expects a uint8 H x W x 3 image and a uint8 H x W label, got %s %s / %s %s"
                            % (img.dtype, img.shape, gt.dtype, gt.shape))
        h, w = img.shape[:2]
        record = np.array((h, w) + draw(h, w, self.config) + (int(self.config.image_height), int(self.config.image_width))
                          + label_size(self.config), dtype=np.int32)
        return np.zeros(0, np.float32), np.zeros(0, np.uint8), {SRC_KEY: img, GT_KEY: gt, GEOM_KEY: record}


def check_geometry(records):
    """worker records int32 [N, RECORD] -> (kernel geometry int32 [N, 8] with the packed pixel offsets, (crop_h, crop_w, label_h,
    label_w)).  Raises ValueError for a record the kernel must not be given."""
    r = np.asarray(records, dtype=np.int64).reshape(-1, RECORD)
    H, W, mirror, sh, sw, ph, pw = (r[:, i] for i in range(7))
    sizes = r[:, 7:]
    if (sizes != sizes[0]).any():
        raise ValueError("train_pre: every image of a batch needs the same crop and label size")
    ch, cw, lh, lw = (int(v) for v in sizes[0])
    if not (0 < lh <= ch and 0 < lw <= cw):
        raise ValueError("train_pre: bad crop / label size %s" % (sizes[0].tolist(),))
    ok = (H > 0) & (W > 0) & (sh > 0) & (sw > 0) & ((mirror == 0) | (mirror == 1)) & (ph >= 0) & (ph < sh) & (pw >= 0) & (pw < sw)
    if not ok.all():
        raise ValueError("train_pre: bad geometry record(s) %s" % r[~ok].tolist())
    pixels = H * W
    offsets = np.concatenate(([0], np.cumsum(pixels)[:-1]))
    if int(pixels.sum()) * 3 >= 2 ** 31:
        raise ValueError("train_pre: a batch's sources must stay below 2^31 bytes")
    geom = np.stack([H, W, mirror, sh, sw, ph, pw, offsets], axis=1).astype(np.int32)
    return torch.from_numpy(geom), (ch, cw, lh, lw)


def _cat(tensors):
    """the tensors flattened back to back; in a worker straight into shared memory, as default_collate stacks"""
    flat = [t.reshape(-1) for t in tensors]
    out = None
    if torch.utils.data.get_worker_info() is not None:
        n = sum(t.numel() for t in flat)
        out = flat[0].new(flat[0]._typed_storage()._new_shared(n, device=flat[0].device)).resize_(n)
    return torch.cat(flat, out=out)


def collate(batch):
    """DataLoader collate_fn of a patched loader: default_collate of the dataset's own keys (the placeholders, `fn`, `n`), and the
    packed sources, labels and geometry under BATCH_KEY"""
    srcs = [d.pop(SRC_KEY) for d in batch]
    gts = [d.pop(GT_KEY) for d in batch]
    geom, size = check_geometry(np.stack([np.asarray(d.pop(GEOM_KEY)) for d in batch]))
    out = default_collate(batch)
    out[BATCH_KEY] = {"src": _cat(srcs), "gt": _cat(gts), "geom": geom, "size": torch.tensor(size, dtype=torch.int32)}
    return out


def _device():
    return torch.device("cuda", torch.cuda.current_device())


class DeviceTrainLoader:
    """What the wrapped get_train_loader returns: the reference's DataLoader (every attribute is its), whose iterators hand out
    batches with `data` / `label` already computed on the current CUDA device"""

    def __init__(self, loader, mean, std):
        self.loader = loader
        self.lut_host = normalization_lut(mean, std)
        self._luts = {}

    def __getattr__(self, name):
        return getattr(self.__dict__["loader"], name)

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        return DeviceBatches(self, iter(self.loader))

    def to_device(self, batch):
        """a collated batch -> the same dict with `data` / `label` computed on the current device and BATCH_KEY dropped"""
        p = batch.pop(BATCH_KEY)
        dev = _device()
        if dev not in self._luts:
            self._luts[dev] = self.lut_host.to(dev)
        # The sources are in pinned memory (pin_memory=True); a non_blocking copy from it records an event with torch's host
        # allocator, which keeps the block from being reused until the copy has completed, even after `p` is dropped.
        src = p["src"].to(dev, non_blocking=True)
        gt = p["gt"].to(dev, non_blocking=True)
        geom = p["geom"].to(dev, non_blocking=True)
        ch, cw, lh, lw = (int(v) for v in p["size"])
        batch["data"], batch["label"] = functional.train_pre(src, gt, geom, self._luts[dev], (ch, cw), (lh, lw))
        return batch


class DeviceBatches:
    """iterator of a DeviceTrainLoader (`next()` is the spelling train.py:237 / train_search.py:226,235 use)"""

    def __init__(self, owner, it):
        self.owner, self.it = owner, it

    def __iter__(self):
        return self

    def __len__(self):
        return len(self.it)

    def __next__(self):
        return self.owner.to_device(next(self.it))

    next = __next__


def _getitem_owner(dataset):
    for cls in type(dataset).__mro__:
        if "__getitem__" in vars(cls):
            return cls
    return None


def _defined_in(cls, path):
    """True when `cls` is a class named BaseDataset defined in the file `path`"""
    mod = sys.modules.get(getattr(cls, "__module__", None) or "")
    f = getattr(mod, "__file__", None)
    return (path is not None and f is not None and getattr(cls, "__name__", None) == "BaseDataset"
            and os.path.realpath(f) == os.path.realpath(path))


def eligible(loader, trainpre_cls, base_dataset_file):
    """True when the device path computes what `loader` yields: CUDA is available, the dataset's preprocess is exactly the
    reference's TrainPre (`trainpre_cls`), its items come from the reference's BaseDataset.__getitem__ (defined in
    `base_dataset_file`; it passes extra_dict through), and the loader collates with default_collate"""
    ds = getattr(loader, "dataset", None)
    return (torch.cuda.is_available() and type(getattr(ds, "preprocess", None)) is trainpre_cls
            and _defined_in(_getitem_owner(ds), base_dataset_file) and getattr(loader, "collate_fn", None) is default_collate)


def wrap_loader(loader, trainpre_cls, base_dataset_file):
    """-> a DeviceTrainLoader over `loader` (its dataset's preprocess and its collate_fn replaced), or `loader` unchanged"""
    if not eligible(loader, trainpre_cls, base_dataset_file):
        return loader
    pre = loader.dataset.preprocess
    loader.dataset.preprocess = DeviceTrainPre(pre)
    loader.collate_fn = collate
    return DeviceTrainLoader(loader, pre.img_mean, pre.img_std)


def reference_base_dataset(module):
    """<FasterSeg>/tools/datasets/BaseDataset.py for the dataloader module <FasterSeg>/<dir>/dataloader.py, or None"""
    f = getattr(module, "__file__", None)
    return None if f is None else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(f))), "tools", "datasets",
                                                "BaseDataset.py")


def install(module):
    """Wrap `module.get_train_loader` (train/dataloader.py:34, search/dataloader.py:34) in place; idempotent"""
    orig = module.get_train_loader
    if getattr(orig, "_fsb_original", None) is not None:
        return module
    base = reference_base_dataset(module)

    def get_train_loader(*a, **k):
        return wrap_loader(orig(*a, **k), module.TrainPre, base)

    get_train_loader.__doc__ = orig.__doc__
    get_train_loader._fsb_original = orig
    module.get_train_loader = get_train_loader
    return module
