"""Test-set prediction on the device behind the reference's `Tester` (tools/engine/tester.py), for train/train.py's `test()`
(train/train.py:283-291), which writes the Cityscapes submission files when `config.is_test` is set.

Per image the reference normalises on the host, runs the fp32 frame, copies the 19 x H x W fp32 `exp` of the logits back, takes
the argmax with numpy, remaps trainId -> Cityscapes id with a Python loop over every pixel (train/test.py:66-68), optionally
builds the colour map with one `np.where` pass per class (tools/utils/visualize.py:6-21), and writes both with `cv2.imwrite`.
`install(module)` patches `Tester.run_online` and `run_online_multiprocess` in place; for the testers the device path covers
(`eligible`) they instead

  * read `dataset[idx]` through the evaluator's DataLoader (host workers, pinned memory), ignoring the test split's dummy labels,
  * run the network on the uint8 image with the normalisation folded into the stem, and produce both uint8 images in one kernel
    after the forward (`predict_label_maps`: the trainId -> id table and the colour table in shared memory),
  * copy them into a ring of pinned host buffers and hand them to a thread pool that calls `cv2.imwrite` on the reference's paths.

The id table is the one the driver's own `func_per_iteration` reads (its module's `cityscapes_trainID2id`), the colours those of
`dataset.get_class_colors()` with `set_img_color`'s rule for `config.background`.  The files are byte-identical to the
reference's wherever the labels agree.  Every write has finished when the method returns (train.py moves the directory on the next
line).  Any other tester -- another `func_per_iteration`, several scales, flipping, a network that is not ours or not on the
device `devices[0]` names, an id table or colour list whose values `imwrite` would not store as given -- runs the reference's
method unchanged."""
import numbers
import os
from concurrent.futures import ThreadPoolExecutor

import torch

from . import evaluator
from .model_seg import Network_Multi_Path_Infer

PATCHED = ("run_online", "run_online_multiprocess")
ID_TABLE = "cityscapes_trainID2id"
RING = 4                 # host buffer sets in flight: one being copied into while the writers encode the others


def _byte(v):
    return isinstance(v, numbers.Integral) and 0 <= v <= 255


def tables(id_table, n, colors=None, background=None):
    """-> (lut uint8 [n], palette uint8 [n, 4] or None) for labels 0..n-1, or None where the reference would not write these bytes.
    lut[k] = id_table[k].  palette rows (B, G, R, use_image): set_img_color paints label k with colors[k] unless k == background
    or k >= len(colors), where it keeps the image pixel (use_image = 1); the written array is the RGB composite reversed to BGR."""
    if not isinstance(id_table, dict) or not all(k in id_table and _byte(id_table[k]) for k in range(n)):
        return None
    lut = torch.tensor([int(id_table[k]) for k in range(n)], dtype=torch.uint8)
    if colors is None:
        return lut, None
    try:
        colors = [list(c) for c in colors]
    except TypeError:
        return None
    if not all(len(c) == 3 and all(_byte(v) for v in c) for c in colors):
        return None
    palette = torch.zeros((n, 4), dtype=torch.uint8)
    for k in range(n):
        if k < len(colors) and k != background:
            palette[k, :3] = torch.tensor([int(v) for v in colors[k][::-1]], dtype=torch.uint8)
        else:
            palette[k, 3] = 1
    return lut, palette


def _device(net):
    """the CUDA device of `net`'s parameters, or None"""
    p = next(iter(net.parameters()), None)
    return p.device if p is not None and p.is_cuda else None


def _plan(t):
    """(device, lut, palette or None) when `t` (a Tester) writes what the device path computes, else None"""
    net = getattr(t, "network", None)
    dev = _device(net) if isinstance(net, Network_Multi_Path_Infer) else None
    devices = getattr(t, "devices", None)
    if dev is None or not devices or devices[0] != dev.index:
        return None
    func = getattr(type(t), "func_per_iteration", None)
    code = getattr(func, "__code__", None)
    test_py = getattr(type(t), "_fsb_test_py", None)
    if code is None or test_py is None or os.path.realpath(code.co_filename) != test_py:
        return None
    config = getattr(t, "config", None)
    if config is None or len(config.eval_scale_array) != 1 or t.is_flip:
        return None
    colors = t.dataset.get_class_colors() if t.show_prediction else None
    tab = tables(func.__globals__.get(ID_TABLE), net._num_classes, colors, getattr(config, "background", None))
    if tab is None or (t.show_prediction and tab[1] is None):
        return None
    return (dev,) + tab


def eligible(t):
    """True when the device path writes exactly the files `t`'s own run_online would: the train/ network on CUDA device
    devices[0], the reference's own SegTester.func_per_iteration (train/test.py next to the tools/ directory of the patched
    tester), one scale, no flipping, and id / colour tables of bytes"""
    return _plan(t) is not None


def _write(event, files):
    import cv2
    if event is not None:
        event.synchronize()
    for path, array in files:
        cv2.imwrite(path, array)         # a False return is ignored, as train/test.py:64,69 ignore it


class Writer:
    """Ring of host buffer sets and a thread pool of cv2.imwrite calls.  put() copies device images into the next set without
    blocking the host and queues their writes behind the copy's event; a set is reused only after its write has finished (which
    waited for its copy).  Leaving the block waits for every write and re-raises a writer's exception."""

    def __init__(self, slots=RING):
        self.buffers = [[] for _ in range(slots)]
        self.futures = [None] * slots
        self.pool = ThreadPoolExecutor(max_workers=slots, thread_name_prefix="fsb-imwrite")
        self.i = 0

    def put(self, files):
        """files: [(path, uint8 tensor H x W or H x W x 3)], written in that order"""
        s = self.i % len(self.buffers)
        self.i += 1
        if self.futures[s] is not None:
            self.futures[s].result()
            self.futures[s] = None
        bufs = self.buffers[s]
        out, on_cuda = [], False
        for k, (path, src) in enumerate(files):
            if k == len(bufs) or bufs[k].shape != src.shape:
                buf = torch.empty(src.shape, dtype=torch.uint8, pin_memory=src.is_cuda)
                bufs[k:k + 1] = [buf]
            bufs[k].copy_(src, non_blocking=True)
            on_cuda = on_cuda or src.is_cuda
            out.append((path, bufs[k].numpy()))
        event = None
        if on_cuda:
            event = torch.cuda.Event()
            event.record()
        self.futures[s] = self.pool.submit(_write, event, out)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.pool.shutdown(wait=True)
        if exc[0] is None:
            for f in self.futures:
                if f is not None:
                    f.result()
        return False


def _collate(batch):
    """dataset items -> (uint8 image N x H x W x 3, [fn]); the test split's labels are not read"""
    return torch.stack([evaluator.image(d) for d in batch]), [d["fn"] for d in batch]


def predict(t):
    """The device path: writes <cwd>/<config.save>/test/<fn>.png (and <fn>.viz.png with show_prediction) for every image"""
    dev, lut, palette = _plan(t)
    net = t.network
    folder = os.path.join(os.path.realpath("."), t.config.save, "test")
    with torch.cuda.device(dev), torch.random.fork_rng(devices=[dev.index]), torch.no_grad():
        net.eval()                       # val_func_process leaves the network in eval mode (tools/engine/tester.py:275)
        net.set_input_normalization(t.image_mean, t.image_std)
        lut = lut.to(dev)
        palette = palette.to(dev) if palette is not None else None
        with Writer() as writer:
            for img, names in evaluator.loader(t, collate_fn=_collate):
                x = img.to(dev, non_blocking=True).permute(0, 3, 1, 2)
                ids, viz = net.predict_label_maps(x, lut=lut, palette=palette)
                files = [(os.path.join(folder, names[0] + ".png"), ids[0])]
                if viz is not None:
                    files.insert(0, (os.path.join(folder, names[0] + ".viz.png"), viz[0]))
                writer.put(files)


def _device_or(name, orig):
    def method(self):
        if eligible(self):
            self.val_func = self.network
            return predict(self)
        return orig(self)
    method.__name__ = name
    method.__doc__ = orig.__doc__
    method._fsb_original = orig
    return method


def install(module):
    """Patch `module.Tester` (tools/engine/tester.py) in place; idempotent.  The device path serves only the SegTester of the
    train/test.py next to that module's tools/ directory."""
    cls = module.Tester
    root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.realpath(module.__file__))))
    cls._fsb_test_py = os.path.realpath(os.path.join(root, "train", "test.py"))
    for name in PATCHED:
        orig = getattr(cls, name)
        if getattr(orig, "_fsb_original", None) is None:
            setattr(cls, name, _device_or(name, orig))
    return cls
