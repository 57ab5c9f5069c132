"""Golden vectors of the reference's training augmentation (train/dataloader.py:8-31 TrainPre; get_train_loader end to end) ->
tests/golden/trainpre.npz.  Run where a reference checkout is available:

    python -m oracle.make_golden_trainpre

The inputs are the closed-form `synthetic_pair`, so only the reference's outputs are stored.  For every case the reference's own
TrainPre runs under a fixed `random.seed`; its random draws are recorded by a proxy of the `random` module that img_utils calls,
together with the next `random.random()` after the call (which pins how much of the stream TrainPre consumed)."""
import hashlib
import os
import random
import tempfile

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "trainpre.npz")
STRIDE = 997   # sample stride of the full-size outputs


def synthetic_pair(H, W, k):
    """closed-form uint8 RGB image (H x W x 3) and uint8 label (values 0..18 and 255) number k"""
    y, x = np.mgrid[0:H, 0:W].astype(np.int64)
    img = np.stack([((x * 131 + y * 71 + c * 29 + k * 53) ^ ((x * y) >> 3)) & 255 for c in range(3)], axis=2).astype(np.uint8)
    gt = ((x // 5 + (y // 3) * 7 + k) % 19).astype(np.uint8)
    gt[(x * 3 + y * 5 + k) % 31 == 0] = 255
    return img, gt


class Config(dict):
    def __getattr__(self, k):
        return self[k]


def config(crop, scales, g):
    return Config(image_height=crop[0], image_width=crop[1], train_scale_array=scales, gt_down_sampling=g)


# (name, H, W, crop, train_scale_array, gt_down_sampling, predicate on the draws (mirror, sh, sw, pos_h, pos_w))
SMALL = [
    ("mirror_s075_pos0", 37, 53, (24, 32), [0.75], 1, lambda d: d[0] == 1 and d[3] == 0 and d[4] == 0),
    ("s125_edge_rows", 37, 53, (24, 32), [1.25], 1, lambda d: d[0] == 0 and d[3] == d[1] - 24 + 1),
    ("mirror_s125_edge_both", 37, 53, (24, 32), [1.25], 8, lambda d: d[0] == 1 and d[3] == d[1] - 24 + 1 and d[4] == d[2] - 32 + 1),
    ("s1_pad_both", 37, 53, (48, 64), [1], 1, lambda d: d[0] == 0),
    ("mirror_s1_pad_both_g8", 37, 53, (48, 64), [1], 8, lambda d: d[0] == 1),
    ("s125_pad_cols", 37, 53, (40, 72), [1.25], 8, lambda d: d[0] == 1 and d[3] > 0),
    ("mixed_scales", 64, 96, (32, 48), [0.75, 1, 1.25], 1, lambda d: True),
    ("mixed_scales_mirror", 64, 96, (32, 48), [0.75, 1, 1.25], 8, lambda d: d[0] == 1),
    ("odd_s075_edge_cols", 33, 17, (16, 8), [0.75], 1, lambda d: d[4] == d[2] - 8 + 1),
    ("no_scale_array", 37, 53, (24, 32), None, 1, lambda d: d[0] == 1),
]
# the drivers' geometries: train.py (1024 x 2048 -> 512 x 1024) and the search (512 x 1024 after down_sampling -> 256 x 512, labels
# 32 x 64), once per scale
FULL = [("train_s%s" % s, 1024, 2048, (512, 1024), [s], 1, lambda d: True) for s in ("0.75", "1", "1.25")] + \
       [("search_s%s" % s, 512, 1024, (256, 512), [s], 8, lambda d: True) for s in ("0.75", "1", "1.25")]
E2E = dict(H=96, W=160, crop=(64, 128), scales=[0.75, 1, 1.25], g=1, images=4, batch=2, workers=2, seed=7)


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class _Recorder:
    """stands in for the `random` module inside img_utils and records what TrainPre drew"""

    def __init__(self):
        self.calls = []

    def random(self):
        v = random.random()
        self.calls.append(("random", v))
        return v

    def choice(self, seq):
        v = random.choice(seq)
        self.calls.append(("choice", v))
        return v

    def randint(self, a, b):
        v = random.randint(a, b)
        self.calls.append(("randint", v))
        return v


def run_case(ns, H, W, k, crop, scales, g, seed):
    """the reference's TrainPre on synthetic_pair(H, W, k) -> (draws, next random, data float32, label int64)"""
    import torch
    img_utils = ns.dataloader.random_mirror.__globals__
    img, gt = synthetic_pair(H, W, k)
    rec = _Recorder()
    saved = img_utils["random"]
    img_utils["random"] = rec
    try:
        random.seed(seed)
        p_img, p_gt, _ = ns.dataloader.TrainPre(config(crop, scales, g), np.array([0.485, 0.456, 0.406]),
                                                np.array([0.229, 0.224, 0.225]))(img, gt)
        nxt = random.random()
    finally:
        img_utils["random"] = saved
    data = torch.from_numpy(np.ascontiguousarray(p_img)).float().numpy()     # BaseDataset.py:47-48
    label = torch.from_numpy(np.ascontiguousarray(p_gt)).long().numpy()
    mirror = int(rec.calls[0][1] >= 0.5)
    s = rec.calls[1][1] if scales is not None else 1
    sh, sw = (int(H * s), int(W * s)) if scales is not None else (H, W)
    ints = [v for kind, v in rec.calls if kind == "randint"]
    pos_h = ints.pop(0) if sh > crop[0] else 0
    pos_w = ints.pop(0) if sw > crop[1] else 0
    return (mirror, sh, sw, pos_h, pos_w), nxt, data, label


def make_e2e(ns, datasets, out):
    """4 synthetic PNG pairs through the reference's get_train_loader (Cityscapes dataset, batch 2, 2 workers)"""
    import cv2
    import torch
    e = E2E
    root = tempfile.mkdtemp(prefix="fsb_trainpre_")
    lines = []
    for k in range(e["images"]):
        img, gt = synthetic_pair(e["H"], e["W"], k)
        cv2.imwrite(os.path.join(root, "img%d.png" % k), img[:, :, ::-1])      # the dataset flips BGR -> RGB again
        cv2.imwrite(os.path.join(root, "gt%d.png" % k), gt)
        lines.append("img%d.png gt%d.png\n" % (k, k))
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.writelines(lines)
    loader = e2e_loader(ns.dataloader, datasets, root)
    batches = list(iter(loader))
    for i, b in enumerate(batches):
        out["e2e_data_%d" % i] = b["data"].numpy()
        out["e2e_label_%d" % i] = b["label"].numpy()
        out["e2e_fn_%d" % i] = np.array(b["fn"])
        out["e2e_n_%d" % i] = b["n"].numpy()
    out["e2e_batches"] = np.array(len(batches))


def e2e_loader(dataloader_module, datasets_module, root):
    """the end-to-end case's loader, built by the reference's get_train_loader over the PNGs under `root` (seeds fixed)"""
    import torch
    e = E2E
    cfg = Config(img_root_folder=root, gt_root_folder=root, train_source=os.path.join(root, "train.txt"),
                 eval_source=os.path.join(root, "train.txt"), down_sampling=1, image_height=e["crop"][0],
                 image_width=e["crop"][1], train_scale_array=e["scales"], gt_down_sampling=e["g"],
                 image_mean=np.array([0.485, 0.456, 0.406]), image_std=np.array([0.229, 0.224, 0.225]),
                 batch_size=e["batch"], niters_per_epoch=e["images"] // e["batch"], num_workers=e["workers"])
    random.seed(e["seed"])
    torch.manual_seed(e["seed"])
    return dataloader_module.get_train_loader(cfg, datasets_module.Cityscapes)


def load_reference():
    """the reference's train/dataloader.py and datasets package (the Cityscapes class) through oracle.ref_harness"""
    import collections
    import collections.abc
    from oracle import ref_harness
    collections.Iterable = collections.abc.Iterable      # img_utils.get_2dshape (py3.10+ moved it; the launcher does the same)
    ns = ref_harness.load_reference("train", "dataloader")
    import importlib
    import sys
    sys.path.insert(0, os.path.join(ns.root, "tools"))
    try:
        datasets = importlib.import_module("datasets.cityscapes.cityscapes")
    finally:
        sys.path.remove(os.path.join(ns.root, "tools"))
    return ns, datasets


def main():
    ns, datasets = load_reference()
    out = {}
    names = []
    for full, cases in ((False, SMALL), (True, FULL)):
        for k, (name, H, W, crop, scales, g, want) in enumerate(cases):
            scales = None if scales is None else [float(s) if isinstance(s, str) else s for s in scales]
            for seed in range(1000):
                draws, nxt, data, label = run_case(ns, H, W, k, crop, scales, g, seed)
                if want(draws):
                    break
            else:
                raise RuntimeError("no seed gives the draws case %s wants" % name)
            names.append(name)
            out[name + "/meta"] = np.array([H, W, k, crop[0], crop[1], g, seed] + list(draws), np.int64)
            out[name + "/scales"] = np.array([] if scales is None else scales, np.float64)
            out[name + "/next_random"] = np.array(nxt)
            if full:
                out[name + "/data_sha256"] = np.array(digest(data))
                out[name + "/label_sha256"] = np.array(digest(label))
                out[name + "/data_sample"] = data.reshape(-1)[::STRIDE].copy()
                out[name + "/label_sample"] = label.reshape(-1)[::STRIDE].copy()
            else:
                out[name + "/data"] = data
                out[name + "/label"] = label
            print(name, "seed", seed, "draws", draws, data.shape, label.shape)
    out["cases"] = np.array(names)
    out["full_cases"] = np.array([c[0] for c in FULL])
    make_e2e(ns, datasets, out)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
