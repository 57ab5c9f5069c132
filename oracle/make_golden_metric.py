#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- goldens of the evaluator's metrics and input normalisation from the UNMODIFIED reference
(tools/seg_opr/metric.py:7-27 `hist_info` / `compute_score`, tools/utils/img_utils.py:179-185 `normalize`), for the evaluator path
(SURVEY section 8 row N4; tools/engine/evaluator.py:206-225,329).  Inputs are regenerated from the seeds (numpy MT19937), so the
file only holds the reference's outputs.  Written to tests/golden/metric.json.
Run in the build container:  python oracle/make_golden_metric.py"""
import importlib.util
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "metric.json")

# name -> (seed, n_cl, shape, fraction of ignored pixels, ignore value, classes that never occur in pred AND gt)
CASES = {
    "cityscapes_small": (1, 19, (2, 64, 128), 0.05, 255, ()),
    "absent_classes": (2, 19, (1, 48, 96), 0.10, 255, (0, 7, 18)),      # nan IoU rows: nanmean skips them
    "negative_ignore": (3, 19, (1, 32, 64), 0.20, -1, ()),              # gt >= 0 is part of the reference's mask
    "all_ignored_row": (4, 5, (1, 16, 16), 0.50, 255, (4,)),
    "perfect": (5, 19, (1, 32, 32), 0.0, 255, ()),
}
NORMALIZE_CASES = {"imagenet_stats": (11, (2, 24, 40, 3), [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]),
                   "odd_stats": (12, (1, 7, 9, 3), [0.1, 0.5, 0.9], [0.5, 0.25, 1.5])}


def metric_inputs(name):
    seed, n_cl, shape, p_ign, ign, absent = CASES[name]
    rs = np.random.RandomState(seed)
    present = np.array([c for c in range(n_cl) if c not in absent])
    gt = present[rs.randint(0, len(present), size=shape)].astype(np.int64)
    pred = gt.copy()
    if name != "perfect":
        flip = rs.uniform(size=shape) < 0.35
        pred[flip] = present[rs.randint(0, len(present), size=int(flip.sum()))]
    gt[rs.uniform(size=shape) < p_ign] = ign
    return n_cl, pred.astype(np.uint8), gt


def normalize_inputs(name):
    seed, shape, mean, std = NORMALIZE_CASES[name]
    rs = np.random.RandomState(seed)
    return rs.randint(0, 256, size=shape).astype(np.uint8), np.array(mean), np.array(std)


def hist_info_restated(n_cl, pred, gt):
    """oracle restatement of tools/seg_opr/metric.py:7-15 hist_info: confusion matrix (row = ground truth, column = prediction)
    over the pixels whose ground truth lies in [0, n_cl), their count, and how many of them are predicted correctly"""
    valid = (gt >= 0) & (gt < n_cl)
    g, p = gt[valid].astype(np.int64), pred[valid].astype(np.int64)
    hist = np.bincount(n_cl * g + p, minlength=n_cl * n_cl).reshape(n_cl, n_cl)
    return hist, int(valid.sum()), int((p == g).sum())


def normalize_restated(img, mean, std):
    """oracle restatement of tools/utils/img_utils.py:179-185 normalize, same dtypes: uint8 -> float32 / 255, then the float64
    mean and std per channel"""
    return (img.astype(np.float32) / np.float32(255) - mean) / std


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_modules():
    root = ref_harness.REFERENCE_ROOT
    metric = _load(os.path.join(root, "tools", "seg_opr", "metric.py"), "_ref_metric")
    # img_utils imports cv2 at module level (not installed here); `normalize` itself is numpy only -> execute just that function
    src = open(os.path.join(root, "tools", "utils", "img_utils.py")).read()
    start = src.index("def normalize(")
    end = src.index("\ndef ", start + 1) if "\ndef " in src[start + 1:] else len(src)
    ns = {"np": np}
    exec(compile(src[start:end], "img_utils.normalize", "exec"), ns)      # noqa: S102 -- the reference's own function body, unmodified
    return metric, ns["normalize"]


def _f(x):
    return None if (isinstance(x, float) and np.isnan(x)) else x


def main():
    metric, normalize = reference_modules()
    out = {"metric": {}, "normalize": {}}
    for name in CASES:
        n_cl, pred, gt = metric_inputs(name)
        hist, labeled, correct = metric.hist_info(n_cl, pred, gt)
        iu, miou, miou_nb, acc = metric.compute_score(hist, correct, labeled)
        out["metric"][name] = {"hist": hist.astype(np.int64).tolist(), "labeled": int(labeled), "correct": int(correct),
                               "iu": [_f(float(v)) for v in iu], "mean_IU": _f(float(miou)), "mean_IU_no_back": _f(float(miou_nb)),
                               "mean_pixel_acc": _f(float(acc))}
    for name in NORMALIZE_CASES:
        img, mean, std = normalize_inputs(name)
        got = np.stack([normalize(im, mean, std) for im in img]).astype(np.float32)      # evaluator.py:329 feeds one HWC image at a time
        out["normalize"][name] = {"sum": float(got.astype(np.float64).sum()), "first": got.reshape(-1)[:12].tolist(),
                                  "last": got.reshape(-1)[-12:].tolist()}
    with open(OUT, "w") as f:
        json.dump(out, f)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
