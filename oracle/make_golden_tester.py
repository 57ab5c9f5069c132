#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- goldens of the drivers' test-set files from the UNMODIFIED reference (train/test.py:49-69
`SegTester.func_per_iteration`, tools/utils/visualize.py:6-21 `show_prediction`), for fasterseg_b200/tester.py.  The reference's
own method runs with `whole_eval` replaced by a closed-form int64 prediction map (so no network and no GPU are involved) and writes
its PNGs with cv2.imwrite into a scratch directory; the golden keeps the inputs and the bytes of every file (for the full
1024 x 2048 frame only their sha256 -- the inputs are `pred_map` / `image_map` below).  Written to tests/golden/tester.npz.
Run in the build container:  python oracle/make_golden_tester.py"""
import hashlib
import os
import sys
import tempfile
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "tester.npz")

# name -> (H, W, n_classes, show_prediction, config.background, number of colours (None = the dataset's 19))
CASES = {
    "ids_37x53": (37, 53, 19, False, -1, None),
    "viz_37x53": (37, 53, 19, True, -1, None),
    "viz_background3_64x128": (64, 128, 19, True, 3, None),
    "viz_short_colours_64x128": (64, 128, 19, True, -1, 15),
    "viz_11cls_background3_37x53": (37, 53, 11, True, 3, None),
    "ids_11cls_64x128": (64, 128, 11, False, -1, None),
    "viz_11cls_7colours_64x128": (64, 128, 11, True, 3, 7),
    "viz_1024x2048": (1024, 2048, 19, True, -1, None),
    "viz_background3_1024x2048": (1024, 2048, 19, True, 3, None),
}
HASHED = 1024 * 2048          # cases this large keep only the sha256 of their files


def pred_map(h, w, n):
    """closed-form int64 trainId map with every class present and long runs as well as isolated pixels"""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    return (y // 3 * 7 + x // 5 * 3 + (x * y) % 5) % n


def image_map(h, w):
    """closed-form uint8 RGB image"""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    return np.stack([(y * 5 + x * 11 + c * 70 + (x * y) % 7) % 256 for c in range(3)], axis=2).astype(np.uint8)


def main():
    ns = ref_harness.load_reference("train", "test")
    test = ns.test
    colors19 = test.Cityscapes.get_class_colors()
    table = test.cityscapes_trainID2id
    out = {"id_table_keys": np.array(sorted(table), np.int64), "id_table_values": np.array([table[k] for k in sorted(table)], np.int64),
           "colors": np.array(colors19, np.int64)}
    for name, (h, w, n, show, background, ncol) in CASES.items():
        colors = colors19 if ncol is None else colors19[:ncol]
        pred, img = pred_map(h, w, n), image_map(h, w)
        with tempfile.TemporaryDirectory() as tmp:
            cwd = os.getcwd()
            os.makedirs(os.path.join(tmp, "out", "test"))
            os.chdir(tmp)
            try:
                t = object.__new__(test.SegTester)
                t.config = types.SimpleNamespace(eval_scale_array=[1], background=background, save="out")
                t.show_prediction = show
                t.dataset = types.SimpleNamespace(get_class_colors=lambda c=colors: c)
                t.whole_eval = lambda img_, out_size, device, p=pred: p.copy()
                t.func_per_iteration(dict(data=img, label=np.zeros((h, w), np.uint8), fn=name), 0, iter=0)
            finally:
                os.chdir(cwd)
            files = {}
            for suffix in (".png", ".viz.png"):
                path = os.path.join(tmp, "out", "test", name + suffix)
                if os.path.exists(path):
                    files[suffix] = open(path, "rb").read()
        assert (".viz.png" in files) == show and ".png" in files
        out[name + "/case"] = np.array([h, w, n, int(show), background, -1 if ncol is None else ncol], np.int64)
        for suffix, data in files.items():
            key = name + "/" + suffix.lstrip(".")
            if h * w >= HASHED:
                out[key + ".sha256"] = np.frombuffer(hashlib.sha256(data).digest(), np.uint8)
            else:
                out[key] = np.frombuffer(data, np.uint8)
        if h * w < HASHED:
            out[name + "/pred"] = pred
            out[name + "/image"] = img
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
