#!/usr/bin/env python
"""Validation throughput (images/s) of the device path behind the reference's Evaluator (fasterseg_b200.evaluator) on seeded synthetic
data: the student at 1024x2048, the supernet at 512x1024 (the search's down_sampling = 2) for one out_idx and for the search's loop
over the five heads, and -- given a reference checkout (--reference) -- the reference's own
run_online_multiprocess (3 spawned workers, host normalise / exp / argmax / numpy histogram) against the device path, alternated.
Every case is timed twice: images already decoded in RAM, and PNG files decoded from a temporary directory by the loader's host
workers.  Weights are seeded; the numbers do not depend on them.  Prints the card, its power limit and SM clock, and one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fasterseg_b200 import evaluator, metric, zoo  # noqa: E402
from fasterseg_b200.model_search import Network_Multi_Path  # noqa: E402

MEAN, STD = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
WML = [4. / 12, 6. / 12, 8. / 12, 10. / 12, 1.]


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


class SyntheticSet:
    """the 'val' items of tools/datasets/BaseDataset.py:34-60: RGB uint8 image as the flipped view of a BGR array, uint8 label.
    png_dir: decode <i>.png / <i>_gt.png with cv2 on every access (as the dataset does); else the arrays stay in RAM"""

    def __init__(self, n, h, w, seed, png_dir=None):
        rs = np.random.RandomState(seed)
        self.n, self.png_dir, self.items = n, png_dir, []
        for i in range(n):
            # smooth-ish content so that PNG compression (and decode cost) resembles a photo more than noise does
            base = rs.randint(0, 256, size=(h // 16 + 1, w // 16 + 1, 3)).astype(np.uint8)
            bgr = np.ascontiguousarray(np.repeat(np.repeat(base, 16, 0), 16, 1)[:h, :w] + rs.randint(0, 8, size=(h, w, 3)).astype(np.uint8))
            lab = np.repeat(np.repeat(rs.randint(0, 19, size=(h // 32 + 1, w // 32 + 1)).astype(np.uint8), 32, 0), 32, 1)[:h, :w].copy()
            lab[rs.uniform(size=lab.shape) < 0.05] = 255
            if png_dir is None:
                self.items.append((bgr, lab))
            else:
                import cv2
                cv2.imwrite(os.path.join(png_dir, "%d.png" % i), bgr)
                cv2.imwrite(os.path.join(png_dir, "%d_gt.png" % i), lab)

    def get_length(self):
        return self.n

    def __len__(self):
        return self.n

    def __getitem__(self, idx):
        if self.png_dir is None:
            bgr, lab = self.items[idx]
        else:
            import cv2
            bgr = cv2.imread(os.path.join(self.png_dir, "%d.png" % idx), cv2.IMREAD_COLOR)
            lab = cv2.imread(os.path.join(self.png_dir, "%d_gt.png" % idx), cv2.IMREAD_GRAYSCALE)
        return dict(data=bgr[:, :, ::-1], label=lab, fn=str(idx), n=self.n)

    def get_class_names(self):
        return ["class%d" % i for i in range(19)]


class StandInEvaluator:
    """the attributes tools/engine/evaluator.py:17-44 sets; used when no copy of the reference is around"""

    def __init__(self, dataset, class_num, image_mean, image_std, network, multi_scales, is_flip, devices=0, out_idx=0, threds=3,
                 config=None, logger=None, verbose=False, save_path=None, show_image=False, show_prediction=False):
        self.dataset, self.ndata, self.class_num, self.image_mean, self.image_std = dataset, dataset.get_length(), class_num, image_mean, image_std
        self.network, self.multi_scales, self.is_flip, self.devices, self.out_idx, self.threds = network, multi_scales, is_flip, [devices], out_idx, threds
        self.config, self.logger, self.save_path, self.show_image, self.show_prediction = config, logger, save_path, show_image, show_prediction

    def run_online_multiprocess(self):
        raise RuntimeError("no reference evaluator")

    def compute_metric(self, results):
        hist = sum(r["hist"] for r in results)
        iu, miou, _, _ = metric.compute_score(hist, sum(r["correct"] for r in results), sum(r["labeled"] for r in results))
        return "mean_IU %.3f%%" % (miou * 100), miou


def _reference_evaluator(root):
    """engine.evaluator and train/eval.py's SegEvaluator of the reference checkout at `root`, or (None, None)"""
    if not root or not os.path.isfile(os.path.join(root, "tools", "engine", "evaluator.py")):
        return None, None
    import collections
    import collections.abc
    for n in ("Iterable", "Mapping", "Sequence"):                 # tools/utils/img_utils.py predates python 3.10
        if not hasattr(collections, n):
            setattr(collections, n, getattr(collections.abc, n))
    sys.path[:0] = [os.path.join(root, "train"), os.path.join(root, "tools")]   # the spawned workers import the same modules
    import importlib
    return importlib.import_module("engine.evaluator"), importlib.import_module("eval").SegEvaluator


def _seeded(model, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in model.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (2.0 / max(1, p[0].numel())) ** 0.5)
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d) and m.running_mean is not None:
                m.running_mean.normal_(0, 0.1, generator=g)
                m.running_var.uniform_(0.5, 1.5, generator=g)
    return model


def _time(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--images", type=int, default=24, help="validation images per timed pass")
    ap.add_argument("--rounds", type=int, default=3, help="timed passes per case (median reported)")
    ap.add_argument("--ref-images", type=int, default=6, help="images per pass of the reference's multiprocess path")
    ap.add_argument("--workers", type=int, default=3, help="Evaluator.threds: the reference's processes / our loader's workers")
    ap.add_argument("--reference", default=os.environ.get("FASTERSEG_REFERENCE"),
                    help="a FasterSeg checkout: also time its own run_online_multiprocess (default $FASTERSEG_REFERENCE)")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "eval_bench needs a GPU"
    card = _card()
    print("card: %s" % card)
    ev_mod, Seg = _reference_evaluator(a.reference)
    Eval = Seg if Seg is not None else StandInEvaluator
    if ev_mod is not None:
        originals = {n: ev_mod.Evaluator.__dict__[n] for n in evaluator.PATCHED}
        evaluator.install(ev_mod)
    else:
        evaluator.install(types.SimpleNamespace(Evaluator=StandInEvaluator))
    config = types.SimpleNamespace(num_classes=19, eval_scale_array=[1], eval_crop_size=1024, eval_stride_rate=5 / 6, background=0)

    student = _seeded(zoo.build_network(1), 1).cuda().eval()
    supernet = _seeded(Network_Multi_Path(19, 16, torch.nn.CrossEntropyLoss(ignore_index=255), Fch=12, width_mult_list=WML,
                                          prun_modes=["max", "arch_ratio"], stem_head_width=[(1, 1), (8. / 12, 8. / 12)]), 2).cuda().eval()
    supernet.arch_idx = 0
    results = {"card": card, "images": a.images, "workers": a.workers}
    tmp = tempfile.mkdtemp(prefix="fsb_eval_bench_")
    for source in ("ram", "png"):
        sets = {}
        for name, (h, w) in (("student", (1024, 2048)), ("supernet", (512, 1024))):
            d = os.path.join(tmp, "%s_%s" % (name, source))
            if source == "png":
                os.makedirs(d)
            sets[name] = SyntheticSet(a.images, h, w, seed=3, png_dir=d if source == "png" else None)

        def device(model, ds, heads):
            def run():
                miou = []
                for h in heads:
                    ev = Eval(ds, 19, MEAN, STD, model, [1], False, 0, out_idx=h, threds=a.workers, config=config)
                    miou.append(ev.run_online_multiprocess()[1])
                return miou
            return run

        cases = {"student": device(student, sets["student"], [0]), "supernet_1head": device(supernet, sets["supernet"], [0]),
                 "supernet_5heads": device(supernet, sets["supernet"], range(5))}
        for name, run in cases.items():
            run()                                                       # warm-up: module loads, allocator, loader workers
            ts = [_time(run)[0] for _ in range(a.rounds)]
            n = a.images * (5 if name.endswith("5heads") else 1)
            results["%s_%s_img_per_s" % (name, source)] = n / statistics.median(ts)
            print("%-16s %-3s device path: %8.1f images/s (median of %d passes over %d images; min-max %.3f-%.3f s)"
                  % (name, source, n / statistics.median(ts), a.rounds, n, min(ts), max(ts)))
        if ev_mod is not None:
            ref_set = SyntheticSet(a.ref_images, 1024, 2048, seed=4,
                                   png_dir=(os.makedirs(os.path.join(tmp, "ref_" + source)) or os.path.join(tmp, "ref_" + source))
                                   if source == "png" else None)
            ref_t, dev_t, err = [], [], None
            for _ in range(2):                                          # alternated: reference, device, reference, device
                ev = Seg(ref_set, 19, MEAN, STD, student, [1], False, 0, threds=a.workers, config=config)
                try:
                    t, r_ref = _time(lambda: originals["run_online_multiprocess"](ev))
                    ref_t.append(t)
                except Exception as e:  # noqa: BLE001 -- reported, not hidden
                    err = "%s: %s" % (type(e).__name__, e)
                    break
                t, r_dev = _time(lambda: Seg(ref_set, 19, MEAN, STD, student, [1], False, 0, threds=a.workers,
                                             config=config).run_online_multiprocess())
                dev_t.append(t)
            if err is None:
                results["reference_vs_device_%s" % source] = {"reference_img_per_s": a.ref_images / min(ref_t),
                                                              "device_img_per_s": a.ref_images / min(dev_t),
                                                              "miou_reference": float(r_ref[1]), "miou_device": float(r_dev[1])}
                print("student %-3s reference run_online_multiprocess: %.2f images/s, device path %.1f images/s (best of 2, %d images); "
                      "mIoU %.6f vs %.6f" % (source, a.ref_images / min(ref_t), a.ref_images / min(dev_t), a.ref_images,
                                            float(r_ref[1]), float(r_dev[1])))
            else:
                results["reference_vs_device_%s" % source] = {"error": err}
                print("student %-3s reference run_online_multiprocess failed: %s" % (source, err))
    print(json.dumps(results))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
