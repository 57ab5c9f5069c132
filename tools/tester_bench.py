#!/usr/bin/env python
"""Test-set prediction images/s: the reference's own `SegTester.run_online` (train/test.py:49-69; host normalise, fp32 score map
copied back, numpy argmax, Python trainId -> id loop, optional colour map) against the same call after `fasterseg_b200.tester`
patched it (one kernel writes the id / colour maps, pinned ring, imwrite thread pool), alternated, on the seeded student.

    python tools/tester_bench.py [--images 8] [--runs 3] [--threds 3]

Input: seeded synthetic 1024 x 2048 PNGs in a temporary directory, read through a dataset with BaseDataset's item protocol.  Both
arms run with and without show_prediction.  Where no copy of the reference is around (oracle/_ref), the reference arm is the
reference arithmetic restated here, and labelled so.  The two arms' files must be byte-identical.  Also times the kernel against
fsb_upsample_argmax with CUDA events at 1 x 19 x 128 x 256 -> 1024 x 2048.  Prints the card, its power limit and one JSON line."""
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
from fasterseg_b200 import tester, zoo  # noqa: E402

MEAN, STD = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
# the id table and colours of train/test.py:25-46 and the Cityscapes dataset, as the golden of oracle/make_golden_tester.py keeps them
_GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "tester.npz"))
ID_TABLE = dict(zip(_GOLDEN["id_table_keys"].tolist(), _GOLDEN["id_table_values"].tolist()))
COLORS = _GOLDEN["colors"].tolist()


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


class PngSet:
    """the 'test' items of tools/datasets/BaseDataset.py:34-64: cv2-decoded BGR flipped to RGB, a dummy label, fn"""

    def __init__(self, n, h, w, seed, folder):
        import cv2
        rs = np.random.RandomState(seed)
        self.n, self.folder = n, folder
        for i in range(n):
            base = rs.randint(0, 256, size=(h // 16 + 1, w // 16 + 1, 3)).astype(np.uint8)
            bgr = np.ascontiguousarray(np.repeat(np.repeat(base, 16, 0), 16, 1)[:h, :w] + rs.randint(0, 8, size=(h, w, 3)).astype(np.uint8))
            cv2.imwrite(os.path.join(folder, "%d.png" % i), bgr)

    def get_length(self):
        return self.n

    def __len__(self):
        return self.n

    def __getitem__(self, idx):
        import cv2
        bgr = cv2.imread(os.path.join(self.folder, "%d.png" % idx), cv2.IMREAD_COLOR)
        return dict(data=bgr[:, :, ::-1], label=np.zeros(bgr.shape[:2], np.uint8), fn="img%d" % idx, n=self.n)

    @staticmethod
    def get_class_colors():
        return COLORS


def _reference_classes(root):
    """(engine.tester module, train/test.py's SegTester) of the reference copy at `root`, or (None, None)"""
    if not root or not os.path.isfile(os.path.join(root, "tools", "engine", "tester.py")):
        return None, None
    import collections
    import collections.abc
    for n in ("Iterable", "Mapping", "Sequence"):                 # tools/utils/img_utils.py predates python 3.10
        if not hasattr(collections, n):
            setattr(collections, n, getattr(collections.abc, n))
    sys.path[:0] = [os.path.join(root, "train"), os.path.join(root, "tools")]
    import importlib
    return importlib.import_module("engine.tester"), importlib.import_module("test").SegTester


def _restated_classes(folder):
    """a Tester / SegTester pair whose func_per_iteration restates train/test.py:49-69 (with tools/engine/tester.py:179-204,
    270-291 and tools/utils/visualize.py:6-21) in a file laid out like the reference, so that the patch serves it"""
    os.makedirs(os.path.join(folder, "tools", "engine"))
    os.makedirs(os.path.join(folder, "train"))
    with open(os.path.join(folder, "tools", "engine", "tester.py"), "w") as f:
        f.write("class Tester(object):\n"
                "    def run_online(self):\n        self.val_func = self.network\n"
                "        for idx in range(self.ndata):\n            self.func_per_iteration(self.dataset[idx], self.devices[0], iter=idx)\n\n"
                "    def run_online_multiprocess(self):\n        return self.run_online()\n")
    with open(os.path.join(folder, "train", "test.py"), "w") as f:
        f.write('''import os
import cv2
import numpy as np
import torch

cityscapes_trainID2id = %r


def func_per_iteration(self, data, device, iter=None):
    config = self.config
    img, name = data["data"], data["fn"]
    x = (img.astype(np.float32) / 255.0 - self.image_mean) / self.image_std
    x = torch.FloatTensor(np.ascontiguousarray(x.transpose(2, 0, 1)[None], dtype=np.float32)).cuda(device)
    with torch.no_grad():
        self.val_func.eval()
        score = torch.exp(self.val_func(x)[0])
    pred = score.permute(1, 2, 0).cpu().numpy().argmax(2)
    if self.show_prediction:
        im = np.array(img, np.uint8)
        for i, c in enumerate(self.dataset.get_class_colors()):
            if i != config.background:
                im[np.where(pred == i)] = c
        cv2.imwrite(os.path.join(os.path.realpath("."), config.save, "test", name + ".viz.png"), im[:, :, ::-1])
    for a in range(pred.shape[0]):
        for b in range(pred.shape[1]):
            pred[a, b] = cityscapes_trainID2id[pred[a, b]]
    cv2.imwrite(os.path.join(os.path.realpath("."), config.save, "test", name + ".png"), pred)
''' % ID_TABLE)
    import importlib.util
    mods = []
    for name, path in (("fsb_bench_engine_tester", ("tools", "engine", "tester.py")), ("fsb_bench_test", ("train", "test.py"))):
        spec = importlib.util.spec_from_file_location(name, os.path.join(folder, *path))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        mods.append(mod)
    eng, test = mods

    class SegTester(eng.Tester):
        func_per_iteration = test.func_per_iteration

        def __init__(self, dataset, class_num, image_mean, image_std, network, multi_scales, is_flip, devices=0, out_idx=0, threds=3,
                     config=None, logger=None, verbose=False, save_path=None, show_prediction=False):
            self.dataset, self.ndata, self.class_num, self.image_mean, self.image_std = dataset, dataset.get_length(), class_num, image_mean, image_std
            self.network, self.multi_scales, self.is_flip, self.devices, self.out_idx = network, multi_scales, is_flip, [devices], out_idx
            self.threds, self.config, self.show_prediction = threds, config, show_prediction

    return eng, SegTester


def _seeded_student(seed):
    """the student with the seeded weights of smoke() / tests/test_student_gpu.py (logits of a trained network's magnitude)"""
    from oracle import fasterseg_oracle as orc
    from tests import helpers as H
    model = zoo.build_network(1)
    _, g = H.student_structure(1)
    sd = orc.random_state_dict({k: tuple(v) for k, v in g["state_dict_shapes"].items() if not k.endswith("num_batches_tracked")},
                               seed=seed)
    own, seen = model.state_dict(), set()
    for k in sorted(sd):
        if own[k].data_ptr() not in seen:
            seen.add(own[k].data_ptr())
            own[k].copy_(sd[k])
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eps, m.momentum = orc.BN_EPS, orc.BN_MOMENTUM
    return model.cuda().eval()


def _tied_only(model, ds, idx, a, b):
    """number of pixels where the id maps a (reference) and b (device) of image idx differ; asserts that at each of them the
    fp32 logits of the two labels are exp-tied or a rounding step apart (the reference takes the first of equal exp values)"""
    import cv2
    pa, pb = (cv2.imread(p, cv2.IMREAD_UNCHANGED) for p in (a, b))
    diff = pa != pb
    if not diff.any():
        return 0
    inv = np.zeros(256, np.int64)
    for k in range(19):
        inv[ID_TABLE[k]] = k
    img = np.ascontiguousarray(ds[idx]["data"])
    x = ((img.astype(np.float32) / 255.0 - MEAN) / STD).astype(np.float32).transpose(2, 0, 1)[None]
    with torch.no_grad():
        logits = model(torch.from_numpy(np.ascontiguousarray(x)).cuda())[0].float()
    m = torch.from_numpy(diff).cuda()
    la = torch.from_numpy(inv[pa]).cuda()[m]
    lb = torch.from_numpy(inv[pb]).cuda()[m]
    flat = logits.reshape(19, -1)[:, m.reshape(-1)]
    va, vb = flat.gather(0, la[None])[0], flat.gather(0, lb[None])[0]
    tie = (torch.exp(va) == torch.exp(vb)) | ((va - vb).abs() <= 4 * torch.finfo(torch.float32).eps * torch.maximum(va.abs(), vb.abs()))
    assert bool(tie.all()), "image %d: labels differ at pixels that are not tied" % idx
    return int(diff.sum())


def _events(fn, iters=200, warmup=20):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1000.0)
    return statistics.median(times)


def kernel_times():
    from fasterseg_b200 import functional as F_
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(1, 128, 256, 24, generator=g) * 3).half().cuda().permute(0, 3, 1, 2)[:, :19]
    lut, pal = tester.tables(ID_TABLE, 19, COLORS, -1)
    lut, pal = lut.cuda(), pal.cuda()
    img = torch.randint(0, 256, (1, 1024, 2048, 3), dtype=torch.uint8, device="cuda")
    labels = torch.empty(1, 1024, 2048, dtype=torch.uint8, device="cuda")
    ids = torch.empty_like(labels)
    viz = torch.empty(1, 1024, 2048, 3, dtype=torch.uint8, device="cuda")
    return {"upsample_argmax_us": _events(lambda: F_.upsample_argmax(x, (1024, 2048), out=labels)),
            "map_ids_us": _events(lambda: F_.upsample_argmax_map(x, (1024, 2048), lut=lut, ids_out=ids)),
            "map_ids_viz_us": _events(lambda: F_.upsample_argmax_map(x, (1024, 2048), lut=lut, palette=pal, image=img, ids_out=ids,
                                                                      viz_out=viz))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--threds", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    card = _card()
    print("card:", card)
    from oracle import ref_harness
    work = tempfile.mkdtemp(prefix="fsb_tester_bench_")
    eng, SegTester = _reference_classes(ref_harness.REFERENCE_ROOT if ref_harness.reference_available() else None)
    arm = "reference SegTester.run_online"
    if eng is None:
        eng, SegTester = _restated_classes(os.path.join(work, "FasterSeg"))
        arm = "restated reference arithmetic (no reference copy)"
    originals = {n: eng.Tester.__dict__[n] for n in tester.PATCHED}
    os.makedirs(os.path.join(work, "png"))
    ds = PngSet(args.images, 1024, 2048, 31, os.path.join(work, "png"))
    model = _seeded_student(77)
    result = {"card": card, "reference_arm": arm, "images": args.images, "threds": args.threds, "size": [1024, 2048], "cases": {}}
    cwd = os.getcwd()
    try:
        for show in (False, True):
            runs = {"reference": [], "device": []}
            tied_pixels = files_differing = 0
            for r in range(args.runs):
                for side in ("reference", "device"):
                    for n, f in originals.items():
                        setattr(eng.Tester, n, f)
                    if side == "device":
                        tester.install(eng)
                    d = os.path.join(work, "run_%d_%d_%s" % (show, r, side))
                    os.makedirs(os.path.join(d, "out", "test"))
                    os.chdir(d)
                    config = types.SimpleNamespace(num_classes=19, eval_scale_array=[1], background=-1, save="out")
                    t = SegTester(ds, 19, MEAN, STD, model, [1], False, 0, threds=args.threds, config=config, show_prediction=show)
                    if side == "device":
                        assert tester.eligible(t)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    t.run_online()
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    os.chdir(cwd)
                    runs[side].append(args.images / dt)
                    print("show_prediction=%s run %d %s: %.3f images/s" % (show, r, side, args.images / dt), flush=True)
                a, b = (os.path.join(work, "run_%d_%d_%s" % (show, r, s), "out", "test") for s in ("reference", "device"))
                names = sorted(os.listdir(a))
                assert names == sorted(os.listdir(b)) and len(names) == args.images * (2 if show else 1), (names, os.listdir(b))
                differ = [n for n in names if open(os.path.join(a, n), "rb").read() != open(os.path.join(b, n), "rb").read()]
                tied = sum(_tied_only(model, ds, int(n[3:-4]), os.path.join(a, n), os.path.join(b, n)) for n in differ if n.endswith(".png")
                           and not n.endswith(".viz.png"))
                assert all(n.replace(".viz.png", ".png") in differ for n in differ), "a colour map differs where its ids do not"
                assert tied or not differ, "files differ without a tied label: %s" % differ
                tied_pixels = max(tied_pixels, tied)
                files_differing = max(files_differing, len(differ))
            result["cases"]["show_prediction" if show else "ids_only"] = {
                "reference_images_per_s": statistics.median(runs["reference"]), "device_images_per_s": statistics.median(runs["device"]),
                "reference_runs": runs["reference"], "device_runs": runs["device"],
                "device_faster_every_run": all(d > r for d, r in zip(runs["device"], runs["reference"])), "files_identical": files_differing == 0,
                "files_differing_at_tied_labels": files_differing, "tied_pixels": tied_pixels}
    finally:
        os.chdir(cwd)
        for n, f in originals.items():
            setattr(eng.Tester, n, f)
    result["kernel_us_1x19x128x256_to_1024x2048"] = kernel_times()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
