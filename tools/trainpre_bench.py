#!/usr/bin/env python
"""Training-loader throughput of the reference's get_train_loader (train/dataloader.py) with the host TrainPre against the device path
of fasterseg_b200.trainpre, at the distillation driver's settings (1024 x 2048 Cityscapes-sized PNGs, 512 x 1024 crops, scales
0.75 / 1 / 1.25, batch 12) for 6 workers (config_train.py:62) and for every host core, and the distillation step
(tools/distill_step_bench.measure) fed by each loader at 6 workers.

Steady state: each DataLoader worker assembles a whole batch, so with w workers batches arrive in waves of w.  Every run is one
epoch of w x (1 + --waves) batches (the file list repeats, as BaseDataset's file_length does); the clock starts when the first wave
has arrived and the rate counts only the --waves waves after it, so neither worker start-up nor the prefetched first wave is in the
window.  Loader and step are measured over the same window, so the step's images/s can never exceed its loader's.  The arms
alternate, --runs runs each.  Needs the reference's dataloader / dataset modules: a checkout, or the copy __graft_entry__.build()
keeps in oracle/_ref.  Prints the card, its power limit, the host CPU and its core count, and one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fasterseg_b200 import trainpre  # noqa: E402
from oracle import make_golden_trainpre as G  # noqa: E402


def _card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e


def _cpu():
    try:
        out = subprocess.run(["lscpu"], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError):
        out = ""
    names = [ln.split(":", 1)[1].strip() for ln in out.splitlines() if ln.startswith(("Model name", "Vendor ID"))]
    return "%s, %d logical cores (%d usable by this process)" % (" / ".join(names) or "?", os.cpu_count(), len(os.sched_getaffinity(0)))


def write_pngs(root, n, seed=0):
    """n street-scene-sized pairs: a smooth image (a cubic upsample of coarse noise plus fine noise, ~4 MB as PNG) and a blocky label"""
    import cv2
    rs = np.random.RandomState(seed)
    lines = []
    for i in range(n):
        base = cv2.resize(rs.randint(0, 256, (64, 128, 3)).astype(np.uint8), (2048, 1024), interpolation=cv2.INTER_CUBIC)
        img = np.clip(base.astype(np.int16) + rs.randint(-6, 7, base.shape), 0, 255).astype(np.uint8)
        gt = cv2.resize(rs.randint(0, 19, (32, 64)).astype(np.uint8), (2048, 1024), interpolation=cv2.INTER_NEAREST)
        cv2.imwrite(os.path.join(root, "img%d.png" % i), img)
        cv2.imwrite(os.path.join(root, "gt%d.png" % i), gt)
        lines.append("img%d.png gt%d.png\n" % (i, i))
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.writelines(lines)


def make_loader(ns, datasets, root, n, workers, device, batches=None):
    cfg = G.Config(img_root_folder=root, gt_root_folder=root, train_source=os.path.join(root, "train.txt"),
                   eval_source=os.path.join(root, "train.txt"), down_sampling=1, image_height=512, image_width=1024,
                   train_scale_array=[0.75, 1, 1.25], gt_down_sampling=1, image_mean=np.array([0.485, 0.456, 0.406]),
                   image_std=np.array([0.229, 0.224, 0.225]), batch_size=12, niters_per_epoch=batches or n // 12, num_workers=workers)
    get = getattr(ns.dataloader.get_train_loader, "_fsb_original", ns.dataloader.get_train_loader)
    loader = get(cfg, datasets.Cityscapes)
    if device:
        loader = trainpre.wrap_loader(loader, ns.dataloader.TrainPre, trainpre.reference_base_dataset(ns.dataloader))
        assert isinstance(loader, trainpre.DeviceTrainLoader)
    return loader


def loader_rate(loader, workers):
    """steady-state images/s: batches after the first wave, over the time from the first wave's arrival to the last batch, each
    batch moved to the GPU as the drivers do (train.py:239-240)"""
    arrived = []
    for b in loader:
        b["data"].cuda(non_blocking=True)
        b["label"].cuda(non_blocking=True)
        torch.cuda.synchronize()
        arrived.append(time.perf_counter())
    return 12 * (len(arrived) - workers) / (arrived[-1] - arrived[workers - 1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=96)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workers", type=int, nargs="*", default=None, help="default: 6 and every usable core")
    ap.add_argument("--waves", type=int, default=4, help="timed waves of batches after the first (one batch per worker each)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "trainpre_bench measures on the GPU"
    workers = args.workers or sorted({6, len(os.sched_getaffinity(0))})
    print("card:", _card())
    print("host:", _cpu())
    ns, datasets = G.load_reference()
    root = tempfile.mkdtemp(prefix="fsb_trainpre_bench_")
    write_pngs(root, args.images)
    n = args.images - args.images % 12
    result = {"metric": "train_loader_images_per_s", "png_pairs": n, "batch": 12, "crop": [512, 1024], "source": [1024, 2048],
              "runs": args.runs, "waves": args.waves, "window": "steady state: the --waves waves after the first", "loader": {}}
    for w in workers:
        rates = {"reference": [], "device": []}
        for _ in range(args.runs):
            for arm in ("reference", "device"):
                loader = make_loader(ns, datasets, root, n, w, arm == "device", batches=w * (1 + args.waves))
                rates[arm].append(loader_rate(loader, w))
        result["loader"]["workers_%d" % w] = {arm: {"median": round(statistics.median(v), 1), "all": [round(r, 1) for r in v]}
                                              for arm, v in rates.items()}
        print(w, "workers:", json.dumps(result["loader"]["workers_%d" % w]), flush=True)

    from tools import distill_step_bench
    result["step"] = {}
    w = 6
    batches = w * (1 + args.waves)
    for arm in ("reference", "device"):
        # the loader's workers start at the first step, after the networks are built; the first wave also serves measure's two
        # warm-up steps
        loader = make_loader(ns, datasets, root, n, w, arm == "device", batches=batches)
        state = {"calls": []}

        def data():
            if "it" not in state:
                state["it"] = iter(loader)
            state["calls"].append(time.perf_counter())
            b = next(state["it"])
            return b["data"].cuda(non_blocking=True), b["label"].cuda(non_blocking=True)

        r = distill_step_bench.measure(steps=batches - 2, warmup=2, data=data)
        # the steps on batches w .. end, from the request for batch w (the first of the second wave) to the end of the last step
        # (measure synchronises after every step)
        rate = (batches - w) / (time.perf_counter() - state["calls"][w])
        result["step"][arm] = {"steps_per_s": round(rate, 2), "images_per_s": round(12 * rate, 1), "ms_per_step_median": r["value"],
                               "min_ms": r["min_ms"]}
        print("step fed by the", arm, "loader:", json.dumps(result["step"][arm]), flush=True)
        state.pop("it")
    r = distill_step_bench.measure(steps=16, warmup=2)
    result["step"]["synthetic_on_device"] = {"ms_per_step_median": r["value"], "steps_per_s": round(1e3 / r["value"], 2)}
    result["card"], result["host"] = _card(), _cpu()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
