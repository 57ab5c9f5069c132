#!/usr/bin/env python
"""Training steps of the UNMODIFIED drivers, before and after the launcher's criterion / metric hooks (DESIGN section 3.9).

train.py arm: the reference's own train/train.py is imported from the copy that build() keeps in oracle/_ref/FasterSeg, as
`python -m fasterseg_b200.launch train.py` runs it (shadow modules, import hooks), and its own `train()` (train/train.py:219-271)
runs teacher arch_0 + student arch_1 (built as train.py:95-140 does, synthetic weights as bench.synth_weights_) on a
device-resident synthetic loader, so the loader is not measured.
  ref:     today's path without the hooks -- the reference's ProbOhemCrossEntropy2d.forward (argsort, two host syncs),
           Seg_Metrics.update on the host, label-resolution logits;
  patched: the launcher's hooks -- lazy logits, the fused OHEM / KL kernels, K9c for the per-step mIoU.
search arm: `_loss` + backward + clip + SGD step of the 16-layer supernet (tools/search_step_bench.py) with the reference's own
criterion, built as search/train_search.py:62-66 builds it, reference forward vs the patched one.
The paths alternate, `--runs` times each; median steps/s and peak memory per path.  The API step of tools/distill_step_bench.py
and the card's name, power limit and SM clock are recorded in the same call.  Prints one JSON line."""
import argparse
import contextlib
import importlib.util
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "oracle", "_ref", "FasterSeg")       # made by __graft_entry__.build(); the reference checkout is not read


def load_train_driver(root=REF):
    """import <root>/train/train.py as `python -m fasterseg_b200.launch train.py` runs it: compat patches, shadow modules, the
    criterion / metric hooks and the lazy-logits default, cwd = train/ (config_train.py derives its paths from it).  Stubs for
    easydict / tensorboardX / matplotlib where they are not installed.  Returns the module; `main()` is not run."""
    from fasterseg_b200 import launch
    from oracle import ref_harness
    ref_harness._install_stubs()
    launch.install_compat_patches()
    script = os.path.join(root, "train", "train.py")
    launch.install_shadow_modules(script)
    launch.install_criterion_patch(script)
    launch.install_train_metrics_patch(script)
    launch.install_lazy_logits_default(script)
    cwd = os.getcwd()
    # config_train.py adds <first ancestor named FasterSeg>/tools, which is another directory when a parent path also carries
    # that name: put this copy's tools/ first, as ref_harness does
    sys.path.insert(0, os.path.join(root, "tools"))
    sys.path.insert(0, os.path.dirname(script))
    os.chdir(os.path.dirname(script))
    try:
        spec = importlib.util.spec_from_file_location("fsb_train_driver", script)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        os.chdir(cwd)
    return mod


@contextlib.contextmanager
def loaded_train_driver(root=REF):
    """load_train_driver(root) for the duration of the block (tests): afterwards the modules it imported from `root` and the
    shadow names are gone again, and sys.path, sys.meta_path, the cwd and the lazy-logits default are as before"""
    from fasterseg_b200 import launch, model_seg
    modules, path, meta, cwd, lazy = dict(sys.modules), list(sys.path), list(sys.meta_path), os.getcwd(), model_seg.LAZY_LOGITS
    top = os.path.realpath(root) + os.sep
    try:
        yield load_train_driver(root)
    finally:
        for name, mod in list(sys.modules.items()):
            if name in launch.SHADOWED or os.path.realpath(getattr(mod, "__file__", None) or "/").startswith(top):
                del sys.modules[name]
        sys.modules.update(modules)
        sys.path[:], sys.meta_path[:] = path, meta
        os.chdir(cwd)
        model_seg.LAZY_LOGITS = lazy


@contextlib.contextmanager
def reference_path(driver):
    """today's path for a driver loaded by load_train_driver: the reference's criterion forward and metric update, and
    label-resolution logits"""
    from fasterseg_b200 import model_seg
    crit, metrics = driver.ProbOhemCrossEntropy2d, driver.seg_metrics.Seg_Metrics
    patched = crit.forward, metrics.update, model_seg.LAZY_LOGITS
    crit.forward, metrics.update, model_seg.LAZY_LOGITS = crit.forward._fsb_original, metrics.update._fsb_original, False
    try:
        yield
    finally:
        crit.forward, metrics.update, model_seg.LAZY_LOGITS = patched


class SyntheticLoader:
    """device-resident batches in the reference loader's format; its iterator has the `.next()` train.py:237 calls"""

    def __init__(self, batch, hw, steps, device="cuda", seed=0):
        g = torch.Generator().manual_seed(seed)
        self.data = torch.randn(batch, 3, hw[0], hw[1], generator=g).to(device)
        label = torch.randint(0, 19, (batch,) + tuple(hw), generator=g)
        label[torch.rand(label.shape, generator=g) < 0.05] = 255
        self.label = label.to(device)
        self.steps = steps

    def __len__(self):
        return self.steps

    def __iter__(self):
        return self

    def next(self):
        return {"data": self.data, "label": self.label, "fn": [""] * self.data.shape[0], "n": self.data.shape[0]}

    __next__ = next


class NullWriter:
    def add_scalar(self, *a, **k):
        pass


def build_driver_models(device="cuda"):
    """[teacher arch_0, student arch_1] as train.py:95-140 builds them, with synthetic weights"""
    from bench import synth_weights_
    from fasterseg_b200 import zoo
    teacher = zoo.build_network(0)
    synth_weights_(teacher, 1)
    student = zoo.build_network(1, training=True)
    synth_weights_(student, 2)
    return [teacher.to(device), student.to(device)]


def driver_criteria(driver, batch, hw):
    """the criteria of train.py:62-64"""
    cfg = driver.config
    min_kept = int(batch * hw[0] * hw[1] // (16 * cfg.gt_down_sampling ** 2))
    return driver.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False), nn.KLDivLoss()


def run_train(driver, models, optimizer, loader, criteria, steps):
    """train.py's own train() for `steps` steps, its progress bar on stderr; -> (seconds, per-model train mIoU)"""
    driver.config.niters_per_epoch = steps
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(sys.stderr):
        mious = driver.train(loader, models, criteria[0], criteria[1], optimizer, NullWriter(), 0)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, [float(m) for m in mious]


def train_arm(driver, batch, hw, steps, warmup, runs):
    models = build_driver_models()
    optimizer = torch.optim.SGD(models[1].parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
    loader = SyntheticLoader(batch, hw, steps)
    criteria = driver_criteria(driver, batch, hw)
    paths = {"ref": lambda: reference_path(driver), "patched": contextlib.nullcontext}
    out = {p: {"steps_per_s": [], "peak_GB": []} for p in paths}
    for name, ctx in paths.items():
        with ctx():
            run_train(driver, models, optimizer, loader, criteria, warmup)
    for _ in range(runs):
        for name, ctx in paths.items():
            with ctx():
                torch.cuda.reset_peak_memory_stats()
                dt, mious = run_train(driver, models, optimizer, loader, criteria, steps)
            out[name]["steps_per_s"].append(round(steps / dt, 3))
            out[name]["peak_GB"].append(round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
            out[name]["train_mIoU"] = mious
    return out


def search_arm(driver, mode, steps, warmup, runs):
    """tools/search_step_bench.py's step with the reference's criterion (search/train_search.py:62-66)"""
    from fasterseg_b200 import optim as FO
    from tools import search_step_bench as SB
    FO.install()
    torch.manual_seed(12345)
    B, H, W = (3, 256, 512) if mode == "pretrain" else (2, 224, 448)
    gt_down = 8                                                   # config_search.py: the supernet's loss is at 1/8 resolution
    crit = driver.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=int(B * H * W // (16 * gt_down ** 2)),
                                         use_weight=False)
    model = SB.build(16, "ce")
    model._criterion = crit
    opt = torch.optim.SGD(SB.weight_params(model), lr=0.02, momentum=0.9, weight_decay=5e-4)
    g = torch.Generator().manual_seed(977)
    x = torch.randn(B, 3, H, W, generator=g).cuda()
    t = torch.randint(0, 19, (B, H // gt_down, W // gt_down), generator=g)
    t[torch.rand(t.shape, generator=g) < 0.05] = 255
    t = t.cuda()
    cls = type(crit)
    forwards = {"ref": cls.forward._fsb_original, "patched": cls.forward}

    def steps_of(n):
        for _ in range(n):
            opt.zero_grad()
            loss = model._loss(x, t, True if mode == "pretrain" else "dir")
            loss.backward()
            nn.utils.clip_grad_norm_(model.parameters(), 5)
            opt.step()

    out = {p: {"steps_per_s": [], "peak_GB": []} for p in forwards}
    try:
        for name, fwd in forwards.items():
            cls.forward = fwd
            steps_of(warmup)
        for _ in range(runs):
            for name, fwd in forwards.items():
                cls.forward = fwd
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                steps_of(steps)
                torch.cuda.synchronize()
                out[name]["steps_per_s"].append(round(steps / (time.perf_counter() - t0), 3))
                out[name]["peak_GB"].append(round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
    finally:
        cls.forward = forwards["patched"]
        FO.uninstall()
    out["batch"] = [B, 3, H, W]
    return out


def summarise(arm):
    for p in ("ref", "patched"):
        r = arm[p]
        v = sorted(r["steps_per_s"])
        r["median_steps_per_s"] = v[len(v) // 2]
        r["peak_GB_max"] = max(r["peak_GB"])
    arm["speedup"] = round(arm["patched"]["median_steps_per_s"] / arm["ref"]["median_steps_per_s"], 2)
    return arm


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (v.strip() for v in line.split(","))))
    except Exception as e:  # noqa: BLE001 -- recorded, not fatal
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=12)
    ap.add_argument("--hw", type=int, nargs=2, default=[512, 1024])
    ap.add_argument("--steps", type=int, default=None, help="steps per timed run (default: config.niters_per_epoch)")
    ap.add_argument("--search-steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("driver_step_bench: needs a CUDA device")
    if not os.path.isfile(os.path.join(REF, "train", "train.py")):
        raise SystemExit("driver_step_bench: no copy of the reference in %s (made by __graft_entry__.build())" % REF)
    driver = load_train_driver()
    steps = args.steps or int(driver.config.niters_per_epoch)
    res = {"gpu": gpu_info(), "train_py": summarise(train_arm(driver, args.batch, tuple(args.hw), steps, args.warmup, args.runs))}
    res["train_py"].update(batch=[args.batch, 3] + list(args.hw), steps_per_run=steps, runs=args.runs)
    for mode in ("pretrain", "search"):
        res["search_" + mode] = summarise(search_arm(driver, mode, args.search_steps, args.warmup, args.runs))
    from tools import distill_step_bench
    res["api_distill_step"] = distill_step_bench.measure(args.batch, tuple(args.hw))
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
