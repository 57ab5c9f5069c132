"""TEST INFRASTRUCTURE ONLY -- loader for the *unmodified* reference (VITA-Group/FasterSeg).

This module exists so that `oracle/make_golden*.py` (run where a checkout of the reference is
available) can import the reference's own Python modules, run them on CPU fp32 and write golden
vectors to `tests/golden/`.  Nothing in the product path (`fasterseg_b200/`) imports it, and no
test depends on the reference tree: the tests read the stored goldens.

Why a harness is needed (SURVEY.md section 5 "compat list", section 8c):
  * `operations.py:12-17` computes `root_dir = abs_dir[:abs_dir.index('FasterSeg')...]`
    from `osp.realpath('.')` -> cwd must be a REAL directory whose path contains
    `FasterSeg`, so we work from a scratch copy `<tmp>/FasterSeg/`.
  * `thop`, `easydict`, `matplotlib`, `tensorboardX` are not installed -> stub modules.
  * `train/operations.py:36` / `train/seg_oprs.py:15` call `np.load` on a pickled dict
    without `allow_pickle` -> patched default.
  * `arch_*.pt` need `torch.load(weights_only=False)`.
  * `model_search.py:16` hard-codes `.cuda()` in `sample_gumbel` -> neutralised on CPU.
"""
from __future__ import annotations

import importlib
import os
import shutil
import sys
import tempfile
import types

# Where the reference checkout lives: $FASTERSEG_REFERENCE, else a directory `reference` next to this repository, else the verbatim
# copy that install_local_copy() (called by __graft_entry__.build()) keeps in the git-ignored oracle/_ref/FasterSeg, so that
# `bench.py --impl reference` and the cpu_baseline leg can time the UNMODIFIED reference on machines without the checkout.
_LOCAL_COPY = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "FasterSeg")
_SIBLING = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "..", "reference")
REFERENCE_ROOT = os.environ.get("FASTERSEG_REFERENCE") or (os.path.normpath(_SIBLING) if os.path.isdir(os.path.join(_SIBLING, "search"))
                                                          else _LOCAL_COPY)
_SCRATCH = None
_REF_MODULE_NAMES = (
    "operations", "slimmable_ops", "seg_oprs", "model_seg", "model_search", "genotypes",
    "architect", "utils", "utils.darts_utils", "utils.init_func", "seg_opr", "seg_opr.loss_opr",
    "engine", "engine.logger",
)


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "search"))


def _install_stubs() -> None:
    if "thop" not in sys.modules:
        thop = types.ModuleType("thop")
        thop.profile = lambda *a, **k: (0, 0)
        sys.modules["thop"] = thop
    if "easydict" not in sys.modules:
        ed = types.ModuleType("easydict")

        class EasyDict(dict):
            def __getattr__(self, k):
                try:
                    return self[k]
                except KeyError as e:
                    raise AttributeError(k) from e

            def __setattr__(self, k, v):
                self[k] = v

        ed.EasyDict = EasyDict
        sys.modules["easydict"] = ed
    try:
        import matplotlib  # noqa: F401
    except Exception:
        mpl = types.ModuleType("matplotlib")
        mpl.use = lambda *a, **k: None
        plt = types.ModuleType("matplotlib.pyplot")
        mpl.pyplot = plt
        sys.modules["matplotlib"] = mpl
        sys.modules["matplotlib.pyplot"] = plt
    if "tensorboardX" not in sys.modules:
        tb = types.ModuleType("tensorboardX")

        class SummaryWriter:  # pragma: no cover - never exercised
            def __init__(self, *a, **k):
                pass

            def __getattr__(self, name):
                return lambda *a, **k: None

        tb.SummaryWriter = SummaryWriter
        sys.modules["tensorboardX"] = tb


def install_local_copy() -> None:
    """Copy the reference checkout (without images) to oracle/_ref/FasterSeg once, if a checkout is available."""
    if REFERENCE_ROOT == _LOCAL_COPY or not reference_available() or os.path.isdir(os.path.join(_LOCAL_COPY, "search")):
        return
    os.makedirs(os.path.dirname(_LOCAL_COPY), exist_ok=True)
    shutil.copytree(REFERENCE_ROOT, _LOCAL_COPY, ignore=shutil.ignore_patterns("images", "*.png", "*.jpg", "*.gif", ".git"))


def scratch_copy() -> str:
    """Copy the reference tree to `<tmp>/FasterSeg` once per process and return that path."""
    global _SCRATCH
    if _SCRATCH is None:
        if not reference_available():
            raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
        base = tempfile.mkdtemp(prefix="fsb200_ref_")
        dst = os.path.join(base, "FasterSeg")
        shutil.copytree(REFERENCE_ROOT, dst, ignore=shutil.ignore_patterns("images", "*.png"))
        _SCRATCH = dst
    return _SCRATCH


class ReferenceNamespace:
    """Holds the reference modules imported with cwd = `<scratch>/<flavour>`."""

    def __init__(self, flavour: str):
        assert flavour in ("search", "train", "latency")
        self.flavour = flavour
        self.root = scratch_copy()
        self.dir = os.path.join(self.root, flavour)
        self.modules = {}

    def load(self, *names: str):
        import numpy as np
        import torch

        _install_stubs()
        for n in _REF_MODULE_NAMES:
            sys.modules.pop(n, None)
        old_cwd = os.getcwd()
        old_path = list(sys.path)
        old_np_load = np.load

        def np_load(*a, **k):
            k.setdefault("allow_pickle", True)
            return old_np_load(*a, **k)

        np.load = np_load
        try:
            os.chdir(self.dir)
            sys.path.insert(0, os.path.join(self.root, "tools"))
            sys.path.insert(0, self.dir)
            for n in names:
                self.modules[n] = importlib.import_module(n)
        finally:
            np.load = old_np_load
            os.chdir(old_cwd)
            sys.path[:] = old_path
            for n in _REF_MODULE_NAMES:
                sys.modules.pop(n, None)
        if "model_search" in self.modules and not torch.cuda.is_available():
            ms = self.modules["model_search"]

            def sample_gumbel(shape, eps=1e-20):  # model_search.py:14-17 minus `.cuda()`
                U = torch.rand(shape)
                return -torch.log(-torch.log(U + eps) + eps)

            ms.sample_gumbel = sample_gumbel
        return self

    def __getattr__(self, name):
        try:
            return self.__dict__["modules"][name]
        except KeyError as e:
            raise AttributeError(name) from e


def load_reference(flavour: str, *names: str) -> ReferenceNamespace:
    return ReferenceNamespace(flavour).load(*names)


def load_arch(idx: int):
    """`torch.load` of the shipped genotype `train/fasterseg/arch_{idx}.pt` (train.py:93-99)."""
    import torch

    return torch.load(os.path.join(REFERENCE_ROOT, "train", "fasterseg", "arch_%d.pt" % idx),
                      map_location="cpu", weights_only=False)


def build_reference_student(ns: ReferenceNamespace, arch_idx: int = 1, train_mode: bool = False,
                            lasts=None, stem_head_width=None):
    """Build `Network_Multi_Path_Infer` exactly as `train/train.py:95-118` does (arch_1 = student)."""
    import torch
    import torch.nn as nn

    state = load_arch(arch_idx)
    if stem_head_width is None:
        # config_train.py: C.stem_head_width = [(1, 1), (8./12, 8./12)]
        stem_head_width = (1.0, 1.0) if arch_idx == 0 else (8.0 / 12, 8.0 / 12)
    width_mult_list = [4. / 12, 6. / 12, 8. / 12, 10. / 12, 1.]
    Net = ns.model_seg.Network_Multi_Path_Infer
    model = Net(
        [state["alpha_%d_0" % arch_idx].detach(), state["alpha_%d_1" % arch_idx].detach(),
         state["alpha_%d_2" % arch_idx].detach()],
        [None, state["beta_%d_1" % arch_idx].detach(), state["beta_%d_2" % arch_idx].detach()],
        [state["ratio_%d_0" % arch_idx].detach(), state["ratio_%d_1" % arch_idx].detach(),
         state["ratio_%d_2" % arch_idx].detach()],
        num_classes=19, layers=16, Fch=12, width_mult_list=width_mult_list,
        stem_head_width=stem_head_width, ignore_skip=(arch_idx == 0))
    if lasts is None:
        # darts_utils.py:343-348 objective_acc_lat; train.py:101-104
        def obj(acc, lat, lat_target=8.3, alpha=-0.07, beta=-0.07):
            w = alpha if lat <= lat_target else beta
            return acc * (lat / lat_target) ** w
        lasts = [2, 0] if obj(state["mIoU02"], state["latency02"]) > obj(state["mIoU12"], state["latency12"]) else [2, 1]
    model.train(train_mode)
    model.build_structure(lasts)
    return model, state, lasts
