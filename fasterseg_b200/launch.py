"""Run an UNMODIFIED reference driver (search/train_search.py, train/train.py, latency/run_latency.py) on the H100 (sm_90a) path.

    cd <FasterSeg>/search && python -m fasterseg_b200.launch train_search.py
    torchrun --nproc-per-node 8 -m fasterseg_b200.launch train_search.py        # data parallel
    cd <FasterSeg>/latency && python -m fasterseg_b200.launch run_latency.py

The reference resolves `operations`, `slimmable_ops`, `seg_oprs`, `model_seg`, `model_search`, `genotypes` from the script's
directory (search/model_search.py:4-9, train/train.py:32); registering our modules under those names in `sys.modules` BEFORE the
script imports them swaps the whole L1/L2 layer with zero script edits (SURVEY section 8b).  The three directories hold
different copies: for a script in a directory named `latency`, `operations` and `model_seg` are the latency/ deployment
network (fasterseg_b200.latency_variant: nearest resizes, single-conv stride-2 FactorizedReduce) that run_latency.py builds and
times; every other directory gets the train/ modules.  The shim also applies the
py3.12 / torch 2.x compat patches the old scripts need (SURVEY section 5 "compat list") and, under torchrun, the
data-parallel hooks of `fasterseg_b200.parallel`.
"""
from __future__ import annotations

import importlib
import os
import runpy
import sys
import types

SHADOWED = ("genotypes", "slimmable_ops", "operations", "seg_oprs", "model_seg", "model_search")


LATENCY_VARIANT = ("operations", "model_seg")   # modules of latency/ that differ from train/


def shadow_module_names(script=None):
    """{module name the script imports: our module} -- the latency/ variant for a script whose directory is named `latency`"""
    latency = script is not None and os.path.basename(os.path.dirname(os.path.abspath(script))) == "latency"
    return {name: "fasterseg_b200." + ("latency_variant." + name if latency and name in LATENCY_VARIANT else name)
            for name in SHADOWED}


def install_shadow_modules(script=None):
    for name, target in shadow_module_names(script).items():
        sys.modules[name] = importlib.import_module(target)
    return [sys.modules[n] for n in SHADOWED]


def install_compat_patches():
    import numpy as np
    import torch
    # `dataloader.next()` (train_search.py:226,235; train.py:237)
    from torch.utils.data.dataloader import _BaseDataLoaderIter
    if not hasattr(_BaseDataLoaderIter, "next"):
        _BaseDataLoaderIter.next = _BaseDataLoaderIter.__next__
    # pickled dicts / genotype files
    if not getattr(np.load, "_fsb_patched", False):
        orig = np.load

        def load(*a, **k):
            k.setdefault("allow_pickle", True)
            return orig(*a, **k)

        load._fsb_patched = True
        np.load = load
    if not getattr(torch.load, "_fsb_patched", False):
        torig = torch.load

        def tload(*a, **k):
            k.setdefault("weights_only", False)
            return torig(*a, **k)

        tload._fsb_patched = True
        torch.load = tload
    import collections
    import collections.abc
    for n in ("Iterable", "Mapping", "Sequence"):
        if not hasattr(collections, n):
            setattr(collections, n, getattr(collections.abc, n))
    for name, attrs in (("thop", {"profile": lambda *a, **k: (0, 0)}),):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except ImportError:
                m = types.ModuleType(name)
                m.__dict__.update(attrs)
                sys.modules[name] = m


class RankShardSampler:
    """Sampler the launcher gives every training DataLoader under torchrun: one permutation of the dataset per epoch drawn from a
    PRIVATE generator that is identical on all ranks (so the global torch / numpy RNG streams -- width sampling, gumbel noise --
    stay in lock-step), of which this rank takes every world-th index: the ranks see disjoint shards of
    the same shuffle, like DistributedSampler, without the script knowing."""

    def __init__(self, data_source, rank, world, shuffle=True, seed=12345):
        self.n, self.rank, self.world, self.shuffle, self.seed, self.epoch = len(data_source), rank, world, shuffle, seed, 0

    def __iter__(self):
        import torch
        if self.shuffle:
            g = torch.Generator()
            g.manual_seed(self.seed + self.epoch)
            order = torch.randperm(self.n, generator=g).tolist()
        else:
            order = list(range(self.n))
        self.epoch += 1
        per = self.n // self.world
        return iter(order[self.rank::self.world][:per])

    def __len__(self):
        return self.n // self.world


def install_rank_sharded_loaders(rank, world):
    """Patch torch.utils.data.DataLoader so that every loader the unmodified script builds with `shuffle=True` or a RandomSampler /
    SequentialSampler over a map-style dataset iterates this rank's shard only (ADVICE round 1: without it every rank saw the same
    batches and N GPUs computed one gradient N times)."""
    import torch.utils.data as tud
    if getattr(tud.DataLoader, "_fsb_sharded", False):
        return
    orig_init = tud.DataLoader.__init__

    def init(self, dataset, *a, **k):
        names = ("batch_size", "shuffle", "sampler", "batch_sampler")
        args = dict(zip(names, a))
        args.update({n: k[n] for n in names if n in k})
        explicit = args.get("sampler") is not None or args.get("batch_sampler") is not None
        if not explicit and hasattr(dataset, "__len__") and not isinstance(dataset, tud.IterableDataset):
            shuffle = bool(args.get("shuffle", False))
            a = a[:1] + (False,) + a[2:] if len(a) >= 2 else a      # positional shuffle -> False
            k.pop("shuffle", None)
            if len(a) >= 3:
                a = a[:2] + (RankShardSampler(dataset, rank, world, shuffle),) + a[3:]
            else:
                k["sampler"] = RankShardSampler(dataset, rank, world, shuffle)
        orig_init(self, dataset, *a, **k)

    tud.DataLoader.__init__ = init
    tud.DataLoader._fsb_sharded = True


def install_rank0_side_effects(rank):
    """Non-zero ranks must not race rank 0 on the experiment directory: `os.mkdir(path/'scripts')` in the drivers' create_exp_dir
    raises FileExistsError on the second rank, and every rank would write checkpoints / arch_*.pt / tensorboard logs into the same
    place.  On ranks > 0: directory creation tolerates existing paths, torch.save and np.save-style checkpointing are dropped and
    SummaryWriter-like loggers become no-ops."""
    import os as _os
    import torch
    orig_mkdir, orig_makedirs = _os.mkdir, _os.makedirs

    def mkdir(path, *a, **k):
        try:
            return orig_mkdir(path, *a, **k)
        except FileExistsError:
            return None

    def makedirs(path, *a, **k):
        k["exist_ok"] = True
        return orig_makedirs(path, *a, **k)

    _os.mkdir, _os.makedirs = mkdir, makedirs     # all ranks: creation is idempotent (rank 0 may come second)
    if rank == 0:
        return
    torch.save = lambda *a, **k: None

    class _NullWriter:
        def __init__(self, *a, **k):
            pass

        def __getattr__(self, name):
            return lambda *a, **k: None

    import importlib
    for mod in ("tensorboardX", "torch.utils.tensorboard"):
        try:
            m = importlib.import_module(mod)
            m.SummaryWriter = _NullWriter
        except Exception:  # noqa: BLE001 -- the module may be absent; the drivers import it lazily
            pass


def discover_parameters():
    """Parameters of every nn.Module the script has built, in a DETERMINISTIC order that is identical on all ranks: top-level modules
    (those that are no other module's child) sorted by class name and parameter count, then `named_parameters()` order -- not
    `gc.get_objects()` order, which is an address-dependent heap walk."""
    import gc
    import torch
    mods = [o for o in gc.get_objects() if isinstance(o, torch.nn.Module)]
    children = {id(c) for m in mods for c in m.children()}
    tops = [m for m in mods if id(m) not in children]
    tops.sort(key=lambda m: (type(m).__name__, sum(p.numel() for p in m.parameters()), len(list(m.parameters()))))
    seen, params, names = set(), [], []
    for ti, m in enumerate(tops):
        for name, p in m.named_parameters():
            if id(p) not in seen and p.requires_grad:
                seen.add(id(p))
                params.append(p)
                names.append("%d:%s:%s" % (ti, type(m).__name__, name))
    return params, names


def install_data_parallel():
    """Under torchrun: NCCL process group, SyncBN statistics, rank-sharded data loaders, rank-0-only side effects, and the gradient
    all-reduce at the end of every backward for all parameters of every nn.Module the script builds (registered lazily at the first
    backward, in a deterministic order whose NAMES are hashed into the handshake)."""
    from . import parallel
    rank, local_rank, world = parallel.init_from_env()
    if world == 1:
        return None
    parallel.seed_all_ranks_identically()
    install_rank_sharded_loaders(rank, world)
    install_rank0_side_effects(rank)

    class _Lazy(parallel.GradSync):
        def sync(self):
            if not self.params:
                params, names = discover_parameters()
                self.params.extend(params)
                self.set_names(names)
            super().sync()

    return _Lazy([]).install()


def reference_tools_dir(script):
    """<FasterSeg>/tools for a driver at <FasterSeg>/<dir>/<script>.py (config_*.py puts the same directory on sys.path), or None"""
    tools = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(script))), "tools")
    return tools if os.path.isfile(os.path.join(tools, "engine", "evaluator.py")) else None


class _PatchAfterImport:
    """sys.meta_path finder: when `name` is imported from `origin`, loads it with its own loader and then calls patch(module)"""

    def __init__(self, name, origin, patch):
        self.name, self.origin, self.patch = name, os.path.realpath(origin), patch

    def find_spec(self, fullname, path=None, target=None):
        if fullname != self.name:
            return None
        from importlib.machinery import PathFinder
        spec = PathFinder.find_spec(fullname, path)
        if spec is None or spec.origin is None or os.path.realpath(spec.origin) != self.origin:
            return None
        spec.loader = _PatchingLoader(spec.loader, self.patch)
        return spec


class _PatchingLoader:
    def __init__(self, loader, patch):
        self.loader, self.patch = loader, patch

    def create_module(self, spec):
        return self.loader.create_module(spec)

    def exec_module(self, module):
        self.loader.exec_module(module)
        self.patch(module)


def install_evaluator_patch(script):
    """Validation on the device (fasterseg_b200.evaluator): when the driver imports the reference's engine.evaluator from the
    tools/ directory next to its own, patch Evaluator.run_online / run_online_multiprocess.  Returns the finder, or None (and
    changes nothing) when no reference tools/ directory is found."""
    tools = reference_tools_dir(script)
    if tools is None:
        return None
    from . import evaluator
    finder = _PatchAfterImport("engine.evaluator", os.path.join(tools, "engine", "evaluator.py"), evaluator.install)
    sys.meta_path.insert(0, finder)
    return finder


def install_tester_patch(script):
    """Test-set prediction on the device (fasterseg_b200.tester): when the driver imports the reference's engine.tester from the
    tools/ directory next to its own (train.py:29 via train/test.py:17), patch Tester.run_online / run_online_multiprocess.
    Returns the finder, or None (and changes nothing) when there is no such tools/engine/tester.py."""
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(script))), "tools", "engine", "tester.py")
    if not os.path.isfile(path):
        return None
    from . import tester
    finder = _PatchAfterImport("engine.tester", path, tester.install)
    sys.meta_path.insert(0, finder)
    return finder


def install_dataloader_patch(script):
    """Training augmentation on the device (fasterseg_b200.trainpre): when the driver imports the `dataloader` module next to it
    (train/dataloader.py, search/dataloader.py), wrap its get_train_loader.  Returns the finder, or None (and changes nothing)
    when the script's directory has no dataloader.py."""
    path = os.path.join(os.path.dirname(os.path.abspath(script)), "dataloader.py")
    if not os.path.isfile(path):
        return None
    from . import trainpre
    finder = _PatchAfterImport("dataloader", path, trainpre.install)
    sys.meta_path.insert(0, finder)
    return finder


def install_criterion_patch(script):
    """Training criterion without host syncs (losses.install_reference_ohem): when the driver imports the reference's
    seg_opr.loss_opr from the tools/ directory next to its own (train.py:27, train_search.py), patch
    ProbOhemCrossEntropy2d.forward.  Returns the finder, or None (and changes nothing) when no reference tools/ directory is
    found."""
    tools = reference_tools_dir(script)
    if tools is None:
        return None
    from . import losses
    finder = _PatchAfterImport("seg_opr.loss_opr", os.path.join(tools, "seg_opr", "loss_opr.py"), losses.install_reference_ohem)
    sys.meta_path.insert(0, finder)
    return finder


def install_train_metrics_patch(script):
    """Per-step training mIoU on the device (fasterseg_b200.train_metrics): when the driver imports the `seg_metrics` module
    next to it (train/seg_metrics.py), patch Seg_Metrics.update.  Returns the finder, or None (and changes nothing) when the
    script's directory has no seg_metrics.py."""
    path = os.path.join(os.path.dirname(os.path.abspath(script)), "seg_metrics.py")
    if not os.path.isfile(path):
        return None
    from . import train_metrics
    finder = _PatchAfterImport("seg_metrics", path, train_metrics.install)
    sys.meta_path.insert(0, finder)
    return finder


def install_lazy_logits_default(script):
    """Every train/ Network_Multi_Path_Infer the driver builds returns losses.LazyLogits (an instance's own `lazy_logits` still
    wins): the patched criteria and metric take them without materialising label-resolution logits.  Not for the latency/
    variant, which has no lazy path.  Returns whether the default was switched on."""
    if "latency_variant" in shadow_module_names(script)["model_seg"]:
        return False
    from . import model_seg
    model_seg.LAZY_LOGITS = True
    return True


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        raise SystemExit("usage: python -m fasterseg_b200.launch <reference_script.py> [args...]")
    from . import _lib
    _lib.lib()  # fail loudly up front if the native library has not been built
    script = argv[0]
    install_compat_patches()
    install_shadow_modules(script)
    install_data_parallel()
    install_evaluator_patch(script)
    install_tester_patch(script)
    install_dataloader_patch(script)
    install_criterion_patch(script)
    install_train_metrics_patch(script)
    install_lazy_logits_default(script)
    from . import optim
    optim.install()      # torch.optim.SGD / nn.utils.clip_grad_norm_ take the flat path after a captured `_loss` (torch's otherwise)
    sys.argv = argv
    sys.path.insert(0, os.path.dirname(os.path.abspath(script)) or ".")
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main()
