"""The drivers' training step on the fused criteria without a GPU: the launcher's hooks on the reference's
seg_opr.loss_opr (losses.install_reference_ohem) and train/seg_metrics.py (train_metrics.install), the lazy-logits default, which
path the patched criterion takes, the per-step mIoU counters against the reference's own Seg_Metrics (tests/golden/seg_metrics.json),
LazyLogits.data / __getitem__, and train.py's own train() on the CPU stand-in backend where a copy of the reference is available.
The kernels themselves: tests/test_driver_train_gpu.py."""
import json
import os
import sys
import textwrap
import types

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from fasterseg_b200 import autograd as AG
from fasterseg_b200 import functional as F_
from fasterseg_b200 import launch, losses, model_seg, train_metrics
from fasterseg_b200.losses import LazyLogits
from oracle import make_golden_seg_metrics as G
from tests import cpu_backend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "seg_metrics.json")))
HOOKED = ("seg_opr", "seg_opr.loss_opr", "seg_metrics")


# ---- launcher hooks ------------------------------------------------------------------------------------------------------------------
_STUB_LOSS_OPR = textwrap.dedent('''
    class ProbOhemCrossEntropy2d(object):
        def forward(self, pred, target):
            return "stub"
''')
_STUB_SEG_METRICS = textwrap.dedent('''
    class Seg_Metrics(object):
        def update(self, pred, target):
            return "stub"
''')


def _fake_checkout(base, flavour="train"):
    root = base / "FasterSeg"
    (root / flavour).mkdir(parents=True)
    (root / flavour / "script.py").write_text("")
    (root / flavour / "seg_metrics.py").write_text(_STUB_SEG_METRICS)
    eng, seg = root / "tools" / "engine", root / "tools" / "seg_opr"
    eng.mkdir(parents=True)
    seg.mkdir(parents=True)
    (eng / "__init__.py").write_text("")
    (eng / "evaluator.py").write_text("")
    (seg / "__init__.py").write_text("")
    (seg / "loss_opr.py").write_text(_STUB_LOSS_OPR)
    return str(root / flavour / "script.py"), str(root / "tools"), str(root / flavour)


@pytest.fixture
def clean_import_state():
    path, meta, lazy = list(sys.path), list(sys.meta_path), model_seg.LAZY_LOGITS
    saved = {n: sys.modules[n] for n in HOOKED if n in sys.modules}
    for n in HOOKED:
        sys.modules.pop(n, None)
    yield
    sys.path[:] = path
    sys.meta_path[:] = meta
    model_seg.LAZY_LOGITS = lazy
    for n in HOOKED:
        sys.modules.pop(n, None)
    sys.modules.update(saved)


def _import_hooked(tools, script_dir):
    sys.path.insert(0, tools)
    sys.path.insert(0, script_dir)
    import seg_metrics
    import seg_opr.loss_opr
    return seg_opr.loss_opr, seg_metrics


def test_launcher_patches_the_reference_criterion_and_metric_in_place(tmp_path, clean_import_state):
    script, tools, script_dir = _fake_checkout(tmp_path)
    assert launch.install_criterion_patch(script) is not None and launch.install_train_metrics_patch(script) is not None
    loss_opr, seg_metrics = _import_hooked(tools, script_dir)
    crit, metrics = loss_opr.ProbOhemCrossEntropy2d, seg_metrics.Seg_Metrics
    assert crit.forward._fsb_original is not None and crit.forward.__name__ == "forward"
    assert metrics.update._fsb_original is not None and metrics.update.__name__ == "update"
    assert losses.install_reference_ohem(loss_opr).forward is crit.forward          # idempotent: no double wrapping
    assert train_metrics.install(seg_metrics).update is metrics.update


def test_modules_of_the_same_name_from_elsewhere_are_untouched(tmp_path, clean_import_state):
    script, _, _ = _fake_checkout(tmp_path / "a")
    _, other_tools, other_dir = _fake_checkout(tmp_path / "b")
    launch.install_criterion_patch(script)
    launch.install_train_metrics_patch(script)
    loss_opr, seg_metrics = _import_hooked(other_tools, other_dir)
    assert not hasattr(loss_opr.ProbOhemCrossEntropy2d.forward, "_fsb_original")
    assert not hasattr(seg_metrics.Seg_Metrics.update, "_fsb_original")


def test_hooks_change_nothing_without_the_reference_files(tmp_path, clean_import_state):
    (tmp_path / "x").mkdir()
    script = str(tmp_path / "x" / "script.py")
    meta = list(sys.meta_path)
    assert launch.install_criterion_patch(script) is None and launch.install_train_metrics_patch(script) is None
    assert sys.meta_path == meta


def test_lazy_logits_default_for_train_drivers_only(tmp_path, clean_import_state):
    assert model_seg.LAZY_LOGITS is False                          # programs that build the network themselves
    latency, _, _ = _fake_checkout(tmp_path / "l", "latency")
    assert launch.install_lazy_logits_default(latency) is False and model_seg.LAZY_LOGITS is False
    train, _, _ = _fake_checkout(tmp_path / "t", "train")
    assert launch.install_lazy_logits_default(train) is True and model_seg.LAZY_LOGITS is True


def test_lazy_default_reaches_the_network_and_an_instance_setting_wins(clean_import_state):
    from tests.test_boundary_cpu import _build_student
    net, _ = _build_student(1)
    x = torch.randn(1, 3, 64, 128)
    with cpu_backend.installed(), torch.no_grad():
        assert isinstance(net(x), torch.Tensor)
        model_seg.LAZY_LOGITS = True
        out = net(x)
        assert isinstance(out, LazyLogits) and out.size == (64, 128)
        net.lazy_logits = False
        assert isinstance(net(x), torch.Tensor)


# ---- criterion dispatch ------------------------------------------------------------------------------------------------------------
class _RefOhem(nn.Module):
    """the attributes of tools/seg_opr/loss_opr.py:43-61's class; forward records what it was called with"""

    def __init__(self, ignore_label=255, reduction="mean", thresh=0.7, min_kept=100, use_weight=False):
        super().__init__()
        self.ignore_label, self.thresh, self.min_kept, self.down_ratio = ignore_label, float(thresh), int(min_kept), 1
        weight = torch.rand(19) if use_weight else None
        self.criterion = nn.CrossEntropyLoss(reduction=reduction, weight=weight, ignore_index=ignore_label)
        self.calls = []

    def forward(self, pred, target):
        self.calls.append(pred)
        return torch.tensor(7.0)


@pytest.fixture
def rig(monkeypatch):
    calls = []
    monkeypatch.setattr(model_seg, "_upsample_logits",
                        lambda x, size, dtype: F.interpolate(x.float(), size=size, mode="bilinear", align_corners=True).to(dtype))
    monkeypatch.setattr(AG, "fused_ohem_ce", lambda *a: calls.append(a) or torch.tensor(2.5))
    monkeypatch.setattr(_RefOhem, "forward", _RefOhem.forward)       # the patch below is undone with the class attribute
    losses.install_reference_ohem(types.SimpleNamespace(ProbOhemCrossEntropy2d=_RefOhem))
    g = torch.Generator().manual_seed(0)
    low = torch.randn(2, 19, 4, 8, generator=g)
    tgt = torch.randint(0, 19, (2, 32, 64), generator=g)
    tgt[0, :3] = 255
    return calls, low, tgt


def test_lazy_logits_take_the_fused_kernels(rig):
    calls, low, tgt = rig
    crit = _RefOhem(thresh=0.7, min_kept=100)
    assert float(crit(LazyLogits(low, (32, 64)), tgt)) == 2.5
    assert not crit.calls and len(calls) == 1
    assert calls[0][0] is low and calls[0][1] is tgt and calls[0][2:] == ((32, 64), 255, 0.7, 100)


def test_dense_logits_take_the_sync_free_restatement(rig):
    calls, low, tgt = rig
    dense = F.interpolate(low, size=(32, 64), mode="bilinear", align_corners=True)
    crit = _RefOhem(thresh=0.7, min_kept=100)
    got = crit(dense, tgt)
    want = losses.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=100)(dense, tgt)
    assert not crit.calls and not calls and float(got) == float(want)


@pytest.mark.parametrize("kw", [dict(use_weight=True), dict(reduction="sum"), dict(reduction="none")])
def test_weights_or_another_reduction_run_the_reference_forward_on_materialised_logits(rig, kw):
    calls, low, tgt = rig
    crit = _RefOhem(**kw)
    assert float(crit(LazyLogits(low, (32, 64)), tgt)) == 7.0
    dense = F.interpolate(low, size=(32, 64), mode="bilinear", align_corners=True)
    assert float(crit(dense, tgt)) == 7.0
    assert not calls and len(crit.calls) == 2
    assert torch.equal(crit.calls[0], dense) and crit.calls[1] is dense


# ---- per-step mIoU: counters -> (inter, union) ----------------------------------------------------------------------------------------
def _upsample_argmax_confusion(x, size, gt, n_cl, out):
    """stand-in: the two-kernel composition the fused kernel is bit-identical to"""
    return cpu_backend.confusion_matrix(cpu_backend.upsample_argmax(x, size), gt, n_cl, out)


@pytest.fixture
def device_metric(monkeypatch):
    monkeypatch.setattr(train_metrics, "_on_device", lambda x, target: True)
    monkeypatch.setattr(F_, "upsample_argmax_confusion", _upsample_argmax_confusion)


class _Metrics:
    """Seg_Metrics' state (train/seg_metrics.py:6-9); the original update must not be reached"""

    def __init__(self, n_classes):
        self.n_classes = n_classes
        self.total_inter, self.total_union = np.zeros(n_classes), np.zeros(n_classes)

    def update(self, pred, target):
        raise AssertionError("reference update reached")


def _lowres(logits):
    N, C, H, W = logits.shape
    buf = F_.empty_nhwc(N, C, H, W, "cpu")
    buf.copy_(torch.from_numpy(logits).half())
    return buf


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_counters_give_the_reference_intersection_and_union(name):
    n = G.CASES[name][1]
    for (logits, target), want in zip(G.inputs(name), GOLDEN[name]):
        hist = cpu_backend.confusion_matrix(torch.from_numpy(logits.argmax(1)).to(torch.uint8), torch.from_numpy(target), n)
        inter, union = train_metrics.inter_union(hist[:n * n].reshape(n, n).numpy())
        assert inter.tolist() == want["inter"] and union.tolist() == want["union"]


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_patched_update_accumulates_the_reference_totals(name, device_metric, monkeypatch):
    monkeypatch.setattr(_Metrics, "update", _Metrics.update)
    train_metrics.install(types.SimpleNamespace(Seg_Metrics=_Metrics))
    n = G.CASES[name][1]
    m = _Metrics(n)
    for (logits, target), want in zip(G.inputs(name), GOLDEN[name]):
        m.update(LazyLogits(_lowres(logits), target.shape[1:]).data, torch.from_numpy(target))
        assert m.total_inter.tolist() == want["total_inter"] and m.total_union.tolist() == want["total_union"]


def test_ineligible_inputs_run_the_reference_update(device_metric, monkeypatch):
    seen = []
    monkeypatch.setattr(_Metrics, "update", lambda self, pred, target: seen.append(pred))
    train_metrics.install(types.SimpleNamespace(Seg_Metrics=_Metrics))
    logits, target = G.inputs("camvid_11")[0]
    lazy = LazyLogits(_lowres(logits), target.shape[1:])
    t = torch.from_numpy(target)
    for pred, tgt, n in ((torch.from_numpy(logits), t, 11), (lazy, t, 19), (lazy, t[:, :4], 11), (lazy, t.to(torch.int16), 11)):
        _Metrics(n).update(pred, tgt)
    assert len(seen) == 4
    monkeypatch.setattr(train_metrics, "_on_device", lambda x, target: False)
    _Metrics(11).update(lazy, t)
    assert len(seen) == 5


# ---- LazyLogits additions ----------------------------------------------------------------------------------------------------------
def test_lazy_logits_data_and_indexing(monkeypatch):
    monkeypatch.setattr(model_seg, "_upsample_logits",
                        lambda x, size, dtype: F.interpolate(x.float(), size=size, mode="bilinear", align_corners=True).to(dtype))
    low = torch.randn(2, 19, 4, 8, requires_grad=True)
    lazy = LazyLogits(low, (32, 64))
    d = lazy.data
    assert isinstance(d, LazyLogits) and d.size == (32, 64) and not d.lowres.requires_grad and torch.equal(d.lowres, low)
    dense = F.interpolate(low.detach(), size=(32, 64), mode="bilinear", align_corners=True)
    assert torch.equal(lazy[0], dense[0]) and torch.equal(lazy[1, 3], dense[1, 3])    # tools/engine/evaluator.py:308 `score[0]`


# ---- train.py's own train() on the CPU stand-in ------------------------------------------------------------------------------------
@pytest.fixture
def driver(monkeypatch):
    from tools import driver_step_bench as D
    if not os.path.isfile(os.path.join(D.REF, "train", "train.py")):
        pytest.skip("no copy of the reference in oracle/_ref")
    with D.loaded_train_driver() as drv:
        yield D, drv


class _Writer:
    def __init__(self):
        self.losses = []

    def add_scalar(self, tag, value, step):
        self.losses.append(float(value.detach()))


def _run(D, drv, steps, batch=2, hw=(64, 128)):
    from bench import synth_weights_
    from tests.test_boundary_cpu import _build_student
    teacher, _ = _build_student(0)
    synth_weights_(teacher, 1)
    student, _ = _build_student(1, training=True)
    synth_weights_(student, 2)
    opt = torch.optim.SGD(student.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
    ohem, kl = D.driver_criteria(drv, batch, hw)
    drv.config.niters_per_epoch = steps
    writer = _Writer()
    mious = drv.train(D.SyntheticLoader(batch, hw, steps, device="cpu"), [teacher, student], ohem, kl, opt, writer, 0)
    return [float(m) for m in mious], writer.losses


def test_train_py_steps_through_both_paths(driver, device_metric, monkeypatch):
    D, drv = driver
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)
    dense_update = drv.seg_metrics.Seg_Metrics.update._fsb_original
    fused = []
    fused_ohem = AG.fused_ohem_ce
    monkeypatch.setattr(AG, "fused_ohem_ce", lambda *a: fused.append(1) or fused_ohem(*a))
    with cpu_backend.installed():
        with D.reference_path(drv):
            assert drv.seg_metrics.Seg_Metrics.update is dense_update
            ref1, ref_loss1 = _run(D, drv, 1)
            ref2, ref_loss2 = _run(D, drv, 2)
        assert not fused
        new1, new_loss1 = _run(D, drv, 1)
        assert len(fused) == 3                                        # logits8 / 16 / 32
        new2, new_loss2 = _run(D, drv, 2)
    assert new1 == ref1                                               # same weights, same labels: the same mIoU on step 1
    assert new_loss1[0] == pytest.approx(ref_loss1[0], rel=2e-3)
    assert len(new_loss2) == len(ref_loss2) == 2 and new_loss2[1] == pytest.approx(ref_loss2[1], rel=2e-3)
    assert new2 == pytest.approx(ref2, abs=1e-2)
