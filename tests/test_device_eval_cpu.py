"""Host side of validation on the device (fasterseg_b200.evaluator, fsb_upsample_argmax_confusion) without a GPU: which evaluations
take the device path, the launcher's patch of the reference's engine.evaluator, the marshalling of the new wrapper against the
header, and the network entry points on the CPU stand-in backend."""
import ctypes as C
import os
import re
import sys
import textwrap
import types

import numpy as np
import pytest
import torch

from fasterseg_b200 import _lib
from fasterseg_b200 import evaluator
from fasterseg_b200 import functional as F_
from fasterseg_b200 import launch
from fasterseg_b200 import metric
from tests import cpu_backend
from tests.test_boundary_cpu import _build_student, _build_supernet
from tests.test_marshalling_cpu import act, fake  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- eligibility ----------------------------------------------------------------------------------------------------------------------
def _ev(net, **kw):
    ev = types.SimpleNamespace(network=net, multi_scales=[1], is_flip=False, save_path=None, show_image=False,
                               show_prediction=False, logger=None)
    for k, v in kw.items():
        setattr(ev, k, v)
    return ev


@pytest.fixture(scope="module")
def student():
    model, _ = _build_student(1)
    return model.eval()


def test_eligibility(monkeypatch, student):
    assert not evaluator.eligible(_ev(student))                       # our network, but on the CPU
    monkeypatch.setattr(evaluator, "_on_cuda", lambda net: True)
    assert evaluator.eligible(_ev(student))
    assert evaluator.eligible(_ev(_build_supernet(3)))
    for kw in (dict(multi_scales=[0.75, 1]), dict(multi_scales=[]), dict(is_flip=True), dict(save_path="/tmp/x"),
               dict(show_image=True), dict(show_prediction=True), dict(logger=object()), dict(network=torch.nn.Conv2d(3, 3, 1)),
               dict(network=None)):
        assert not evaluator.eligible(_ev(student, **kw)), kw


def test_install_patches_in_place_once_and_keeps_the_originals(monkeypatch):
    class Evaluator:
        def run_online(self):
            return "orig-online"

        def run_online_multiprocess(self):
            return "orig-mp"

    mod = types.SimpleNamespace(Evaluator=Evaluator)
    assert evaluator.install(mod) is Evaluator
    first = Evaluator.run_online_multiprocess
    evaluator.install(mod)                                             # idempotent: no double wrapping
    assert Evaluator.run_online_multiprocess is first
    ev = Evaluator()
    for k, v in vars(_ev(None)).items():
        setattr(ev, k, v)
    assert ev.run_online() == "orig-online" and ev.run_online_multiprocess() == "orig-mp"    # not eligible -> the original
    monkeypatch.setattr(evaluator, "eligible", lambda e: True)
    monkeypatch.setattr(evaluator, "evaluate", lambda e: ("device", e.val_func))
    assert ev.run_online_multiprocess() == ("device", None)


# ---- launcher ------------------------------------------------------------------------------------------------------------------------
_STUB_EVALUATOR = textwrap.dedent('''
    class Evaluator(object):
        def run_online(self):
            return "online"

        def run_online_multiprocess(self):
            return "multiprocess"
''')


def _fake_checkout(tmp_path, with_tools):
    root = tmp_path / "FasterSeg"
    (root / "train").mkdir(parents=True)
    (root / "train" / "train.py").write_text("")
    if with_tools:
        eng = root / "tools" / "engine"
        eng.mkdir(parents=True)
        (eng / "__init__.py").write_text("")
        (eng / "evaluator.py").write_text(_STUB_EVALUATOR)
    return str(root / "train" / "train.py"), str(root / "tools")


@pytest.fixture
def clean_import_state():
    path, meta = list(sys.path), list(sys.meta_path)
    mods = {n: sys.modules[n] for n in ("engine", "engine.evaluator") if n in sys.modules}
    yield
    sys.path[:] = path
    sys.meta_path[:] = meta
    for n in ("engine", "engine.evaluator"):
        sys.modules.pop(n, None)
    sys.modules.update(mods)


def test_launcher_patches_the_reference_evaluator_when_it_is_imported(tmp_path, clean_import_state):
    script, tools = _fake_checkout(tmp_path, True)
    assert launch.reference_tools_dir(script) == tools
    for n in ("engine", "engine.evaluator"):
        sys.modules.pop(n, None)
    finder = launch.install_evaluator_patch(script)
    assert finder is not None and sys.meta_path[0] is finder
    sys.path.insert(0, tools)                                           # what config_*.py's add_path does
    import engine.evaluator as ev_mod
    for name in evaluator.PATCHED:
        m = getattr(ev_mod.Evaluator, name)
        assert m._fsb_original is not None and m.__name__ == name
    e = ev_mod.Evaluator()
    for k, v in vars(_ev(None)).items():
        setattr(e, k, v)
    assert e.run_online() == "online" and e.run_online_multiprocess() == "multiprocess"


def test_launcher_leaves_other_modules_named_engine_evaluator_alone(tmp_path, clean_import_state):
    script, _ = _fake_checkout(tmp_path / "a", True)
    _, other_tools = _fake_checkout(tmp_path / "b", True)
    for n in ("engine", "engine.evaluator"):
        sys.modules.pop(n, None)
    launch.install_evaluator_patch(script)
    sys.path.insert(0, other_tools)
    import engine.evaluator as ev_mod
    assert not hasattr(ev_mod.Evaluator.run_online, "_fsb_original")


def test_launcher_changes_nothing_without_a_reference_tools_dir(tmp_path, clean_import_state):
    script, _ = _fake_checkout(tmp_path, False)
    meta = list(sys.meta_path)
    assert launch.reference_tools_dir(script) is None
    assert launch.install_evaluator_patch(script) is None
    assert sys.meta_path == meta


# ---- marshalling -----------------------------------------------------------------------------------------------------------------------
_P = C.c_void_p
_CTYPES = {"int": C.c_int, "int64_t": C.c_int64, "float": C.c_float}


def test_signature_table_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "fsb200.h")).read(), flags=re.S)
    m = re.search(r"int\s+fsb_upsample_argmax_confusion\s*\(([^)]*)\)", src)
    params = [p.strip() for p in m.group(1).split(",")]
    want = [_P if "*" in p else _CTYPES[p.rsplit(None, 1)[0]] for p in params]
    res, args = _lib._SIGS["fsb_upsample_argmax_confusion"]
    assert res is C.c_int and args == want


def test_upsample_argmax_confusion_marshalling(fake):  # noqa: F811
    x = act(2, 19, 16, 32, wide=5)                                     # channel stride 24
    gt = torch.empty(2, 128, 256, dtype=torch.int32)
    out = torch.zeros(19 * 19 + 2, dtype=torch.int64)
    assert F_.upsample_argmax_confusion(x, (128, 256), gt, 19, out) is out
    a = fake.last("fsb_upsample_argmax_confusion")
    assert a[:6] == [2, 19, 16, 32, 128, 256]
    assert a[6:] == [x.data_ptr(), 24, gt.data_ptr(), 4, out.data_ptr(), None]
    for dtype, nbytes in ((torch.uint8, 1), (torch.int64, 8)):
        F_.upsample_argmax_confusion(x, (128, 256), gt.to(dtype), 19, out)
        assert fake.last("fsb_upsample_argmax_confusion")[9] == nbytes
    for bad in (dict(n_cl=11), dict(gt=gt[:, :, :128]), dict(gt=gt.to(torch.int16)), dict(gt=gt.transpose(1, 2)),
                dict(out=out[:-1]), dict(out=out.to(torch.int32))):
        kw = dict(gt=gt, n_cl=19, out=out)
        kw.update(bad)
        with pytest.raises(ValueError):
            F_.upsample_argmax_confusion(x, (128, 256), kw["gt"], kw["n_cl"], kw["out"])


# ---- network entry points on the CPU stand-in backend -----------------------------------------------------------------------------------
def _upsample_argmax_confusion(x, size, gt, n_cl, out):
    """stand-in: the two-kernel composition the fused kernel is bit-identical to"""
    return cpu_backend.confusion_matrix(cpu_backend.upsample_argmax(x, size), gt, n_cl, out)


@pytest.fixture
def cpu_path(monkeypatch):
    with cpu_backend.installed():
        monkeypatch.setattr(F_, "upsample_argmax_confusion", _upsample_argmax_confusion)
        yield


def _gt(shape, seed):
    rs = np.random.RandomState(seed)
    g = rs.randint(0, 19, size=shape).astype(np.int64)
    g[rs.uniform(size=shape) < 0.1] = 255
    return torch.from_numpy(g)


def test_student_accumulate_confusion(cpu_path, student):
    x = torch.randn(1, 3, 64, 128)
    gt = _gt((1, 64, 128), 1)
    cm = metric.ConfusionMatrix(19, device="cpu")
    student.accumulate_confusion(x, gt, cm)
    student.accumulate_confusion(x, gt, cm)
    want = metric.ConfusionMatrix(19, device="cpu")
    with torch.no_grad():
        lab = student(x).argmax(1).to(torch.uint8)
    want.update(lab, gt)
    want.update(lab, gt)
    assert torch.equal(cm.acc, want.acc) and int(cm.acc[-2]) > 0


@pytest.mark.parametrize("mode", ["max", "random"])
def test_supernet_single_head_entry_points_draw_widths_like_forward(cpu_path, mode):
    model = _build_supernet(3).eval()
    model.arch_idx, model.prun_mode = 0, mode
    x = torch.randn(1, 3, 64, 128)
    gt = _gt((1, 64, 128), 2)
    for head in range(5):
        np.random.seed(head)
        with torch.no_grad():
            want = model(x)[head].argmax(1).to(torch.uint8)
        after = np.random.get_state()[2]
        np.random.seed(head)
        got = model.predict_labels(x, head=head)
        assert np.random.get_state()[2] == after                        # same numpy draws as the full forward
        assert torch.equal(got, want), head
        np.random.seed(head)
        cm = metric.ConfusionMatrix(19, device="cpu")
        model.accumulate_confusion(x, gt, cm, head=head)
        ref = metric.ConfusionMatrix(19, device="cpu")
        ref.update(want, gt)
        assert torch.equal(cm.acc, ref.acc)
    assert len(model(x)) == 5                                            # the default path still returns the 5-tuple
