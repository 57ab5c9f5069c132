"""Host side of test-set prediction on the device (fasterseg_b200.tester, fsb_upsample_argmax_map) without a GPU: the writer's
files against the reference's own (tests/golden/tester.npz, oracle/make_golden_tester.py), which testers take the device path,
the launcher's patch of the reference's engine.tester, the marshalling of the new wrapper against the header, and the network
entry point on the CPU stand-in backend."""
import ctypes as C
import hashlib
import os
import re
import sys
import textwrap
import types

import numpy as np
import pytest
import torch

from fasterseg_b200 import _lib
from fasterseg_b200 import functional as F_
from fasterseg_b200 import launch
from fasterseg_b200 import tester
from tests import cpu_backend
from tests.test_boundary_cpu import _build_student
from tests.test_marshalling_cpu import act, fake  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "tester.npz"))
ID_TABLE = dict(zip(GOLDEN["id_table_keys"].tolist(), GOLDEN["id_table_values"].tolist()))
COLORS = GOLDEN["colors"].tolist()


# ---- numpy model of the kernel's per-pixel rule ---------------------------------------------------------------------------------------
def apply_tables(label, lut, palette, image):
    """ids = lut[label]; viz = palette[label] (B, G, R), or the RGB image pixel reversed where palette[label].use_image is set"""
    label = np.asarray(label, np.int64)
    ids = np.asarray(lut)[label]
    if palette is None:
        return ids, None
    pal = np.asarray(palette)[label]
    keep = pal[..., 3:] != 0
    viz = np.where(keep, np.asarray(image)[..., ::-1], pal[..., :3]) if keep.any() else pal[..., :3]
    viz = np.ascontiguousarray(viz, dtype=np.uint8)
    return ids, viz


# ---- files against the reference's own SegTester.func_per_iteration ---------------------------------------------------------------------
def _pred_map(h, w, n):
    """oracle/make_golden_tester.py pred_map"""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    return (y // 3 * 7 + x // 5 * 3 + (x * y) % 5) % n


def _image_map(h, w):
    """oracle/make_golden_tester.py image_map"""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    return np.stack([(y * 5 + x * 11 + c * 70 + (x * y) % 7) % 256 for c in range(3)], axis=2).astype(np.uint8)


CASES = sorted(k[:-len("/case")] for k in GOLDEN.files if k.endswith("/case"))


@pytest.mark.parametrize("name", CASES)
def test_writer_reproduces_the_reference_files(tmp_path, name):
    h, w, n, show, background, ncol = GOLDEN[name + "/case"].tolist()
    colors = COLORS if ncol < 0 else COLORS[:ncol]
    if name + "/pred" in GOLDEN.files:
        pred, image = GOLDEN[name + "/pred"], GOLDEN[name + "/image"]
        assert np.array_equal(pred, _pred_map(h, w, n)) and np.array_equal(image, _image_map(h, w))
    else:
        pred, image = _pred_map(h, w, n), _image_map(h, w)
    lut, palette = tester.tables(ID_TABLE, n, colors if show else None, background)
    ids, viz = apply_tables(pred, lut.numpy(), None if palette is None else palette.numpy(), image)
    files = [(str(tmp_path / (name + ".png")), torch.from_numpy(ids.astype(np.uint8)))]
    if show:
        files.insert(0, (str(tmp_path / (name + ".viz.png")), torch.from_numpy(viz)))
    with tester.Writer() as wr:
        wr.put(files)
    assert sorted(os.listdir(tmp_path)) == sorted(os.path.basename(p) for p, _ in files)
    for suffix in (["png", "viz.png"] if show else ["png"]):
        data = (tmp_path / (name + "." + suffix)).read_bytes()
        key = name + "/" + suffix
        if key + ".sha256" in GOLDEN.files:
            assert hashlib.sha256(data).digest() == GOLDEN[key + ".sha256"].tobytes(), key
        else:
            assert data == GOLDEN[key].tobytes(), key


def test_palette_follows_set_img_color():
    lut, pal = tester.tables(ID_TABLE, 19, COLORS[:15], 3)
    assert lut.tolist() == [ID_TABLE[k] for k in range(19)]
    for k in range(19):
        if k < 15 and k != 3:
            assert pal[k].tolist() == COLORS[k][::-1] + [0]
        else:
            assert pal[k, 3] == 1
    assert tester.tables(ID_TABLE, 19)[1] is None


# ---- eligibility ----------------------------------------------------------------------------------------------------------------------
_STUB_TESTER = textwrap.dedent('''
    class Tester(object):
        def run_online(self):
            return "online"

        def run_online_multiprocess(self):
            return "multiprocess"
''')


def _fake_checkout(base, with_tools=True, table="ID_TABLE"):
    """<base>/FasterSeg with train/train.py, train/test.py (a func_per_iteration and the id table in its globals) and, optionally,
    tools/engine/tester.py"""
    root = base / "FasterSeg"
    (root / "train").mkdir(parents=True)
    (root / "train" / "train.py").write_text("")
    (root / "train" / "test.py").write_text("cityscapes_trainID2id = %s\n\n\ndef func_per_iteration(self, data, device, iter=None):\n"
                                            "    return None\n" % (repr(ID_TABLE) if table == "ID_TABLE" else table))
    if with_tools:
        eng = root / "tools" / "engine"
        eng.mkdir(parents=True)
        (eng / "__init__.py").write_text("")
        (eng / "tester.py").write_text(_STUB_TESTER)
    return str(root / "train" / "train.py"), str(root / "tools")


def _load(path, name):
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _classes(base, table="ID_TABLE"):
    """(patched Tester class, SegTester subclass whose func_per_iteration is the checkout's train/test.py's)"""
    script, tools = _fake_checkout(base, table=table)
    eng = _load(os.path.join(tools, "engine", "tester.py"), "fsb_test_engine_tester_%d" % id(base))
    test = _load(os.path.join(os.path.dirname(script), "test.py"), "fsb_test_train_test_%d" % id(base))
    tester.install(eng)
    seg = type("SegTester", (eng.Tester,), {"func_per_iteration": test.func_per_iteration})
    return eng.Tester, seg


class _Colors:
    def __init__(self, colors):
        self.colors = colors

    def get_class_colors(self):
        return self.colors


def _t(cls, net, **kw):
    t = cls()
    cfg = types.SimpleNamespace(eval_scale_array=[1], background=-1, save="out")
    for k, v in dict(network=net, devices=[0], config=cfg, is_flip=False, show_prediction=False, dataset=_Colors(COLORS)).items():
        setattr(t, k, v)
    for k, v in kw.items():
        setattr(t, k, v)
    return t


@pytest.fixture(scope="module")
def student():
    model, _ = _build_student(1)
    return model.eval()


@pytest.fixture
def on_cuda0(monkeypatch):
    monkeypatch.setattr(tester, "_device", lambda net: torch.device("cuda", 0))


def test_not_on_cuda_is_not_eligible(tmp_path, student):
    _, seg = _classes(tmp_path)
    assert not tester.eligible(_t(seg, student))


def test_eligibility_matrix(tmp_path, student, on_cuda0):
    base, seg = _classes(tmp_path / "a")
    assert tester.eligible(_t(seg, student))
    assert tester.eligible(_t(seg, student, show_prediction=True))
    cfg = lambda **kw: types.SimpleNamespace(**dict(dict(eval_scale_array=[1], background=-1, save="out"), **kw))  # noqa: E731
    for kw in (dict(devices=[1]), dict(devices=[]), dict(network=torch.nn.Conv2d(3, 3, 1)), dict(network=None), dict(config=None),
               dict(config=cfg(eval_scale_array=[0.75, 1])), dict(is_flip=True),
               dict(show_prediction=True, dataset=_Colors([[0, 0, 256]] + COLORS[1:])),
               dict(show_prediction=True, dataset=_Colors([[0, 0, -1]] + COLORS[1:])),
               dict(show_prediction=True, dataset=_Colors([[0.5, 0, 0]] + COLORS[1:])),
               dict(show_prediction=True, dataset=_Colors([[0, 0]] + COLORS[1:])),
               dict(show_prediction=True, dataset=_Colors([7] + COLORS[1:]))):
        assert not tester.eligible(_t(seg, student, **kw)), kw
    # func_per_iteration overridden in a subclass, or from another checkout's train/test.py
    over = type("Over", (seg,), {"func_per_iteration": lambda self, data, device, iter=None: None})
    assert not tester.eligible(_t(over, student))
    _, other = _classes(tmp_path / "b")
    mixed = type("Mixed", (base,), {"func_per_iteration": other.func_per_iteration})
    assert not tester.eligible(_t(mixed, student))
    assert not tester.eligible(_t(base, student))                       # the base Tester's own func_per_iteration: none
    # id tables with a missing, out-of-range or non-integer entry
    for i, table in enumerate(("{k: k for k in range(18)}", "{**{k: 7 for k in range(19)}, 4: 256}", "{**{k: 7 for k in range(19)}, 4: -1}",
                               "{**{k: 7 for k in range(19)}, 4: 7.0}", "[7] * 19")):
        _, bad = _classes(tmp_path / ("t%d" % i), table=table)
        assert not tester.eligible(_t(bad, student)), table
    _, fine = _classes(tmp_path / "t9", table="{k: k for k in range(19)}")
    assert tester.eligible(_t(fine, student))


def test_install_is_idempotent_and_ineligible_testers_reach_the_original(tmp_path, monkeypatch):
    base, seg = _classes(tmp_path)
    first = base.run_online
    mod = types.SimpleNamespace(Tester=base, __file__=os.path.join(str(tmp_path), "FasterSeg", "tools", "engine", "tester.py"))
    assert tester.install(mod) is base
    assert base.run_online is first and base.run_online._fsb_original is not None
    t = _t(seg, None)
    assert t.run_online() == "online" and t.run_online_multiprocess() == "multiprocess"
    monkeypatch.setattr(tester, "eligible", lambda x: True)
    monkeypatch.setattr(tester, "predict", lambda x: ("device", x.val_func))
    t.network = "net"
    assert t.run_online() == ("device", "net") and t.run_online_multiprocess() == ("device", "net")


# ---- launcher ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def clean_import_state():
    path, meta = list(sys.path), list(sys.meta_path)
    mods = {n: sys.modules[n] for n in ("engine", "engine.tester") if n in sys.modules}
    yield
    sys.path[:] = path
    sys.meta_path[:] = meta
    for n in ("engine", "engine.tester"):
        sys.modules.pop(n, None)
    sys.modules.update(mods)


def test_launcher_patches_the_reference_tester_when_it_is_imported(tmp_path, clean_import_state):
    script, tools = _fake_checkout(tmp_path)
    for n in ("engine", "engine.tester"):
        sys.modules.pop(n, None)
    finder = launch.install_tester_patch(script)
    assert finder is not None and sys.meta_path[0] is finder
    sys.path.insert(0, tools)
    import engine.tester as t_mod
    for name in tester.PATCHED:
        m = getattr(t_mod.Tester, name)
        assert m._fsb_original is not None and m.__name__ == name
    assert t_mod.Tester._fsb_test_py == os.path.realpath(os.path.join(os.path.dirname(script), "test.py"))
    t = t_mod.Tester()
    assert t.run_online() == "online" and t.run_online_multiprocess() == "multiprocess"


def test_launcher_leaves_other_modules_named_engine_tester_alone(tmp_path, clean_import_state):
    script, _ = _fake_checkout(tmp_path / "a")
    _, other_tools = _fake_checkout(tmp_path / "b")
    for n in ("engine", "engine.tester"):
        sys.modules.pop(n, None)
    launch.install_tester_patch(script)
    sys.path.insert(0, other_tools)
    import engine.tester as t_mod
    assert not hasattr(t_mod.Tester.run_online, "_fsb_original")


def test_launcher_changes_nothing_without_a_tools_dir(tmp_path, clean_import_state):
    script, _ = _fake_checkout(tmp_path, with_tools=False)
    meta = list(sys.meta_path)
    assert launch.install_tester_patch(script) is None
    assert sys.meta_path == meta


# ---- marshalling -----------------------------------------------------------------------------------------------------------------------
_P = C.c_void_p
_CTYPES = {"int": C.c_int, "int64_t": C.c_int64, "float": C.c_float}


def test_signature_table_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "fsb200.h")).read(), flags=re.S)
    m = re.search(r"int\s+fsb_upsample_argmax_map\s*\(([^)]*)\)", src)
    params = [p.strip() for p in m.group(1).split(",")]
    want = [_P if "*" in p else _CTYPES[p.rsplit(None, 1)[0]] for p in params]
    res, args = _lib._SIGS["fsb_upsample_argmax_map"]
    assert res is C.c_int and args == want


def test_upsample_argmax_map_marshalling(fake):  # noqa: F811
    x = act(2, 19, 16, 32, wide=5)                                     # channel stride 24
    lut = torch.arange(19, dtype=torch.uint8)
    pal = torch.zeros(19, 4, dtype=torch.uint8)
    img = torch.zeros(2, 128, 256, 3, dtype=torch.uint8)
    ids, viz = F_.upsample_argmax_map(x, (128, 256), lut=lut, palette=pal, image=img)
    assert ids.shape == (2, 128, 256) and viz.shape == (2, 128, 256, 3) and ids.dtype == viz.dtype == torch.uint8
    a = fake.last("fsb_upsample_argmax_map")
    assert a[:6] == [2, 19, 16, 32, 128, 256]
    assert a[6:] == [x.data_ptr(), 24, lut.data_ptr(), ids.data_ptr(), pal.data_ptr(), img.data_ptr(), viz.data_ptr(), None]
    ids, viz = F_.upsample_argmax_map(x, (128, 256))                    # ids only, identity table
    assert viz is None and fake.last("fsb_upsample_argmax_map")[8:] == [None, ids.data_ptr(), None, None, None, None]
    ids, viz = F_.upsample_argmax_map(x, (128, 256), palette=pal)       # viz only; no use_image row, so no image needed
    assert ids is None and fake.last("fsb_upsample_argmax_map")[8:] == [None, None, pal.data_ptr(), None, viz.data_ptr(), None]
    ids_out, viz_out = torch.empty(2, 128, 256, dtype=torch.uint8), torch.empty(2, 128, 256, 3, dtype=torch.uint8)
    assert F_.upsample_argmax_map(x, (128, 256), palette=pal, ids_out=ids_out, viz_out=viz_out) == (ids_out, viz_out)
    use = pal.clone()
    use[3, 3] = 1
    bad_cases = (dict(lut=lut[:18]), dict(lut=lut.to(torch.int32)), dict(palette=pal[:, :3]), dict(palette=pal.t().contiguous().t()),
                 dict(palette=use), dict(palette=use, image=img[:, :64]), dict(palette=use, image=img.to(torch.int32)),
                 dict(palette=pal, image=img.permute(0, 2, 1, 3)), dict(image=img), dict(viz_out=viz_out),
                 dict(ids_out=ids_out[:1]), dict(ids_out=ids_out.to(torch.int64)), dict(palette=pal, viz_out=viz_out[..., :2]),
                 dict(lut=lut.to("meta")))
    for bad in bad_cases:
        with pytest.raises(ValueError):
            F_.upsample_argmax_map(x, (128, 256), **bad)
    with pytest.raises(ValueError):
        F_.upsample_argmax_map(x.float(), (128, 256))
    with pytest.raises(ValueError):
        F_.upsample_argmax_map(act(1, 256, 4, 4), (32, 32))


# ---- network entry point on the CPU stand-in backend -------------------------------------------------------------------------------------
_REAL = F_.upsample_argmax_map


@pytest.fixture
def cpu_path(fake, monkeypatch):  # noqa: F811
    """the real wrapper's checks and allocation against the fake library, then the numpy model of the kernel"""
    def standin(x, size, lut=None, palette=None, image=None, ids_out=None, viz_out=None):
        ids, viz = _REAL(x, size, lut=lut, palette=palette, image=image, ids_out=ids_out, viz_out=viz_out)
        label = cpu_backend.upsample_argmax(x, size)
        want_ids, want_viz = apply_tables(label.numpy(), (lut if lut is not None else torch.arange(x.shape[1])).numpy(),
                                          None if palette is None else palette.numpy(), None if image is None else image.numpy())
        if ids is not None:
            ids.copy_(torch.from_numpy(want_ids.astype(np.uint8)))
        if viz is not None:
            viz.copy_(torch.from_numpy(want_viz))
        return ids, viz

    with cpu_backend.installed():
        monkeypatch.setattr(F_, "upsample_argmax_map", standin)
        yield


def test_student_predict_label_maps(cpu_path, student):
    g = torch.Generator().manual_seed(3)
    img = torch.randint(0, 256, (1, 64, 128, 3), dtype=torch.uint8, generator=g)
    x = ((img.float() / 255 - torch.tensor([0.485, 0.456, 0.406])) / torch.tensor([0.229, 0.224, 0.225])).permute(0, 3, 1, 2)
    lut, pal = tester.tables(ID_TABLE, 19, COLORS[:12], 5)
    ids, viz = student.predict_label_maps(x.contiguous(), lut=lut)
    with torch.no_grad():
        label = student(x.contiguous()).argmax(1)
    assert viz is None and torch.equal(ids, lut[label])
    ids, viz = student.predict_label_maps(x.contiguous(), palette=torch.zeros(19, 4, dtype=torch.uint8))
    assert ids is None and torch.equal(viz, torch.zeros_like(viz))
    with pytest.raises(ValueError):                                      # a float input cannot serve use_image rows
        student.predict_label_maps(x.contiguous(), lut=lut, palette=pal)


def test_predict_label_maps_takes_use_image_pixels_from_a_uint8_input(cpu_path, student, monkeypatch):
    img = torch.randint(0, 256, (1, 64, 128, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(4))
    logits = act(1, 19, 8, 16)
    logits.copy_(torch.randn(1, 19, 8, 16))
    monkeypatch.setattr(type(student), "_features", lambda self, inp: logits)
    lut, pal = tester.tables(ID_TABLE, 19, COLORS[:12], 5)
    ids, viz = student.predict_label_maps(img.permute(0, 3, 1, 2), lut=lut, palette=pal)
    label = cpu_backend.upsample_argmax(logits, (64, 128)).long()
    want_ids, want_viz = apply_tables(label.numpy(), lut.numpy(), pal.numpy(), img.numpy())
    assert np.array_equal(ids.numpy(), want_ids) and np.array_equal(viz.numpy(), want_viz)
    keep = pal[label][..., 3] == 1
    assert bool(keep.any()) and torch.equal(viz[keep], img[keep].flip(-1))


# ---- writer ---------------------------------------------------------------------------------------------------------------------------
def test_writer_finishes_every_file_before_returning(tmp_path, monkeypatch):
    import threading
    import time
    import cv2
    real = cv2.imwrite
    threads = set()

    def slow(path, arr):
        threads.add(threading.get_ident())
        time.sleep(0.02)
        return real(path, arr)

    monkeypatch.setattr(cv2, "imwrite", slow)
    imgs = [torch.full((9, 13), k, dtype=torch.uint8) for k in range(11)]
    with tester.Writer(slots=3) as wr:
        for k, im in enumerate(imgs):
            wr.put([(str(tmp_path / ("%d.png" % k)), im)])
    for k, im in enumerate(imgs):                       # ring buffers reused 3-4 times, each file still has its own image
        assert np.array_equal(cv2.imread(str(tmp_path / ("%d.png" % k)), cv2.IMREAD_UNCHANGED), im.numpy())
    assert threading.get_ident() not in threads


def test_writer_propagates_a_writer_exception(tmp_path, monkeypatch):
    import cv2

    def boom(path, arr):
        if path.endswith("2.png"):
            raise RuntimeError("disk full")
        return True

    monkeypatch.setattr(cv2, "imwrite", boom)
    with pytest.raises(RuntimeError, match="disk full"):
        with tester.Writer(slots=2) as wr:
            for k in range(3):
                wr.put([(str(tmp_path / ("%d.png" % k)), torch.zeros(4, 4, dtype=torch.uint8))])
    monkeypatch.setattr(cv2, "imwrite", lambda path, arr: False)      # a False return is ignored
    with tester.Writer() as wr:
        wr.put([(str(tmp_path / "x.png"), torch.zeros(4, 4, dtype=torch.uint8))])
