"""Test-set prediction on the device (fasterseg_b200.tester, the fused upsample + argmax + id / colour map kernel): the maps
against fsb_upsample_argmax followed by the tables applied with torch, and the patched Tester's files against those the reference
arithmetic writes (train/test.py:49-69 after tools/engine/tester.py:179-204,270-291: model(x) fp32 -> exp -> argmax -> trainId ->
id -> cv2.imwrite; tools/utils/visualize.py:6-21 for the colour map)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ref_harness
from tests.test_device_eval_gpu import MEAN, STD, SyntheticSet, _logits, _reference_labels, _student
from tests.test_device_tester_cpu import COLORS, ID_TABLE, _classes, _t

pytestmark = pytest.mark.gpu


def _F():
    from fasterseg_b200 import functional as F_
    return F_


# ---- kernel -------------------------------------------------------------------------------------------------------------------------
def _tables(n_cl, seed, use_image=True):
    g = torch.Generator().manual_seed(seed)
    lut = torch.randperm(256, generator=g)[:n_cl].to(torch.uint8)
    pal = torch.randint(0, 256, (n_cl, 4), generator=g, dtype=torch.int64).to(torch.uint8)
    pal[:, 3] = 0
    if use_image:
        pal[torch.randperm(n_cl, generator=g)[:max(1, n_cl // 3)], 3] = 1
    return lut.cuda(), pal.cuda()


def _want(labels, lut, pal, image):
    lab = labels.long()
    rows = pal[lab]
    viz = torch.where(rows[..., 3:] != 0, image.flip(-1), rows[..., :3]) if image is not None else rows[..., :3]
    return lut[lab], viz


@pytest.mark.parametrize("N,Hi,Wi,Ho,Wo", [(1, 128, 256, 1024, 2048), (2, 64, 128, 512, 1024), (2, 37, 53, 301, 419), (1, 9, 12, 9, 12)])
@pytest.mark.parametrize("n_cl,cs", [(19, 24), (11, 16), (11, 32)])
def test_maps_equal_upsample_argmax_then_tables(N, Hi, Wi, Ho, Wo, n_cl, cs):
    F_ = _F()
    x = _logits(N, n_cl, Hi, Wi, cs, seed=Hi * 7 + n_cl)
    labels = F_.upsample_argmax(x, (Ho, Wo))
    lut, pal = _tables(n_cl, Wo)
    image = torch.randint(0, 256, (N, Ho, Wo, 3), dtype=torch.uint8, device="cuda")
    ids, viz = F_.upsample_argmax_map(x, (Ho, Wo), lut=lut, palette=pal, image=image)
    want_ids, want_viz = _want(labels, lut, pal, image)
    assert torch.equal(ids, want_ids) and torch.equal(viz, want_viz)
    assert bool((pal[labels.long()][..., 3] == 1).any())                    # use_image rows were hit
    # each output alone, the identity table, and outputs at odd byte offsets (the byte-store path)
    ids2, none = F_.upsample_argmax_map(x, (Ho, Wo))
    assert none is None and torch.equal(ids2, labels)
    pal0 = pal.clone()
    pal0[:, 3] = 0
    none, viz0 = F_.upsample_argmax_map(x, (Ho, Wo), palette=pal0)
    assert none is None and torch.equal(viz0, _want(labels, lut, pal0, None)[1])
    raw = torch.full((N * Ho * Wo * 4 + 8,), 7, dtype=torch.uint8, device="cuda")
    ids_out = raw[1:1 + N * Ho * Wo].view(N, Ho, Wo)
    viz_out = raw[N * Ho * Wo + 3:N * Ho * Wo + 3 + N * Ho * Wo * 3].view(N, Ho, Wo, 3)
    got = F_.upsample_argmax_map(x, (Ho, Wo), lut=lut, palette=pal, image=image, ids_out=ids_out, viz_out=viz_out)
    torch.cuda.synchronize()
    assert got[0] is ids_out and got[1] is viz_out
    assert torch.equal(ids_out, want_ids) and torch.equal(viz_out, want_viz)
    assert int(raw[0]) == 7 and int(raw[N * Ho * Wo + 1]) == 7 and int(raw[-1]) == 7      # nothing written outside


def test_library_rejects_bad_arguments():
    F_ = _F()
    from fasterseg_b200 import _lib
    lib = _lib.lib()
    x = _logits(1, 19, 8, 8, 24, 1)
    lut, pal = _tables(19, 1)
    ids = torch.empty(1, 64, 64, dtype=torch.uint8, device="cuda")
    viz = torch.empty(1, 64, 64, 3, dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    s = F_._stream()
    ok = lib.fsb_upsample_argmax_map(1, 19, 8, 8, 64, 64, p(x), 24, p(lut), p(ids), None, None, None, s)
    assert ok == 0
    for args in ((1, 19, 8, 8, 64, 64, p(x), 24, p(lut), None, p(pal), None, None),      # no output
                 (1, 19, 8, 8, 64, 64, p(x), 24, p(lut), p(ids), None, None, p(viz)),     # viz without a palette
                 (1, 0, 8, 8, 64, 64, p(x), 24, p(lut), p(ids), None, None, None),        # C = 0
                 (1, 256, 8, 8, 64, 64, p(x), 256, p(lut), p(ids), None, None, None),     # C > 255
                 (1, 19, 8, 8, 64, 64, p(x), 16, p(lut), p(ids), None, None, None),       # channel stride < C
                 (0, 19, 8, 8, 64, 64, p(x), 24, p(lut), p(ids), None, None, None),
                 (1, 19, 8, 8, 0, 64, p(x), 24, p(lut), p(ids), None, None, None),
                 (1, 19, 8, 8, 64, 64, None, 24, p(lut), p(ids), None, None, None)):
        assert lib.fsb_upsample_argmax_map(*args, s) == -1                   # FSB_ERR_INVALID
    with pytest.raises(ValueError):
        F_.upsample_argmax_map(x, (64, 64), palette=pal)                 # use_image rows without an image
    with pytest.raises(ValueError):
        F_.upsample_argmax_map(x, (64, 64), lut=lut.cpu())
    torch.cuda.synchronize()


# ---- the patched tester -------------------------------------------------------------------------------------------------------------
class PredictionSet(SyntheticSet):
    def get_class_colors(self):
        return COLORS


def _expected_files(model, ds, folder, show, background=-1):
    """what train/test.py:49-69 writes, restated: labels of the reference arithmetic (fp32 logits -> exp -> argmax), trainId -> id
    through the table, set_img_color's composite, cv2.imwrite of the int64 map and of the composite reversed to BGR.  A label may
    differ from ours only where the two classes' fp32 logits are exp-tied or a rounding step apart; there ours is taken."""
    import cv2
    model.set_input_normalization(MEAN, STD)
    table = np.array([ID_TABLE[k] for k in range(19)], np.int64)
    differ = 0
    for i in range(ds.get_length()):
        d = ds[i]
        img = np.ascontiguousarray(d["data"])
        logits, ref, ours = _reference_labels(model, img)
        mism = ref != ours
        if bool(mism.any()):
            lr = logits.gather(0, ref.long()[None])[0][mism]
            lo = logits.gather(0, ours.long()[None])[0][mism]
            tie = (torch.exp(lr) == torch.exp(lo)) | ((lr - lo).abs() <= 4 * torch.finfo(torch.float32).eps * torch.maximum(lr.abs(), lo.abs()))
            assert bool(tie.all())
            differ += int(mism.sum())
        lab = ref.clone()
        lab[mism] = ours[mism]
        pred = lab.cpu().numpy().astype(np.int64)
        if show:
            comp = np.array(img, np.uint8)
            for k in range(len(COLORS)):
                if k != background:
                    comp[np.where(pred == k)] = COLORS[k]
            cv2.imwrite(os.path.join(folder, d["fn"] + ".viz.png"), comp[:, :, ::-1])
        cv2.imwrite(os.path.join(folder, d["fn"] + ".png"), table[pred])
    print("labels differing from the reference arithmetic at exp- or rounding-tied pixels: %d" % differ)


def _same_files(a, b):
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(b)) and names
    for n in names:
        assert open(os.path.join(a, n), "rb").read() == open(os.path.join(b, n), "rb").read(), n
    return names


def _standin(tmp_path, model, ds, **kw):
    _, seg = _classes(tmp_path / "checkout")
    t = _t(seg, model, dataset=ds, ndata=ds.get_length(), threds=3, image_mean=MEAN, image_std=STD, class_num=19, **kw)
    return t


@pytest.mark.parametrize("show", [False, True])
def test_patched_tester_writes_the_reference_files(tmp_path, monkeypatch, show):
    model = _student()
    ds = PredictionSet(6, 1024, 2048, seed=21)
    t = _standin(tmp_path, model, ds, show_prediction=show)
    from fasterseg_b200 import tester
    assert tester.eligible(t)
    run = tmp_path / "run"
    (run / "out" / "test").mkdir(parents=True)
    monkeypatch.chdir(run)
    model.train()
    torch.manual_seed(5)
    rng = torch.get_rng_state()
    assert t.run_online() is None
    assert not model.training and all(not m.training for m in model.modules())      # left in eval mode, like val_func_process
    assert torch.equal(torch.get_rng_state(), rng)
    want = tmp_path / "want"
    want.mkdir()
    _expected_files(model, ds, str(want), show)
    names = _same_files(str(run / "out" / "test"), str(want))
    assert len(names) == 6 * (2 if show else 1)
    assert t.run_online_multiprocess() is None
    _same_files(str(run / "out" / "test"), str(want))


def test_testers_the_device_path_does_not_cover_run_the_original(tmp_path):
    model = _student()
    ds = PredictionSet(1, 64, 128, seed=22)
    for kw in (dict(is_flip=True), dict(config=type("Cfg", (), dict(eval_scale_array=[0.75, 1], background=-1, save="out"))())):
        t = _standin(tmp_path / str(len(kw)) / ("flip" if "is_flip" in kw else "scales"), model, ds, **kw)
        assert t.run_online() == "online" and t.run_online_multiprocess() == "multiprocess"


# ---- the reference's own tester, where build() kept a copy of the reference ------------------------------------------------------------
def _reference_seg_tester():
    if not ref_harness.reference_available():
        pytest.skip("no copy of the reference under oracle/_ref")
    import collections
    import collections.abc
    for n in ("Iterable", "Mapping", "Sequence"):            # tools/utils/img_utils.py predates python 3.10
        if not hasattr(collections, n):
            setattr(collections, n, getattr(collections.abc, n))
    root = ref_harness.REFERENCE_ROOT
    tools, train = os.path.join(root, "tools"), os.path.join(root, "train")
    before = set(sys.modules)
    old_path = list(sys.path)
    sys.path[:0] = [train, tools]
    try:
        import importlib
        t_mod = importlib.import_module("engine.tester")
        seg_test = importlib.import_module("test")
    finally:
        sys.path[:] = old_path
        for n in set(sys.modules) - before:
            f = getattr(sys.modules[n], "__file__", None) or ""
            if os.path.realpath(f).startswith(os.path.realpath(root)):
                del sys.modules[n]
    return t_mod, seg_test.SegTester


@pytest.mark.parametrize("show", [False, True])
def test_reference_seg_tester_unpatched_and_patched_write_the_same_files(tmp_path, monkeypatch, show):
    from fasterseg_b200 import tester
    t_mod, SegTester = _reference_seg_tester()
    model = _student()
    ds = PredictionSet(2, 1024, 2048, seed=23)
    config = type("Cfg", (), dict(num_classes=19, eval_scale_array=[1], background=-1, save="out"))()
    t = SegTester(ds, 19, MEAN, STD, model, [1], False, 0, config=config, show_prediction=show)
    for d in ("ref", "dev"):
        (tmp_path / d / "out" / "test").mkdir(parents=True)
    saved = {n: t_mod.Tester.__dict__[n] for n in tester.PATCHED}
    monkeypatch.chdir(tmp_path / "ref")
    t.run_online()                                       # unpatched: the reference's per-image loop
    try:
        tester.install(t_mod)
        assert tester.eligible(t)
        monkeypatch.chdir(tmp_path / "dev")
        t.run_online()
    finally:
        for n, f in saved.items():
            setattr(t_mod.Tester, n, f)
    ref_dir, dev_dir = str(tmp_path / "ref" / "out" / "test"), str(tmp_path / "dev" / "out" / "test")
    if sorted(os.listdir(ref_dir)) == sorted(os.listdir(dev_dir)) and all(
            open(os.path.join(ref_dir, n), "rb").read() == open(os.path.join(dev_dir, n), "rb").read() for n in os.listdir(ref_dir)):
        return
    want = tmp_path / "want"                              # only where the reference arithmetic has exp- / rounding-tied pixels
    want.mkdir()
    _expected_files(model, ds, str(want), show)
    _same_files(dev_dir, str(want))
