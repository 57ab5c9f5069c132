"""Validation on the device (fasterseg_b200.evaluator, the fused upsample + argmax + confusion kernel): counters bit-identical to
upsample_argmax + confusion_matrix, and the patched Evaluator against the reference evaluator's arithmetic
(tools/engine/evaluator.py:297-318: model(x) fp32 -> exp -> argmax; tools/seg_opr/metric.py:7-15 hist_info)."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import fasterseg_oracle as orc
from oracle import ref_harness
from tests import helpers as H
from tests.test_boundary_cpu import _build_student, _build_supernet
from tests.test_student_gpu import _load_seeded
from tests.test_supernet_oracle import make_sd

pytestmark = pytest.mark.gpu

MEAN, STD = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])


def _F():
    from fasterseg_b200 import functional as F_
    return F_


# ---- kernel -------------------------------------------------------------------------------------------------------------------------
def _logits(N, C, H_, W_, cs, seed):
    """NHWC fp16 view with channel stride cs >= C; a quarter of the pixels are quantised to 0.5 steps so exact ties between
    classes occur (the tie rule: first maximum wins)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H_, W_, cs, generator=g) * 3
    q = torch.rand(N, H_, W_, 1, generator=g) < 0.25
    x = torch.where(q, torch.round(x * 2) / 2, x)
    return x.half().cuda().permute(0, 3, 1, 2)[:, :C]


def _gt(N, Ho, Wo, n_cl, dtype, seed):
    rs = np.random.RandomState(seed)
    g = rs.randint(0, n_cl, size=(N, Ho, Wo)).astype(np.int64)
    g[rs.uniform(size=g.shape) < 0.1] = 255
    if dtype != torch.uint8:
        g[rs.uniform(size=g.shape) < 0.05] = -1
        g[rs.uniform(size=g.shape) < 0.02] = n_cl + 3
    return torch.from_numpy(g).to(dtype).cuda()


@pytest.mark.parametrize("N,Hi,Wi,Ho,Wo", [(1, 128, 256, 1024, 2048), (2, 64, 128, 512, 1024), (2, 37, 53, 301, 419), (1, 9, 12, 9, 12)])
@pytest.mark.parametrize("n_cl,cs", [(19, 24), (11, 16), (11, 32)])
def test_fused_confusion_equals_upsample_argmax_then_confusion_matrix(N, Hi, Wi, Ho, Wo, n_cl, cs):
    F_ = _F()
    x = _logits(N, n_cl, Hi, Wi, cs, seed=Hi * 7 + n_cl)
    labels = F_.upsample_argmax(x, (Ho, Wo))
    for k, dtype in enumerate((torch.uint8, torch.int32, torch.int64)):
        gt = _gt(N, Ho, Wo, n_cl, dtype, seed=k + Wo)
        want = F_.confusion_matrix(labels, gt, n_cl)
        got = torch.full((n_cl * n_cl + 2,), 5, device="cuda", dtype=torch.int64)   # accumulates into what is there
        F_.upsample_argmax_confusion(x, (Ho, Wo), gt, n_cl, got)
        torch.cuda.synchronize()
        assert torch.equal(got - 5, want), (dtype, int((got - 5 - want).abs().sum()))
        assert int(want[n_cl * n_cl]) > 0 and int(want[:n_cl * n_cl].sum()) == int(want[n_cl * n_cl])


def test_fused_confusion_rejects_bad_arguments():
    F_ = _F()
    x = _logits(1, 19, 8, 8, 24, 1)
    gt = torch.zeros(1, 64, 64, dtype=torch.int64, device="cuda")
    out = torch.zeros(19 * 19 + 2, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError):
        F_.upsample_argmax_confusion(x, (64, 64), gt, 11, torch.zeros(123, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError):
        F_.upsample_argmax_confusion(x, (64, 64), gt.to(torch.int16), 19, out)
    big = _logits(1, 70, 8, 8, 72, 2)
    with pytest.raises(Exception):
        F_.upsample_argmax_confusion(big, (64, 64), gt, 70, torch.zeros(70 * 70 + 2, dtype=torch.int64, device="cuda"))


# ---- evaluator --------------------------------------------------------------------------------------------------------------------
class SyntheticSet:
    """what tools/datasets/BaseDataset.py:34-60 hands the evaluator for the 'val' split: the uint8 RGB image as the BGR->RGB
    flipped view of the decoded array, and the uint8 label map (255 = ignore)"""

    def __init__(self, n, h, w, seed):
        rs = np.random.RandomState(seed)
        self.items = []
        for i in range(n):
            bgr = rs.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
            lab = rs.randint(0, 19, size=(h, w)).astype(np.uint8)
            lab[rs.uniform(size=lab.shape) < 0.1] = 255
            self.items.append((bgr, lab))

    def get_length(self):
        return len(self.items)

    def __len__(self):
        return len(self.items)

    def __getitem__(self, idx):
        bgr, lab = self.items[idx]
        return dict(data=bgr[:, :, ::-1], label=lab, fn="img%d" % idx, n=len(self.items))

    def get_class_names(self):
        return ["class%d" % i for i in range(19)]


def _compute_metric(ev, results):
    """SegEvaluator.compute_metric's arithmetic (tools/seg_opr/metric.py:18-27 compute_score; one line per class and the means)"""
    from fasterseg_b200 import metric
    hist = np.zeros((ev.class_num, ev.class_num))
    correct = labeled = 0
    for d in results:
        hist += d["hist"]
        correct += d["correct"]
        labeled += d["labeled"]
    iu, mean_iu, _, acc = metric.compute_score(hist, correct, labeled)
    line = "\n".join("%d %s\t%.3f%%" % (i + 1, n, u * 100) for i, (n, u) in enumerate(zip(ev.dataset.get_class_names(), iu)))
    return line + "\nmean_IU %.3f%% mean_pixel_ACC %.3f%%" % (mean_iu * 100, acc * 100), mean_iu


class StandInEvaluator:
    """the attributes tools/engine/evaluator.py:17-44 sets, and originals that record that they ran"""

    def __init__(self, dataset, network, multi_scales=(1,), is_flip=False, out_idx=0, threds=3):
        self.dataset, self.ndata, self.class_num = dataset, dataset.get_length(), 19
        self.image_mean, self.image_std = MEAN, STD
        self.multi_scales, self.is_flip, self.network, self.out_idx, self.threds = list(multi_scales), is_flip, network, out_idx, threds
        self.devices, self.config, self.logger, self.save_path, self.show_image, self.show_prediction = [0], None, None, None, False, False
        self.original_calls = []
        self.seen = []

    def run_online(self):
        self.original_calls.append("run_online")
        return "original", 0.0

    def run_online_multiprocess(self):
        self.original_calls.append("run_online_multiprocess")
        return "original", 0.0

    def compute_metric(self, results):
        self.seen.extend(results)
        return _compute_metric(self, results)


def _patched_class():
    from fasterseg_b200 import evaluator
    cls = type("Evaluator", (StandInEvaluator,), {})
    evaluator.install(types.SimpleNamespace(Evaluator=cls))
    return cls


def _reference_labels(model, img_rgb, out_idx=None):
    """tools/engine/evaluator.py:297-339 restated: normalise on the host, model(x) in fp32, exp, argmax; also our labels (the fused
    kernel's argmax = predict_labels on the uint8 frame) and the fp32 logits"""
    x = ((img_rgb.astype(np.float32) / 255.0 - MEAN) / STD).astype(np.float32).transpose(2, 0, 1)[None]
    with torch.no_grad():
        score = model(torch.from_numpy(np.ascontiguousarray(x)).cuda())
        if out_idx is not None:
            score = score[out_idx]
        logits = score[0].float()
        ref = torch.exp(logits).argmax(0).to(torch.uint8)
        u8 = torch.from_numpy(np.ascontiguousarray(img_rgb)).cuda()[None].permute(0, 3, 1, 2)
        ours = model.predict_labels(u8)[0] if out_idx is None else model.predict_labels(u8, head=out_idx)[0]
    return logits, ref, ours


def _expected(model, ds, out_idx=None):
    """hist / labeled / correct of the reference arithmetic.  A label may differ from ours only where the two classes' fp32
    logits are exp-tied (the reference's argmax of exp picks the first) or a rounding step apart (model(x) upsamples through the
    logits kernel, whose interpolation rounds differently from the argmax kernel's); there ours is taken, and the count reported."""
    from fasterseg_b200 import metric
    hist, labeled, correct, differ = np.zeros((19, 19), np.int64), 0, 0, 0
    for i in range(ds.get_length()):
        d = ds[i]
        logits, ref, ours = _reference_labels(model, np.ascontiguousarray(d["data"]), out_idx)
        mism = ref != ours
        if bool(mism.any()):
            lr = logits.gather(0, ref.long()[None])[0][mism]
            lo = logits.gather(0, ours.long()[None])[0][mism]
            exp_tie = torch.exp(lr) == torch.exp(lo)
            ulp = torch.finfo(torch.float32).eps * torch.maximum(lr.abs(), lo.abs())
            near = (lr - lo).abs() <= 4 * ulp
            assert bool((exp_tie | near).all()), "label differs at a pixel whose logits are %s apart" % float((lr - lo).abs().max())
            differ += int(mism.sum())
        lab = ref.clone()
        lab[mism] = ours[mism]
        p, g = lab.cpu().numpy(), d["label"]
        k = (g >= 0) & (g < 19)
        hist += np.bincount(19 * g[k].astype(int) + p[k].astype(int), minlength=19 * 19).reshape(19, 19)
        labeled += int(k.sum())
        correct += int((p[k] == g[k]).sum())
    print("labels differing from the reference arithmetic at exp- or rounding-tied pixels: %d" % differ)
    return hist, labeled, correct


def _check(ev, result, want):
    hist, labeled, correct = want
    assert ev.original_calls == []
    assert len(ev.seen) == 1
    got = ev.seen[0]
    assert np.array_equal(got["hist"], hist) and got["labeled"] == labeled and got["correct"] == correct
    line, miou = _compute_metric(ev, [{"hist": hist, "labeled": labeled, "correct": correct}])
    assert result == (line, miou)


def _student():
    model, g = _build_student(1)
    model = model.cuda().eval()
    _load_seeded(model, g, 77)
    return model


def test_patched_evaluator_on_the_student_matches_the_reference_arithmetic():
    model = _student()
    ds = SyntheticSet(6, 1024, 2048, seed=11)
    cls = _patched_class()
    ev = cls(ds, model)
    result = ev.run_online_multiprocess()
    _check(ev, result, _expected(model, ds))
    ev2 = cls(ds, model, threds=0)
    assert ev2.run_online() == result and ev2.original_calls == []


def _supernet(mode):
    model = _build_supernet(6).cuda()
    own = model.state_dict()
    for k, v in make_sd().items():
        own[k].copy_(v)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eps, m.momentum = orc.BN_EPS, orc.BN_MOMENTUM
    model.eval()
    model.arch_idx, model.prun_mode = 0, mode
    return model


@pytest.mark.parametrize("mode", ["max", "min"])
def test_patched_evaluator_on_the_supernet_matches_the_reference_arithmetic(mode):
    model = _supernet(mode)
    ds = SyntheticSet(2, 512, 1024, seed=12)
    cls = _patched_class()
    for out_idx in range(5):
        ev = cls(ds, model, out_idx=out_idx)
        result = ev.run_online_multiprocess()
        _check(ev, result, _expected(model, ds, out_idx))


def test_device_path_leaves_the_driver_rng_streams_alone_under_arch_ratio():
    model = _supernet(None)
    model.arch_idx = 1                                    # prun_modes[1] == 'arch_ratio': gumbel draws from torch's generator
    ds = SyntheticSet(2, 256, 512, seed=13)
    torch.manual_seed(5)
    np.random.seed(6)
    t0, n0 = torch.get_rng_state(), np.random.get_state()
    ev = _patched_class()(ds, model, out_idx=2)
    ev.run_online_multiprocess()
    assert ev.original_calls == [] and len(ev.seen) == 1
    assert torch.equal(torch.get_rng_state(), t0)
    n1 = np.random.get_state()
    assert n1[0] == n0[0] and np.array_equal(n1[1], n0[1]) and n1[2:] == n0[2:]
    with torch.no_grad():                                 # without the fork the eval forward does move torch's stream
        model(torch.zeros(1, 3, 256, 512, device="cuda"))
    assert not torch.equal(torch.get_rng_state(), t0)
    model.prun_mode = "random"                            # 'random' widths come from numpy
    np.random.set_state(n0)
    ev = _patched_class()(ds, model, out_idx=0)
    ev.run_online()
    n2 = np.random.get_state()
    assert np.array_equal(n2[1], n0[1]) and n2[2] == n0[2]


def test_evaluations_the_device_path_does_not_cover_run_the_original_method():
    model = _student()
    ds = SyntheticSet(1, 64, 128, seed=14)
    cls = _patched_class()
    for kw in (dict(is_flip=True), dict(multi_scales=(0.75, 1.0))):
        ev = cls(ds, model, **kw)
        assert ev.run_online_multiprocess() == ("original", 0.0) and ev.run_online() == ("original", 0.0)
        assert ev.original_calls == ["run_online_multiprocess", "run_online"] and ev.seen == []


# ---- the reference's own evaluator, where build() kept a copy of the reference ------------------------------------------------------
def _reference_seg_evaluator():
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
        ev_mod = importlib.import_module("engine.evaluator")
        seg_eval = importlib.import_module("eval")
    finally:
        sys.path[:] = old_path
        for n in set(sys.modules) - before:
            f = getattr(sys.modules[n], "__file__", None) or ""
            if os.path.realpath(f).startswith(os.path.realpath(root)):
                del sys.modules[n]
    return ev_mod, seg_eval.SegEvaluator


def test_reference_seg_evaluator_unpatched_and_patched_agree():
    from fasterseg_b200 import evaluator
    ev_mod, SegEvaluator = _reference_seg_evaluator()
    model = _student()
    ds = SyntheticSet(2, 1024, 2048, seed=15)
    config = types.SimpleNamespace(num_classes=19, eval_scale_array=[1], eval_crop_size=1024, eval_stride_rate=5 / 6, background=0)
    seen = []

    class Capturing(SegEvaluator):
        def compute_metric(self, results):
            seen.append([dict(r) for r in results])
            return super().compute_metric(results)

    ev = Capturing(ds, 19, MEAN, STD, model, [1], False, 0, config=config)
    saved = {n: ev_mod.Evaluator.__dict__[n] for n in evaluator.PATCHED}
    ref_line, ref_miou = ev.run_online()                 # unpatched: the reference's per-image loop
    try:
        evaluator.install(ev_mod)
        seen.clear()
        line, miou = ev.run_online()
    finally:
        for n, f in saved.items():
            setattr(ev_mod.Evaluator, n, f)
    assert len(seen) == 1 and len(seen[0]) == 1
    want = _expected(model, ds)
    got = seen[0][0]
    assert np.array_equal(got["hist"], want[0]) and got["labeled"] == want[1] and got["correct"] == want[2]
    if ref_line == line:
        assert ref_miou == miou
    else:   # only where _expected reported exp- / rounding-tied pixels
        assert abs(ref_miou - miou) < 1e-6
