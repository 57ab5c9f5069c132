"""The drivers' training step on the fused criteria, on the GPU, against the reference's own code from the copy that build() keeps in
oracle/_ref/FasterSeg (skipped where that copy is absent): the patched ProbOhemCrossEntropy2d on lazy and on dense logits against
the reference's forward, no host synchronisation in it, the patched Seg_Metrics.update against the reference's on the
materialised logits, and train.py's own train() through both paths (DESIGN section 3.9)."""
import math
import os
import sys

import pytest
import torch

from fasterseg_b200 import functional as F_
from fasterseg_b200.losses import LazyLogits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def driver():
    sys.path.insert(0, ROOT)
    from tools import driver_step_bench as D
    if not os.path.isfile(os.path.join(D.REF, "train", "train.py")):
        pytest.skip("no copy of the reference in oracle/_ref")
    with D.loaded_train_driver() as drv:
        yield D, drv


def _grad_close(got, ref, what):
    scale = float(ref.abs().max()) + 1e-30
    err = float((got.double() - ref.double()).abs().max())
    assert err <= 2e-3 * scale, "%s: max |diff| %.3e vs max |ref| %.3e" % (what, err, scale)


def _target(shape, seed, p_ignore=0.05, labels=19):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, labels, shape, generator=g)
    t[torch.rand(shape, generator=g) < p_ignore] = 255
    return t.cuda()


def _lowres(x):
    N, C, H, W = x.shape
    buf = F_.empty_nhwc(N, C, H, W, x.device)
    buf.copy_(x.half())
    return buf.requires_grad_(True)


def _check_ohem(crit, low, size, tgt, what):
    """patched forward on LazyLogits(low) vs the reference's forward on the materialised logits: loss and d/d(low)"""
    x_ref, x = _lowres(low), _lowres(low)
    want = type(crit).forward._fsb_original(crit, LazyLogits(x_ref, size).dense(), tgt.clone())
    got = crit(LazyLogits(x, size), tgt)
    if math.isnan(float(want)):
        assert math.isnan(float(got)), what
        return
    assert float(got) == pytest.approx(float(want), rel=2e-5), what
    want.backward()
    got.backward()
    _grad_close(x.grad.float(), x_ref.grad.float(), what)


@pytest.mark.parametrize("factor", [8, 16, 32])
def test_patched_ohem_on_lazy_logits_matches_the_reference(driver, factor):
    D, drv = driver
    B, H, W = 2, 512, 1024
    crit, _ = D.driver_criteria(drv, B, (H, W))                     # train.py:62-63
    g = torch.Generator().manual_seed(factor)
    low = (torch.randn(B, 19, H // factor, W // factor, generator=g) * 2.5).cuda()
    _check_ohem(crit, low, (H, W), _target((B, H, W), factor), "x%d" % factor)


# branch -> (scale of the logits, fraction ignored, min_kept, the target is the argmax of the logits)
BRANCHES = {
    "fewer_valid_than_min_kept": (2.5, 0.99, 4096, False),
    "everything_ignored": (2.5, 1.0, 4096, False),
    "kth_below_thresh": (1.0, 0.05, 4096, False),
    "kth_above_thresh": (12.0, 0.05, 4096, True),
}


@pytest.mark.parametrize("name", sorted(BRANCHES))
def test_patched_ohem_branches_on_lazy_logits(driver, name):
    _, drv = driver
    scale, p_ign, min_kept, confident = BRANCHES[name]
    B, h, w, size = 2, 16, 32, (128, 256)
    g = torch.Generator().manual_seed(len(name))
    low = (torch.randn(B, 19, h, w, generator=g) * scale).cuda()
    tgt = _target((B,) + size, len(name), p_ign)
    if confident:
        up = LazyLogits(_lowres(low).detach(), size).dense()
        tgt = torch.where(tgt == 255, tgt, up.argmax(1))
    crit = drv.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=min_kept, use_weight=False)
    _check_ohem(crit, low, size, tgt, name)


@pytest.mark.parametrize("shape", [(3, 32, 64), (2, 28, 56)])             # configs[2] / configs[4] at 1/8 (gt_down_sampling = 8)
def test_patched_ohem_on_dense_logits_matches_the_reference(driver, shape):
    _, drv = driver
    B, H, W = shape
    crit = drv.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=int(B * H * W // 16), use_weight=False)
    g = torch.Generator().manual_seed(H)
    pred = (torch.randn(B, 19, H, W, generator=g) * 2.5).cuda()
    tgt = _target((B, H, W), W)
    p_ref, p = pred.clone().requires_grad_(True), pred.clone().requires_grad_(True)
    want = type(crit).forward._fsb_original(crit, p_ref, tgt.clone())
    got = crit(p, tgt)
    assert float(got) == pytest.approx(float(want), rel=2e-5)
    want.backward()
    got.backward()
    _grad_close(p.grad, p_ref.grad, "dense %s" % (shape,))


@pytest.mark.parametrize("lazy", [True, False])
def test_patched_ohem_does_not_synchronise_the_host(driver, lazy):
    _, drv = driver
    B, H, W = 2, 256, 512
    crit = drv.ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=B * H * W // 16, use_weight=False)
    low = torch.randn(B, 19, H // 8, W // 8, device="cuda") * 2.5
    pred = LazyLogits(_lowres(low), (H, W)) if lazy else torch.randn(B, 19, H // 8, W // 8, device="cuda", requires_grad=True)
    tgt = _target((B, H, W) if lazy else (B, H // 8, W // 8), 5)
    crit(pred, tgt)                                                      # warm-up: first-call allocations
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = crit(pred, tgt)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert math.isfinite(float(loss))


def _out_of_range_target(shape, seed):
    t = _target(shape, seed, 0.05)
    g = torch.Generator().manual_seed(seed + 1)
    odd = (torch.rand(shape, generator=g) < 0.05).cuda()
    return torch.where(odd, torch.tensor([19, 300, -1], device="cuda")[torch.randint(0, 3, shape, generator=g).cuda()], t)


def test_patched_seg_metrics_equal_the_reference_update(driver):
    D, drv = driver
    Metrics = drv.seg_metrics.Seg_Metrics
    teacher, student = D.build_driver_models()
    teacher.lazy_logits = student.lazy_logits = True
    B, H, W = 2, 512, 1024
    x = torch.randn(B, 3, H, W, device="cuda")
    with torch.no_grad():
        outs = [teacher.eval()(x), student.train()(x)[0]]
    for k, out in enumerate(outs):
        assert isinstance(out, LazyLogits)
        new, ref = Metrics(n_classes=19), Metrics(n_classes=19)
        for step in range(2):
            t = _out_of_range_target((B, H, W), 10 * k + step)
            new.update(out.data, t)
            Metrics.update._fsb_original(ref, out.data.dense(), t)
            assert new.total_inter.tolist() == ref.total_inter.tolist() and new.total_union.tolist() == ref.total_union.tolist()
        assert new.get_scores() == ref.get_scores() and ref.total_union.sum() > 0


class _Writer:
    def __init__(self):
        self.losses = []

    def add_scalar(self, tag, value, step):
        self.losses.append(float(value.detach()))


def _train(D, drv, steps, B=2, hw=(512, 1024)):
    models = D.build_driver_models()
    opt = torch.optim.SGD(models[1].parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
    ohem, kl = D.driver_criteria(drv, B, hw)
    drv.config.niters_per_epoch = steps
    writer = _Writer()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    mious = drv.train(D.SyntheticLoader(B, hw, steps), models, ohem, kl, opt, writer, 0)
    torch.cuda.synchronize()
    return [float(m) for m in mious], writer.losses, torch.cuda.max_memory_allocated()


def test_train_py_through_both_paths(driver):
    D, drv = driver
    with D.reference_path(drv):
        ref1, ref_loss1, _ = _train(D, drv, 1)
        ref2, ref_loss2, ref_peak = _train(D, drv, 2)
    new1, new_loss1, _ = _train(D, drv, 1)
    new2, new_loss2, new_peak = _train(D, drv, 2)
    print("\ntrain.py train(), batch 2 x 512 x 1024, 2 steps: peak memory %.2f GB (reference path) vs %.2f GB (fused path)"
          % (ref_peak / 2 ** 30, new_peak / 2 ** 30))
    assert new1 == ref1                                                  # step 1: the same mIoU description
    assert new_loss1[0] == pytest.approx(ref_loss1[0], rel=2e-5)
    assert len(new_loss2) == 2 and new_loss2[1] == pytest.approx(ref_loss2[1], rel=2e-3)
    assert new2 == pytest.approx(ref2, abs=1e-2)
    assert new_peak < ref_peak
