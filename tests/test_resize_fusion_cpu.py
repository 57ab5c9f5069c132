"""Host side of the fused resizes (fsb_conv_fwd_half, fsb_bilinear_fwd_half and the network's plan in model_seg._trunk):
the 2x2 locality the kernels rely on, checked exhaustively with the library's fp32 index rule, and the launch list of the
student frame on the CPU stand-in backend."""
import contextlib
import os
import re

import numpy as np
import torch

from fasterseg_b200 import functional as F_
from fasterseg_b200 import roofline
from tests import cpu_backend
from tests.test_boundary_cpu import _build_student

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def _standin():
    """the CPU stand-in backend, with the /2 output (out_half) of F_.conv_fwd and F_.bilinear: one call where the library makes it in
    the same launch (fsb_conv_fwd_half, fsb_bilinear_fwd_half for an exact x2), a second bilinear call otherwise"""
    with cpu_backend.installed():
        conv, bil = F_.conv_fwd, F_.bilinear

        def conv_fwd(*a, out_half=None, **kw):
            y = conv(*a, **kw)
            if out_half is not None:
                bil(y, (y.shape[2] // 2, y.shape[3] // 2), out=out_half)
            return y

        def bilinear(x, size, relu=False, out=None, out_half=None):
            y = bil(x, size, relu=relu, out=out)
            if out_half is not None:
                half = (y.shape[2] // 2, y.shape[3] // 2)
                (bil if tuple(y.shape[2:]) == (2 * x.shape[2], 2 * x.shape[3]) else F_.bilinear)(y, half, out=out_half)
            return y

        F_.conv_fwd, F_.bilinear = conv_fwd, bilinear
        try:
            yield
        finally:
            F_.conv_fwd, F_.bilinear = conv, bil


def _local_max():
    src = open(os.path.join(ROOT, "fasterseg_b200", "csrc", "fsb_internal.h")).read()
    return int(re.search(r"constexpr int kBilinearLocalMax = (\d+);", src).group(1))


def _src_index(n_out, n_in):
    """(i0, i1) of every output index: src_index / ac_scale of fsb_common.cuh in float32 (scale * float(dst), truncation, clamp)"""
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0)
    src = np.float32(scale) * np.arange(n_out, dtype=np.float32)
    i0 = np.minimum(src.astype(np.int64), n_in - 1)
    return i0, i0 + (i0 < n_in - 1)


def test_bilinear_half_footprints_are_local_for_every_even_extent():
    limit = _local_max()
    assert limit == 4096
    for n in range(2, limit + 1, 2):
        # /2 of an n-pixel axis: output pixel i reads only pixels 2i and 2i + 1 (its aligned 2x2 block)
        i0, i1 = _src_index(n // 2, n)
        k = np.arange(n // 2)
        assert np.all(i0 // 2 == k) and np.all(i1 // 2 == k), n
        # exact x2 of an n/2-pixel axis: output pixels 2k and 2k + 1 read only source pixels k - 1 .. k + 1
        j0, j1 = _src_index(n, n // 2)
        lo, hi = np.minimum(j0[0::2], j0[1::2]), np.maximum(j1[0::2], j1[1::2])
        assert np.all(lo >= k - 1) and np.all(hi <= k + 1), n


def test_student_frame_launch_list_with_fused_resizes():
    """arch_1 at 1024x2048: the 12 bilinear /2 launches of the zoomed cells and the 3 skip copies of the refines are gone; every
    other launch stays, and the logits are those of the unfused frame."""
    with _standin():
        model, _ = _build_student(1)
        model.eval()
        model.logits_dtype = torch.float16
        x = torch.zeros(1, 3, 1024, 2048)
        with torch.no_grad():
            before = roofline.trace_launches(lambda: model(x))
            model.fuse_resizes = True
            first = roofline.trace_launches(lambda: model(x))      # records the plan for this input size
            after = roofline.trace_launches(lambda: model(x))
            small = torch.randn(1, 3, 256, 512, generator=torch.Generator().manual_seed(3))
            model(small)
            fused = model(small)
            model.fuse_resizes = False
            plain = model(small)
    kinds = [r["kernel"] for r in after]
    assert len(before) == len(first) == 74 and len(after) == len(before) - 15
    assert "copy_channels" not in kinds and [r["kernel"] for r in before].count("copy_channels") == 3
    assert [r for r in before if r["kernel"] == "bilinear" and _is_down2(r["shape"])] != []
    assert [r for r in after if r["kernel"] == "bilinear" and _is_down2(r["shape"])] == []
    assert kinds.count("bilinear") == 13 and kinds.count("conv") == 44
    assert torch.equal(fused, plain)


def _is_down2(shape):
    hi, wi, ho, wo = map(int, re.search(r"(\d+)x(\d+) -> (\d+)x(\d+)", shape).groups())
    return (ho, wo) == (hi // 2, wi // 2)


def test_plan_keeps_the_unfused_path_in_training_autograd_and_by_default_on_the_cpu():
    with _standin():
        model, _ = _build_student(1)
        model.eval()
        x = torch.zeros(1, 3, 64, 128)
        assert not model._fuse_resizes_for(x)             # None: CUDA inputs only
        model.fuse_resizes = True
        with torch.no_grad():
            assert model._fuse_resizes_for(x)
        assert not model._fuse_resizes_for(x)             # autograd on
        model.train()
        with torch.no_grad():
            assert not model._fuse_resizes_for(x)
        model.eval()
        model.fuse_resizes = None
        with torch.no_grad():
            model(x)
        assert model.__dict__.get("_fsb_resize_plans") is None      # nothing recorded while the plan is off
        model.fuse_resizes = True
        with torch.no_grad():
            model(x)
    plan = model.__dict__["_fsb_resize_plans"][(1, 3, 64, 128)]
    assert len(plan.reads_half) == 12 and len(plan.half) == 11 and len(plan.skip) == 3
    assert plan.shapes[0] == (1, 32, 8, 16)


def test_producers_with_batch_statistics_still_fill_the_half_map():
    """a network put in eval mode before build_structure keeps train-mode BatchNorms in its cells: their convs normalise with batch
    statistics and the /2 map comes from a separate resize, with the same values as the unfused forward"""
    with _standin():
        model, _ = _build_student(1)
        model.eval()
        model.cells["1-0"].train()          # producer of the first zoomed cell's input
        x = torch.randn(1, 3, 128, 256, generator=torch.Generator().manual_seed(5))
        with torch.no_grad():
            model.fuse_resizes = True
            model(x)
            fused = model(x)
            model.fuse_resizes = False
            plain = model(x)
    assert torch.equal(fused, plain)
