"""conv_tc residency: 160-thread CTAs (the MMA warpgroup and one producer warp) compiled for 3 CTAs per SM at N tiles of <= 64
channels and 2 at 96 / 128, and a launcher that sizes the shared memory for that residency, or for CTAs / SMs (rounded up) when
the grid fills fewer slots.

fsb_conv_residency (the CUDA occupancy calculator on the instance and shared memory the launcher picks) must report the planned
residency on the frame's large convs.  One multi-wave case per instance class (per-tap, window, Y_UP2, BN-train statistics
with fp32 output, data gradient) is checked against the CPU oracle at the tolerances of test_kernels_gpu.py /
test_conv_window_gpu.py, and twice in a row for the same bits, statistics rows included.
"""
import ctypes as C
import re

import numpy as np
import pytest
import torch

from oracle import fasterseg_oracle as orc
from tests import helpers as H

pytestmark = pytest.mark.gpu

REL = 1e-3
_INSTANCE = re.compile(r"conv_tc_(?:up2_)?kernel(?:<\s*(\d+),\s*(\d+),\s*(true|false)\s*>|ILi(\d+)ELi(\d+)ELb([01])E)")


def _F():
    from fasterseg_b200 import functional as F_
    return F_


def _planned(nt, ctas):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return min(3 if nt <= 64 else 2, -(-ctas // sms))


def _instances(fn, tmp_path):
    """[(BK, NT, window)] of the conv_tc launches of fn, read from the kernel nodes of a CUDA graph capture"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)  # kept for debug_dump only; never replayed
    g.enable_debug_mode()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    dot = tmp_path / "conv.dot"
    g.debug_dump(str(dot))
    out = []
    for m in _INSTANCE.finditer(dot.read_text()):
        bk, nt, win = (m.group(1), m.group(2), m.group(3)) if m.group(1) else (m.group(4), m.group(5), m.group(6))
        out.append((int(bk), int(nt), win in ("true", "1")))
    assert out, "no conv_tc launch captured"
    return sorted(set(out))


def _close(got, ref, rel=REL):
    got, ref = got.double(), ref.double()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    err = (got - ref).abs()
    bad = err > rel * ref.abs() + rel * rms
    assert not bad.any(), "max err %.3e (rms %.3e), %d/%d outside tolerance" % (err.max().item(), rms, int(bad.sum()), bad.numel())


def _rand(shape, seed, scale=1.0):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal(shape).astype(np.float32) * scale)


def _nhwc(x_nchw_f32):
    return x_nchw_f32.cuda().half().contiguous(memory_format=torch.channels_last)


def _problem(N, Cin, Cout, k, Hh, Ww, seed):
    x = _rand((N, Cin, Hh, Ww), seed).half().float()
    w = (_rand((Cout, Cin, k, k), seed + 1) * (2.0 / (Cin * k * k)) ** 0.5).half().float()
    scale = torch.from_numpy(np.random.RandomState(seed + 2).uniform(0.5, 1.5, Cout).astype(np.float32))
    shift = _rand((Cout,), seed + 3, 0.2)
    return x, w, scale, shift


def _bits(t):
    t = t.detach().contiguous().cpu()
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


# name, Cin, Cout, k, stride, H, W (input), CTAs -- the student frame's shapes (tools/conv_bench.py)
LAYERS = [
    ("stem.1.conv1", 32, 64, 3, 2, 512, 1024, 1024),
    ("stem.1.conv2", 64, 64, 3, 1, 256, 512, 1024),
    ("refines32.0", 192, 128, 3, 1, 64, 128, 192),
    ("ffm", 128, 128, 1, 1, 128, 256, 256),
    ("heads8.conv3x3", 128, 128, 3, 1, 128, 256, 256),
]


@pytest.mark.parametrize("layer", LAYERS, ids=[layer[0] for layer in LAYERS])
def test_frame_convs_reach_planned_residency(layer, tmp_path):
    from fasterseg_b200 import _lib
    F_ = _F()
    _, Cin, Cout, k, s, Hh, Ww, ctas = layer
    pad = k // 2
    x = F_.empty_nhwc(1, Cin, Hh, Ww, "cuda").normal_()
    wp = F_.pack_conv_weight(torch.randn(Cout, Cin, k, k, device="cuda") * 0.05, Cin, Cout, k)
    sc, sh = torch.ones(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
    (inst,) = _instances(lambda: F_.conv_fwd(x, wp, Cout, k, s, pad, sc, sh, relu=True), tmp_path)
    d = F_.make_conv_desc(1, Hh, Ww, Cin, Cout, k, s, pad, Cin, Cout, _lib.FSB_CONV_RELU | _lib.FSB_CONV_AFFINE)
    assert _lib.lib().fsb_conv_residency(C.byref(d)) == _planned(inst[1], ctas), inst


def test_residency_query_rejects_the_direct_kernel():
    from fasterseg_b200 import _lib
    F_ = _F()
    d = F_.make_conv_desc(1, 64, 64, 8, 16, 3, 1, 1, 8, 16, 0)  # Cin < 16: CUDA-core direct kernel
    assert _lib.lib().fsb_conv_residency(C.byref(d)) == -3  # FSB_ERR_UNSUPPORTED


def _twice(fn):
    a = fn()
    b = fn()
    torch.cuda.synchronize()
    return a, b


# N, Cin, Cout, k, stride, H, W: grids of more CTAs than SMs (the residency-sized shared memory)
FWD_CASES = [
    (1, 64, 128, 3, 2, 256, 256),   # per-tap, BK 64, NT 128 (2 per SM)
    (1, 32, 64, 3, 2, 256, 256),    # per-tap, BK 32, NT 64 (3 per SM)
    (1, 96, 96, 1, 1, 128, 128),    # per-tap 1x1, NT 96
    (1, 64, 64, 3, 1, 128, 256),    # window, NT 64
    (1, 128, 128, 3, 1, 128, 128),  # window, NT 128
]


@pytest.mark.parametrize("case", FWD_CASES)
def test_forward_matches_oracle_and_repeats(case, tmp_path):
    F_ = _F()
    N, Cin, Cout, k, s, Hh, Ww = case
    pad = k // 2
    x, w, scale, shift = _problem(N, Cin, Cout, k, Hh, Ww, Cin * 7 + Cout + k)
    ref = torch.relu(orc.conv2d(x, w, None, s, pad) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, k)
    xg, sc, sh = _nhwc(x), scale.cuda(), shift.cuda()
    (inst,) = _instances(lambda: F_.conv_fwd(xg, wp, Cout, k, s, pad, sc, sh, relu=True), tmp_path)
    assert inst[2] == (k == 3 and s == 1), inst
    a, b = _twice(lambda: F_.conv_fwd(xg, wp, Cout, k, s, pad, sc, sh, relu=True))
    _close(a.float().cpu(), ref)
    assert torch.equal(_bits(a), _bits(b))


def test_up2_matches_oracle_and_repeats():
    """FSB_CONV_Y_UP2 (conv_tc_up2_kernel): the output is nearest x2 of the conv, written by four lattice stores"""
    F_ = _F()
    N, Cin, Cout, Hh, Ww = 1, 64, 64, 128, 128
    x, w, scale, shift = _problem(N, Cin, Cout, 3, Hh, Ww, 77)
    ref = torch.relu(orc.conv2d(x, w, None, 1, 1) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    ref = ref.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, 3)
    xg, sc, sh = _nhwc(x), scale.cuda(), shift.cuda()
    a, b = _twice(lambda: F_.conv_fwd(xg, wp, Cout, 3, 1, 1, sc, sh, relu=True, up2=True))
    assert tuple(a.shape) == (N, Cout, 2 * Hh, 2 * Ww)
    _close(a.float().cpu(), ref)
    assert torch.equal(_bits(a), _bits(b))


@pytest.mark.parametrize("case", [(1, 64, 64, 128, 256), (1, 128, 128, 64, 256)])
def test_statistics_fp32_matches_oracle_and_repeats(case):
    """BN-train forward: fp32 raw output and one partial statistics row per tile; the rows repeat bit for bit"""
    F_ = _F()
    N, Cin, Cout, Hh, Ww = case
    x, w, _, _ = _problem(N, Cin, Cout, 3, Hh, Ww, 300 + Cin)
    ref = orc.conv2d(x, w, None, 1, 1)
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, 3)
    xg = _nhwc(x)
    runs = []
    for _ in range(2):
        stats = F_.conv_stats_buffer(xg, Cout, 3, 1, 1)
        stats.fill_(float("nan"))  # every entry must be written
        y = F_.conv_fwd(xg, wp, Cout, 3, 1, 1, stats=stats, out_f32=True)
        runs.append((y, stats))
    torch.cuda.synchronize()
    (y, stats), (y2, stats2) = runs
    assert y.dtype == torch.float32
    _close(y.cpu(), ref)
    assert torch.equal(_bits(y), _bits(y2)) and torch.equal(_bits(stats), _bits(stats2))
    s = F_.rowsum(stats)[0].cpu().double()
    np.testing.assert_allclose(s[:Cout].numpy(), ref.double().sum(dim=(0, 2, 3)).numpy(), rtol=2e-4, atol=2e-2)
    np.testing.assert_allclose(s[Cout:].numpy(), ref.double().pow(2).sum(dim=(0, 2, 3)).numpy(), rtol=2e-4, atol=2e-2)


@pytest.mark.parametrize("case", [(1, 64, 64, 1, 128, 128), (1, 32, 64, 2, 128, 128)])
def test_dgrad_matches_oracle_and_repeats(case):
    """data gradient (stride 1: one conv of dy with the flipped, transposed weights; stride 2: custom tap tables per parity)"""
    F_ = _F()
    N, Cin, Cout, s, Hh, Ww = case
    x = _rand((N, Cin, Hh, Ww), 90 + Cin).half().float().requires_grad_(True)
    w = (_rand((Cout, Cin, 3, 3), 91 + Cin) * (2.0 / (Cin * 9)) ** 0.5).half().float()
    y = orc.conv2d(x, w, None, s, 1)
    gy = _rand(tuple(y.shape), 92 + Cin).half().float()
    y.backward(gy)
    wg = w.cuda()
    wt = F_.pack_conv_weight_dgrad(wg, Cin, Cout, 3)
    gyg = _nhwc(gy)
    a, b = _twice(lambda: F_.conv_dgrad(gyg, wg, (N, Cin, Hh, Ww), Cin, Cout, 3, s, 1, wpacked_t=wt))
    err = H.rel_err(a.float().cpu().numpy(), x.grad.numpy())
    assert err < 1.5e-3, "dgrad rel err %.3e" % err
    assert torch.equal(_bits(a), _bits(b))
