"""Window mode of conv_tc (3x3 stride-1 convs: one halo window of the input per 64-channel chunk, the nine taps read from it
through shifted descriptors) against the CPU oracle, on the cases that stress it: ragged tiles, 8 x 16 tiles (Wo < 16),
windows at the edges of a batch of images, every Cin residue mod 64, inputs that are channel slices of a wider buffer,
desc.off_h/off_w, fused BN-train statistics with fp32 output, and the stride-1 data gradient.  The cases run with
FSB_CONV_TC2=1 (window mode on any grid) and check, from the kernel nodes of a CUDA graph capture, that the launch ran a
window instance of conv_tc_kernel; one test checks the default choice between the window and the per-tap mode.

Tolerance as in test_kernels_gpu.py: operands rounded to fp16 once, fp32 accumulation, result rounded once.
"""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from oracle import fasterseg_oracle as orc
from tests import helpers as H

pytestmark = pytest.mark.gpu

REL = 1e-3
# demangled (conv_tc_kernel<64, 64, true>) or mangled (conv_tc_kernelILi64ELi64ELb1E) name of a window-mode instance
_WINDOW = re.compile(r"conv_tc_kernel(<\s*64,\s*\d+,\s*true\s*>|ILi64ELi\d+ELb1E)")
_PER_TAP = re.compile(r"conv_tc_kernel(<\s*\d+,\s*\d+,\s*false\s*>|ILi\d+ELi\d+ELb0E)")


def _F():
    from fasterseg_b200 import functional as F_
    return F_


@pytest.fixture(autouse=True)
def _window_mode(lib_option):
    # these small problems have fewer CTAs than SMs, where the default is the per-tap mode: force the window mode
    lib_option("FSB_CONV_TC2", 1)


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


def _run_in_mode(fn, pattern, tmp_path):
    """-> fn()'s result; asserts that fn launches conv_tc_kernel only in the instances `pattern` matches, read from the kernel
    nodes of a CUDA graph capture of fn (its debug dump names each node's function)"""
    out = fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)  # the captured cudaGraph_t stays for debug_dump; the graph is never replayed
    g.enable_debug_mode()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    dot = tmp_path / "conv.dot"
    g.debug_dump(str(dot))
    names = re.findall(r"conv_tc_kernel[\w<>, ]*", dot.read_text())
    assert names and all(pattern.search(n) for n in names), "conv_tc ran another mode than %s: %s" % (pattern.pattern, names)
    return out


def _ref_conv(x, w, pad, off=(0, 0)):
    """y[ho, wo] = sum x[ho + r - pad + off_h, wo + s - pad + off_w] * w[r, s] (zero outside the image)"""
    xp = TF.pad(x, (pad, pad, pad, pad))[:, :, off[0]:, off[1]:]
    return orc.conv2d(xp, w, None, 1, 0)


def _problem(N, Cin, Cout, Hh, Ww, seed):
    x = _rand((N, Cin, Hh, Ww), seed).half().float()
    w = (_rand((Cout, Cin, 3, 3), seed + 1) * (2.0 / (Cin * 9)) ** 0.5).half().float()
    scale = torch.from_numpy(np.random.RandomState(seed + 2).uniform(0.5, 1.5, Cout).astype(np.float32))
    shift = _rand((Cout,), seed + 3, 0.2)
    return x, w, scale, shift


@pytest.mark.parametrize("case,window", [((1, 64, 64, 128, 256), True), ((1, 128, 128, 32, 64), False),
                                         ((2, 96, 64, 64, 128), True)])
def test_default_picks_window_mode_on_large_grids(case, window, lib_option, tmp_path):
    """unset FSB_CONV_TC2: inference convs take the window mode when the grid has more CTAs than SMs (bandwidth-bound), the
    per-tap mode otherwise; BN-train convs (statistics) stay per-tap"""
    lib_option("FSB_CONV_TC2", -1)
    F_ = _F()
    N, Cin, Cout, Hh, Ww = case
    x, w, scale, shift = _problem(N, Cin, Cout, Hh, Ww, 500 + Cin)
    ref = torch.relu(_ref_conv(x, w, 1) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, 3)
    xg, sc, sh = _nhwc(x), scale.cuda(), shift.cuda()
    y = _run_in_mode(lambda: F_.conv_fwd(xg, wp, Cout, 3, 1, 1, sc, sh, relu=True), _WINDOW if window else _PER_TAP, tmp_path)
    _close(y.float().cpu(), ref)
    stats = F_.conv_stats_buffer(xg, Cout, 3, 1, 1)
    _run_in_mode(lambda: F_.conv_fwd(xg, wp, Cout, 3, 1, 1, stats=stats, out_f32=True), _PER_TAP, tmp_path)


WINDOW_CASES = [
    # N, Cin, Cout, H, W, off
    (1, 64, 64, 13, 37, (0, 0)),      # ragged 16 x 8 tiles in both directions
    (1, 64, 64, 21, 12, (0, 0)),      # Wo < 16: 8 x 16 tiles, ragged in height
    (2, 96, 48, 35, 9, (0, 0)),       # 8 x 16 tiles, two images
    (3, 64, 32, 10, 20, (0, 0)),      # windows at the edges of neighbouring images
    (3, 32, 64, 17, 7, (0, 0)),
    (1, 16, 16, 8, 8, (0, 0)),
    (1, 32, 128, 20, 36, (0, 0)),
    (2, 48, 80, 9, 13, (0, 0)),
    (1, 80, 48, 5, 97, (0, 0)),
    (1, 96, 64, 12, 40, (0, 0)),
    (1, 192, 128, 24, 40, (0, 0)),
    (1, 256, 256, 6, 20, (0, 0)),
    (1, 64, 96, 14, 30, (1, 1)),      # desc.off_h / off_w
    (2, 80, 32, 11, 19, (1, 0)),
]


@pytest.mark.parametrize("case", WINDOW_CASES)
def test_window_conv_matches_oracle(case, tmp_path):
    F_ = _F()
    N, Cin, Cout, Hh, Ww, off = case
    x, w, scale, shift = _problem(N, Cin, Cout, Hh, Ww, hash(case) % 100000)
    ref = torch.relu(_ref_conv(x, w, 1, off) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, 3)
    xg, sc, sh = _nhwc(x), scale.cuda(), shift.cuda()
    y = _run_in_mode(lambda: F_.conv_fwd(xg, wp, Cout, 3, 1, 1, sc, sh, relu=True, off=off), _WINDOW, tmp_path)
    assert tuple(y.shape) == tuple(ref.shape)
    _close(y.float().cpu(), ref)


@pytest.mark.parametrize("Cin", [16, 32, 48, 80, 96, 192, 256])
def test_window_conv_reads_only_its_channel_slice(Cin, lib_option, tmp_path):
    """x = channels [24, 24 + Cin) of a wider buffer whose other channels are NaN: a ragged last chunk must be zero-filled,
    never read from the neighbouring channels.  The per-tap mode on the same problem agrees to fp32 summation order."""
    F_ = _F()
    N, Cout, Hh, Ww = 2, 48, 11, 29
    x, w, scale, shift = _problem(N, Cin, Cout, Hh, Ww, 900 + Cin)
    ref = torch.relu(_ref_conv(x, w, 1) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    wide = F_.empty_nhwc(N, Cin + 48, Hh, Ww, "cuda")
    wide.fill_(float("nan"))
    wide[:, 24:24 + Cin].copy_(_nhwc(x))
    xs = wide[:, 24:24 + Cin]
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, 3)
    sc, sh = scale.cuda(), shift.cuda()
    y = _run_in_mode(lambda: F_.conv_fwd(xs, wp, Cout, 3, 1, 1, sc, sh, relu=True), _WINDOW, tmp_path)
    assert not torch.isnan(y).any()
    _close(y.float().cpu(), ref)
    lib_option("FSB_CONV_TC2", 0)
    y0 = _run_in_mode(lambda: F_.conv_fwd(xs, wp, Cout, 3, 1, 1, sc, sh, relu=True), _PER_TAP, tmp_path)
    _close(y0.float().cpu(), y.float().cpu())


@pytest.mark.parametrize("case", [(3, 64, 96, 40, 72), (2, 32, 48, 9, 14), (1, 80, 64, 33, 10)])
def test_window_conv_statistics_and_fp32_output(case, tmp_path):
    """BN-train forward: fp32 raw output and one partial statistics row per 128-pixel tile, summed against the oracle."""
    F_ = _F()
    N, Cin, Cout, Hh, Ww = case
    x, w, _, _ = _problem(N, Cin, Cout, Hh, Ww, 40 + Cin)
    ref = _ref_conv(x, w, 1)
    xg = _nhwc(x)
    stats = F_.conv_stats_buffer(xg, Cout, 3, 1, 1)
    tw = 16 if Ww >= 16 else 8
    assert stats.shape[0] == N * -(-Ww // tw) * -(-Hh // (128 // tw))  # the 16 x 8 / 8 x 16 tiles of the per-tap mode
    stats.fill_(float("nan"))  # every entry must be written
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, 3)
    y = _run_in_mode(lambda: F_.conv_fwd(xg, wp, Cout, 3, 1, 1, stats=stats, out_f32=True), _WINDOW, tmp_path)
    assert y.dtype == torch.float32
    _close(y.cpu(), ref)
    s = F_.rowsum(stats)[0].cpu().double()
    np.testing.assert_allclose(s[:Cout].numpy(), ref.double().sum(dim=(0, 2, 3)).numpy(), rtol=2e-4, atol=2e-2)
    np.testing.assert_allclose(s[Cout:].numpy(), ref.double().pow(2).sum(dim=(0, 2, 3)).numpy(), rtol=2e-4, atol=2e-2)


@pytest.mark.parametrize("case", [(2, 64, 64, 16, 24), (1, 48, 96, 13, 10), (2, 96, 32, 9, 37)])
def test_window_dgrad_stride1(case, tmp_path):
    """stride-1 data gradient: a 3x3 stride-1 conv of dy with the flipped, transposed weights"""
    F_ = _F()
    N, Cin, Cout, Hh, Ww = case
    x = _rand((N, Cin, Hh, Ww), 70 + Cin).half().float().requires_grad_(True)
    w = (_rand((Cout, Cin, 3, 3), 71 + Cin) * (2.0 / (Cin * 9)) ** 0.5).half().float()
    y = orc.conv2d(x, w, None, 1, 1)
    gy = _rand(tuple(y.shape), 72 + Cin).half().float()
    y.backward(gy)
    wg = w.cuda()
    wt = F_.pack_conv_weight_dgrad(wg, Cin, Cout, 3)
    gyg = _nhwc(gy)
    dx = _run_in_mode(lambda: F_.conv_dgrad(gyg, wg, (N, Cin, Hh, Ww), Cin, Cout, 3, 1, 1, wpacked_t=wt), _WINDOW, tmp_path)
    err = H.rel_err(dx.float().cpu().numpy(), x.grad.numpy())
    assert err < 1.5e-3, "dgrad rel err %.3e" % err
