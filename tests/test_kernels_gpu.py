"""GPU parity tests of the individual CUDA kernels (through the C ABI) against the CPU oracle.

Tolerance for the fp16-storage path (north_star: "within 1e-3 relative fp16 tolerance"): inputs and
weights are rounded to fp16 ONCE, the oracle computes in fp32 on those same rounded values, our kernels
accumulate in fp32 and round the result to fp16 once -> elementwise |err| <= 1e-3 * |ref| + 1e-3 * rms(ref).
"""
import numpy as np
import pytest
import torch

from oracle import fasterseg_oracle as orc
from tests import helpers as H

pytestmark = pytest.mark.gpu

REL = 1e-3


def _F():
    from fasterseg_b200 import functional as F_
    return F_


def _close(got, ref, rel=REL):
    got = got.double()
    ref = ref.double()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    err = (got - ref).abs()
    bound = rel * ref.abs() + rel * rms
    bad = (err > bound)
    assert not bad.any(), "max err %.3e (rms %.3e), %d/%d outside tolerance" % (err.max().item(), rms, int(bad.sum()), bad.numel())


def _rand(shape, seed, scale=1.0):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal(shape).astype(np.float32) * scale)


def _nhwc(x_nchw_f32):
    """CPU NCHW fp32 -> CUDA NHWC fp16 view (plain torch plumbing for test inputs)."""
    return x_nchw_f32.cuda().half().contiguous(memory_format=torch.channels_last)


CONV_CASES = [
    # N, Cin, Cout, k, stride, H, W
    (1, 32, 32, 3, 1, 16, 32),
    (2, 64, 64, 3, 1, 24, 40),
    (1, 64, 128, 3, 2, 32, 48),
    (1, 96, 64, 3, 1, 16, 16),
    (1, 128, 64, 1, 1, 16, 32),
    (1, 256, 128, 1, 1, 8, 16),
    (1, 128, 19, 1, 1, 16, 32),
    (2, 48, 80, 3, 1, 9, 13),
    (2, 384, 384, 3, 1, 8, 16),
    (1, 32, 128, 3, 1, 20, 36),
    (2, 32, 64, 3, 2, 9, 13),
    (1, 64, 64, 3, 2, 18, 30),
    (1, 160, 320, 3, 1, 5, 7),
    (1, 192, 128, 3, 1, 32, 64),
    (3, 80, 48, 1, 1, 6, 10),
    (1, 16, 16, 3, 1, 8, 8),
    # wide maps: many spatial tiles, ragged last tiles
    (1, 64, 64, 3, 1, 20, 256),
    (2, 32, 32, 3, 1, 9, 130),
    (1, 128, 128, 3, 1, 16, 128),
    (1, 96, 64, 3, 1, 12, 256),
    (1, 64, 192, 3, 1, 8, 200),
    (1, 256, 256, 3, 1, 6, 128),
    (1, 80, 48, 3, 1, 5, 97),
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("direct", [False, True])
def test_conv_bn_relu_matches_oracle(case, direct):
    F_ = _F()
    N, Cin, Cout, k, stride, Hh, Ww = case
    seed = hash(case) % 100000
    x = _rand((N, Cin, Hh, Ww), seed).half().float()
    w = (_rand((Cout, Cin, k, k), seed + 1) * (2.0 / (Cin * k * k)) ** 0.5).half().float()
    scale = torch.from_numpy(np.random.RandomState(seed + 2).uniform(0.5, 1.5, Cout).astype(np.float32))
    shift = _rand((Cout,), seed + 3, 0.2)
    pad = 1 if k == 3 else 0
    ref = torch.relu(orc.conv2d(x, w, None, stride, pad) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, k)
    y = F_.conv_fwd(_nhwc(x), wp, Cout, k, stride, pad, scale.cuda(), shift.cuda(), relu=True, force_direct=direct)
    torch.cuda.synchronize()
    assert tuple(y.shape) == tuple(ref.shape)
    _close(y.float().cpu(), ref)


# conv_tc written into a channel slice of a wider buffer (zero-copy concat: the TMA store must respect offset and stride).
# Cases: ragged tiles, batch > 1, 1x1 and stride 2, Wo < 16 (8 x 16 tiles), every N-tile width (Cout 16 .. 256, split into 128-wide
# tiles), 1 .. 4 channel chunks, single-row images, maps with far more tiles than SMs.
SLICE_CASES = [
    # N, Cin, Cout, k, stride, H, W
    (1, 128, 128, 3, 1, 32, 64),
    (1, 192, 128, 3, 1, 24, 40),
    (2, 64, 192, 3, 1, 9, 21),
    (1, 128, 128, 1, 1, 16, 48),
    (1, 64, 128, 3, 2, 34, 50),
    (1, 256, 256, 3, 1, 8, 12),
    (1, 128, 128, 3, 1, 16, 256),
    (1, 64, 64, 3, 1, 40, 256),
    (1, 64, 64, 3, 1, 600, 128),
    (1, 64, 64, 3, 1, 1500, 128),
    (1, 128, 128, 3, 1, 700, 128),
    (2, 64, 128, 3, 1, 9, 200),
    (1, 64, 64, 3, 1, 7, 130),
    (3, 64, 64, 3, 1, 5, 128),
    (1, 192, 128, 3, 1, 12, 128),
    (1, 128, 256, 3, 1, 6, 128),
    (1, 64, 192, 3, 1, 10, 256),
    (1, 64, 64, 3, 1, 24, 256),
    (1, 64, 32, 3, 1, 33, 100),
    (2, 64, 64, 3, 1, 7, 130),
    (1, 128, 32, 3, 1, 9, 64),
    (1, 128, 48, 3, 1, 5, 37),
    (1, 256, 16, 3, 1, 3, 500),
    (1, 192, 32, 3, 1, 6, 90),
    (1, 64, 64, 3, 1, 1, 300),
    (3, 64, 64, 3, 1, 160, 128),
]


@pytest.mark.parametrize("case", SLICE_CASES)
def test_conv_tc_into_channel_slice(case):
    F_ = _F()
    from fasterseg_b200 import _lib
    import ctypes as C
    N, Cin, Cout, k, stride, Hh, Ww = case
    seed = hash(case) % 100000
    x = _rand((N, Cin, Hh, Ww), seed).half().float()
    w = (_rand((Cout, Cin, k, k), seed + 1) * (2.0 / (Cin * k * k)) ** 0.5).half().float()
    scale = torch.from_numpy(np.random.RandomState(seed + 2).uniform(0.5, 1.5, Cout).astype(np.float32))
    shift = _rand((Cout,), seed + 3, 0.2)
    pad = 1 if k == 3 else 0
    ref = torch.relu(orc.conv2d(x, w, None, stride, pad) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, k)
    Ho, Wo = ref.shape[2], ref.shape[3]
    cat = F_.empty_nhwc(N, Cout + 64, Ho, Wo, "cuda")
    cat.fill_(7.0)
    out = cat[:, 32:32 + Cout]
    d = _lib.ConvDesc(N, Hh, Ww, Cin, Cout, k, stride, pad, 1, 0, 0, Ho, Wo, Cin, Cout + 64, _lib.FSB_CONV_RELU | _lib.FSB_CONV_AFFINE)
    assert _lib.lib().fsb_conv_kernel_id(C.byref(d), C.c_void_p(out.data_ptr()), 0) == 1, "case does not reach the tensor-core kernel"
    y = F_.conv_fwd(_nhwc(x), wp, Cout, k, stride, pad, scale.cuda(), shift.cuda(), relu=True, out=out)
    torch.cuda.synchronize()
    _close(y.float().cpu(), ref)
    assert float((cat[:, :32] - 7.0).abs().max()) == 0.0 and float((cat[:, 32 + Cout:] - 7.0).abs().max()) == 0.0
    # the same kernel into a dense tensor: the destination layout must not change a single bit
    y0 = F_.conv_fwd(_nhwc(x), wp, Cout, k, stride, pad, scale.cuda(), shift.cuda(), relu=True)
    torch.cuda.synchronize()
    assert float((y0.float() - y.float()).abs().max()) == 0.0


def test_statistics_are_bit_reproducible():
    """conv with fused statistics, bn_stats, bn_bwd sums and wsum scalar gradients: no floating-point atomics -> the same call
    gives the same bits every time (round 1 differed run to run)."""
    F_ = _F()
    x = _nhwc(_rand((3, 64, 40, 72), 31))
    w = (_rand((96, 64, 3, 3), 32) * 0.05)
    wp = F_.pack_conv_weight(w.cuda(), 64, 96, 3)
    outs = []
    for _ in range(3):
        st = F_.conv_stats_buffer(x, 96, 3, 1, 1)
        raw = F_.conv_fwd(x, wp, 96, 3, 1, 1, stats=st, out_f32=True)
        scale, shift, mean, invstd = F_.bn_finalize(st, 3 * 40 * 72, torch.ones(96, device="cuda"), torch.zeros(96, device="cuda"),
                                                    1e-5, 0.1, None, None, want_save=True)
        y = F_.affine_act(raw, scale, shift, relu=True)
        dy = _nhwc(_rand((3, 96, 40, 72), 33))
        sums = F_.bn_bwd_sums(dy, y, raw, mean, invstd, True).clone()
        xs = [y, _nhwc(_rand((3, 96, 40, 72), 34))]
        _, dw = F_.wsum_bwd(dy, xs, torch.tensor([0.3, 0.7], device="cuda"), [False, False], True, 1024.0)
        torch.cuda.synchronize()
        outs.append([t.clone() for t in (F_.rowsum(st)[0], mean, invstd, F_.bn_stats(y), sums, dw)])
    for other in outs[1:]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)


def test_conv_no_epilogue_and_stats():
    F_ = _F()
    N, Cin, Cout, Hh, Ww = 2, 64, 96, 12, 20
    x = _rand((N, Cin, Hh, Ww), 5).half().float()
    w = (_rand((Cout, Cin, 3, 3), 6) * 0.06).half().float()
    ref = orc.conv2d(x, w, None, 1, 1)
    wp = F_.pack_conv_weight(w.cuda(), Cin, Cout, 3)
    for direct in (False, True):
        xg = _nhwc(x)
        stats = F_.conv_stats_buffer(xg, Cout, 3, 1, 1, force_direct=direct)
        stats.fill_(float("nan"))    # every entry must be written by the launch (no zeroing contract)
        y = F_.conv_fwd(xg, wp, Cout, 3, 1, 1, stats=stats, force_direct=direct, out_f32=True)
        torch.cuda.synchronize()
        _close(y.float().cpu(), ref)
        s = F_.rowsum(stats)[0].cpu().double()
        np.testing.assert_allclose(s[:Cout].numpy(), ref.double().sum(dim=(0, 2, 3)).numpy(), rtol=2e-4, atol=2e-2)
        np.testing.assert_allclose(s[Cout:].numpy(), ref.double().pow(2).sum(dim=(0, 2, 3)).numpy(), rtol=2e-4, atol=2e-2)


def test_conv_sliced_weights_and_concat_views():
    """USConv2d slicing (slimmable_ops.py:42) + torch.cat(dim=1) as channel-offset stores/loads."""
    F_ = _F()
    Cmax_o, Cmax_i, co, ci = 96, 64, 48, 32
    wmax = (_rand((Cmax_o, Cmax_i, 3, 3), 11) * 0.08).half().float()
    x_full = _rand((2, 64, 10, 14), 12).half().float()  # conv reads channels [16:48) of a 64-channel buffer
    xs = x_full[:, 16:16 + ci]
    ref = torch.relu(orc.conv2d(xs, wmax[:co, :ci], None, 1, 1))
    wp = F_.pack_conv_weight(wmax.cuda(), ci, co, 3)
    xg = _nhwc(x_full)[:, 16:16 + ci]
    cat = F_.empty_nhwc(2, 80, 10, 14, "cuda")
    cat.zero_()
    F_.conv_fwd(xg, wp, co, 3, 1, 1, relu=True, out=cat[:, 32:32 + co])
    torch.cuda.synchronize()
    _close(cat[:, 32:32 + co].float().cpu(), ref)
    assert float(cat[:, :32].abs().max()) == 0.0


def test_factorized_reduce_offset_conv():
    """1x1 stride-2 conv on x[:, :, 1:, 1:] (operations.py:523) through desc.off_h/off_w."""
    F_ = _F()
    x = _rand((2, 64, 12, 16), 21).half().float()
    w = (_rand((48, 64, 1, 1), 22) * 0.15).half().float()
    ref0 = orc.conv2d(x, w, None, 2, 0)
    ref1 = orc.conv2d(x[:, :, 1:, 1:], w, None, 2, 0)
    wp = F_.pack_conv_weight(w.cuda(), 64, 48, 1)
    for direct in (False, True):
        y0 = F_.conv_fwd(_nhwc(x), wp, 48, 1, 2, 0, force_direct=direct)
        y1 = F_.conv_fwd(_nhwc(x), wp, 48, 1, 2, 0, off=(1, 1), force_direct=direct)
        torch.cuda.synchronize()
        _close(y0.float().cpu(), ref0)
        _close(y1.float().cpu(), ref1)


@pytest.mark.parametrize("co", [32, 48])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_stem_conv_nchw(co, dtype):
    F_ = _F()
    x = _rand((2, 3, 33, 50), 31)
    if dtype == torch.float16:
        x = x.half().float()
    w = _rand((co, 3, 3, 3), 32) * 0.27
    scale = torch.from_numpy(np.random.RandomState(33).uniform(0.5, 1.5, co).astype(np.float32))
    shift = _rand((co,), 34, 0.2)
    # declared semantics: image and weights are rounded to fp16 once, products accumulate in fp32 (tensor cores)
    ref = torch.relu(orc.conv2d(x.half().float(), w.half().float(), None, 2, 1) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    y = F_.stem_conv_nchw(x.cuda().to(dtype), w.cuda(), scale.cuda(), shift.cuda())
    torch.cuda.synchronize()
    _close(y.float().cpu(), ref)
    ref32 = torch.relu(orc.conv2d(x, w, None, 2, 1) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
    assert H.rel_err(y.float().cpu().numpy(), ref32.numpy()) < 1e-3  # vs un-rounded fp32 operands: norm-wise


def test_convnorm_gate_config0():
    """BASELINE.json configs[0]: ConvNorm(3->32/48, k3, s2) on 1x3x256x512 vs the REFERENCE's golden sample."""
    F_ = _F()
    z = H.load_npz("convnorm_gate.npz")
    x = orc.random_input((1, 3, 256, 512), seed=12345)
    for co in (32, 48):
        shapes = {"conv.0.weight": (co, 3, 3, 3), "conv.1.weight": (co,), "conv.1.bias": (co,),
                  "conv.1.running_mean": (co,), "conv.1.running_var": (co,)}
        sd = orc.random_state_dict(shapes, seed=12345 + co)
        sc, sh = F_.bn_fold(sd["conv.1.weight"].cuda(), sd["conv.1.bias"].cuda(), sd["conv.1.running_mean"].cuda(),
                            sd["conv.1.running_var"].cuda(), orc.BN_EPS)
        y = F_.stem_conv_nchw(x.cuda(), sd["conv.0.weight"].cuda(), sc, sh).float().cpu()
        ref_s = torch.from_numpy(z["co%d.eval/sample" % co])
        # vs the REFERENCE (fp32 operands): norm-wise 1e-3 (north_star) + elementwise 2e-3 * (|ref| + rms)
        assert H.rel_err(y[:, :, ::8, ::8].numpy(), ref_s.numpy()) < 1e-3
        _close(y[:, :, ::8, ::8], ref_s, rel=4e-3)  # tails of 27-term sums of fp16-rounded operands
        full = orc.conv_norm(x, orc.Params(sd), 3, 2, 1, False)
        assert H.rel_err(y.numpy(), full.numpy()) < 1e-3
        _close(y, full, rel=4e-3)


def test_bilinear_golden_and_random():
    F_ = _F()
    z = H.load_npz("bilinear.npz")
    n = len([k for k in z.files if k.endswith("/x")])
    for i in range(n):
        x = torch.from_numpy(z["%d/x" % i])
        # pad channels 5 -> 8 for the 16-byte vector path
        xp = torch.zeros(x.shape[0], 8, x.shape[2], x.shape[3])
        xp[:, :5] = x
        xh = xp.half().float()
        ref = orc.bilinear_ac(xh, z["%d/y" % i].shape[2:])
        y = F_.bilinear(_nhwc(xh), ref.shape[2:])
        torch.cuda.synchronize()
        _close(y.float().cpu(), ref)
        _close(y.float().cpu()[:, :5], torch.from_numpy(z["%d/y" % i]), rel=2e-3)  # vs the reference itself (fp32 input)
    x = _rand((2, 64, 17, 23), 41).half().float()
    for size in ((8, 11), (34, 46), (17, 23)):
        ref = torch.relu(orc.bilinear_ac(x, size))
        y = F_.bilinear(_nhwc(x), size, relu=True)
        _close(y.float().cpu(), ref)


def test_upsample_logits_and_argmax():
    F_ = _F()
    x = _rand((2, 19, 9, 12), 51).half().float()
    xp = torch.zeros(2, 24, 9, 12)
    xp[:, :19] = x
    xg = _nhwc(xp)[:, :19]
    ref = orc.bilinear_ac(x, (72, 96))
    for dt in (torch.float32, torch.float16):
        y = F_.upsample_logits(xg, (72, 96), dtype=dt)
        torch.cuda.synchronize()
        assert y.is_contiguous() and tuple(y.shape) == (2, 19, 72, 96)
        _close(y.float().cpu(), ref, rel=1e-3 if dt == torch.float16 else 1e-5)
    lab = F_.upsample_argmax(xg, (72, 96)).cpu()
    ref_lab = ref.argmax(1).to(torch.uint8)
    mism = lab != ref_lab
    if mism.any():  # only fp32 rounding-order near-ties may differ
        top2 = ref.topk(2, dim=1).values
        margin = (top2[:, 0] - top2[:, 1])[mism]
        assert float(margin.max()) < 1e-5, "argmax mismatch with margin %g" % float(margin.max())
    assert float(mism.float().mean()) < 1e-3
    # bit-exact against argmax of OUR OWN fp32 upsampled logits
    own = F_.upsample_logits(xg, (72, 96), dtype=torch.float32).argmax(1).to(torch.uint8).cpu()
    assert torch.equal(lab, own)
    # odd output width / non-multiple-of-8 tails
    ref2 = orc.bilinear_ac(x, (13, 21))
    y2 = F_.upsample_logits(xg, (13, 21), dtype=torch.float32)
    _close(y2.cpu(), ref2, rel=1e-5)
    lab2 = F_.upsample_argmax(xg, (13, 21)).cpu()
    assert torch.equal(lab2, y2.argmax(1).to(torch.uint8).cpu())


def test_layout_roundtrip_and_copy():
    F_ = _F()
    x = _rand((2, 19, 7, 11), 61)
    y = F_.to_nhwc_half(x.cuda())
    assert tuple(y.shape) == (2, 19, 7, 11)
    torch.testing.assert_close(y.float().cpu(), x.half().float(), rtol=0, atol=0)
    back = F_.to_nchw(y, torch.float32)
    torch.testing.assert_close(back.cpu(), x.half().float(), rtol=0, atol=0)
    a = _nhwc(_rand((2, 32, 5, 6), 62))
    cat = F_.empty_nhwc(2, 64, 5, 6, "cuda")
    cat.zero_()
    F_.copy_channels(a, cat[:, 16:48])
    assert torch.equal(cat[:, 16:48].contiguous(), a.contiguous())


def test_bn_train_kernels():
    F_ = _F()
    Cc = 48
    x = (_rand((3, Cc, 9, 14), 71) * 1.7 + 0.3).half().float()
    gamma = torch.from_numpy(np.random.RandomState(72).uniform(0.5, 1.5, Cc).astype(np.float32))
    beta = _rand((Cc,), 73, 0.2)
    rm, rv = _rand((Cc,), 74, 0.1), torch.from_numpy(np.random.RandomState(75).uniform(0.5, 1.5, Cc).astype(np.float32))
    rm_ref, rv_ref = rm.clone(), rv.clone()
    ref = torch.relu(orc.batchnorm(x, gamma, beta, rm_ref, rv_ref, True))
    xg = _nhwc(x)
    stats = F_.bn_stats(xg)
    rm_g, rv_g = rm.cuda(), rv.cuda()
    scale, shift, mean, invstd = F_.bn_finalize(stats, 3 * 9 * 14, gamma.cuda(), beta.cuda(), orc.BN_EPS, orc.BN_MOMENTUM,
                                                rm_g, rv_g, want_save=True)
    y = F_.affine_act(xg, scale, shift, relu=True)
    torch.cuda.synchronize()
    _close(y.float().cpu(), ref)
    np.testing.assert_allclose(rm_g.cpu().numpy(), rm_ref.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(rv_g.cpu().numpy(), rv_ref.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(mean.cpu().numpy(), x.mean(dim=(0, 2, 3)).numpy(), rtol=1e-5, atol=1e-6)


def test_errors_are_loud():
    F_ = _F()
    from fasterseg_b200._lib import FsbError
    x = _nhwc(_rand((1, 32, 8, 8), 81))
    wp = F_.pack_conv_weight(_rand((32, 32, 3, 3), 82).cuda(), 32, 32, 3)
    bad_out = F_.empty_nhwc(1, 32, 7, 8, "cuda")
    with pytest.raises((FsbError, AssertionError)):
        F_.conv_fwd(x, wp, 32, 3, 1, 1, out=bad_out)


WGRAD_CASES = [
    # N, Cin, Cout, k, stride, H, W
    (2, 64, 64, 3, 1, 16, 24),
    (1, 32, 128, 3, 1, 20, 36),
    (2, 96, 48, 3, 1, 9, 13),
    (1, 128, 64, 1, 1, 16, 32),
    (2, 64, 128, 3, 2, 18, 30),
    (1, 192, 320, 3, 1, 8, 16),
    (3, 80, 160, 1, 1, 6, 10),
    (2, 32, 64, 3, 2, 9, 13),
    (1, 384, 384, 3, 1, 8, 16),
    # FactorizedReduce's second conv: 1x1 stride 2 on x[:, :, 1:, 1:] (operations.py:523) through desc.off_h / off_w
    (2, 64, 48, 1, 2, 12, 16, (1, 1)),
]


@pytest.mark.parametrize("case", WGRAD_CASES)
def test_conv_wgrad_and_dgrad_match_oracle(case):
    """K7: tensor-core weight gradient (MN-major operands) and data gradient vs CPU autograd of F.conv2d; the CUDA-core
    kernels are checked on the same inputs."""
    F_ = _F()
    N, Cin, Cout, k, stride, Hh, Ww = case[:7]
    off = case[7] if len(case) > 7 else (0, 0)
    seed = hash(case) % 100000
    pad = 1 if k == 3 else 0
    x = _rand((N, Cin, Hh, Ww), seed).half().float().requires_grad_(True)
    w = (_rand((Cout, Cin, k, k), seed + 1) * (2.0 / (Cin * k * k)) ** 0.5).half().float().requires_grad_(True)
    y = orc.conv2d(x[:, :, off[0]:, off[1]:], w, None, stride, pad)
    gy = _rand(tuple(y.shape), seed + 2).half().float()
    y.backward(gy)
    xg, gyg, wg = _nhwc(x.detach()), _nhwc(gy), w.detach().cuda()
    for direct in (False, True):
        dw = F_.conv_wgrad(xg, gyg, wg, Cin, Cout, k, stride, pad, 1.0, off=off, force_direct=direct)
        torch.cuda.synchronize()
        err = H.rel_err(dw.cpu().numpy(), w.grad.numpy())
        assert err < 1e-3, "wgrad (direct=%s) rel err %.3e" % (direct, err)
        wt = F_.pack_conv_weight_dgrad(wg, Cin, Cout, k)
        dx = F_.conv_dgrad(gyg, wg, (N, Cin, Hh, Ww), Cin, Cout, k, stride, pad, off=off, wpacked_t=wt, force_direct=direct)
        torch.cuda.synchronize()
        errx = H.rel_err(dx.float().cpu().numpy(), x.grad.numpy())
        assert errx < 1.5e-3, "dgrad (direct=%s) rel err %.3e" % (direct, errx)
    # accumulation into an existing gradient (a cell invoked twice, model_search.py:326-329)
    acc = dw.clone()
    F_.conv_wgrad(xg, gyg, wg, Cin, Cout, k, stride, pad, 1.0, off=off, accumulate_into=acc)
    torch.cuda.synchronize()
    assert H.rel_err(acc.cpu().numpy(), 2 * w.grad.numpy()) < 1e-3
