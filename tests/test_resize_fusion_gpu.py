"""The fused resizes on the GPU: fsb_conv_fwd_half must give exactly the bits of fsb_conv_fwd followed by fsb_bilinear_fwd (/2),
fsb_bilinear_fwd_half those of the x2 (+ReLU) upsample followed by the /2, and the student frame with its resize plan those of the
same network without it."""
import pytest
import torch

from fasterseg_b200 import _lib, roofline
from fasterseg_b200 import functional as F_

pytestmark = pytest.mark.gpu


def _act(N, C, H, W, seed, cpad=0):
    g = torch.Generator().manual_seed(seed)
    buf = F_.empty_nhwc(N, C + cpad, H, W, "cuda")
    buf.copy_(torch.randn(N, C + cpad, H, W, generator=g).half().cuda())
    return buf[:, cpad:]


def _conv_params(Cin, Cout, seed):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) * (2.0 / (9 * Cin)) ** 0.5).cuda()
    scale = (torch.rand(Cout, generator=g) + 0.5).cuda()
    shift = (torch.randn(Cout, generator=g) * 0.1).cuda()
    return F_.pack_conv_weight(w, Cin, Cout, 3), scale, shift


@pytest.fixture
def no_separate_launch(monkeypatch):
    """fails if a wrapper falls back to a second bilinear launch: the half output must come from the one kernel"""
    def refuse(*a, **kw):
        raise AssertionError("the /2 output took the separate bilinear launch")
    monkeypatch.setattr(F_, "bilinear", refuse)


# (N, Cin, Cout, Ho, Wo): the four /2-producing convs of the student frame (arch_1, 1024x2048), N tiles of 32 / 64 / 128, 8x16 tiles
# (Wo < 16), partial border tiles, two images
CONV_SHAPES = [(1, 32, 32, 128, 256), (1, 32, 128, 64, 128), (1, 64, 64, 64, 128), (1, 128, 128, 32, 64),
               (1, 64, 32, 20, 36), (2, 64, 64, 22, 12), (1, 32, 128, 14, 8), (1, 96, 128, 128, 256), (2, 16, 48, 18, 26)]


@pytest.mark.parametrize("mode", [0, 1])            # FSB_CONV_TC2: per-tap, window
@pytest.mark.parametrize("offset", [False, True])   # outputs as channel slices of wider buffers
@pytest.mark.parametrize("shape", CONV_SHAPES)
def test_conv_fwd_half_equals_conv_then_bilinear(shape, offset, mode, no_separate_launch):
    N, Cin, Cout, Ho, Wo = shape
    x = _act(N, Cin, Ho, Wo, seed=Cin + Ho, cpad=8 if offset else 0)
    wp, scale, shift = _conv_params(Cin, Cout, seed=Cout)
    _lib.set_option("FSB_CONV_TC2", mode)
    try:
        if offset:
            y = F_.empty_nhwc(N, Cout + 24, Ho, Wo, "cuda")[:, 16:16 + Cout]
            yh = F_.empty_nhwc(N, Cout + 16, Ho // 2, Wo // 2, "cuda")[:, 8:8 + Cout]
        else:
            y, yh = F_.empty_nhwc(N, Cout, Ho, Wo, "cuda"), F_.empty_nhwc(N, Cout, Ho // 2, Wo // 2, "cuda")
        F_.conv_fwd(x, wp, Cout, 3, 1, 1, scale, shift, relu=True, out=y, out_half=yh)
        ref = F_.conv_fwd(x, wp, Cout, 3, 1, 1, scale, shift, relu=True)
    finally:
        _lib.set_option("FSB_CONV_TC2", -1)
    ref_h = torch.empty_like(yh)
    check = _lib.lib().fsb_bilinear_fwd(N, Cout, Ho, Wo, Ho // 2, Wo // 2, F_._ptr(ref), ref.stride(3), F_._ptr(ref_h), ref_h.stride(3),
                                        0, F_._stream())
    _lib.check(check, "fsb_bilinear_fwd")
    torch.cuda.synchronize()
    assert torch.equal(y, ref) and torch.equal(yh, ref_h)


def test_conv_fwd_half_falls_back_where_the_kernel_does_not_apply():
    """odd output extent, and the direct kernel (Cin < 16): the wrapper makes the /2 with a second launch, same bits"""
    for Cin, H, W in ((32, 21, 34), (8, 20, 34)):
        x = _act(1, Cin, H, W, seed=7)
        wp, scale, shift = _conv_params(Cin, 32, seed=8)
        yh = F_.empty_nhwc(1, 32, H // 2, W // 2, "cuda")
        y = F_.conv_fwd(x, wp, 32, 3, 1, 1, scale, shift, relu=True, out_half=yh)
        assert torch.equal(yh, F_.bilinear(y, (H // 2, W // 2)))


# (N, C, Hi, Wi): the x2 upsamples of the frame whose output a zoomed cell reads, odd sizes, two images
UP_SHAPES = [(1, 32, 64, 128), (1, 64, 32, 64), (1, 192, 32, 64), (1, 128, 16, 32), (1, 128, 32, 64), (2, 24, 7, 9), (1, 8, 1, 5)]


@pytest.mark.parametrize("offset", [False, True])
@pytest.mark.parametrize("shape", UP_SHAPES)
def test_bilinear_fwd_half_equals_up2_relu_then_down2(shape, offset, no_separate_launch):
    N, C, Hi, Wi = shape
    x = _act(N, C, Hi, Wi, seed=C + Hi, cpad=8 if offset else 0)
    if offset:
        y = F_.empty_nhwc(N, C + 40, 2 * Hi, 2 * Wi, "cuda")[:, 32:32 + C]
        yh = F_.empty_nhwc(N, C + 8, Hi, Wi, "cuda")[:, 8:]
    else:
        y, yh = F_.empty_nhwc(N, C, 2 * Hi, 2 * Wi, "cuda"), F_.empty_nhwc(N, C, Hi, Wi, "cuda")
    rc = _lib.lib().fsb_bilinear_fwd_half(N, C, Hi, Wi, F_._ptr(x), x.stride(3), F_._ptr(y), y.stride(3), F_._ptr(yh), yh.stride(3),
                                          _lib.FSB_CONV_RELU, F_._stream())
    _lib.check(rc, "fsb_bilinear_fwd_half")
    ref, ref_h = F_.empty_nhwc(N, C, 2 * Hi, 2 * Wi, "cuda"), F_.empty_nhwc(N, C, Hi, Wi, "cuda")
    for src, dst, (hi, wi), (ho, wo), flags in ((x, ref, (Hi, Wi), (2 * Hi, 2 * Wi), _lib.FSB_CONV_RELU),
                                                (ref, ref_h, (2 * Hi, 2 * Wi), (Hi, Wi), 0)):
        _lib.check(_lib.lib().fsb_bilinear_fwd(N, C, hi, wi, ho, wo, F_._ptr(src), src.stride(3), F_._ptr(dst), dst.stride(3), flags,
                                               F_._stream()), "fsb_bilinear_fwd")
    torch.cuda.synchronize()
    assert torch.equal(y, ref) and torch.equal(yh, ref_h)


def _student():
    from bench import synth_weights_
    from fasterseg_b200 import zoo
    model = zoo.build_network(1)
    synth_weights_(model)
    model = model.cuda().eval()
    model.logits_dtype = torch.float16
    return model


def test_student_frame_with_fused_resizes_is_bit_identical_and_15_launches_shorter():
    """the first forward at an input size records the plan and runs the parent's 73 launches; from the second on the frame is 58
    launches, the fused stem still first, the same work and the same bits as without the plan"""
    model = _student()
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, 3, 1024, 2048, generator=g).cuda()
    with torch.no_grad():
        first = roofline.trace_launches(lambda: model(x))
        recs = roofline.trace_launches(lambda: model(x))
        fused = model(x)
        labels = model.predict_labels(x)
        model.fuse_resizes = False
        plain_recs = roofline.trace_launches(lambda: model(x))
        plain = model(x)
        plain_labels = model.predict_labels(x)
    kinds = [r["kernel"] for r in recs]
    assert len(first) == len(plain_recs) == 73 and len(recs) == 58
    assert kinds[0] == "stem_fused" and "stem_conv" not in kinds and "copy_channels" not in kinds
    assert abs(roofline.sigma_roofline(recs, tensor_tflops=989.0, hbm_gbs=3350.0)["gflop"] - 55.54) < 0.01
    assert torch.equal(fused, plain) and torch.equal(labels, plain_labels)
