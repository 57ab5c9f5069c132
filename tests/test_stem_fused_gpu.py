"""K1f (csrc/stem_fused.cu): the RGB stem and stem.1's first conv as one kernel must give exactly the bits of the two-kernel path
(stem_conv_* then conv_fwd) for every input kind, frame size and output placement, and the network must take it only where it
applies."""
import numpy as np
import pytest
import torch

from fasterseg_b200 import functional as F_
from fasterseg_b200 import roofline, zoo

pytestmark = pytest.mark.gpu

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _params(C0, C1, seed=0):
    g = torch.Generator().manual_seed(seed)
    dev = torch.device("cuda")
    w0 = (torch.randn(C0, 3, 3, 3, generator=g) * (2.0 / 27) ** 0.5).to(dev)
    w1 = (torch.randn(C1, C0, 3, 3, generator=g) * (2.0 / (9 * C0)) ** 0.5).to(dev)
    s0, b0 = (torch.rand(C0, generator=g) + 0.5).to(dev), (torch.randn(C0, generator=g) * 0.1).to(dev)
    s1, b1 = (torch.rand(C1, generator=g) + 0.5).to(dev), (torch.randn(C1, generator=g) * 0.1).to(dev)
    return w0, s0, b0, F_.pack_conv_weight(w1, C0, C1, 3), C1, s1, b1


def _frame(kind, N, H, W, seed=1):
    g = torch.Generator().manual_seed(seed)
    if kind == "u8":
        img = torch.randint(0, 256, (N, H, W, 3), generator=g, dtype=torch.uint8).cuda()
        return img.permute(0, 3, 1, 2), F_.normalization_lut(MEAN, STD, torch.device("cuda"))
    x = torch.randn(N, 3, H, W, generator=g).cuda()
    return (x if kind == "f32" else x.half()), None


def _two_kernels(x, lut, w0, s0, b0, w1p, C1, s1, b1, out=None):
    y0 = F_.stem_conv_u8hwc(x, lut, w0, s0, b0) if x.dtype == torch.uint8 else F_.stem_conv_nchw(x, w0, s0, b0)
    return F_.conv_fwd(y0, w1p, C1, 3, 2, 1, s1, b1, relu=True, out=out)


@pytest.mark.parametrize("kind", ["f32", "f16", "u8"])
@pytest.mark.parametrize("N,H,W", [(2, 1024, 2048), (1, 520, 1000), (1, 517, 1029), (1, 64, 96)])
def test_stem_fused_is_bit_identical_to_the_two_kernels(kind, N, H, W):
    p = _params(32, 64)
    x, lut = _frame(kind, N, H, W)
    ref = _two_kernels(x, lut, *p)
    y = F_.stem_fused(x, lut, *p)
    torch.cuda.synchronize()
    assert y is not None and tuple(y.shape) == tuple(ref.shape)
    assert torch.equal(y, ref), "max-abs difference %.3e" % (y.float() - ref.float()).abs().max().item()
    assert ref.float().abs().max().item() > 0


@pytest.mark.parametrize("kind", ["f32", "u8"])
def test_stem_fused_writes_a_channel_slice_and_nothing_else(kind):
    p = _params(32, 64, seed=3)
    x, lut = _frame(kind, 1, 260, 500, seed=4)
    H1, W1 = 65, 125
    wide = torch.full((1, H1, W1, 96), 7.0, device="cuda", dtype=torch.float16)
    ref_wide = wide.clone()
    y = F_.stem_fused(x, lut, *p, out=wide.permute(0, 3, 1, 2)[:, 16:80])
    _two_kernels(x, lut, *p, out=ref_wide.permute(0, 3, 1, 2)[:, 16:80])
    torch.cuda.synchronize()
    assert y is not None
    assert torch.equal(wide, ref_wide)
    assert bool((wide[..., :16] == 7).all()) and bool((wide[..., 80:] == 7).all())


@pytest.mark.parametrize("C0,C1", [(48, 96), (32, 48), (12, 64)])
def test_other_stem_widths_are_unsupported(C0, C1):
    x, _ = _frame("f32", 1, 64, 96)
    assert F_.stem_fused(x, None, *_params(C0, C1)) is None


def _student():
    from bench import synth_weights_
    model = zoo.build_network(1)
    synth_weights_(model)
    model = model.cuda().eval()
    model.logits_dtype = torch.float16
    return model


def test_network_takes_the_fused_stem_and_matches_the_two_kernel_path(monkeypatch):
    model = _student()
    x = torch.randn(1, 3, 512, 1024, generator=torch.Generator().manual_seed(5)).cuda()
    calls = []
    fused = F_.stem_fused

    def spy(*a, **kw):
        y = fused(*a, **kw)
        calls.append(y is not None)
        return y
    with torch.no_grad():
        monkeypatch.setattr(F_, "stem_fused", spy)
        y = model(x)
        monkeypatch.setattr(F_, "stem_fused", lambda *a, **kw: None)   # the library declines: the network runs self.stem
        ref = model(x)
    torch.cuda.synchronize()
    assert calls == [True]
    assert torch.equal(y, ref)
    # training mode, or autograd, keeps the two-kernel stem
    calls.clear()
    monkeypatch.setattr(F_, "stem_fused", spy)
    model(x[:, :, :64, :128].contiguous())
    assert calls == []


def test_student_frame_traces_one_stem_launch_on_the_gpu():
    model = _student()
    x = torch.zeros(1, 3, 1024, 2048, device="cuda")
    with torch.no_grad():
        recs = roofline.trace_launches(lambda: model(x))
    kinds = [r["kernel"] for r in recs]
    assert len(recs) == 73 and kinds[0] == "stem_fused" and "stem_conv" not in kinds
    s = roofline.sigma_roofline(recs, tensor_tflops=989.0, hbm_gbs=3350.0)
    assert abs(s["gflop"] - 55.54) < 0.01
    assert np.isfinite(s["sum_us"])
