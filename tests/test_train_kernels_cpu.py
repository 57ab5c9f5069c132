"""The float64 references of the training kernels (tests/train_kernel_refs.py) checked without a GPU: against torch autograd of
the same float64 composite, and against the CPU stand-ins of tests/cpu_backend.py that the whole CPU suite trusts."""
import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from tests import train_kernel_refs as R

F64 = torch.float64


def _randn(shape, seed, mean=0.0):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal(shape)).to(F64) + mean


def _autograd_bn(x, gamma, beta, eps, relu):
    x = x.clone().requires_grad_(True)
    g = gamma.clone().requires_grad_(True)
    b = beta.clone().requires_grad_(True)
    y = TF.batch_norm(x, None, None, g, b, training=True, eps=eps)
    return x, g, b, (y.relu() if relu else y)


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("shape", [(2, 8, 5, 7), (1, 16, 1, 2), (3, 24, 4, 1)])
def test_bn_train_forward_and_backward_match_autograd(shape, relu):
    C = shape[1]
    x = _randn(shape, 1, mean=0.7)
    gamma, beta = _randn((C,), 2) * 0.5 + 1.0, _randn((C,), 3) * 0.2
    eps, mom = 1e-5, 0.1
    rm, rv = _randn((C,), 4) * 0.1, _randn((C,), 5).abs() + 0.5
    xr, g, b, y = _autograd_bn(x, gamma, beta, eps, relu)
    rm_t, rv_t = rm.clone(), rv.clone()
    TF.batch_norm(x, rm_t, rv_t, gamma, beta, training=True, momentum=mom, eps=eps)

    s, q = R.bn_sums(x)
    st = R.bn_finalize(s, q, x.numel() // C, gamma, beta, eps, mom, rm, rv)
    torch.testing.assert_close(R.affine_act(x, st["scale"], st["shift"], relu), y.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(st["running_mean"], rm_t, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(st["running_var"], rv_t, rtol=1e-12, atol=1e-12)

    dy = _randn(shape, 6)
    y.backward(dy)
    ref = R.bn_bwd(dy, y.detach(), x, st["mean"], st["invstd"], gamma, relu)
    torch.testing.assert_close(ref["draw"], xr.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(ref["dgamma"], g.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(ref["dbeta"], b.grad, rtol=1e-10, atol=1e-10)


def test_bn_finalize_edges():
    # count = 2: unbiased factor 2; a variance that rounds below zero is clamped to 0 (invstd = 1 / sqrt(eps))
    st = R.bn_finalize(torch.tensor([2.0, 6.0], dtype=F64), torch.tensor([2.0, 18.0 - 1e-9], dtype=F64), 2, None, None, 1e-5, 0.5,
                       torch.zeros(2, dtype=F64), torch.ones(2, dtype=F64))
    assert st["var"][0] == 0.0 and st["var"][1] == 0.0
    assert torch.allclose(st["invstd"], torch.full((2,), 1e-5, dtype=F64).rsqrt())
    x = torch.tensor([1.0, 3.0], dtype=F64)
    assert torch.allclose(R.bn_finalize(x.sum().reshape(1), (x * x).sum().reshape(1), 2, None, None, 0.0, 1.0,
                                        torch.zeros(1, dtype=F64), torch.zeros(1, dtype=F64))["running_var"],
                          x.var(unbiased=True).reshape(1))


@pytest.mark.parametrize("hmax", [8, 16, 32, 64])
def test_split_perm_is_the_defined_bijection_and_matches_the_stand_in(hmax):
    from tests import cpu_backend
    for h in range(0, hmax + 1):
        p = R.split_perm(h, hmax)
        assert sorted(p.tolist()) == list(range(2 * hmax))
        assert p[:h].tolist() == list(range(h)) and p[h:2 * h].tolist() == list(range(hmax, hmax + h))
        assert torch.equal(cpu_backend._split_perm(h, hmax), p)


@pytest.mark.parametrize("io", [((9, 13), (18, 26)), ((17, 23), (34, 46)), ((18, 26), (9, 13)), ((16, 32), (128, 256)),
                                ((7, 5), (7, 5)), ((5, 6), (1, 11)), ((1, 6), (4, 9)), ((1, 1), (3, 4)), ((64, 128), (512, 1024)),
                                ((9, 12), (13, 21))])
def test_bilinear_matrices_match_interpolate_and_its_autograd(io):
    (Hi, Wi), (Ho, Wo) = io
    x = _randn((2, 3, Hi, Wi), 11).requires_grad_(True)
    y = TF.interpolate(x, size=(Ho, Wo), mode="bilinear", align_corners=True)
    # the taps are computed in fp32: src = fp32(scale * dst) carries an error of ~2 ulps of src < 2 * n_in * 2^-24, which moves
    # each of the two weights of an axis by as much; torch computes them in float64
    tap_err = 4 * (Hi + Wi) * 2.0 ** -24
    torch.testing.assert_close(R.bilinear_fwd(x.detach(), Ho, Wo), y.detach(), rtol=0, atol=tap_err * float(x.detach().abs().max()))
    dy = _randn((2, 3, Ho, Wo), 12)
    mask = _randn((2, 3, Ho, Wo), 13)
    y.backward(dy * (mask > 0))
    dx, mag = R.bilinear_bwd(dy, Hi, Wi, mask)
    torch.testing.assert_close(dx, x.grad, rtol=0, atol=tap_err * float(mag.max()))
    assert bool((mag >= dx.abs() - 1e-12).all())
    dl, _ = R.upsample_logits_bwd(dy, Hi, Wi, 3.0)
    torch.testing.assert_close(dl, 3.0 * R.bilinear_bwd(dy, Hi, Wi)[0], rtol=1e-15, atol=0)


def test_wsum_matches_autograd():
    xs = [_randn((2, 8, 3, 5), 20 + k) for k in range(5)]
    w = _randn((5,), 30).requires_grad_(True)
    xr = [x.clone().requires_grad_(True) for x in xs]
    out = sum(w[k] * xr[k] for k in range(5))
    torch.testing.assert_close(R.wsum_fwd(xs, w.detach()), out.detach(), rtol=1e-14, atol=1e-14)
    dout = _randn(out.shape, 31)
    out.backward(dout)
    dxs, dw, mag = R.wsum_bwd(dout, xs, w.detach(), 4.0)
    for k in range(5):
        torch.testing.assert_close(dxs[k], xr[k].grad, rtol=1e-14, atol=1e-14)
    torch.testing.assert_close(dw * 4.0, w.grad, rtol=1e-12, atol=1e-12)
    assert bool((mag >= dw.abs()).all())


@pytest.mark.parametrize("geom", [(3, 1, 1, (0, 0)), (3, 2, 1, (0, 0)), (1, 1, 0, (0, 0)), (1, 2, 0, (0, 0)), (1, 2, 0, (1, 1))])
def test_conv_unit_matches_autograd(geom):
    k, stride, pad, off = geom
    N, Cin, Cout, H, W = 2, 5, 8, 9, 11
    x = _randn((N, Cin, H, W), 40).requires_grad_(True)
    w = (_randn((Cout, Cin, k, k), 41) * 0.3).requires_grad_(True)
    gamma, beta = _randn((Cout,), 42) * 0.3 + 1.0, _randn((Cout,), 43) * 0.1
    # autograd of the float64 composite: slice, conv, batch_norm(training), relu
    g = gamma.clone().requires_grad_(True)
    b = beta.clone().requires_grad_(True)
    raw = TF.conv2d(x[:, :, off[0]:, off[1]:], w, None, stride, pad)
    y = TF.batch_norm(raw, None, None, g, b, training=True, eps=1e-5).relu()
    dy = _randn(tuple(y.shape), 44)
    y.backward(dy)
    st = R.conv_bn_act_fwd(x.detach(), w.detach(), stride, pad, off, gamma, beta, 1e-5, 0.1, None, None, True)
    torch.testing.assert_close(st["raw"], raw.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(st["y"], y.detach(), rtol=1e-10, atol=1e-10)
    bw = R.bn_bwd(dy, st["y"], st["raw"], st["mean"], st["invstd"], gamma, True)
    torch.testing.assert_close(bw["dgamma"], g.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(bw["dbeta"], b.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(R.conv_dgrad(bw["draw"], w.detach(), (N, Cin, H, W), stride, pad, off), x.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(R.conv_wgrad(x.detach(), bw["draw"], tuple(w.shape), stride, pad, off), w.grad, rtol=1e-10, atol=1e-10)


# ---- the references against the CPU stand-ins (same edge cases) -------------------------------------------------------------
def _nhwc16(x):
    from fasterseg_b200 import functional as F_
    N, Cc, H, W = x.shape
    out = F_.empty_nhwc(N, Cc, H, W, "cpu")
    out.copy_(x.half())
    return out


def test_stand_ins_agree_with_the_references():
    from tests import cpu_backend as cb
    N, C, H, W = 2, 16, 5, 7
    x = _nhwc16(_randn((N, C, H, W), 50, mean=0.5))
    x64 = x.to(F64)
    gamma, beta = (_randn((C,), 51) * 0.3 + 1).float(), (_randn((C,), 52) * 0.1).float()
    rm, rv = torch.zeros(C), torch.ones(C)
    s, q = R.bn_sums(x64)
    st = R.bn_finalize(s, q, N * H * W, gamma, beta, 1e-5, 0.1, rm, rv)
    stats = cb.bn_stats(x)
    torch.testing.assert_close(stats.to(F64), torch.cat([s, q]), rtol=1e-6, atol=1e-5)
    scale, shift, mean, invstd = cb.bn_finalize(stats, N * H * W, gamma, beta, 1e-5, 0.1, rm, rv, want_save=True)
    torch.testing.assert_close(mean.to(F64), st["mean"], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(invstd.to(F64), st["invstd"], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(rm.to(F64), st["running_mean"], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(rv.to(F64), st["running_var"], rtol=1e-5, atol=1e-6)
    y = cb.affine_act(x, scale, shift, relu=True)
    torch.testing.assert_close(y.to(F64), R.affine_act(x64, st["scale"], st["shift"], True), rtol=2e-3, atol=2e-3)
    # exact zeros and -0.0 in y take the ReLU mask's "not > 0" branch in both
    y[0, :, 0, 0] = 0.0
    y[1, :, 2, 3] = -0.0
    dy = _nhwc16(_randn((N, C, H, W), 53))
    sums = cb.bn_bwd_sums(dy, y, x, mean, invstd, True)
    ref = R.bn_bwd(dy, y, x, mean, invstd, gamma, True)
    torch.testing.assert_close(sums.to(F64), torch.cat([ref["sum_dz"], ref["sum_dzxhat"]]), rtol=1e-5, atol=1e-4)
    draw, dg, db = cb.bn_bwd_apply(dy, y, x, mean, invstd, gamma, sums, N * H * W, True, 8.0)
    torch.testing.assert_close(draw.to(F64), ref["draw"], rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(dg.to(F64), ref["dgamma"] / 8.0, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(db.to(F64), ref["dbeta"] / 8.0, rtol=1e-5, atol=1e-5)
    # resize backward, wsum, the fused unit (with the FactorizedReduce offset)
    for (Hi, Wi), (Ho, Wo) in (((9, 13), (18, 26)), ((18, 26), (9, 13)), ((1, 4), (5, 1))):
        g = _nhwc16(_randn((N, 8, Ho, Wo), 54))
        ref_dx, _ = R.bilinear_bwd(g.to(F64), Hi, Wi, g.to(F64))
        torch.testing.assert_close(cb.bilinear_bwd(g, (Hi, Wi), relu_mask_y=g).to(F64), ref_dx, rtol=2e-3, atol=2e-3)
    xs = [_nhwc16(_randn((N, C, H, W), 60 + k)) for k in range(3)]
    wts = torch.tensor([0.3, -1.25, 2.0])
    dxs, dw = cb.wsum_bwd(dy, xs, wts, [True, False, True], True, 16.0)
    rdx, rdw, _ = R.wsum_bwd(dy.to(F64), [t.to(F64) for t in xs], wts, 16.0)
    torch.testing.assert_close(dw.to(F64), rdw, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(dxs[0].to(F64), rdx[0], rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(cb.wsum_fwd(xs, wts).to(F64), R.wsum_fwd([t.to(F64) for t in xs], wts), rtol=2e-3, atol=2e-3)
    w = (_randn((8, C, 1, 1), 70) * 0.2).float()
    wp = cb.pack_conv_weight(w, C, 8, 1)
    for off in ((0, 0), (1, 1)):
        cb.PRECISE["on"] = True
        try:
            yb, raw, vec, d = cb.conv_bn_act_train_fwd(x, wp, 8, 1, 2, 0, off, gamma[:8], beta[:8], 1e-5, 0.1, None, None, None, True)
            st = R.conv_bn_act_fwd(x64, wp.to(F64), 2, 0, off, gamma[:8], beta[:8], 1e-5, 0.1, None, None, True)
            torch.testing.assert_close(raw.to(F64), st["raw"], rtol=1e-6, atol=1e-6)
            torch.testing.assert_close(yb.to(F64), st["y"], rtol=2e-3, atol=2e-3)
            dyu = _nhwc16(_randn(tuple(yb.shape), 71))
            dwa = torch.zeros_like(w)
            dx, dg, db = cb.conv_bn_act_train_bwd(d, x, dyu, yb, raw, vec, gamma[:8], True, None, w, True, dwa, 4.0)
            bw = R.bn_bwd(dyu, yb, raw, vec[32:40], vec[40:48], gamma[:8], True)
            torch.testing.assert_close(dg.to(F64), bw["dgamma"] / 4.0, rtol=1e-5, atol=1e-5)
            draw16 = bw["draw"].half().to(F64)
            torch.testing.assert_close(dx.to(F64), R.conv_dgrad(draw16, wp.to(F64), tuple(x.shape), 2, 0, off), rtol=2e-3, atol=2e-3)
            torch.testing.assert_close(dwa.to(F64), R.conv_wgrad(x64, draw16, tuple(w.shape), 2, 0, off) / 4.0, rtol=1e-3, atol=1e-3)
        finally:
            cb.PRECISE["on"] = False
