"""TEST INFRASTRUCTURE ONLY -- a torch-CPU stand-in for the tensor-level wrappers of `fasterseg_b200.functional`.

The product has no CPU path (`_lib.lib()` raises without the CUDA library).  To test the HOST LOGIC of the boundary on the
build machine -- which operator calls which unit with which channel slice, the zero-copy concat offsets, the autograd wiring of
the training units, gradient accumulation into `param.grad`, the branch / cell / MixedOp plumbing of both networks -- the
`-m "not gpu"` tests swap the ~35 wrappers for the functions below (same signatures, same tensor conventions: logical NCHW
fp16 views with channels-last strides, fp32 master weights, fp16 gradients carrying GRAD_SCALE) and run the real
`fasterseg_b200` modules on CPU tensors against the oracle.  Arithmetic is fp32 with results rounded where the kernels store
fp16, i.e. the storage semantics documented in include/fsb200.h.  Nothing here is imported by the package.
"""
import contextlib
import types

import numpy as np

import torch
import torch.nn.functional as TF

from fasterseg_b200 import functional as F_
from fasterseg_b200._lib import ConvDesc

_empty = F_.empty_nhwc  # pure torch, device-agnostic: reused as is


def nhwc_info(t, dtype=torch.float16):
    if t.dtype != dtype or t.dim() != 4:
        raise ValueError("expected a 4-D %s tensor, got %s %s" % (dtype, t.dtype, tuple(t.shape)))
    N, Cc, H, W = t.shape
    sn, sc, sh, sw = t.stride()
    cs = sw
    ok = (Cc == 1 or sc == 1) and cs >= Cc and (H == 1 or sh == W * cs) and (N == 1 or sn == H * W * cs)
    if W == 1:
        cs = sh if H > 1 else (sn if N > 1 else max(Cc, 1))
        ok = (Cc == 1 or sc == 1)
    if not ok:
        raise ValueError("tensor is not NHWC-addressable: shape %s strides %s" % (tuple(t.shape), t.stride()))
    return N, Cc, H, W, cs


def _put(out, val):
    """store `val` (fp32, logical NCHW) into the view `out`, rounding to its dtype"""
    out.copy_(val.to(out.dtype))
    return out


def to_nhwc_half(x):
    if F_.is_nhwc_half(x):
        return x
    if x.dim() != 4 or x.dtype not in (torch.float32, torch.float16):
        raise ValueError("expected an NCHW fp32/fp16 tensor")
    N, Cc, H, W = x.shape
    return _put(_empty(N, Cc, H, W, x.device), x.detach().float())


def to_nchw(x, dtype=torch.float32):
    nhwc_info(x)
    return x.detach().to(dtype).contiguous()


def pack_conv_weight(w, Cin, Cout, ksize, out=None):
    assert w.dtype == torch.float32 and w.dim() == 4 and w.shape[2] == ksize and w.shape[3] == ksize
    packed = w[:Cout, :Cin].detach().half().contiguous()
    if out is not None:
        out.copy_(packed)
        return out
    return packed


def bn_fold(gamma, beta, mean, var, eps, conv_bias=None):
    g = torch.ones_like(mean) if gamma is None else gamma.float()
    b = torch.zeros_like(mean) if beta is None else beta.float()
    scale = g / torch.sqrt(var.float() + eps)
    shift = b - mean.float() * scale
    if conv_bias is not None:
        shift = shift + conv_bias.float() * scale
    return scale.contiguous(), shift.contiguous()


# float64 accumulation in the stand-in convs / gradients: makes results independent of the summation order (needed where two
# code paths that differ only in zero-padded channels must agree to the last fp32 bit, tests/test_graphed_cpu.py)
PRECISE = {"on": False}


# shape-only convs and conv gradients: zeros of the right shape instead of the arithmetic, for recording which calls a network
# makes where its control flow does not depend on the data (tests/conv_fwd_census.py)
SHAPES_ONLY = {"on": False}


@contextlib.contextmanager
def shapes_only():
    SHAPES_ONLY["on"] = True
    try:
        yield
    finally:
        SHAPES_ONLY["on"] = False


def _conv2d(x, w, stride, pad):
    if SHAPES_ONLY["on"]:
        N, _, H, W = x.shape
        k = w.shape[2]
        return torch.zeros((N, w.shape[0], (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1), dtype=torch.float32)
    return TF.conv2d(x, w, None, stride, pad)


def _raw_conv(x, w16, stride, pad, off):
    xin = x[:, :, off[0]:, off[1]:].float()
    if SHAPES_ONLY["on"]:
        return _conv2d(xin, w16, stride, pad)
    if PRECISE["on"]:
        return TF.conv2d(xin.double(), w16.double(), None, stride, pad).float()
    return TF.conv2d(xin, w16.float(), None, stride, pad)


def _add_stats(stats, y, Cout, at=0):
    """stats: [rows, 2 * SC] (the stand-in uses ONE zero-initialised row) or [2 * SC]"""
    row = stats[0] if stats.dim() == 2 else stats
    SC = row.numel() // 2
    yd = y.double()
    row[at:at + Cout] += yd.sum((0, 2, 3)).float()
    row[SC + at:SC + at + Cout] += (yd * yd).sum((0, 2, 3)).float()


def conv_stats_buffer(x, Cout, ksize, stride, pad, off=(0, 0), total_C=None, force_direct=False):
    return torch.zeros((1, 2 * (Cout if total_C is None else int(total_C))), dtype=torch.float32)


def rowsum(rows):
    return rows.double().sum(0, keepdim=True).float()


def conv_fwd(x, wpacked, Cout, ksize, stride, pad, scale=None, shift=None, relu=False, out=None, off=(0, 0),
             stats=None, force_direct=False, out_f32=False, stats_off=0, down2=False, up2=False):
    N, Cin, H, W, _ = nhwc_info(x)
    assert tuple(wpacked.shape) == (Cout, Cin, ksize, ksize), (tuple(wpacked.shape), (Cout, Cin, ksize, ksize))
    if down2:      # nearest(x, (H/2, W/2)): the even rows and columns (FSB_CONV_X_DOWN2)
        assert H % 2 == 0 and W % 2 == 0 and stride == 1 and stats is None and not out_f32
        x = x[:, :, ::2, ::2]
        H, W = H // 2, W // 2
    y = _raw_conv(x, wpacked, stride, pad, off)
    Ho, Wo = F_.conv_out_size(H, W, ksize, stride, pad, 1, off[0], off[1])
    assert tuple(y.shape) == (N, Cout, Ho, Wo)
    if stats is not None:
        _add_stats(stats, y, Cout, stats_off)
    if scale is not None:
        y = y * scale.view(1, -1, 1, 1)
    if shift is not None:
        y = y + shift.view(1, -1, 1, 1)
    if relu:
        y = y.relu()
    if up2:        # nearest(y, (2Ho, 2Wo)): every output pixel to its 2x2 block (FSB_CONV_Y_UP2)
        assert stats is None and not out_f32
        y = y.repeat_interleave(2, 2).repeat_interleave(2, 3)
        Ho, Wo = 2 * Ho, 2 * Wo
    odt = torch.float32 if out_f32 else torch.float16
    if out is None:
        out = _empty(N, Cout, Ho, Wo, x.device, dtype=odt)
    assert tuple(out.shape) == (N, Cout, Ho, Wo) and out.dtype == odt
    nhwc_info(out, odt)
    return _put(out, y)


def stem_conv_nchw(x, w, scale, shift, relu=True, out=None):
    assert x.dim() == 4 and x.shape[1] == 3 and tuple(w.shape[1:]) == (3, 3, 3)
    y = _conv2d(x.half().float(), w.half().float(), 2, 1)
    if scale is not None:
        y = y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    if relu:
        y = y.relu()
    if out is None:
        out = _empty(y.shape[0], y.shape[1], y.shape[2], y.shape[3], x.device)
    return _put(out, y)


def stem_conv_u8hwc(x_u8, lut, w, scale, shift, relu=True, out=None):
    N, _, H, W = x_u8.shape
    xn = torch.stack([lut.view(3, 256)[c][x_u8[:, c].long()] for c in range(3)], dim=1).float()   # fp16 table values
    y = _conv2d(xn, w.half().float(), 2, 1)
    if scale is not None:
        y = y * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    if relu:
        y = y.relu()
    if out is None:
        out = _empty(y.shape[0], y.shape[1], y.shape[2], y.shape[3], x_u8.device)
    return _put(out, y)


def confusion_matrix(pred_u8, gt, n_cl, out=None):
    if out is None:
        out = torch.zeros(n_cl * n_cl + 2, dtype=torch.int64)
    g = gt.reshape(-1).long()
    p = pred_u8.reshape(-1).long()
    k = (g >= 0) & (g < n_cl)
    out[:n_cl * n_cl] += torch.bincount(n_cl * g[k] + p[k], minlength=n_cl * n_cl)
    out[n_cl * n_cl] += int(k.sum())
    out[n_cl * n_cl + 1] += int((p[k] == g[k]).sum())
    return out


def _interp(x32, size):
    return TF.interpolate(x32, size=(int(size[0]), int(size[1])), mode="bilinear", align_corners=True)


def bilinear(x, size, relu=False, out=None):
    N, Cc, _, _, _ = nhwc_info(x)
    y = _interp(x.float(), size)
    if relu:
        y = y.relu()
    if out is None:
        out = _empty(N, Cc, int(size[0]), int(size[1]), x.device)
    assert tuple(out.shape) == tuple(y.shape)
    return _put(out, y)


def upsample_logits(x, size, dtype=torch.float32, out=None):
    nhwc_info(x)
    y = _interp(x.float(), size).to(dtype).contiguous()
    if out is not None:
        out.copy_(y)
        return out
    return y


def upsample_argmax(x, size, out=None):
    nhwc_info(x)
    lab = _interp(x.float(), size).argmax(1).to(torch.uint8)
    if out is not None:
        out.copy_(lab)
        return out
    return lab


def _nearest(x32, size):
    """torch's legacy 'nearest' index rule (src = floor(dst * in / out)), as the library's nearest kernels (include/fsb200.h)"""
    return TF.interpolate(x32, size=(int(size[0]), int(size[1])), mode="nearest")


def nearest(x, size, out=None):
    N, Cc, _, _, _ = nhwc_info(x)
    y = _nearest(x.float(), size)
    if out is None:
        out = _empty(N, Cc, int(size[0]), int(size[1]), x.device)
    assert tuple(out.shape) == tuple(y.shape)
    nhwc_info(out)
    return _put(out, y)


def upsample_logits_nearest(x, size, dtype=torch.float32, out=None):
    nhwc_info(x)
    y = _nearest(x.float(), size).to(dtype).contiguous()
    if out is not None:
        out.copy_(y)
        return out
    return y


def upsample_argmax_nearest(x, size, out=None):
    nhwc_info(x)
    lab = _nearest(x.float(), size).argmax(1).to(torch.uint8)
    if out is not None:
        out.copy_(lab)
        return out
    return lab


def copy_channels(x, out):
    assert tuple(x.shape) == tuple(out.shape)
    nhwc_info(x), nhwc_info(out)
    out.copy_(x)
    return out


def bn_stats(x):
    N, Cc, H, W, _ = nhwc_info(x)
    stats = torch.zeros(2 * Cc, dtype=torch.float32)
    _add_stats(stats, x.float(), Cc)
    return stats


def bn_finalize(stats, count, gamma, beta, eps, momentum, running_mean, running_var, want_save=False):
    if stats.dim() == 2:
        stats = stats.double().sum(0).float()
    Cc = stats.numel() // 2
    mean = stats[:Cc].double() / count
    var = (stats[Cc:].double() / count - mean * mean).clamp_min(0)
    invstd = 1.0 / torch.sqrt(var + eps)
    scale = gamma.detach().double() * invstd
    shift = beta.detach().double() - mean * scale
    if running_mean is not None:
        with torch.no_grad():
            running_mean.mul_(1 - momentum).add_(momentum * mean.float())
            unbiased = var * (count / max(count - 1, 1))
            running_var.mul_(1 - momentum).add_(momentum * unbiased.float())
    return scale.float(), shift.float(), mean.float(), invstd.float()


def affine_act(x, scale, shift, relu=False, out=None):
    N, Cc, H, W, _ = nhwc_info(x, x.dtype)
    y = x.float() * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    if relu:
        y = y.relu()
    if out is None:
        out = _empty(N, Cc, H, W, x.device)
    return _put(out, y)


def _dz_xhat(dy, y, raw, mean, invstd, relu):
    dz = dy.float()
    if relu:
        dz = dz * (y.float() > 0)
    v = lambda t: t.detach().float().view(1, -1, 1, 1)
    return dz, (raw.float() - v(mean)) * v(invstd)


def bn_bwd_sums(dy, y, raw, mean, invstd, relu):
    nhwc_info(dy)
    dz, xhat = _dz_xhat(dy, y, raw, mean, invstd, relu)
    return torch.cat([dz.double().sum((0, 2, 3)), (dz.double() * xhat.double()).sum((0, 2, 3))]).float()


def bn_bwd_apply(dy, y, raw, mean, invstd, gamma, sums, count, relu, gscale, want_param_grads=True):
    N, Cc, H, W, _ = nhwc_info(dy)
    dz, xhat = _dz_xhat(dy, y, raw, mean, invstd, relu)
    v = lambda t: t.detach().float().view(1, -1, 1, 1)
    draw = v(gamma) * v(invstd) * (dz - v(sums[:Cc]) / count - xhat * v(sums[Cc:]) / count)
    out = _put(_empty(N, Cc, H, W, dy.device), draw)
    if not want_param_grads:
        return out, None, None
    return out, sums[Cc:] / gscale, sums[:Cc] / gscale


def relu_bwd(dy, y):
    N, Cc, H, W, _ = nhwc_info(dy)
    return _put(_empty(N, Cc, H, W, dy.device), dy.float() * (y.float() > 0))


def pack_conv_weight_dgrad(w, Cin, Cout, ksize, out=None):
    return pack_conv_weight(w, Cin, Cout, ksize, out=out)


def conv_dgrad(dy, w, x_shape, Cin, Cout, ksize, stride, pad, off=(0, 0), wpacked_t=None, force_direct=False):
    N, _, H, W = x_shape
    nhwc_info(dy)
    w16 = w[:Cout, :Cin].detach().half().float()
    eff = (N, Cin, H - off[0], W - off[1])
    if SHAPES_ONLY["on"]:
        g = torch.zeros(eff, dtype=torch.float32)
    elif PRECISE["on"]:
        g = torch.nn.grad.conv2d_input(eff, w16.double(), dy.double(), stride=stride, padding=pad).float()
    else:
        g = torch.nn.grad.conv2d_input(eff, w16, dy.float(), stride=stride, padding=pad)
    full = torch.zeros((N, Cin, H, W), dtype=torch.float32)
    full[:, :, off[0]:, off[1]:] = g
    return _put(_empty(N, Cin, H, W, dy.device), full)


def conv_wgrad(x, dy, w_like, Cin, Cout, ksize, stride, pad, gscale, off=(0, 0), accumulate_into=None, force_direct=False):
    xin = x[:, :, off[0]:, off[1]:].float()
    if SHAPES_ONLY["on"]:
        g = torch.zeros((Cout, Cin, ksize, ksize), dtype=torch.float32)
    elif PRECISE["on"]:
        g = (torch.nn.grad.conv2d_weight(xin.double(), (Cout, Cin, ksize, ksize), dy.double(), stride=stride, padding=pad) / gscale).float()
    else:
        g = torch.nn.grad.conv2d_weight(xin, (Cout, Cin, ksize, ksize), dy.float(), stride=stride, padding=pad) / gscale
    if accumulate_into is not None:
        assert accumulate_into.dtype == torch.float32 and accumulate_into.shape == w_like.shape
        with torch.no_grad():
            accumulate_into[:Cout, :Cin] += g
        return accumulate_into
    dw = torch.zeros(w_like.shape, dtype=torch.float32)
    dw[:Cout, :Cin] = g
    return dw


def _interp_bwd(g32, in_hw):
    x0 = torch.zeros((g32.shape[0], g32.shape[1], in_hw[0], in_hw[1]), dtype=torch.float32, requires_grad=True)
    with torch.enable_grad():
        y0 = _interp(x0, g32.shape[2:])
    return torch.autograd.grad(y0, x0, g32)[0]


def bilinear_bwd(dy, in_hw, relu_mask_y=None):
    N, Cc, _, _, _ = nhwc_info(dy)
    g = dy.float()
    if relu_mask_y is not None:
        g = g * (relu_mask_y.float() > 0)
    return _put(_empty(N, Cc, in_hw[0], in_hw[1], dy.device), _interp_bwd(g, in_hw))


def upsample_logits_bwd(dy_nchw, in_hw, gscale):
    N, Cc = dy_nchw.shape[:2]
    return _put(_empty(N, Cc, in_hw[0], in_hw[1], dy_nchw.device), _interp_bwd(dy_nchw.float() * gscale, in_hw))


def nchw_grad_to_nhwc(dy_nchw, gscale):
    N, Cc, H, W = dy_nchw.shape
    return _put(_empty(N, Cc, H, W, dy_nchw.device), dy_nchw.float() * gscale)


def wsum_fwd(xs, wts, out=None):
    N, Cc, H, W, _ = nhwc_info(xs[0])
    acc = sum(float(wts[k]) * xs[k].float() for k in range(len(xs)))
    if out is None:
        out = _empty(N, Cc, H, W, xs[0].device)
    return _put(out, acc)


def wsum_bwd(dout, xs, wts, need_dx, need_dw, gscale):
    N, Cc, H, W, _ = nhwc_info(dout)
    g = dout.float()
    dxs = [_put(_empty(N, Cc, H, W, dout.device), float(wts[k]) * g) if need_dx[k] else None for k in range(len(xs))]
    dw = torch.stack([(g * xs[k].float()).sum() / gscale for k in range(len(xs))]).float() if need_dw else None
    return dxs, dw


def add_inplace(x, y):
    y.copy_((y.float() + x.float()).to(y.dtype))
    return y


def conv_bn_act_train_fwd(x, wpacked, Cout, ksize, stride, pad, off, gamma, beta, eps, momentum, running_mean, running_var,
                          num_batches_tracked, relu, sel=None, width_idx=None):
    assert sel is None and width_idx is None, "device-selected BatchNorm sets exist on the GPU only"
    N, Cin, H, W, xcs = nhwc_info(x)
    Ho, Wo = F_.conv_out_size(H, W, ksize, stride, pad, 1, off[0], off[1])
    stats = torch.zeros(2 * Cout, dtype=torch.float32)
    raw = conv_fwd(x, wpacked, Cout, ksize, stride, pad, off=off, stats=stats, out_f32=True)
    scale, shift, mean, invstd = bn_finalize(stats, N * Ho * Wo, gamma, beta, eps, momentum, running_mean, running_var, True)
    if num_batches_tracked is not None:
        num_batches_tracked += 1
    y = affine_act(raw, scale, shift, relu=relu)
    vec = torch.cat([stats, scale, shift, mean, invstd])
    cpad = (Cout + 7) // 8 * 8
    d = ConvDesc(N, H, W, Cin, Cout, ksize, stride, pad, 1, off[0], off[1], Ho, Wo, xcs, cpad, 0)
    return y, raw, vec, d


def conv_bn_act_train_bwd(d, x, dy, y, raw, vec, gamma, relu, wpacked_t, w, need_dx, dw_accum, gscale, sel=None, width_idx=None):
    N, Cout, Ho, Wo, _ = nhwc_info(dy)
    mean, invstd = vec[4 * Cout:5 * Cout], vec[5 * Cout:6 * Cout]
    sums = bn_bwd_sums(dy, y, raw, mean, invstd, relu)
    draw, dg, db = bn_bwd_apply(dy, y, raw, mean, invstd, gamma, sums, N * Ho * Wo, relu, gscale)
    off = (d.off_h, d.off_w)
    dx = conv_dgrad(draw, w, (N, d.Cin, d.H, d.W), d.Cin, Cout, d.ksize, d.stride, d.pad, off=off) if need_dx else None
    if dw_accum is not None:
        conv_wgrad(x, draw, w, d.Cin, Cout, d.ksize, d.stride, d.pad, gscale, off=off, accumulate_into=dw_accum)
    return dx, dg, db


# ---- device-selected BatchNorm sets (engine.SelBN): the stand-in reads the width index from the context's vector ----------
def _sel_bn(sel):
    return sel.bns[int(sel.ctx.width_idx[sel.slot])]


def _split_perm(h, hmax):
    """compact channel -> raw channel of a FactorizedReduce at maximum width (csrc/bn.cu split_remap)"""
    def remap(c):
        if c < h:
            return c
        if c < 2 * h:
            return hmax + (c - h)
        k = c - 2 * h
        return h + k if k < hmax - h else hmax + h + (k - (hmax - h))
    return torch.tensor([remap(c) for c in range(2 * hmax)], dtype=torch.long)


def _pad(v, C):
    out = torch.zeros(C, dtype=torch.float32)
    out[:v.numel()] = v
    return out


def bn_finalize_sel(stats, count, sel, hmax=0):
    bn = _sel_bn(sel)
    Ca, Cc = bn.num_features, stats.shape[1] // 2
    tot = stats.double().sum(0).float()
    s, q = tot[:Cc], tot[Cc:]
    if hmax:
        perm = _split_perm(Ca // 2, hmax)
        s, q = s[perm], q[perm]
    scale, shift, mean, invstd = bn_finalize(torch.cat([s[:Ca], q[:Ca]]), count, bn.weight, bn.bias, sel.eps, sel.momentum,
                                             bn.running_mean, bn.running_var, True)
    if bn.num_batches_tracked is not None:
        bn.num_batches_tracked += 1
    return _pad(scale, Cc), _pad(shift, Cc), _pad(mean, Cc), _pad(invstd, Cc)


def affine_act_sel(x, scale, shift, sel, hmax, relu=False):
    if hmax:
        perm = _split_perm(_sel_bn(sel).num_features // 2, hmax)
        xc = _put(_empty(x.shape[0], x.shape[1], x.shape[2], x.shape[3], x.device, dtype=x.dtype), x[:, perm].float())
        return affine_act(xc, scale, shift, relu=relu)
    return affine_act(x, scale, shift, relu=relu)


def bn_bwd_sel(dy, y, raw, mean, invstd, count, relu, gscale, sel, hmax=0, world=1):
    assert world == 1, "the CPU stand-in has no peer exchange (SyncBN over sel kernels is covered on the GPU)"
    bn = _sel_bn(sel)
    Ca, Cc = bn.num_features, dy.shape[1]
    perm = _split_perm(Ca // 2, hmax) if hmax else None
    rawc = raw if perm is None else raw[:, perm]
    sums = bn_bwd_sums(dy, y, rawc, mean, invstd, relu)
    gamma = _pad(bn.weight.detach().float(), Cc)
    draw, _, _ = bn_bwd_apply(dy, y, rawc, mean, invstd, gamma, sums, count, relu, gscale, want_param_grads=False)
    with torch.no_grad():
        sel.ctx.flat.sview(bn.weight).add_(sums[Cc:Cc + Ca] / gscale)
        sel.ctx.flat.sview(bn.bias).add_(sums[:Ca] / gscale)
    if perm is None:
        return draw
    out = _empty(dy.shape[0], Cc, dy.shape[2], dy.shape[3], dy.device)
    out[:, perm] = draw
    return out


def conv_bn_act_train_fwd_sel(x, wpacked, Cout, ksize, stride, pad, off, sel, relu):
    N, Cin, H, W, xcs = nhwc_info(x)
    Ho, Wo = F_.conv_out_size(H, W, ksize, stride, pad, 1, off[0], off[1])
    stats = torch.zeros((1, 2 * Cout), dtype=torch.float32)
    raw = conv_fwd(x, wpacked, Cout, ksize, stride, pad, off=off, stats=stats, out_f32=True)
    scale, shift, mean, invstd = bn_finalize_sel(stats, N * Ho * Wo, sel)
    y = affine_act(raw, scale, shift, relu=relu)
    cpad = (Cout + 7) // 8 * 8
    d = ConvDesc(N, H, W, Cin, Cout, ksize, stride, pad, 1, off[0], off[1], Ho, Wo, xcs, cpad, 0)
    return y, raw, (mean, invstd), d


def conv_bn_act_train_bwd_sel(d, x, dy, y, raw, vec, sel, relu, wpacked_t, w, need_dx, dw_accum, gscale):
    N, Cout, Ho, Wo, _ = nhwc_info(dy)
    mean, invstd = vec
    draw = bn_bwd_sel(dy, y, raw, mean, invstd, N * Ho * Wo, relu, gscale, sel)
    off = (d.off_h, d.off_w)
    dx = conv_dgrad(draw, w, (N, d.Cin, d.H, d.W), d.Cin, Cout, d.ksize, d.stride, d.pad, off=off) if need_dx else None
    if dw_accum is not None:
        conv_wgrad(x, draw, w, d.Cin, Cout, d.ksize, d.stride, d.pad, gscale, off=off, accumulate_into=dw_accum)
    return dx


_PATCHED = ("nhwc_info", "to_nhwc_half", "to_nchw", "pack_conv_weight", "bn_fold", "conv_stats_buffer", "rowsum", "conv_fwd", "stem_conv_nchw", "bilinear",
            "upsample_logits", "upsample_argmax", "nearest", "upsample_logits_nearest", "upsample_argmax_nearest", "copy_channels", "bn_stats", "bn_finalize", "affine_act", "bn_bwd_sums", "bn_bwd_apply", "relu_bwd",
            "pack_conv_weight_dgrad", "conv_dgrad", "conv_wgrad", "bilinear_bwd", "upsample_logits_bwd", "nchw_grad_to_nhwc",
            "wsum_fwd", "wsum_bwd", "add_inplace", "conv_bn_act_train_fwd", "conv_bn_act_train_bwd",
            "stem_conv_u8hwc", "confusion_matrix", "bn_finalize_sel", "affine_act_sel", "bn_bwd_sel", "conv_bn_act_train_fwd_sel", "conv_bn_act_train_bwd_sel",
            "flat_chunk", "flat_grad_norm", "flat_scale", "flat_sgd",
            "loss_logp_fwd", "kth_smallest", "ohem_reduce", "loss_ce_bwd", "loss_kl_fwd", "loss_kl_bwd")


# ---- fused criteria (csrc/loss.cu): same contracts, arithmetic by torch autograd through F.interpolate -----------------------------
def _valid_labels(target, ignore_label, Cc):
    return (target != ignore_label) & (target >= 0) & (target < Cc)


def _logp_true(up, target, valid):
    t = torch.where(valid, target, torch.zeros_like(target))
    return up.gather(1, t.unsqueeze(1)).squeeze(1) - torch.logsumexp(up, dim=1)


def loss_logp_fwd(x, target, size, ignore_label):
    N, Cc, _, _, _ = nhwc_info(x)
    up = _interp(x.float(), size)
    valid = _valid_labels(target, ignore_label, Cc)
    logp = torch.where(valid, _logp_true(up, target, valid), torch.zeros((), dtype=torch.float32))      # ignored pixels: probability 1
    return logp.contiguous(), torch.logsumexp(up, dim=1).contiguous()


def kth_smallest(x, k):
    assert x.dtype == torch.float32 and x.is_contiguous() and 1 <= k <= x.numel()
    return torch.kthvalue(x.reshape(-1), int(k)).values.clone()


def _kept(logp_t, target, ignore_label, Cc, thr):
    kept = _valid_labels(target, ignore_label, Cc)
    if thr is not None:
        kept = kept & (logp_t.reshape(target.shape) <= thr)
    return kept


def ohem_reduce(logp_t, target, ignore_label, num_classes, thr=None):
    kept = _kept(logp_t, target, ignore_label, num_classes, thr).reshape(-1)
    lp = logp_t.reshape(-1)
    return torch.stack([-(lp[kept].double().sum()).float(), kept.sum().float()])


def _to_grad_buffer(g32, gscale, like, out):
    g = (g32 * gscale).half()
    if out is None:
        out = F_.empty_nhwc(*like.shape, like.device)
        out.copy_(g)
    else:
        out.copy_((out.float() + g.float()).half())
    return out


def loss_ce_bwd(x, target, size, ignore_label, lse, logp_t, thr, coef, gscale, out=None):
    N, Cc, _, _, _ = nhwc_info(x)
    with torch.enable_grad():
        xr = x.detach().float().requires_grad_(True)
        up = _interp(xr, size)
        valid = _valid_labels(target, ignore_label, Cc)
        kept = _kept(logp_t, target, ignore_label, Cc, thr)       # the FORWARD's log-probabilities decide, as in the kernel
        loss = -(torch.where(kept, _logp_true(up, target, valid), torch.zeros((), dtype=torch.float32))).sum() * coef.reshape(())
        g, = torch.autograd.grad(loss, xr)
    return _to_grad_buffer(g, gscale, x, out)


def _kl_sum(us, ut):
    logp = torch.log_softmax(us, dim=1)
    logq = torch.log_softmax(ut, dim=1)
    return (logq.exp() * (logq - logp)).sum()


def loss_kl_fwd(xs, xt, size):
    us, ut = _interp(xs.float(), size), _interp(xt.float(), size)
    return _kl_sum(us.double(), ut.double()).float(), torch.logsumexp(us, dim=1).contiguous(), torch.logsumexp(ut, dim=1).contiguous()


def loss_kl_bwd(xs, xt, size, lse_s, lse_t, coef, gscale, out=None):
    with torch.enable_grad():
        xr = xs.detach().float().requires_grad_(True)
        loss = _kl_sum(_interp(xr, size), _interp(xt.detach().float(), size)) * coef.reshape(())
        g, = torch.autograd.grad(loss, xr)
    return _to_grad_buffer(g, gscale, xs, out)


# ---- flat step tail (csrc/optim.cu) on host memory: the segment table holds raw storage pointers, exactly as on the device ------------
FLAT_CHUNK = 4096


def flat_chunk():
    return FLAT_CHUNK


def _flat_tables(block_map, nblocks, segs, live):
    """decode the tables optim.FlatTables built and check their invariants (what the kernels rely on without checking)"""
    import ctypes
    seg = np.frombuffer(segs.numpy().tobytes(), dtype=[("p", "<u8"), ("off", "<u4"), ("n", "<u4")])
    bm = block_map.numpy().reshape(-1, 2)
    assert bm.shape[0] == nblocks and block_map.dtype == torch.int32 and live.dtype == torch.uint8 and live.numel() == len(seg)
    want = np.concatenate([np.stack([np.full((int(n) + FLAT_CHUNK - 1) // FLAT_CHUNK, i), np.arange((int(n) + FLAT_CHUNK - 1) // FLAT_CHUNK)], axis=1)
                           for i, n in enumerate(seg["n"])])
    assert np.array_equal(bm, want), "block map does not cover every segment chunk by chunk"
    ends = seg["off"].astype(np.int64) + seg["n"]
    assert np.all(seg["off"] % 4 == 0) and np.all(seg["off"][1:] >= ends[:-1]), "segments overlap or are misaligned"

    def param(i):
        n = int(seg["n"][i])
        return np.ctypeslib.as_array((ctypes.c_float * n).from_address(int(seg["p"][i])))
    return seg, live.numpy(), param


def flat_grad_norm(block_map, nblocks, segs, live, G, partial, extra_sq, max_norm, out2):
    seg, lv, _ = _flat_tables(block_map, nblocks, segs, live)
    g = G.numpy()
    sq = 0.0
    for i in np.nonzero(lv)[0]:
        v = g[int(seg["off"][i]):int(seg["off"][i]) + int(seg["n"][i])].astype(np.float64)
        sq += float((v * v).sum())
    if extra_sq is not None:
        sq += float(extra_sq[0])
    norm = np.float32(np.sqrt(sq))
    out2[0] = float(norm)
    out2[1] = float(min(np.float32(1.0), np.float32(max_norm) / (norm + np.float32(1e-6))))


def flat_scale(block_map, nblocks, segs, live, G, coef):
    seg, lv, _ = _flat_tables(block_map, nblocks, segs, live)
    g = G.numpy()
    c = np.float32(float(coef[0]))
    for i in np.nonzero(lv)[0]:
        g[int(seg["off"][i]):int(seg["off"][i]) + int(seg["n"][i])] *= c


def flat_sgd(block_map, nblocks, segs, live, G, M, lr, momentum, weight_decay):
    seg, lv, param = _flat_tables(block_map, nblocks, segs, live)
    g, m = G.numpy(), M.numpy()
    lr, momentum, wd = np.float32(lr), np.float32(momentum), np.float32(weight_decay)
    for i in np.nonzero(lv)[0]:
        lo, hi = int(seg["off"][i]), int(seg["off"][i]) + int(seg["n"][i])
        p = param(i)
        m[lo:hi] = momentum * m[lo:hi] + (g[lo:hi] + wd * p)
        p -= lr * m[lo:hi]


@contextlib.contextmanager
def installed():
    """Swap the wrappers of fasterseg_b200.functional for the CPU stand-ins for the duration of the block."""
    saved = {name: getattr(F_, name) for name in _PATCHED}
    here = globals()
    try:
        for name in _PATCHED:
            setattr(F_, name, here[name])
        yield types.SimpleNamespace(names=_PATCHED)
    finally:
        for name, fn in saved.items():
            setattr(F_, name, fn)
