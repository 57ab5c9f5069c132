"""Float64 references of the training kernels (csrc/bn.cu, csrc/train.cu, csrc/train_fused.cu), one plain function per operation.

Written from the operations' definitions (nn.BatchNorm2d training semantics, the transpose of bilinear align_corners=True
interpolation, a weighted sum, conv -> BatchNorm -> ReLU), not from the kernels.  Tensors are logical NCHW, CPU, float64.
The callers round the inputs once to the type the kernel reads (fp16 activations and weights, fp32 `raw`) and hand those
values in, so the only difference left between a kernel and its reference is the kernel's own arithmetic.
"""
import numpy as np
import torch

F64 = torch.float64


def _c(v):
    """per-channel vector -> broadcastable (1, C, 1, 1)"""
    return v.reshape(1, -1, 1, 1)


# ---- BatchNorm, training forward ------------------------------------------------------------------------------------------
def bn_sums(x):
    """per-channel sum and sum of squares over (N, H, W)"""
    x = x.to(F64)
    return x.sum((0, 2, 3)), (x * x).sum((0, 2, 3))


def bn_finalize(s, q, count, gamma, beta, eps, momentum, running_mean=None, running_var=None):
    """batch mean and BIASED variance normalise; the running statistics take the UNBIASED variance (count / (count - 1)).
    A variance that rounds below zero is clamped.  -> dict(mean, var, invstd, scale, shift, running_mean, running_var)"""
    mean = s.to(F64) / count
    var = (q.to(F64) / count - mean * mean).clamp_min(0.0)
    invstd = 1.0 / torch.sqrt(var + eps)
    g = torch.ones_like(mean) if gamma is None else gamma.to(F64)
    b = torch.zeros_like(mean) if beta is None else beta.to(F64)
    out = dict(mean=mean, var=var, invstd=invstd, scale=g * invstd, shift=b - mean * g * invstd)
    if running_mean is not None:
        unbiased = var * (count / (count - 1.0)) if count > 1 else var
        out["running_mean"] = (1.0 - momentum) * running_mean.to(F64) + momentum * mean
        out["running_var"] = (1.0 - momentum) * running_var.to(F64) + momentum * unbiased
    return out


def affine_act(x, scale, shift, relu):
    y = x.to(F64) * _c(scale.to(F64)) + _c(shift.to(F64))
    return y.clamp_min(0.0) if relu else y


# ---- BatchNorm (+ReLU), backward ----------------------------------------------------------------------------------------------
def bn_bwd(dy, y, raw, mean, invstd, gamma, relu, count=None, sums=None):
    """Backward of y = act(gamma * (raw - mean) * invstd + beta) with the batch statistics differentiated too.
    dz = dy * (y > 0) (torch's threshold_backward); xhat = (raw - mean) * invstd.
    -> dict(sum_dz, sum_dzxhat, draw, dgamma = sum_dzxhat, dbeta = sum_dz).  gamma None means 1.
    sums = (sum_dz, sum_dzxhat): use these in draw instead of the ones computed here (to test draw from a kernel's own sums)."""
    dz = dy.to(F64)
    if relu:
        dz = dz * (y.to(F64) > 0)
    xhat = (raw.to(F64) - _c(mean.to(F64))) * _c(invstd.to(F64))
    s = dz.sum((0, 2, 3))
    q = (dz * xhat).sum((0, 2, 3))
    n = float(dz.shape[0] * dz.shape[2] * dz.shape[3]) if count is None else float(count)
    g = torch.ones_like(s) if gamma is None else gamma.to(F64)
    sd, qd = (s, q) if sums is None else (sums[0].to(F64), sums[1].to(F64))
    draw = _c(g * invstd.to(F64)) * (dz - _c(sd) / n - xhat * _c(qd) / n)
    return dict(sum_dz=s, sum_dzxhat=q, draw=draw, dgamma=q, dbeta=s, dz=dz, xhat=xhat)


def bn_bwd_abs_terms(dz, xhat):
    """per-channel sums of |dz| and |dz * xhat|: the scale of the rounding error of an fp32 accumulation of the two sums"""
    return dz.abs().sum((0, 2, 3)), (dz * xhat).abs().sum((0, 2, 3))


# ---- FactorizedReduce channel order -------------------------------------------------------------------------------------------
def split_perm(h, hmax):
    """compact channel -> raw channel of a FactorizedReduce at maximum width with active half-width h.
    Raw order is [conv1 0..hmax | conv2 0..hmax]; compact order is [conv1 0..h | conv2 0..h | inactive], the inactive
    channels being conv1 h..hmax followed by conv2 h..hmax."""
    assert 0 <= h <= hmax
    order = list(range(h)) + [hmax + c for c in range(h)] + list(range(h, hmax)) + [hmax + c for c in range(h, hmax)]
    return torch.tensor(order, dtype=torch.long)


# ---- bilinear, align_corners=True ---------------------------------------------------------------------------------------------
def ac_matrix(n_in, n_out):
    """[n_out x n_in] float64 interpolation matrix of one axis.  The taps are computed in fp32 the way the forward computes
    them: scale = fp32(n_in - 1) / fp32(n_out - 1), src = fp32(scale * dst), i0 = trunc(src) (clamped), l1 = fp32(src - i0),
    weights (1 - l1, l1) on (i0, min(i0 + 1, n_in - 1))."""
    f = np.float32
    scale = f(n_in - 1) / f(n_out - 1) if n_out > 1 else f(0.0)
    A = np.zeros((n_out, n_in), dtype=np.float64)
    for o in range(n_out):
        src = f(scale * f(o))
        i0 = min(int(src), n_in - 1)
        i1 = i0 + (1 if i0 < n_in - 1 else 0)
        l1 = f(src - f(i0))
        A[o, i0] += float(f(f(1.0) - l1))
        A[o, i1] += float(l1)
    return torch.from_numpy(A)


def bilinear_fwd(x, Ho, Wo):
    Ah, Aw = ac_matrix(x.shape[2], Ho), ac_matrix(x.shape[3], Wo)
    return torch.einsum("oh,nchw,pw->ncop", Ah, x.to(F64), Aw)


def bilinear_bwd(dy, Hi, Wi, mask_y=None):
    """transpose of bilinear_fwd applied to dy (optionally dy * (mask_y > 0), the ReLU after the upsample):
    dx = A_h^T . dy . A_w.  -> (dx, |A_h|^T . |dy| . |A_w|), the second being the scale of an fp32 accumulation's error"""
    g = dy.to(F64)
    if mask_y is not None:
        g = g * (mask_y.to(F64) > 0)
    Ah, Aw = ac_matrix(Hi, dy.shape[2]), ac_matrix(Wi, dy.shape[3])
    dx = torch.einsum("oh,ncop,pw->nchw", Ah, g, Aw)
    mag = torch.einsum("oh,ncop,pw->nchw", Ah.abs(), g.abs(), Aw.abs())
    return dx, mag


def upsample_logits_bwd(dy_nchw, Hi, Wi, gscale):
    """backward of the logits upsample: bilinear_bwd of dy, times gscale"""
    dx, mag = bilinear_bwd(dy_nchw, Hi, Wi)
    return dx * gscale, mag * abs(gscale)


# ---- weighted multi-tensor sum ------------------------------------------------------------------------------------------------
def wsum_fwd(xs, wts):
    return sum(float(w) * x.to(F64) for w, x in zip(wts.tolist(), xs))


def wsum_bwd(dout, xs, wts, gscale):
    """-> (dxs[k] = wts[k] * dout, dwts[k] = <dout, xs[k]> / gscale, sum |dout * xs[k]| / gscale)"""
    g = dout.to(F64)
    dxs = [float(w) * g for w in wts.tolist()]
    dw = torch.stack([(g * x.to(F64)).sum() for x in xs]) / gscale
    mag = torch.stack([(g * x.to(F64)).abs().sum() for x in xs]) / gscale
    return dxs, dw, mag


# ---- conv -> BatchNorm(train) -> ReLU unit ------------------------------------------------------------------------------------
def conv(x, w, stride, pad, off=(0, 0)):
    """F.conv2d on x[:, :, off_h:, off_w:] (FactorizedReduce's second conv reads the input shifted by one pixel)"""
    return torch.nn.functional.conv2d(x.to(F64)[:, :, off[0]:, off[1]:], w.to(F64), None, stride, pad)


def conv_dgrad(draw, w, x_shape, stride, pad, off=(0, 0)):
    N, Cin, H, W = x_shape
    eff = (N, Cin, H - off[0], W - off[1])
    g = torch.nn.grad.conv2d_input(eff, w.to(F64), draw.to(F64), stride=stride, padding=pad)
    dx = torch.zeros(x_shape, dtype=F64)
    dx[:, :, off[0]:, off[1]:] = g
    return dx


def conv_wgrad(x, draw, w_shape, stride, pad, off=(0, 0)):
    return torch.nn.grad.conv2d_weight(x.to(F64)[:, :, off[0]:, off[1]:], w_shape, draw.to(F64), stride=stride, padding=pad)


def conv_bn_act_fwd(x, w, stride, pad, off, gamma, beta, eps, momentum, running_mean, running_var, relu):
    """-> dict(raw, y, and bn_finalize's entries) of the whole unit in float64"""
    raw = conv(x, w, stride, pad, off)
    s, q = bn_sums(raw)
    st = bn_finalize(s, q, raw.shape[0] * raw.shape[2] * raw.shape[3], gamma, beta, eps, momentum, running_mean, running_var)
    st["raw"] = raw
    st["y"] = affine_act(raw, st["scale"], st["shift"], relu)
    return st
