"""TEST INFRASTRUCTURE ONLY -- a numpy stand-in for `functional.train_pre` (csrc/trainpre.cu) with the same arguments and the same
arithmetic: OpenCV's 8-bit INTER_LINEAR / INTER_NEAREST resize as documented in include/fsb200.h and csrc/trainpre.cu, evaluated
on whole index vectors instead of per thread.  The CPU tests compare it with the goldens the reference wrote, which checks the
arithmetic specification before the kernel is run; nothing in the package imports it."""
import math

import numpy as np
import torch


def linear_coef(src, dst, clamp):
    """cv::resize INTER_LINEAR source index and fixed-point coefficients of every destination index"""
    scale = 1.0 / (dst / src)
    s = np.empty(dst, np.int64)
    a = np.empty((dst, 2), np.int64)
    for d in range(dst):
        f = np.float32((d + 0.5) * scale - 0.5)
        i = math.floor(f)
        f = np.float32(f - np.float32(i))
        if clamp and i < 0:
            i, f = 0, np.float32(0)
        if clamp and i >= src - 1:
            i, f = src - 1, np.float32(0)
        s[d] = i
        a[d] = (int(np.rint(np.float32(np.float32(1) - f) * np.float32(2048))), int(np.rint(f * np.float32(2048))))
    return s, a


def nearest_src(src, dst):
    """cv::resize INTER_NEAREST source index of every destination index"""
    return np.minimum(np.floor(np.arange(dst) * (1.0 / (dst / src))).astype(np.int64), src - 1)


def crop_src(crop, scaled, pos):
    """crop index -> scaled-frame index, -1 in the padding (random_crop_pad_to_shape + pad_image_to_shape)"""
    kept = min(crop, scaled - pos)
    k = np.arange(crop) - (crop - kept) // 2
    return np.where((k >= 0) & (k < kept), pos + k, -1)


def train_pre_one(img, gt, mirror, sh, sw, ph, pw, lut, crop, label_size):
    """one image: uint8 H x W x 3, uint8 H x W -> (float32 3 x ch x cw, int64 lh x lw)"""
    H, W = gt.shape
    ch, cw = crop
    lh, lw = label_size
    ys, xs = crop_src(ch, sh, ph), crop_src(cw, sw, pw)
    sy, b = linear_coef(H, sh, False)
    sx, a = linear_coef(W, sw, True)
    yv, xv = ys >= 0, xs >= 0
    yy, xx = np.where(yv, ys, 0), np.where(xv, xs, 0)
    r0, r1 = np.clip(sy[yy], 0, H - 1), np.clip(sy[yy] + 1, 0, H - 1)
    c0, c1 = sx[xx], np.minimum(sx[xx] + 1, W - 1)
    if mirror:
        c0, c1 = W - 1 - c0, W - 1 - c1
    I = img.astype(np.int64)
    a0, a1 = a[xx, 0][None, :, None], a[xx, 1][None, :, None]
    s0 = I[r0][:, c0] * a0 + I[r0][:, c1] * a1
    s1 = I[r1][:, c0] * a0 + I[r1][:, c1] * a1
    b0, b1 = b[yy, 0][:, None, None], b[yy, 1][:, None, None]
    v = np.clip(((((s0 >> 4) * b0) >> 16) + (((s1 >> 4) * b1) >> 16) + 2) >> 2, 0, 255)
    out = np.stack([lut[c][v[:, :, c]] for c in range(3)])
    out[:, ~(yv[:, None] & xv[None, :])] = 0.0
    yc, xc = crop_src(ch, sh, ph)[nearest_src(ch, lh)], crop_src(cw, sw, pw)[nearest_src(cw, lw)]
    rows = nearest_src(H, sh)[np.where(yc >= 0, yc, 0)]
    cols = nearest_src(W, sw)[np.where(xc >= 0, xc, 0)]
    if mirror:
        cols = W - 1 - cols
    lab = gt[rows][:, cols].astype(np.int64)
    lab[~((yc >= 0)[:, None] & (xc >= 0)[None, :])] = 255
    return out.astype(np.float32), lab


def train_pre(img, gt, geom, lut, crop, label_size, out_img=None, out_gt=None):
    """stand-in of functional.train_pre on CPU tensors (same arguments, same packed layout)"""
    img, gt, geom, lut = img.numpy(), gt.numpy(), geom.numpy(), lut.numpy().reshape(3, 256)
    imgs, labs = [], []
    for H, W, mirror, sh, sw, ph, pw, off in geom.tolist():
        im = img[off * 3:(off + H * W) * 3].reshape(H, W, 3)
        g = gt[off:off + H * W].reshape(H, W)
        a, b = train_pre_one(im, g, mirror, sh, sw, ph, pw, lut, crop, label_size)
        imgs.append(a)
        labs.append(b)
    return torch.from_numpy(np.stack(imgs)), torch.from_numpy(np.stack(labs))
