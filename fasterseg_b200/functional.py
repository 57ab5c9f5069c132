"""Tensor-level wrappers over the C ABI (include/fsb200.h).

Activations are torch fp16 tensors with logical shape (N, C, H, W) and channels-last strides
(N: H*W*cs, C: 1, H: W*cs, W: cs) where the channel stride `cs` may exceed C (a channel slice of a
wider concat buffer).  PyTorch is plumbing here: it owns the device memory and the stream; every
arithmetic kernel is ours.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import (ConvDesc, FSB_ACT_IN_F32, FSB_CONV_AFFINE, FSB_CONV_FORCE_DIRECT, FSB_CONV_OUT_F32, FSB_CONV_RELU,
                   FSB_CONV_STATS, FSB_CONV_X_DOWN2, FSB_CONV_Y_UP2, check)


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream() -> int:
    """cudaStream_t of torch's current stream.  torch.cuda.current_stream() costs ~15 us per call (device lookups, Stream
    object construction); the raw accessor is ~50x cheaper and this is called once per kernel launch."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


def _on_device(t: torch.Tensor) -> bool:
    """Every tensor handed to the library must live on the GPU (there is no CPU path).  One predicate, so that the host-side
    tests can run the wrappers' marshalling against a fake library with CPU tensors (tests/test_marshalling_cpu.py)."""
    return t.is_cuda


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def empty_nhwc(N, Cc, H, W, device, dtype=torch.float16) -> torch.Tensor:
    """(N, C, H, W)-shaped view of a fresh NHWC buffer; the pixel stride is rounded up to 8 channels so that
    every pixel starts on a 16-byte boundary (vector stores, TMA strides).  Called ~15 k times per supernet step:
    when no padding is needed the strided tensor is created in ONE torch call (no permute / slice objects)."""
    cpad = (Cc + 7) // 8 * 8
    if cpad == Cc:
        return torch.empty_strided((N, Cc, H, W), (H * W * Cc, 1, W * Cc, Cc), device=device, dtype=dtype)
    # padded: allocate the full (N, H, W, cpad) block -- the pad lanes of the last pixel must belong to the allocation,
    # vector stores touch them -- and hand out the first Cc channels
    return torch.empty((N, H, W, cpad), device=device, dtype=dtype).permute(0, 3, 1, 2)[:, :Cc]


def nhwc_info(t: torch.Tensor, dtype=torch.float16) -> Tuple[int, int, int, int, int]:
    """-> (N, C, H, W, channel_stride); raises unless `t` is a channels-last addressable CUDA tensor of `dtype`."""
    if t.dtype != dtype or t.dim() != 4 or not _on_device(t):
        raise ValueError("expected a 4-D CUDA %s tensor, got %s %s" % (dtype, t.dtype, tuple(t.shape)))
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


def is_nhwc_half(t: torch.Tensor) -> bool:
    try:
        nhwc_info(t)
        return True
    except ValueError:
        return False


def to_nhwc_half(x: torch.Tensor) -> torch.Tensor:
    """Reference-layout tensor (NCHW fp32/fp16 contiguous) -> NHWC fp16 via our layout kernel."""
    if is_nhwc_half(x):
        return x
    if x.dim() != 4 or not _on_device(x) or x.dtype not in (torch.float32, torch.float16):
        raise ValueError("expected a CUDA NCHW fp32/fp16 tensor")
    x = x.contiguous()
    N, Cc, H, W = x.shape
    cpad = (Cc + 7) // 8 * 8
    buf = torch.empty((N, H, W, cpad), device=x.device, dtype=torch.float16)
    if cpad != Cc:
        buf.zero_()
    y = buf.permute(0, 3, 1, 2)[:, :Cc]
    check(_lib.lib().fsb_nchw_to_nhwc_f16(N, Cc, H, W, _ptr(x), int(x.dtype == torch.float32), _ptr(y), cpad, _stream()),
          "fsb_nchw_to_nhwc_f16")
    return y


def to_nchw(x: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    N, Cc, H, W, cs = nhwc_info(x)
    y = torch.empty((N, Cc, H, W), device=x.device, dtype=dtype)
    check(_lib.lib().fsb_nhwc_f16_to_nchw(N, Cc, H, W, _ptr(x), cs, _ptr(y), int(dtype == torch.float32), _stream()),
          "fsb_nhwc_f16_to_nchw")
    return y


# ----------------------------------------------------------------------------------------------
def conv_out_size(H, W, ksize, stride, pad, dil=1, off_h=0, off_w=0):
    ext = dil * (ksize - 1) + 1
    return (H - off_h + 2 * pad - ext) // stride + 1, (W - off_w + 2 * pad - ext) // stride + 1


def make_conv_desc(N, H, W, Cin, Cout, ksize, stride, pad, x_cstride, y_cstride, flags=0, dil=1, off_h=0, off_w=0) -> ConvDesc:
    Ho, Wo = conv_out_size(H, W, ksize, stride, pad, dil, off_h, off_w)
    return ConvDesc(N, H, W, Cin, Cout, ksize, stride, pad, dil, off_h, off_w, Ho, Wo, x_cstride, y_cstride, flags)


def pack_conv_weight(w: torch.Tensor, Cin: int, Cout: int, ksize: int, out=None) -> torch.Tensor:
    """fp32 OIHW master weight (possibly max-width; only [:Cout, :Cin] is read) -> packed fp16 buffer (`out`: re-pack in place)."""
    assert _on_device(w) and w.dtype == torch.float32 and w.dim() == 4 and w.shape[2] == ksize and w.shape[3] == ksize
    assert w.stride(3) == 1 and w.stride(2) == ksize
    d = ConvDesc(1, 8, 8, Cin, Cout, ksize, 1, 0, 1, 0, 0, 8, 8, Cin, Cout, 0)
    nbytes = _lib.lib().fsb_conv_packed_bytes(C.byref(d))
    if out is None:
        out = torch.empty(nbytes // 2, device=w.device, dtype=torch.float16)
    assert out.numel() * 2 == nbytes and out.dtype == torch.float16
    check(_lib.lib().fsb_pack_conv_weight(C.byref(d), _ptr(w), w.stride(0), w.stride(1), _ptr(out), _stream()),
          "fsb_pack_conv_weight")
    return out


def bn_fold(gamma, beta, mean, var, eps, conv_bias=None):
    Cc = mean.numel()
    out = torch.empty((2, Cc), device=mean.device, dtype=torch.float32)
    check(_lib.lib().fsb_bn_fold(Cc, _ptr(gamma), _ptr(beta), _ptr(mean), _ptr(var), float(eps), _ptr(conv_bias),
                                 _ptr(out[0]), _ptr(out[1]), _stream()), "fsb_bn_fold")
    return out[0], out[1]


def conv_stats_buffer(x, Cout, ksize, stride, pad, off=(0, 0), total_C=None, force_direct=False):
    """fp32 [rows, 2 * SC] buffer of partial statistic rows for `conv_fwd(..., stats=buf)` on this geometry (SC = total_C or
    Cout; include/fsb200.h "Deterministic statistics").  Needs no zeroing: the conv writes every row."""
    N, Cin, H, W, xcs = nhwc_info(x)
    Ho, Wo = conv_out_size(H, W, ksize, stride, pad, 1, off[0], off[1])
    SC = Cout if total_C is None else int(total_C)
    flags = FSB_CONV_STATS | FSB_CONV_OUT_F32 | (FSB_CONV_FORCE_DIRECT if force_direct else 0)
    d = ConvDesc(N, H, W, Cin, Cout, ksize, stride, pad, 1, off[0], off[1], Ho, Wo, xcs, (Cout + 7) // 8 * 8, flags)
    rows = _lib.lib().fsb_conv_stats_rows(C.byref(d))
    if rows <= 0:
        raise _lib.FsbError("fsb_conv_stats_rows: invalid geometry")
    return torch.empty((rows, 2 * SC), device=x.device, dtype=torch.float32)


def rowsum(rows):
    """[R, L] fp32 -> [1, L]: rows added in index order in double precision (the deterministic reduction)"""
    assert rows.dim() == 2 and rows.dtype == torch.float32 and rows.is_contiguous()
    out = torch.empty((1, rows.shape[1]), device=rows.device, dtype=torch.float32)
    check(_lib.lib().fsb_rowsum(rows.shape[1], _ptr(rows), rows.shape[0], rows.shape[1], _ptr(out), _stream()), "fsb_rowsum")
    return out


def conv_fwd(x, wpacked, Cout, ksize, stride, pad, scale=None, shift=None, relu=False, out=None, off=(0, 0),
             stats=None, force_direct=False, out_f32=False, stats_off=0, down2=False, up2=False, out_half=None):
    """y = act(conv(x) * scale + shift); x/out NHWC fp16 views (see module docstring).  out_f32: fp32 NHWC output (the
    training path's raw conv result, normalised by BatchNorm from un-rounded values).  stats: a `conv_stats_buffer`; this
    conv's per-channel sums land at column stats_off + c, its sums of squares at SC + stats_off + c of every row.
    down2: the conv runs on nearest(x, (H/2, W/2)), read in place from x (even H, W; stride 1).  up2: the result is
    nearest(y, (2Ho, 2Wo)), written in place (out is the 2Ho x 2Wo map).  Both are bit for bit the separate resize.
    out_half: an NHWC fp16 (N, Cout, Ho // 2, Wo // 2) view that also receives bilinear(y, (Ho // 2, Wo // 2)) -- from the conv's
    own epilogue where the library can (fsb_conv_fwd_half), else from a second launch; the same bits either way."""
    N, Cin, H, W, xcs = nhwc_info(x)
    if down2:
        if H % 2 or W % 2:
            raise ValueError("down2 needs an even input size, got %dx%d" % (H, W))
        H, W = H // 2, W // 2
    Ho, Wo = conv_out_size(H, W, ksize, stride, pad, 1, off[0], off[1])
    odt = torch.float32 if out_f32 else torch.float16
    up = 2 if up2 else 1
    if out is None:
        out = empty_nhwc(N, Cout, Ho * up, Wo * up, x.device, dtype=odt)
    No, Co, Hy, Wy, ycs = nhwc_info(out, odt)
    assert (No, Co, Hy, Wy) == (N, Cout, Ho * up, Wo * up), ((No, Co, Hy, Wy), (N, Cout, Ho * up, Wo * up))
    flags = (FSB_CONV_RELU if relu else 0) | (FSB_CONV_AFFINE if (scale is not None or shift is not None) else 0)
    flags |= (FSB_CONV_X_DOWN2 if down2 else 0) | (FSB_CONV_Y_UP2 if up2 else 0)
    if stats is not None:
        flags |= FSB_CONV_STATS
    if force_direct:
        flags |= FSB_CONV_FORCE_DIRECT
    if out_f32:
        flags |= FSB_CONV_OUT_F32
    d = ConvDesc(N, H, W, Cin, Cout, ksize, stride, pad, 1, off[0], off[1], Ho, Wo, xcs, ycs, flags)
    if out_half is not None:
        _, Ch, Hh, Wh, hcs = nhwc_info(out_half)
        assert (Ch, Hh, Wh) == (Cout, Ho // 2, Wo // 2) and not up2, ((Ch, Hh, Wh), (Cout, Ho // 2, Wo // 2))
        rc = _lib.lib().fsb_conv_fwd_half(C.byref(d), _ptr(x), _ptr(wpacked), _ptr(scale), _ptr(shift), _ptr(out), _ptr(out_half),
                                          hcs, _stream())
        if rc != _lib.FSB_ERR_UNSUPPORTED:
            check(rc, "fsb_conv_fwd_half")
            return out
    if stats is not None:
        assert stats.dim() == 2 and stats.dtype == torch.float32 and stats.is_contiguous()
        d.stats_C, d.stats_off = stats.shape[1] // 2, int(stats_off)
        rows = _lib.lib().fsb_conv_stats_rows(C.byref(d))
        assert rows == stats.shape[0], "statistics buffer has %d rows, this launch writes %d" % (stats.shape[0], rows)
    check(_lib.lib().fsb_conv_fwd(C.byref(d), _ptr(x), _ptr(wpacked), _ptr(scale), _ptr(shift), _ptr(out), _ptr(stats),
                                  _stream()), "fsb_conv_fwd")
    if out_half is not None:
        bilinear(out, (Ho // 2, Wo // 2), out=out_half)
    return out


def stem_conv_nchw(x, w, scale, shift, relu=True, out=None):
    """3x3 s2 p1 RGB stem on the caller's NCHW fp32/fp16 tensor."""
    assert x.dim() == 4 and x.shape[1] == 3 and _on_device(x) and x.is_contiguous()
    assert w.dtype == torch.float32 and w.is_contiguous() and tuple(w.shape[1:]) == (3, 3, 3)
    N, _, H, W = x.shape
    Cout = w.shape[0]
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    if out is None:
        out = empty_nhwc(N, Cout, Ho, Wo, x.device)
    _, _, _, _, ycs = nhwc_info(out)
    flags = (FSB_CONV_RELU if relu else 0) | (FSB_CONV_AFFINE if scale is not None else 0)
    check(_lib.lib().fsb_stem_conv_nchw(N, H, W, Cout, _ptr(x), int(x.dtype == torch.float32), _ptr(w), _ptr(scale),
                                        _ptr(shift), _ptr(out), ycs, flags, _stream()), "fsb_stem_conv_nchw")
    return out


def normalization_lut(mean, std, device):
    """3 x 256 fp16 table: the normalised value of every byte per channel, computed like the reference does
    (tools/utils/img_utils.py:179-185: float32 byte / 255.0, then float64 `- mean` and `/ std`, evaluator.py:329 casts the image
    to float32) and rounded to fp16 once -- what the stem kernel would make of the normalised fp32 frame."""
    import numpy as np
    v = np.arange(256, dtype=np.uint8).astype(np.float32) / 255.0                     # float32, like img.astype(np.float32) / 255.0
    table = (v[None, :] - np.asarray(mean, dtype=np.float64)[:, None]) / np.asarray(std, dtype=np.float64)[:, None]
    return torch.from_numpy(table.astype(np.float32)).to(torch.float16).contiguous().to(device)


def stem_conv_u8hwc(x_u8, lut, w, scale, shift, relu=True, out=None):
    """3x3 s2 p1 RGB stem on a uint8 HWC frame given as a logical (N, 3, H, W) view of an (N, H, W, 3) buffer, normalisation
    folded into the gather through `lut` (normalization_lut)."""
    assert x_u8.dtype == torch.uint8 and x_u8.dim() == 4 and x_u8.shape[1] == 3 and _on_device(x_u8)
    N, _, H, W = x_u8.shape
    assert x_u8.stride() == (H * W * 3, 1, W * 3, 3), "expected the permute(0, 3, 1, 2) view of a contiguous (N, H, W, 3) uint8 frame"
    assert lut.dtype == torch.float16 and lut.numel() == 768 and lut.is_contiguous()
    assert w.dtype == torch.float32 and w.is_contiguous() and tuple(w.shape[1:]) == (3, 3, 3)
    Cout = w.shape[0]
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    if out is None:
        out = empty_nhwc(N, Cout, Ho, Wo, x_u8.device)
    _, _, _, _, ycs = nhwc_info(out)
    flags = (FSB_CONV_RELU if relu else 0) | (FSB_CONV_AFFINE if scale is not None else 0)
    check(_lib.lib().fsb_stem_conv_u8hwc(N, H, W, Cout, _ptr(x_u8), _ptr(lut), _ptr(w), _ptr(scale), _ptr(shift), _ptr(out), ycs, flags,
                                         _stream()), "fsb_stem_conv_u8hwc")
    return out


def stem_fused(x, lut, w0, scale0, shift0, w1_packed, C1, scale1, shift1, out=None):
    """relu(BN(conv1(relu(BN(stem0(x)))))) in one kernel: the RGB stem (w0, fp32 OIHW [C0, 3, 3, 3]) and the 3x3 stride-2 conv1 of
    stem.1 (w1_packed: pack_conv_weight of its [C1, C0, 3, 3] weight), without the 1/2-resolution map.  x: NCHW fp32 / fp16, or the
    uint8 HWC view of stem_conv_u8hwc with its `lut`.  Returns `out` (NHWC fp16, 1/4 resolution), or None when the library has no
    fused kernel for these widths (FSB_ERR_UNSUPPORTED): the caller then runs stem_conv_* and conv_fwd."""
    assert x.dim() == 4 and x.shape[1] == 3 and _on_device(x)
    N, _, H, W = x.shape
    if x.dtype == torch.uint8:
        assert x.stride() == (H * W * 3, 1, W * 3, 3), "expected the permute(0, 3, 1, 2) view of a contiguous (N, H, W, 3) uint8 frame"
        assert lut is not None and lut.dtype == torch.float16 and lut.numel() == 768 and lut.is_contiguous()
        kind = 2
    else:
        assert x.dtype in (torch.float32, torch.float16) and x.is_contiguous()
        kind = 0 if x.dtype == torch.float32 else 1
    assert w0.dtype == torch.float32 and w0.is_contiguous() and tuple(w0.shape[1:]) == (3, 3, 3)
    C0 = w0.shape[0]
    H1, W1 = conv_out_size((H + 1) // 2, (W + 1) // 2, 3, 2, 1)
    if out is None:
        out = empty_nhwc(N, C1, H1, W1, x.device)
    _, _, _, _, ycs = nhwc_info(out)
    assert tuple(out.shape) == (N, C1, H1, W1), (tuple(out.shape), (N, C1, H1, W1))
    rc = _lib.lib().fsb_stem_fused(N, H, W, kind, _ptr(x), _ptr(lut if kind == 2 else None), C0, _ptr(w0), _ptr(scale0), _ptr(shift0),
                                   C1, _ptr(w1_packed), _ptr(scale1), _ptr(shift1), _ptr(out), ycs, _stream())
    if rc == _lib.FSB_ERR_UNSUPPORTED:
        return None
    check(rc, "fsb_stem_fused")
    return out


def confusion_matrix(pred_u8, gt, n_cl, out=None):
    """accumulate hist_info (tools/seg_opr/metric.py:7-15) of `pred_u8` vs `gt` into the int64 [n_cl^2 + 2] tensor `out`"""
    assert pred_u8.dtype == torch.uint8 and pred_u8.is_contiguous() and gt.is_contiguous() and pred_u8.numel() == gt.numel()
    assert gt.dtype in (torch.uint8, torch.int32, torch.int64)
    if out is None:
        out = torch.zeros(n_cl * n_cl + 2, device=pred_u8.device, dtype=torch.int64)
    check(_lib.lib().fsb_confusion_matrix(pred_u8.numel(), _ptr(pred_u8), _ptr(gt), gt.element_size(), int(n_cl), _ptr(out), _stream()),
          "fsb_confusion_matrix")
    return out


TRAIN_PRE_GEOM = 8   # int32 per image: H, W, mirror, sh, sw, pos_h, pos_w, pixel offset (fasterseg_b200/trainpre.py builds them)


def train_pre(img, gt, geom, lut, crop, label_size, out_img=None, out_gt=None):
    """TrainPre (train/dataloader.py:14-31) of a batch on the device, bit-identical to the reference: img / gt are the packed uint8
    HWC RGB sources and uint8 labels, geom the int32 [N, 8] geometry records (validated on the host by trainpre.check_geometry),
    lut the float32 [3, 256] normalisation table, crop = (image_height, image_width), label_size = the label map's (h, w).
    -> (float32 [N, 3, crop_h, crop_w], int64 [N, label_h, label_w])"""
    if geom.dtype != torch.int32 or geom.dim() != 2 or geom.shape[1] != TRAIN_PRE_GEOM or not geom.is_contiguous():
        raise ValueError("train_pre: geom must be a contiguous int32 [N, %d] tensor, got %s %s"
                         % (TRAIN_PRE_GEOM, geom.dtype, tuple(geom.shape)))
    for name, t in (("img", img), ("gt", gt)):
        if t.dtype != torch.uint8 or not t.is_contiguous():
            raise ValueError("train_pre: %s must be a contiguous uint8 tensor" % name)
    if lut.dtype != torch.float32 or lut.numel() != 3 * 256 or not lut.is_contiguous():
        raise ValueError("train_pre: lut must be a contiguous float32 [3, 256] tensor")
    N = geom.shape[0]
    ch, cw = int(crop[0]), int(crop[1])
    lh, lw = int(label_size[0]), int(label_size[1])
    if out_img is None:
        out_img = torch.empty(N, 3, ch, cw, dtype=torch.float32, device=img.device)
    if out_gt is None:
        out_gt = torch.empty(N, lh, lw, dtype=torch.int64, device=img.device)
    if out_img.dtype != torch.float32 or tuple(out_img.shape) != (N, 3, ch, cw) or not out_img.is_contiguous():
        raise ValueError("train_pre: out_img must be a contiguous float32 [%d, 3, %d, %d] tensor" % (N, ch, cw))
    if out_gt.dtype != torch.int64 or tuple(out_gt.shape) != (N, lh, lw) or not out_gt.is_contiguous():
        raise ValueError("train_pre: out_gt must be a contiguous int64 [%d, %d, %d] tensor" % (N, lh, lw))
    if not all(_on_device(t) for t in (img, gt, geom, lut, out_img, out_gt)):
        raise ValueError("train_pre: every tensor must be on the GPU")
    if len({t.device for t in (img, gt, geom, lut, out_img, out_gt)}) != 1:
        raise ValueError("train_pre: every tensor must be on the same device")
    desc = _lib.TrainPreDesc(N, ch, cw, lh, lw)
    check(_lib.lib().fsb_train_pre(C.byref(desc), _ptr(img), _ptr(gt), _ptr(geom), _ptr(lut), _ptr(out_img), _ptr(out_gt), _stream()),
          "fsb_train_pre")
    return out_img, out_gt


# ---- flat step tail (csrc/optim.cu): tables are built by optim.FlatTables ---------------------------------------------------------
def flat_chunk() -> int:
    """elements of one block of the flat kernels' block map"""
    return int(_lib.lib().fsb_flat_chunk())


def flat_grad_norm(block_map, nblocks, segs, live, G, partial, extra_sq, max_norm, out2):
    """out2[0] = 2-norm over the live segments of the flat gradient buffer G (+ extra_sq[0], gradients living elsewhere),
    out2[1] = min(1, max_norm / (norm + 1e-6)) -- nn.utils.clip_grad_norm_'s total norm and clip coefficient, on the device"""
    check(_lib.lib().fsb_flat_grad_norm(_ptr(block_map), int(nblocks), _ptr(segs), _ptr(live), _ptr(G), _ptr(partial), _ptr(extra_sq),
                                        float(max_norm), _ptr(out2), _stream()), "fsb_flat_grad_norm")


def flat_scale(block_map, nblocks, segs, live, G, coef):
    """G[live segments] *= coef[0]"""
    check(_lib.lib().fsb_flat_scale(_ptr(block_map), int(nblocks), _ptr(segs), _ptr(live), _ptr(G), _ptr(coef), _stream()), "fsb_flat_scale")


def flat_sgd(block_map, nblocks, segs, live, G, M, lr, momentum, weight_decay):
    """torch.optim.SGD arithmetic over the live segments: d = g + wd * p; m = momentum * m + d; p -= lr * m (p through the segment
    table's storage pointers, g / m in the flat buffers)"""
    check(_lib.lib().fsb_flat_sgd(_ptr(block_map), int(nblocks), _ptr(segs), _ptr(live), _ptr(G), _ptr(M), float(lr), float(momentum),
                                  float(weight_decay), _stream()), "fsb_flat_sgd")


def _f32_ptrs(ts, what):
    for t in ts:
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or not _on_device(t)):
            raise ValueError("%s: expected contiguous CUDA float32 tensors, got %s %s" % (what, t.dtype, tuple(t.shape)))
    return [_ptr(t) for t in ts]


def supernet_latency_workspace_bytes(plan_host: torch.Tensor) -> int:
    """bytes of the caller-owned workspace that fsb_supernet_latency_fwd fills and _bwd reads (host math on the plan header)"""
    assert plan_host.dtype == torch.int32 and not plan_host.is_cuda
    n = int(_lib.lib().fsb_supernet_latency_workspace_bytes(_ptr(plan_host)))
    if n == 0:
        raise _lib.FsbError("fsb_supernet_latency_workspace_bytes: invalid plan")
    return n


def supernet_latency_fwd(plan_host, plan, params, noise, workspace, out):
    """out[()] = expected latency of the supernet (K14).  params: the 8 arch logit tensors (alphas x3, betas x2, ratios x3), None where
    the plan does not read them; noise: gumbel uniforms or forced width indices on the device; workspace: saved for the backward"""
    assert len(params) == 8 and plan.dtype == torch.int32 and _on_device(plan)
    ptrs = _f32_ptrs(list(params) + [noise, workspace, out], "fsb_supernet_latency_fwd")
    check(_lib.lib().fsb_supernet_latency_fwd(_ptr(plan_host), _ptr(plan), *ptrs, _stream()), "fsb_supernet_latency_fwd")
    return out


def supernet_latency_bwd(plan_host, plan, gout, workspace, grads):
    """grads: 8 tensors shaped like the arch logits (None where the plan does not differentiate), overwritten with d latency * gout"""
    assert len(grads) == 8 and plan.dtype == torch.int32 and _on_device(plan)
    ptrs = _f32_ptrs([gout, workspace] + list(grads), "fsb_supernet_latency_bwd")
    check(_lib.lib().fsb_supernet_latency_bwd(_ptr(plan_host), _ptr(plan), *ptrs, _stream()), "fsb_supernet_latency_bwd")
    return grads


def bilinear(x, size, relu=False, out=None, out_half=None):
    """F.interpolate(x, size, mode='bilinear', align_corners=True) (then ReLU if relu).  out_half: an NHWC fp16
    (N, C, Ho // 2, Wo // 2) view that also receives bilinear(y, (Ho // 2, Wo // 2)) -- for an exact x2 upsample from the same
    launch (fsb_bilinear_fwd_half), else from a second one; the same bits either way."""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    if out is None:
        out = empty_nhwc(N, Cc, Ho, Wo, x.device)
    _, Co, Hy, Wy, ycs = nhwc_info(out)
    assert (Co, Hy, Wy) == (Cc, Ho, Wo)
    flags = FSB_CONV_RELU if relu else 0
    if out_half is not None:
        _, Ch, Hh, Wh, hcs = nhwc_info(out_half)
        assert (Ch, Hh, Wh) == (Cc, Ho // 2, Wo // 2), ((Ch, Hh, Wh), (Cc, Ho // 2, Wo // 2))
        if (Ho, Wo) == (2 * Hi, 2 * Wi):
            rc = _lib.lib().fsb_bilinear_fwd_half(N, Cc, Hi, Wi, _ptr(x), xcs, _ptr(out), ycs, _ptr(out_half), hcs, flags, _stream())
            if rc != _lib.FSB_ERR_UNSUPPORTED:
                check(rc, "fsb_bilinear_fwd_half")
                return out
    check(_lib.lib().fsb_bilinear_fwd(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(out), ycs, flags, _stream()), "fsb_bilinear_fwd")
    if out_half is not None:
        bilinear(out, (Ho // 2, Wo // 2), out=out_half)
    return out


def upsample_logits(x, size, dtype=torch.float32, out=None):
    """NHWC fp16 logits -> NCHW (contiguous) logits at `size`, bilinear align_corners=True."""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    if out is None:
        out = torch.empty((N, Cc, Ho, Wo), device=x.device, dtype=dtype)
    assert out.is_contiguous() and out.dtype in (torch.float16, torch.float32)
    check(_lib.lib().fsb_upsample_logits_nchw(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(out),
                                              int(out.dtype == torch.float32), _stream()), "fsb_upsample_logits_nchw")
    return out


def upsample_argmax(x, size, out=None):
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    if out is None:
        out = torch.empty((N, Ho, Wo), device=x.device, dtype=torch.uint8)
    check(_lib.lib().fsb_upsample_argmax(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(out), _stream()), "fsb_upsample_argmax")
    return out


def upsample_argmax_confusion(x, size, gt, n_cl, out):
    """confusion_matrix(upsample_argmax(x, size), gt, n_cl, out) in one launch that never writes the label map: x holds the n_cl
    class logits (NHWC fp16 view), gt the N x Ho x Wo ground truth (uint8 / int32 / int64, values outside [0, n_cl) ignored), out the
    int64 [n_cl^2 + 2] counters, accumulated into.  The counters are bit-identical to the two-kernel path."""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    n_cl = int(n_cl)
    if Cc != n_cl:
        raise ValueError("upsample_argmax_confusion: logits have %d classes, n_cl is %d" % (Cc, n_cl))
    if gt.dtype not in (torch.uint8, torch.int32, torch.int64) or not gt.is_contiguous() or gt.numel() != N * Ho * Wo or not _on_device(gt):
        raise ValueError("upsample_argmax_confusion: gt must be a contiguous CUDA uint8 / int32 / int64 tensor of %d x %d x %d elements, "
                         "got %s %s" % (N, Ho, Wo, gt.dtype, tuple(gt.shape)))
    if out.dtype != torch.int64 or not out.is_contiguous() or out.numel() != n_cl * n_cl + 2 or not _on_device(out):
        raise ValueError("upsample_argmax_confusion: out must be a contiguous CUDA int64 tensor of n_cl^2 + 2 elements")
    check(_lib.lib().fsb_upsample_argmax_confusion(N, n_cl, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(gt), gt.element_size(), _ptr(out),
                                                   _stream()), "fsb_upsample_argmax_confusion")
    return out


def upsample_argmax_map(x, size, lut=None, palette=None, image=None, ids_out=None, viz_out=None):
    """The test-set writer's two images (train/test.py:49-69) from the 1/8 logits in one launch, with label = upsample_argmax(x, size):
      ids = lut[label]                   uint8 N x Ho x Wo; written when `lut` or `ids_out` is given, or when there is no palette
      viz = palette[label] rule          uint8 N x Ho x Wo x 3, BGR; written when `palette` is given
    lut: uint8 [C] (None = identity).  palette: uint8 [C, 4] rows (B, G, R, use_image); where use_image is set the pixel is
    `image`'s (uint8 N x Ho x Wo x 3, RGB) reversed to BGR, as set_img_color + `[:, :, ::-1]` (tools/utils/visualize.py:6-21) leave
    it.  -> (ids, viz), None for an output not asked for.  Without `image` the palette's use_image column is read on the host."""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    if not 1 <= Cc <= 255:
        raise ValueError("upsample_argmax_map: 1 <= C <= 255 classes, got %d" % Cc)

    def u8(t, shape, name):
        if t.dtype != torch.uint8 or tuple(t.shape) != shape or not t.is_contiguous() or not _on_device(t) or t.device != x.device:
            raise ValueError("upsample_argmax_map: %s must be a contiguous uint8 tensor of shape %s on %s, got %s %s on %s"
                             % (name, shape, x.device, t.dtype, tuple(t.shape), t.device))
        return t

    if lut is not None:
        u8(lut, (Cc,), "lut")
    if palette is not None:
        u8(palette, (Cc, 4), "palette")
    elif viz_out is not None or image is not None:
        raise ValueError("upsample_argmax_map: viz_out / image need a palette")
    if image is not None:
        u8(image, (N, Ho, Wo, 3), "image")
    elif palette is not None and bool(palette[:, 3].any()):
        raise ValueError("upsample_argmax_map: the palette takes image pixels (use_image set) but no image was given")
    ids = viz = None
    if ids_out is not None or lut is not None or palette is None:
        ids = torch.empty((N, Ho, Wo), device=x.device, dtype=torch.uint8) if ids_out is None else u8(ids_out, (N, Ho, Wo), "ids_out")
    if palette is not None:
        viz = torch.empty((N, Ho, Wo, 3), device=x.device, dtype=torch.uint8) if viz_out is None else u8(viz_out, (N, Ho, Wo, 3), "viz_out")
    check(_lib.lib().fsb_upsample_argmax_map(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(lut), _ptr(ids), _ptr(palette), _ptr(image),
                                             _ptr(viz), _stream()), "fsb_upsample_argmax_map")
    return ids, viz


def nearest(x, size, out=None):
    """F.interpolate(x, size, mode='nearest') on NHWC fp16 views (torch's legacy index rule; a copy, so bit-exact)"""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    if out is None:
        out = empty_nhwc(N, Cc, Ho, Wo, x.device)
    _, Co, Hy, Wy, ycs = nhwc_info(out)
    assert (Co, Hy, Wy) == (Cc, Ho, Wo)
    check(_lib.lib().fsb_nearest_fwd(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(out), ycs, _stream()), "fsb_nearest_fwd")
    return out


def upsample_logits_nearest(x, size, dtype=torch.float32, out=None):
    """NHWC fp16 logits -> NCHW (contiguous) logits at `size`, mode='nearest'."""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    if out is None:
        out = torch.empty((N, Cc, Ho, Wo), device=x.device, dtype=dtype)
    assert out.is_contiguous() and out.dtype in (torch.float16, torch.float32) and tuple(out.shape) == (N, Cc, Ho, Wo)
    check(_lib.lib().fsb_upsample_logits_nearest_nchw(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(out),
                                                      int(out.dtype == torch.float32), _stream()),
          "fsb_upsample_logits_nearest_nchw")
    return out


def upsample_argmax_nearest(x, size, out=None):
    """uint8 argmax over classes of upsample_logits_nearest(x, size), without materialising the logits"""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    if out is None:
        out = torch.empty((N, Ho, Wo), device=x.device, dtype=torch.uint8)
    assert out.is_contiguous() and out.dtype == torch.uint8 and tuple(out.shape) == (N, Ho, Wo)
    check(_lib.lib().fsb_upsample_argmax_nearest(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(out), _stream()),
          "fsb_upsample_argmax_nearest")
    return out


def copy_channels(x, out):
    N, Cc, H, W, xcs = nhwc_info(x)
    No, Co, Ho, Wo, ycs = nhwc_info(out)
    assert (N, Cc, H, W) == (No, Co, Ho, Wo)
    check(_lib.lib().fsb_copy_channels(N * H * W, Cc, _ptr(x), xcs, _ptr(out), ycs, _stream()), "fsb_copy_channels")
    return out


def bn_stats(x):
    """-> fp32 [2C] = per-channel (sum | sum of squares); deterministic (partial rows + ordered row sum)"""
    N, Cc, H, W, xcs = nhwc_info(x)
    rows = _lib.lib().fsb_stat_rows(N * H * W)
    buf = torch.empty((1 + rows, 2 * Cc), device=x.device, dtype=torch.float32)
    check(_lib.lib().fsb_bn_stats(N * H * W, Cc, _ptr(x), xcs, _ptr(buf), _stream()), "fsb_bn_stats")
    return buf[0]


def bn_finalize(stats, count, gamma, beta, eps, momentum, running_mean, running_var, want_save=False):
    """stats: [rows, 2C] partial rows (conv_stats_buffer / rowsum output) or [2C] totals"""
    if stats.dim() == 1:
        stats = stats.view(1, -1)
    Cc = stats.shape[1] // 2
    buf = torch.empty((4, Cc), device=stats.device, dtype=torch.float32)
    check(_lib.lib().fsb_bn_finalize(Cc, _ptr(stats), stats.shape[0], Cc, float(count), _ptr(gamma), _ptr(beta), float(eps), float(momentum),
                                     _ptr(running_mean), _ptr(running_var), _ptr(buf[0]), _ptr(buf[1]),
                                     _ptr(buf[2]) if want_save else None, _ptr(buf[3]) if want_save else None, _stream()),
          "fsb_bn_finalize")
    return buf[0], buf[1], buf[2], buf[3]


def affine_act(x, scale, shift, relu=False, out=None):
    N, Cc, H, W, xcs = nhwc_info(x, x.dtype)
    if out is None:
        out = empty_nhwc(N, Cc, H, W, x.device)
    _, _, _, _, ycs = nhwc_info(out)
    flags = (FSB_CONV_RELU if relu else 0) | (FSB_ACT_IN_F32 if x.dtype == torch.float32 else 0)
    check(_lib.lib().fsb_affine_act(N * H * W, Cc, _ptr(x), xcs, _ptr(scale), _ptr(shift), _ptr(out), ycs, flags, _stream()),
          "fsb_affine_act")
    return out


# ----------------------------------------------------------------------------------------------
# backward / training wrappers (kernels in csrc/train.cu)
# ----------------------------------------------------------------------------------------------
def bn_bwd_sums(dy, y, raw, mean, invstd, relu):
    """First pass of the BatchNorm(+ReLU) backward: fp32 [2C] = per-channel (sum dz | sum dz * xhat), dz = dy masked by y > 0."""
    N, Cc, H, W, dcs = nhwc_info(dy)
    _, _, _, _, rcs = nhwc_info(raw, raw.dtype)
    rf32 = int(raw.dtype == torch.float32)
    ycs = nhwc_info(y)[4] if relu else 0
    rows = _lib.lib().fsb_stat_rows(N * H * W)
    sums = torch.empty((1 + rows, 2 * Cc), device=dy.device, dtype=torch.float32)   # row 0 = totals, rows 1.. = per-CTA partials
    check(_lib.lib().fsb_bn_bwd_reduce(N * H * W, Cc, _ptr(dy), dcs, _ptr(y) if relu else None, ycs, _ptr(raw), rcs, rf32, _ptr(mean),
                                       _ptr(invstd), int(relu), _ptr(sums), _stream()), "fsb_bn_bwd_reduce")
    return sums[0]


def bn_bwd_apply(dy, y, raw, mean, invstd, gamma, sums, count, relu, gscale, want_param_grads=True):
    """Second pass: draw = gamma * invstd * (dz - sums[:C] / count - xhat * sums[C:] / count) as fp16 NHWC, and (when asked)
    dgamma = sums[C:] / gscale, dbeta = sums[:C] / gscale written by the same kernel."""
    N, Cc, H, W, dcs = nhwc_info(dy)
    _, _, _, _, rcs = nhwc_info(raw, raw.dtype)
    rf32 = int(raw.dtype == torch.float32)
    ycs = nhwc_info(y)[4] if relu else 0
    draw = empty_nhwc(N, Cc, H, W, dy.device)
    dg = torch.empty(Cc, device=dy.device, dtype=torch.float32) if want_param_grads else None
    db = torch.empty(Cc, device=dy.device, dtype=torch.float32) if want_param_grads else None
    check(_lib.lib().fsb_bn_bwd_apply(N * H * W, Cc, _ptr(dy), dcs, _ptr(y) if relu else None, ycs, _ptr(raw), rcs, rf32, _ptr(mean),
                                      _ptr(invstd), _ptr(gamma), _ptr(sums), float(count), int(relu), _ptr(draw),
                                      nhwc_info(draw)[4], _ptr(dg), _ptr(db), float(gscale), 0, _stream()), "fsb_bn_bwd_apply")
    return draw, dg, db


def bn_bwd(dy, y, raw, mean, invstd, gamma, count, relu, gscale, want_param_grads=True, allreduce=None):
    """BatchNorm(+ReLU) backward -> (draw, dgamma, dbeta).  `allreduce(sums)` hook = SyncBN backward, `count` then being the
    GLOBAL number of pixels per channel."""
    Cc = dy.shape[1]
    sums = bn_bwd_sums(dy, y, raw, mean, invstd, relu)
    if allreduce is None:
        return bn_bwd_apply(dy, y, raw, mean, invstd, gamma, sums, count, relu, gscale, want_param_grads)
    # SyncBN: dx needs the GLOBAL sums, but gamma/beta gradients must stay LOCAL sums -- the data-parallel gradient average
    # (parallel.GradSync) divides every parameter gradient by the world size afterwards, like DDP + torch SyncBatchNorm
    dg = db = None
    if want_param_grads:
        db = sums[:Cc] / gscale
        dg = sums[Cc:] / gscale
    sums = allreduce(sums.clone() if want_param_grads else sums)
    draw, _, _ = bn_bwd_apply(dy, y, raw, mean, invstd, gamma, sums, count, relu, gscale, want_param_grads=False)
    return draw, dg, db


def relu_bwd(dy, y):
    N, Cc, H, W, dcs = nhwc_info(dy)
    ycs = nhwc_info(y)[4]
    dx = empty_nhwc(N, Cc, H, W, dy.device)
    check(_lib.lib().fsb_relu_bwd(N * H * W, Cc, _ptr(dy), dcs, _ptr(y), ycs, _ptr(dx), nhwc_info(dx)[4], _stream()), "fsb_relu_bwd")
    return dx


def pack_conv_weight_dgrad(w, Cin, Cout, ksize, out=None):
    d = ConvDesc(1, 8, 8, Cin, Cout, ksize, 1, (ksize - 1) // 2, 1, 0, 0, 8, 8, Cin, Cout, 0)
    nbytes = _lib.lib().fsb_conv_packed_dgrad_bytes(C.byref(d))
    if out is None:
        out = torch.empty(nbytes // 2, device=w.device, dtype=torch.float16)
    assert out.numel() * 2 == nbytes and out.dtype == torch.float16
    check(_lib.lib().fsb_pack_conv_weight_dgrad(C.byref(d), _ptr(w), w.stride(0), w.stride(1), _ptr(out), _stream()),
          "fsb_pack_conv_weight_dgrad")
    return out


def conv_dgrad(dy, w, x_shape, Cin, Cout, ksize, stride, pad, off=(0, 0), wpacked_t=None, force_direct=False):
    """dx of conv(x, w[:Cout, :Cin]); x_shape = (N, Cin, H, W) of the forward input."""
    N, _, H, W = x_shape
    Nd, Cd, Ho, Wo, dcs = nhwc_info(dy)
    assert Cd == Cout and Nd == N
    dx = empty_nhwc(N, Cin, H, W, dy.device)
    flags = FSB_CONV_FORCE_DIRECT if force_direct else 0
    d = ConvDesc(N, H, W, Cin, Cout, ksize, stride, pad, 1, off[0], off[1], Ho, Wo, Cin, Cout, flags)
    check(_lib.lib().fsb_conv_dgrad(C.byref(d), _ptr(dy), dcs, _ptr(wpacked_t), _ptr(w), w.stride(0), w.stride(1), _ptr(dx),
                                    nhwc_info(dx)[4], _stream()), "fsb_conv_dgrad")
    return dx


def conv_wgrad(x, dy, w_like, Cin, Cout, ksize, stride, pad, gscale, off=(0, 0), accumulate_into=None, force_direct=False):
    """fp32 gradient with the shape/strides of the master weight `w_like` (zero outside the active corner).
    accumulate_into: an existing fp32 gradient tensor (e.g. param.grad) to add into instead of allocating -- for max-width
    slimmable weights this avoids writing a full-size zero tensor per invocation (4 GB per supernet step otherwise)."""
    N, Cx, H, W, xcs = nhwc_info(x)
    _, Cd, Ho, Wo, dcs = nhwc_info(dy)
    assert Cx == Cin and Cd == Cout
    d = ConvDesc(N, H, W, Cin, Cout, ksize, stride, pad, 1, off[0], off[1], Ho, Wo, xcs, Cout,
                 FSB_CONV_FORCE_DIRECT if force_direct else 0)
    if accumulate_into is not None:
        dw = accumulate_into
        assert dw.dtype == torch.float32 and dw.shape == w_like.shape and dw.stride(3) == 1 and dw.stride(2) == ksize
        check(_lib.lib().fsb_conv_wgrad(C.byref(d), _ptr(x), _ptr(dy), dcs, _ptr(dw), dw.stride(0), dw.stride(1), 1, float(gscale),
                                        _stream()), "fsb_conv_wgrad")
        return dw
    full = (w_like.shape[0] == Cout and w_like.shape[1] == Cin)
    dw = torch.empty_like(w_like, dtype=torch.float32, memory_format=torch.contiguous_format) if full else \
        torch.zeros_like(w_like, dtype=torch.float32, memory_format=torch.contiguous_format)
    check(_lib.lib().fsb_conv_wgrad(C.byref(d), _ptr(x), _ptr(dy), dcs, _ptr(dw), dw.stride(0), dw.stride(1), 0, float(gscale),
                                    _stream()), "fsb_conv_wgrad")
    return dw


def bilinear_bwd(dy, in_hw, relu_mask_y=None):
    N, Cc, Ho, Wo, dcs = nhwc_info(dy)
    Hi, Wi = in_hw
    dx = empty_nhwc(N, Cc, Hi, Wi, dy.device)
    ycs = nhwc_info(relu_mask_y)[4] if relu_mask_y is not None else 0
    check(_lib.lib().fsb_bilinear_bwd(N, Cc, Hi, Wi, Ho, Wo, _ptr(dy), dcs, _ptr(relu_mask_y), ycs, _ptr(dx), nhwc_info(dx)[4],
                                      _stream()), "fsb_bilinear_bwd")
    return dx


def upsample_logits_bwd(dy_nchw, in_hw, gscale):
    dy_nchw = dy_nchw.contiguous()
    N, Cc, Ho, Wo = dy_nchw.shape
    Hi, Wi = in_hw
    dx = empty_nhwc(N, Cc, Hi, Wi, dy_nchw.device)
    check(_lib.lib().fsb_upsample_logits_bwd(N, Cc, Hi, Wi, Ho, Wo, _ptr(dy_nchw), int(dy_nchw.dtype == torch.float32), _ptr(dx),
                                             nhwc_info(dx)[4], float(gscale), _stream()), "fsb_upsample_logits_bwd")
    return dx


def nchw_grad_to_nhwc(dy_nchw, gscale):
    dy_nchw = dy_nchw.contiguous()
    N, Cc, H, W = dy_nchw.shape
    dx = empty_nhwc(N, Cc, H, W, dy_nchw.device)
    check(_lib.lib().fsb_nchw_grad_to_nhwc(N, Cc, H, W, _ptr(dy_nchw), int(dy_nchw.dtype == torch.float32), _ptr(dx),
                                           nhwc_info(dx)[4], float(gscale), _stream()), "fsb_nchw_grad_to_nhwc")
    return dx


def _ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])
    return arr


def wsum_fwd(xs, wts, out=None):
    N, Cc, H, W, _ = nhwc_info(xs[0])
    if out is None:
        out = empty_nhwc(N, Cc, H, W, xs[0].device)
    strides = (C.c_int * len(xs))(*[nhwc_info(t)[4] for t in xs])
    check(_lib.lib().fsb_wsum_fwd(len(xs), N * H * W, Cc, _ptr_array(xs), strides, _ptr(wts), _ptr(out), nhwc_info(out)[4],
                                  _stream()), "fsb_wsum_fwd")
    return out


def wsum_bwd(dout, xs, wts, need_dx, need_dw, gscale):
    N, Cc, H, W, docs = nhwc_info(dout)
    K = len(xs)
    dxs = [empty_nhwc(N, Cc, H, W, dout.device) if need_dx[k] else None for k in range(K)]
    dw = None
    if need_dw:   # (1 + rows) x 8: row 0 = totals (ordered row sum of the per-CTA partials below it); needs no zeroing
        dw = torch.empty((1 + _lib.lib().fsb_wsum_rows(N * H * W, Cc), 8), device=dout.device, dtype=torch.float32)
    xstr = (C.c_int * K)(*[nhwc_info(t)[4] for t in xs])
    dxstr = (C.c_int * K)(*[0 if t is None else nhwc_info(t)[4] for t in dxs])
    check(_lib.lib().fsb_wsum_bwd(K, N * H * W, Cc, _ptr(dout), docs, _ptr_array(xs), xstr, _ptr(wts), _ptr_array(dxs), dxstr,
                                  _ptr(dw), float(gscale), _stream()), "fsb_wsum_bwd")
    return dxs, (dw[0, :K] if need_dw else None)


def add_inplace(x, y):
    N, Cc, H, W, xcs = nhwc_info(x)
    check(_lib.lib().fsb_add_inplace(N * H * W, Cc, _ptr(x), xcs, _ptr(y), nhwc_info(y)[4], _stream()), "fsb_add_inplace")
    return y


# ----------------------------------------------------------------------------------------------
# fused training unit (one C-ABI call per direction; see csrc/train_fused.cu)
# ----------------------------------------------------------------------------------------------
def conv_bn_act_train_fwd(x, wpacked, Cout, ksize, stride, pad, off, gamma, beta, eps, momentum, running_mean, running_var,
                          num_batches_tracked, relu, sel=None, width_idx=None):
    """-> (y fp16 NHWC, raw fp32 NHWC, vec fp32[(6 + 2R)*Cout] = [sum|sumsq|scale|shift|mean|invstd|R partial rows], desc).
    sel / width_idx: device pointers (ints) of an fsb_bn_sel table and an int32 width index -- the BatchNorm parameter set is
    then chosen on the device (captured training graphs) and gamma / beta / running stats arguments are ignored."""
    N, Cin, H, W, xcs = nhwc_info(x)
    Ho, Wo = conv_out_size(H, W, ksize, stride, pad, 1, off[0], off[1])
    cpad = (Cout + 7) // 8 * 8
    dev = x.device
    raw = empty_nhwc(N, Cout, Ho, Wo, dev, torch.float32)    # views at offset 0 of their buffers, pixel stride cpad
    y = empty_nhwc(N, Cout, Ho, Wo, dev)
    d = ConvDesc(N, H, W, Cin, Cout, ksize, stride, pad, 1, off[0], off[1], Ho, Wo, xcs, cpad, FSB_CONV_OUT_F32 | FSB_CONV_STATS)
    rows = _lib.lib().fsb_conv_stats_rows(C.byref(d))
    d.flags = 0
    vec = torch.empty((6 + 2 * rows) * Cout, device=dev, dtype=torch.float32)
    check(_lib.lib().fsb_conv_bn_act_train_fwd(C.byref(d), x.data_ptr(), wpacked.data_ptr(),
                                               None if gamma is None else gamma.data_ptr(), None if beta is None else beta.data_ptr(),
                                               float(eps), float(momentum),
                                               None if running_mean is None else running_mean.data_ptr(),
                                               None if running_var is None else running_var.data_ptr(),
                                               None if num_batches_tracked is None else num_batches_tracked.data_ptr(),
                                               raw.data_ptr(), cpad, y.data_ptr(), cpad, vec.data_ptr(), int(relu), sel, width_idx,
                                               _stream()),
          "fsb_conv_bn_act_train_fwd")
    return y, raw, vec, d


def conv_bn_act_train_bwd(d, x, dy, y, raw, vec, gamma, relu, wpacked_t, w, need_dx, dw_accum, gscale, sel=None, width_idx=None):
    """-> (dx or None, dgamma, dbeta); the weight gradient is accumulated into `dw_accum` (fp32, master layout) when given.
    With sel / width_idx (see conv_bn_act_train_fwd) dgamma / dbeta are accumulated into the selected parameter set's gradient
    slots by the kernel and the returned tensors are meaningless."""
    N, Cout, Ho, Wo, dcs = nhwc_info(dy)
    dev = dy.device
    cpad = d.y_cstride
    draw = empty_nhwc(N, Cout, Ho, Wo, dev)
    assert draw.stride(3) == cpad
    rows = _lib.lib().fsb_stat_rows(N * Ho * Wo)
    vb = torch.empty((4 + 2 * rows) * Cout, device=dev, dtype=torch.float32)   # [totals 2C | partial rows | dgamma | dbeta]
    dx = None
    xcs = 0
    if need_dx:
        dx = empty_nhwc(N, d.Cin, d.H, d.W, dev)
        xcs = dx.stride(3)
    check(_lib.lib().fsb_conv_bn_act_train_bwd(C.byref(d), x.data_ptr(), dy.data_ptr(), dcs, y.data_ptr(), y.stride(3), raw.data_ptr(),
                                               raw.stride(3), vec.data_ptr(), None if gamma is None else gamma.data_ptr(), int(relu),
                                               None if wpacked_t is None else wpacked_t.data_ptr(), w.data_ptr(), w.stride(0),
                                               w.stride(1), draw.data_ptr(), cpad, vb.data_ptr(),
                                               None if dx is None else dx.data_ptr(), xcs,
                                               None if dw_accum is None else dw_accum.data_ptr(), float(gscale), sel, width_idx,
                                               _stream()),
          "fsb_conv_bn_act_train_bwd")
    at = (2 + 2 * rows) * Cout
    return dx, vb[at:at + Cout], vb[at + Cout:at + 2 * Cout]


# ----------------------------------------------------------------------------------------------
# device-selected BatchNorm sets (captured training graphs, fasterseg_b200/graphed.py).  `sel` is an engine.SelBN: `.table_ptr`
# = device address of its fsb_bn_sel table (one entry per width), `.idx_ptr` = device address of the int32 width index of the
# current pass.  Units run at their maximum width; the kernels zero the inactive tail (include/fsb200.h).
# ----------------------------------------------------------------------------------------------
def conv_bn_act_train_fwd_sel(x, wpacked, Cout, ksize, stride, pad, off, sel, relu):
    return conv_bn_act_train_fwd(x, wpacked, Cout, ksize, stride, pad, off, None, None, sel.eps, sel.momentum, None, None, None, relu,
                                 sel=sel.table_ptr, width_idx=sel.idx_ptr)


def conv_bn_act_train_bwd_sel(d, x, dy, y, raw, vec, sel, relu, wpacked_t, w, need_dx, dw_accum, gscale):
    dx, _, _ = conv_bn_act_train_bwd(d, x, dy, y, raw, vec, None, relu, wpacked_t, w, need_dx, dw_accum, gscale,
                                     sel=sel.table_ptr, width_idx=sel.idx_ptr)
    return dx


def bn_finalize_sel(stats, count, sel, hmax=0):
    """-> (scale, shift, mean, invstd) fp32 [C]; C = stats columns / 2 (the unit's maximum width)"""
    Cc = stats.shape[1] // 2
    buf = torch.empty((4, Cc), device=stats.device, dtype=torch.float32)
    check(_lib.lib().fsb_bn_finalize_sel(Cc, _ptr(stats), stats.shape[0], Cc, float(count), float(sel.eps), float(sel.momentum),
                                         _ptr(buf[0]), _ptr(buf[1]), _ptr(buf[2]), _ptr(buf[3]), sel.table_ptr, sel.idx_ptr, int(hmax),
                                         _stream()), "fsb_bn_finalize_sel")
    return buf[0], buf[1], buf[2], buf[3]


def affine_act_sel(x, scale, shift, sel, hmax, relu=False):
    N, Cc, H, W, xcs = nhwc_info(x, x.dtype)
    out = empty_nhwc(N, Cc, H, W, x.device)
    flags = (FSB_CONV_RELU if relu else 0) | (FSB_ACT_IN_F32 if x.dtype == torch.float32 else 0)
    check(_lib.lib().fsb_affine_act_sel(N * H * W, Cc, _ptr(x), xcs, _ptr(scale), _ptr(shift), _ptr(out), nhwc_info(out)[4], flags,
                                        sel.table_ptr, sel.idx_ptr, int(hmax), _stream()), "fsb_affine_act_sel")
    return out


def dp_allreduce(t):
    """in-place sum over the data-parallel ranks through the library's own exchange (peer memory for small vectors, NCCL
    otherwise; csrc/peer.cu, csrc/dp.cu) on the current stream -- capturable, no host synchronisation"""
    assert t.dtype == torch.float32 and t.is_contiguous()
    check(_lib.lib().fsb_dp_allreduce_f32(_ptr(t), t.numel(), _stream()), "fsb_dp_allreduce_f32")
    return t


def bn_bwd_sel(dy, y, raw, mean, invstd, count, relu, gscale, sel, hmax=0, world=1):
    """BatchNorm(+ReLU) backward of a device-selected set -> draw (raw channel order when hmax > 0); gamma / beta gradients are
    accumulated into the selected set's gradient slots by the kernel.  world > 1 (SyncBN): the sums are exchanged between the
    two kernels, `count` is the global pixel count, and the parameter gradients come from the rank-local sums."""
    N, Cc, H, W, dcs = nhwc_info(dy)
    _, _, _, _, rcs = nhwc_info(raw, raw.dtype)
    rf32 = int(raw.dtype == torch.float32)
    ycs = nhwc_info(y)[4] if relu else 0
    rows = _lib.lib().fsb_stat_rows(N * H * W)
    sums = torch.empty((1 + rows, 2 * Cc), device=dy.device, dtype=torch.float32)
    check(_lib.lib().fsb_bn_bwd_reduce_sel(N * H * W, Cc, _ptr(dy), dcs, _ptr(y) if relu else None, ycs, _ptr(raw), rcs, rf32, _ptr(mean),
                                           _ptr(invstd), int(relu), _ptr(sums), sel.table_ptr, sel.idx_ptr, int(hmax), _stream()),
          "fsb_bn_bwd_reduce_sel")
    local = None
    if world > 1:
        local = sums[0].clone()
        dp_allreduce(sums[0])
    draw = empty_nhwc(N, Cc, H, W, dy.device)
    check(_lib.lib().fsb_bn_bwd_apply_sel(N * H * W, Cc, _ptr(dy), dcs, _ptr(y) if relu else None, ycs, _ptr(raw), rcs, rf32, _ptr(mean),
                                          _ptr(invstd), _ptr(sums), _ptr(local), float(count), int(relu), _ptr(draw), nhwc_info(draw)[4],
                                          float(gscale), sel.table_ptr, sel.idx_ptr, int(hmax), _stream()), "fsb_bn_bwd_apply_sel")
    return draw


# ---- N1: criteria evaluated from the low-resolution logits (csrc/loss.cu) ---------------------------------------------------------------
def loss_logp_fwd(x, target, size, ignore_label):
    """x: NHWC fp16 logits (N, C, Hi, Wi); target int64 (N, Ho, Wo) -> (logp_t, lse), both fp32 (N, Ho, Wo): log-probability of the true
    class of the bilinearly upsampled (align_corners=True) logits (0 where the label is ignored) and their log-sum-exp."""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    assert target.dtype == torch.int64 and tuple(target.shape) == (N, Ho, Wo) and target.is_contiguous(), (target.dtype, tuple(target.shape))
    logp = torch.empty((N, Ho, Wo), device=x.device, dtype=torch.float32)
    lse = torch.empty((N, Ho, Wo), device=x.device, dtype=torch.float32)
    check(_lib.lib().fsb_loss_logp_fwd(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(target), int(ignore_label), _ptr(logp), _ptr(lse),
                                       _stream()), "fsb_loss_logp_fwd")
    return logp, lse


def kth_smallest(x, k):
    """exact k-th smallest (1-based) element of a contiguous fp32 tensor as a 0-d device tensor; no sort, no host synchronisation"""
    assert x.dtype == torch.float32 and x.is_contiguous() and 1 <= k <= x.numel()
    out = torch.empty((), device=x.device, dtype=torch.float32)
    ws = torch.empty((_lib.lib().fsb_kth_workspace_bytes(),), device=x.device, dtype=torch.uint8)
    check(_lib.lib().fsb_kth_smallest_f32(_ptr(x), x.numel(), int(k), _ptr(out), _ptr(ws), _stream()), "fsb_kth_smallest_f32")
    return out


def ohem_reduce(logp_t, target, ignore_label, num_classes, thr=None):
    """-> fp32 tensor [sum(-logp_t * kept), count(kept)], kept = valid label & (logp_t <= thr); thr: 0-d device tensor or None"""
    out = torch.empty((2,), device=logp_t.device, dtype=torch.float32)
    partial = torch.empty((2 * _lib.lib().fsb_loss_rows(),), device=logp_t.device, dtype=torch.float32)
    check(_lib.lib().fsb_ohem_reduce(_ptr(logp_t), _ptr(target), logp_t.numel(), int(ignore_label), int(num_classes), _ptr(thr), _ptr(partial),
                                     _ptr(out), _stream()), "fsb_ohem_reduce")
    return out


def loss_ce_bwd(x, target, size, ignore_label, lse, logp_t, thr, coef, gscale, out=None):
    """gradient of sum over kept pixels of coef * (-logp_t) w.r.t. the low-resolution logits x: NHWC fp16, times gscale.  out: accumulate."""
    N, Cc, Hi, Wi, xcs = nhwc_info(x)
    Ho, Wo = int(size[0]), int(size[1])
    acc = out is not None
    dx = out if acc else empty_nhwc(N, Cc, Hi, Wi, x.device)
    check(_lib.lib().fsb_loss_ce_bwd(N, Cc, Hi, Wi, Ho, Wo, _ptr(x), xcs, _ptr(target), int(ignore_label), _ptr(lse), _ptr(logp_t), _ptr(thr),
                                     _ptr(coef), _ptr(dx), nhwc_info(dx)[4], float(gscale), int(acc), _stream()), "fsb_loss_ce_bwd")
    return dx


def loss_kl_fwd(xs, xt, size):
    """sum over pixels and classes of q (log q - log p), p = softmax(up(xs)), q = softmax(up(xt)) -> (0-d sum, lse_s, lse_t)"""
    N, Cc, Hs, Ws, scs = nhwc_info(xs)
    Nt, Ct, Ht, Wt, tcs = nhwc_info(xt)
    assert (N, Cc) == (Nt, Ct)
    Ho, Wo = int(size[0]), int(size[1])
    lse_s = torch.empty((N, Ho, Wo), device=xs.device, dtype=torch.float32)
    lse_t = torch.empty((N, Ho, Wo), device=xs.device, dtype=torch.float32)
    out = torch.empty((2,), device=xs.device, dtype=torch.float32)
    partial = torch.empty((2 * _lib.lib().fsb_loss_rows(),), device=xs.device, dtype=torch.float32)
    check(_lib.lib().fsb_loss_kl_fwd(N, Cc, Hs, Ws, Ht, Wt, Ho, Wo, _ptr(xs), scs, _ptr(xt), tcs, _ptr(lse_s), _ptr(lse_t), _ptr(partial),
                                     _ptr(out), _stream()), "fsb_loss_kl_fwd")
    return out[0], lse_s, lse_t


def loss_kl_bwd(xs, xt, size, lse_s, lse_t, coef, gscale, out=None):
    N, Cc, Hs, Ws, scs = nhwc_info(xs)
    _, _, Ht, Wt, tcs = nhwc_info(xt)
    Ho, Wo = int(size[0]), int(size[1])
    acc = out is not None
    dx = out if acc else empty_nhwc(N, Cc, Hs, Ws, xs.device)
    check(_lib.lib().fsb_loss_kl_bwd(N, Cc, Hs, Ws, Ht, Wt, Ho, Wo, _ptr(xs), scs, _ptr(xt), tcs, _ptr(lse_s), _ptr(lse_t), _ptr(coef), _ptr(dx),
                                     nhwc_info(dx)[4], float(gscale), int(acc), _stream()), "fsb_loss_kl_bwd")
    return dx
