"""Frame-level roofline accounting (SURVEY section 8d: "report both per-kernel fraction and frame-level Sigma-roofline
fraction").

`trace_launches(fn)` runs `fn()` once with the launching wrappers of `fasterseg_b200.functional` instrumented and returns,
per kernel launch, its ALGORITHMIC work: FLOPs and the bytes it must move if every operand is read once and every result
written once (activations at their storage width, packed fp16 weights).  `sigma_roofline` turns that list into the time the
same launches would take if each ran exactly at the measured machine peaks -- sum over launches of
max(flops / tensor peak, bytes / HBM peak) -- which is the denominator for a whole-frame efficiency figure.
Pure bookkeeping on tensor shapes: no device work beyond the forward it wraps."""
from __future__ import annotations

import contextlib
from typing import Callable, Dict, List

from . import functional as F_


def _esize(t):
    return t.element_size()


def _conv_record(name, x, Cout, k, stride, pad, off, out):
    N, Cin, H, W = x.shape
    Ho, Wo = out.shape[2], out.shape[3]
    flops = 2.0 * k * k * Cin * Cout * N * Ho * Wo
    nbytes = N * Cin * (H - off[0]) * (W - off[1]) * _esize(x) + N * Cout * Ho * Wo * _esize(out) + k * k * Cin * Cout * 2
    return {"kernel": name, "flops": flops, "bytes": float(nbytes), "shape": "%dx%d %d->%d @%dx%d s%d" % (k, k, Cin, Cout, Ho, Wo, stride)}


def _rec_conv(res, a, kw):
    x, _, Cout, k, stride, pad = a[:6]
    return _conv_record("conv", x, Cout, k, stride, pad, kw.get("off", (0, 0)), res)


def _rec_stem(res, a, kw):
    x, w = a[0], a[1]
    N, Co, Ho, Wo = res.shape
    return {"kernel": "stem_conv", "flops": 2.0 * 27 * Co * N * Ho * Wo,
            "bytes": float(x.numel() * _esize(x) + N * Co * Ho * Wo * 2 + w.numel() * 4), "shape": "3x3 3->%d @%dx%d s2" % (Co, Ho, Wo)}


def _rec_stem_fused(res, a, kw):
    x, w0, w1 = a[0], a[2], a[5]
    if res is None:   # no fused kernel for these widths: the caller's two launches are recorded instead
        return None
    N, C1, H1, W1 = res.shape
    C0 = w0.shape[0]
    H0, W0 = (x.shape[2] + 1) // 2, (x.shape[3] + 1) // 2
    return {"kernel": "stem_fused", "flops": 2.0 * 27 * C0 * N * H0 * W0 + 2.0 * 9 * C0 * C1 * N * H1 * W1,
            "bytes": float(x.numel() * _esize(x) + N * C1 * H1 * W1 * 2 + w0.numel() * 4 + w1.numel() * 2),
            "shape": "3x3 3->%d->%d @%dx%d s2 s2" % (C0, C1, H1, W1)}


def _rec_bilinear(res, a, kw):
    x = a[0]
    N, Cc, Hi, Wi = x.shape
    return {"kernel": "bilinear", "flops": 0.0, "bytes": float(N * Cc * (Hi * Wi + res.shape[2] * res.shape[3]) * 2),
            "shape": "%d ch %dx%d -> %dx%d" % (Cc, Hi, Wi, res.shape[2], res.shape[3])}


def _rec_copy(res, a, kw):
    x = a[0]
    return {"kernel": "copy_channels", "flops": 0.0, "bytes": float(2 * x.shape[0] * x.shape[1] * x.shape[2] * x.shape[3] * 2),
            "shape": "%d ch @%dx%d" % (x.shape[1], x.shape[2], x.shape[3])}


def _rec_upsample(res, a, kw):
    x = a[0]
    return {"kernel": "upsample_logits", "flops": 0.0,
            "bytes": float(x.shape[0] * x.shape[1] * x.shape[2] * x.shape[3] * 2 + res.numel() * _esize(res)),
            "shape": "%d ch %dx%d -> %dx%d %s" % (x.shape[1], x.shape[2], x.shape[3], res.shape[2], res.shape[3], str(res.dtype)[6:])}


def _rec_argmax(res, a, kw):
    x = a[0]
    return {"kernel": "upsample_argmax", "flops": 0.0, "bytes": float(x.shape[0] * x.shape[1] * x.shape[2] * x.shape[3] * 2 + res.numel()),
            "shape": "%d ch %dx%d -> %dx%d u8" % (x.shape[1], x.shape[2], x.shape[3], res.shape[1], res.shape[2])}


_RECORDERS = {"conv_fwd": _rec_conv, "stem_conv_nchw": _rec_stem, "stem_fused": _rec_stem_fused, "bilinear": _rec_bilinear, "copy_channels": _rec_copy,
              "upsample_logits": _rec_upsample, "upsample_argmax": _rec_argmax}


@contextlib.contextmanager
def _instrumented(records: List[Dict]):
    saved = {name: getattr(F_, name) for name in _RECORDERS}

    def traced(orig, make_record):
        def call(*a, **kw):
            res = orig(*a, **kw)
            rec = make_record(res, a, kw)
            if rec is not None:
                records.append(rec)
            return res
        return call

    try:
        for name, rec in _RECORDERS.items():
            setattr(F_, name, traced(saved[name], rec))
        yield
    finally:
        for name, orig in saved.items():
            setattr(F_, name, orig)


def trace_launches(fn: Callable[[], object]) -> List[Dict]:
    """Run `fn()` once and return one record {"kernel", "shape", "flops", "bytes"} per launch of the inference path."""
    records: List[Dict] = []
    with _instrumented(records):
        fn()
    return records


def sigma_roofline(records: List[Dict], tensor_tflops: float, hbm_gbs: float) -> Dict:
    """Sum over launches of max(flops / tensor peak, bytes / HBM peak) and the totals that go with it."""
    t_total = 0.0
    n_tensor = 0
    for r in records:
        t_tensor = r["flops"] / (tensor_tflops * 1e12)
        t_hbm = r["bytes"] / (hbm_gbs * 1e9)
        r["roof_us"] = max(t_tensor, t_hbm) * 1e6
        r["bound"] = "tensor" if t_tensor >= t_hbm else "hbm"
        n_tensor += r["bound"] == "tensor"
        t_total += max(t_tensor, t_hbm)
    return {"launches": len(records), "tensor_bound_launches": n_tensor, "sum_us": t_total * 1e6,
            "gflop": sum(r["flops"] for r in records) / 1e9, "mbytes": sum(r["bytes"] for r in records) / 1e6}
