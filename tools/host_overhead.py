#!/usr/bin/env python
"""Host-side cost of one supernet step, measured WITHOUT a GPU: every tensor-level wrapper of `fasterseg_b200.functional`
is replaced by a stub that only allocates correctly-shaped outputs, so what remains is exactly the Python the real step
executes between kernel launches (module dispatch, autograd Functions, cache lookups, descriptor building, scalar
arithmetic on the architecture parameters).  The real step is host-launch-bound (~20 k launches, DESIGN.md section 3), so
this is the number to push down; the ctypes call itself (~2-4 us each) is not included.
Usage: python tools/host_overhead.py [--mode pretrain|search] [--layers 16] [--steps 3] [--profile]"""
import argparse
import cProfile
import os
import pstats
import sys
import time

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fasterseg_b200 import functional as F_  # noqa: E402
from fasterseg_b200._lib import ConvDesc  # noqa: E402

CALLS = {}
WORK = {"flops": 0.0, "bytes": 0.0, "roof_s": 0.0}   # algorithmic work of the launches the stubs stand for
PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0                # H100 SXM data sheet (dense FP16, HBM3), not measured


def _count(name):
    CALLS[name] = CALLS.get(name, 0) + 1


def _work(flops, nbytes):
    """one launch (or fused group of launches) worth `flops` and `nbytes` of algorithmic traffic"""
    WORK["flops"] += flops
    WORK["bytes"] += nbytes
    WORK["roof_s"] += max(flops / (PEAK_TFLOPS * 1e12), nbytes / (PEAK_GBS * 1e9))


def _numel(t):
    return float(t.shape[0] * t.shape[1] * t.shape[2] * t.shape[3])


def _e(N, C, H, W, dtype=torch.float16):
    return F_.empty_nhwc(N, C, H, W, "cpu", dtype=dtype)


def install_null_backend():
    def nhwc_info(t, dtype=torch.float16):
        N, Cc, H, W = t.shape
        return N, Cc, H, W, t.stride(3) if W > 1 else max(Cc, 1)

    def to_nhwc_half(x):
        if x.dtype == torch.float16 and x.dim() == 4 and (x.shape[1] == 1 or x.stride(1) == 1):
            return x
        _count("to_nhwc_half")
        return _e(*x.shape)

    def conv_fwd(x, wp, Cout, k, s, p, scale=None, shift=None, relu=False, out=None, off=(0, 0), stats=None, force_direct=False,
                 out_f32=False):
        _count("conv_fwd")
        N, Cin, H, W = x.shape
        Ho, Wo = F_.conv_out_size(H, W, k, s, p, 1, off[0], off[1])
        _work(2.0 * k * k * Cin * Cout * N * Ho * Wo, 2 * _numel(x) + (4 if out_f32 else 2) * N * Cout * Ho * Wo + 2 * k * k * Cin * Cout)
        return out if out is not None else _e(N, Cout, Ho, Wo, torch.float32 if out_f32 else torch.float16)

    def stem_conv_nchw(x, w, scale, shift, relu=True, out=None):
        _count("stem_conv")
        return out if out is not None else _e(x.shape[0], w.shape[0], (x.shape[2] + 1) // 2, (x.shape[3] + 1) // 2)

    def bilinear(x, size, relu=False, out=None):
        _count("bilinear")
        _work(0.0, 2 * _numel(x) + 2.0 * x.shape[0] * x.shape[1] * int(size[0]) * int(size[1]))
        return out if out is not None else _e(x.shape[0], x.shape[1], int(size[0]), int(size[1]))

    def train_fwd(x, wp, Cout, k, s, p, off, gamma, beta, eps, momentum, rm, rv, nbt, relu):
        _count("conv_bn_act_train_fwd")
        N, Cin, H, W = x.shape
        Ho, Wo = F_.conv_out_size(H, W, k, s, p, 1, off[0], off[1])
        d = ConvDesc(N, H, W, Cin, Cout, k, s, p, 1, off[0], off[1], Ho, Wo, x.stride(3), (Cout + 7) // 8 * 8, 0)
        px = float(N * Cout * Ho * Wo)
        # conv (x in, fp32 raw out, weights) + apply (raw in, fp16 y out)
        _work(2.0 * k * k * Cin * Cout * N * Ho * Wo, 2 * _numel(x) + 4 * px + 2 * k * k * Cin * Cout + 4 * px + 2 * px)
        return _e(N, Cout, Ho, Wo), _e(N, Cout, Ho, Wo, torch.float32), torch.empty(6 * Cout), d

    def train_bwd(d, x, dy, y, raw, vec, gamma, relu, wt, w, need_dx, dw_acc, gscale):
        _count("conv_bn_act_train_bwd")
        Cout = dy.shape[1]
        px, kk = _numel(dy), d.ksize * d.ksize
        gemm = 2.0 * kk * d.Cin * Cout * dy.shape[0] * dy.shape[2] * dy.shape[3]
        # BN backward: two passes over (dy, y, raw) + draw out; dgrad: draw + weights in, dx out; wgrad: x + draw in, dW out
        _work((2.0 if need_dx else 1.0) * gemm,
              2 * (2 + 2 + 4) * px + 2 * px + (2 * px + 2 * _numel(x) if need_dx else 0) + 2 * _numel(x) + 2 * px + 6 * kk * d.Cin * Cout)
        dx = _e(dy.shape[0], d.Cin, d.H, d.W) if need_dx else None
        return dx, torch.empty(Cout), torch.empty(Cout)

    def bn_finalize(stats, count, gamma, beta, eps, momentum, rm, rv, want_save=False):
        _count("bn_finalize")
        b = torch.empty((4, stats.numel() // 2))
        return b[0], b[1], b[2], b[3]

    def wsum_bwd(dout, xs, wts, need_dx, need_dw, gscale):
        _count("wsum_bwd")
        _work(0.0, 2 * _numel(dout) * (1 + len(xs) + sum(1 for n in need_dx if n)))
        return [_e(*dout.shape) if n else None for n in need_dx], (torch.empty(len(xs)) if need_dw else None)

    def conv_wgrad(x, dy, w_like, Cin, Cout, k, s, p, gscale, off=(0, 0), accumulate_into=None, force_direct=False):
        _count("conv_wgrad")
        _work(2.0 * k * k * Cin * Cout * dy.shape[0] * dy.shape[2] * dy.shape[3], 2 * _numel(x) + 2 * _numel(dy) + 4 * k * k * Cin * Cout)
        return accumulate_into if accumulate_into is not None else torch.empty_like(w_like)

    simple = {
        "to_nchw": lambda x, dtype=torch.float32: torch.zeros(tuple(x.shape), dtype=dtype),
        "pack_conv_weight": lambda w, ci, co, k: torch.empty(1, dtype=torch.float16),
        "pack_conv_weight_dgrad": lambda w, ci, co, k: torch.empty(1, dtype=torch.float16),
        "bn_fold": lambda g, b, m, v, eps, conv_bias=None: (torch.empty_like(m), torch.empty_like(m)),
        "upsample_logits": lambda x, size, dtype=torch.float32, out=None: torch.zeros((x.shape[0], x.shape[1], int(size[0]), int(size[1])), dtype=dtype),
        "copy_channels": lambda x, out: out,
        "bn_stats": lambda x, stats=None: torch.empty(2 * x.shape[1]) if stats is None else stats,
        "affine_act": lambda x, scale, shift, relu=False, out=None: out if out is not None else _e(*x.shape),
        "bn_bwd_sums": lambda dy, y, raw, mean, invstd, relu: torch.empty(2 * dy.shape[1]),
        "bn_bwd_apply": lambda dy, y, raw, mean, invstd, gamma, sums, count, relu, gscale, want_param_grads=True:
            (_e(*dy.shape), torch.empty(dy.shape[1]), torch.empty(dy.shape[1])),
        "relu_bwd": lambda dy, y: _e(*dy.shape),
        "conv_dgrad": lambda dy, w, xs, ci, co, k, s, p, off=(0, 0), wpacked_t=None, force_direct=False: _e(*xs),
        "bilinear_bwd": lambda dy, in_hw, relu_mask_y=None: _e(dy.shape[0], dy.shape[1], *in_hw),
        "upsample_logits_bwd": lambda dy, in_hw, gscale: _e(dy.shape[0], dy.shape[1], *in_hw),
        "nchw_grad_to_nhwc": lambda dy, gscale: _e(*dy.shape),
        "wsum_fwd": lambda xs, wts, out=None: out if out is not None else _e(*xs[0].shape),
        "add_inplace": lambda x, y: y,
    }
    for name, fn in simple.items():
        def wrapped(*a, _fn=fn, _name=name, **k):
            _count(_name)
            res = _fn(*a, **k)
            # elementwise / layout kernels: every 4-D tensor argument read once, every 4-D result written once
            touched = [t for t in list(a) + (list(res) if isinstance(res, tuple) else [res]) if isinstance(t, torch.Tensor) and t.dim() == 4]
            if _name == "conv_dgrad":
                dy, w, xs, ci, co, kk = a[0], a[1], a[2], a[3], a[4], a[5]
                _work(2.0 * kk * kk * ci * co * dy.shape[0] * dy.shape[2] * dy.shape[3], 2 * _numel(dy) + 2.0 * xs[0] * xs[1] * xs[2] * xs[3] + 2 * kk * kk * ci * co)
            elif _name == "wsum_fwd":
                _work(0.0, 2 * _numel(a[0][0]) * (len(a[0]) + 1))
            elif _name not in ("pack_conv_weight", "pack_conv_weight_dgrad", "bn_fold", "bn_finalize"):
                _work(0.0, sum(t.element_size() * _numel(t) for t in touched))
            return res
        setattr(F_, name, wrapped)
    for name, fn in (("nhwc_info", nhwc_info), ("to_nhwc_half", to_nhwc_half), ("conv_fwd", conv_fwd), ("stem_conv_nchw", stem_conv_nchw),
                     ("bilinear", bilinear), ("conv_bn_act_train_fwd", train_fwd), ("conv_bn_act_train_bwd", train_bwd),
                     ("bn_finalize", bn_finalize), ("wsum_bwd", wsum_bwd), ("conv_wgrad", conv_wgrad)):
        setattr(F_, name, fn)
    F_.is_nhwc_half = lambda t: t.dtype == torch.float16 and t.dim() == 4 and (t.shape[1] == 1 or t.stride(1) == 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="pretrain", choices=["pretrain", "search"])
    ap.add_argument("--layers", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    torch.set_num_threads(1)
    install_null_backend()
    from fasterseg_b200.model_search import Network_Multi_Path
    WML = [4. / 12, 6. / 12, 8. / 12, 10. / 12, 1.]
    model = Network_Multi_Path(19, args.layers, nn.CrossEntropyLoss(ignore_index=255), Fch=12, width_mult_list=WML,
                               prun_modes=['max', 'arch_ratio'], stem_head_width=[(1, 1), (8. / 12, 8. / 12)]).train()
    B, H, W = (3, 256, 512) if args.mode == "pretrain" else (2, 224, 448)
    x = torch.zeros(B, 3, H, W)
    t = torch.randint(0, 19, (B, H // 8, W // 8))
    np.random.seed(1)
    torch.manual_seed(1)

    def step():
        # gradients stay allocated between steps: re-creating 1 GB of zero-filled fp32 buffers costs seconds on a CPU and
        # microseconds of host time on the GPU (one memset kernel per parameter) -- it would drown what is measured here
        loss = model._loss(x, t, True if args.mode == "pretrain" else "dir")
        loss.backward()

    step()  # warm-up: weight-pack caches, grad buffers
    CALLS.clear()
    for k_ in WORK:
        WORK[k_] = 0.0
    prof = cProfile.Profile() if args.profile else None
    times = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        if prof:
            prof.enable()
        step()
        if prof:
            prof.disable()
        times.append(time.perf_counter() - t0)
    n_calls = sum(CALLS.values()) // args.steps
    print("mode %s layers %d: host time per step (forward x4 + backward, null backend) median %.0f ms, min %.0f ms; %d backend calls/step -> %.1f us of Python per call"
          % (args.mode, args.layers, 1e3 * sorted(times)[len(times) // 2], 1e3 * min(times), n_calls, 1e6 * min(times) / max(n_calls, 1)))
    print("algorithmic work per step: %.2f TFLOP, %.1f GB -> sum over launches of max(FLOPs / %.0f TFLOP/s, bytes / %.0f GB/s) = %.1f ms"
          % (WORK["flops"] / args.steps / 1e12, WORK["bytes"] / args.steps / 1e9, PEAK_TFLOPS, PEAK_GBS, 1e3 * WORK["roof_s"] / args.steps))
    print("calls/step:", {k: v // args.steps for k, v in sorted(CALLS.items(), key=lambda kv: -kv[1])})
    if prof:
        pstats.Stats(prof).sort_stats("tottime").print_stats(28)


if __name__ == "__main__":
    main()
