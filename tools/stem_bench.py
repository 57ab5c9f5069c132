#!/usr/bin/env python
"""The fused stem kernel (K1f, F_.stem_fused) against the two launches it replaces (stem_conv_* + conv_fwd of stem.1.conv1) at
the student's widths (3 -> 32 -> 64) on 1x3x1024x2048 frames, fp32 NCHW and uint8 HWC input.  Each variant is a CUDA graph of
`--reps` launches that rotates through a pool of distinct frames larger than the 50 MB L2, so every launch reads its frame from HBM
as in the frame forward.  The two paths are alternated for `--rounds` rounds; prints median (min-max) us per frame, the card, its
power limit and SM clock, and whether the outputs are bit-identical."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fasterseg_b200 import functional as F_  # noqa: E402

H, W = 1024, 2048
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = "nvidia-smi unavailable: %s" % e
    return q


def _graph(fn, frames, reps):
    for x in frames[:2]:
        fn(x)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(reps):
            fn(frames[i % len(frames)])
    return g


def _time(g, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g.replay()
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--pool-mb", type=float, default=160.0)
    a = ap.parse_args()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    w0 = (torch.randn(32, 3, 3, 3, generator=g) * (2.0 / 27) ** 0.5).to(dev)
    w1 = (torch.randn(64, 32, 3, 3, generator=g) * (2.0 / 288) ** 0.5).to(dev)
    s0, b0 = (torch.rand(32, generator=g) + 0.5).to(dev), (torch.randn(32, generator=g) * 0.1).to(dev)
    s1, b1 = (torch.rand(64, generator=g) + 0.5).to(dev), (torch.randn(64, generator=g) * 0.1).to(dev)
    w1p = F_.pack_conv_weight(w1, 32, 64, 3)
    lut = F_.normalization_lut(MEAN, STD, dev)
    print("card: %s" % _card())
    for kind in ("fp32", "uint8"):
        nbytes = 3 * H * W * (4 if kind == "fp32" else 1)
        n = max(2, int(a.pool_mb * 1e6 / nbytes) + 1)
        if kind == "fp32":
            frames = [torch.randn(1, 3, H, W, generator=g).to(dev) for _ in range(n)]
        else:
            frames = [torch.randint(0, 256, (1, H, W, 3), generator=g, dtype=torch.uint8).to(dev).permute(0, 3, 1, 2) for _ in range(n)]
        out_pair = F_.empty_nhwc(1, 64, H // 4, W // 4, dev)
        out_fused = F_.empty_nhwc(1, 64, H // 4, W // 4, dev)

        def pair(x):
            y0 = F_.stem_conv_u8hwc(x, lut, w0, s0, b0) if x.dtype == torch.uint8 else F_.stem_conv_nchw(x, w0, s0, b0)
            return F_.conv_fwd(y0, w1p, 64, 3, 2, 1, s1, b1, relu=True, out=out_pair)

        def fused(x):
            y = F_.stem_fused(x, lut, w0, s0, b0, w1p, 64, s1, b1, out=out_fused)
            assert y is not None, "no fused kernel for the student's stem"
            return y

        pair(frames[0])
        fused(frames[0])
        torch.cuda.synchronize()
        same = torch.equal(out_pair, out_fused)
        gp, gf = _graph(pair, frames, a.reps), _graph(fused, frames, a.reps)
        tp, tf = [], []
        for _ in range(a.rounds):
            tp.append(_time(gp, a.reps))
            tf.append(_time(gf, a.reps))
        mp, mf = statistics.median(tp), statistics.median(tf)
        print("%-5s pool %d frames (%.0f MB): stem_conv + conv_fwd %.2f us (%.2f-%.2f), stem_fused %.2f us (%.2f-%.2f), "
              "gain %.2f us, outputs bit-identical: %s"
              % (kind, n, n * nbytes / 1e6, mp, min(tp), max(tp), mf, min(tf), max(tf), mp - mf, same))


if __name__ == "__main__":
    main()
