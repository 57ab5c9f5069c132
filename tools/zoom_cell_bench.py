#!/usr/bin/env python
"""One zoomed cell of the student frame with its producer, with and without the fused resizes, on one GPU.

The pair is the frame's conv that feeds a zoomed cell (3x3 64 -> 64 on the 64x128 map, BN + ReLU) followed by that cell
(conv_2x_downup at stride 1: bilinear /2, two 3x3 convs, bilinear x2 + ReLU).  Unfused: four launches as the parent ran them
(conv, /2, conv, conv, x2 -- five).  Fused: the producer conv also stores the /2 map (fsb_conv_fwd_half) and the cell starts from
it (x_half) -- four launches.  Both are captured in CUDA graphs and replayed alternately; the outputs must be the same bits.
Prints the card name, power limit and SM clock read in the same run, and one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fasterseg_b200 import engine  # noqa: E402
from fasterseg_b200 import functional as F_  # noqa: E402
from fasterseg_b200.operations import BasicResidual_downup_2x  # noqa: E402


def gpu_line():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name()


def randomise_(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(module.state_dict().items()):
            if name.endswith("num_batches_tracked"):
                continue
            if p.dim() == 4:
                p.copy_(torch.randn(p.shape, generator=g) * (2.0 / (p.shape[1] * 9)) ** 0.5)
            elif name.endswith("running_var") or name.endswith("weight"):
                p.copy_(torch.rand(p.shape, generator=g) + 0.5)
            else:
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=2000)
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda")
    C, H, W = 64, 64, 128
    conv, bn = nn.Conv2d(C, C, 3, 1, 1, bias=False), nn.BatchNorm2d(C)
    cell = BasicResidual_downup_2x(C, C, stride=1, slimmable=False)
    for i, m in enumerate((conv, bn, cell)):
        randomise_(m, 100 + i)
    conv, bn, cell = conv.to(dev).eval(), bn.to(dev).eval(), cell.to(dev).eval()
    x = F_.to_nhwc_half(torch.randn(1, C, H, W, generator=torch.Generator().manual_seed(7)).to(dev))
    half = F_.empty_nhwc(1, C, H // 2, W // 2, dev)

    def unfused():
        return cell(engine.conv_bn_act(x, conv, bn, relu=True))

    def fused():
        return cell(engine.conv_bn_act(x, conv, bn, relu=True, out_half=half), x_half=half)

    graphs, outs = {}, {}
    with torch.no_grad():
        for name, fn in (("unfused", unfused), ("fused", fused)):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                outs[name] = fn()
            graphs[name] = g
    for g in graphs.values():
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(outs["fused"], outs["unfused"]), "fused and unfused cell outputs differ"
    times = {name: [] for name in graphs}
    for _ in range(args.runs):
        for name, g in graphs.items():
            for _ in range(50):
                g.replay()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.replays):
                g.replay()
            t1.record()
            torch.cuda.synchronize()
            times[name].append(t0.elapsed_time(t1) * 1000.0 / args.replays)
    med = {name: statistics.median(v) for name, v in times.items()}
    line = {"gpu": gpu_line(), "cell": "conv 3x3 %d->%d @%dx%d + conv_2x_downup s1" % (C, C, H, W),
            "us_per_replay": {k: round(v, 2) for k, v in med.items()}, "runs_us": {k: [round(t, 2) for t in v] for k, v in times.items()},
            "saved_us": round(med["unfused"] - med["fused"], 2), "bit_identical": True}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
