#!/usr/bin/env python
"""Train/ vs latency/ network variant of the student (arch_1) at 1x3x1024x2048 on one GPU.

Per run, alternating the two variants (--runs times): device-resident CUDA-graph replay FPS over a rotating pool of seeded input
frames larger than L2 (logits mode, fp16 logits, and labels mode), and launches per replay.  Then one zoomed cell (conv_2x_downup at
stride 1 on the 1/8 map) through `functional` with the nearest /2 and x2 folded into its convs against the same cell with
standalone nearest kernels, both captured in CUDA graphs.  Prints the card name, power limit and SM clock read in the same run,
and one JSON line with everything."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fasterseg_b200 import functional as F_  # noqa: E402
from fasterseg_b200 import zoo  # noqa: E402
from fasterseg_b200.runtime import GraphedInference  # noqa: E402
from oracle import fasterseg_oracle as orc  # noqa: E402


def gpu_line():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name()


def build(variant):
    model = zoo.build_network(1, variant=variant).cuda().eval()
    shapes = {k: tuple(v.shape) for k, v in model.state_dict().items() if not k.endswith("num_batches_tracked")}
    sd = orc.random_state_dict(shapes, seed=2025)
    own, seen = model.state_dict(), set()
    with torch.no_grad():
        for k in sorted(sd):
            if own[k].data_ptr() not in seen:
                seen.add(own[k].data_ptr())
                own[k].copy_(sd[k])
    return model


def replay_fps(g, pool, iters, warmup):
    for i in range(warmup):
        g(pool[i % len(pool)])
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(iters):
        g(pool[i % len(pool)])
    t1.record()
    t1.synchronize()
    return iters * 1000.0 / t0.elapsed_time(t1)


def graph_us(fn, iters, warmup):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(warmup):
        g.replay()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        g.replay()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) * 1000.0 / iters


def cell_times(iters, warmup, runs):
    """conv_2x_downup (stride 1) on the 1/8 map of the frame: 64 channels at 128x256"""
    N, C, H, W = 1, 64, 128, 256
    x = F_.empty_nhwc(N, C, H, W, "cuda")
    x.copy_(orc.random_input((N, C, H, W), seed=11).cuda())
    packs = []
    for s in (1, 2):
        w = orc.random_input((C, C, 3, 3), seed=20 + s).cuda() * (2.0 / (9 * C)) ** 0.5
        packs.append(F_.pack_conv_weight(w, C, C, 3))
    sc = torch.ones(C, device="cuda")
    sh = torch.zeros(C, device="cuda")
    out = F_.empty_nhwc(N, C, H, W, "cuda")

    def folded():
        y = F_.conv_fwd(x, packs[0], C, 3, 1, 1, sc, sh, relu=True, down2=True)
        F_.conv_fwd(y, packs[1], C, 3, 1, 1, sc, sh, relu=True, out=out, up2=True)

    def standalone():
        y = F_.conv_fwd(F_.nearest(x, (H // 2, W // 2)), packs[0], C, 3, 1, 1, sc, sh, relu=True)
        F_.nearest(F_.conv_fwd(y, packs[1], C, 3, 1, 1, sc, sh, relu=True), (H, W), out=out)

    res = {"folded": [], "standalone": []}
    for _ in range(runs):
        res["folded"].append(graph_us(folded, iters, warmup))
        res["standalone"].append(graph_us(standalone, iters, warmup))
    folded()
    a = out.clone()
    standalone()
    assert torch.equal(a, out), "folded and standalone cell differ"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--pool", type=int, default=4, help="input frames rotated through (4 x 25 MB fp32 > 50 MB L2)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    hw = gpu_line()
    print("gpu:", hw, flush=True)
    pool = [orc.random_input((1, 3, 1024, 2048), seed=100 + i).cuda() for i in range(args.pool)]
    models = {v: build(v) for v in ("train", "latency")}
    graphs = {(v, m): GraphedInference(models[v], pool[0], mode=m, logits_dtype=torch.float16)
              for v in models for m in ("logits", "labels")}
    res = {v: {"logits_fps": [], "labels_fps": [], "launches": graphs[(v, "logits")].launches_per_replay,
               "launches_labels": graphs[(v, "labels")].launches_per_replay} for v in models}
    for r in range(args.runs):
        for v in ("train", "latency"):
            for m in ("logits", "labels"):
                fps = replay_fps(graphs[(v, m)], pool, args.iters, args.warmup)
                res[v][m + "_fps"].append(fps)
                print("run %d %-7s %-6s %8.1f FPS" % (r, v, m, fps), flush=True)
    cell = cell_times(args.iters, args.warmup, args.runs)
    for k, v in cell.items():
        print("cell conv_2x_downup 64ch 128x256 %-10s %s us" % (k, " / ".join("%.1f" % t for t in v)))
    for v in models:
        print("%-7s logits median %.1f FPS, labels median %.1f FPS, launches per replay %d (labels %d)"
              % (v, statistics.median(res[v]["logits_fps"]), statistics.median(res[v]["labels_fps"]), res[v]["launches"],
                 res[v]["launches_labels"]))
    print("gpu:", gpu_line())
    print(json.dumps({"gpu": hw, "variants": res, "cell_us": cell}))


if __name__ == "__main__":
    main()
