#!/usr/bin/env python
"""Per-layer micro-benchmark of the conv / resize kernels on the student's layer shapes (1x3x1024x2048 frame).
Prints us/launch, achieved TFLOP/s and algorithmic GB/s per layer; `--only i` restricts to one layer.
`--compare`: on every layer time conv_tc's per-tap mode (FSB_CONV_TC2=0) and, on 3x3 stride-1 convs, its window mode
(FSB_CONV_TC2=1), alternating them `--rounds` times in this process; print the median us of each and the L2 -> SM bytes each
mode moves (TMA boxes of input and weights, from conv_plan's tiling rule)."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fasterseg_b200 import _lib  # noqa: E402
from fasterseg_b200 import functional as F_  # noqa: E402

# name, Cin, Cout, k, stride, H, W (input)
LAYERS = [
    ("stem.1.conv1", 32, 64, 3, 2, 512, 1024),
    ("stem.1.conv2", 64, 64, 3, 1, 256, 512),
    ("stem.2.conv1", 64, 64, 3, 2, 256, 512),
    ("stem.2.conv2", 64, 64, 3, 1, 128, 256),
    ("cell0.conv1", 64, 32, 3, 1, 128, 256),
    ("cell1.conv", 32, 32, 3, 1, 128, 256),
    ("cell2.conv(down)", 32, 32, 3, 1, 64, 128),
    ("cell3-0.conv", 32, 128, 3, 1, 64, 128),
    ("cell4-0.conv1", 128, 64, 3, 1, 32, 64),
    ("cell5-0.conv", 64, 64, 3, 1, 32, 64),
    ("cell5-1.conv1", 32, 64, 3, 2, 128, 256),
    ("cell7-0.conv1", 64, 128, 3, 1, 32, 64),
    ("cell7-0.conv2", 128, 128, 3, 1, 32, 64),
    ("cell7-1.conv1", 64, 192, 3, 1, 32, 64),
    ("cell7-1.conv2", 192, 192, 3, 1, 32, 64),
    ("cell8-0.conv", 128, 128, 3, 1, 16, 32),
    ("cell8-1.conv1", 192, 128, 3, 1, 32, 64),
    ("cell9-0.conv1", 128, 256, 3, 1, 16, 32),
    ("cell9-0.conv2", 256, 256, 3, 1, 16, 32),
    ("arms32.0", 256, 128, 1, 1, 32, 64),
    ("arms16", 128, 64, 1, 1, 64, 128),
    ("refines32.0", 192, 128, 3, 1, 64, 128),
    ("refines16", 96, 64, 3, 1, 128, 256),
    ("ffm", 128, 128, 1, 1, 128, 256),
    ("heads8.conv3x3", 128, 128, 3, 1, 128, 256),
    ("heads8.conv1x1", 128, 19, 1, 1, 128, 256),
]


SMS = 132  # H100 SXM


def l2_to_sm_mb(ci, co, k, s, h, w, mode):
    """(MB of TMA boxes one launch loads into shared memory in `mode` ("per-tap" or "window"), CTAs), following
    conv_plan: 16 x 8 tiles (8 x 16 when Wo < 16), N tile of <= 128 channels split while the grid has fewer CTAs than SMs;
    per-tap: one input box of 128 px x BK and one weight box per (tap, chunk); window: one (th + 2) x (tw + 2) px x 64-channel
    window per chunk and one weight box per (chunk, tap)."""
    pad = 1 if k == 3 else 0
    ho, wo = (h + 2 * pad - k) // s + 1, (w + 2 * pad - k) // s + 1
    tw = 16 if wo >= 16 else 8
    th = 128 // tw
    m_tiles = -(-wo // tw) * -(-ho // th)
    npad = -(-co // 16) * 16
    nts = [16, 32, 48, 64, 96, 128]
    n_tiles = -(-npad // 128)
    ni = next(i for i, nt in enumerate(nts) if nt * n_tiles >= npad)
    n_tiles = -(-npad // nts[ni])
    while m_tiles * n_tiles < SMS and ni > 0 and nts[ni - 1] >= 32:
        ni -= 1
        n_tiles = -(-npad // nts[ni])
    nt = nts[ni]
    bk = 64 if (mode != "per-tap" or ci % 64 == 0) else 32
    chunks = -(-ci // bk)
    if mode == "per-tap":
        per_cta = k * k * chunks * (128 + nt) * bk * 2
    else:
        per_cta = chunks * ((th + 2) * (tw + 2) * 128 + 9 * nt * 128)
    return m_tiles * n_tiles * per_cta / 1e6, m_tiles * n_tiles


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", type=int, default=-1)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--direct", action="store_true")
    ap.add_argument("--compare", action="store_true")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda")
    tot = 0.0
    for li, (name, ci, co, k, s, h, w) in enumerate(LAYERS):
        if args.only >= 0 and li != args.only:
            continue
        pad = 1 if k == 3 else 0
        ho, wo = F_.conv_out_size(h, w, k, s, pad)
        in_b, out_b = ci * h * w * 2, co * ho * wo * 2
        nbuf = max(2, min(16, int(260e6 // (in_b + out_b)) + 1))
        xs = [F_.empty_nhwc(1, ci, h, w, dev).normal_() for _ in range(nbuf)]
        ys = [F_.empty_nhwc(1, co, ho, wo, dev) for _ in range(nbuf)]
        wp = F_.pack_conv_weight(torch.randn(co, ci, k, k, device=dev) * 0.05, ci, co, k)
        sc, sh = torch.rand(co, device=dev) + 0.5, torch.randn(co, device=dev) * 0.1

        def timed_graph():
            for i in range(nbuf):
                F_.conv_fwd(xs[i], wp, co, k, s, pad, sc, sh, relu=True, out=ys[i], force_direct=args.direct)
            torch.cuda.synchronize()
            # capture `reps` back-to-back launches (rotating buffers) in a CUDA graph: device time without Python launch cost
            graph = torch.cuda.CUDAGraph()
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                with torch.cuda.graph(graph, stream=side):
                    for r in range(args.reps):
                        i = r % nbuf
                        F_.conv_fwd(xs[i], wp, co, k, s, pad, sc, sh, relu=True, out=ys[i], force_direct=args.direct)
            torch.cuda.synchronize()
            graph.replay()
            torch.cuda.synchronize()
            return graph

        def replay_us(graph):
            st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            st.record()
            graph.replay()
            en.record()
            en.synchronize()
            return st.elapsed_time(en) * 1000 / args.reps

        if args.compare:
            # FSB_CONV_TC2: 0 = per-tap, 1 = window; unset (the default) = window on grids of more CTAs than SMs
            modes = {"per-tap": 0, "window": 1} if k == 3 and s == 1 else {"per-tap": 0}
            graphs = {}
            for label, v in modes.items():
                _lib.set_option("FSB_CONV_TC2", v)
                graphs[label] = timed_graph()
            _lib.set_option("FSB_CONV_TC2", -1)
            ts = {label: [] for label in modes}
            for _ in range(args.rounds):
                for label in modes:
                    ts[label].append(replay_us(graphs[label]))
            med = {label: sorted(v)[len(v) // 2] for label, v in ts.items()}
            cols = "  ".join("%s %8.2f us %6.1f MB" % (label, med[label], l2_to_sm_mb(ci, co, k, s, h, w, label)[0])
                             for label in modes)
            ctas = l2_to_sm_mb(ci, co, k, s, h, w, "per-tap")[1]
            default = "window" if "window" in modes and ctas > SMS else "per-tap"
            print("%2d %-18s %3d->%3d k%d s%d %4dx%-4d %4d CTAs  %s  per-tap/window %.2fx  default %s" % (
                li, name, ci, co, k, s, h, w, ctas, cols, med["per-tap"] / med.get("window", med["per-tap"]), default))
            continue
        us = replay_us(timed_graph())
        flops = 2.0 * k * k * ci * co * ho * wo
        byts = in_b + out_b + k * k * ci * co * 2
        tot += us
        import ctypes as C
        d = _lib.ConvDesc(1, h, w, ci, co, k, s, pad, 1, 0, 0, ho, wo, ci, co, _lib.FSB_CONV_RELU | _lib.FSB_CONV_AFFINE)
        kid = _lib.lib().fsb_conv_kernel_id(C.byref(d), C.c_void_p(ys[0].data_ptr()), 0)
        print("%2d %-18s %3d->%3d k%d s%d %4dx%-4d %8.2f us  %7.1f TFLOP/s %7.1f GB/s  (roof %.1f us)  K%d" % (
            li, name, ci, co, k, s, h, w, us, flops / us / 1e6, byts / us / 1e3, max(flops / 989e12, byts / 3350e9) * 1e6, kid))   # H100 SXM data sheet
    print("total %.1f us" % tot)


if __name__ == "__main__":
    main()
