#!/usr/bin/env python
"""The architect's latency regulariser (search/architect.py:60-75: three weighted Network_Multi_Path.forward_latency((3, 1024, 2048))
calls for the student, then loss_latency.backward()) on its two paths: the Python walk (`_latency_walk`, scalar arithmetic on the
device of the arch parameters) and K14 (csrc/latency.cu, one launch forward and one backward).

  (a) the latency term alone: the three weighted calls + backward, walk vs kernel;
  (b) the whole first-order search step of configs[4] (architect step on a 2 x 3 x 224 x 448 batch with latency_weight = [0, 1e-2]
      for the student, then the weight step), with the latency term on the walk, on the kernel, and off.

The paths alternate, `--runs` runs each, every run timed with a synchronised host clock.  The table is latency_lookup_table.npy from
the working directory if it covers every reachable key, else the synthetic table of the tests; the JSON says which.  The card
name, power limit and SM clock are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fasterseg_b200 import operations  # noqa: E402
from fasterseg_b200 import supernet_latency as SL  # noqa: E402
from tools import search_step_bench as ssb  # noqa: E402
from tools.latency_variant_bench import gpu_line  # noqa: E402

SIZE = (3, 1024, 2048)
CALLS = ((1. / 500, (True, False, False)), (497. / 500, (False, True, False)), (2. / 500, (False, False, True)))
LATENCY_WEIGHT = [0, 1e-2]


def choose_table(model):
    """'latency_lookup_table.npy' if it has every key the student's three calls can reach, else the synthetic table"""
    from oracle.make_golden_decode import SyntheticLatencyTable
    table = operations.latency_lookup_table
    model.arch_idx, model.prun_mode = 1, None
    try:
        for _, flags in CALLS:
            SL.build_plan(model, SIZE, *flags, model._current_mode() if flags[2] else "max", table)
        return "latency_lookup_table.npy (%d entries)" % len(table)
    except SL.Missing:
        operations.latency_lookup_table = SyntheticLatencyTable()
        return "synthetic (oracle/make_golden_decode.py::SyntheticLatencyTable)"


def loss_latency(model):
    """architect._backward_step's latency term"""
    total = 0
    model.prun_mode = None
    for idx, w in enumerate(LATENCY_WEIGHT):
        model.arch_idx = idx
        if w > 0:
            lat = 0
            for r, flags in CALLS:
                lat = lat + r * model.forward_latency(SIZE, *flags)
            total = total + lat * w
    return total


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5, help="latency terms per run in (a)")
    ap.add_argument("--steps", type=int, default=3, help="search steps per run in (b)")
    ap.add_argument("--layers", type=int, default=16)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "architect_step_bench measures on the GPU"
    from fasterseg_b200 import optim as FO
    FO.install()
    torch.manual_seed(12345)
    model = ssb.build(args.layers)
    table = choose_table(model)
    arch_opts = [torch.optim.Adam(ps, lr=3e-4, betas=(0.5, 0.999)) for ps in model._arch_parameters]
    opt = torch.optim.SGD(ssb.weight_params(model), lr=0.02, momentum=0.9, weight_decay=5e-4)
    B, H, W = 2, 224, 448
    g = torch.Generator().manual_seed(977)
    x = torch.randn(B, 3, H, W, generator=g).cuda()
    t = torch.randint(0, 19, (B, H // 8, W // 8), generator=g)
    t[torch.rand(t.shape, generator=g) < 0.05] = 255
    t = t.cuda()
    from fasterseg_b200.losses import ProbOhemCrossEntropy2d
    model._criterion = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=int(B * (H // 8) * (W // 8) // 16))

    def term():
        for o in arch_opts:
            o.zero_grad()
        loss_latency(model).backward()

    def search_step(with_latency):
        for o in arch_opts:
            o.zero_grad()
        loss = model._loss(x, t, "dir")
        lat = loss_latency(model) if with_latency else 0
        loss.backward()
        if lat != 0:
            lat.backward()
        for o in arch_opts:
            o.step()
        opt.zero_grad()
        loss = model._loss(x, t, "dir")
        loss.backward()
        nn.utils.clip_grad_norm_(model.parameters(), 5)
        opt.step()

    paths = {"walk": False, "kernel": True}
    for kernel in paths.values():          # warm-up: plans, captured passes, allocator
        SL.ENABLED = kernel
        term()
        search_step(True)
    search_step(False)
    term_ms = {k: [] for k in paths}
    step_ms = {k: [] for k in list(paths) + ["off"]}
    for _ in range(args.runs):
        for name, kernel in paths.items():
            SL.ENABLED = kernel
            term_ms[name].append(round(timed(term, args.reps), 3))
        for name, kernel in list(paths.items()) + [("off", True)]:
            SL.ENABLED = kernel
            step_ms[name].append(round(timed(lambda: search_step(name != "off"), args.steps), 2))
    SL.ENABLED = True
    FO.uninstall()
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    print(json.dumps({
        "gpu": gpu_line(), "table": table, "layers": args.layers, "size": list(SIZE),
        "latency_term_ms": term_ms, "latency_term_median_ms": {k: med(v) for k, v in term_ms.items()},
        "latency_term_speedup": round(med(term_ms["walk"]) / med(term_ms["kernel"]), 1),
        "search_step_ms": step_ms, "search_step_median_ms": {k: med(v) for k, v in step_ms.items()},
        "batch": [B, 3, H, W], "runs": args.runs, "reps": args.reps, "steps": args.steps}))


if __name__ == "__main__":
    main()
