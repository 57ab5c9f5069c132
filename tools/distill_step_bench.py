#!/usr/bin/env python
"""BASELINE.json configs[3]: teacher -> student KL-distillation train step (train/train.py:219-271), synthetic data.
  teacher (arch_0, eval, no_grad) forward; student (arch_1, train) forward -> 3 full-resolution logits;
  loss = CE(l8) + 0.2 CE(l16) + 0.2 CE(l32) + KLDiv(log_softmax(student l8), softmax(teacher l8)); backward; SGD step.
--criterion ohem (default): the reference's ProbOhemCrossEntropy2d(thresh 0.7, min_kept = B*H*W/16) for the three CE terms;
--lazy 1 (default): N1 fused criteria (csrc/loss.cu) on the low-resolution logits; --lazy 0: label-resolution logits materialised
(478 MB each at the default size) and the criteria as torch ops on them (the round-1 path).
Prints one JSON line; --batch / --hw scale the per-GPU shard (default 12 x 3 x 512 x 1024)."""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import synth_weights_  # noqa: E402
from fasterseg_b200 import zoo  # noqa: E402


def measure(batch=12, hw=(512, 1024), steps=5, warmup=2, lazy=True, criterion="ohem", data=None):
    """data: optional callable -> (x, t) on the GPU, called once per step (a loader feeding the step); the fixed synthetic batch
    otherwise"""
    from fasterseg_b200.losses import ProbOhemCrossEntropy2d
    B, (H, W) = batch, hw
    teacher = zoo.build_network(0).cuda().eval()
    synth_weights_(teacher, 1)
    teacher.logits_dtype = torch.float16
    student = zoo.build_network(1, training=True).cuda().train()
    synth_weights_(student, 2)
    teacher.lazy_logits = bool(lazy)
    student.lazy_logits = bool(lazy)
    opt = torch.optim.SGD(student.parameters(), lr=0.01, momentum=0.9, weight_decay=5e-4)
    if criterion == "ohem":   # train/train.py:79-81
        ce = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=int(B * H * W // 16))
    else:
        ce = nn.CrossEntropyLoss(ignore_index=255)
    kl = nn.KLDivLoss(reduction="mean")
    x = torch.randn(B, 3, H, W, device="cuda")
    t = torch.randint(0, 19, (B, H, W), device="cuda")
    t[torch.rand(t.shape, device="cuda") < 0.05] = 255

    def step():
        nonlocal x, t
        if data is not None:
            x, t = data()
        opt.zero_grad()
        with torch.no_grad():
            tl = teacher(x).float()   # LazyLogits.float() is the identity
        l8, l16, l32 = student(x)
        # the reference's expression, verbatim (train/train.py:254-260); on LazyLogits it dispatches to the fused kernels
        loss = ce(l8, t) + 0.2 * ce(l16, t) + 0.2 * ce(l32, t) + kl(F.softmax(l8, dim=1).log(), F.softmax(tl, dim=1))
        loss.backward()
        opt.step()
        return loss

    torch.cuda.reset_peak_memory_stats()
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        loss = step()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    times.sort()
    dt = times[len(times) // 2]
    return {"metric": "distill_step_ms", "value": round(dt * 1e3, 1), "min_ms": round(times[0] * 1e3, 1), "unit": "ms/step",
            "batch": [B, 3, H, W], "images_per_s": round(B / dt, 1), "loss": float(loss.detach()), "criterion": criterion,
            "logits": "lazy: fused criteria on low-resolution logits (csrc/loss.cu)" if lazy else "materialised at label resolution",
            "mem_GB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=12)
    ap.add_argument("--hw", type=int, nargs=2, default=[512, 1024])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lazy", type=int, default=1)
    ap.add_argument("--criterion", default="ohem", choices=["ohem", "ce"])
    args = ap.parse_args()
    print(json.dumps(measure(args.batch, tuple(args.hw), args.steps, args.warmup, bool(args.lazy), args.criterion)))


if __name__ == "__main__":
    main()
