#!/usr/bin/env python
"""Secondary metric of BASELINE.json: supernet step time.
  pretrain step (configs[2]): search/train_search.py:246-250 with C.pretrain=True -- _loss = 4 forwards (max, min, random,
                              random) + backward + clip_grad_norm_(5) + SGD step, batch 3 x 3 x 256 x 512 per GPU
  search step   (configs[4]): architect.step (first-order: _loss on the search batch + Adam on arch params, architect.py:42-76,
                              latency term omitted; tools/architect_step_bench.py times the step with the student's latency
                              term on the walk and on K14) followed by the weight step, batch 2 x 3 x 224 x 448 per GPU
Synthetic data per SURVEY 8(d).  Prints one JSON line.
Data parallel: launch with torchrun (--nproc-per-node N): per-rank shard of the same per-GPU batch (weak scaling), SyncBN
statistics + end-of-backward gradient all-reduce (fasterseg_b200/parallel.py); the time is the max over ranks."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import synth_weights_  # noqa: E402
from fasterseg_b200 import parallel  # noqa: E402
from fasterseg_b200.model_search import Network_Multi_Path  # noqa: E402

WML = [4. / 12, 6. / 12, 8. / 12, 10. / 12, 1.]


def build(layers, criterion="ohem"):
    # the reference's search criterion: ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept = batch * H * W / 8^2 / 16
    # (search/train_search.py:104-105 with config_search.py:47,84-86); "ce" = plain cross entropy (round-1 numbers)
    if criterion == "ohem":
        from fasterseg_b200.losses import ProbOhemCrossEntropy2d
        crit = None   # needs the batch geometry: set by measure()
    else:
        crit = nn.CrossEntropyLoss(ignore_index=255)
    m = Network_Multi_Path(19, layers, crit, Fch=12, width_mult_list=WML, prun_modes=['max', 'arch_ratio'],
                           stem_head_width=[(1, 1), (8. / 12, 8. / 12)])
    synth_weights_(m)
    with torch.no_grad():
        for ps in m._arch_parameters:
            for p in ps:
                p.fill_(1e-3)
    return m.cuda().train()


def weight_params(m):
    ps = []
    for mod in (m.stem, m.cells, m.refine32, m.refine16, m.head0, m.head1, m.head2, m.head02, m.head12):
        ps += list(mod.parameters())
    return ps


def measure(mode="pretrain", layers=16, steps=3, warmup=1, rank=0, world=1, tape=None, graph=None, criterion="ohem", flat_optim=True):
    """Time `steps` optimizer steps; returns the result dict (identical on every rank).
    tape: None = whatever FSB_TAPE says; True / False = force the one-node-per-forward autograd mode of the EAGER path.
    graph: None = default (captured passes, fasterseg_b200/graphed.py); False = eager per-unit path."""
    from fasterseg_b200 import autograd as AG
    from fasterseg_b200 import optim as FO
    if tape is not None:
        AG.TAPE_ENABLED = bool(tape)
    # what fasterseg_b200.launch does for the unmodified drivers: torch.optim.SGD / nn.utils.clip_grad_norm_ become flat-aware
    # (csrc/optim.cu); the step below keeps the reference's own lines (search/train_search.py:246-250)
    if flat_optim:
        FO.install()
    else:
        FO.uninstall()
    args = argparse.Namespace(mode=mode, layers=layers, steps=steps, warmup=warmup)
    parallel.seed_all_ranks_identically(12345)   # identical weights + lock-step width sampling / gumbel noise on every rank
    model = build(args.layers, criterion)
    if graph is not None:
        model.__dict__["_fsb_graph_mode"] = None if graph else False
    params = weight_params(model)
    opt = torch.optim.SGD(params, lr=0.02, momentum=0.9, weight_decay=5e-4)
    arch_opts = [torch.optim.Adam(ps, lr=3e-4, betas=(0.5, 0.999)) for ps in model._arch_parameters]
    if args.mode == "pretrain":
        B, H, W = 3, 256, 512
    else:
        B, H, W = 2, 224, 448
    g = torch.Generator().manual_seed(977 + rank)  # private per-rank data stream (different shard on every rank)
    x = torch.randn(B, 3, H, W, generator=g).cuda()
    t = torch.randint(0, 19, (B, H // 8, W // 8), generator=g)
    t[torch.rand(t.shape, generator=g) < 0.05] = 255
    t = t.cuda()
    if criterion == "ohem":
        from fasterseg_b200.losses import ProbOhemCrossEntropy2d
        model._criterion = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=int(B * (H // 8) * (W // 8) // 16))
    from fasterseg_b200 import engine
    # captured passes with the library-owned exchange all-reduce their flat gradient buffer themselves (graphed.py); the
    # hook-based GradSync is for the eager per-unit path
    graph_dp = world > 1 and engine.dp_native() and graph is not False
    sync = parallel.GradSync(list(model.parameters())).install() if (world > 1 and not graph_dp) else None

    def step():
        if args.mode == "search":
            for o in arch_opts:
                o.zero_grad()
            loss = model._loss(x, t, "dir")          # architect._backward_step on the search batch
            loss.backward()
            for o in arch_opts:
                o.step()
        opt.zero_grad()
        loss = model._loss(x, t, True if args.mode == "pretrain" else "dir")
        loss.backward()
        nn.utils.clip_grad_norm_(model.parameters(), 5)
        opt.step()
        return loss

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        loss = step()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    times.sort()
    stat = torch.tensor([times[len(times) // 2], times[0], times[-1]], device="cuda", dtype=torch.float64)
    if world > 1:
        torch.distributed.all_reduce(stat, op=torch.distributed.ReduceOp.MAX)   # a step ends when the slowest rank ends
    dt, tmin, tmax = (float(v) for v in stat)  # median: the step is host-bound and shares the host with other tenants
    if sync:
        sync.uninstall()
    FO.uninstall()
    return {"metric": "supernet_%s_step_ms" % args.mode, "value": round(dt * 1e3, 1), "min_ms": round(tmin * 1e3, 1),
            "max_ms": round(tmax * 1e3, 1), "unit": "ms/step", "n_gpus": world, "layers": args.layers, "steps": args.steps,
            "warmup": args.warmup, "criterion": criterion,
            "step_tail": "flat clip_grad_norm_ + SGD kernels (%d flat steps)" % getattr(opt, "flat_steps", 0) if flat_optim else "torch clip_grad_norm_ + torch.optim.SGD",
            "autograd": "captured passes (CUDA graphs)" if model.__dict__.get("_fsb_graph_runner") is not None else ("tape" if AG.TAPE_ENABLED else "per-unit"), "batch_per_gpu": [B, 3, H, W], "images_per_s": round(B * world / dt, 2),
            "grad_syncs": sync.syncs if sync else 0, "loss": float(loss.detach()),
            "params_M": round(sum(p.numel() for p in model.parameters()) / 1e6, 2),
            "mem_GB": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--mode", default="pretrain", choices=["pretrain", "search"])
    ap.add_argument("--graph", type=int, default=1, help="1 = captured passes (default), 0 = eager per-unit path")
    ap.add_argument("--criterion", default="ohem", choices=["ohem", "ce"])
    ap.add_argument("--flat-optim", type=int, default=1, help="1 = flat clip + SGD kernels (default, what the launcher installs), 0 = torch's")
    args = ap.parse_args()
    rank, local_rank, world = parallel.init_from_env()
    torch.cuda.set_device(local_rank)
    res = measure(args.mode, args.layers, args.steps, args.warmup, rank, world, graph=bool(args.graph), criterion=args.criterion,
                  flat_optim=bool(args.flat_optim))
    if rank == 0:
        print(json.dumps(res))
    if world > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
