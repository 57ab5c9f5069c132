"""Census of the conv backward geometries the training steps run: every call of F_.conv_dgrad, F_.conv_wgrad and the fused
unit's backward (F_.conv_bn_act_train_bwd / _sel), de-duplicated, recorded on the CPU stand-in backend (tests/cpu_backend.py).

The runs are the supernet `_loss` backward of tools/search_step_bench.build(16) -- pretrain (max, min and two random-width passes)
and search (one pass per architecture, max and min) -- and the distillation student (zoo.build_network(1, training=True)).  They
are recorded at batch 1: the batch only changes the number of pixel tiles and chunks, so the GPU test (tests/test_conv_bwd_gpu.py)
runs each geometry at the driver's batch, which the census keeps beside each run.

The supernet runs are the eager `_loss` (the CPU stand-ins run no captured passes): every pass at its own widths, so sliced
master weights and the sampled widths are in the census.  On the GPU the step runs as captured passes (fasterseg_b200/graphed.py)
with every unit at its maximum width.  Recorded the same way with the captured passes forced (`_fsb_graph_mode = True`, run
eagerly on the stand-ins), every one of those calls is already in the census, so the eager recording is the superset.

    python -m tests.conv_bwd_census        # rewrite tests/golden/conv_bwd_census.json
"""
import json
import os

import numpy as np
import torch

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_bwd_census.json")
FIELDS = ("op", "N", "H", "W", "Cin", "Cout", "k", "stride", "pad", "dil", "off_h", "off_w", "x_cstride", "dy_cstride",
          "dx_cstride", "w_stride_o", "w_stride_i", "accumulate", "gscale")
# run -> (the driver's batch and image size, the batch the census records at)
RUNS = {
    "pretrain": dict(batch=3, hw=[256, 512], recorded_batch=1),
    "search": dict(batch=2, hw=[224, 448], recorded_batch=1),
    "distill": dict(batch=12, hw=[512, 1024], recorded_batch=1),
}


def _cpad(c):
    return (c + 7) // 8 * 8


class Recorder:
    """Wraps the four functional entry points that reach fsb_conv_dgrad / fsb_conv_wgrad and records each kernel call."""
    NAMES = ("conv_dgrad", "conv_wgrad", "conv_bn_act_train_bwd", "conv_bn_act_train_bwd_sel")

    def __init__(self, F_):
        self.F_ = F_
        self.seen = set()
        self.saved = {}

    def add(self, **kw):
        self.seen.add(tuple(kw[f] for f in FIELDS))

    def __enter__(self):
        F_ = self.F_
        self.saved = {n: getattr(F_, n) for n in self.NAMES}
        s = self.saved
        cs = lambda t: F_.nhwc_info(t)[4]

        def conv_dgrad(dy, w, x_shape, Cin, Cout, ksize, stride, pad, off=(0, 0), wpacked_t=None, force_direct=False):
            N, _, H, W = x_shape
            self.add(op="dgrad", N=N, H=H, W=W, Cin=Cin, Cout=Cout, k=ksize, stride=stride, pad=pad, dil=1, off_h=off[0], off_w=off[1],
                     x_cstride=0, dy_cstride=cs(dy), dx_cstride=_cpad(Cin), w_stride_o=w.stride(0), w_stride_i=w.stride(1),
                     accumulate=0, gscale=0.0)
            return s["conv_dgrad"](dy, w, x_shape, Cin, Cout, ksize, stride, pad, off=off, wpacked_t=wpacked_t, force_direct=force_direct)

        def conv_wgrad(x, dy, w_like, Cin, Cout, ksize, stride, pad, gscale, off=(0, 0), accumulate_into=None, force_direct=False):
            N, _, H, W, xcs = F_.nhwc_info(x)
            # without accumulate_into the wrapper allocates a contiguous gradient of w_like's shape
            so, si = ((accumulate_into.stride(0), accumulate_into.stride(1)) if accumulate_into is not None else
                      (w_like.shape[1] * ksize * ksize, ksize * ksize))
            self.add(op="wgrad", N=N, H=H, W=W, Cin=Cin, Cout=Cout, k=ksize, stride=stride, pad=pad, dil=1, off_h=off[0], off_w=off[1],
                     x_cstride=xcs, dy_cstride=cs(dy), dx_cstride=0, w_stride_o=so, w_stride_i=si,
                     accumulate=int(accumulate_into is not None), gscale=float(gscale))
            return s["conv_wgrad"](x, dy, w_like, Cin, Cout, ksize, stride, pad, gscale, off=off, accumulate_into=accumulate_into,
                                   force_direct=force_direct)

        def unit(d, x, w, need_dx, dw_accum, gscale):
            g = dict(N=d.N, H=d.H, W=d.W, Cin=d.Cin, Cout=d.Cout, k=d.ksize, stride=d.stride, pad=d.pad, dil=d.dil, off_h=d.off_h,
                     off_w=d.off_w, dy_cstride=_cpad(d.Cout), w_stride_o=w.stride(0), w_stride_i=w.stride(1))
            if need_dx:
                self.add(op="dgrad", x_cstride=0, dx_cstride=_cpad(d.Cin), accumulate=0, gscale=0.0, **g)
            if dw_accum is not None:
                self.add(op="wgrad", x_cstride=cs(x), dx_cstride=0, accumulate=1, gscale=float(gscale), **g)

        def conv_bn_act_train_bwd(d, x, dy, y, raw, vec, gamma, relu, wpacked_t, w, need_dx, dw_accum, gscale, sel=None, width_idx=None):
            unit(d, x, w, need_dx, dw_accum, gscale)
            return s["conv_bn_act_train_bwd"](d, x, dy, y, raw, vec, gamma, relu, wpacked_t, w, need_dx, dw_accum, gscale, sel=sel,
                                              width_idx=width_idx)

        def conv_bn_act_train_bwd_sel(d, x, dy, y, raw, vec, sel, relu, wpacked_t, w, need_dx, dw_accum, gscale):
            unit(d, x, w, need_dx, dw_accum, gscale)
            return s["conv_bn_act_train_bwd_sel"](d, x, dy, y, raw, vec, sel, relu, wpacked_t, w, need_dx, dw_accum, gscale)

        for n in self.NAMES:
            setattr(F_, n, locals()[n])
        return self

    def __exit__(self, *exc):
        for n, fn in self.saved.items():
            setattr(self.F_, n, fn)

    def entries(self):
        return [list(t) for t in sorted(self.seen)]


def _supernet():
    """tools/search_step_bench.build(16) without the move to the device"""
    from bench import synth_weights_
    from fasterseg_b200.model_search import Network_Multi_Path
    from fasterseg_b200.losses import ProbOhemCrossEntropy2d
    from tools.search_step_bench import WML
    m = Network_Multi_Path(19, 16, None, Fch=12, width_mult_list=WML, prun_modes=['max', 'arch_ratio'],
                           stem_head_width=[(1, 1), (8. / 12, 8. / 12)])
    synth_weights_(m)
    with torch.no_grad():
        for ps in m._arch_parameters:
            for p in ps:
                p.fill_(1e-3)
    m._criterion = ProbOhemCrossEntropy2d(ignore_label=255, thresh=0.7, min_kept=1)
    return m.train()


def _record_supernet(F_, run, pretrain):
    from fasterseg_b200 import parallel
    parallel.seed_all_ranks_identically(12345)
    model = _supernet()
    B, (H, W) = RUNS[run]["recorded_batch"], RUNS[run]["hw"]
    g = torch.Generator().manual_seed(977)
    x = torch.randn(B, 3, H, W, generator=g)
    t = torch.randint(0, 19, (B, H // 8, W // 8), generator=g)
    with Recorder(F_) as rec:
        model._loss(x, t, pretrain).backward()
    return rec.entries()


def _record_distill(F_):
    from bench import synth_weights_
    from fasterseg_b200 import zoo
    torch.manual_seed(0)
    np.random.seed(0)
    student = zoo.build_network(1, training=True).train()
    synth_weights_(student, 2)
    B, (H, W) = RUNS["distill"]["recorded_batch"], RUNS["distill"]["hw"]
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(5))
    with Recorder(F_) as rec:
        outs = student(x)
        sum(o.float().sum() for o in outs).backward()
    return rec.entries()


def generate():
    """-> the census dict; runs the three networks on the CPU stand-ins"""
    from fasterseg_b200 import functional as F_
    from tests import cpu_backend
    runs = {}
    with cpu_backend.installed():
        runs["pretrain"] = _record_supernet(F_, "pretrain", True)
        runs["search"] = _record_supernet(F_, "search", "dir")
        runs["distill"] = _record_distill(F_)
    return {"fields": list(FIELDS), "runs": {r: dict(RUNS[r], entries=runs[r]) for r in RUNS}}


def dumps(census):
    """one entry (a row of FIELDS) per line"""
    out = ['{"fields": %s,' % json.dumps(census["fields"]), ' "runs": {']
    runs = list(census["runs"].items())
    for i, (r, v) in enumerate(runs):
        head = {k: v[k] for k in sorted(v) if k != "entries"}
        out.append('  %s: %s, "entries": [' % (json.dumps(r), json.dumps(head)[:-1]))
        out.append(",\n".join("   " + json.dumps(e) for e in v["entries"]))
        out.append("  ]}" + ("," if i + 1 < len(runs) else ""))
    out.append(" }}")
    return "\n".join(out) + "\n"


def load():
    with open(PATH) as f:
        return json.load(f)


def geometries(census=None):
    """-> [dict(FIELDS..., run=...)] with N = the driver's batch, de-duplicated over the runs (first run wins)"""
    census = census or load()
    seen, out = set(), []
    for r, v in census["runs"].items():
        for row in v["entries"]:
            g = dict(zip(census["fields"], row))
            g["N"] = v["batch"]
            key = tuple(g[f] for f in FIELDS)
            if key not in seen:
                seen.add(key)
                out.append(dict(g, run=r))
    return out


if __name__ == "__main__":
    c = generate()
    with open(PATH, "w") as f:
        f.write(dumps(c))
    print({r: len(v["entries"]) for r, v in c["runs"].items()})
