"""Census of the forward conv launches the networks run: every call of F_.conv_fwd, the fused training unit's conv
(F_.conv_bn_act_train_fwd / _sel: FSB_CONV_STATS | FSB_CONV_OUT_F32 into its fp32 `raw`) and the RGB stems (F_.stem_conv_nchw,
F_.stem_conv_u8hwc), de-duplicated, recorded on the CPU stand-in backend (tests/cpu_backend.py).  F_.pack_conv_weight is
recorded too, for the strides of the master weight each packed buffer was cut from (slimmable slices).

The runs are the student frame of bench.py (zoo.build_network(1), eval, 1 x 1024 x 2048), the latency/ deployment network
(variant="latency", eval, same frame), the distillation teacher (zoo.build_network(0), eval) and student
(zoo.build_network(1, training=True), train forward) of tools/distill_step_bench.py, and the supernet `_loss` forward of
pretrain and search (the runs of tests/conv_bwd_census.py, whose builders this module reuses).  They are recorded at batch 1:
the batch only changes the number of pixel tiles, so the GPU test (tests/test_conv_fwd_gpu.py) runs each geometry at the
driver's batch, which the census keeps beside each run.  The inference networks have no data-dependent control flow, so they
are recorded with shape-only stand-ins (cpu_backend.SHAPES_ONLY): the calls are the same and the 1024 x 2048 frame costs no
CPU arithmetic.

On CPU tensors the frame's stem never takes F_.stem_fused (it needs a CUDA input): it is recorded as the stem conv plus the
conv_fwd of stem.1.conv1, which is the geometry the GPU test runs stem_fused at.

The supernet runs are recorded twice, eagerly (every pass at its own widths: sliced master weights and the sampled widths) and
with the captured passes forced (`_fsb_graph_mode = True`, run eagerly on the stand-ins: every unit at its maximum width, as
the GPU step runs them), and the census keeps the union.  Every call of the captured recording is already in the eager one, so
the union is the eager recording.  A captured pass also runs its backward; its convs and conv gradients run shape-only, which
changes no call (the widths are sampled before the pass).

    python -m tests.conv_fwd_census        # rewrite tests/golden/conv_fwd_census.json
"""
import contextlib
import json
import os

import numpy as np
import torch

from tests import conv_bwd_census as BC

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_fwd_census.json")
# op: conv (F_.conv_fwd), unit (the fused training unit's conv), stem_nchw / stem_u8hwc (the RGB stems; Cin = 3, k 3, s 2, p 1).
# H, W: the descriptor's (the half size with X_DOWN2); x_coff / y_coff: channel offset of the x / y view inside its buffer;
# scale / shift: whether each is passed; stats_C, stats_off: 0 without FSB_CONV_STATS
FIELDS = ("op", "N", "H", "W", "Cin", "Cout", "k", "stride", "pad", "dil", "off_h", "off_w", "x_cstride", "y_cstride", "x_coff",
          "y_coff", "flags", "scale", "shift", "stats_C", "stats_off", "w_stride_o", "w_stride_i")
# run -> the driver's batch and image size, the batch the census records at
RUNS = {
    "frame": dict(batch=1, hw=[1024, 2048], recorded_batch=1),
    "latency": dict(batch=1, hw=[1024, 2048], recorded_batch=1),
    "teacher": dict(batch=12, hw=[512, 1024], recorded_batch=1),
    "distill": dict(batch=12, hw=[512, 1024], recorded_batch=1),
    "pretrain": dict(BC.RUNS["pretrain"]),
    "search": dict(BC.RUNS["search"]),
}


def _coff(t):
    """channel offset of an NHWC view inside its buffer"""
    cs = t.stride(3) if t.shape[3] > 1 else t.stride(2)
    return t.storage_offset() % cs if cs else 0


class Recorder:
    """Wraps the functional entry points that reach fsb_conv_fwd, the fused unit's conv and the stems, and records each call"""
    NAMES = ("pack_conv_weight", "conv_fwd", "conv_bn_act_train_fwd", "conv_bn_act_train_fwd_sel", "stem_conv_nchw",
             "stem_conv_u8hwc")

    def __init__(self, F_):
        self.F_ = F_
        self.seen = set()
        self.saved = {}
        self.wstrides = {}      # packed buffer's data_ptr -> strides of the master weight it was packed from

    def add(self, **kw):
        self.seen.add(tuple(kw[f] for f in FIELDS))

    def _ws(self, wpacked):
        return self.wstrides[wpacked.data_ptr()]

    def __enter__(self):
        F_ = self.F_
        self.saved = {n: getattr(F_, n) for n in self.NAMES}
        s = self.saved

        def pack_conv_weight(w, Cin, Cout, ksize, out=None):
            packed = s["pack_conv_weight"](w, Cin, Cout, ksize, out=out)
            self.wstrides[packed.data_ptr()] = (w.stride(0), w.stride(1))
            return packed

        def conv_fwd(x, wpacked, Cout, ksize, stride, pad, scale=None, shift=None, relu=False, out=None, off=(0, 0), stats=None,
                     force_direct=False, out_f32=False, stats_off=0, down2=False, up2=False):
            y = s["conv_fwd"](x, wpacked, Cout, ksize, stride, pad, scale=scale, shift=shift, relu=relu, out=out, off=off,
                              stats=stats, force_direct=force_direct, out_f32=out_f32, stats_off=stats_off, down2=down2, up2=up2)
            N, Cin, H, W, xcs = F_.nhwc_info(x)
            if down2:
                H, W = H // 2, W // 2
            ycs = F_.nhwc_info(y, y.dtype)[4]
            flags = ((1 if relu else 0) | (2 if (scale is not None or shift is not None) else 0) | (4 if force_direct else 0) |
                     (8 if stats is not None else 0) | (16 if out_f32 else 0) | (64 if down2 else 0) | (128 if up2 else 0))
            so, si = self._ws(wpacked)
            self.add(op="conv", N=N, H=H, W=W, Cin=Cin, Cout=Cout, k=ksize, stride=stride, pad=pad, dil=1, off_h=off[0],
                     off_w=off[1], x_cstride=xcs, y_cstride=ycs, x_coff=_coff(x), y_coff=_coff(y), flags=flags,
                     scale=int(scale is not None), shift=int(shift is not None),
                     stats_C=stats.shape[1] // 2 if stats is not None else 0, stats_off=int(stats_off) if stats is not None else 0,
                     w_stride_o=so, w_stride_i=si)
            return y

        def unit(x, wpacked, Cout, ksize, stride, pad, off):
            N, Cin, H, W, xcs = F_.nhwc_info(x)
            so, si = self._ws(wpacked)
            self.add(op="unit", N=N, H=H, W=W, Cin=Cin, Cout=Cout, k=ksize, stride=stride, pad=pad, dil=1, off_h=off[0], off_w=off[1],
                     x_cstride=xcs, y_cstride=BC._cpad(Cout), x_coff=_coff(x), y_coff=0, flags=8 | 16, scale=0, shift=0,
                     stats_C=Cout, stats_off=0, w_stride_o=so, w_stride_i=si)

        def conv_bn_act_train_fwd(x, wpacked, Cout, ksize, stride, pad, off, gamma, beta, eps, momentum, running_mean, running_var,
                                  num_batches_tracked, relu, sel=None, width_idx=None):
            unit(x, wpacked, Cout, ksize, stride, pad, off)
            return s["conv_bn_act_train_fwd"](x, wpacked, Cout, ksize, stride, pad, off, gamma, beta, eps, momentum, running_mean,
                                              running_var, num_batches_tracked, relu, sel=sel, width_idx=width_idx)

        def conv_bn_act_train_fwd_sel(x, wpacked, Cout, ksize, stride, pad, off, sel, relu):
            unit(x, wpacked, Cout, ksize, stride, pad, off)
            return s["conv_bn_act_train_fwd_sel"](x, wpacked, Cout, ksize, stride, pad, off, sel, relu)

        def stem(op, x, w, scale, shift, relu, y):
            N, _, H, W = x.shape
            self.add(op=op, N=N, H=H, W=W, Cin=3, Cout=w.shape[0], k=3, stride=2, pad=1, dil=1, off_h=0, off_w=0, x_cstride=0,
                     y_cstride=F_.nhwc_info(y)[4], x_coff=0, y_coff=_coff(y), flags=(1 if relu else 0) | (2 if scale is not None else 0),
                     scale=int(scale is not None), shift=int(shift is not None), stats_C=0, stats_off=0, w_stride_o=w.stride(0),
                     w_stride_i=w.stride(1))

        def stem_conv_nchw(x, w, scale, shift, relu=True, out=None):
            y = s["stem_conv_nchw"](x, w, scale, shift, relu=relu, out=out)
            stem("stem_nchw", x, w, scale, shift, relu, y)
            return y

        def stem_conv_u8hwc(x_u8, lut, w, scale, shift, relu=True, out=None):
            y = s["stem_conv_u8hwc"](x_u8, lut, w, scale, shift, relu=relu, out=out)
            stem("stem_u8hwc", x_u8, w, scale, shift, relu, y)
            return y

        for n in self.NAMES:
            setattr(F_, n, locals()[n])
        return self

    def __exit__(self, *exc):
        for n, fn in self.saved.items():
            setattr(self.F_, n, fn)

    def entries(self):
        return [list(t) for t in sorted(self.seen)]


def _record_inference(F_, run):
    from bench import synth_weights_
    from fasterseg_b200 import zoo
    from tests import cpu_backend
    torch.manual_seed(0)
    np.random.seed(0)
    arch, variant, seed = {"frame": (1, "train", 12345), "latency": (1, "latency", 12345), "teacher": (0, "train", 1)}[run]
    model = zoo.build_network(arch, variant=variant).eval()
    synth_weights_(model, seed)
    model.logits_dtype = torch.float16
    B, (H, W) = RUNS[run]["recorded_batch"], RUNS[run]["hw"]
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(5))
    with Recorder(F_) as rec, cpu_backend.shapes_only(), torch.no_grad():
        model(x)
    return rec.entries()


def _record_supernet(F_, run, pretrain):
    from fasterseg_b200 import parallel
    from tests import cpu_backend
    out = set()
    for graph in (None, True):
        parallel.seed_all_ranks_identically(12345)
        model = BC._supernet()
        if graph:
            model.__dict__["_fsb_graph_mode"] = True
        B, (H, W) = RUNS[run]["recorded_batch"], RUNS[run]["hw"]
        g = torch.Generator().manual_seed(977)
        x = torch.randn(B, 3, H, W, generator=g)
        t = torch.randint(0, 19, (B, H // 8, W // 8), generator=g)
        with Recorder(F_) as rec, (cpu_backend.shapes_only() if graph else contextlib.nullcontext()):
            model._loss(x, t, pretrain)
        out |= {tuple(e) for e in rec.entries()}
    return [list(e) for e in sorted(out)]


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
        student(x)
    return rec.entries()


def generate():
    """-> the census dict; runs the six networks on the CPU stand-ins"""
    from fasterseg_b200 import functional as F_
    from tests import cpu_backend
    runs = {}
    with cpu_backend.installed():
        for r in ("frame", "latency", "teacher"):
            runs[r] = _record_inference(F_, r)
        runs["distill"] = _record_distill(F_)
        runs["pretrain"] = _record_supernet(F_, "pretrain", True)
        runs["search"] = _record_supernet(F_, "search", "dir")
    return {"fields": list(FIELDS), "runs": {r: dict(RUNS[r], entries=runs[r]) for r in RUNS}}


dumps = BC.dumps


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
