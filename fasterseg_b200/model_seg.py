"""Derived (teacher / student) network -- drop-in for the reference's train/model_seg.py.

Same public surface as the reference (train/model_seg.py:138-408): `MixedOp` / `Cell` / `Network_Multi_Path_Infer` with the
same constructor arguments, `build_structure`, `num_filters`, `forward`, `forward_latency`, attribute names (`ops0.. path2..
branch_groups, cells, ch_16 ...`) and every parameter name (`stem.0.conv.0.weight`, `cells.3-1._op._op.conv1.weight`,
`arms32.0...`, `ffm...`, `heads8...`); the decoder functions it exports live in `decode.py`.

Organisation (ours): `build_structure` compiles the decoded branches into a flat *schedule* -- one `_CellStep` per distinct
cell in execution order (which branches share it, where a stream fork happens) plus one `_Tail` per branch (its
arm / refine chain towards the 1/8 feature) -- and `forward`, `predict_labels` and `forward_latency` are interpreters of
that schedule.  GPU side: NHWC fp16 activations, each conv+BN+ReLU one fused wgmma kernel, the torch.cat call sites
(:307,312,319,331) replaced by producers writing into channel slices of one buffer, independent branches on their own CUDA
streams inside one CUDA graph, the final x8 upsample as one kernel writing NCHW logits (or, via `predict_labels`, a fused
upsample+argmax that never materialises them).
"""
from collections import OrderedDict, namedtuple

import numpy as np
import torch
import torch.nn as nn

from . import decode
from . import engine
from . import functional as F_
from .decode import (alphas2ops_path_width, betas2path, downs2path, network_metas, path2downs, path2widths,  # noqa: F401
                     softmax)
from .genotypes import PRIMITIVES
from .operations import *  # noqa: F401,F403  (the reference does `from operations import *`)
from .operations import OPS, BasicResidual2x, ConvNorm, _Residual
from .seg_oprs import FeatureFusion, Head

BatchNorm2d = nn.BatchNorm2d

SCALES = (8, 16, 32)                      # feature strides the decoder tails tap
_CellStep = namedtuple("_CellStep", "key layer lead members fork")   # one distinct cell of the trunk
_Tail = namedtuple("_Tail", "branch last")                          # how branch b reaches the 1/8 fusion input
# Inference outputs a step's producer writes for later kernels (see Network_Multi_Path_Infer._trunk): `half` = steps whose output a
# zoomed op reads, made by a kernel that also stores the output's bilinear /2; `reads_half` = the zoomed steps that take that /2;
# `skip` = step -> (branch, link) of the one refine whose concat buffer receives the step's output as its skip feature;
# `shapes` = each step's output shape.
_ResizePlan = namedtuple("_ResizePlan", "half reads_half skip shapes")


class MixedOp(nn.Module):
    """Single selected primitive (non-slimmable, fixed channels)."""

    def __init__(self, C_in, C_out, op_idx, stride=1):
        super(MixedOp, self).__init__()
        self._op = OPS[PRIMITIVES[op_idx]](C_in, C_out, stride, slimmable=False, width_mult_list=[1.])

    def forward(self, x, out=None, **fused):
        """fused: out_half / x_half of the residual primitives (operations._Residual.forward), passed on when given"""
        fused = {k: v for k, v in fused.items() if v is not None}
        if out is not None:
            fused["out"] = out
        return self._op(x, **fused)

    def forward_latency(self, size):
        latency, size_out = self._op.forward_latency(size)
        return latency, size_out


class Cell(nn.Module):
    def __init__(self, op_idx, C_in, C_out, down):
        super(Cell, self).__init__()
        self._C_in, self._C_out, self._down = C_in, C_out, down
        self._op = MixedOp(C_in, C_out, op_idx, stride=2 if down else 1)

    def forward(self, input, out=None, **fused):
        return self._op(input, out=out, **fused)

    def forward_latency(self, size):
        return self._op.forward_latency(size)


# Default of `Network_Multi_Path_Infer.lazy_logits` for instances that do not set their own.  Off for programs that build the
# network themselves; the launcher switches it on for the train/ drivers, whose criteria and metric take the lazy logits.
LAZY_LOGITS = False


class Network_Multi_Path_Infer(nn.Module):
    _cell_cls = Cell   # the latency/ variant (latency_variant/model_seg.py) builds its cells from its own operators
    # Inference on the GPU writes a zoomed op's bilinear /2 input and a refine's skip feature from the kernels that produce them
    # (_trunk), from the second forward at an input size on.  None: whenever the forward runs in eval mode without autograd on a
    # CUDA input; False: never; True: also on the stand-in backend of the host tests.  The results are the same bits either way.
    fuse_resizes = None

    def __init__(self, alphas, betas, ratios, num_classes=19, layers=9, criterion=nn.CrossEntropyLoss(ignore_index=-1),
                 Fch=12, width_mult_list=[1., ], stem_head_width=(1., 1.), ignore_skip=False):
        super(Network_Multi_Path_Infer, self).__init__()
        assert layers >= 2
        self._num_classes, self._layers, self._criterion, self._Fch = num_classes, layers, criterion, Fch
        single_width = ratios[0].size(1) == 1          # genotypes searched without width options (model_seg.py:183-189)
        self._width_mult_list = ([1., ] if ignore_skip else [4. / 12, ]) if single_width else width_mult_list
        self._stem_head_width = stem_head_width
        self.latency = 0
        self.logits_dtype = torch.float32  # dtype of the upsampled logits returned by forward (fp16 halves the HBM write)
        # Branches are independent dependency chains of small, latency-bound kernels once their cells stop being shared
        # (model_seg.py:347-355): run each on its own CUDA stream (captured as parallel arms of the CUDA graph) and join
        # before the feature-fusion module.
        self.parallel_branches = True

        c2, c4, c8 = (self.num_filters(s, stem_head_width[0]) for s in (2, 4, 8))
        self.stem = nn.Sequential(
            ConvNorm(3, c2 * 2, kernel_size=3, stride=2, padding=1, bias=False, groups=1, slimmable=False),
            BasicResidual2x(c2 * 2, c4 * 2, kernel_size=3, stride=2, groups=1, slimmable=False),
            BasicResidual2x(c4 * 2, c8, kernel_size=3, stride=2, groups=1, slimmable=False))

        # one decoder for the three candidate branches; the order 0, 1, 2 matters (decode.py: the stages talk through
        # in-place edits of alphas / betas)
        decoder = decode.BranchDecoder(alphas, betas, ratios, self._width_mult_list, layers, ignore_skip)
        for last in (0, 1, 2):
            g = decoder.decode(last)
            for field in ("ops", "path", "downs", "widths"):
                setattr(self, "%s%d" % (field, last), getattr(g, field))

    def num_filters(self, scale, width=1.0):
        return int(np.round(scale * self._Fch * width))

    # ---------------------------------------------------------------------------------------------------------
    # structure
    # ---------------------------------------------------------------------------------------------------------
    def build_structure(self, lasts):
        self._branch = len(lasts)
        self.lasts = lasts
        self.ops, self.paths, self.downs, self.widths = ([getattr(self, name % last) for last in lasts]
                                                         for name in ("ops%d", "path%d", "downs%d", "widths%d"))
        self.branch_groups, self.cells = self.get_branch_groups_cells(self.ops, self.paths, self.downs, self.widths, self.lasts)
        self.build_arm_ffm_head()
        self._compile_schedule()

    def _cell_channels(self, branch, layer):
        """(C_in, C_out) of the cell of `branch` at `layer`: stem width in, head width out, searched widths in between."""
        path, widths = self.paths[branch], self.widths[branch]
        stride = 2 ** (path[layer] + 3)
        grow = self.downs[branch][layer] + 1
        first, final = layer == 0, layer == len(path) - 1
        if final and not first:
            assert self.downs[branch][layer] == 0
        w_in = self._stem_head_width[0] if first else widths[layer - 1]
        if first or not final:
            return self.num_filters(stride, w_in), self.num_filters(stride * grow, widths[layer])
        return self.num_filters(stride, w_in), self.num_filters(stride, self._stem_head_width[1])

    def get_branch_groups_cells(self, ops, paths, downs, widths, lasts):
        """Branches share a cell for as long as, layer after layer, they agree on (next scale, op, width)
        (model_seg.py:241-296).  Returns ([per layer: groups of branch ids], ModuleDict "layer-branch" -> Cell)."""
        n_branch = len(ops)

        def fingerprint(b, layer):
            if len(paths[b]) <= layer + 1:
                return ("last-cell-of", b)     # a branch's final cell is never shared
            return (paths[b][layer + 1], int(ops[b][layer]), widths[b][layer])

        self.ch_16 = self.ch_8_2 = self.ch_8_1 = 0
        taps = {}   # which branch's skip feature feeds which refine conv: (last, stride) -> attribute
        for attr, last, stride in (("ch_16", 2, 16), ("ch_8_2", 2, 8), ("ch_8_1", 1, 8)):
            if last in lasts:
                taps[(lasts.index(last), stride)] = attr

        cells, groups_per_layer = nn.ModuleDict(), []
        history = [() for _ in range(n_branch)]        # fingerprints so far; equal histories = still the same cell
        for layer in range(max(len(p) for p in paths)):
            buckets = OrderedDict()
            for b in range(n_branch):
                history[b] = history[b] + (fingerprint(b, layer),)
                if len(paths[b]) >= layer + 1:
                    buckets.setdefault(history[b], []).append(b)
            groups = list(buckets.values())
            for members in groups:
                lead = members[0]
                for other in members[1:]:
                    assert (ops[lead][layer] == ops[other][layer] and paths[lead][layer + 1] == paths[other][layer + 1]
                            and downs[lead][layer] == downs[other][layer] and widths[lead][layer] == widths[other][layer])
                down = downs[lead][layer]
                assert down in [0, 1]
                if layer < len(paths[lead]) - 1:
                    assert down == paths[lead][layer + 1] - paths[lead][layer]
                c_in, c_out = self._cell_channels(lead, layer)
                cell = self._cell_cls(ops[lead][layer], c_in, c_out, down)
                if down:   # the feature entering a down-sampling cell is what the refine conv of the finer scale concatenates
                    stride = 2 ** (paths[lead][layer] + 3)
                    for b in members:
                        if (b, stride) in taps:
                            setattr(self, taps[(b, stride)], cell._C_in)
                for b in members:
                    cells["%d-%d" % (layer, b)] = cell
            groups_per_layer.append(groups)
        return groups_per_layer, cells

    def build_arm_ffm_head(self):
        """Decoder modules (model_seg.py:214-239); attribute names are the checkpoint format."""
        n_cls, bn = self._num_classes, BatchNorm2d
        f8, f16, f32 = (self.num_filters(s, self._stem_head_width[1]) for s in SCALES)
        has16, has32 = 1 in self.lasts, 2 in self.lasts
        if self.training:  # auxiliary heads only exist in a train-mode build (model_seg.py:217-226)
            if has32:
                self.heads32 = Head(f32, n_cls, True, norm_layer=bn)
                self.heads16 = Head(f16 + self.ch_16 if has16 else self.ch_16, n_cls, True, norm_layer=bn)
            else:
                self.heads16 = Head(f16, n_cls, True, norm_layer=bn)
        fused = f8 * self._branch
        self.heads8 = Head(fused, n_cls, Fch=self._Fch, scale=4, branch=self._branch, is_aux=False, norm_layer=bn)
        point = dict(kernel_size=1, stride=1, padding=0, slimmable=False)
        box = dict(kernel_size=3, stride=1, padding=1, slimmable=False)
        if has32:
            self.arms32 = nn.ModuleList([ConvNorm(f32, f16, **point), ConvNorm(f16, f8, **point)])
            self.refines32 = nn.ModuleList([ConvNorm(f16 + self.ch_16, f16, **box), ConvNorm(f8 + self.ch_8_2, f8, **box)])
        if has16:
            self.arms16 = ConvNorm(f16, f8, **point)
            self.refines16 = ConvNorm(f8 + self.ch_8_1, f8, **box)
        self.ffm = FeatureFusion(fused, fused, reduction=1, Fch=self._Fch, scale=8, branch=self._branch, norm_layer=bn)

    def _compile_schedule(self):
        steps = []
        for layer, groups in enumerate(self.branch_groups):
            for n, members in enumerate(groups):
                steps.append(_CellStep("%d-%d" % (layer, members[0]), layer, members[0], tuple(members),
                                       fork=(n == 0 and len(groups) > 1)))
        # plain (non-Module, non-persistent) attributes: the schedule is derived data
        self.__dict__["_steps"] = steps
        self.__dict__["_tails"] = [_Tail(b, last) for b, last in enumerate(self.lasts)]
        self.__dict__.pop("_fsb_resize_plans", None)   # recorded per input size from the schedule's first forward (_trunk)

    def _tail_modules(self, last):
        """[(arm 1x1, refine 3x3, stride of the coarse input, stride of the skip input, extra skip channels)] for a branch
        ending at scale index `last`, coarse to fine."""
        if last == 2:
            return [(self.arms32[0], self.refines32[0], 32, 16, self.ch_16), (self.arms32[1], self.refines32[1], 16, 8, self.ch_8_2)]
        if last == 1:
            return [(self.arms16, self.refines16, 16, 8, self.ch_8_1)]
        return []

    # ---------------------------------------------------------------------------------------------------------
    # execution
    # ---------------------------------------------------------------------------------------------------------
    def _arm_refine(self, arm, refine, coarse, skip, out=None, cat=None):
        """arm 1x1 -> bilinear to skip's size -> cat([up, skip]) -> refine 3x3, with the concat done by writing both
        producers into one buffer (model_seg.py:304-307, 309-312, 316-319).  cat: that buffer, its skip channels already written
        by the skip's producer (_trunk)."""
        a = arm(coarse)
        from . import autograd as AG
        if AG.grad_mode(a):
            up = AG.bilinear(a, (skip.shape[2], skip.shape[3]))
            return refine(AG.cat_channels([up, skip]))
        N, c_up = a.shape[0], a.shape[1]
        c_skip, Hs, Ws = skip.shape[1], skip.shape[2], skip.shape[3]
        if cat is None:
            cat = F_.empty_nhwc(N, c_up + c_skip, Hs, Ws, a.device)
            F_.copy_channels(F_.to_nhwc_half(skip), cat[:, c_up:])
        F_.bilinear(a, (Hs, Ws), out=cat[:, :c_up])
        return refine(cat, out=out)

    def _side_streams(self, device):
        """one extra CUDA stream per additional branch (inference only)"""
        if not self.parallel_branches or self._branch < 2 or self.training or device.type != "cuda":
            return None
        streams = self.__dict__.get("_fsb_streams")
        if streams is None or streams[0].device != device:
            streams = [torch.cuda.Stream(device) for _ in range(self._branch - 1)]
            self.__dict__["_fsb_streams"] = streams
        return streams

    def _stem(self, input):
        """self.stem(input).  At inference on a CUDA input, stem.0 and the first conv of stem.1 run as one kernel
        (F_.stem_fused), so the 1/2-resolution map never goes through HBM; the rest of the stem runs unchanged.  Anything the
        fused kernel was not written for -- training, autograd, other stem layers or widths -- runs self.stem as before."""
        stem0, stem1 = self.stem[0], self.stem[1]
        if (self.training or torch.is_grad_enabled() or not input.is_cuda or type(stem0) is not ConvNorm
                or type(stem1) is not BasicResidual2x):
            return self.stem(input)
        conv0, bn0, conv1, bn1 = stem0.conv[0], stem0.conv[1], stem1.conv1, stem1.bn1
        lut = None
        if input.dtype == torch.uint8:
            lut = stem0.__dict__.get("_fsb_norm_lut")
            usable = lut is not None
        else:
            usable = input.dtype in (torch.float32, torch.float16) and input.is_contiguous() and not F_.is_nhwc_half(input)
        usable = usable and (stem0.C_in == 3 and stem0.kernel_size == 3 and stem0.stride == 2 and stem0.padding == 1
                             and not stem0.slimmable and conv0.bias is None and not bn0.training)
        usable = usable and (not stem1.slimmable and conv1.kernel_size[0] == 3 and conv1.stride[0] == 2 and conv1.padding[0] == 1
                             and conv1.dilation[0] == 1 and conv1.groups == 1 and not bn1.training and not stem1.bn2.training)
        if not usable:
            return self.stem(input)
        scale0, shift0 = engine.folded_bn(bn0, stem0.C_out, None)
        w0 = conv0.weight.detach()
        ci, co = engine.active_channels(conv1)
        scale1, shift1 = engine.folded_bn(engine.active_bn(bn1), co, conv1.bias)
        y = F_.stem_fused(input, lut, w0 if w0.dtype == torch.float32 else w0.float(), scale0, shift0,
                          engine.packed_weight(conv1, ci, co), co, scale1, shift1)
        if y is None:
            return self.stem(input)
        y = engine.conv_bn_act(y, stem1.conv2, stem1.bn2, relu=True)
        return self.stem[2](y)

    def _fuse_resizes_for(self, input):
        if self.fuse_resizes is False or self.training or torch.is_grad_enabled():
            return False
        return self.fuse_resizes or input.is_cuda

    def _record_resize_plan(self, input, src_step, tap_step, shapes):
        """The _ResizePlan of this input size, from what the first forward at that size ran: which step produced the input of each
        step (src_step[i], None for the stem), which step's output each refine took as its skip (tap_step, the same taps the tails
        read) and the shape of every step's output.  Buffers are then sized from the shapes the kernels produced, not re-derived
        from each operator's stride rules."""
        def residual(op):   # a primitive whose forward takes out_half / x_half
            return isinstance(op, _Residual) and type(op).forward is _Residual.forward

        ops = [self.cells[step.key]._op._op for step in self._steps]
        half, reads_half = set(), set()
        for i, p in enumerate(src_step):
            if residual(ops[i]) and ops[i]._zoom and p is not None and residual(ops[p]):
                half.add(p)
                reads_half.add(i)
        uses = {}
        for tail in self._tails:
            for n, (_, _, _, s_skip, _) in enumerate(self._tail_modules(tail.last)):
                uses.setdefault(tap_step[s_skip][tail.branch], []).append((tail.branch, n))
        skip = {p: u[0] for p, u in uses.items() if p is not None and len(u) == 1}   # a skip of two refines is copied
        plans = self.__dict__.setdefault("_fsb_resize_plans", {})
        plans[tuple(input.shape)] = _ResizePlan(frozenset(half), frozenset(reads_half), skip, tuple(shapes))

    def _fused_outputs(self, plan, i, src_half, device, cats):
        """keyword arguments of step i's cell under `plan`: its input's /2 (x_half), the buffer for its own /2 (out_half) and
        its output slice of a refine's concat buffer (out, the buffer recorded in cats[(branch, link)])"""
        kw = {}
        if i in plan.reads_half and src_half is not None:
            kw["x_half"] = src_half
        N, C, Ho, Wo = plan.shapes[i]
        if i in plan.half:
            kw["out_half"] = F_.empty_nhwc(N, C, Ho // 2, Wo // 2, device)
        if i in plan.skip:
            b, n = plan.skip[i]
            c_up = self._tail_modules(self.lasts[b])[n][0].C_out
            cat = F_.empty_nhwc(N, c_up + C, Ho, Wo, device)
            kw["out"] = cat[:, c_up:]
            cats[(b, n)] = (cat, kw["out"])
        return kw

    def _trunk(self, input, ctx=None):
        """stem + cells -> per scale, the latest feature of every branch ({8: [...], 16: [...], 32: [...]}).
        At inference (fuse_resizes) the kernels that produce a feature also write what later launches would have made of it:
        - a feature that a zoomed op reads also goes out as its bilinear /2, stored by the producing kernel (the last conv of the
          cell, or its bilinear x2 -- a /2 pixel reads only its own 2x2 block), and the zoomed op starts from that map;
        - a refine's skip feature is written straight into the channels of the refine's concat buffer (ctx.cats).
        Each is the same bits as the separate launch it replaces.  The first forward at an input size runs without them and
        records the plan for that size (_record_resize_plan), like the packed-weight and folded-BN caches that it also fills."""
        full_h = input.size(2)
        ctx = ctx if ctx is not None else _BranchCtx(None)
        stem = self._stem(input)
        # The concat buffer that the side streams will write into is allocated on the main stream BEFORE the fork, so the
        # block the caching allocator hands out cannot still be in use by main-stream work the side streams do not wait for.
        f8 = self.num_filters(8, self._stem_head_width[1])
        ctx.fused_in = F_.empty_nhwc(stem.shape[0], f8 * self._branch, stem.shape[2], stem.shape[3], stem.device)
        fuse = self._fuse_resizes_for(input)
        plan = self.__dict__.get("_fsb_resize_plans", {}).get(tuple(input.shape)) if fuse else None
        latest = [stem] * self._branch
        halves = [None] * self._branch     # bilinear /2 of latest[b], where its producer wrote one
        taps = {s: [stem] * self._branch for s in SCALES}
        src_step, shapes = [], []          # what the plan is recorded from: the producer of each step's input, each output's shape
        last_step = [None] * self._branch
        tap_step = {s: [None] * self._branch for s in SCALES}
        for i, step in enumerate(self._steps):
            if step.fork:
                ctx.fork()
            with ctx.on(step.lead):
                src = latest[step.lead]
                # the /2 maps and concat buffers cross the branch streams like the features: allocated on the producer's stream
                # and held until the join
                kw = self._fused_outputs(plan, i, halves[step.lead], src.device, ctx.cats) if plan is not None else {}
                feat = self.cells[step.key](src, **kw)
                ctx.hold(src, feat, *kw.values())
            src_step.append(last_step[step.lead])
            shapes.append(tuple(feat.shape))
            stride = int(full_h // feat.size(2))
            for b in step.members:
                latest[b] = feat
                halves[b] = kw.get("out_half")
                last_step[b] = i
                if stride in taps:
                    taps[stride][b] = feat
                    tap_step[stride][b] = i
        if fuse and plan is None:
            self._record_resize_plan(input, src_step, tap_step, shapes)
        return taps[8], taps[16], taps[32]

    def agg_ffm(self, outputs8, outputs16, outputs32, ctx=None):
        """per-branch arm/refine tails -> concat at 1/8 -> FeatureFusion -> heads (model_seg.py:298-335)"""
        training = self.training
        ctx = ctx if ctx is not None else _BranchCtx(None)
        taps = {8: outputs8, 16: outputs16, 32: outputs32}
        f8 = self.num_filters(8, self._stem_head_width[1])
        fused_in = getattr(ctx, "fused_in", None)  # allocated before the fork (see _trunk)
        if fused_in is None:
            ref = outputs8[0]
            fused_in = F_.empty_nhwc(ref.shape[0], f8 * self._branch, ref.shape[2], ref.shape[3], ref.device)  # cat(pred8)
        from . import autograd as AG
        grad = AG.grad_mode(*(outputs8 + outputs16 + outputs32))
        aux = {16: [], 32: []}          # train mode: inputs of the auxiliary heads, in branch order
        at8 = []
        for tail in self._tails:
            b = tail.branch
            slot = None if grad else fused_in[:, b * f8:(b + 1) * f8]
            with ctx.on(b):
                chain = self._tail_modules(tail.last)
                feat = None
                for n, (arm, refine, s_coarse, s_skip, _) in enumerate(chain):
                    coarse = taps[s_coarse][b] if n == 0 else feat
                    if training and n == 0:
                        aux[s_coarse].append(coarse)
                    if training and n == 1:
                        aux[s_coarse].append(taps[s_coarse][b])   # the trunk's 1/16 feature, not the refined one
                    skip = taps[s_skip][b]
                    cat, view = ctx.cats.get((b, n), (None, None))
                    fused = {"cat": cat} if view is skip else {}   # the skip's producer wrote it into this refine's concat buffer
                    feat = self._arm_refine(arm, refine, coarse, skip, out=slot if n == len(chain) - 1 else None, **fused)
                    ctx.hold(coarse, taps[s_skip][b], feat)
                if not chain:
                    feat = outputs8[b]
                    if not grad:
                        F_.copy_channels(F_.to_nhwc_half(feat), slot)
                at8.append(feat)
        ctx.join()
        if grad:
            fused_in = _cat_channels(at8)
        pred8 = self.heads8(self.ffm(fused_in))
        if not training:
            return pred8
        pred32 = self.heads32(_cat_channels(aux[32])) if aux[32] else None
        pred16 = self.heads16(_cat_channels(aux[16])) if aux[16] else None
        return pred8, pred16, pred32

    def _features(self, input):
        ctx = _BranchCtx(self._side_streams(input.device))
        outputs8, outputs16, outputs32 = self._trunk(input, ctx)
        return self.agg_ffm(outputs8, outputs16, outputs32, ctx)

    def forward(self, input):
        from . import autograd as AG
        if AG.TAPE_ENABLED and AG._TAPE is None and self.training and torch.is_grad_enabled():
            # EXPERIMENTAL: the whole pass as one autograd node; absent auxiliary predictions come back as None
            live = [0] + ([1] if any(last in (1, 2) for last in self.lasts) else []) + ([2] if 2 in self.lasts else [])
            outs = AG.run_taped(self, lambda x: tuple(p for p in self._forward(x) if p is not None), input)
            full = [None, None, None]
            for i, o in zip(live, outs):
                full[i] = o
            return tuple(full)
        return self._forward(input)

    def _forward(self, input):
        lazy = self.__dict__.get("lazy_logits", LAZY_LOGITS)   # N1: hand the criteria the low-resolution logits (losses.LazyLogits)
        if lazy:
            from .losses import LazyLogits
        if not self.training:
            pred8 = self._features(input)
            size = (int(pred8.size(2)) * 8, int(pred8.size(3)) * 8)
            if lazy:
                return LazyLogits(pred8, size, self.logits_dtype)
            return F_.upsample_logits(pred8, size, dtype=self.logits_dtype)
        outs = []
        for pred, factor in zip(self._features(input), SCALES):   # (pred8, pred16, pred32)
            if pred is not None:
                size = (pred.size(2) * factor, pred.size(3) * factor)
                pred = LazyLogits(pred, size, self.logits_dtype) if lazy else _upsample_logits(pred, size, self.logits_dtype)
            outs.append(pred)
        return tuple(outs)

    def set_input_normalization(self, mean, std):
        """Evaluator path (tools/engine/evaluator.py:206-225,329): after this the network also accepts the uint8 HWC image itself
        -- `img_u8` of shape (N, H, W, 3), passed as `img_u8.permute(0, 3, 1, 2)` -- and applies (v / 255 - mean) / std inside the
        stem kernel.  mean / std: per-channel sequences (config.image_mean / image_std)."""
        stem0 = self.stem[0]
        stem0.__dict__["_fsb_norm_lut"] = F_.normalization_lut(mean, std, next(self.parameters()).device)
        stem0.__dict__["_fsb_norm"] = (tuple(float(m) for m in mean), tuple(float(s) for s in std))

    @torch.no_grad()
    def predict_labels(self, input, out=None):
        """argmax(forward(input), dim=1) as uint8, fused into the x8 upsample: the evaluator's
        `exp -> cpu -> argmax` (tools/engine/evaluator.py:315-318) without materialising full-resolution logits."""
        assert not self.training
        pred8 = self._features(input)
        return F_.upsample_argmax(pred8, (int(pred8.size(2)) * 8, int(pred8.size(3)) * 8), out=out)

    @torch.no_grad()
    def accumulate_confusion(self, input, gt, cm):
        """Validation of one batch (tools/engine/evaluator.py:297-318 + tools/seg_opr/metric.py:7-15): the eval forward to the 1/8
        logits, then one kernel upsamples, takes the argmax and adds hist_info against `gt` (N x H x W) into `cm`
        (metric.ConfusionMatrix).  The counters equal those of predict_labels followed by cm.update."""
        assert not self.training
        pred8 = self._features(input)
        cm.update_from_logits(pred8, (int(pred8.size(2)) * 8, int(pred8.size(3)) * 8), gt)

    # ---------------------------------------------------------------------------------------------------------
    # latency model (table lookups, model_seg.py:368-408)
    # ---------------------------------------------------------------------------------------------------------
    def forward_latency(self, size):
        full_h = size[1]
        total = 0

        def run(module, shape):
            nonlocal total
            ms, shape = module.forward_latency(shape)
            total += ms
            return shape

        for block in self.stem:
            size = run(block, size)
        latest = [size] * self._branch
        # kept quirk: the reference never records the 1/8 shape of a cell here (it tests `scale == 4`), so the entry of a
        # branch that ends at 1/8 stays the stem's shape; only the 1/16 and 1/32 shapes are tracked
        taps = {s: [size] * self._branch for s in SCALES}
        for step in self._steps:
            shape = run(self.cells[step.key], latest[step.lead])
            stride = int(full_h // shape[1])
            for b in step.members:
                latest[b] = shape
                if stride in (16, 32):
                    taps[stride][b] = shape
        for tail in self._tails:
            chain = self._tail_modules(tail.last)
            shape = taps[8][tail.branch]
            for n, (arm, refine, s_coarse, _, c_skip) in enumerate(chain):
                shape = run(arm, taps[s_coarse][tail.branch] if n == 0 else shape)
                shape = run(refine, (shape[0] + c_skip, shape[1] * 2, shape[2] * 2))
        shape = run(self.ffm, (shape[0] * self._branch, shape[1], shape[2]))   # shape of the LAST branch, like the reference
        shape = run(self.heads8, shape)
        return total, shape


class _NullCtx:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


class _BranchCtx:
    """Routes the work of branch b to its own stream after `fork()`; `join()` makes the main stream wait for all.
    Every tensor that work on a side stream reads or writes is parked in `self.keep` until `join()`: the caching allocator
    frees a block on the stream it was ALLOCATED on, so a feature that a side-stream cell still reads must not lose its last
    Python reference while that cell is only enqueued (e.g. two branches that stay at the same stride after the fork overwrite
    `latest[b]` / `taps[..][b]` as they advance)."""

    def __init__(self, streams):
        self.streams, self.forked = streams, False
        self.main = torch.cuda.current_stream() if streams else None
        self.fused_in = None
        self.cats = {}    # (branch, link) -> (concat buffer, skip channels) a trunk cell wrote its output into
        self.keep = []

    def hold(self, *tensors):
        """keep these tensors alive until join() (no-op without side streams)"""
        if self.streams and self.forked:
            self.keep.extend(t for t in tensors if t is not None)

    def fork(self):
        if self.streams and not self.forked:
            for s in self.streams:
                s.wait_stream(self.main)
            self.forked = True

    def on(self, branch):
        if not self.streams:
            return _NullCtx()
        if not self.forked or branch == 0:
            return torch.cuda.stream(self.main)
        return torch.cuda.stream(self.streams[branch - 1])

    def join(self):
        if self.forked:
            for s in self.streams:
                self.main.wait_stream(s)
            self.forked = False
        self.keep = []   # after the join the main stream is ordered behind every side-stream reader


def _upsample_logits(x, size, dtype):
    from . import autograd as AG
    if AG.grad_mode(x):
        return AG.upsample_logits(x, size, dtype)
    return F_.upsample_logits(x, size, dtype=dtype)


def _cat_channels(tensors):
    """torch.cat(dim=1) of NHWC fp16 views through the strided copy kernel."""
    tensors = [F_.to_nhwc_half(t) for t in tensors]
    if len(tensors) == 1:
        return tensors[0]
    from . import autograd as AG
    if AG.grad_mode(*tensors):
        return AG.cat_channels(tensors)
    N, _, H, W = tensors[0].shape
    total = sum(t.shape[1] for t in tensors)
    out = F_.empty_nhwc(N, total, H, W, tensors[0].device)
    at = 0
    for t in tensors:
        F_.copy_channels(t, out[:, at:at + t.shape[1]])
        at += t.shape[1]
    return out
