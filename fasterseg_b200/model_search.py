"""Multi-resolution search supernet -- drop-in for the reference's search/model_search.py.

Same public surface as the reference (search/model_search.py:14-548): gumbel helpers, `MixedOp` / `Cell` /
`Network_Multi_Path` with the same constructor arguments, `sample_prun_ratio`, `forward`, `forward_latency`, `_loss`,
`_build_arch_parameters`, `_reset_arch_parameters`, attributes (`_arch_names`, `_arch_parameters`, `arch_idx`, `prun_mode`,
`_prun_modes` ...) and every parameter name (`stem.0.0.conv.0.weight`, `cells.3.1._op._ops.4.bn2.bn.2.running_var`,
`alpha_0_1`, `beta_1_2`, `ratio_1_0` ...), so search/train_search.py and search/architect.py drive it unchanged.

Organisation (ours): the trellis of cells is described once as a list of `_Node`s (layer, scale, which outputs of the
previous layer feed it, which beta row mixes them); `forward` and `forward_latency` walk that list, and `_loss` runs a list
of (architecture, width-mode) passes.  GPU side: NHWC fp16 activations; every conv+BN+ReLU is one fused wgmma unit (train
mode: conv with fused statistics, finalize, apply); the `result + op(x) * w * r0 * r1` accumulation over the five
primitives and the beta-weighted mix of the two cell invocations are single weighted-sum kernels (K5) whose backward also
yields the scalar gradients of alphas / betas / ratios; logits leave as NCHW fp32 through one layout kernel.
"""
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Variable

from . import autograd as AG
from . import engine
from . import functional as F_
from .genotypes import PRIMITIVES
from .operations import *  # noqa: F401,F403
from .operations import OPS, BasicResidual2x, ConvNorm
from .seg_oprs import Head

KEEP, DOWN = 0, 1   # the two outputs of a cell: same scale / next coarser scale
_Node = namedtuple("_Node", "layer scale feeds beta_row")   # feeds: ((source scale, KEEP | DOWN), ...) in invocation order


def _trellis(layers):
    """Cells of the supernet in execution order.  Scale j appears from layer j on; a cell on the diagonal (layer == scale) or
    at scale 0 has one input; any other cell runs twice per forward -- first on the down output of the finer scale, then on
    the keep output of its own scale -- and mixes the results with betas[scale][layer - scale - 1] (model_search.py:289-334)."""
    nodes = []
    for layer in range(layers):
        for scale in range(min(layer, 2) + 1):
            if scale == 0:
                nodes.append(_Node(layer, scale, ((0, KEEP),), None))
            elif layer == scale:
                nodes.append(_Node(layer, scale, ((scale - 1, DOWN),), None))
            else:
                nodes.append(_Node(layer, scale, ((scale - 1, DOWN), (scale, KEEP)), layer - scale - 1))
    return nodes


# ---- gumbel-softmax width sampling (model_search.py:13-43; technique: github.com/YongfeiYan/Gumbel_Softmax_VAE) ---------
def sample_gumbel(shape, eps=1e-20, device=None):
    uniform = torch.rand(shape)          # drawn from the CPU generator like the reference, then moved
    if device is not None:
        uniform = uniform.to(device)
    return -torch.log(eps - torch.log(uniform + eps))


def gumbel_softmax_sample(logits, temperature=1):
    noisy = logits + sample_gumbel(logits.size(), device=logits.device)
    return F.softmax(noisy / temperature, dim=-1)


def gumbel_softmax(logits, temperature=1, hard=False):
    """Straight-through estimator: the forward value is the one-hot of the sample, the gradient that of the soft sample."""
    soft = gumbel_softmax_sample(logits, temperature)
    if not hard:
        return soft
    winner = soft.max(dim=-1)[1]
    one_hot = torch.zeros_like(soft).view(-1, soft.size(-1)).scatter_(1, winner.view(-1, 1), 1).view(*soft.size())
    return (one_hot - soft).detach() + soft


def _resolve_ratio(r, width_mult_list):
    """tensor -> (width_mult_list[argmax], score tensor = r[argmax]) ; float -> (forced width, 1.)  (model_search.py:63-74);
    engine.SymRatio (width chosen on the device in a captured pass) -> itself, score folded into the planned weights"""
    if isinstance(r, engine.SymRatio):
        return r, 1.
    if isinstance(r, torch.Tensor):
        idx = int(r.argmax())
        return width_mult_list[idx], r[idx]
    return r, 1.


def _needs_graph(*tensors):
    return AG.grad_mode(*tensors)


class MixedOp(nn.Module):
    def __init__(self, C_in, C_out, stride=1, width_mult_list=[1.]):
        super(MixedOp, self).__init__()
        self._width_mult_list = width_mult_list
        self._ops = nn.ModuleList(OPS[name](C_in, C_out, stride, True, width_mult_list=width_mult_list) for name in PRIMITIVES)

    def set_prun_ratio(self, ratio):
        for op in self._ops:
            op.set_ratio(ratio)

    def _scaled_weights(self, weights, ratios):
        """switch every primitive to the (in, out) widths and fold the two width scores into the op weights"""
        (w_in, score_in), (w_out, score_out) = (_resolve_ratio(r, self._width_mult_list) for r in ratios[:2])
        self.set_prun_ratio((w_in, w_out))
        if hasattr(weights, "take_slot"):       # planned pass (graphed.py): a static slot holding softmax(alpha) x width scores
            return weights.take_slot(ratios[0], ratios[1])
        return weights * score_in * score_out  # [len(PRIMITIVES)] scalar arithmetic (plumbing)

    def forward(self, x, weights, ratios):
        # a ratio is a tensor (searched width distribution) or a float (forced width)
        return self._mix(x, self._scaled_weights(weights, ratios))

    def _mix(self, x, wvec):
        """sum_k wvec[k] * op_k(x) at the widths `_scaled_weights` just configured"""
        ctx = engine.graph_ctx()
        if ctx is not None:     # captured pass: the five primitives are independent chains of small kernels -> side streams
            outs = ctx.parallel([(lambda op=op: F_.to_nhwc_half(op(x))) for op in self._ops])
        else:
            outs = [F_.to_nhwc_half(op(x)) for op in self._ops]
        if _needs_graph(wvec, *outs):
            return AG.weighted_sum(wvec, outs)
        return F_.wsum_fwd(outs, wvec.detach().float().contiguous())

    def forward_latency(self, size, weights, ratios):
        wvec = self._scaled_weights(weights, ratios)
        expected = 0
        for w, op in zip(wvec, self._ops):
            ms, size_out = op.forward_latency(size)
            expected = expected + ms * w
        return expected, size_out


class Cell(nn.Module):
    def __init__(self, C_in, C_out=None, down=True, width_mult_list=[1.]):
        super(Cell, self).__init__()
        self._C_in = C_in
        self._C_out = C_in if C_out is None else C_out
        self._down = down
        self._width_mult_list = width_mult_list
        self._op = MixedOp(C_in, self._C_out, width_mult_list=width_mult_list)
        if self._down:
            self.downsample = MixedOp(C_in, C_in * 2, stride=2, width_mult_list=width_mult_list)

    def _both(self, method, x, alphas, ratios):
        """(keep, down) through `method` of the two MixedOps; ratios = (in, out, down) and `down` is None iff no down path"""
        assert (ratios[2] is not None) == bool(self._down)
        ctx = engine.graph_ctx() if method == "forward" else None
        if ctx is not None and self._down:     # captured pass: the two MixedOps read the same x and are independent
            # (the mixing-weight slots are taken in program order BEFORE forking, so slot numbering stays deterministic)
            w_keep = self._op._scaled_weights(alphas, (ratios[0], ratios[1]))
            w_down = self.downsample._scaled_weights(alphas, (ratios[0], ratios[2]))
            keep, down = ctx.parallel([lambda: self._op._mix(x, w_keep), lambda: self.downsample._mix(x, w_down)])
            return keep, down
        keep = getattr(self._op, method)(x, alphas, (ratios[0], ratios[1]))
        down = getattr(self.downsample, method)(x, alphas, (ratios[0], ratios[2])) if self._down else None
        return keep, down

    def forward(self, input, alphas, ratios):
        return self._both("forward", input, alphas, ratios)

    def forward_latency(self, size, alphas, ratios):
        return self._both("forward_latency", size, alphas, ratios)


def _mix(betas_row, a, b):
    """beta-weighted sum of the two invocations of a cell (model_search.py:330-333)."""
    if a is None and b is None:
        return 0
    a, b = F_.to_nhwc_half(a), F_.to_nhwc_half(b)
    if _needs_graph(betas_row, a, b):
        return AG.weighted_sum(betas_row, [a, b])
    return F_.wsum_fwd([a, b], betas_row.detach().float().contiguous())


def _blend(brow, results):
    """(keep, down) of a twice-invoked cell from its [(keep, down) | None, (keep, down) | None] results."""
    first, second = results
    if first is not None and second is not None:
        return _mix(brow, first[KEEP], second[KEEP]), (_mix(brow, first[DOWN], second[DOWN]) if first[DOWN] is not None else 0)
    # a beta underflowed to 0 and its invocation was skipped: plain scaled term, like the reference's sum()
    alive, w = (second, brow[1]) if first is None else (first, brow[0])
    if alive is None:
        return 0, 0
    solo = torch.stack([w, w * 0])
    return _mix(solo, alive[KEEP], alive[KEEP]), (0 if alive[DOWN] is None else _mix(solo, alive[DOWN], alive[DOWN]))


class Network_Multi_Path(nn.Module):
    def __init__(self, num_classes=19, layers=16, criterion=nn.CrossEntropyLoss(ignore_index=-1), Fch=12, width_mult_list=[1., ],
                 prun_modes=['arch_ratio', ], stem_head_width=[(1., 1.), ]):
        super(Network_Multi_Path, self).__init__()
        assert layers >= 3
        self._num_classes, self._layers, self._criterion, self._Fch = num_classes, layers, criterion, Fch
        self._width_mult_list = width_mult_list
        self._prun_modes = prun_modes
        self.prun_mode = None  # prun_mode is higher priority than _prun_modes
        self._stem_head_width = stem_head_width
        self._flops = 0
        self._params = 0
        nf = self.num_filters
        stem_widths = [w for w, _ in stem_head_width]
        head_widths = [w for _, w in stem_head_width]

        def per(widths, make):
            return nn.ModuleList([make(w) for w in widths])    # one copy per architecture (teacher / student)

        def cn(ci, co, k):
            return ConvNorm(ci, co, kernel_size=k, padding=1 if k == 3 else None, bias=False, groups=1, slimmable=False)

        self.stem = per(stem_widths, lambda w: nn.Sequential(
            ConvNorm(3, nf(2, w) * 2, kernel_size=3, stride=2, padding=1, bias=False, groups=1, slimmable=False),
            BasicResidual2x(nf(2, w) * 2, nf(4, w) * 2, kernel_size=3, stride=2, groups=1, slimmable=False),
            BasicResidual2x(nf(4, w) * 2, nf(8, w), kernel_size=3, stride=2, groups=1, slimmable=False)))

        self.__dict__["_nodes"] = _trellis(layers)
        self.cells = nn.ModuleList(nn.ModuleList() for _ in range(layers))
        for node in self._nodes:
            # a cell has a down path unless it sits at the coarsest scale or in the last layer
            has_down = node.scale < 2 and node.layer < max(layers - 1, 2)
            self.cells[node.layer].append(Cell(nf(8 * 2 ** node.scale), down=has_down, width_mult_list=width_mult_list))

        self.refine32 = per(head_widths, lambda w: nn.ModuleList([cn(nf(32, w), nf(16, w), 1), cn(nf(32, w), nf(16, w), 3),
                                                                  cn(nf(16, w), nf(8, w), 1), cn(nf(16, w), nf(8, w), 3)]))
        self.refine16 = per(head_widths, lambda w: nn.ModuleList([cn(nf(16, w), nf(8, w), 1), cn(nf(16, w), nf(8, w), 3)]))
        for name, mult in (("head0", 1), ("head1", 1), ("head2", 1), ("head02", 2), ("head12", 2)):
            setattr(self, name, per(head_widths, lambda w: Head(nf(8, w) * mult, num_classes, False)))

        # arch parameter names: {"alphas": [...], "betas": [...], "ratios": [...]} per architecture (teacher / student)
        self._arch_names = []
        self._arch_parameters = []
        for i in range(len(self._prun_modes)):
            arch_name, arch_param = self._build_arch_parameters(i)
            self._arch_names.append(arch_name)
            self._arch_parameters.append(arch_param)
            self._reset_arch_parameters(i)
        self.arch_idx = 0  # which architecture's stem / heads / arch parameters the next forward uses

    def num_filters(self, scale, width=1.0):
        return int(np.round(scale * self._Fch * width))

    def new(self):
        """(dead in the reference too: it references an undefined `Network`, model_search.py:203-207)"""
        model_new = Network_Multi_Path(self._num_classes, self._layers, self._criterion, self._Fch).cuda()
        for x, y in zip(model_new._arch_parameters, self._arch_parameters):
            for a, b in zip(x, y):
                a.data.copy_(b.data)
        return model_new

    # ---------------------------------------------------------------------------------------------------------
    # width sampling
    # ---------------------------------------------------------------------------------------------------------
    def sample_prun_ratio(self, mode="arch_ratio"):
        '''mode: "min"|"max"|"random"|"arch_ratio"(default)'''
        assert mode in ["min", "max", "random", "arch_ratio"]
        rows = (self._layers - 1, self._layers - 1, self._layers - 2)     # ratio rows per scale
        if mode == "arch_ratio":
            params = [getattr(self, name) for name in self._arch_names[self.arch_idx]["ratios"]]
            return [[gumbel_softmax(F.log_softmax(p[row], dim=-1), hard=True) for row in range(n)] for p, n in zip(params, rows)]
        choices = self._width_mult_list
        draw = {"min": lambda: choices[0], "max": lambda: choices[-1], "random": lambda: np.random.choice(choices)}[mode]
        # drawing order (all rows of scale 0, then scale 1, then scale 2) is part of the contract: shared numpy RNG stream
        return [[draw() for _ in range(n)] for n in rows]

    def _arch(self, kind, i):
        return getattr(self, self._arch_names[self.arch_idx][kind][i])

    def _ratio_triple(self, i, j, ratios):
        """(in, out, down) width ratios of the cell at layer i, scale j (model_search.py:300-316)."""
        shw = self._stem_head_width[self.arch_idx]
        if i == 0 and j == 0:
            return (shw[0], ratios[j][i - j], ratios[j + 1][i - j])
        if i == self._layers - 1:
            return (ratios[j][i - j - 1] if j == 0 else ratios[j][i - j], shw[1], None)
        if j == 2:
            return (ratios[j][i - j], ratios[j][i - j + 1], None)
        if j == 0:
            return (ratios[j][i - j - 1], ratios[j][i - j], ratios[j + 1][i - j])
        return (ratios[j][i - j], ratios[j][i - j + 1], ratios[j + 1][i - j])

    def _distributions(self, alpha=True, beta=True):
        """softmax of the architecture parameters, or uniform stand-ins (forward_latency's switches)"""
        dev = self._arch("alphas", 0).device
        if alpha:
            alphas = [F.softmax(self._arch("alphas", s), dim=-1) for s in range(3)]
        else:
            alphas = [torch.ones_like(self._arch("alphas", s)).to(dev) * 1. / len(PRIMITIVES) for s in range(3)]
        if beta:
            betas = [None] + [F.softmax(self._arch("betas", s), dim=-1) for s in range(2)]
        else:
            betas = [None] + [torch.ones_like(self._arch("betas", s)).to(dev) * 1. / 2 for s in range(2)]
        return alphas, betas

    def _current_mode(self):
        return self.prun_mode if self.prun_mode is not None else self._prun_modes[self.arch_idx]

    # ---------------------------------------------------------------------------------------------------------
    # execution
    # ---------------------------------------------------------------------------------------------------------
    def forward(self, input):
        if AG.TAPE_ENABLED and AG._TAPE is None and self.training and torch.is_grad_enabled():
            return AG.run_taped(self, self._forward, input)   # EXPERIMENTAL: the whole pass as one autograd node
        return self._forward(input)

    def _forward(self, input, plan=None, head=None):
        """plan (graphed.PassContext): a captured pass -- mixing weights and widths come from static device slots instead of being
        computed here; the tensor work is identical.  head (eval, no plan): return only that head's 1/8 NHWC logits, running only
        the refine chains it reads; widths are drawn exactly as for the full pass."""
        idx = self.arch_idx
        refine16, refine32 = self.refine16[idx], self.refine32[idx]
        if plan is None:
            alphas, betas = self._distributions()
            # one host read instead of a GPU->CPU sync per `betas[...] > 0` test (model_search.py:326-329)
            alive = [None] + [(b.detach() > 0).tolist() for b in betas[1:]]
            ratios = self.sample_prun_ratio(mode=self._current_mode())
        else:
            ratios = plan.sym_ratios

        def run_cell(node, prev):
            cell = self.cells[node.layer][node.scale]
            arow = node.layer - node.scale
            alpha = alphas[node.scale][arow] if plan is None else plan.alpha(node.scale, arow)
            ratio = self._ratio_triple(node.layer, node.scale, ratios)
            if node.beta_row is None:
                (src, port), = node.feeds
                return cell(prev[src][port], alpha, ratio)
            # same weights, two inputs ("0: from down", then "1: from keep"); BN running stats see both, in this order
            flags = alive[node.scale][node.beta_row] if plan is None else (True, True)   # softmax(beta) > 0 barring underflow
            results = [cell(prev[src][port], alpha, ratio) if flags[n] else None for n, (src, port) in enumerate(node.feeds)]
            brow = betas[node.scale][node.beta_row] if plan is None else plan.beta(node.scale, node.beta_row)
            return _blend(brow, results)

        def fan(thunks):
            """independent pieces: on side streams in a captured pass, in order otherwise"""
            return plan.parallel(thunks) if plan is not None else [t() for t in thunks]

        cur = {0: (self.stem[idx](input), None)}
        for layer in range(self._layers):
            nodes = [n for n in self._nodes if n.layer == layer]      # the cells of a layer only read the previous layer
            prev = cur
            outs = fan([(lambda n=n, prev=prev: run_cell(n, prev)) for n in nodes])
            cur = {n.scale: o for n, o in zip(nodes, outs)}
        f8, f16, f32 = (cur[s][KEEP] for s in range(3))

        def chain16():
            return refine16[1](_cat([_resize2x(refine16[0](f16)), f8]))

        def chain32():
            o = refine32[1](_cat([_resize2x(refine32[0](f32)), f16]))
            return refine32[3](_cat([_resize2x(refine32[2](o)), f8]))

        out0 = f8
        heads = [lambda: self.head0[idx](out0), lambda: self.head1[idx](out1), lambda: self.head2[idx](out2),
                 lambda: self.head02[idx](_cat([out0, out2])), lambda: self.head12[idx](_cat([out1, out2]))]
        if head is not None:
            out1 = chain16() if head in (1, 4) else None
            out2 = chain32() if head in (2, 3, 4) else None
            return heads[head]()
        out1, out2 = fan([chain16, chain32])
        preds = fan(heads)
        leave = _to_nchw if self.training else _upsample8
        return tuple(leave(p) for p in preds)

    def set_input_normalization(self, mean, std):
        """After this every architecture's stem also accepts the uint8 HWC image itself, passed as `img_u8.permute(0, 3, 1, 2)`,
        and applies (v / 255 - mean) / std in its gather (Network_Multi_Path_Infer.set_input_normalization)"""
        lut = F_.normalization_lut(mean, std, next(self.parameters()).device)
        for stem in self.stem:
            stem[0].__dict__["_fsb_norm_lut"] = lut

    def _head_logits(self, input, head):
        assert not self.training and 0 <= int(head) < 5
        return F_.to_nhwc_half(self._forward(input, head=int(head)))

    @torch.no_grad()
    def predict_labels(self, input, head=0):
        """argmax(forward(input)[head], dim=1) as uint8 (the evaluator's `score[out_idx]` -> exp -> argmax,
        tools/engine/evaluator.py:306-318): the eval forward with that head only, and the fused x8 upsample + argmax"""
        p = self._head_logits(input, head)
        return F_.upsample_argmax(p, (int(p.size(2)) * 8, int(p.size(3)) * 8))

    @torch.no_grad()
    def accumulate_confusion(self, input, gt, cm, head=0):
        """hist_info of predict_labels(input, head) against `gt` into `cm` (metric.ConfusionMatrix), in one kernel after the
        eval forward and without a label map"""
        p = self._head_logits(input, head)
        cm.update_from_logits(p, (int(p.size(2)) * 8, int(p.size(3)) * 8), gt)

    def forward_latency(self, size, alpha=True, beta=True, ratio=True):
        """Expected latency of the current architecture distribution from the per-op lookup table
        (model_search.py:361-475).  With the arch parameters on CUDA and every reachable table entry present, one kernel
        evaluates it (supernet_latency.py, K14) and one more differentiates it; otherwise `_latency_walk` runs as scalar
        arithmetic on the arch parameters' device, measuring and persisting any missing table entry."""
        from . import supernet_latency
        mode = self._current_mode() if ratio else 'max'
        if supernet_latency.usable(self):
            plan = supernet_latency.plan_for(self, size, alpha, beta, ratio, mode)
            if plan is not None:
                return supernet_latency.expected_latency(self, plan)
        alphas, betas = self._distributions(alpha, beta)
        ratios = self.sample_prun_ratio(mode=mode)
        return self._latency_walk(size, alphas, betas, ratios, lambda cell, size, a, r: cell.forward_latency(size, a, r))

    def _latency_walk(self, size, alphas, betas, ratios, cell_latency):
        """The expected-latency recurrence over the trellis.  cell_latency(cell, size, alphas row, (in, out, down) ratios) ->
        ((keep ms, size), (down ms, size) | None).  The recurrences reproduce the reference's, including which beta row weights
        the running totals (see `settle`); supernet_latency.py traces this same code into the kernel's plan."""
        stem_ms = 0
        for block in self.stem[self.arch_idx]:
            ms, size = block.forward_latency(size)
            stem_ms = stem_ms + ms
        total = [[stem_ms, 0], [0, 0], [0, 0]]            # expected latency up to (scale, KEEP | DOWN)
        prev, cur, pending, at_layer = {0: (size, None)}, {}, [], 0

        def settle(layer, pending):
            """fold the per-cell latencies of one finished layer into the running totals"""
            coarsest = len(pending) - 1
            for scale, ms in enumerate(pending):
                if scale == 0:
                    if ms[KEEP] is not None: total[0][KEEP] = total[0][KEEP] + ms[KEEP]
                    if ms[DOWN] is not None: total[0][DOWN] = total[0][KEEP] + ms[DOWN]
                elif layer == scale:
                    if ms[KEEP] is not None: total[scale][KEEP] = total[scale - 1][DOWN] + ms[KEEP]
                    if ms[DOWN] is not None: total[scale][DOWN] = total[scale - 1][DOWN] + ms[DOWN]
                else:
                    # kept quirk: the mixing row is the one of the layer's COARSEST cell, for every scale of the layer
                    b = betas[coarsest][layer - coarsest - 1]
                    if ms[KEEP] is not None:
                        total[scale][KEEP] = b[1] * total[scale][KEEP] + b[0] * total[scale - 1][DOWN] + ms[KEEP]
                    if ms[DOWN] is not None:
                        total[scale][DOWN] = b[1] * total[scale][KEEP] + b[0] * total[scale - 1][DOWN] + ms[DOWN]

        for node in self._nodes:
            if node.layer != at_layer:
                settle(at_layer, pending)
                prev, cur, pending, at_layer = cur, {}, [], node.layer
            cell = self.cells[node.layer][node.scale]
            a = alphas[node.scale][node.layer - node.scale]
            r = self._ratio_triple(node.layer, node.scale, ratios)
            if node.beta_row is None:
                (src, port), = node.feeds
                keep, down = cell_latency(cell, prev[src][port], a, r)
                cur[node.scale] = (keep[1], down[1] if down is not None else None)
                pending.append([keep[0], down[0] if down is not None else None])
            else:
                b = betas[node.scale][node.beta_row]
                runs = [cell_latency(cell, prev[src][port], a, r) if b[n] > 0 else (None, None)
                        for n, (src, port) in enumerate(node.feeds)]
                (keep0, down0), (keep1, down1) = runs
                assert (keep0 is None and keep1 is None) or keep0[1] == keep1[1]
                assert (down0 is None and down1 is None) or down0[1] == down1[1]
                cur[node.scale] = (keep0[1], down0[1] if down0 is not None else None)
                pending.append([sum(w * k for w, k in zip(b, [keep0[0], keep1[0]])),
                                sum(w * d if d is not None else 0
                                    for w, d in zip(b, [None if down0 is None else down0[0], None if down1 is None else down1[0]]))])
        settle(at_layer, pending)
        return sum([total[0][KEEP], total[1][KEEP], total[2][KEEP]])

    def _loss(self, input, target, pretrain=False):
        """Sum of the criterion over the 5 logits of every pass (model_search.py:478-505): search = one pass per architecture
        with its own width mode, plus max / min width; pretrain = max, min and two random-width passes."""
        passes = []   # (architecture to switch to | None = leave as is, width mode)
        if pretrain is not True:
            passes += [(idx, None) for idx in range(len(self._arch_names))]   # "random width": sampled by gumbel softmax
        if len(self._width_mult_list) > 1:
            passes += [(None, mode) for mode in ["max", "min"] + (["random", "random"] if pretrain == True else [])]  # noqa: E712
        elif pretrain == True and len(self._width_mult_list) == 1:  # noqa: E712
            passes.append((None, "max"))
        runner = self._graph_runner(input)
        if runner is not None:
            return runner.loss(input, target, passes)
        loss = 0
        for arch, mode in passes:
            if arch is not None:
                self.arch_idx = arch
            self.prun_mode = mode
            loss = loss + sum(self._criterion(logit, target) for logit in self(input))
        return loss

    def _graph_runner(self, input):
        """graphed.GraphedLoss of this model when `_loss` can run as captured passes (training mode, gradients on, CUDA, single
        process or library-owned data parallelism, more than one width), else None -> the eager path above."""
        from . import graphed
        forced = self.__dict__.get("_fsb_graph_mode")          # tests: True forces (eager passes on CPU), False disables
        if forced is False or (forced is None and not (graphed.ENABLED and input.is_cuda)):
            return None
        if not (self.training and torch.is_grad_enabled() and len(self._width_mult_list) > 1 and AG.FUSED_WGRAD_ACCUMULATION):
            return None
        if engine.dp_world_size() > 1 and not engine.dp_native():
            return None
        runner = self.__dict__.get("_fsb_graph_runner")
        if runner is None:
            runner = graphed.GraphedLoss(self, capture=input.is_cuda)
            self.__dict__["_fsb_graph_runner"] = runner
        return runner

    def _arch_shapes(self, idx):
        num_ops = len(PRIMITIVES)
        num_widths = len(self._width_mult_list) if self._prun_modes[idx] == 'arch_ratio' else 1
        L = self._layers
        return {"alphas": [(L, num_ops), (L - 1, num_ops), (L - 2, num_ops)],
                "betas": [(L - 2, 2), (L - 3, 2)],  # in-degree probs; 0: from down, 1: from keep
                "ratios": [(L - 1, num_widths), (L - 1, num_widths), (L - 2, num_widths)]}

    def _build_arch_parameters(self, idx):
        names = {"alphas": ["alpha_" + str(idx) + "_" + str(s) for s in [0, 1, 2]],
                 "betas": ["beta_" + str(idx) + "_" + str(s) for s in [1, 2]],
                 "ratios": ["ratio_" + str(idx) + "_" + str(s) for s in [0, 1, 2]]}
        shapes = self._arch_shapes(idx)
        for kind in ("alphas", "betas", "ratios"):
            for name, shape in zip(names[kind], shapes[kind]):
                setattr(self, name, nn.Parameter(Variable(1e-3 * torch.ones(*shape), requires_grad=True)))
        params = [getattr(self, n) for kind in ("alphas", "betas", "ratios") for n in names[kind]]
        return names, params

    def _reset_arch_parameters(self, idx):
        shapes = self._arch_shapes(idx)
        for kind in ("alphas", "betas", "ratios"):
            for name, shape in zip(self._arch_names[idx][kind], shapes[kind]):
                getattr(self, name).data = Variable(1e-3 * torch.ones(*shape), requires_grad=True)


# ------------------------------------------------------------------------------------------------------------
def _grad(*ts):
    return AG.grad_mode(*ts)


def _cat(tensors):
    tensors = [F_.to_nhwc_half(t) for t in tensors]
    if _grad(*tensors):
        return AG.cat_channels(tensors)
    N, _, H, W = tensors[0].shape
    out = F_.empty_nhwc(N, sum(t.shape[1] for t in tensors), H, W, tensors[0].device)
    at = 0
    for t in tensors:
        F_.copy_channels(t, out[:, at:at + t.shape[1]])
        at += t.shape[1]
    return out


def _resize2x(t):
    t = F_.to_nhwc_half(t)
    size = (t.shape[2] * 2, t.shape[3] * 2)
    return AG.bilinear(t, size) if _grad(t) else F_.bilinear(t, size)


def _upsample8(p):
    p = F_.to_nhwc_half(p)
    size = (p.shape[2] * 8, p.shape[3] * 8)
    return AG.upsample_logits(p, size) if _grad(p) else F_.upsample_logits(p, size, dtype=torch.float32)


def _to_nchw(p):
    p = F_.to_nhwc_half(p)
    return AG.to_nchw(p) if _grad(p) else F_.to_nchw(p, torch.float32)
