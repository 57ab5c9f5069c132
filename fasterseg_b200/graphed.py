"""Captured training passes of the search supernet ("graph mode" of Network_Multi_Path._loss).

Why: one supernet step is ~3 400 conv units per `_loss` (search/model_search.py:478-505: four forwards, one backward),
~27 k kernel launches of a few microseconds each.  Driven from Python the step costs 1-2 s of host time against ~5 ms of
roofline (DESIGN.md); nothing short of removing the host from the loop changes that.  The obstacle to CUDA graphs is that two
to three of the four passes run at SAMPLED widths (np.random.choice / gumbel-softmax, model_search.py:209-261), i.e. different
tensor shapes every step.

How: a pass is captured ONCE per architecture at MAXIMUM width, and the width choice becomes data:
  * every slimmable unit gets its width index from a slot of an int32 vector in device memory (engine.SymRatio);
  * its BatchNorm kernels pick the per-width parameter set from a device table (fsb_bn_sel) and force the inactive channel
    tail to zero -- zero activations meet the unused weight columns of the consumer, zero gradients meet the unused weight rows
    of the producer, so the arithmetic of USConv2d / USBatchNorm2d slicing (search/slimmable_ops.py:36-69) is reproduced
    exactly while every tensor keeps a static shape (FactorizedReduce's concat moves with the width: fsb_*_sel `hmax`);
  * the op / branch mixing weights (softmax(alpha) x width scores, softmax(beta)) are computed eagerly by ordinary torch
    autograd -- a handful of tiny kernels per pass -- copied into static slots, and their gradients come back out of the
    backward graph and are pushed through that torch graph: alphas, betas and ratios get exactly the gradients of
    model_search.py:60-78,326-333;
  * weight gradients accumulate in a flat staging buffer; `loss.backward()` releases them into `param.grad` for exactly the
    parameters the step touched (parameters of unsampled widths keep grad None, as in the reference, so SGD's weight decay and
    momentum skip them).
A step then is: 4 x (few tiny torch ops + forward replay + the caller's criterion + backward replay) -- no per-unit host work.
Without a GPU (tests) the same code runs the passes eagerly (capture=False) on the CPU stand-in backend.
"""
from __future__ import annotations

import ctypes as C
import gc
import os
import weakref

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, autograd as AG, engine
from . import functional as F_

ENABLED = os.environ.get("FSB_GRAPH", "1") != "0"


# Registries the flat step tail (optim.py) looks buffers up in.  Weak values: the runner of a model owns its FlatGrads, so a model that
# goes away takes its flat buffers (2 x 4 bytes per parameter) and its registry entries with it -- and a FlatGrads keeps its parameters
# alive, so an id() in here can never have been recycled for another tensor.
FLAT_BY_PARAM = weakref.WeakValueDictionary()      # id(parameter) -> the FlatGrads that stages its gradient
FLAT_BY_MODEL = weakref.WeakValueDictionary()      # id(model) -> its FlatGrads


class FlatGrads:
    """Two flat fp32 buffers over all parameters of a model: `S` (staging: the captured kernels accumulate here) and `G`
    (what `param.grad` views point into after a release)."""

    def __init__(self, model):
        self.params = [p for p in model.parameters() if p.requires_grad]
        dev = self.params[0].device
        self.offsets, total = {}, 0
        for p in self.params:
            self.offsets[id(p)] = total
            total += (p.numel() + 3) // 4 * 4      # 16-byte aligned views
        self.total = total
        self.S = torch.zeros(total, device=dev, dtype=torch.float32)
        self.G = torch.zeros(total, device=dev, dtype=torch.float32)
        self.index = {id(p): i for i, p in enumerate(self.params)}
        self._sviews, self._gviews = {}, {}
        self.dirty = False      # S holds un-released gradients
        # bookkeeping for the flat step tail (optim.py): which parameters the LAST release handed a gradient view of G, and whether G
        # is exactly "scale * staging" (every other region zero) -- the precondition of the flat clip / SGD kernels
        self.live_flags = np.zeros(len(self.params), dtype=np.uint8)
        self.ever_live = np.zeros(len(self.params), dtype=np.uint8)
        self.fresh_release = None
        for p in self.params:
            FLAT_BY_PARAM[id(p)] = self
        self.model_ref = weakref.ref(model)
        self.other_params = [p for p in model.parameters() if not p.requires_grad]      # never carry gradients; kept for completeness
        FLAT_BY_MODEL[id(model)] = self

    def _view(self, flat, cache, p):
        v = cache.get(id(p))
        if v is None:
            off = self.offsets[id(p)]
            v = flat[off:off + p.numel()].view(p.shape)
            cache[id(p)] = v
        return v

    def sview(self, p):
        return self._view(self.S, self._sviews, p)

    def gview(self, p):
        return self._view(self.G, self._gviews, p)

    def begin(self):
        """start of a `_loss`: forget staged gradients nobody asked for"""
        if self.dirty:
            self.S.zero_()
        self.dirty = True

    def release(self, touched, scale=1.0):
        """staged gradients -> param.grad of the `touched` parameters (list of Parameters)"""
        fresh = all(p.grad is None for p in touched)
        self.fresh_release = bool(fresh)
        self.live_flags[:] = 0
        self.live_flags[[self.index[id(p)] for p in touched]] = 1
        self.ever_live |= self.live_flags
        if fresh:
            if scale == 1.0:
                self.G.copy_(self.S)
            else:
                torch.mul(self.S, scale, out=self.G)
            for p in touched:
                p.grad = self.gview(p)
        else:   # some gradients are alive (e.g. the architect step left them): accumulate parameter by parameter
            for p in touched:
                s = self.sview(p)
                if p.grad is None:
                    g = self.gview(p)
                    g.copy_(s) if scale == 1.0 else torch.mul(s, scale, out=g)
                    p.grad = g
                else:
                    p.grad.add_(s, alpha=scale)
        self.S.zero_()
        self.dirty = False


class _PlanAlpha:
    """stands for one row of softmax(alpha) during a planned pass; `take_slot` hands a MixedOp its static weight slot"""

    def __init__(self, ctx, scale, row):
        self.ctx, self.scale, self.row = ctx, scale, row

    def take_slot(self, r_in, r_out):
        return self.ctx._next_wslot(self.scale, self.row, r_in, r_out)


_PEER_REGIONS = 0


class PassContext:
    """Everything static about one (architecture, input shape): slots, device tables, packed weights, graphs."""

    def __init__(self, model, arch_idx, flat, x_shape, capture, index=0):
        self.model, self.arch_idx, self.flat, self.capture, self.index = model, arch_idx, flat, capture, index
        # peer-exchange regions (csrc/peer.cu) are process-wide: forward / backward of every pass context ever built get their own ids
        # (the construction order is the same on every rank)
        global _PEER_REGIONS
        self._peer_regions = (_PEER_REGIONS, _PEER_REGIONS + 1)
        _PEER_REGIONS += 2
        self.dev = flat.S.device
        L = model._layers
        self.rows = (L - 1, L - 1, L - 2)
        self.slot_base = (0, L - 1, 2 * (L - 1))
        self.n_slots = sum(self.rows)
        self.width_idx = torch.zeros(self.n_slots, device=self.dev, dtype=torch.int32)
        self.sym_ratios = [[engine.SymRatio(self.slot_base[s] + r) for r in range(self.rows[s])] for s in range(3)]
        self.X = torch.zeros(x_shape, device=self.dev, dtype=torch.float32)
        self._wmeta, self._bmeta = [], []       # (alpha flat row, in slot, out slot) / (beta flat row)
        # static mixing-weight slots: row i of Wbuf / Bbuf is what the i-th MixedOp / beta mix of the pass reads; each slot is a
        # leaf view of its row, so the tape returns its gradient
        self.Wbuf = torch.full((1024, 5), 0.2, device=self.dev, dtype=torch.float32)
        self.Bbuf = torch.full((256, 2), 0.5, device=self.dev, dtype=torch.float32)
        self._wslots, self._bslots = [], []
        self._wcount = self._bcount = 0
        self._packs, self._pack_list = {}, []
        self._sel, self._sel_tables = {}, {}
        self.static_touched = {}               # id -> Parameter staged by this context outside device-selected sets
        # independent ops of a MixedOp / the two MixedOps of a Cell run on side streams (GPU only): the pass is a chain of ~8 000
        # kernels that each occupy a fraction of the machine for a few microseconds
        self.use_streams = self.dev.type == "cuda" and os.environ.get("FSB_GRAPH_STREAMS", "1") != "0"
        self._streams, self._stream_cursor, self._child_top = [], 0, 0
        self.built = False
        self.graphs = None
        self._pack_versions = None
        # alpha rows flattened over scales: scale s row r -> arow_base[s] + r
        self.arow_base = (0, L, 2 * L - 1)
        self.brow_base = (None, 0, L - 2)

    # ---- engine-facing API (engine.graph_ctx()) -------------------------------------------------------------------
    def stage(self, p):
        self.static_touched[id(p)] = p
        return self.flat.sview(p)

    def packed(self, conv, ci, co, dgrad):
        key = (id(conv), ci, co, dgrad)
        t = self._packs.get(key)
        if t is None:
            assert not self._capturing, "weight pack requested during capture that the warm-up pass did not see"
            pack = F_.pack_conv_weight_dgrad if dgrad else F_.pack_conv_weight
            w = conv.weight.detach()
            t = pack(w if w.dtype == torch.float32 else w.float(), ci, co, conv.kernel_size[0])
            self._packs[key] = t
            self._pack_list.append((conv, ci, co, dgrad, t))
        return t

    def sel_bn(self, usbn, slot):
        key = (id(usbn), slot)
        s = self._sel.get(key)
        if s is None:
            s = engine.SelBN(usbn, slot, self)
            self._sel[key] = s
        return s

    def sel_table_ptr(self, sel):
        t = self._sel_tables.get(id(sel))
        if t is None:
            assert not self._capturing, "BatchNorm table requested during capture that the warm-up pass did not see"
            arr = (_lib.BnSel * len(sel.bns))()
            for i, bn in enumerate(sel.bns):
                arr[i].gamma, arr[i].beta = bn.weight.data_ptr(), bn.bias.data_ptr()
                arr[i].running_mean, arr[i].running_var = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
                arr[i].num_batches_tracked = bn.num_batches_tracked.data_ptr() if bn.num_batches_tracked is not None else None
                arr[i].dgamma = self.flat.sview(bn.weight).data_ptr()
                arr[i].dbeta = self.flat.sview(bn.bias).data_ptr()
                arr[i].C = bn.num_features
            raw = bytes(arr)
            t = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.dev)
            self._sel_tables[id(sel)] = t
        return t.data_ptr()

    def width_idx_ptr(self, slot):
        return self.width_idx.data_ptr() + 4 * slot

    _capturing = False

    # ---- plan: what _forward asks for instead of computing distributions ------------------------------------------------
    def alpha(self, scale, row):
        return _PlanAlpha(self, scale, row)

    def _slot_of(self, r):
        return r.slot if isinstance(r, engine.SymRatio) else self.n_slots      # index n_slots = constant score 1

    def _next_wslot(self, scale, row, r_in, r_out):
        i = self._wcount
        self._wcount += 1
        meta = (self.arow_base[scale] + row, self._slot_of(r_in), self._slot_of(r_out))
        if i == len(self._wslots):
            assert not self.built and i < self.Wbuf.shape[0]
            self._wmeta.append(meta)
            self._wslots.append(self.Wbuf[i].detach().requires_grad_(True))
        assert self._wmeta[i] == meta, "the pass changed shape between builds"
        return self._wslots[i]

    def beta(self, scale, row):
        i = self._bcount
        self._bcount += 1
        meta = self.brow_base[scale] + row
        if i == len(self._bslots):
            assert not self.built and i < self.Bbuf.shape[0]
            self._bmeta.append(meta)
            self._bslots.append(self.Bbuf[i].detach().requires_grad_(True))
        assert self._bmeta[i] == meta
        return self._bslots[i]

    def parallel(self, thunks):
        """run independent pieces of the pass concurrently: thunk i on its own side stream, forked from and joined to the
        current stream with events.  Stream indices are assigned by CALL STRUCTURE: the thunks of one call get consecutive
        indices, everything a thunk forks in turn is numbered above all indices its earlier siblings used, and two calls made one
        after the other inside the same thunk get the SAME indices.  So a module always runs on the same stream: the two
        invocations of a twice-run cell (model_search.py:326-329) stay ordered -- BatchNorm running statistics are updated in
        program order and the in-place gradient accumulations of the backward never race."""
        if not self.use_streams or len(thunks) < 2:
            return [t() for t in thunks]
        base = self._stream_cursor
        top = base + len(thunks)
        while len(self._streams) < top:
            self._streams.append(torch.cuda.Stream(device=self.dev))
        main = torch.cuda.current_stream()
        fork = torch.cuda.Event()
        fork.record(main)
        outs, joins = [], []
        try:
            for i, t in enumerate(thunks):
                s = self._streams[base + i]
                s.wait_event(fork)
                self._stream_cursor = top          # whatever this thunk forks is numbered above its earlier siblings' forks
                self._child_top = top
                with torch.cuda.stream(s):
                    outs.append(t())
                    e = torch.cuda.Event()
                    e.record(s)
                    joins.append(e)
                top = max(top, self._child_top)
        finally:
            self._stream_cursor = base
            self._child_top = max(getattr(self, "_child_top", 0), top)
        for e in joins:
            main.wait_event(e)
        return outs

    # ---- one planned forward + backward on the tape ------------------------------------------------------------------
    def _peer_begin(self, direction):
        """data parallel: the SyncBN exchanges of this pass belong to one region of the peer-memory protocol (csrc/peer.cu)"""
        if engine.dp_native():
            _lib.check(_lib.lib().fsb_peer_begin(self._peer_regions[direction], F_._stream()), "fsb_peer_begin")

    def _run_forward(self):
        self._wcount = self._bcount = 0
        self._peer_begin(0)
        tape = AG.Tape(streams=self.use_streams)
        prev_tape, prev_ctx = AG._TAPE, engine._GRAPH_CTX
        AG._TAPE, engine._GRAPH_CTX = tape, self
        try:
            with torch.no_grad():
                outs = self.model._forward(self.X, plan=self)
        finally:
            AG._TAPE, engine._GRAPH_CTX = prev_tape, prev_ctx
        return tape, list(outs)

    def _run_backward(self, tape, outs, dlogits):
        self._peer_begin(1)
        prev_ctx = engine._GRAPH_CTX
        engine._GRAPH_CTX = self
        try:
            with torch.no_grad():
                leaves = tape.backward({id(o): g for o, g in zip(outs, dlogits)})
                dW = [None] * len(self._wslots)
                dB = [None] * len(self._bslots)
                wid = {id(t): i for i, t in enumerate(self._wslots)}
                bid = {id(t): i for i, t in enumerate(self._bslots)}
                for key, (t, g) in leaves.items():
                    if key in wid:
                        dW[wid[key]] = g
                    elif key in bid:
                        dB[bid[key]] = g
                    else:   # a parameter whose gradient came back as a tensor (BatchNorm of fixed-width units, conv bias)
                        self.stage(t).add_(g.to(torch.float32).reshape(t.shape))
        finally:
            engine._GRAPH_CTX = prev_ctx
        zero5 = torch.zeros(5, device=self.dev)
        zero2 = torch.zeros(2, device=self.dev)
        return (torch.stack([g if g is not None else zero5 for g in dW]) if dW else None,
                torch.stack([g if g is not None else zero2 for g in dB]) if dB else None)

    def _weight_versions(self):
        return (engine.WEIGHTS_EPOCH,) + tuple(c.weight._version for c, _, _, _, _ in self._pack_list)

    def _repack(self):
        for conv, ci, co, dgrad, t in self._pack_list:
            pack = F_.pack_conv_weight_dgrad if dgrad else F_.pack_conv_weight
            w = conv.weight.detach()
            fresh = pack(w if w.dtype == torch.float32 else w.float(), ci, co, conv.kernel_size[0], out=t)
            assert fresh.data_ptr() == t.data_ptr()

    def build(self):
        """warm-up pass (creates slots, tables, packs; its side effects on BatchNorm buffers and the staging buffer are undone),
        then -- on a GPU -- capture of the pack / forward / backward graphs."""
        model = self.model
        buffers = {k: v.clone() for k, v in model.state_dict().items() if "running_" in k or "num_batches_tracked" in k}
        staged = self.flat.S.clone() if self.flat.dirty else None
        tape, outs = self._run_forward()
        self.dlogits = [torch.zeros_like(o) for o in outs]
        self._run_backward(tape, outs, self.dlogits)     # warm-up of the backward kernels (tables for dgrad packs etc.)
        del tape, outs
        with torch.no_grad():
            sd = model.state_dict()
            for k, v in buffers.items():
                sd[k].copy_(v)
            if staged is not None:
                self.flat.S.copy_(staged)
            else:
                self.flat.S.zero_()
        dev = self.dev
        self.w_arow = torch.tensor([m[0] for m in self._wmeta], device=dev, dtype=torch.long)
        self.w_in = torch.tensor([m[1] for m in self._wmeta], device=dev, dtype=torch.long)
        self.w_out = torch.tensor([m[2] for m in self._wmeta], device=dev, dtype=torch.long)
        self.b_row = torch.tensor(self._bmeta, device=dev, dtype=torch.long)
        # device-selected BatchNorm sets: parameter indices [unit, width, (gamma, beta)] into flat.params for the touched-set
        sels = list(self._sel.values())
        self.sel_slots = np.array([s.slot for s in sels], dtype=np.int64)
        self.sel_param_index = np.array([[[self.flat.index[id(b.weight)], self.flat.index[id(b.bias)]] for b in s.bns] for s in sels],
                                        dtype=np.int64).reshape(len(sels), -1, 2)
        for s in sels:      # their gradient slots are reached through the tables, not through stage()
            for b in s.bns:
                self.static_touched.pop(id(b.weight), None)
                self.static_touched.pop(id(b.bias), None)
        self.static_index = np.array(sorted(self.flat.index[i] for i in self.static_touched), dtype=np.int64)
        self.built = True
        if self.capture:
            self._capture()
        self._pack_versions = self._weight_versions()

    def _capture(self):
        pool = torch.cuda.graph_pool_handle()
        self.g_pack, self.g_fwd, self.g_bwd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        self._capturing = True
        # No automatic garbage collection while capturing: an unreachable earlier pass whose graphs the cyclic collector frees in
        # the middle of a capture destroys them while a stream is capturing, which invalidates this capture.  Collect first, so
        # that such passes are freed here instead.
        gc.collect()
        gc_enabled = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(self.g_pack, pool=pool):
                self._repack()
            with torch.cuda.graph(self.g_fwd, pool=pool):
                self._tape, self.outs = self._run_forward()
            with torch.cuda.graph(self.g_bwd, pool=pool):
                self.dW, self.dB = self._run_backward(self._tape, self.outs, self.dlogits)
        finally:
            self._capturing = False
            if gc_enabled:
                gc.enable()
        self.graphs = (self.g_pack, self.g_fwd, self.g_bwd)

    # ---- per-step execution ----------------------------------------------------------------------------------------
    def forward(self, x):
        if self._weight_versions() != self._pack_versions:
            if self.capture:
                self.g_pack.replay()
            else:
                self._repack()
            self._pack_versions = self._weight_versions()
        self.X.copy_(x)
        if self.capture:
            self.g_fwd.replay()
        else:
            self._tape, self.outs = self._run_forward()
        return self.outs

    def backward(self, dl):
        for buf, g in zip(self.dlogits, dl):
            buf.copy_(g)
        if self.capture:
            self.g_bwd.replay()
        else:
            self.dW, self.dB = self._run_backward(self._tape, self.outs, self.dlogits)
            self._tape = None
        return self.dW, self.dB


class _Release(torch.autograd.Function):
    """loss value with a backward that (1) hands the mixing-weight gradients of every pass to torch autograd (-> alphas, betas,
    ratios) and (2) releases the staged weight gradients into param.grad."""

    @staticmethod
    def forward(ctx, value, anchor, runner, *mix):
        ctx.runner = runner
        return value.clone()

    @staticmethod
    def backward(ctx, gout):
        runner = ctx.runner
        ctx.runner = None
        grads = runner._release(gout)
        return (None, None, None) + tuple(grads)


class GraphedLoss:
    """`Network_Multi_Path._loss` in graph mode (see module docstring)."""

    def __init__(self, model, capture=None):
        self.model = model
        self.capture = torch.cuda.is_available() if capture is None else capture
        self.flat = FlatGrads(model)
        self.contexts = {}
        self.anchor = torch.zeros((), device=self.flat.S.device, requires_grad=True)
        self._pending = None

    def _context(self, arch_idx, x):
        key = (arch_idx, tuple(x.shape))
        ctx = self.contexts.get(key)
        if ctx is None:
            ctx = PassContext(self.model, arch_idx, self.flat, tuple(x.shape), self.capture, index=len(self.contexts))
            with torch.no_grad():
                ctx.X.copy_(x)
            ctx.build()
            self.contexts[key] = ctx
        return ctx

    # width sampling of one pass -> (int32 index vector [n_slots] on the device, score vector [n_slots + 1] with grad or None)
    def _sample(self, ctx, mode):
        model = self.model
        choices = model._width_mult_list
        dev = ctx.dev
        if mode == "arch_ratio":
            params = [getattr(model, name) for name in model._arch_names[model.arch_idx]["ratios"]]
            # one CPU draw per row in the reference's order (model_search.py:14-17,214-228), then ONE host->device copy
            uniform = torch.stack([torch.rand(p.shape[1]) for p, n in zip(params, ctx.rows) for _ in range(n)]).to(dev)
            logits = torch.cat([F.log_softmax(p[:n], dim=-1) for p, n in zip(params, ctx.rows)])
            noisy = logits - torch.log(1e-20 - torch.log(uniform + 1e-20))
            soft = F.softmax(noisy, dim=-1)
            winner = soft.max(dim=-1)[1]
            one_hot = torch.zeros_like(soft).scatter_(1, winner.view(-1, 1), 1)
            hard = (one_hot - soft).detach() + soft
            score = hard.gather(1, winner.view(-1, 1)).view(-1)
            return winner.to(torch.int32), torch.cat([score, torch.ones(1, device=dev)])
        if mode == "max":
            idx = np.full(ctx.n_slots, len(choices) - 1, dtype=np.int32)
        elif mode == "min":
            idx = np.zeros(ctx.n_slots, dtype=np.int32)
        else:   # "random": same draws, same order as model_search.py:254-260
            idx = np.array([choices.index(np.random.choice(choices)) for _ in range(ctx.n_slots)], dtype=np.int32)
        return torch.from_numpy(idx).to(dev), None

    def loss(self, input, target, passes):
        """passes: [(architecture to switch to | None, width mode | None)] exactly as Network_Multi_Path._loss builds them"""
        model = self.model
        self.flat.begin()
        total = 0
        mix, records = [], []
        for arch, mode in passes:
            if arch is not None:
                model.arch_idx = arch
            model.prun_mode = mode
            ctx = self._context(model.arch_idx, input)
            idx, score = self._sample(ctx, model._current_mode())
            alphas, betas = model._distributions()
            A = torch.cat(alphas)                                   # [sum rows, 5]
            W = A[ctx.w_arow]
            if score is not None:
                W = W * (score[ctx.w_in] * score[ctx.w_out]).unsqueeze(1)
            Bm = torch.cat(betas[1:])[ctx.b_row] if len(ctx._bmeta) else None
            with torch.no_grad():
                ctx.width_idx.copy_(idx)
                ctx.Wbuf[:W.shape[0]].copy_(W)
                if Bm is not None:
                    ctx.Bbuf[:Bm.shape[0]].copy_(Bm)
            outs = ctx.forward(input)
            logits = [o.detach().requires_grad_(True) for o in outs]
            with torch.enable_grad():
                loss_i = sum(model._criterion(l, target) for l in logits)
            dl = torch.autograd.grad(loss_i, logits)
            dW, dB = ctx.backward(dl)
            total = total + loss_i.detach()
            mix.append(W)
            records.append((ctx, idx, dW.clone() if dW is not None else None))
            if Bm is not None:
                mix.append(Bm)
                records.append((None, None, dB.clone()))
        self._pending = records
        return _Release.apply(total, self.anchor, self, *mix)

    def _release(self, gout):
        records, self._pending = self._pending, None
        scale = float(gout)     # loss.backward() passes 1; a scaled loss is honoured
        grads = []
        touched = np.zeros(len(self.flat.params), dtype=bool)
        for ctx, idx, dmix in records:
            grads.append(dmix * gout if dmix is not None else None)
            if ctx is None:
                continue
            touched[ctx.static_index] = True
            if len(ctx.sel_slots):
                w = idx.cpu().numpy()[ctx.sel_slots]
                touched[ctx.sel_param_index[np.arange(len(w)), w].reshape(-1)] = True
        params = self.flat.params
        world = engine.dp_world_size()
        if world > 1:
            # data parallel: ONE all-reduce of the flat staging buffer (the whole step's gradients, 4 bytes per parameter) and the
            # mean over ranks folded into the release scale; mixing-weight gradients likewise (tiny)
            torch.distributed.all_reduce(self.flat.S)
            scale = scale / world
            for g in grads:
                if g is not None:
                    torch.distributed.all_reduce(g)
                    g.div_(world)
        self.flat.release([params[i] for i in np.nonzero(touched)[0]], scale)
        return grads
