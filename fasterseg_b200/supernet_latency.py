"""K14: the supernet's expected latency (`Network_Multi_Path.forward_latency`, model_search.py:361-475) and its gradient as one
kernel launch each (csrc/latency.cu).

The Python walk (`Network_Multi_Path._latency_walk`) does scalar arithmetic on the device of the arch parameters: ~2 300 to
4 000 tiny kernels and up to 275 device->host reads per call, three calls per architect step.  Here the walk is traced ONCE per
(table, architecture, input size, switches, width mode, stem/head widths) into a compact plan:

* MixedOp terms: one per MixedOp invocation, ms = sum_k lat[k][w_in][w_out] * a_k * s_in * s_out, with the alpha row, the in / out
  ratio rows (or a forced width) and the [5 ops][n_w][n_w] latency slice of every width pair the mode can reach;
* the recurrence: the beta-weighted `pending` sums and `settle` updates of the walk as a straight-line program of ADD / MUL
  instructions over registers (constants, beta softmax values, term values, instruction results), recorded by running
  `_latency_walk` itself with symbolic values -- so the plan cannot drift from the walk.

The forward kernel takes the softmaxes, the gumbel width samples (uniforms drawn on the host exactly like `sample_prun_ratio`,
one pinned non-blocking copy), evaluates the terms in parallel and the program in one thread; the backward kernel runs the
program in reverse and folds the adjoints back through the softmaxes and the straight-through gumbel estimator.

The plan builder never measures: if any reachable key is missing from `operations.latency_lookup_table`, `plan_for` returns None
and forward_latency takes the walk, which measures and persists like the reference."""
import os

import numpy as np
import torch

from . import operations
from .genotypes import PRIMITIVES

ENABLED = os.environ.get("FSB_LATENCY_KERNEL", "1") != "0"   # 0: forward_latency always takes the walk

PLAN_VERSION = 1
HDR = 32
ADD, MUL = 0, 1
N_OPS = len(PRIMITIVES)
# header fields (int32 slots of the plan)
(H_VERSION, H_NW, H_AROWS, H_BROWS, H_RROWS, H_FLAGS, H_TERMS, H_REGS, H_INSTRS, H_OUT, H_CONSTS, H_OFF_CONST, H_OFF_TERMS,
 H_OFF_INSTR, H_OFF_LAT, H_OFF_APTR, H_OFF_AIDX, H_OFF_RPTR, H_OFF_RIDX, H_REG_BETA, H_REG_TERM, H_REG_INSTR, H_LEN) = (
    0, 1, 2, 5, 7, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27)
F_ALPHA, F_BETA, F_SAMPLED = 1, 2, 4


class Missing(KeyError):
    """a reachable latency-table key is absent"""


class _Tracer:
    def __init__(self):
        self.consts, self.const_ix = [], {}
        self.instrs = []      # (op, operand, operand); operands are ("c" | "b" | "t" | "i", index)
        self.terms = []       # (alpha row, in ratio row | -1, out ratio row | -1, lat [N_OPS, n_w, n_w])

    def const(self, v):
        v = float(np.float32(v))
        if v not in self.const_ix:
            self.const_ix[v] = len(self.consts)
            self.consts.append(v)
        return _Sym(self, ("c", self.const_ix[v]))

    def lift(self, x):
        return x if isinstance(x, _Sym) else self.const(x)

    def op(self, code, a, b):
        self.instrs.append((code, a.ref, b.ref))
        return _Sym(self, ("i", len(self.instrs) - 1))


class _Sym:
    """a scalar of the traced walk: records + and * into the tracer's program"""

    def __init__(self, tracer, ref):
        self.tr, self.ref = tracer, ref

    def __add__(self, o):
        if not isinstance(o, _Sym) and o == 0:
            return self
        return self.tr.op(ADD, self, self.tr.lift(o))

    def __radd__(self, o):
        if not isinstance(o, _Sym) and o == 0:
            return self
        return self.tr.op(ADD, self.tr.lift(o), self)

    def __mul__(self, o):
        return self.tr.op(MUL, self, self.tr.lift(o))

    def __rmul__(self, o):
        return self.tr.op(MUL, self.tr.lift(o), self)

    def __gt__(self, o):
        # `b[n] > 0`: the kernel runs every invocation; a softmax weight that underflowed to 0 contributes 0 * ms
        return True


class _Row:
    def __init__(self, index):
        self.index = index


class _BetaRow(_Row):
    def __init__(self, tracer, index):
        super().__init__(index)
        self.tr = tracer

    def __getitem__(self, j):
        assert j in (0, 1)
        return _Sym(self.tr, ("b", 2 * self.index + j))

    def __iter__(self):
        return iter((self[0], self[1]))


class _Chan:
    """channel count of a traced size: one value per width slot of the ratio row (or forced width) that produced it"""

    def __init__(self, side, by_slot):
        self.side, self.by_slot = side, by_slot

    def __eq__(self, o):
        return isinstance(o, _Chan) and o.side is self.side and o.by_slot == self.by_slot

    def __hash__(self):
        return hash(tuple(sorted(self.by_slot.items())))


def _rows(model):
    L = model._layers
    return (L, L - 1, L - 2), (L - 2, L - 3), (L - 1, L - 1, L - 2)


def reachable_slots(mode, n_w):
    return {"arch_ratio": range(n_w), "random": range(n_w), "max": [n_w - 1], "min": [0]}[mode]


def _sides(r, mode, wml):
    """(slot, width) pairs a ratio can take: every width the mode can draw for a ratio row, the one width of a forced ratio"""
    if isinstance(r, _Row):
        return [(i, wml[i]) for i in reachable_slots(mode, len(wml))]
    return [(0, r)]


def _trace(model, size, mode, table):
    tr = _Tracer()
    arows, brows, rrows = _rows(model)
    wml = model._width_mult_list
    n_w = len(wml)
    s = size
    for block in model.stem[model.arch_idx]:       # the walk sums the stem from the table too: check before it looks up
        name, s = block.latency_key(s)
        if name not in table:
            raise Missing(name)
    aoff = np.cumsum((0,) + arows)
    boff = np.cumsum((0,) + brows)
    roff = np.cumsum((0,) + rrows)
    alphas = [[_Row(int(aoff[s]) + r) for r in range(arows[s])] for s in range(3)]
    betas = [None] + [[_BetaRow(tr, int(boff[s]) + r) for r in range(brows[s])] for s in range(2)]
    ratios = [[_Row(int(roff[s]) + r) for r in range(rrows[s])] for s in range(3)]

    def mixed(mop, size, arow, r_in, r_out):
        c, h, w = size
        if isinstance(c, _Chan):
            assert c.side is r_in, "a cell reads its input at the width that produced it"
        lat = np.zeros((N_OPS, n_w, n_w), np.float64)
        by_slot, hw = {}, None
        for i, w_in in _sides(r_in, mode, wml):
            for j, w_out in _sides(r_out, mode, wml):
                mop.set_prun_ratio((w_in, w_out))
                for k, op in enumerate(mop._ops):
                    name, (co, ho, wo) = op.latency_key((c.by_slot[i] if isinstance(c, _Chan) else c, h, w))
                    if name not in table:
                        raise Missing(name)
                    lat[k, i, j] = table[name]
                    assert by_slot.setdefault(j, co) == co and (hw is None or hw == (ho, wo))
                    hw = (ho, wo)
        tr.terms.append((arow.index, r_in.index if isinstance(r_in, _Row) else -1, r_out.index if isinstance(r_out, _Row) else -1, lat))
        return _Sym(tr, ("t", len(tr.terms) - 1)), (_Chan(r_out, by_slot),) + hw

    def cell_latency(cell, size, a, r):
        # Cell.forward_latency with the two MixedOps recorded as terms
        assert (r[2] is not None) == bool(cell._down)
        keep = mixed(cell._op, size, a, r[0], r[1])
        down = mixed(cell.downsample, size, a, r[0], r[2]) if cell._down else None
        return keep, down

    total = model._latency_walk(size, alphas, betas, ratios, cell_latency)
    return tr, tr.lift(total), (arows, brows, rrows)


class Plan:
    """a traced walk: `host` (int32 CPU tensor; float sections bit-cast) and its copy on each device it ran on"""

    def __init__(self, host, table, mode, flags, rows, n_w):
        self.host, self.table, self.mode, self.flags, self.rows, self.n_w = host, table, mode, flags, rows, n_w
        self.sampled = bool(flags & F_SAMPLED)
        self.n_ratio_rows = sum(rows[2])
        self._dev = {}

    def on(self, device):
        d = self._dev.get(device)
        if d is None:
            d = self.host.to(device)
            self._dev[device] = d
        return d


def _pad4(n):
    return (n + 3) // 4 * 4


def build_plan(model, size, alpha, beta, ratio, mode, table=None):
    """trace the walk of the model's current architecture into a Plan; raises Missing if the table lacks a reachable key"""
    table = operations.latency_lookup_table if table is None else table
    tr, out, rows = _trace(model, tuple(size), mode, table)
    arows, brows, rrows = rows
    n_w = len(model._width_mult_list)
    RA, RB, RR = sum(arows), sum(brows), sum(rrows)
    M, NI, NC = len(tr.terms), len(tr.instrs), len(tr.consts)
    reg_beta, reg_term = NC, NC + 2 * RB
    reg_instr = reg_term + M
    base = {"c": 0, "b": reg_beta, "t": reg_term, "i": reg_instr}

    def reg(ref):
        return base[ref[0]] + ref[1]

    aptr, aidx = [[] for _ in range(RA)], []
    rptr, ridx = [[] for _ in range(RR)], []
    for t, (ar, ri, ro, _) in enumerate(tr.terms):
        aptr[ar].append(t)
        if ri >= 0:
            rptr[ri].append(2 * t)
        if ro >= 0:
            rptr[ro].append(2 * t + 1)

    def csr(lists):
        ptr, idx = [0], []
        for l in lists:
            idx += l
            ptr.append(len(idx))
        return ptr, idx

    aptr, aidx = csr(aptr)
    rptr, ridx = csr(rptr)
    secs = [("const", np.asarray(tr.consts, np.float32).view(np.int32)),
            ("terms", np.asarray([(ar, ri, ro, 0) for ar, ri, ro, _ in tr.terms], np.int32).reshape(-1)),
            ("instr", np.asarray([(c, reg(a), reg(b), 0) for c, a, b in tr.instrs], np.int32).reshape(-1)),
            ("lat", np.concatenate([lat.astype(np.float32).reshape(-1) for *_, lat in tr.terms]).view(np.int32)),
            ("aptr", np.asarray(aptr, np.int32)), ("aidx", np.asarray(aidx, np.int32)),
            ("rptr", np.asarray(rptr, np.int32)), ("ridx", np.asarray(ridx, np.int32))]
    offs, at = {}, HDR
    for name, arr in secs:
        offs[name] = at
        at = _pad4(at + arr.size)
    plan = np.zeros(at, np.int32)
    for name, arr in secs:
        plan[offs[name]:offs[name] + arr.size] = arr
    stride = N_OPS * n_w * n_w
    terms = plan[offs["terms"]:offs["terms"] + 4 * M].reshape(M, 4)
    terms[:, 3] = np.arange(M) * stride          # lat offset of each term inside the lat section
    sampled = ratio and mode == "arch_ratio"
    flags = (F_ALPHA if alpha else 0) | (F_BETA if beta else 0) | (F_SAMPLED if sampled else 0)
    hdr = {H_VERSION: PLAN_VERSION, H_NW: n_w, H_FLAGS: flags, H_TERMS: M, H_REGS: reg_instr + NI, H_INSTRS: NI, H_OUT: reg(out.ref),
           H_CONSTS: NC, H_OFF_CONST: offs["const"], H_OFF_TERMS: offs["terms"], H_OFF_INSTR: offs["instr"], H_OFF_LAT: offs["lat"],
           H_OFF_APTR: offs["aptr"], H_OFF_AIDX: offs["aidx"], H_OFF_RPTR: offs["rptr"], H_OFF_RIDX: offs["ridx"],
           H_REG_BETA: reg_beta, H_REG_TERM: reg_term, H_REG_INSTR: reg_instr, H_LEN: at}
    for k, v in hdr.items():
        plan[k] = v
    plan[H_AROWS:H_AROWS + 3] = arows
    plan[H_BROWS:H_BROWS + 2] = brows
    plan[H_RROWS:H_RROWS + 3] = rrows
    return Plan(torch.from_numpy(plan), table, mode, flags, rows, n_w)


def usable(model):
    """the kernel path applies: arch parameters of the current architecture are float32 on CUDA"""
    p = model._arch("alphas", 0)
    return ENABLED and p.is_cuda and p.dtype == torch.float32


def plan_for(model, size, alpha, beta, ratio, mode):
    """cached Plan for the model's current architecture, or None when the table lacks a reachable key"""
    table = operations.latency_lookup_table
    key = (id(table), model.arch_idx, tuple(size), bool(alpha), bool(beta), bool(ratio), mode,
           tuple(model._stem_head_width[model.arch_idx]))
    cache = model.__dict__.setdefault("_fsb_latency_plans", {})
    plan = cache.get(key)
    if plan is not None and plan.table is table:      # the plan holds the table, so its id cannot be reused while cached
        return plan
    try:
        plan = build_plan(model, size, alpha, beta, ratio, mode, table)
    except Missing:
        return None
    cache[key] = plan
    return plan


def draw(model, plan, pin=True):
    """the per-call random input of the kernel, drawn from the host generators exactly like `sample_prun_ratio(plan.mode)`:
    gumbel uniforms (one torch.rand(n_w) per ratio row, scale 0 rows first) in arch_ratio mode, else the width index of
    every row (numpy draws in 'random' mode)"""
    if plan.sampled:
        buf = torch.empty((plan.n_ratio_rows, plan.n_w), dtype=torch.float32, pin_memory=pin)
        size = torch.Size([plan.n_w])
        for i in range(plan.n_ratio_rows):
            torch.rand(size, out=buf[i])
        return buf
    wml = model._width_mult_list
    idx = [wml.index(w) for row in model.sample_prun_ratio(mode=plan.mode) for w in row]
    buf = torch.empty(len(idx), dtype=torch.float32, pin_memory=pin)
    buf.copy_(torch.tensor(idx, dtype=torch.float32))
    return buf


def arch_inputs(model):
    return [model._arch(kind, i) for kind, n in (("alphas", 3), ("betas", 2), ("ratios", 3)) for i in range(n)]


def differentiated(plan, params):
    """which of the 8 arch tensors the walk differentiates (the others keep .grad None, so Adam skips them)"""
    d = [bool(plan.flags & F_ALPHA)] * 3 + [bool(plan.flags & F_BETA)] * 2 + [plan.sampled] * 3
    return [di and p.numel() > 0 for di, p in zip(d, params)]


def expected_latency(model, plan):
    from . import autograd as AG
    params = arch_inputs(model)
    noise = draw(model, plan).to(params[0].device, non_blocking=True)
    diff = differentiated(plan, params)
    return AG.supernet_latency(plan, noise, [p if d else p.detach() for p, d in zip(params, diff)], diff)

