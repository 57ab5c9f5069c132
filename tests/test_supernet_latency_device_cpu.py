"""K14 without a GPU: the walk (`Network_Multi_Path._latency_walk`, the CPU path of forward_latency) against the reference's values
AND gradients (oracle/make_golden_latency_grad.py), the traced plan run through a float32 numpy restatement of the two kernels
(csrc/latency.cu) against the walk, the plan cache and its fallback, the host-side random draws, and the ctypes marshalling."""
import ctypes as C

import numpy as np
import pytest
import torch

from fasterseg_b200 import _lib
from fasterseg_b200 import functional as F_
from fasterseg_b200 import operations
from fasterseg_b200 import supernet_latency as SL
from oracle import make_golden_latency as mk
from oracle import make_golden_latency_grad as mkg
from oracle.make_golden_decode import SyntheticLatencyTable
from tests import helpers as H
from tests.test_marshalling_cpu import FakeLib

GOLD = H.load_npz("supernet_latency_grad.npz")
IDS = lambda c: "L%d-%dx%d" % (c["layers"], c["hw"][0], c["hw"][1])  # noqa: E731


def _model(case, monkeypatch):
    from fasterseg_b200.model_search import Network_Multi_Path
    monkeypatch.setattr(operations, "latency_lookup_table", SyntheticLatencyTable())
    model = mk.build(Network_Multi_Path, case["layers"])
    mk.randomise_arch(model, case["seed"])
    return model


def assert_matches(got, want, what):
    """value within rel 2e-6; every gradient within 1e-5 * max|g| of its tensor; the same None pattern.  The gradient tolerance
    has a floor at float32 rounding of the latency (1e-6 * value): where two invocations of a cell have the same latency, the
    beta gradient is b_j * (k - (b_0 + b_1) * k), zero in real arithmetic and rounding noise of the order of k in float32."""
    assert got.keys() == want.keys(), what
    for k in want:
        if k.endswith("/value"):
            assert got[k][0] == pytest.approx(want[k][0], rel=2e-6), (what, k)
        elif k.endswith("/none"):
            assert (got[k] == want[k]).all(), (what, k, got[k], want[k])
        else:
            value = abs(float(want[k[:k.rindex("/") + 1] + "value"][0]))
            tol = max(1e-5 * float(np.abs(want[k]).max()), 1e-6 * value)
            assert np.abs(got[k] - want[k]).max() <= tol, (what, k, np.abs(got[k] - want[k]).max(), tol)


def golden_of(case):
    g = GOLD
    pre = "%d/" % case["seed"]
    return {k: g[k] for k in g.files if k.startswith(pre)}


@pytest.mark.parametrize("case", mk.CASES, ids=IDS)
def test_walk_value_and_gradients_match_reference(case, monkeypatch):
    model = _model(case, monkeypatch)
    assert_matches(mkg.evaluate_grad(model, case), golden_of(case), IDS(case))


# ---- float32 restatement of csrc/latency.cu ---------------------------------------------------------------------------------
def _f(h, off, n):
    return h[off:off + n].view(np.float32)


def interpret(plan, params, noise):
    """-> (value, [8 gradients | None]) of the plan, in float32 like the kernels"""
    h = plan.host.numpy()
    f32 = np.float32
    nw, flags = int(h[SL.H_NW]), int(h[SL.H_FLAGS])
    arows, brows, rrows = h[SL.H_AROWS:SL.H_AROWS + 3], h[SL.H_BROWS:SL.H_BROWS + 2], h[SL.H_RROWS:SL.H_RROWS + 3]
    P = [p.detach().numpy().astype(np.float32) for p in params]
    A = np.concatenate([P[i].reshape(-1, 5) for i in range(3)]) if flags & SL.F_ALPHA else np.zeros((sum(arows), 5), f32)
    A = (np.exp(A - A.max(1, keepdims=True)) / np.exp(A - A.max(1, keepdims=True)).sum(1, keepdims=True)).astype(f32) \
        if flags & SL.F_ALPHA else np.full((sum(arows), 5), f32(0.2))
    B = np.concatenate([P[3 + i].reshape(-1, 2) for i in range(2)]) if flags & SL.F_BETA else None
    B = (np.exp(B - B.max(1, keepdims=True)) / np.exp(B - B.max(1, keepdims=True)).sum(1, keepdims=True)).astype(f32) \
        if flags & SL.F_BETA else np.full((sum(brows), 2), f32(0.5))
    RR = int(sum(rrows))
    noise = noise.numpy()
    if flags & SL.F_SAMPLED:
        Rp = np.concatenate([P[5 + i].reshape(-1, nw) for i in range(3)])
        pi = np.exp(Rp - Rp.max(1, keepdims=True))
        pi = (pi / pi.sum(1, keepdims=True)).astype(f32)
        g = -np.log(f32(1e-20) - np.log(noise.reshape(RR, nw) + f32(1e-20)))
        z = np.log(pi) + g
        soft = np.exp(z - z.max(1, keepdims=True))
        soft = (soft / soft.sum(1, keepdims=True)).astype(f32)
        win = soft.argmax(1)
        sw = soft[np.arange(RR), win]
        score = (f32(1) - sw) + sw
    else:
        win, score = noise.astype(np.int64), np.ones(RR, f32)
    M, NR, NI = int(h[SL.H_TERMS]), int(h[SL.H_REGS]), int(h[SL.H_INSTRS])
    terms = h[h[SL.H_OFF_TERMS]:h[SL.H_OFF_TERMS] + 4 * M].reshape(M, 4)
    lat_all = h[h[SL.H_OFF_LAT]:].view(np.float32)
    ins = h[h[SL.H_OFF_INSTR]:h[SL.H_OFF_INSTR] + 4 * NI].reshape(NI, 4)
    reg = np.zeros(NR, f32)
    reg[:int(h[SL.H_CONSTS])] = _f(h, int(h[SL.H_OFF_CONST]), int(h[SL.H_CONSTS]))
    rb, rt, ri = int(h[SL.H_REG_BETA]), int(h[SL.H_REG_TERM]), int(h[SL.H_REG_INSTR])
    reg[rb:rb + B.size] = B.reshape(-1)

    def side(r):
        return (int(win[r]), score[r]) if r >= 0 else (0, f32(1))

    def lat(tm):
        (i, si), (j, so) = side(tm[1]), side(tm[2])
        return lat_all[tm[3]:tm[3] + 5 * nw * nw].reshape(5, nw, nw)[:, i, j], si, so

    for m, tm in enumerate(terms):
        l, si, so = lat(tm)
        reg[rt + m] = np.sum(l * (A[tm[0]] * si * so), dtype=f32)
    for i, (op, a, b, _) in enumerate(ins):
        reg[ri + i] = reg[a] + reg[b] if op == SL.ADD else reg[a] * reg[b]
    value = reg[int(h[SL.H_OUT])]

    adj = np.zeros(NR, f32)
    adj[int(h[SL.H_OUT])] = 1
    for i in range(NI - 1, -1, -1):
        op, a, b, _ = ins[i]
        d = adj[ri + i]
        if op == SL.ADD:
            adj[a] += d
            adj[b] += d
        else:
            va, vb = reg[a], reg[b]
            adj[a] += d * vb
            adj[b] += d * va
    dA, dS = np.zeros_like(A), np.zeros(RR, f32)
    for m, tm in enumerate(terms):
        l, si, so = lat(tm)
        g_m = adj[rt + m]
        dA[tm[0]] += g_m * l * so * si
        if tm[1] >= 0:
            dS[tm[1]] += g_m * np.sum(l * A[tm[0]]) * so
        if tm[2] >= 0:
            dS[tm[2]] += g_m * np.sum(l * A[tm[0]]) * si
    grads = [None] * 8

    def split(x, counts, width, first):
        at = 0
        for n, c in enumerate(counts):
            grads[first + n] = x[at:at + c].reshape(c, width)
            at += c

    if flags & SL.F_ALPHA:
        split(A * (dA - (A * dA).sum(1, keepdims=True)), arows, 5, 0)
    if flags & SL.F_BETA:
        dB = adj[rb:rb + B.size].reshape(-1, 2)
        d = B[:, 0] * B[:, 1] * (dB[:, 0] - dB[:, 1])
        split(np.stack([d, -d], 1), brows, 2, 3)
    if flags & SL.F_SAMPLED:
        dsoft = np.zeros_like(soft)
        dsoft[np.arange(RR), win] = dS
        dz = soft * (dsoft - (soft * dsoft).sum(1, keepdims=True))
        split(dz - pi * dz.sum(1, keepdims=True), rrows, nw, 5)
    return value, grads


def evaluate_plan(model, case):
    """mkg.evaluate_grad's record, computed by tracing the plan and interpreting it (same seeds, same host draws)"""
    out = {}
    H_, W = case["hw"]
    for arch_idx in (0, 1):
        for flags in mk.FLAGS:
            model.arch_idx, model.prun_mode = arch_idx, None
            names, params = mkg.arch_tensors(model, arch_idx)
            mode = model._current_mode() if flags[2] else "max"
            plan = SL.plan_for(model, (3, H_, W), *flags, mode)
            torch.manual_seed(case["seed"] * 7 + arch_idx)
            np.random.seed(case["seed"] * 11 + arch_idx)
            value, grads = interpret(plan, params, SL.draw(model, plan, pin=False))
            diff = SL.differentiated(plan, params)
            key = "%d/a%d.%d%d%d/" % ((case["seed"], arch_idx) + tuple(int(f) for f in flags))
            out[key + "value"] = np.array([float(value)], np.float64)
            out[key + "none"] = np.array([not d for d in diff], np.uint8)
            for n, g, d in zip(names, grads, diff):
                if d:
                    out[key + n] = g
    return out


@pytest.mark.parametrize("case", mk.CASES, ids=IDS)
def test_plan_interpreter_matches_walk(case, monkeypatch):
    model = _model(case, monkeypatch)
    walk = mkg.evaluate_grad(model, case)
    assert_matches(evaluate_plan(model, case), walk, IDS(case))


# ---- plan cache and fallback --------------------------------------------------------------------------------------------------
def test_plan_cache_keys(monkeypatch):
    model = _model(mk.CASES[0], monkeypatch)
    model.arch_idx = 1
    p = SL.plan_for(model, (3, 256, 512), True, True, True, "arch_ratio")
    assert p is not None and p.sampled
    assert SL.plan_for(model, (3, 256, 512), True, True, True, "arch_ratio") is p
    others = [SL.plan_for(model, (3, 512, 512), True, True, True, "arch_ratio"),
              SL.plan_for(model, (3, 256, 512), False, True, True, "arch_ratio"),
              SL.plan_for(model, (3, 256, 512), True, True, True, "random")]
    model.arch_idx = 0
    others.append(SL.plan_for(model, (3, 256, 512), True, True, True, "arch_ratio"))
    model.arch_idx = 1
    monkeypatch.setattr(operations, "latency_lookup_table", SyntheticLatencyTable())    # a new table object -> a new plan
    others.append(SL.plan_for(model, (3, 256, 512), True, True, True, "arch_ratio"))
    assert all(o is not None and o is not p for o in others) and len(set(map(id, others))) == len(others)
    assert not others[1].flags & SL.F_ALPHA and not others[2].sampled


class _Partial(SyntheticLatencyTable):
    """the synthetic table without the entries of one width"""

    def __init__(self, hole):
        super().__init__()
        self.hole = hole

    def __contains__(self, key):
        return self.hole not in key


def test_incomplete_table_takes_the_walk(monkeypatch, tmp_path):
    model = _model(mk.CASES[0], monkeypatch)
    model.arch_idx = 1
    measured = []
    monkeypatch.setattr(operations, "compute_latency", lambda layer, size, iterations=None: measured.append(size) or 1.0)
    monkeypatch.setattr(operations, "table_file_name", str(tmp_path / "table.npy"))
    hole = "_Cin128_"     # 8/12 of scale 1, 4/12 of scale 2: reachable only by sampling (the stem's widths are 32 and 64)
    monkeypatch.setattr(operations, "latency_lookup_table", _Partial(hole))
    assert SL.plan_for(model, (3, 256, 512), True, True, True, "arch_ratio") is None and not measured   # never measures
    assert SL.plan_for(model, (3, 256, 512), True, True, False, "max") is not None    # forced max width: the hole is unreachable
    monkeypatch.setattr(SL, "usable", lambda *a: True)
    calls = []
    monkeypatch.setattr(SL, "expected_latency", lambda m, plan: calls.append(plan) or torch.tensor(0.))
    torch.manual_seed(1)
    for _ in range(3):    # gumbel sampling sooner or later draws the narrowest width: the walk measures and persists it
        model.forward_latency((3, 256, 512))
    assert not calls and measured and (tmp_path / "table.npy").exists()
    model.forward_latency((3, 256, 512), ratio=False)
    assert len(calls) == 1


# ---- host-side random draws ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["arch_ratio", "random", "max", "min"])
def test_draws_leave_the_walks_rng_state(mode, monkeypatch):
    model = _model(mk.CASES[1], monkeypatch)
    model.arch_idx = 1
    plan = SL.plan_for(model, (3, 224, 448), True, True, True, mode)
    torch.manual_seed(5)
    np.random.seed(6)
    ratios = model.sample_prun_ratio(mode=mode)
    want = torch.get_rng_state(), np.random.get_state()
    torch.manual_seed(5)
    np.random.seed(6)
    buf = SL.draw(model, plan, pin=False)
    assert torch.equal(torch.get_rng_state(), want[0])
    got_np = np.random.get_state()
    assert got_np[0] == want[1][0] and (got_np[1] == want[1][1]).all() and got_np[2:] == want[1][2:]
    wml = model._width_mult_list
    if mode == "arch_ratio":
        torch.manual_seed(5)
        rows = [torch.rand(len(wml)) for _ in range(plan.n_ratio_rows)]
        assert torch.equal(buf, torch.stack(rows))
        assert [int(r.argmax()) for row in ratios for r in row] == [int(i) for i in interpret_winners(plan, model, buf)]
    else:
        assert buf.tolist() == [float(wml.index(w)) for row in ratios for w in row]


def interpret_winners(plan, model, buf):
    """winners of the gumbel sample the kernel takes from `buf` (float32 restatement)"""
    Rp = torch.cat([model._arch("ratios", i).detach().reshape(-1, plan.n_w) for i in range(3)])
    g = -torch.log(1e-20 - torch.log(buf + 1e-20))
    return torch.softmax(torch.log_softmax(Rp, -1) + g, -1).argmax(-1)


# ---- ABI ----------------------------------------------------------------------------------------------------------------------
def test_workspace_bytes_is_host_math(monkeypatch):
    model = _model(mk.CASES[-1], monkeypatch)
    model.arch_idx = 1
    plan = SL.plan_for(model, (3, 1024, 2048), True, True, True, "arch_ratio")
    h = plan.host.numpy()
    RA, RR = int(h[SL.H_AROWS:SL.H_AROWS + 3].sum()), int(h[SL.H_RROWS:SL.H_RROWS + 3].sum())
    want = 4 * (int(h[SL.H_REGS]) + 5 * RA + RR * (2 * plan.n_w + 2))
    assert F_.supernet_latency_workspace_bytes(plan.host) == want
    bad = plan.host.clone()
    bad[SL.H_VERSION] = 99
    assert _lib.lib().fsb_supernet_latency_workspace_bytes(C.c_void_p(bad.data_ptr())) == 0


def test_marshalling(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_lib, "lib", lambda: lib)
    monkeypatch.setattr(F_, "_stream", lambda: 0)
    monkeypatch.setattr(F_, "_on_device", lambda t: True)
    plan_host = torch.zeros(64, dtype=torch.int32)
    plan = torch.zeros(64, dtype=torch.int32)
    params = [torch.empty(4, 5) for _ in range(3)] + [torch.empty(3, 2), None] + [torch.empty(4, 5) for _ in range(3)]
    noise, ws, out = torch.empty(20), torch.empty(100), torch.empty(())
    F_.supernet_latency_fwd(plan_host, plan, params, noise, ws, out)
    got = lib.last("fsb_supernet_latency_fwd")
    assert got[0] == plan_host.data_ptr() and got[1] == plan.data_ptr()
    assert got[2:10] == [None if p is None else p.data_ptr() for p in params]
    assert got[10:] == [noise.data_ptr(), ws.data_ptr(), out.data_ptr(), None]     # stream 0 arrives as NULL
    gout = torch.empty(())
    grads = [torch.empty(4, 5), None, None, None, None, torch.empty(4, 5), None, None]
    F_.supernet_latency_bwd(plan_host, plan, gout, ws, grads)
    got = lib.last("fsb_supernet_latency_bwd")
    assert got[:4] == [plan_host.data_ptr(), plan.data_ptr(), gout.data_ptr(), ws.data_ptr()]
    assert got[4:12] == [None if g is None else g.data_ptr() for g in grads]
    with pytest.raises(ValueError):
        F_.supernet_latency_fwd(plan_host, plan, params[:7] + [torch.empty(4, 5, dtype=torch.float64)], noise, ws, out)
