"""The conv data and weight gradients (fsb_conv_dgrad, fsb_conv_wgrad; csrc/train.cu, csrc/wgrad_tc.cu) through the C ABI, at
every geometry the training steps run (tests/golden/conv_bwd_census.json, at the drivers' batch) and on a synthetic grid of the
kernels' edges, on every path that can take each geometry.  Which kernel ran is read from torch.profiler.

Exact family (the main one): x, dy and w are sparse integers in {-1, 0, 1}, gscale = 1024 and the initial dw of accumulate = 1
is integers / 1024.  Every product and partial sum is then an integer far below 2^24, so fp32 accumulation is exact in any
order (atomics, pixel chunks, deterministic mode): dw must equal the float64 reference rounded to a multiple of 1/gscale and dx
the float64 reference (|dx| <= 2048, exact in fp16) bit for bit.  One missing, duplicated or misplaced contribution changes an
entry by at least 1/1024.

Random family: normal inputs against elementwise float64 bounds (u = 2^-24): dx within 2^-11 |ref| + (Cout k^2 + 2) u sum|dy||w|,
dw within (n + 6) u sum|x||dy| / gscale over n pixels -- only where n is small enough for that bound to mean something.

Buffer discipline: x and dy are channel slices of wider buffers whose other channels hold a sentinel; dx is a slice at channel
offset 8 of a buffer whose own channels start as NaN, with sentinels around it and a spare pixel after its end; dw is the
[:Cout, :Cin] corner of a wider fp32 master tensor.  Every owned element must be written and every other bit must survive.
"""
import collections
import ctypes as C

import pytest
import torch

from tests import conv_bwd_census as CC
from tests.conv_harness import (F64, INVALID, SENT16, SENT32, U, L, Options, Slice, _assert_kernels, _bits32, _cpad, _ints, _n_tile,
                                _normal, _out_size, _report, _s, profiled)

pytestmark = pytest.mark.gpu

GSCALE = 1024.0            # autograd.GRAD_SCALE


class G:
    """one backward conv geometry (the census fields; cstrides 0 = dense)"""

    def __init__(self, N, H, W, Cin, Cout, k, stride, pad, dil=1, off=(0, 0), x_cstride=0, dy_cstride=0, dx_cstride=0, w_stride_o=0,
                 accumulate=0, gscale=GSCALE, name=""):
        self.N, self.H, self.W, self.Cin, self.Cout, self.k, self.stride, self.pad, self.dil = N, H, W, Cin, Cout, k, stride, pad, dil
        self.off = tuple(off)
        self.Ho, self.Wo = _out_size(H, W, k, stride, pad, dil, self.off)
        self.xcs = x_cstride or _cpad(Cin)
        self.dcs = dy_cstride or _cpad(Cout)
        self.dxcs = dx_cstride or _cpad(Cin)
        self.cin_m = (w_stride_o or Cin * k * k) // (k * k)     # master weight's input channels (> Cin: a slimmable slice)
        self.accumulate, self.gscale, self.name = accumulate, gscale, name

    @classmethod
    def from_census(cls, g):
        return cls(g["N"], g["H"], g["W"], g["Cin"], g["Cout"], g["k"], g["stride"], g["pad"], g["dil"], (g["off_h"], g["off_w"]),
                   g["x_cstride"], g["dy_cstride"], g["dx_cstride"], g["w_stride_o"], g["accumulate"], g["gscale"] or GSCALE,
                   "%s/%s" % (g["run"], g["op"]))

    def __repr__(self):
        return ("%s N%d %dx%d ci%d co%d k%d s%d p%d d%d off%s cs(%d,%d,%d) cin_m%d acc%d g%g" %
                (self.name, self.N, self.H, self.W, self.Cin, self.Cout, self.k, self.stride, self.pad, self.dil, self.off, self.xcs,
                 self.dcs, self.dxcs, self.cin_m, self.accumulate, self.gscale))

    def desc(self, x_cstride, dy_cstride, flags=0):
        from fasterseg_b200 import _lib
        return _lib.ConvDesc(self.N, self.H, self.W, self.Cin, self.Cout, self.k, self.stride, self.pad, self.dil, self.off[0], self.off[1],
                             self.Ho, self.Wo, x_cstride, dy_cstride, flags)


# ---- which path a geometry takes (mirrors the routing of conv_dgrad_launch / conv_wgrad_launch / conv_plan) ------------------------
def _s2_planes(g):
    """-> [(Hl, Wl, ntaps)] of the four parity planes of a stride-2 dgrad"""
    out = []
    for ph in (0, 1):
        for pw in (0, 1):
            Hl, Wl = (g.H - ph + 1) // 2, (g.W - pw + 1) // 2
            n = sum(1 for r in range(g.k) for s in range(g.k)
                    if (ph - g.off[0] + g.pad - r * g.dil) % 2 == 0 and (pw - g.off[1] + g.pad - s * g.dil) % 2 == 0)
            out.append((Hl, Wl, n))
    return out


def _empty_wgrad_plane(g):
    """a stride-2 tap whose parity plane of x has no pixel (H or W of 1): the wgrad takes the direct kernel"""
    if g.stride != 2:
        return False
    for r in range(g.k):
        for s in range(g.k):
            ph, pw = (r - g.pad + g.off[0]) % 2, (s - g.pad + g.off[1]) % 2
            if (g.H - ph + 1) // 2 <= 0 or (g.W - pw + 1) // 2 <= 0:
                return True
    return False


def wgrad_paths(g, xcs, dcs, aligned=True):
    """-> [(path, flags, {option: value}, expected kernel counts)]"""
    from fasterseg_b200 import _lib
    zero = {} if g.accumulate else {"zero_wgrad_kernel": 1}
    direct = dict(zero, conv_wgrad_kernel=1)
    out = []
    for det in (-1, 1):
        opts = {"FSB_DETERMINISTIC": det}
        if g.k in (1, 3) and g.dil == 1 and g.Cin >= 16 and g.Cout >= 16 and xcs % 8 == 0 and dcs % 8 == 0 and aligned and \
                not _empty_wgrad_plane(g):
            ci64 = (g.Cin + 63) // 64 * 64
            out.append(("tc", 0, opts, dict(zero, **{"conv_wgrad_tc_kernel<%d>" % (128 if ci64 % 128 == 0 else 64): 1})))
            out.append(("direct", _lib.FSB_CONV_FORCE_DIRECT, opts, direct))
        else:
            out.append(("direct", 0, opts, direct))
    return out


def dgrad_paths(g, dcs, dxcs, aligned=True):
    from fasterseg_b200 import _lib
    direct = {"conv_dgrad_direct_kernel": 1}
    FD = _lib.FSB_CONV_FORCE_DIRECT
    if g.stride == 1 and g.off == (0, 0) and aligned and g.Cout >= 16 and dcs % 8 == 0:
        nt = _n_tile(g.Cin, g.H, g.W, g.N)
        out = [("tap", 0, {"FSB_CONV_TC2": -1}, {"conv_tc<%d>" % nt: 1})]
        if g.k == 3 and g.dil == 1:
            out.append(("window", 0, {"FSB_CONV_TC2": 1}, {"conv_tc_win<%d>" % nt: 1}))
        return out + [("direct", FD, {}, direct)]
    if g.stride == 2 and aligned and g.Cin % 8 == 0 and dxcs % 8 == 0 and dcs % 8 == 0 and g.Cout >= 16:
        exp = collections.Counter()
        for Hl, Wl, n in _s2_planes(g):
            if n and Hl > 0 and Wl > 0:
                exp["conv_tc<%d>" % _n_tile(g.Cin, Hl, Wl, g.N)] += 1
        return [("planes", 0, {"FSB_DGRAD_S2_DIRECT": -1}, dict(exp)), ("s2_direct", 0, {"FSB_DGRAD_S2_DIRECT": 1}, direct),
                ("direct", FD, {}, direct)]
    return [("direct", 0, {}, direct)]


def _ref_dgrad(g, dy, w):
    eff = (g.N, g.Cin, g.H - g.off[0], g.W - g.off[1])
    r = torch.nn.grad.conv2d_input(eff, w, dy, stride=g.stride, padding=g.pad, dilation=g.dil)
    dx = torch.zeros((g.N, g.Cin, g.H, g.W), dtype=F64, device="cuda")
    dx[:, :, g.off[0]:, g.off[1]:] = r
    return dx


def _ref_wgrad(g, x, dy):
    return torch.nn.grad.conv2d_weight(x[:, :, g.off[0]:, g.off[1]:], (g.Cout, g.Cin, g.k, g.k), dy, stride=g.stride, padding=g.pad,
                                       dilation=g.dil)


def _master(g, corner, fill_corner=None):
    """fp32 master weight (Cout + 8, cin_m, k, k) with `corner` in [:Cout, :Cin] and a sentinel elsewhere"""
    m = torch.full((g.Cout + 8, g.cin_m, g.k, g.k), SENT32, dtype=torch.float32, device="cuda")
    m[:g.Cout, :g.Cin] = corner if fill_corner is None else fill_corner
    return m


# ---- one run of each kernel -----------------------------------------------------------------------------------------------------
def run_wgrad(g, x, dy, dw0, flags, xoff=8, dyoff=8):
    """-> (rc, master after the call, master before it); x, dy: float64 NCHW on the device"""
    xs = Slice(g.N, g.H, g.W, g.Cin, g.xcs + 8, xoff, torch.float16, None, SENT16).put(x)
    ds = Slice(g.N, g.Ho, g.Wo, g.Cout, g.dcs + 8, dyoff, torch.float16, None, SENT16).put(dy)
    m = _master(g, None, dw0 if g.accumulate else float("nan"))
    before = m.clone()
    d = g.desc(g.xcs + 8, g.dcs + 8, flags)
    rc = L().fsb_conv_wgrad(C.byref(d), xs.ptr(), ds.ptr(), g.dcs + 8, m.data_ptr(), m.stride(0), m.stride(1), int(g.accumulate),
                            float(g.gscale), _s())
    return rc, m, before


def run_dgrad(g, dy, w, flags, dyoff=8, with_w=True):
    """-> (rc, dx Slice, its bits before the call)"""
    from fasterseg_b200 import functional as F_
    ds = Slice(g.N, g.Ho, g.Wo, g.Cout, g.dcs + 8, dyoff, torch.float16, None, SENT16).put(dy)
    m = _master(g, w.float())
    wt = F_.pack_conv_weight_dgrad(m, g.Cin, g.Cout, g.k)
    xs = Slice(g.N, g.H, g.W, g.Cin, g.dxcs + 8, 8, torch.float16, float("nan"), SENT16)
    before = xs.bits().clone()
    d = g.desc(g.dxcs + 8, g.dcs + 8, flags)
    rc = L().fsb_conv_dgrad(C.byref(d), ds.ptr(), g.dcs + 8, wt.data_ptr(), m.data_ptr() if with_w else None, m.stride(0), m.stride(1),
                            xs.ptr(), g.dxcs + 8, _s())
    return rc, xs, before


def _dw_expected(before, g, corner):
    exp = before.clone()
    exp[:g.Cout, :g.Cin] = corner.float()
    return exp


def exact_case(g, op, seed, fails, kernels):
    """every path of one geometry on exact operands; appends failure strings; counts the expected kernel launches"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if op == "wgrad":
        x = _ints((g.N, g.Cin, g.H, g.W), gen)
        dy = _ints((g.N, g.Cout, g.Ho, g.Wo), gen)
        dw0 = torch.randint(-8, 9, (g.Cout, g.Cin, g.k, g.k), generator=gen, device="cuda").to(F64) / g.gscale
        ref = torch.round(_ref_wgrad(g, x, dy)) / g.gscale + (dw0 if g.accumulate else 0.0)
        for path, flags, opts, exp in wgrad_paths(g, g.xcs + 8, g.dcs + 8):
            with Options(opts):
                rc, m, before = run_wgrad(g, x, dy, dw0, flags)
            kernels.update(exp)
            if rc != 0:
                fails.append("%r %s %s: rc %d %s" % (g, path, opts, rc, L().fsb_last_error_string()))
            elif not torch.equal(_bits32(m), _bits32(_dw_expected(before, g, ref))):
                bad = (_bits32(m) != _bits32(_dw_expected(before, g, ref)))
                fails.append("%r %s %s: %d dw bits differ (inside the corner %d)" % (g, path, opts, int(bad.sum()),
                                                                                   int(bad[:g.Cout, :g.Cin].sum())))
    else:
        dy = _ints((g.N, g.Cout, g.Ho, g.Wo), gen)
        w = _ints((g.Cout, g.Cin, g.k, g.k), gen)
        ref = torch.round(_ref_dgrad(g, dy, w))     # an integer sum: rounding removes any float64 algorithm noise
        assert float(ref.abs().max()) <= 2048, "%r: |dx| exceeds the fp16-exact range" % g
        for path, flags, opts, exp in dgrad_paths(g, g.dcs + 8, g.dxcs + 8):
            with Options(opts):
                rc, xs, before = run_dgrad(g, dy, w, flags)
            kernels.update(exp)
            if rc != 0:
                fails.append("%r %s %s: rc %d %s" % (g, path, opts, rc, L().fsb_last_error_string()))
                continue
            want = Slice(g.N, g.H, g.W, g.Cin, g.dxcs + 8, 8, torch.float16, None, SENT16)
            want.flat.view(torch.int16).copy_(before)
            want.put(ref)
            if not torch.equal(xs.bits(), want.bits()):
                bad = xs.bits() != want.bits()
                own = bad[:-(g.dxcs + 8)].view(g.N, g.H, g.W, g.dxcs + 8)[..., 8:8 + g.Cin]
                fails.append("%r %s %s: %d dx bits differ (%d owned, %d NaN left)" % (g, path, opts, int(bad.sum()), int(own.sum()),
                                                                                    int(torch.isnan(xs.view).sum())))


def _run_exact(geoms, op, seed0):
    def run():
        fails, expected = [], collections.Counter()
        for i, g in enumerate(geoms):
            exact_case(g, op, seed0 + i, fails, expected)
        return fails, expected
    (fails, expected), k = profiled(run)
    print("%s: %d geometries, kernels %s, %d stale records" % (op, len(geoms), dict(sorted(k.counts.items())), k.stale))
    assert not fails, "%d failures:\n%s" % (len(fails), "\n".join(fails[:12]))
    _assert_kernels(k.counts, expected)


# ---- the census ----------------------------------------------------------------------------------------------------------------
def _census(op):
    return [G.from_census(g) for g in CC.geometries() if g["op"] == op]


@pytest.mark.parametrize("op", ["wgrad", "dgrad"])
def test_census_exact(op):
    geoms = _census(op)
    assert len(geoms) > 100
    _run_exact(geoms, op, 1000 if op == "wgrad" else 5000)


# ---- synthetic edge grid: (purpose, geometry) ------------------------------------------------------------------------------------
EDGE = [
    # ci tile: 64 or 128 channels (ci64 % 128), ragged last ci tile
    *[("Cin%d" % ci, G(1, 20, 36, ci, 64, 3, 1, 1)) for ci in (16, 48, 96, 128, 192, 384)],
    # dy sub-tile wholly past Cout (co0 + 64 >= Cout); co_tiles > 1 with a ragged tail
    *[("Cout%d" % co, G(1, 20, 36, 64, co, 3, 1, 1)) for co in (16, 24, 160, 320)],
    # direct fallbacks: Cin / Cout < 16, channel strides not multiples of 8
    ("Cin8", G(2, 11, 13, 8, 32, 3, 1, 1)),
    ("Cout8", G(2, 11, 13, 32, 8, 3, 1, 1)),
    ("xcs12", G(2, 11, 13, 12, 24, 3, 1, 1, x_cstride=12, dx_cstride=12)),
    ("dcs20", G(2, 11, 13, 16, 20, 1, 1, 0, dy_cstride=20)),
    ("s2_xcs20", G(2, 11, 13, 20, 32, 3, 2, 1, x_cstride=20, dx_cstride=20)),
    # tile width 8 or 16 with a ragged last tile
    *[("Wo%d" % wo, G(2, 9, wo, 32, 48, 3, 1, 1)) for wo in (7, 15, 16, 17)],
    # more wgrad chunks than tiles (empty chunks, n_iters <= 0) with per < stages; one tile, one chunk
    ("empty_chunks", G(1, 80, 64, 64, 64, 3, 1, 1)),
    ("one_tile", G(1, 16, 8, 64, 64, 1, 1, 0)),
    # stride 2: odd / even maps, parity planes of unequal size, planes without taps (1x1), FactorizedReduce's offset
    *[("s2k3_%dx%d" % hw, G(2, hw[0], hw[1], 32, 64, 3, 2, 1)) for hw in ((17, 33), (16, 32), (17, 32), (16, 33))],
    *[("s2k1_%dx%d_off%d" % (hw + (o,)), G(2, hw[0], hw[1], 32, 48, 1, 2, 0, off=(o, o))) for hw in ((17, 33), (16, 32), (15, 18))
      for o in (0, 1)],
    ("s2k3_tiny", G(3, 3, 5, 16, 16, 3, 2, 1)),
    # a 1-row input: the wgrad's parity plane of the taps above it is empty (direct kernel), the dgrad's second row plane too
    ("s2k3_h1", G(2, 1, 9, 32, 32, 3, 2, 1)),
    # each dgrad N tile of conv_plan (16 .. 128): dx channels against the grid's m_tiles
    *[("nt_ci%d" % ci, G(3, 64, 128, ci, 32, 3, 1, 1)) for ci in (16, 32, 48, 64, 96, 128)],
    ("nt_small_grid", G(1, 16, 16, 128, 32, 3, 1, 1)),
    ("nt_s2_planes", G(2, 32, 64, 96, 64, 3, 2, 1)),
    # dilation 2: conv_tc (dgrad_as_fwd_desc) for the dgrad, the direct kernel for the wgrad
    ("dil2", G(2, 20, 24, 32, 32, 3, 1, 2, dil=2)),
    # accumulate = 1 into a slimmable slice of the master weight
    ("acc_slice", G(2, 20, 36, 40, 24, 3, 1, 1, w_stride_o=64 * 9, accumulate=1)),
    ("acc_slice_s2", G(2, 17, 35, 48, 40, 1, 2, 0, off=(1, 1), w_stride_o=64, accumulate=1)),
]
EDGE_IDS = [e[0] for e in EDGE]


def test_edge_grid_covers_every_dgrad_n_tile():
    nts = set()
    for _, g in EDGE:
        for _, _, _, exp in dgrad_paths(g, g.dcs + 8, g.dxcs + 8):
            nts |= {int(k.split("<")[1][:-1]) for k in exp if k.startswith("conv_tc")}
    assert nts == {16, 32, 48, 64, 96, 128}, nts


@pytest.mark.parametrize("op", ["wgrad", "dgrad"])
@pytest.mark.parametrize("case", EDGE, ids=EDGE_IDS)
def test_edge_exact(case, op):
    _run_exact([case[1]], op, 77)


# ---- random family ------------------------------------------------------------------------------------------------------------
def _random_wgrad(g, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x, dy = _normal((g.N, g.Cin, g.H, g.W), gen), _normal((g.N, g.Cout, g.Ho, g.Wo), gen)
    ref = _ref_wgrad(g, x, dy) / g.gscale
    mag = _ref_wgrad(g, x.abs(), dy.abs()) / g.gscale
    n = g.N * g.Ho * g.Wo
    worst = {}
    for path, flags, opts, _ in wgrad_paths(g, g.xcs + 8, g.dcs + 8):
        with Options(opts):
            rc, m, before = run_wgrad(g, x, dy, None, flags)
        assert rc == 0, L().fsb_last_error_string()
        got = m[:g.Cout, :g.Cin].to(F64)
        assert bool(torch.isfinite(got).all())
        ratio = float(((got - ref).abs() / ((n + 6) * U * mag + 1e-300)).max())
        worst[path] = max(worst.get(path, 0.0), ratio)
        outside = _bits32(m).clone()
        outside[:g.Cout, :g.Cin] = 0
        ob = _bits32(before).clone()
        ob[:g.Cout, :g.Cin] = 0
        assert torch.equal(outside, ob)
    return worst


def _random_dgrad(g, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dy, w = _normal((g.N, g.Cout, g.Ho, g.Wo), gen), _normal((g.Cout, g.Cin, g.k, g.k), gen) * 0.25
    ref = _ref_dgrad(g, dy, w)
    mag = _ref_dgrad(g, dy.abs(), w.abs())
    bound = 2.0 ** -11 * ref.abs() + (g.Cout * g.k * g.k + 2) * U * mag + 2.0 ** -24
    worst = {}
    for path, flags, opts, _ in dgrad_paths(g, g.dcs + 8, g.dxcs + 8):
        with Options(opts):
            rc, xs, before = run_dgrad(g, dy, w, flags)
        assert rc == 0, L().fsb_last_error_string()
        got = xs.nchw()
        assert bool(torch.isfinite(got).all()), "%r %s: dx not written" % (g, path)
        worst[path] = max(worst.get(path, 0.0), float(((got - ref).abs() / bound).max()))
        own = torch.zeros_like(xs.bits(), dtype=torch.bool)
        own[:-(g.dxcs + 8)].view(g.N, g.H, g.W, g.dxcs + 8)[..., 8:8 + g.Cin] = True
        assert torch.equal(xs.bits()[~own], before[~own]), "%r %s: dx sentinels overwritten" % (g, path)
    return worst


@pytest.mark.parametrize("gscale", [1024.0, 3.0])
def test_wgrad_random_small_n(gscale):
    worst = collections.Counter()
    for i, (_, g) in enumerate(EDGE):
        g = G(1, g.H, g.W, g.Cin, g.Cout, g.k, g.stride, g.pad, g.dil, g.off, g.xcs, g.dcs, g.dxcs, g.cin_m * g.k * g.k, 0, gscale)
        if g.Ho * g.Wo > 1024:
            continue
        for p, r in _random_wgrad(g, 300 + i).items():
            worst[p] = max(worst[p], r)
    _report("wgrad random gscale %g" % gscale, worst)


def test_dgrad_random_census_and_edges():
    geoms = [G.from_census(g) for g in CC.geometries() if g["op"] == "dgrad" and g["run"] == "distill"] + [g for _, g in EDGE]
    worst = collections.Counter()
    for i, g in enumerate(geoms):
        for p, r in _random_dgrad(g, 900 + i).items():
            worst[p] = max(worst[p], r)
    _report("dgrad random", worst)


# ---- determinism -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direct", [False, True])
def test_deterministic_wgrad_is_bit_identical(direct):
    from fasterseg_b200 import _lib
    g = G(3, 64, 128, 64, 64, 3, 1, 1)        # splits into many pixel chunks in the default mode
    gen = torch.Generator(device="cuda").manual_seed(11)
    x, dy = _normal((g.N, g.Cin, g.H, g.W), gen), _normal((g.N, g.Cout, g.Ho, g.Wo), gen)
    flags = _lib.FSB_CONV_FORCE_DIRECT if direct else 0
    with Options({"FSB_DETERMINISTIC": 1}):
        a = run_wgrad(g, x, dy, None, flags)
        b = run_wgrad(g, x, dy, None, flags)
    assert a[0] == 0 and b[0] == 0
    assert torch.equal(_bits32(a[1]), _bits32(b[1]))


# ---- misaligned slices: the tensor-core kernels read through TMA; the call must fall back, not fail ------------------------------
@pytest.mark.parametrize("k,stride,off", [(3, 1, (0, 0)), (3, 2, (0, 0)), (1, 2, (1, 1))])
def test_misaligned_slices_fall_back_to_the_direct_kernels(k, stride, off):
    g = G(2, 17, 20, 32, 48, k, stride, (k - 1) // 2, off=off, accumulate=0)
    gen = torch.Generator(device="cuda").manual_seed(21)
    x, dy = _ints((g.N, g.Cin, g.H, g.W), gen), _ints((g.N, g.Cout, g.Ho, g.Wo), gen)
    w = _ints((g.Cout, g.Cin, g.k, g.k), gen)
    (rc, m, before), kn = profiled(lambda: run_wgrad(g, x, dy, None, 0, xoff=4, dyoff=4))
    assert rc == 0, L().fsb_last_error_string()
    assert torch.equal(_bits32(m), _bits32(_dw_expected(before, g, torch.round(_ref_wgrad(g, x, dy)) / g.gscale)))
    _assert_kernels(kn.counts, {"zero_wgrad_kernel": 1, "conv_wgrad_kernel": 1})
    (rc, xs, before), kn = profiled(lambda: run_dgrad(g, dy, w, 0, dyoff=4))
    assert rc == 0, L().fsb_last_error_string()
    assert torch.equal(xs.nchw(), torch.round(_ref_dgrad(g, dy, w)))
    _assert_kernels(kn.counts, {"conv_dgrad_direct_kernel": 1})
    # without the fp32 weight there is no fallback: rejected before anything is written
    rc, xs, before = run_dgrad(g, dy, w, 0, dyoff=4, with_w=False)
    torch.cuda.synchronize()
    assert rc == INVALID
    assert torch.equal(xs.bits(), before)
