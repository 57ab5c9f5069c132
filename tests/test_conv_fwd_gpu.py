"""The forward conv (fsb_conv_fwd: conv_tc in csrc/conv_tc.cu, conv_direct_kernel in csrc/conv_direct.cu), the fused training
unit's conv (fsb_conv_bn_act_train_fwd) and the RGB stems through the C ABI, at every launch the networks make
(tests/golden/conv_fwd_census.json, at the drivers' batch) and on a synthetic grid of the kernels' edges, on every path that
can take each geometry: the default plan, per-tap (FSB_CONV_TC2=0), window (FSB_CONV_TC2=1) and direct (FSB_CONV_FORCE_DIRECT).
Which kernel ran is read from torch.profiler and checked against fwd_plan, the Python mirror of conv_plan; the mirror is also
checked against the library's own fsb_conv_kernel_id and fsb_conv_stats_rows.

Exact family (the main one): x and w are sparse integers in {-1, 0, 1}, scale is in {0.5, 1, 2, -1} and shift an integer in
[-3, 3].  Every partial sum of the conv is then an integer far below 2^24, exact in fp32 in any order, and so are the affine and
ReLU: the fp16 output (|y| <= 2048 asserted) and the fp32 output must equal the float64 reference bit for bit.  With
FSB_CONV_STATS every partial row must equal the float64 sum and sum of squares of its 128-pixel tile (conv_tc: one row per tile
in blockIdx.x order (img * tiles_h + tile_h) * tiles_w + tile_w; the sums of squares of a row stay below 2^24, asserted), and
the direct kernel's rows must add up (fsb_rowsum) to the float64 totals exactly.  Dropping one tap of one k-step, or reading one
window row a pixel off, changes some output by at least 1.

Random family: normal fp16-rounded operands, which catch a precision downgrade that small integers cannot (an fp16 accumulator,
a truncated operand).  Elementwise float64 bound, u = 2^-24, K = Cin k^2: the operands are exact fp16 values, so each product is
exact in fp32 and the K-term fp32 sum is within (K + 2) u sum|x||w| of the exact one in any order (the usual (n - 1) u bound
plus slack); the affine y = acc * scale + shift in fp32 adds |scale| times that, and its own two roundings add at most
2u (|scale acc| + |shift|); ReLU is 1-Lipschitz; the fp16 store adds 2^-11 |ref|.  Hence
    |y - ref| <= 2^-11 |ref| + |scale| (K + 2) u sum|x||w| + 2u (|scale acc| + |shift|),
and the worst err / bound per path is reported (<= 1).

Buffer discipline: x is a channel slice of a wider buffer whose other channels hold a large sentinel (with FSB_CONV_X_DOWN2 the
odd rows and columns of the 2H x 2W map hold it too); y is a slice at the recorded channel offset + 8 of a buffer whose own
channels start as NaN, with sentinels around it and a spare pixel after its end (with FSB_CONV_Y_UP2 all four pixels of every
2x2 block are owned); the statistics buffer starts as NaN in this conv's columns and as a sentinel in the other columns of
stats_C; the master weight is the [:Cout, :Cin] corner of a wider fp32 tensor with a sentinel outside it; the packed buffer is
pre-filled with NaN and packed in place, so its kpad / npad zero padding must be written by the packer.  Every owned element
must be written and every other bit must survive.
"""
import collections
import ctypes as C

import pytest
import torch
import torch.nn.functional as TF

from tests import conv_fwd_census as FC
from tests.conv_harness import (AFFINE, F64, FORCE_DIRECT, INVALID, N_TILES, OUT_F32, RELU, SENT16, SENT32, STATS, U, X_DOWN2, Y_UP2,
                                L, Options, Slice, _assert_kernels, _bits32, _cpad, _ints, _normal, _out_size, _report, _s, _sms, fwd_plan,
                                profiled)

pytestmark = pytest.mark.gpu

UNSUPPORTED = -3
DIRECT_MACS = 2 ** 33      # the forced direct path only where the CUDA-core kernel takes milliseconds, not seconds


class FG:
    """one forward conv geometry (the census fields; H, W are the descriptor's, cstrides 0 = dense)"""

    def __init__(self, N, H, W, Cin, Cout, k, stride, pad, dil=1, off=(0, 0), x_cstride=0, y_cstride=0, x_coff=0, y_coff=0, flags=0,
                 scale=1, shift=1, stats_C=0, stats_off=0, w_stride_o=0, name=""):
        self.N, self.H, self.W, self.Cin, self.Cout, self.k, self.stride, self.pad, self.dil = N, H, W, Cin, Cout, k, stride, pad, dil
        self.off, self.flags = tuple(off), flags
        self.f32 = bool(flags & OUT_F32)
        self.xcs = (x_cstride or _cpad(Cin)) + 8       # 8 sentinel channels ahead of the view: same 16-byte alignment class
        self.ycs = (y_cstride or _cpad(Cout)) + 8
        self.xoff, self.yoff = x_coff + 8, y_coff + 8
        self.scale, self.shift = bool(scale), bool(shift)
        self.SC = (stats_C or Cout) if flags & STATS else 0
        self.stats_off = stats_off
        self.cin_m = (w_stride_o or Cin * k * k) // (k * k)     # master weight's input channels (> Cin: a slimmable slice)
        self.name = name
        self.Ho, self.Wo = _out_size(H, W, k, stride, pad, dil, self.off)
        self.up = 2 if flags & Y_UP2 else 1
        self.down = 2 if flags & X_DOWN2 else 1

    @classmethod
    def from_census(cls, g):
        flags = g["flags"] if g["op"] == "conv" else STATS | OUT_F32
        return cls(g["N"], g["H"], g["W"], g["Cin"], g["Cout"], g["k"], g["stride"], g["pad"], g["dil"], (g["off_h"], g["off_w"]),
                   g["x_cstride"], g["y_cstride"], g["x_coff"], g["y_coff"], flags, g["scale"], g["shift"], g["stats_C"], g["stats_off"],
                   g["w_stride_o"], "%s/%s" % (g["run"], g["op"]))

    def plan(self, flags=0, tc2=-1):
        return fwd_plan(self.N, self.H, self.W, self.Cin, self.Cout, self.k, self.stride, self.pad, self.dil, self.off, self.xcs,
                        self.flags | flags, tc2=tc2)

    def desc(self, flags=0):
        from fasterseg_b200 import _lib
        d = _lib.ConvDesc(self.N, self.H, self.W, self.Cin, self.Cout, self.k, self.stride, self.pad, self.dil, self.off[0], self.off[1],
                          self.Ho, self.Wo, self.xcs, self.ycs, self.flags | flags)
        if self.SC:
            d.stats_C, d.stats_off = self.SC, self.stats_off
        return d

    def macs(self):
        return self.N * self.Ho * self.Wo * self.Cout * self.Cin * self.k * self.k

    def __repr__(self):
        return ("%s N%d %dx%d ci%d co%d k%d s%d p%d d%d off%s cs(%d,%d) coff(%d,%d) flags%d aff(%d,%d) stats(%d,%d) cin_m%d" %
                (self.name, self.N, self.H, self.W, self.Cin, self.Cout, self.k, self.stride, self.pad, self.dil, self.off, self.xcs,
                 self.ycs, self.xoff, self.yoff, self.flags, self.scale, self.shift, self.SC, self.stats_off, self.cin_m))


# ---- which paths take a geometry, and the kernels they launch ----------------------------------------------------------------------
def _expected(g, p):
    if p["direct"]:
        return {"conv_direct_kernel": 1, **({"bn_stats_generic_kernel<float>": 1} if g.flags & STATS else {})}
    return {"conv_tc%s%s<%d>" % ("_up2" if g.flags & Y_UP2 else "", "_win" if p["win"] else "", p["n_tile"]): 1}


def fwd_paths(g):
    """-> [(path, extra flags, {option: value}, plan, expected kernel counts)]: the default plan, and per-tap, window and direct
    wherever they can take the geometry and launch something else than the default"""
    default = g.plan()
    out = [("default", 0, {"FSB_CONV_TC2": -1}, default, _expected(g, default))]
    if default["direct"]:
        return out
    for path, tc2 in (("tap", 0), ("window", 1)):
        p = g.plan(tc2=tc2)
        if p["win"] != default["win"]:
            out.append((path, 0, {"FSB_CONV_TC2": tc2}, p, _expected(g, p)))
    if not g.flags & (X_DOWN2 | Y_UP2) and g.macs() <= DIRECT_MACS:
        p = g.plan(FORCE_DIRECT)
        out.append(("direct", FORCE_DIRECT, {"FSB_CONV_TC2": -1}, p, _expected(g, p)))
    return out


def stat_rows(g, p):
    return p["m_tiles"] if not p["direct"] else L().fsb_stat_rows(g.N * g.Ho * g.Wo)


# ---- operands and one launch ------------------------------------------------------------------------------------------------------
def operands(g, gen, exact):
    xin = (_ints if exact else _normal)((g.N, g.Cin, g.H, g.W), gen)
    w = (_ints if exact else _normal)((g.Cout, g.Cin, g.k, g.k), gen)
    if exact:
        scale = torch.tensor([0.5, 1.0, 2.0, -1.0], dtype=F64, device="cuda")[torch.randint(0, 4, (g.Cout,), generator=gen, device="cuda")]
        shift = torch.randint(-3, 4, (g.Cout,), generator=gen, device="cuda").to(F64)
    else:
        w = w * 0.25
        scale = torch.randn(g.Cout, generator=gen, device="cuda", dtype=torch.float32).to(F64)
        shift = torch.randn(g.Cout, generator=gen, device="cuda", dtype=torch.float32).to(F64)
    if not g.flags & AFFINE:
        scale, shift = None, None
    else:
        scale = scale if g.scale else None
        shift = shift if g.shift else None
    return xin, w, scale, shift


def ref_conv(g, xin, w):
    return TF.conv2d(xin[:, :, g.off[0]:, g.off[1]:], w, None, g.stride, g.pad, g.dil)


def ref_epilogue(g, acc, scale, shift):
    y = acc
    if scale is not None:
        y = y * scale.view(1, -1, 1, 1)
    if shift is not None:
        y = y + shift.view(1, -1, 1, 1)
    if g.flags & RELU:
        y = y.clamp_min(0)
    if g.up == 2:
        y = y.repeat_interleave(2, 2).repeat_interleave(2, 3)
    return y


def packed_weight(g, w):
    """the NaN-prefilled packed buffer, packed in place from the [:Cout, :Cin] corner of a sentinel-filled master weight"""
    from fasterseg_b200 import functional as F_
    m = torch.full((g.Cout + 8, g.cin_m, g.k, g.k), SENT32, dtype=torch.float32, device="cuda")
    m[:g.Cout, :g.Cin] = w.float()
    nbytes = L().fsb_conv_packed_bytes(C.byref(g.desc()))
    packed = torch.full((nbytes // 2,), float("nan"), dtype=torch.float16, device="cuda")
    return F_.pack_conv_weight(m, g.Cin, g.Cout, g.k, out=packed)


def x_slice(g, xin, xoff=None):
    xoff = g.xoff if xoff is None else xoff
    xs = Slice(g.N, g.H * g.down, g.W * g.down, g.Cin, g.xcs, xoff, torch.float16, SENT16, SENT16)
    xs.view[:, ::g.down, ::g.down].copy_(xin.permute(0, 2, 3, 1).half())
    return xs


def stats_buffer(g, rows):
    st = torch.full((rows, 2 * g.SC), SENT32, dtype=torch.float32, device="cuda")
    st[:, g.stats_off:g.stats_off + g.Cout] = float("nan")
    st[:, g.SC + g.stats_off:g.SC + g.stats_off + g.Cout] = float("nan")
    return st


def run_fwd(g, xs, wp, scale, shift, flags, rows):
    """-> (rc, y Slice, its bits before the call, statistics buffer or None, its bits before the call)"""
    ys = Slice(g.N, g.Ho * g.up, g.Wo * g.up, g.Cout, g.ycs, g.yoff, torch.float32 if g.f32 else torch.float16, float("nan"),
               SENT32 if g.f32 else SENT16)
    st = stats_buffer(g, rows) if g.SC else None
    yb, sb = ys.bits().clone(), None if st is None else _bits32(st).clone()
    sc = None if scale is None else scale.float().contiguous()
    sh = None if shift is None else shift.float().contiguous()
    d = g.desc(flags)
    rc = L().fsb_conv_fwd(C.byref(d), xs.ptr(), wp.data_ptr(), None if sc is None else sc.data_ptr(), None if sh is None else sh.data_ptr(),
                          ys.ptr(), None if st is None else st.data_ptr(), _s())
    torch.cuda.synchronize()
    return rc, ys, yb, st, sb


def tile_rows(acc, p):
    """float64 per-tile (sum, sum of squares) of acc [N, C, Ho, Wo] in conv_tc's blockIdx.x order -> [m_tiles, C] each"""
    N, Cc, Ho, Wo = acc.shape
    th, tw = p["th"], p["tw"]
    a = torch.zeros((N, Cc, p["tiles_h"] * th, p["tiles_w"] * tw), dtype=F64, device=acc.device)
    a[:, :, :Ho, :Wo] = acc

    def rows(t):
        return t.view(N, Cc, p["tiles_h"], th, p["tiles_w"], tw).sum((3, 5)).permute(0, 2, 3, 1).reshape(-1, Cc)
    return rows(a), rows(a * a)


def check_y(g, ys, yb, want_nchw):
    want = Slice(g.N, g.Ho * g.up, g.Wo * g.up, g.Cout, g.ycs, g.yoff, ys.flat.dtype, None, 0.0)
    want.bits().copy_(yb)
    want.put(want_nchw)
    if torch.equal(ys.bits(), want.bits()):
        return None
    bad = ys.bits() != want.bits()
    own = bad[:-g.ycs].view(g.N, g.Ho * g.up, g.Wo * g.up, g.ycs)[..., g.yoff:g.yoff + g.Cout]
    return "%d y bits differ (%d owned, %d NaN left)" % (int(bad.sum()), int(own.sum()), int(torch.isnan(ys.view).sum()))


def check_stats(g, p, st, sb, acc, kernels):
    cols = torch.zeros(2 * g.SC, dtype=torch.bool, device="cuda")
    cols[g.stats_off:g.stats_off + g.Cout] = True
    cols[g.SC + g.stats_off:g.SC + g.stats_off + g.Cout] = True
    if not torch.equal(_bits32(st)[:, ~cols], sb[:, ~cols]):
        return "statistics sentinels overwritten"
    own = torch.cat([st[:, g.stats_off:g.stats_off + g.Cout], st[:, g.SC + g.stats_off:g.SC + g.stats_off + g.Cout]], 1)
    if bool(torch.isnan(own).any()):
        return "%d statistics entries not written" % int(torch.isnan(own).sum())
    if not p["direct"]:
        s, q = tile_rows(acc, p)
        assert float(q.max()) < 2 ** 24, "%r: a tile's sum of squares leaves the fp32-exact range" % g
        if not torch.equal(own, torch.cat([s, q], 1).float()):
            return "%d statistics row entries differ" % int((own != torch.cat([s, q], 1).float()).sum())
        return None
    tot = torch.empty((1, 2 * g.Cout), dtype=torch.float32, device="cuda")
    ownc = own.contiguous()
    assert L().fsb_rowsum(2 * g.Cout, ownc.data_ptr(), ownc.shape[0], 2 * g.Cout, tot.data_ptr(), _s()) == 0
    kernels["rowsum_kernel"] += 1
    want = torch.cat([acc.sum((0, 2, 3)), (acc * acc).sum((0, 2, 3))]).float()
    if not torch.equal(tot[0], want):
        return "statistics totals differ"
    return None


def check_queries(g, flags, opts, p, fails):
    d = g.desc(flags)
    with Options(opts):
        kid, rows = L().fsb_conv_kernel_id(C.byref(d), None, 0), L().fsb_conv_stats_rows(C.byref(d))
    if kid != (0 if p["direct"] else 1) or rows != stat_rows(g, p):
        fails.append("%r %s: library plan (kernel id %d, %d stat rows) differs from the mirror (%s, %d)" %
                     (g, opts, kid, rows, "direct" if p["direct"] else "conv_tc", stat_rows(g, p)))


def exact_case(g, seed, fails, kernels):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    xin, w, scale, shift = operands(g, gen, True)
    acc = torch.round(ref_conv(g, xin, w))     # an integer sum: rounding removes any float64 algorithm noise
    want = ref_epilogue(g, acc, scale, shift)
    if not g.f32:
        assert float(want.abs().max()) <= 2048, "%r: |y| exceeds the fp16-exact range" % g
    xs, wp = x_slice(g, xin), packed_weight(g, w)
    for path, flags, opts, p, exp in fwd_paths(g):
        if g.SC and p["direct"] and float((acc * acc).sum((0, 2, 3)).max()) >= 2 ** 24:
            assert path != "default", "%r: direct statistics leave the fp32-exact range" % g
            continue
        check_queries(g, flags, opts, p, fails)
        with Options(opts):
            rc, ys, yb, st, sb = run_fwd(g, xs, wp, scale, shift, flags, stat_rows(g, p))
        kernels.update(exp)
        if rc != 0:
            fails.append("%r %s: rc %d %s" % (g, path, rc, L().fsb_last_error_string()))
            continue
        for err in (check_y(g, ys, yb, want), check_stats(g, p, st, sb, acc, kernels) if g.SC else None):
            if err:
                fails.append("%r %s: %s" % (g, path, err))
    if bool(torch.isnan(wp).any()):
        fails.append("%r: packed weight padding not written" % g)
    if g.flags & (X_DOWN2 | Y_UP2):
        # the direct kernel has no nearest folds: rejected before anything is written
        rc, ys, yb, st, sb = run_fwd(g, xs, wp, scale, shift, FORCE_DIRECT, 1)
        if rc != UNSUPPORTED or not torch.equal(ys.bits(), yb):
            fails.append("%r forced direct: rc %d, %d y bits written" % (g, rc, int((ys.bits() != yb).sum())))


def _run_exact(geoms, seed0):
    def run():
        fails, expected = [], collections.Counter()
        for i, g in enumerate(geoms):
            exact_case(g, seed0 + i, fails, expected)
        return fails, expected
    (fails, expected), k = profiled(run)
    print("%d geometries, kernels %s, %d stale records" % (len(geoms), dict(sorted(k.counts.items())), k.stale))
    assert not fails, "%d failures:\n%s" % (len(fails), "\n".join(fails[:12]))
    _assert_kernels(k.counts, expected)
    return k.counts


# ---- the census ----------------------------------------------------------------------------------------------------------------
def _census(run=None, ops=("conv", "unit")):
    return [FG.from_census(g) for g in FC.geometries() if g["op"] in ops and (run is None or g["run"] == run)]


def test_census_has_every_run():
    per_run = collections.Counter(g["run"] for g in FC.geometries())
    print("census geometries per run: %s, %d in all" % (dict(per_run), sum(per_run.values())))
    assert set(per_run) == set(FC.RUNS) and sum(per_run.values()) > 100


@pytest.mark.parametrize("run", list(FC.RUNS))
def test_census_exact(run):
    geoms = _census(run)
    assert geoms
    _run_exact(geoms, 1000 * (1 + list(FC.RUNS).index(run)))


# ---- synthetic edge grid: (purpose, geometry) ------------------------------------------------------------------------------------
def _grid_cases():
    """grids of about 1, 2, 3 and 5 CTAs per SM on this device, at n tiles of 64 (3 CTAs per SM) and 128 (2 per SM): every res"""
    sms = _sms()
    out = []
    for per_sm in (1, 2, 3, 5):
        for co in (64, 128):
            out.append(("res%d_co%d" % (per_sm, co), FG(1, 8 * per_sm, 16 * sms, 64, co, 3, 1, 1)))
    return out


EDGE = [
    # every forward N tile: Cout against the grid's m_tiles
    *[("nt_co%d" % co, FG(2, 64, 128, 64, co, 3, 1, 1)) for co in (16, 32, 48, 64, 96, 128)],
    ("nt16_small_grid", FG(1, 16, 16, 64, 16, 3, 1, 1)),
    # BK 32 and 64, ragged last chunk
    *[("Cin%d" % ci, FG(2, 20, 36, ci, 64, 3, 1, 1)) for ci in (16, 24, 48, 80, 96, 200, 384)],
    *[("Cin%d_k1" % ci, FG(2, 20, 36, ci, 64, 1, 1, 0)) for ci in (24, 200)],
    # tail_w slabs, the scalar epilogue (Cout % 8), several N tiles
    *[("Cout%d" % co, FG(2, 20, 36, 64, co, 3, 1, 1, flags=AFFINE | RELU)) for co in (8, 12, 19, 24, 48, 96, 160, 320)],
    # 8 x 16 and 16 x 8 tiles with ragged last tiles; maps of one row or column
    *[("Wo%d" % wo, FG(2, 9, wo, 32, 48, 3, 1, 1)) for wo in (7, 8, 15, 16, 17)],
    *[("s2_Wo%d" % wo, FG(2, 9, 2 * wo, 32, 48, 3, 2, 1)) for wo in (7, 8, 15, 16, 17)],
    ("h1", FG(2, 1, 37, 32, 32, 3, 1, 1)),
    ("w1", FG(2, 37, 1, 32, 32, 3, 1, 1)),
    ("h1_k1_s2", FG(2, 1, 37, 32, 32, 1, 2, 0)),
    # stride 2 on odd and even maps, FactorizedReduce's offset, dilation 2
    *[("s2k3_%dx%d" % hw, FG(2, hw[0], hw[1], 32, 64, 3, 2, 1)) for hw in ((17, 33), (16, 32), (17, 32), (16, 33))],
    *[("s2k1_%dx%d_off%d" % (hw + (o,)), FG(2, hw[0], hw[1], 32, 48, 1, 2, 0, off=(o, o))) for hw in ((17, 33), (16, 32))
      for o in (0, 1)],
    ("dil2", FG(2, 20, 24, 32, 32, 3, 1, 2, dil=2)),
    # a 3x3 stride-2 conv whose tap row 0 (column 0) reads an empty parity plane: the direct kernel
    ("s2k3_h1", FG(2, 1, 9, 32, 32, 3, 2, 1)),
    ("s2k3_w1", FG(2, 9, 1, 32, 32, 3, 2, 1)),
    # fp32 output with y_cstride % 4 != 0 (no vector stores); an fp16 y slice off 16 bytes (no TMA store)
    ("f32_ycs_odd", FG(2, 20, 36, 32, 40, 3, 1, 1, y_cstride=42, flags=OUT_F32 | AFFINE)),
    ("y_unaligned", FG(2, 20, 36, 32, 48, 3, 1, 1, y_cstride=56, y_coff=4, flags=AFFINE | RELU)),
    # statistics: conv_tc and direct rows, a half of a shared row (stats_off > 0)
    ("stats", FG(2, 20, 36, 32, 48, 3, 1, 1, flags=STATS | OUT_F32)),
    ("stats_off", FG(2, 17, 35, 32, 24, 1, 2, 0, off=(1, 1), flags=STATS | OUT_F32, stats_C=48, stats_off=24, y_cstride=48, y_coff=24)),
    ("stats_cin8", FG(2, 20, 36, 8, 32, 3, 1, 1, flags=STATS | OUT_F32)),
    # nearest x2 folds: ragged tiles, Cout 24 (tail slabs in every lattice), both together
    ("up2_ragged", FG(2, 9, 13, 32, 24, 3, 1, 1, flags=Y_UP2 | AFFINE | RELU)),
    ("up2_co64", FG(1, 16, 24, 64, 64, 3, 1, 1, flags=Y_UP2 | AFFINE)),
    ("down2", FG(2, 10, 18, 32, 48, 3, 1, 1, flags=X_DOWN2 | AFFINE | RELU)),
    ("down2_up2", FG(2, 9, 13, 32, 24, 3, 1, 1, flags=X_DOWN2 | Y_UP2 | AFFINE | RELU)),
    # a sliced master weight, channel strides off the dense ones
    ("slice", FG(2, 20, 36, 40, 24, 3, 1, 1, x_cstride=64, w_stride_o=64 * 9)),
    ("xcs12_direct", FG(2, 11, 13, 12, 24, 3, 1, 1, x_cstride=12)),
]


def _edges():
    return EDGE + _grid_cases()


def test_edge_grid_covers_every_fwd_n_tile_and_residency():
    nts, res = set(), set()
    for _, g in _edges():
        for _, _, _, p, _ in fwd_paths(g):
            if not p["direct"]:
                nts.add(p["n_tile"])
                res.add(min(-(-p["ctas"] // _sms()), 3 if p["n_tile"] <= 64 else 2))
    assert nts == set(N_TILES), nts
    assert res == {1, 2, 3}, res


@pytest.mark.parametrize("case", EDGE, ids=[e[0] for e in EDGE])
def test_edge_exact(case):
    _run_exact([case[1]], 77)


def test_grid_residency_exact():
    _run_exact([g for _, g in _grid_cases()], 88)


def test_every_instance_ran():
    """the census and the edge grid together launch every N tile in both modes, the up2 instances and the direct kernel"""
    seen = set()
    for g in _census() + [g for _, g in _edges()]:
        for _, _, _, _, exp in fwd_paths(g):
            seen |= set(exp)
    print("kernel instances: %s" % sorted(seen))
    for nt in N_TILES:
        assert "conv_tc<%d>" % nt in seen and "conv_tc_win<%d>" % nt in seen, nt
    assert any(k.startswith("conv_tc_up2") for k in seen) and "conv_direct_kernel" in seen


# ---- random family ------------------------------------------------------------------------------------------------------------
def random_case(g, seed, worst):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    xin, w, scale, shift = operands(g, gen, False)
    acc = ref_conv(g, xin, w)
    ref = ref_epilogue(g, acc, scale, shift)
    mag = ref_conv(g, xin.abs(), w.abs())
    s = scale.view(1, -1, 1, 1) if scale is not None else torch.ones((), dtype=F64, device="cuda")
    b = shift.abs().view(1, -1, 1, 1) if shift is not None else 0.0
    K = g.Cin * g.k * g.k
    bound = s.abs() * (K + 2) * U * mag + 2 * U * ((s * acc).abs() + b)
    if g.up == 2:
        bound = bound.repeat_interleave(2, 2).repeat_interleave(2, 3)
    if not g.f32:
        bound = bound + 2.0 ** -11 * ref.abs()
    bound = bound + 1e-300
    xs, wp = x_slice(g, xin), packed_weight(g, w)
    for path, flags, opts, p, _ in fwd_paths(g):
        with Options(opts):
            rc, ys, yb, st, sb = run_fwd(g, xs, wp, scale, shift, flags, stat_rows(g, p))
        assert rc == 0, "%r %s: %s" % (g, path, L().fsb_last_error_string())
        got = ys.nchw()
        assert bool(torch.isfinite(got).all()), "%r %s: y not written" % (g, path)
        worst[path] = max(worst.get(path, 0.0), float(((got - ref).abs() / bound).max()))


def test_random_census_and_edges():
    worst = {}
    geoms = _census() + [g for _, g in _edges()]
    for i, g in enumerate(geoms):
        random_case(g, 900 + i, worst)
    _report("conv_fwd random (%d geometries)" % len(geoms), worst)


# ---- the fused training unit ---------------------------------------------------------------------------------------------------
def test_train_unit_exact():
    """fsb_conv_bn_act_train_fwd at the census's unit geometries: raw and the R partial rows of vec equal the references"""
    geoms = _census(ops=("unit",))
    fails = []
    for i, g in enumerate(geoms):
        gen = torch.Generator(device="cuda").manual_seed(3000 + i)
        xin, w, _, _ = operands(g, gen, True)
        acc = torch.round(ref_conv(g, xin, w))
        xs, wp = x_slice(g, xin), packed_weight(g, w)
        p = g.plan()
        R = stat_rows(g, p)
        raw = Slice(g.N, g.Ho, g.Wo, g.Cout, g.ycs, g.yoff, torch.float32, float("nan"), SENT32)
        y = torch.empty((g.N * g.Ho * g.Wo * _cpad(g.Cout),), dtype=torch.float16, device="cuda")
        vec = torch.full(((6 + 2 * R) * g.Cout,), float("nan"), dtype=torch.float32, device="cuda")
        gamma = torch.ones(g.Cout, device="cuda")
        beta = torch.zeros(g.Cout, device="cuda")
        rm, rv = torch.zeros(g.Cout, device="cuda"), torch.ones(g.Cout, device="cuda")
        rb = raw.bits().clone()
        d = g.desc(0)
        d.flags, d.stats_C, d.stats_off = 0, 0, 0
        rc = L().fsb_conv_bn_act_train_fwd(C.byref(d), xs.ptr(), wp.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1e-5, 0.1,
                                           rm.data_ptr(), rv.data_ptr(), None, raw.ptr(), g.ycs, y.data_ptr(), _cpad(g.Cout),
                                           vec.data_ptr(), 1, None, None, _s())
        torch.cuda.synchronize()
        if rc != 0:
            fails.append("%r: rc %d %s" % (g, rc, L().fsb_last_error_string()))
            continue
        err = check_y(g, raw, rb, acc)
        if err:
            fails.append("%r: raw: %s" % (g, err))
        rows = vec[6 * g.Cout:].view(R, 2 * g.Cout)
        if not p["direct"]:
            s, q = tile_rows(acc, p)
            if not torch.equal(rows, torch.cat([s, q], 1).float()):
                fails.append("%r: %d partial row entries differ" % (g, int((rows != torch.cat([s, q], 1).float()).sum())))
        elif not torch.equal(rows.double().sum(0).float(), torch.cat([acc.sum((0, 2, 3)), (acc * acc).sum((0, 2, 3))]).float()):
            fails.append("%r: direct partial rows do not add up to the totals" % g)
    print("train unit: %d geometries" % len(geoms))
    assert not fails, "%d failures:\n%s" % (len(fails), "\n".join(fails[:12]))


# ---- the stems at the frame geometry ---------------------------------------------------------------------------------------------
def _frame_stem():
    """(C0, C1): the frame's stem width and stem.1.conv1's, from the census"""
    gs = [g for g in FC.geometries() if g["run"] == "frame"]
    stem = [g for g in gs if g["op"] == "stem_nchw"][0]
    C0 = stem["Cout"]
    c1 = [g for g in gs if g["op"] == "conv" and (g["H"], g["W"], g["Cin"], g["k"], g["stride"]) ==
          ((stem["H"] + 1) // 2, (stem["W"] + 1) // 2, C0, 3, 2)][0]
    return C0, c1["Cout"], c1["H"], c1["W"]


def _stem_operands(gen, C0, C1):
    sc = torch.tensor([0.5, 1.0, 2.0, -1.0], dtype=torch.float32, device="cuda")
    w0 = _ints((C0, 3, 3, 3), gen).float().contiguous()
    w1 = _ints((C1, C0, 3, 3), gen)
    s0 = sc[torch.randint(0, 4, (C0,), generator=gen, device="cuda")].contiguous()
    b0 = torch.randint(-3, 4, (C0,), generator=gen, device="cuda").float()
    s1 = sc[torch.randint(0, 4, (C1,), generator=gen, device="cuda")].contiguous()
    b1 = torch.randint(-3, 4, (C1,), generator=gen, device="cuda").float()
    return w0, w1, s0, b0, s1, b1


def _affine_relu(acc, s, b):
    return (acc * s.double().view(1, -1, 1, 1) + b.double().view(1, -1, 1, 1)).clamp_min(0)


@pytest.mark.parametrize("kind", ["f32", "f16", "u8"])
def test_stems_exact_at_the_frame_geometry(kind):
    C0, C1, H1, W1 = _frame_stem()
    N, H, W = 1, 2 * H1, 2 * W1
    gen = torch.Generator(device="cuda").manual_seed(41)
    w0, w1, s0, b0, s1, b1 = _stem_operands(gen, C0, C1)
    if kind == "u8":
        lut = torch.randint(-1, 2, (768,), generator=gen, device="cuda").half()
        frame = torch.randint(0, 256, (N, H, W, 3), generator=gen, device="cuda", dtype=torch.uint8)
        x = frame.permute(0, 3, 1, 2)
        xv = torch.stack([lut.view(3, 256)[c][x[:, c].long()] for c in range(3)], 1).to(F64)
    else:
        xv = _ints((N, 3, H, W), gen)
        x = xv.to(torch.float32 if kind == "f32" else torch.float16).contiguous()
    z0 = _affine_relu(torch.round(TF.conv2d(xv, w0.double(), None, 2, 1)), s0, b0)
    ys = Slice(N, H1, W1, C0, C0 + 8, 8, torch.float16, float("nan"), SENT16)
    yb = ys.bits().clone()
    if kind == "u8":
        rc = L().fsb_stem_conv_u8hwc(N, H, W, C0, frame.data_ptr(), lut.data_ptr(), w0.data_ptr(), s0.data_ptr(), b0.data_ptr(),
                                     ys.ptr(), C0 + 8, RELU | AFFINE, _s())
    else:
        rc = L().fsb_stem_conv_nchw(N, H, W, C0, x.data_ptr(), int(kind == "f32"), w0.data_ptr(), s0.data_ptr(), b0.data_ptr(),
                                    ys.ptr(), C0 + 8, RELU | AFFINE, _s())
    torch.cuda.synchronize()
    assert rc == 0, L().fsb_last_error_string()
    g0 = FG(N, H, W, 3, C0, 3, 2, 1)
    assert check_y(g0, ys, yb, z0) is None
    # stem_fused: relu(bn1(conv1(relu(bn0(conv0(x)))))) without the 1/2-resolution map
    z1 = _affine_relu(torch.round(2 * TF.conv2d(z0, w1, None, 2, 1)) / 2, s1, b1)     # z0: multiples of 1/2
    assert float(z1.abs().max()) <= 2048
    g1 = FG(N, H1, W1, C0, C1, 3, 2, 1)
    wp = packed_weight(g1, w1)
    out = Slice(N, g1.Ho, g1.Wo, C1, C1 + 8, 8, torch.float16, float("nan"), SENT16)
    ob = out.bits().clone()
    kinds = {"f32": 0, "f16": 1, "u8": 2}
    rc = L().fsb_stem_fused(N, H, W, kinds[kind], (frame if kind == "u8" else x).data_ptr(), lut.data_ptr() if kind == "u8" else None,
                            C0, w0.data_ptr(), s0.data_ptr(), b0.data_ptr(), C1, wp.data_ptr(), s1.data_ptr(), b1.data_ptr(), out.ptr(),
                            C1 + 8, _s())
    torch.cuda.synchronize()
    assert rc == 0, L().fsb_last_error_string()
    assert check_y(g1, out, ob, z1) is None


# ---- rejected descriptors write nothing ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direct", [False, True])
@pytest.mark.parametrize("flags", [STATS | OUT_F32 | AFFINE, STATS | OUT_F32 | RELU, STATS])
def test_statistics_need_a_raw_fp32_output(flags, direct):
    """FSB_CONV_STATS sums the raw fp32 output on every kernel: with an epilogue or an fp16 output the call is rejected before any
    launch, on conv_tc and on the direct kernel alike"""
    g = FG(2, 20, 36, 32, 48, 3, 1, 1, flags=flags | (FORCE_DIRECT if direct else 0))
    gen = torch.Generator(device="cuda").manual_seed(5)
    xin, w, scale, shift = operands(g, gen, True)
    xs, wp = x_slice(g, xin), packed_weight(g, w)
    p = g.plan()
    assert p["direct"] == direct
    rc, ys, yb, st, sb = run_fwd(g, xs, wp, scale, shift, 0, stat_rows(g, p))
    assert rc == INVALID
    assert torch.equal(ys.bits(), yb) and torch.equal(_bits32(st), sb)


@pytest.mark.parametrize("k,stride,off", [(3, 1, (0, 0)), (3, 2, (0, 0)), (1, 2, (1, 1))])
def test_misaligned_x_on_conv_tc_is_rejected(k, stride, off):
    """a descriptor conv_tc takes, with an x that TMA cannot load (8-byte aligned): FSB_ERR_INVALID before anything is written, no
    fall-back that would change the statistics rows fsb_conv_stats_rows(d) reported"""
    g = FG(2, 17, 20, 32, 48, k, stride, (k - 1) // 2, off=off, flags=STATS | OUT_F32)
    gen = torch.Generator(device="cuda").manual_seed(21)
    xin, w, _, _ = operands(g, gen, True)
    xs, wp = x_slice(g, xin, xoff=4), packed_weight(g, w)
    p = g.plan()
    assert not p["direct"]
    rc, ys, yb, st, sb = run_fwd(g, xs, wp, None, None, 0, stat_rows(g, p))
    assert rc == INVALID
    assert torch.equal(ys.bits(), yb) and torch.equal(_bits32(st), sb)
