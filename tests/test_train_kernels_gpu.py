"""The training kernels (csrc/bn.cu, csrc/train.cu, csrc/train_fused.cu) one by one through the C ABI, against the float64
references of tests/train_kernel_refs.py.

Each stage is tested from its own inputs: the backward references take the kernel's own y, raw, mean, invstd and sums, dx and dw
the kernel's own draw.  ReLU-mask flips and the fp16 rounding of earlier stages then stay out of the comparison and the bounds
are elementwise and derived, with u = 2^-24 (fp32 unit roundoff) and 2^-11 (fp16 relative rounding):
  - reductions accumulated in fp32:   |got - ref| <= C_SUM * u * sum|term|   (fp32 partial sums of at most a few hundred
    terms whose errors have random signs; a dropped or double-counted block of pixels moves a sum of non-zero-mean terms by
    more than 1e3 times this);
  - fp16 results:                     2^-11 * |ref| + the fp32 error of what was rounded + 2^-24 (fp16 subnormal spacing);
  - elementwise kernels:              bit-exact against the float64 result rounded to fp16.
Outputs that need no zeroing are pre-filled with NaN and must come back finite; channels outside a slice must keep their bits.
Every test prints its worst error / bound ratio.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import train_kernel_refs as R

pytestmark = pytest.mark.gpu

F64 = torch.float64
U = 2.0 ** -24
H11 = 2.0 ** -11
C_SUM = 64
INVALID = -1
EPS, MOM = float(np.float32(1e-5)), float(np.float32(0.1))     # the fp32 values the kernels are given


def L():
    from fasterseg_b200 import _lib
    return _lib.lib()


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def _randn(shape, seed, mean=0.0, scale=1.0):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal(shape).astype(np.float32) * scale + mean)


def _buf(N, H, W, Ctot, dtype=torch.float16, fill=float("nan")):
    """NHWC device buffer; outputs start as NaN (every element a kernel owns must be written)"""
    return torch.full((N, H, W, Ctot), fill, dtype=dtype, device="cuda")


def _inbuf(N, H, W, Ctot, dtype=torch.float16):
    """NHWC device buffer for inputs: the channels outside the slice a kernel reads hold a large finite sentinel"""
    return _buf(N, H, W, Ctot, dtype, 1000.0)


def _put(buf, off, x_nchw):
    """write a CPU NCHW tensor into channels [off, off + C) of an NHWC device buffer; -> the slice (N, H, W, C)"""
    sl = buf[..., off:off + x_nchw.shape[1]]
    sl.copy_(x_nchw.permute(0, 2, 3, 1).to(buf.dtype))
    return sl


def _nchw(sl):
    """device NHWC slice -> CPU float64 NCHW"""
    return sl.permute(0, 3, 1, 2).double().cpu()


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32).cpu().clone()


def _outside(buf, off, Cs):
    b = _bits(buf)
    return torch.cat([b[..., :off].reshape(-1), b[..., off + Cs:].reshape(-1)])


def _check(name, got, ref, bound):
    got, ref, bound = got.double().cpu(), ref.double().cpu(), torch.as_tensor(bound, dtype=F64).cpu()
    assert bool(torch.isfinite(got).all()), "%s: %d entries not written (NaN)" % (name, int((~torch.isfinite(got)).sum()))
    ratio = float(((got - ref).abs() / bound).max()) if got.numel() else 0.0
    print("%-40s worst err/bound %.3f" % (name, ratio))
    assert ratio <= 1.0, "%s: worst err/bound %.3f" % (name, ratio)
    return ratio


def _f16_bound(ref, fp32_err=0.0):
    return H11 * ref.abs() + fp32_err + 2.0 ** -24


def _inject_zeros(y):
    """exact zeros and -0.0 in a ReLU output: the mask is y > 0, so both must block the gradient"""
    flat = y.view(-1)
    flat[::5] = 0.0
    flat[1::11] = -0.0


# ---- BatchNorm backward, plain ------------------------------------------------------------------------------------------------
# C, pixels, raw fp32, relu, accumulate (None = NULL dgamma / dbeta), gscale, sliced views
BWD_CASES = [
    (8, 257, True, True, 0, 1.0, False),
    (40, 257, True, True, 0, 1.0, True),
    (48, 255, False, True, 1, 1024.0, False),
    (56, 257, True, False, 0, 3.0, True),
    (192, 256, True, True, -1, 1.0, False),
    (384, 1, False, True, 0, 1.0, True),
    (2048, 300, True, True, 1, 3.0, False),
    (16, 1, True, True, 0, 1.0, False),
    (16, 255, True, True, None, 1.0, False),
    (16, 264 * 256, False, True, 0, 1024.0, True),
    (16, 264 * 256 + 1, True, True, 1, 1.0, False),
    (24, 800_003, True, True, 0, 3.0, True),
]


def _bn_bwd_inputs(C, pixels, raw_f32, relu, gscale, sliced, seed):
    N, H, W = 1, 1, pixels
    off, Ct = (8, C + 24) if sliced else (0, C)
    raw_c = _randn((N, C, H, W), seed, mean=0.5)
    mean = raw_c.double().mean((0, 2, 3)).float()
    invstd = (1.0 / (raw_c.double().var((0, 2, 3), unbiased=False) + 1e-5).sqrt()).float()
    gamma = torch.from_numpy(np.random.RandomState(seed + 1).uniform(0.5, 1.5, C).astype(np.float32))
    y_c = ((raw_c - R._c(mean)) * R._c(invstd) * R._c(gamma)).clamp_min(0)
    dy_c = _randn((N, C, H, W), seed + 2, mean=0.3) * gscale
    rawb = _inbuf(N, H, W, Ct, torch.float32 if raw_f32 else torch.float16)
    dyb, yb = _inbuf(N, H, W, Ct), _inbuf(N, H, W, Ct)
    raw, dy, y = _put(rawb, off, raw_c), _put(dyb, off, dy_c), _put(yb, off, y_c)
    if relu:
        yz = y.clone()
        _inject_zeros(yz)
        y.copy_(yz)
    return dict(off=off, Ct=Ct, raw=raw, dy=dy, y=y, mean=mean.cuda(), invstd=invstd.cuda(), gamma=gamma.cuda(), N=N, H=H, W=W)


@pytest.mark.parametrize("case", BWD_CASES)
def test_bn_bwd_reduce_and_apply(case):
    C, pixels, raw_f32, relu, acc, gscale, sliced = case
    t = _bn_bwd_inputs(C, pixels, raw_f32, relu, gscale, sliced, seed=C + pixels % 1000)
    P = L().fsb_stat_rows(pixels)
    sums = torch.full(((1 + P), 2 * C), float("nan"), device="cuda")
    rc = L().fsb_bn_bwd_reduce(pixels, C, _p(t["dy"]), t["Ct"], _p(t["y"]), t["Ct"], _p(t["raw"]), t["Ct"], int(raw_f32),
                               _p(t["mean"]), _p(t["invstd"]), int(relu), _p(sums), _s())
    assert rc == 0
    drawb = _buf(t["N"], t["H"], t["W"], t["Ct"])
    draw = drawb[..., t["off"]:t["off"] + C]
    pre_g = _randn((C,), 5, mean=1.0).cuda()
    pre_b = _randn((C,), 6, mean=-1.0).cuda()
    dg, db = pre_g.clone(), pre_b.clone()
    rc = L().fsb_bn_bwd_apply(pixels, C, _p(t["dy"]), t["Ct"], _p(t["y"]), t["Ct"], _p(t["raw"]), t["Ct"], int(raw_f32), _p(t["mean"]),
                              _p(t["invstd"]), _p(t["gamma"]), _p(sums), float(pixels), int(relu), _p(draw), t["Ct"],
                              None if acc is None else _p(dg), None if acc is None else _p(db), gscale, 0 if acc is None else acc, _s())
    assert rc == 0
    torch.cuda.synchronize()
    dy, y, raw = _nchw(t["dy"]), _nchw(t["y"]), _nchw(t["raw"])
    mean, invstd, gamma = t["mean"].double().cpu(), t["invstd"].double().cpu(), t["gamma"].double().cpu()
    ref = R.bn_bwd(dy, y, raw, mean, invstd, gamma, relu)
    sz, sq = R.bn_bwd_abs_terms(ref["dz"], ref["xhat"])
    s = sums.double().cpu()
    assert bool(torch.isfinite(s).all()), "a partial row was not written"
    assert bool(((s[0] - s[1:].sum(0)).abs() <= 2 * U * s[1:].abs().sum(0)).all()), "row 0 is not the total of the partial rows"
    _check("bn_bwd sum dz", s[0, :C], ref["sum_dz"], C_SUM * U * sz + 1e-30)
    _check("bn_bwd sum dz*xhat", s[0, C:], ref["sum_dzxhat"], C_SUM * U * sq + 1e-30)
    # draw from the kernel's own sums: fp32 evaluation (~8 roundings of terms of size |dz|, |s|/n, |xhat q|/n) + fp16 store
    kref = R.bn_bwd(dy, y, raw, mean, invstd, gamma, relu, sums=(s[0, :C], s[0, C:]))
    gis = R._c(gamma * invstd)
    terms = gis * (ref["dz"].abs() + R._c(s[0, :C].abs()) / pixels + (ref["xhat"] * R._c(s[0, C:]) / pixels).abs())
    _check("bn_bwd draw", _nchw(draw), kref["draw"], _f16_bound(kref["draw"], 8 * U * terms))
    assert torch.equal(_outside(drawb, t["off"], C), _outside(_buf(t["N"], t["H"], t["W"], t["Ct"]), t["off"], C))
    if acc is None:
        return
    if acc == -1:
        assert torch.equal(_bits(dg), _bits(pre_g)) and torch.equal(_bits(db), _bits(pre_b))
        return
    base_g = pre_g.double().cpu() if acc else 0.0
    base_b = pre_b.double().cpu() if acc else 0.0
    _check("bn_bwd dgamma", dg, base_g + s[0, C:] / gscale, 4 * U * (abs(base_g) + s[0, C:].abs() / gscale) + 1e-30)
    _check("bn_bwd dbeta", db, base_b + s[0, :C] / gscale, 4 * U * (abs(base_b) + s[0, :C].abs() / gscale) + 1e-30)


def test_bn_bwd_rejects_more_than_2048_channels():
    t = _bn_bwd_inputs(2056, 4, True, True, 1.0, False, seed=3)
    sums = torch.empty((1 + L().fsb_stat_rows(4)) * 2 * 2056, device="cuda")
    assert L().fsb_bn_bwd_reduce(4, 2056, _p(t["dy"]), 2056, _p(t["y"]), 2056, _p(t["raw"]), 2056, 1, _p(t["mean"]), _p(t["invstd"]), 1,
                                 _p(sums), _s()) == INVALID


# ---- BatchNorm forward edges ---------------------------------------------------------------------------------------------------
# C, pixels, channel offset in the buffer, buffer channels: vector path (C % 8 == 0, aligned) and generic path
STATS_CASES = [(48, 257, 0, 48), (384, 264 * 256 + 1, 0, 384), (20, 1000, 0, 24), (16, 300, 4, 32), (2056, 33, 0, 2056), (8, 1, 0, 8)]


@pytest.mark.parametrize("case", STATS_CASES)
def test_bn_stats(case):
    C, pixels, off, Ct = case
    xb = _inbuf(1, 1, pixels, Ct)
    x = _put(xb, off, _randn((1, C, 1, pixels), C + off, mean=0.75))
    P = L().fsb_stat_rows(pixels)
    buf = torch.full((1 + P, 2 * C), float("nan"), device="cuda")
    assert L().fsb_bn_stats(pixels, C, _p(x), Ct, _p(buf), _s()) == 0
    torch.cuda.synchronize()
    x64 = _nchw(x)
    s, q = R.bn_sums(x64)
    b = buf.double().cpu()
    assert bool(torch.isfinite(b).all()), "a partial row was not written"
    _check("bn_stats sum", b[0, :C], s, C_SUM * U * x64.abs().sum((0, 2, 3)))
    _check("bn_stats sumsq", b[0, C:], q, C_SUM * U * q)


def test_bn_finalize_rows_sc_count2_and_negative_variance():
    C, SC, P = 24, 40, 5
    rows = torch.full((P, 2 * SC), float("nan"))
    rs = np.random.RandomState(7)
    rows[:, :C] = torch.from_numpy(rs.standard_normal((P, C)).astype(np.float32))
    rows[:, SC:SC + C] = rows[:, :C] ** 2 + torch.from_numpy(rs.uniform(0.1, 1.0, (P, C)).astype(np.float32))
    # channel 0: sum 6, sum of squares one fp32 ulp below 18 = 6^2 / count: in double the variance is -2^-20, which must be
    # clamped to 0 (unclamped, invstd would move by 5 %)
    rows[:, 0] = 0.0
    rows[0, 0] = 6.0
    rows[:, SC] = 0.0
    rows[0, SC] = float(np.nextafter(np.float32(18.0), np.float32(0.0)))
    assert float(rows[0, SC]) < 18.0
    count = 2.0
    gamma = torch.from_numpy(rs.uniform(0.5, 1.5, C).astype(np.float32))
    beta = torch.from_numpy(rs.standard_normal(C).astype(np.float32) * 0.1)
    rm0, rv0 = torch.from_numpy(rs.standard_normal(C).astype(np.float32)), torch.from_numpy(rs.uniform(0.5, 2, C).astype(np.float32))
    rm, rv = rm0.cuda(), rv0.cuda()
    out = torch.full((4, C), float("nan"), device="cuda")
    eps, mom = EPS, MOM
    rows_d, gamma_d, beta_d = rows.cuda(), gamma.cuda(), beta.cuda()
    assert L().fsb_bn_finalize(C, _p(rows_d), P, SC, count, _p(gamma_d), _p(beta_d), eps, mom, _p(rm), _p(rv),
                               _p(out[0]), _p(out[1]), _p(out[2]), _p(out[3]), _s()) == 0
    torch.cuda.synchronize()
    r64 = rows.double()
    assert float(r64[:, SC].sum() / count - (r64[:, 0].sum() / count) ** 2) < 0
    st = R.bn_finalize(r64[:, :C].sum(0), r64[:, SC:SC + C].sum(0), count, gamma, beta, eps, mom, rm0, rv0)
    assert st["var"][0] == 0.0
    o = out.double().cpu()
    _check("finalize mean", o[2], st["mean"], 2 * U * st["mean"].abs() + 1e-30)
    _check("finalize invstd", o[3], st["invstd"], 2 * U * st["invstd"])
    _check("finalize scale", o[0], st["scale"], 4 * U * st["scale"].abs())
    _check("finalize shift", o[1], st["shift"], 6 * U * (beta.abs().double() + (st["mean"] * st["scale"]).abs()) + 1e-30)
    _check("finalize running_mean", rm, st["running_mean"], 4 * U * (rm0.abs().double() + mom * st["mean"].abs()))
    _check("finalize running_var", rv, st["running_var"], 4 * U * (rv0.abs().double() + mom * 2 * st["var"]))


# ---- device-selected BatchNorm sets --------------------------------------------------------------------------------------------
class SelTable:
    """an fsb_bn_sel table of parameter sets of widths `widths`, all tensors on the device, gradient slots pre-filled"""

    def __init__(self, widths, seed):
        from fasterseg_b200 import _lib
        rs = np.random.RandomState(seed)
        f = lambda a: torch.from_numpy(a.astype(np.float32)).cuda()
        self.sets = []
        for c in widths:
            self.sets.append(dict(C=c, gamma=f(rs.uniform(0.5, 1.5, c)), beta=f(rs.standard_normal(c) * 0.1),
                                  running_mean=f(rs.standard_normal(c) * 0.1), running_var=f(rs.uniform(0.5, 1.5, c)),
                                  num_batches_tracked=torch.tensor([int(rs.randint(0, 100))], dtype=torch.int64, device="cuda"),
                                  dgamma=f(rs.standard_normal(c)), dbeta=f(rs.standard_normal(c))))
        arr = (_lib.BnSel * len(widths))(*[_lib.BnSel(s["gamma"].data_ptr(), s["beta"].data_ptr(), s["running_mean"].data_ptr(),
                                                      s["running_var"].data_ptr(), s["num_batches_tracked"].data_ptr(), s["dgamma"].data_ptr(),
                                                      s["dbeta"].data_ptr(), s["C"], 0) for s in self.sets])
        self.table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).cuda()
        self.idx = torch.zeros(1, dtype=torch.int32, device="cuda")

    def select(self, k):
        self.idx.fill_(k)

    def snapshot(self):
        return [{k: _bits(v) if torch.is_tensor(v) and v.dtype == torch.float32 else (v.cpu().clone() if torch.is_tensor(v) else v)
                 for k, v in s.items()} for s in self.sets]

    def assert_only_changed(self, before, k, keys):
        after = self.snapshot()
        for i, (b, a) in enumerate(zip(before, after)):
            for key in b:
                if key == "C":
                    continue
                if i == k and key in keys:
                    continue
                assert torch.equal(a[key], b[key]), "set %d: %s changed" % (i, key)


def _sel_rows(raw_nchw, P):
    """P partial statistic rows of raw (columns in the buffer's channel order), pixels split into P contiguous groups"""
    C = raw_nchw.shape[1]
    flat = raw_nchw.double().permute(0, 2, 3, 1).reshape(-1, C)
    rows = torch.zeros(P, 2 * C, dtype=F64)
    for r, chunk in enumerate(torch.tensor_split(flat, P)):
        rows[r, :C] = chunk.sum(0)
        rows[r, C:] = (chunk * chunk).sum(0)
    return rows.float()


def _run_sel_chain(tab, k, Cmax, hmax, pixels, seed, relu=True, gscale=4.0, local=True):
    """finalize_sel -> affine_act_sel -> bn_bwd_reduce_sel -> bn_bwd_apply_sel on set k; checks every stage against the
    references from the stage's own inputs"""
    s = tab.sets[k]
    Ca = s["C"]
    h = Ca // 2
    perm = R.split_perm(h, hmax) if hmax else torch.arange(Cmax)
    raw_c = _randn((1, Cmax, 1, pixels), seed, mean=0.4)            # raw channel order
    rawd = _put(_inbuf(1, 1, pixels, Cmax, torch.float32), 0, raw_c)
    P = 3
    rows = _sel_rows(raw_c, P)
    tab.select(k)
    before = tab.snapshot()
    eps, mom = EPS, MOM
    out = torch.full((4, Cmax), float("nan"), device="cuda")
    rows_d = rows.cuda()
    assert L().fsb_bn_finalize_sel(Cmax, _p(rows_d), P, Cmax, float(pixels), eps, mom, _p(out[0]), _p(out[1]), _p(out[2]), _p(out[3]),
                                   _p(tab.table), _p(tab.idx), hmax, _s()) == 0
    torch.cuda.synchronize()
    o = out.double().cpu()
    r64 = rows.double().sum(0)
    sc, qc = r64[:Cmax][perm][:Ca], r64[Cmax:][perm][:Ca]              # compact order
    st = R.bn_finalize(sc, qc, float(pixels), s["gamma"].cpu(), s["beta"].cpu(), eps, mom, before[k]["running_mean"].view(torch.float32),
                       before[k]["running_var"].view(torch.float32))
    _check("sel finalize mean", o[2, :Ca], st["mean"], 2 * U * st["mean"].abs() + 1e-30)
    _check("sel finalize invstd", o[3, :Ca], st["invstd"], 2 * U * st["invstd"])
    _check("sel finalize scale", o[0, :Ca], st["scale"], 4 * U * st["scale"].abs())
    _check("sel finalize shift", o[1, :Ca], st["shift"], 6 * U * (s["beta"].cpu().abs().double() + (st["mean"] * st["scale"]).abs()) + 1e-30)
    assert bool((o[:, Ca:] == 0).all()), "inactive tail of scale / shift / mean / invstd is not 0"
    _check("sel running_mean", s["running_mean"], st["running_mean"], 4 * U * (before[k]["running_mean"].view(torch.float32).abs().double()
                                                                              + mom * st["mean"].abs()))
    _check("sel running_var", s["running_var"], st["running_var"], 4 * U * (before[k]["running_var"].view(torch.float32).abs().double()
                                                                           + mom * 2 * st["var"]))
    assert int(s["num_batches_tracked"].item()) == int(before[k]["num_batches_tracked"].item()) + 1
    # affine_act_sel: x in raw order, y in compact order
    yb = _buf(1, 1, pixels, Cmax)
    from fasterseg_b200 import _lib
    flags = (_lib.FSB_CONV_RELU if relu else 0) | _lib.FSB_ACT_IN_F32
    assert L().fsb_affine_act_sel(pixels, Cmax, _p(rawd), Cmax, _p(out[0]), _p(out[1]), _p(yb), Cmax, flags, _p(tab.table), _p(tab.idx),
                                  hmax, _s()) == 0
    torch.cuda.synchronize()
    raw64 = _nchw(rawd)
    rawc64 = raw64[:, perm]
    yref = R.affine_act(rawc64[:, :Ca], o[0, :Ca], o[1, :Ca], relu)
    y = _nchw(yb)
    _check("sel affine y", y[:, :Ca], yref, _f16_bound(yref, 2 * U * (rawc64[:, :Ca] * R._c(o[0, :Ca])).abs() + 2 * U * R._c(o[1, :Ca]).abs()))
    assert bool((y[:, Ca:] == 0).all()), "y is not 0 on the inactive tail"
    # backward
    dyb = _put(_inbuf(1, 1, pixels, Cmax), 0, _randn((1, Cmax, 1, pixels), seed + 1, mean=0.2) * gscale)
    yz = yb.clone()
    _inject_zeros(yz)
    yb.copy_(yz)
    Pb = L().fsb_stat_rows(pixels)
    sums = torch.full((1 + Pb, 2 * Cmax), float("nan"), device="cuda")
    assert L().fsb_bn_bwd_reduce_sel(pixels, Cmax, _p(dyb), Cmax, _p(yb), Cmax, _p(rawd), Cmax, 1, _p(out[2]), _p(out[3]), int(relu), _p(sums),
                                     _p(tab.table), _p(tab.idx), hmax, _s()) == 0
    lsum = (torch.from_numpy(np.random.RandomState(seed + 2).standard_normal(2 * Cmax).astype(np.float32)).cuda() if local else None)
    drawb = _buf(1, 1, pixels, Cmax)
    assert L().fsb_bn_bwd_apply_sel(pixels, Cmax, _p(dyb), Cmax, _p(yb), Cmax, _p(rawd), Cmax, 1, _p(out[2]), _p(out[3]), _p(sums[0]),
                                    _p(lsum), float(pixels), int(relu), _p(drawb), Cmax, gscale, _p(tab.table), _p(tab.idx), hmax, _s()) == 0
    torch.cuda.synchronize()
    dy, y = _nchw(dyb), _nchw(yb)
    ref = R.bn_bwd(dy[:, :Ca], y[:, :Ca], rawc64[:, :Ca], o[2, :Ca], o[3, :Ca], s["gamma"].cpu(), relu)
    sm = sums.double().cpu()
    assert bool(torch.isfinite(sm).all()), "a partial row was not written"
    sz, sq = R.bn_bwd_abs_terms(ref["dz"], ref["xhat"])
    _check("sel bwd sum dz", sm[0, :Ca], ref["sum_dz"], C_SUM * U * sz + 1e-30)
    _check("sel bwd sum dz*xhat", sm[0, Cmax:Cmax + Ca], ref["sum_dzxhat"], C_SUM * U * sq + 1e-30)
    draw = _nchw(drawb)
    kref = R.bn_bwd(dy[:, :Ca], y[:, :Ca], rawc64[:, :Ca], o[2, :Ca], o[3, :Ca], s["gamma"].cpu(), relu, count=pixels,
                    sums=(sm[0, :Ca], sm[0, Cmax:Cmax + Ca]))
    gis = R._c(s["gamma"].cpu().double() * o[3, :Ca])
    terms = gis * (ref["dz"].abs() + R._c(sm[0, :Ca].abs()) / pixels + (ref["xhat"] * R._c(sm[0, Cmax:Cmax + Ca]) / pixels).abs())
    _check("sel bwd draw (raw order)", draw[:, perm[:Ca]], kref["draw"], _f16_bound(kref["draw"], 8 * U * terms))
    assert bool((draw[:, perm[Ca:]] == 0).all()), "draw is not 0 on the inactive (raw) channels"
    # gamma / beta gradients: added into set k's slots, from local_sums when given
    ps = (lsum.double().cpu() if local else sm[0])
    g0 = before[k]["dgamma"].view(torch.float32).double()
    b0 = before[k]["dbeta"].view(torch.float32).double()
    _check("sel dgamma", s["dgamma"], g0 + ps[Cmax:Cmax + Ca] / gscale, 4 * U * (g0.abs() + ps[Cmax:Cmax + Ca].abs() / gscale))
    _check("sel dbeta", s["dbeta"], b0 + ps[:Ca] / gscale, 4 * U * (b0.abs() + ps[:Ca].abs() / gscale))
    tab.assert_only_changed(before, k, ("running_mean", "running_var", "num_batches_tracked", "dgamma", "dbeta"))


@pytest.mark.parametrize("k", range(5))
def test_sel_chain_every_width(k):
    tab = SelTable([8, 16, 24, 40, 48], seed=100)
    _run_sel_chain(tab, k, 48, 0, 300, seed=200 + k, local=(k % 2 == 0))


@pytest.mark.parametrize("hmax", [16, 32, 64])
def test_sel_chain_factorized_reduce_order(hmax):
    hs = [8, hmax - 8, hmax]
    tab = SelTable([2 * h for h in hs], seed=hmax)
    for k in range(len(hs)):
        _run_sel_chain(tab, k, 2 * hmax, hmax, 257, seed=300 + hmax + k)


# ---- fused conv -> BN(train) -> ReLU unit --------------------------------------------------------------------------------------
# N, Cin, Cout, k, stride, H, W, off, conv_tc mode for 3x3 s1 (-1 = chosen per problem), force direct
UNIT_CASES = [
    (2, 32, 48, 3, 1, 9, 13, (0, 0), 0, False),
    (2, 32, 48, 3, 1, 9, 13, (0, 0), 1, False),
    (2, 32, 64, 3, 2, 11, 15, (0, 0), -1, False),
    (2, 48, 32, 1, 1, 10, 12, (0, 0), -1, False),
    (2, 64, 48, 1, 2, 12, 16, (0, 0), -1, False),
    (2, 64, 48, 1, 2, 12, 16, (1, 1), -1, False),
    (2, 8, 16, 3, 1, 9, 13, (0, 0), -1, False),
    (2, 32, 48, 3, 1, 9, 13, (0, 0), -1, True),
]


def _unit_setup(case, seed):
    from fasterseg_b200 import functional as F_
    from fasterseg_b200 import _lib
    N, Cin, Cout, k, stride, H, W, off, mode, direct = case
    pad = 1 if k == 3 else 0
    Ho, Wo = F_.conv_out_size(H, W, k, stride, pad, 1, off[0], off[1])
    xoff, xct = 8, Cin + 16
    xb = _inbuf(N, H, W, xct)
    x = _put(xb, xoff, _randn((N, Cin, H, W), seed, mean=0.3))
    w = (_randn((Cout, Cin, k, k), seed + 1) * (2.0 / (Cin * k * k)) ** 0.5).half().float().cuda()
    d = _lib.ConvDesc(N, H, W, Cin, Cout, k, stride, pad, 1, off[0], off[1], Ho, Wo, xct, Cout,
                      _lib.FSB_CONV_FORCE_DIRECT if direct else 0)
    return dict(N=N, Cin=Cin, Cout=Cout, k=k, stride=stride, pad=pad, H=H, W=W, Ho=Ho, Wo=Wo, off=off, x=x, xct=xct, w=w, d=d,
                wp=F_.pack_conv_weight(w, Cin, Cout, k), wt=F_.pack_conv_weight_dgrad(w, Cin, Cout, k))


def _unit_fwd(u, gamma, beta, rm, rv, nbt, relu=True, sel=None):
    from fasterseg_b200 import _lib
    N, Cout, Ho, Wo = u["N"], u["Cout"], u["Ho"], u["Wo"]
    dd = _lib.ConvDesc.from_buffer_copy(u["d"])
    dd.flags |= _lib.FSB_CONV_STATS | _lib.FSB_CONV_OUT_F32
    R_ = L().fsb_conv_stats_rows(C.byref(dd))
    raw = _buf(N, Ho, Wo, Cout, torch.float32)
    y = _buf(N, Ho, Wo, Cout)
    vec = torch.full(((6 + 2 * R_) * Cout,), float("nan"), device="cuda")
    rc = L().fsb_conv_bn_act_train_fwd(C.byref(u["d"]), _p(u["x"]), _p(u["wp"]), _p(gamma), _p(beta), EPS, MOM, _p(rm), _p(rv), _p(nbt),
                                       _p(raw), Cout, _p(y), Cout, _p(vec), int(relu), None if sel is None else _p(sel.table),
                                       None if sel is None else _p(sel.idx), _s())
    assert rc == 0, L().fsb_last_error_string()
    torch.cuda.synchronize()
    return raw, y, vec


def _check_unit_fwd(u, raw, y, vec, gamma, beta, relu=True, active=None):
    """raw against the conv of the fp16 operands, then every later stage from the kernel's own raw / statistics on the first
    `active` channels (a device-selected set's width; its inactive tail must be exactly 0).  -> (float64 statistics of the
    active channels, bound of their variance error)"""
    Cout, n = u["Cout"], u["N"] * u["Ho"] * u["Wo"]
    Ca = Cout if active is None else active
    x64 = _nchw(u["x"])
    w64 = u["w"].double().cpu()
    rref = R.conv(x64, w64, u["stride"], u["pad"], u["off"])
    rmag = R.conv(x64.abs(), w64.abs(), u["stride"], u["pad"], u["off"])
    K = u["Cin"] * u["k"] * u["k"]
    r64 = _nchw(raw)
    _check("unit raw", r64, rref, (K + 2) * U * rmag + 1e-30)
    v = vec.double().cpu()
    assert bool(torch.isfinite(v[2 * Cout:]).all()), "vec[2C:] not written"
    for j in range(2, 6):
        assert bool((v[j * Cout + Ca:(j + 1) * Cout] == 0).all()), "vec section %d: inactive tail not 0" % j
    assert bool((_nchw(y)[:, Ca:] == 0).all()), "y is not 0 on the inactive tail"
    r64 = r64[:, :Ca]
    s, q = R.bn_sums(r64)
    st = R.bn_finalize(s, q, n, None, None, EPS, MOM)
    e_s = C_SUM * U * r64.abs().sum((0, 2, 3)) / n
    e_var = C_SUM * U * q / n + 2 * st["mean"].abs() * e_s
    mean_k, inv_k = v[4 * Cout:4 * Cout + Ca], v[5 * Cout:5 * Cout + Ca]
    _check("unit mean", mean_k, st["mean"], e_s + U * st["mean"].abs() + 1e-30)
    _check("unit invstd", inv_k, st["invstd"], 0.5 * st["invstd"] ** 3 * e_var + 2 * U * st["invstd"])
    g = torch.ones(Ca, dtype=F64) if gamma is None else gamma.double().cpu()
    b = torch.zeros(Ca, dtype=F64) if beta is None else beta.double().cpu()
    sc_k, sh_k = v[2 * Cout:2 * Cout + Ca], v[3 * Cout:3 * Cout + Ca]
    _check("unit scale", sc_k, g * inv_k, 2 * U * (g * inv_k).abs())
    _check("unit shift", sh_k, b - mean_k * g * inv_k, 4 * U * (b.abs() + (mean_k * g * inv_k).abs()) + 1e-30)
    yref = R.affine_act(r64, sc_k, sh_k, relu)
    _check("unit y", _nchw(y)[:, :Ca], yref, _f16_bound(yref, 2 * U * ((r64 * R._c(sc_k)).abs() + R._c(sh_k).abs())))
    return st, e_var


def _check_unit_running(u, rm, rv, rm0, rv0, vec, st, e_var):
    """running statistics: momentum update with the kernel's own batch mean and the unbiased variance"""
    Cout, n = u["Cout"], u["N"] * u["Ho"] * u["Wo"]
    Ca = st["mean"].numel()
    mean_k = vec[4 * Cout:4 * Cout + Ca].double().cpu()
    rm0, rv0 = rm0.double().cpu(), rv0.double().cpu()
    _check("unit running_mean", rm, (1 - MOM) * rm0 + MOM * mean_k, 4 * U * (rm0.abs() + MOM * mean_k.abs()))
    _check("unit running_var", rv, (1 - MOM) * rv0 + MOM * st["var"] * n / (n - 1),
           4 * U * (rv0.abs() + 2 * MOM * st["var"]) + MOM * e_var * n / (n - 1))


def _unit_bwd(u, raw, y, vec, gamma, gscale, dw0, relu=True, sel=None, seed=0):
    N, Cout, Ho, Wo = u["N"], u["Cout"], u["Ho"], u["Wo"]
    dyb = _inbuf(N, Ho, Wo, Cout + 16)
    dy = _put(dyb, 8, _randn((N, Cout, Ho, Wo), seed, mean=0.2) * gscale)
    Rb = L().fsb_stat_rows(N * Ho * Wo)
    drawb = _buf(N, Ho, Wo, Cout)
    vb = torch.full(((4 + 2 * Rb) * Cout,), float("nan"), device="cuda")
    dxb = _buf(N, u["H"], u["W"], u["Cin"])
    dw = dw0.clone()
    rc = L().fsb_conv_bn_act_train_bwd(C.byref(u["d"]), _p(u["x"]), _p(dy), Cout + 16, _p(y), Cout, _p(raw), Cout, _p(vec), _p(gamma),
                                       int(relu), _p(u["wt"]), _p(u["w"]), u["w"].stride(0), u["w"].stride(1), _p(drawb), Cout, _p(vb),
                                       _p(dxb), u["Cin"], _p(dw), gscale, None if sel is None else _p(sel.table),
                                       None if sel is None else _p(sel.idx), _s())
    assert rc == 0, L().fsb_last_error_string()
    torch.cuda.synchronize()
    return dy, drawb, vb, dxb, dw


def _check_unit_bwd(u, dy, raw, y, vec, gamma, gscale, drawb, vb, dxb, dw, dw0, sel_C=None, relu=True):
    Cout, n = u["Cout"], u["N"] * u["Ho"] * u["Wo"]
    Ca = Cout if sel_C is None else sel_C
    v = vec.double().cpu()
    mean, inv = v[4 * Cout:5 * Cout], v[5 * Cout:6 * Cout]
    g = torch.ones(Cout, dtype=F64) if gamma is None else gamma.double().cpu()
    dy64, y64, r64 = _nchw(dy), _nchw(y), _nchw(raw)
    ref = R.bn_bwd(dy64, y64, r64, mean, inv, g, relu)
    vbd = vb.double().cpu()
    Rb = L().fsb_stat_rows(n)
    assert bool(torch.isfinite(vbd[:(2 + 2 * Rb) * Cout]).all()), "vec_bwd sums / partial rows not written"
    sz, sq = R.bn_bwd_abs_terms(ref["dz"], ref["xhat"])
    _check("unit bwd sum dz", vbd[:Cout], ref["sum_dz"], C_SUM * U * sz + 1e-30)
    _check("unit bwd sum dz*xhat", vbd[Cout:2 * Cout], ref["sum_dzxhat"], C_SUM * U * sq + 1e-30)
    kref = R.bn_bwd(dy64, y64, r64, mean, inv, g, relu, sums=(vbd[:Cout], vbd[Cout:2 * Cout]))
    terms = R._c(g * inv) * (ref["dz"].abs() + R._c(vbd[:Cout].abs()) / n + (ref["xhat"] * R._c(vbd[Cout:2 * Cout]) / n).abs())
    draw = _nchw(drawb)
    _check("unit draw", draw, kref["draw"], _f16_bound(kref["draw"], 8 * U * terms))
    if sel_C is not None:
        assert bool((draw[:, Ca:] == 0).all())
    else:
        at = (2 + 2 * Rb) * Cout
        _check("unit dgamma", vbd[at:at + Cout], vbd[Cout:2 * Cout] / gscale, 2 * U * vbd[Cout:2 * Cout].abs() / gscale + 1e-30)
        _check("unit dbeta", vbd[at + Cout:at + 2 * Cout], vbd[:Cout] / gscale, 2 * U * vbd[:Cout].abs() / gscale + 1e-30)
    # dx and dw from the kernel's own draw
    w64 = u["w"].double().cpu()
    xs = (u["N"], u["Cin"], u["H"], u["W"])
    dxref = R.conv_dgrad(draw, w64, xs, u["stride"], u["pad"], u["off"])
    dxmag = R.conv_dgrad(draw.abs(), w64.abs(), xs, u["stride"], u["pad"], u["off"])
    Kd = Cout * u["k"] * u["k"]
    _check("unit dx", _nchw(dxb), dxref, _f16_bound(dxref, (Kd + 2) * U * dxmag))
    x64 = _nchw(u["x"])
    dwref = R.conv_wgrad(x64, draw, tuple(u["w"].shape), u["stride"], u["pad"], u["off"]) / gscale
    dwmag = R.conv_wgrad(x64.abs(), draw.abs(), tuple(u["w"].shape), u["stride"], u["pad"], u["off"]) / gscale
    d0 = dw0.double().cpu()
    _check("unit dw (accumulated)", dw, d0 + dwref, (n + 4) * U * dwmag + 2 * U * d0.abs())
    return ref


@pytest.mark.parametrize("det", [0, 1])
@pytest.mark.parametrize("case", UNIT_CASES)
def test_conv_bn_act_unit(case, det, lib_option):
    lib_option("FSB_DETERMINISTIC", det)
    if case[8] >= 0:
        lib_option("FSB_CONV_TC2", case[8])
    u = _unit_setup(case, seed=sum(case[:7]))
    Cout = u["Cout"]
    rs = np.random.RandomState(9)
    gamma = torch.from_numpy(rs.uniform(0.5, 1.5, Cout).astype(np.float32)).cuda()
    beta = torch.from_numpy(rs.standard_normal(Cout).astype(np.float32) * 0.1).cuda()
    rm0, rv0 = torch.from_numpy(rs.standard_normal(Cout).astype(np.float32) * 0.1), torch.from_numpy(rs.uniform(0.5, 1.5, Cout).astype(np.float32))
    rm, rv = rm0.cuda(), rv0.cuda()
    nbt = torch.tensor([41], dtype=torch.int64, device="cuda")
    raw, y, vec = _unit_fwd(u, gamma, beta, rm, rv, nbt)
    st, e_var = _check_unit_fwd(u, raw, y, vec, gamma, beta)
    _check_unit_running(u, rm, rv, rm0, rv0, vec, st, e_var)
    assert int(nbt.item()) == 42
    gscale = 8.0
    dw0 = _randn(tuple(u["w"].shape), 77).cuda()
    dy, drawb, vb, dxb, dw = _unit_bwd(u, raw, y, vec, gamma, gscale, dw0, seed=sum(case[:7]) + 1)
    _check_unit_bwd(u, dy, raw, y, vec, gamma, gscale, drawb, vb, dxb, dw, dw0)
    # loose end-to-end check of the whole unit against float64 autograd (fp16 storage of y, draw and dx included)
    x = _nchw(u["x"]).requires_grad_(True)
    w = u["w"].double().cpu().requires_grad_(True)
    r = torch.nn.functional.conv2d(x[:, :, u["off"][0]:, u["off"][1]:], w, None, u["stride"], u["pad"])
    yy = torch.nn.functional.batch_norm(r, None, None, gamma.double().cpu(), beta.double().cpu(), training=True, eps=EPS).relu()
    yy.backward(_nchw(dy))
    rel = lambda a, b: float((a - b).norm() / b.norm())
    errs = (rel(_nchw(y), yy.detach()), rel(_nchw(dxb), x.grad), rel(dw.double().cpu() - dw0.double().cpu(), w.grad / gscale))
    print("unit end-to-end norm-wise errors y %.2e dx %.2e dw %.2e" % errs)
    assert max(errs) < 2e-2


def test_conv_bn_act_unit_selected_sets():
    case = (2, 32, 48, 3, 1, 9, 13, (0, 0), -1, False)
    u = _unit_setup(case, seed=5)
    tab = SelTable([8, 16, 24, 40, 48], seed=11)
    for k in range(5):
        tab.select(k)
        before = tab.snapshot()
        raw, y, vec = _unit_fwd(u, None, None, None, None, None, sel=tab)
        s = tab.sets[k]
        Ca = s["C"]
        Cout = u["Cout"]
        # the active channels like the plain unit with the selected set's gamma / beta / running statistics, the tail exactly 0
        st, e_var = _check_unit_fwd(u, raw, y, vec, s["gamma"], s["beta"], active=Ca)
        _check_unit_running(u, s["running_mean"], s["running_var"], before[k]["running_mean"].view(torch.float32),
                            before[k]["running_var"].view(torch.float32), vec, st, e_var)
        assert int(s["num_batches_tracked"].item()) == int(before[k]["num_batches_tracked"].item()) + 1
        g = torch.zeros(Cout)
        g[:Ca] = s["gamma"].cpu()
        dw0 = _randn(tuple(u["w"].shape), 78).cuda()
        dy, drawb, vb, dxb, dw = _unit_bwd(u, raw, y, vec, None, 2.0, dw0, sel=tab, seed=k)
        _check_unit_bwd(u, dy, raw, y, vec, g.cuda(), 2.0, drawb, vb, dxb, dw, dw0, sel_C=Ca)
        vbd = vb.double().cpu()
        g0 = before[k]["dgamma"].view(torch.float32).double()
        b0 = before[k]["dbeta"].view(torch.float32).double()
        _check("unit sel dgamma", s["dgamma"], g0 + vbd[Cout:Cout + Ca] / 2.0, 4 * U * (g0.abs() + vbd[Cout:Cout + Ca].abs() / 2.0))
        _check("unit sel dbeta", s["dbeta"], b0 + vbd[:Ca] / 2.0, 4 * U * (b0.abs() + vbd[:Ca].abs() / 2.0))
        tab.assert_only_changed(before, k, ("running_mean", "running_var", "num_batches_tracked", "dgamma", "dbeta"))


def test_conv_bn_act_unit_bwd_rejects_dx_without_w_before_touching_gradients():
    """the direct dgrad (here forced) needs the fp32 master weight: without it the backward must fail before the BatchNorm
    stage has added anything into the selected set's gradient slots"""
    u = _unit_setup((2, 32, 48, 3, 1, 9, 13, (0, 0), -1, True), seed=6)
    tab = SelTable([16, 48], seed=12)
    tab.select(0)
    raw, y, vec = _unit_fwd(u, None, None, None, None, None, sel=tab)
    before = tab.snapshot()
    N, Cout, Ho, Wo = u["N"], u["Cout"], u["Ho"], u["Wo"]
    dy = _put(_inbuf(N, Ho, Wo, Cout), 0, _randn((N, Cout, Ho, Wo), 8))
    Rb = L().fsb_stat_rows(N * Ho * Wo)
    draw = _buf(N, Ho, Wo, Cout)
    vb = torch.full(((4 + 2 * Rb) * Cout,), float("nan"), device="cuda")
    dx = _buf(N, u["H"], u["W"], u["Cin"])
    rc = L().fsb_conv_bn_act_train_bwd(C.byref(u["d"]), _p(u["x"]), _p(dy), Cout, _p(y), Cout, _p(raw), Cout, _p(vec), None, 1, _p(u["wt"]),
                                       None, u["w"].stride(0), u["w"].stride(1), _p(draw), Cout, _p(vb), _p(dx), u["Cin"], None, 1.0,
                                       _p(tab.table), _p(tab.idx), _s())
    torch.cuda.synchronize()
    assert rc == INVALID
    tab.assert_only_changed(before, -1, ())


def test_conv_bn_act_unit_rejects_cout_not_multiple_of_8_before_touching_state():
    from fasterseg_b200 import _lib
    N, Cin, Cout, H, W = 1, 16, 20, 6, 7
    x = _put(_inbuf(N, H, W, Cin), 0, _randn((N, Cin, H, W), 1))
    w = _randn((Cout, Cin, 3, 3), 2).cuda() * 0.1
    from fasterseg_b200 import functional as F_
    wp = F_.pack_conv_weight(w, Cin, Cout, 3)
    d = _lib.ConvDesc(N, H, W, Cin, Cout, 3, 1, 1, 1, 0, 0, H, W, Cin, 24, 0)
    dd = _lib.ConvDesc.from_buffer_copy(d)
    dd.flags = _lib.FSB_CONV_STATS | _lib.FSB_CONV_OUT_F32
    rows = L().fsb_conv_stats_rows(C.byref(dd))
    raw = _buf(N, H, W, 24, torch.float32)
    y = _buf(N, H, W, 24)
    vec = torch.zeros((6 + 2 * rows) * Cout + 64, device="cuda")
    gamma, beta = torch.ones(Cout, device="cuda"), torch.zeros(Cout, device="cuda")
    rm, rv = _randn((Cout,), 3).cuda(), _randn((Cout,), 4).abs().cuda() + 0.5
    nbt = torch.tensor([7], dtype=torch.int64, device="cuda")
    before = (_bits(rm), _bits(rv), nbt.cpu().clone())
    rc = L().fsb_conv_bn_act_train_fwd(C.byref(d), _p(x), _p(wp), _p(gamma), _p(beta), EPS, MOM, _p(rm), _p(rv), _p(nbt), _p(raw), 24,
                                       _p(y), 24, _p(vec), 1, None, None, _s())
    torch.cuda.synchronize()
    assert rc == INVALID
    assert torch.equal(_bits(rm), before[0]) and torch.equal(_bits(rv), before[1]) and torch.equal(nbt.cpu(), before[2])


# ---- resize backward -----------------------------------------------------------------------------------------------------------
def _taps_per_input(n_in, n_out):
    return int((R.ac_matrix(n_in, n_out) != 0).sum(0).max())


BILINEAR_BWD_CASES = [((9, 13), (18, 26)), ((17, 23), (34, 46)), ((18, 26), (9, 13)), ((34, 46), (17, 23)), ((16, 32), (128, 256)),
                      ((11, 7), (11, 7)), ((6, 9), (1, 17)), ((1, 9), (5, 17)), ((1, 5), (1, 12)), ((7, 1), (13, 1))]


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("io", BILINEAR_BWD_CASES)
def test_bilinear_bwd(io, masked):
    (Hi, Wi), (Ho, Wo) = io
    N, Cc, off, Ct = 2, 16, 8, 40
    dyb, yb = _inbuf(N, Ho, Wo, Ct), _inbuf(N, Ho, Wo, Ct)
    dy = _put(dyb, off, _randn((N, Cc, Ho, Wo), Hi * Wo, mean=0.25))
    y = _put(yb, off, _randn((N, Cc, Ho, Wo), Ho * Wi))
    dxb = _buf(N, Hi, Wi, Ct)
    dx = dxb[..., off:off + Cc]
    assert L().fsb_bilinear_bwd(N, Cc, Hi, Wi, Ho, Wo, _p(dy), Ct, _p(y) if masked else None, Ct, _p(dx), Ct, _s()) == 0
    torch.cuda.synchronize()
    ref, mag = R.bilinear_bwd(_nchw(dy), Hi, Wi, _nchw(y) if masked else None)
    taps = _taps_per_input(Hi, Ho) * _taps_per_input(Wi, Wo)
    _check("bilinear_bwd %s" % (io,), _nchw(dx), ref, _f16_bound(ref, (taps + 2) * U * mag))
    assert torch.equal(_outside(dxb, off, Cc), _outside(_buf(N, Hi, Wi, Ct), off, Cc))


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("geom", [((9, 12), (13, 21), 2, 1024.0), ((9, 12), (72, 96), 2, 3.0), ((64, 128), (512, 1024), 1, 256.0)])
def test_upsample_logits_bwd(geom, f32):
    (Hi, Wi), (Ho, Wo), N, gscale = geom
    Cc, Ct = 19, 24
    dy = _randn((N, Cc, Ho, Wo), Ho + Wi, mean=0.1, scale=0.5)
    if not f32:
        dy = dy.half().float()
    dyg = dy.cuda().to(torch.float32 if f32 else torch.float16).contiguous()
    dxb = _buf(N, Hi, Wi, Ct)
    assert L().fsb_upsample_logits_bwd(N, Cc, Hi, Wi, Ho, Wo, _p(dyg), int(f32), _p(dxb), Ct, gscale, _s()) == 0
    torch.cuda.synchronize()
    ref, mag = R.upsample_logits_bwd(dy.double(), Hi, Wi, gscale)
    taps = _taps_per_input(Hi, Ho) * _taps_per_input(Wi, Wo)
    _check("upsample_logits_bwd %s" % (geom[:2],), _nchw(dxb[..., :Cc]), ref, _f16_bound(ref, (taps + 3) * U * mag))
    assert torch.equal(_bits(dxb[..., Cc:]), _bits(_buf(N, Hi, Wi, Ct - Cc))), "channels 19..23 were written"


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("Cc", [19, 33, 64])
def test_nchw_grad_to_nhwc_is_exact(Cc, f32):
    for H, W in ((1, 1), (1, 31), (3, 11), (25, 40)):
        N, Ct, gscale = 3, (Cc + 7) // 8 * 8 + 8, 256.0
        dy = _randn((N, Cc, H, W), Cc + H * W)
        if not f32:
            dy = dy.half().float()
        dyg = dy.cuda().to(torch.float32 if f32 else torch.float16).contiguous()
        dxb = _buf(N, H, W, Ct)
        assert L().fsb_nchw_grad_to_nhwc(N, Cc, H, W, _p(dyg), int(f32), _p(dxb), Ct, gscale, _s()) == 0
        torch.cuda.synchronize()
        want = (dy.double() * gscale).half().permute(0, 2, 3, 1)
        assert torch.equal(_bits(dxb[..., :Cc]), _bits(want.contiguous())), "nchw_grad_to_nhwc (%d, %d) not exact" % (H, W)
        assert torch.equal(_bits(dxb[..., Cc:]), _bits(_buf(N, H, W, Ct - Cc)))


# ---- weighted sum, add, ReLU backward ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", range(1, 9))
@pytest.mark.parametrize("pixels", [1000, 50_000])
def test_wsum_fwd_bwd(K, pixels):
    Cc, gscale = 16, 3.0
    xs_b = [_inbuf(1, 1, pixels, Cc + 8 * (k % 3)) for k in range(K)]
    xs = [_put(b, 8 * (k % 3), _randn((1, Cc, 1, pixels), 10 * K + k, mean=0.5)) for k, b in enumerate(xs_b)]
    xcs = (C.c_int * K)(*[b.shape[3] for b in xs_b])
    xp = (C.c_void_p * K)(*[x.data_ptr() for x in xs])
    wts = torch.from_numpy(np.random.RandomState(K).uniform(-1, 1.5, K).astype(np.float32)).cuda()
    outb = _buf(1, 1, pixels, Cc + 16)
    out = outb[..., 8:8 + Cc]
    assert L().fsb_wsum_fwd(K, pixels, Cc, xp, xcs, _p(wts), _p(out), Cc + 16, _s()) == 0
    dout = _put(_inbuf(1, 1, pixels, Cc + 8), 0, _randn((1, Cc, 1, pixels), 99, mean=0.3) * gscale)
    need = [k % 2 == 0 for k in range(K)]
    dxs_b = [_buf(1, 1, pixels, Cc + 8) if need[k] else None for k in range(K)]
    dxs = [b[..., 8:8 + Cc] if b is not None else None for b in dxs_b]
    dxp = (C.c_void_p * K)(*[None if t is None else t.data_ptr() for t in dxs])
    dxcs = (C.c_int * K)(*[Cc + 8 if need[k] else 0 for k in range(K)])
    rows = L().fsb_wsum_rows(pixels, Cc)
    dwts = torch.full((1 + rows, 8), float("nan"), device="cuda")
    assert L().fsb_wsum_bwd(K, pixels, Cc, _p(dout), Cc + 8, xp, xcs, _p(wts), dxp, dxcs, _p(dwts), gscale, _s()) == 0
    torch.cuda.synchronize()
    x64 = [_nchw(x) for x in xs]
    w64 = wts.double().cpu()
    ref = R.wsum_fwd(x64, w64)
    mag = R.wsum_fwd([x.abs() for x in x64], w64.abs())
    _check("wsum_fwd K=%d" % K, _nchw(out), ref, _f16_bound(ref, (K + 1) * U * mag))
    assert torch.equal(_outside(outb, 8, Cc), _outside(_buf(1, 1, pixels, Cc + 16), 8, Cc))
    rdx, rdw, rmag = R.wsum_bwd(_nchw(dout), x64, w64, gscale)
    for k in range(K):
        if need[k]:
            _check("wsum_bwd dx[%d]" % k, _nchw(dxs[k]), rdx[k], _f16_bound(rdx[k], U * rdx[k].abs()))
    d = dwts.double().cpu()
    assert bool(torch.isfinite(d).all()), "a partial row of dwts was not written"
    _check("wsum_bwd dwts K=%d" % K, d[0, :K], rdw, C_SUM * U * rmag + 1e-30)


def test_add_inplace_and_relu_bwd_are_exact():
    pixels, Cc = 3000, 24
    xb = _inbuf(1, 1, pixels, 40)
    x = _put(xb, 8, _randn((1, Cc, 1, pixels), 1))
    yb = _inbuf(1, 1, pixels, 48)
    y = _put(yb, 16, _randn((1, Cc, 1, pixels), 2))
    want = (_nchw(x) + _nchw(y)).half()
    assert L().fsb_add_inplace(pixels, Cc, _p(x), 40, _p(y), 48, _s()) == 0
    torch.cuda.synchronize()
    assert torch.equal(_bits(y.permute(0, 3, 1, 2).contiguous()), _bits(want.contiguous()))
    assert torch.equal(_outside(yb, 16, Cc), _outside(_inbuf(1, 1, pixels, 48), 16, Cc))
    # ReLU backward: dy where y > 0, exactly; zeros and -0.0 in y block
    mb = _inbuf(1, 1, pixels, 32)
    m = _put(mb, 8, _randn((1, Cc, 1, pixels), 3))
    mz = m.clone()
    _inject_zeros(mz)
    m.copy_(mz)
    dxb = _buf(1, 1, pixels, 40)
    dx = dxb[..., 16:16 + Cc]
    assert L().fsb_relu_bwd(pixels, Cc, _p(x), 40, _p(m), 32, _p(dx), 40, _s()) == 0
    torch.cuda.synchronize()
    want = torch.where(_nchw(m) > 0, _nchw(x), torch.zeros((), dtype=F64)).half()
    assert torch.equal(_bits(dx.permute(0, 3, 1, 2).contiguous()), _bits(want.contiguous()))
    assert torch.equal(_outside(dxb, 16, Cc), _outside(_buf(1, 1, pixels, 40), 16, Cc))


# ---- stride-2 dgrad writes every element of dx ---------------------------------------------------------------------------------
@pytest.mark.parametrize("s2_direct", [0, 1])
@pytest.mark.parametrize("geom", [(1, (0, 0), 12, 16), (1, (1, 1), 12, 16), (3, (0, 0), 1, 16), (3, (0, 0), 9, 13)])
def test_stride2_dgrad_overwrites_nan_filled_dx(geom, s2_direct, lib_option):
    from fasterseg_b200 import _lib
    from fasterseg_b200 import functional as F_
    lib_option("FSB_DGRAD_S2_DIRECT", s2_direct)
    k, off, H, W = geom
    N, Cin, Cout, pad = 2, 32, 48, (k - 1) // 2
    Ho, Wo = F_.conv_out_size(H, W, k, 2, pad, 1, off[0], off[1])
    w = (_randn((Cout, Cin, k, k), 5) * 0.2).half().float().cuda()
    wt = F_.pack_conv_weight_dgrad(w, Cin, Cout, k)
    dy = _put(_inbuf(N, Ho, Wo, Cout), 0, _randn((N, Cout, Ho, Wo), 6))
    dx = _buf(N, H, W, Cin)
    d = _lib.ConvDesc(N, H, W, Cin, Cout, k, 2, pad, 1, off[0], off[1], Ho, Wo, Cin, Cout, 0)
    assert L().fsb_conv_dgrad(C.byref(d), _p(dy), Cout, _p(wt), _p(w), w.stride(0), w.stride(1), _p(dx), Cin, _s()) == 0
    torch.cuda.synchronize()
    w64 = w.double().cpu()
    ref = R.conv_dgrad(_nchw(dy), w64, (N, Cin, H, W), 2, pad, off)
    mag = R.conv_dgrad(_nchw(dy).abs(), w64.abs(), (N, Cin, H, W), 2, pad, off)
    _check("dgrad s2 k=%d off=%s H=%d" % (k, off, H), _nchw(dx), ref, _f16_bound(ref, (Cout * k * k + 2) * U * mag))
    assert bool((_nchw(dx)[ref == 0] == 0).all()), "pixels no tap reaches are not exactly 0"
