"""The latency/ deployment network on the GPU: the nearest kernels against torch's CPU F.interpolate(mode='nearest') bit for bit,
the conv resize folds (FSB_CONV_X_DOWN2 / FSB_CONV_Y_UP2) against conv + the standalone nearest kernel bit for bit (in the conv_tc
instance a CUDA-graph capture shows), the unsupported flag combinations, the network against the reference latency/ goldens
(tests/golden/latency_variant.npz) and the resize census of the 1024x2048 frame."""
import json
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from oracle import fasterseg_oracle as orc
from tests import helpers as H

pytestmark = pytest.mark.gpu

_UP2 = re.compile(r"conv_tc_up2_kernel")
_PLAIN = re.compile(r"conv_tc_kernel")
_WINDOW = re.compile(r"(<\s*64,\s*\d+,\s*true\s*>|ILi64ELi\d+ELb1E)")
_PER_TAP = re.compile(r"(<\s*\d+,\s*\d+,\s*false\s*>|ILi\d+ELi\d+ELb0E)")


def _F():
    from fasterseg_b200 import functional as F_
    return F_


def _instances(fn, tmp_path):
    """conv_tc kernel names of a CUDA-graph capture of fn (never replayed)"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    g.enable_debug_mode()
    with torch.cuda.graph(g):
        fn()
    torch.cuda.synchronize()
    dot = tmp_path / "g.dot"
    g.debug_dump(str(dot))
    return re.findall(r"conv_tc_(?:up2_)?kernel[\w<>, ]*", dot.read_text())


def _nan_slice(N, C, H, W, lo=8, hi=8):
    """(N, C, H, W) fp16 NHWC view into a buffer whose other channels are NaN"""
    buf = torch.full((N, H, W, lo + C + hi), float("nan"), device="cuda", dtype=torch.float16)
    return buf, buf.permute(0, 3, 1, 2)[:, lo:lo + C]


def _rand16(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal(shape).astype(np.float32)).half()


def _torch_nearest(x16, size):
    return TF.interpolate(x16.float(), size=size, mode="nearest").half()


NEAREST_CASES = [((2, 16, 8, 12), (4, 6)), ((1, 24, 7, 9), (3, 4)), ((3, 8, 5, 11), (2, 5)), ((2, 32, 4, 6), (8, 12)),
                 ((1, 16, 3, 5), (24, 40)), ((2, 8, 3, 5), (1, 2)), ((2, 8, 1, 2), (3, 5)), ((1, 64, 16, 32), (128, 256)),
                 ((3, 16, 6, 10), (3, 5)), ((2, 40, 13, 7), (6, 3))]


@pytest.mark.parametrize("shape,size", NEAREST_CASES)
def test_nearest_fwd_bit_exact(shape, size):
    F_ = _F()
    N, C, H, W = shape
    x = _rand16(shape, sum(shape))
    xbuf, xg = _nan_slice(N, C, H, W)
    xg.copy_(x.cuda())
    ybuf, yg = _nan_slice(N, C, size[0], size[1], lo=16, hi=8)
    F_.nearest(xg, size, out=yg)
    torch.cuda.synchronize()
    want = _torch_nearest(x, size)
    assert torch.equal(yg.cpu().view(torch.int16), want.view(torch.int16))
    assert torch.isnan(ybuf[..., :16]).all() and torch.isnan(ybuf[..., 16 + C:]).all()   # neighbouring channels untouched


LOGIT_CASES = [((1, 19, 16, 32), (128, 256)), ((2, 19, 3, 5), (24, 40)), ((1, 19, 7, 9), (3, 4)), ((1, 19, 5, 3), (2, 5)),
               ((2, 7, 4, 6), (33, 50)), ((1, 19, 128, 256), (1024, 2048))]


@pytest.mark.parametrize("shape,size", LOGIT_CASES)
def test_nearest_logits_and_argmax_bit_exact(shape, size):
    F_ = _F()
    N, C, H, W = shape
    # few distinct levels: many ties between classes, so 'first maximum wins' is exercised
    x = (torch.from_numpy(np.random.RandomState(H * W).randint(-3, 4, shape).astype(np.float32)) * 0.25).half()
    _, xg = _nan_slice(N, C, H, W, lo=0, hi=(8 - C % 8) % 8 + 8)
    xg.copy_(x.cuda())
    want = TF.interpolate(x.float(), size=size, mode="nearest")
    for dtype in (torch.float32, torch.float16):
        y = F_.upsample_logits_nearest(xg, size, dtype=dtype)
        torch.cuda.synchronize()
        assert y.dtype == dtype and torch.equal(y.cpu().float(), want)
    lab = F_.upsample_argmax_nearest(xg, size)
    torch.cuda.synchronize()
    assert torch.equal(lab.cpu(), want.argmax(1).to(torch.uint8))
    assert torch.equal(lab, y.argmax(1).to(torch.uint8))


def _conv_problem(N, Cin, Cout, k, seed):
    w = torch.from_numpy(np.random.RandomState(seed).standard_normal((Cout, Cin, k, k)).astype(np.float32)) * (2.0 / (Cin * k * k)) ** 0.5
    rs = np.random.RandomState(seed + 1)
    scale = torch.from_numpy(rs.uniform(0.5, 1.5, Cout).astype(np.float32)).cuda()
    shift = torch.from_numpy(rs.standard_normal(Cout).astype(np.float32) * 0.2).cuda()
    return _F().pack_conv_weight(w.cuda(), Cin, Cout, k), scale, shift


# (N, Cin, Cout, k, H, W of the conv's input at half resolution, FSB_CONV_TC2 mode)
FOLD_CASES = [(1, 32, 32, 3, 16, 32, 1), (1, 32, 32, 3, 16, 32, 0), (2, 64, 64, 3, 24, 40, 1), (2, 64, 96, 3, 20, 36, 0),
              (1, 128, 128, 3, 12, 20, 1), (3, 48, 48, 3, 9, 13, 1), (1, 64, 64, 1, 16, 32, 0), (2, 256, 128, 1, 6, 10, 0),
              (1, 128, 64, 1, 5, 7, 0), (1, 96, 32, 3, 64, 128, 1)]


@pytest.mark.parametrize("case", FOLD_CASES)
def test_conv_folds_bit_exact(case, lib_option, tmp_path):
    F_ = _F()
    N, Cin, Cout, k, H, W, mode = case
    lib_option("FSB_CONV_TC2", mode)
    mode_re = _WINDOW if (mode == 1 and k == 3) else _PER_TAP
    pad = k // 2
    wp, sc, sh = _conv_problem(N, Cin, Cout, k, Cin + Cout + H)
    _, xfull = _nan_slice(N, Cin, 2 * H, 2 * W)
    xfull.copy_(_rand16((N, Cin, 2 * H, 2 * W), H * W).cuda())
    # X_DOWN2: conv(x at 2H x 2W, down2) == conv(nearest /2 (x))
    down = F_.nearest(xfull, (H, W))
    ref = F_.conv_fwd(down, wp, Cout, k, 1, pad, sc, sh, relu=True)
    names = _instances(lambda: F_.conv_fwd(xfull, wp, Cout, k, 1, pad, sc, sh, relu=True, down2=True), tmp_path)
    assert names and all(_PLAIN.search(n) and mode_re.search(n) for n in names), names
    got = F_.conv_fwd(xfull, wp, Cout, k, 1, pad, sc, sh, relu=True, down2=True)
    torch.cuda.synchronize()
    assert torch.equal(got.cpu().view(torch.int16), ref.cpu().view(torch.int16))
    # Y_UP2 into a channel slice: conv(x, up2) == nearest x2 (conv(x))
    ybuf, yg = _nan_slice(N, Cout, 2 * H, 2 * W, lo=8, hi=16)
    names = _instances(lambda: F_.conv_fwd(down, wp, Cout, k, 1, pad, sc, sh, relu=True, out=yg, up2=True), tmp_path)
    assert names and all(_UP2.search(n) and mode_re.search(n) for n in names), names
    want = F_.nearest(ref, (2 * H, 2 * W))
    torch.cuda.synchronize()
    assert torch.equal(yg.cpu().view(torch.int16), want.cpu().view(torch.int16))
    assert torch.isnan(ybuf[..., :8]).all() and torch.isnan(ybuf[..., 8 + Cout:]).all()
    # both folds in one conv (a stride-1 zoomed cell with even sides)
    both = F_.conv_fwd(xfull, wp, Cout, k, 1, pad, sc, sh, relu=True, down2=True, up2=True)
    torch.cuda.synchronize()
    assert torch.equal(both.cpu().view(torch.int16), want.cpu().view(torch.int16))


def test_unsupported_fold_combinations_raise():
    from fasterseg_b200 import _lib
    F_ = _F()
    wp, sc, sh = _conv_problem(1, 32, 32, 3, 7)
    x = _rand16((1, 32, 16, 16), 3).cuda().contiguous(memory_format=torch.channels_last)
    cases = [
        lambda: F_.conv_fwd(x, wp, 32, 3, 1, 1, out_f32=True, up2=True),
        lambda: F_.conv_fwd(x, wp, 32, 3, 1, 1, stats=F_.conv_stats_buffer(x, 32, 3, 1, 1), up2=True),
        lambda: F_.conv_fwd(x, wp, 32, 3, 1, 1, force_direct=True, up2=True),
        lambda: F_.conv_fwd(x, wp, 32, 3, 1, 1, force_direct=True, down2=True),
        lambda: F_.conv_fwd(x, wp, 32, 3, 2, 1, down2=True),
    ]
    wp12, _, _ = _conv_problem(1, 32, 12, 3, 8)
    cases.append(lambda: F_.conv_fwd(x, wp12, 12, 3, 1, 1, up2=True))            # Cout % 8 != 0: no TMA-store epilogue
    x8 = _rand16((1, 8, 16, 16), 4).cuda().contiguous(memory_format=torch.channels_last)
    wp8, _, _ = _conv_problem(1, 8, 16, 3, 9)
    cases.append(lambda: F_.conv_fwd(x8, wp8, 16, 3, 1, 1, up2=True))              # Cin < 16: direct kernel
    for fn in cases:
        with pytest.raises(_lib.FsbError):
            fn()
    torch.cuda.synchronize()   # nothing was launched that could fault


def _load_seeded(model, shapes, seed):
    sd = orc.random_state_dict({k: tuple(v) for k, v in shapes.items()}, seed=seed)
    own = model.state_dict()
    seen = set()
    with torch.no_grad():
        for k in sorted(sd):
            if own[k].data_ptr() not in seen:
                seen.add(own[k].data_ptr())
                own[k].copy_(sd[k])


def _golden():
    g = H.load_npz("latency_variant.npz")
    return g, json.loads(bytes(g["meta"]).decode())


def _network(tag):
    from fasterseg_b200 import zoo
    g, meta = _golden()
    m = meta[tag]
    arch = 0 if tag == "arch0" else 1
    model = zoo.build_network(arch, lasts=m["lasts"], variant="latency").cuda().eval()
    _load_seeded(model, m.get("shapes", meta["arch1"]["shapes"]), m["seed_weights"])   # the full frame is arch_1
    return model, g, m


@pytest.mark.parametrize("arch", [0, 1])
@pytest.mark.parametrize("hw", [(64, 128), (96, 160)])
def test_network_matches_reference_latency_goldens(arch, hw):
    model, g, _ = _network("arch%d" % arch)
    x = orc.random_input((1, 3) + hw, seed=40 + hw[0] + hw[1]).cuda()
    with torch.no_grad():
        y = model(x)
        lab = model.predict_labels(x)
    torch.cuda.synchronize()
    assert y.dtype == torch.float32 and tuple(y.shape) == (1, 19) + hw
    yn = y.cpu().numpy()
    ref = g["arch%d/%dx%d/logits.s4" % (arch, hw[0], hw[1])].astype(np.float64)
    got = yn[:, :, ::4, ::4].astype(np.float64)
    nerr = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    maxerr = np.abs(got - ref).max() / np.abs(ref).max()
    print("arch%d %s: norm-rel %.3e max-abs/max %.3e" % (arch, hw, nerr, maxerr))
    assert maxerr < 3e-3 and nerr < 3e-3
    assert (lab.cpu().numpy() == g["arch%d/%dx%d/argmax" % (arch, hw[0], hw[1])]).mean() > 0.995
    assert np.array_equal(lab.cpu().numpy(), yn.argmax(1).astype(np.uint8))


def test_single_conv_factorized_reduce_matches_golden():
    from fasterseg_b200.latency_variant import operations as lat_ops
    g, meta = _golden()
    fr = meta["factorized_reduce"]
    op = lat_ops.FactorizedReduce(fr["C_in"], fr["C_out"], 2, slimmable=False).cuda().eval()
    _load_seeded(op, fr["shapes"], fr["seed_weights"])
    x = orc.random_input((2, fr["C_in"]) + tuple(fr["hw"]), seed=fr["seed_input"]).cuda()
    with torch.no_grad():
        y = _F().to_nchw(op(x)).cpu().numpy()
    assert H.rel_err(y, g["factorized_reduce/out"]) < 3e-3


def test_full_frame_digest_and_resize_census():
    """arch_1 at 1x3x1024x2048: logits digest within tolerance; a label may differ from the fp32 reference only where its top-2
    margin is below twice the logit tolerance (DESIGN.md section 4); the captured frame runs no standalone nearest kernel and
    exactly one final upsample"""
    from fasterseg_b200.runtime import LaunchCounter
    model, g, m = _network("full")
    x = orc.random_input((1, 3, 1024, 2048), seed=m["seed_input"]).cuda()
    with torch.no_grad():
        y = model(x)
        lab = model.predict_labels(x)
    torch.cuda.synchronize()
    yn = y.cpu().numpy()
    ref = g["full/logits.s32"].astype(np.float64)
    got = yn[:, :, 3::32, 7::32].astype(np.float64)
    tol = 3e-3
    assert np.abs(got - ref).max() / np.abs(ref).max() < tol and np.linalg.norm(got - ref) / np.linalg.norm(ref) < tol
    labs = lab.cpu().numpy()[:, 1::4, 2::4]
    differs = labs != g["full/argmax.s4"]
    bound = 2 * tol * float(g["full/abs_max"])
    print("full frame: %d of %d sampled labels differ, largest margin among them %.3e (bound %.3e)"
          % (int(differs.sum()), differs.size, float(g["full/margin.s4"][differs].max()) if differs.any() else 0.0, bound))
    assert not differs.any() or float(g["full/margin.s4"][differs].max()) <= bound
    assert np.array_equal(lab.cpu().numpy(), yn.argmax(1).astype(np.uint8))
    for mode, final in (("logits", "fsb_upsample_logits_nearest_nchw"), ("labels", "fsb_upsample_argmax_nearest")):
        run = (lambda: model(x)) if mode == "logits" else (lambda: model.predict_labels(x))
        graph = torch.cuda.CUDAGraph()
        with LaunchCounter() as lc, torch.no_grad(), torch.cuda.graph(graph):
            run()
        torch.cuda.synchronize()
        assert lc.by_name["fsb_nearest_fwd"] == 0, lc.by_name
        assert lc.by_name[final] == 1, lc.by_name
        assert sum(v for k, v in lc.by_name.items() if "bilinear" in k or k in ("fsb_upsample_logits_nchw", "fsb_upsample_argmax")) == 0
