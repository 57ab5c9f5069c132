"""GPU parity at the sizes BASELINE.json's configs name (round 1 only covered reduced sizes), against digests of the UNMODIFIED
reference produced by oracle/make_golden_baseline.py (tests/golden/baseline_sizes.*):
  C2  student arch_1 eval forward 1 x 3 x 1024 x 2048 -- the benchmarked configuration; this input size is what sends the big layers
      through the window and per-tap modes and the N-split heuristics of conv_tc;
  C3  16-layer supernet pretrain `_loss` + backward at 3 x 3 x 256 x 512 (captured passes, fasterseg_b200/graphed.py);
  C5  16-layer supernet search `_loss` + backward at 2 x 3 x 224 x 448.
Label maps: "bit-exact argmax" cannot hold literally for an fp16-storage pipeline against an fp32 one wherever two logits are
closer than the arithmetic error; the provable statement, asserted here for EVERY pixel of the 1024 x 2048 frame, is: the label
differs from the fp32 result only where the fp32 top-2 margin is below twice the logit tolerance this test asserts."""
import time

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import fasterseg_oracle as orc
from tests import helpers as H
from tests.test_boundary_cpu import _build_student, _build_supernet
from tests.test_student_gpu import _load_seeded

pytestmark = pytest.mark.gpu

# logits: fp16 storage through 45 layers against fp32 -- norm-wise relative error (north_star's "1e-3 relative fp16 tolerance")
NORM_TOL = 1.5e-3
# per-element: |ours - ref| <= ABS_TOL_REL * max|ref|  (the bound the label-map proof uses)
ABS_TOL_REL = 3e-3


def test_student_eval_1024x2048_vs_reference_and_oracle():
    z = H.load_npz("baseline_sizes.npz")
    model, g = _build_student(1)
    model = model.cuda().eval()
    sd = _load_seeded(model, g, 2025)
    x = orc.random_input((1, 3, 1024, 2048), seed=4242)
    with torch.no_grad():
        y = model(x.cuda())
        lab = model.predict_labels(x.cuda())
    torch.cuda.synchronize()
    y = y.cpu().numpy()
    lab = lab.cpu().numpy()
    assert y.shape == (1, 19, 1024, 2048) and lab.shape == (1, 1024, 2048)
    # fused upsample + argmax kernel == argmax of our own logits, bit for bit
    assert np.array_equal(lab, y.argmax(1).astype(np.uint8))

    # ---- against the reference's digest (strided samples of the fp32 result) ----
    ref_s = z["c2/logits.s32"].astype(np.float64)
    got_s = y[:, :, 3::32, 7::32].astype(np.float64)
    scale = float(z["c2/moments"][2])
    nerr = np.linalg.norm(got_s - ref_s) / np.linalg.norm(ref_s)
    maxerr = np.abs(got_s - ref_s).max() / scale
    print("C2 vs reference digest: norm-wise rel err %.3e, max-abs / max|logit| %.3e (max|logit| %.2f)" % (nerr, maxerr, scale))
    assert nerr < NORM_TOL and maxerr < ABS_TOL_REL
    ref_lab, ref_margin = z["c2/argmax.s4"], z["c2/margin.s4"].astype(np.float64)
    mism = lab[:, 1::4, 2::4] != ref_lab
    print("C2 labels vs reference (every 4th pixel): %d of %d differ; largest fp32 margin among them %.3e (bound %.3e)" % (
        int(mism.sum()), mism.size, float(ref_margin[mism].max()) if mism.any() else 0.0, 2 * ABS_TOL_REL * scale))
    assert not mism.any() or ref_margin[mism].max() <= 2 * ABS_TOL_REL * scale
    assert mism.mean() < 2e-3

    # ---- against the CPU oracle at FULL resolution (the oracle is pinned to the reference by tests/test_oracle_golden.py and,
    #      at this size, by the digest comparison below) ----
    st, _ = H.student_structure(1)
    t0 = time.time()
    with torch.no_grad():
        ref = orc.student_forward(x, sd, st, training=False).numpy()
    print("CPU oracle forward at 1024x2048: %.1f s" % (time.time() - t0))
    assert H.rel_err(ref[:, :, 3::32, 7::32], z["c2/logits.s32"]) < 1e-4      # the oracle itself, at this size
    d = np.abs(y.astype(np.float64) - ref)
    nerr = np.linalg.norm(y.astype(np.float64) - ref) / np.linalg.norm(ref)
    amax = np.abs(ref).max()
    print("C2 vs oracle, all 39.8 M logits: norm-wise rel err %.3e, max-abs/max %.3e, 99.9th pct abs err / max %.3e" % (
        nerr, d.max() / amax, np.percentile(d[:, :, ::3, ::5], 99.9) / amax))
    assert nerr < NORM_TOL and d.max() / amax < ABS_TOL_REL
    ref_lab = ref.argmax(1)
    srt = np.sort(ref, axis=1)
    margin = srt[:, -1] - srt[:, -2]
    mism = lab != ref_lab
    n = int(mism.sum())
    worst = float(margin[mism].max()) if n else 0.0
    print("C2 label map: %d of %d pixels (%.4f %%) differ from the fp32 argmax; every one has an fp32 top-2 margin <= %.3e "
          "(bound 2 x logit tolerance = %.3e; median margin of ALL pixels %.3e)" % (n, mism.size, 100.0 * n / mism.size, worst,
                                                                                 2 * ABS_TOL_REL * amax, float(np.median(margin))))
    assert worst <= 2 * ABS_TOL_REL * amax
    # and per pixel, with the error actually made there: a flip needs |err_a| + |err_b| >= margin
    if n:
        idx = np.nonzero(mism)
        err_here = d[idx[0], :, idx[1], idx[2]].max(axis=1)
        assert np.all(margin[mism] <= 2 * err_here + 1e-12)
    assert n / mism.size < 2e-3


def _supernet16(case, z, meta):
    torch.manual_seed(0)
    m = _build_supernet(16)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items() if not k.endswith("num_batches_tracked")}
    sd = orc.random_state_dict(shapes, seed=777)
    own = m.state_dict()
    for k, v in sd.items():
        own[k].copy_(v)
    for k in own:
        if k.startswith(("alpha_", "beta_", "ratio_")):
            own[k].copy_(torch.from_numpy(z["%s/arch:%s" % (case, k)]))
    for mod in m.modules():
        if isinstance(mod, nn.BatchNorm2d):
            mod.eps, mod.momentum = orc.BN_EPS, orc.BN_MOMENTUM
    return m.cuda().train()


@pytest.mark.parametrize("case", ["c3", "c5"])
def test_supernet_16_layer_loss_and_gradients_at_baseline_size(case):
    """BASELINE configs[2] / configs[4]: the whole `_loss` (4 forwards, 5 logits each) + backward of the 16-layer, 252 M
    parameter supernet.  The chain of ~60 train-mode BatchNorm layers with random weights is ill-conditioned: rounding the
    STORED activations to fp16 (the CPU oracle's EMULATE_FP16, arithmetic still fp32) moves the gradient tensors of the
    reference by 23 % (median) at this depth.  Our path has exactly those storage semantics, so the gate is two-sided: our
    deviation from the fp32 reference must be the deviation fp16 storage causes (stored per tensor in the golden file)."""
    from oracle.make_golden_baseline import SUPERNET_CASES
    from oracle.make_golden_supernet import make_target
    z = H.load_npz("baseline_sizes.npz")
    meta = H.load_json("baseline_sizes.json")
    c = SUPERNET_CASES[case]
    B, (Hh, Ww) = c["batch"], c["hw"]
    x = orc.random_input((B, 3, Hh, Ww), seed=778).cuda()
    tgt = torch.from_numpy(make_target(B, Hh // 8, Ww // 8, 779)).cuda()
    m = _supernet16(case, z, meta)
    m._criterion = nn.CrossEntropyLoss(ignore_index=255)
    np.random.seed(c["np_seed"])
    torch.manual_seed(c["torch_seed"])
    t0 = time.time()
    loss = m._loss(x, tgt, c["pretrain"])
    loss.backward()
    torch.cuda.synchronize()
    print("%s: first step (build + capture) %.1f s; captured = %s" % (case, time.time() - t0, m.__dict__.get("_fsb_graph_runner") is not None))
    l_ref, l_emu, lo = float(z[case + ".ref/loss"][0]), float(z[case + ".emu/loss"][0]), float(loss)
    print("%s: loss ours %.5f | reference %.5f | fp16-emulating oracle %.5f" % (case, lo, l_ref, l_emu))
    assert abs(lo - l_ref) <= 2.0 * abs(l_emu - l_ref) + 1e-3 * abs(l_ref)
    grads = {k: p.grad for k, p in m.named_parameters()}
    keys = meta[case + ".ref.grad_keys"]
    assert sorted(k for k, g in grads.items() if g is not None) == sorted(keys)
    assert sum(1 for g in grads.values() if g is None) == meta[case + ".no_grad_count"]
    n_ref = z[case + ".ref/grad_norms"]
    n_emu = dict(zip(meta[case + ".emu.grad_keys"], z[case + ".emu/grad_norms"]))
    n_ours = np.array([float(grads[k].double().norm()) for k in keys])
    ok = n_ref > 1e-10
    r_ours = np.abs(np.log(n_ours[ok] / n_ref[ok]))
    r_emu = np.abs(np.log(np.array([n_emu[k] for k in keys])[ok] / n_ref[ok]))
    g_ours, g_ref, g_emu = float(np.sqrt((n_ours ** 2).sum())), float(z[case + ".ref/grad_norm"][0]), float(z[case + ".emu/grad_norm"][0])
    print("%s: global gradient norm ours %.5f | reference %.5f | emulation %.5f" % (case, g_ours, g_ref, g_emu))
    print("%s: per-tensor |log(norm / reference norm)| over %d tensors: median ours %.3e emulation %.3e; 99th pct ours %.3e emulation %.3e" % (
        case, int(ok.sum()), np.median(r_ours), np.median(r_emu), np.percentile(r_ours, 99), np.percentile(r_emu, 99)))
    assert abs(g_ours - g_ref) <= 2.0 * abs(g_emu - g_ref) + 2e-2 * g_ref
    assert np.median(r_ours) <= 1.5 * np.median(r_emu) + 1e-2
    assert np.percentile(r_ours, 99) <= 2.0 * np.percentile(r_emu, 99) + 5e-2
    sel = meta[case + ".selected"]
    e_emu = z[case + ".emu/selected_rel_err"]
    e_ours = []
    for k in sel:
        g = grads[k].detach().float().cpu().numpy()
        ref = z["%s.ref/grad:%s" % (case, k)]
        if g.ndim == 4 and g.nbytes > 150_000:       # the strides oracle/make_golden_baseline.py:_strided applied
            g = g[::4, ::4]
        if g.ndim == 4 and g.nbytes > 40_000:
            g = g[::2, ::2]
        assert g.shape == ref.shape, (k, g.shape, ref.shape)
        e_ours.append(H.rel_err(g, ref))
    e_ours = np.array(e_ours)
    arch = [i for i, k in enumerate(sel) if k.startswith(("alpha_", "beta_"))]
    print("%s: %d selected tensors vs reference values: median rel err ours %.3e | emulation %.3e; architecture parameters: ours %s" % (
        case, len(sel), np.median(e_ours), np.median(e_emu), np.round(e_ours[arch], 3).tolist()))
    assert np.median(e_ours) <= 1.5 * np.median(e_emu) + 1e-2
    worst = max((eo / (ee + 1e-9), k) for eo, ee, k in zip(e_ours, np.maximum(e_emu, np.median(e_emu)), sel) if not k.startswith("ratio_"))
    print("%s: worst err(ours) / err(emulation) over selected tensors: %.2f (%s)" % (case, worst[0], worst[1]))
    assert worst[0] <= 3.0
    sda = m.state_dict()
    for k in z.files:
        if k.startswith(case + ".ref/after:"):
            name = k.split("after:")[1]
            np.testing.assert_allclose(sda[name].cpu().numpy(), z[k], rtol=5e-2, atol=5e-3, err_msg=name)
