"""K14 on the GPU: the supernet's expected latency and its gradient (csrc/latency.cu, one launch each) against the reference's
values and gradients (tests/golden/supernet_latency_grad.npz, every case including L16 at 1024x2048), against the walk run on the
same CUDA parameters, without host synchronisation, and through three architect steps with Adam."""
import numpy as np
import pytest
import torch

from fasterseg_b200 import operations
from fasterseg_b200 import supernet_latency as SL
from fasterseg_b200.runtime import LaunchCounter
from oracle import make_golden_latency as mk
from oracle import make_golden_latency_grad as mkg
from oracle.make_golden_decode import SyntheticLatencyTable
from tests.test_supernet_latency_device_cpu import IDS, assert_matches, golden_of

pytestmark = pytest.mark.gpu


def _model(case, monkeypatch):
    from fasterseg_b200.model_search import Network_Multi_Path
    monkeypatch.setattr(operations, "latency_lookup_table", SyntheticLatencyTable())
    model = mk.build(Network_Multi_Path, case["layers"])
    mk.randomise_arch(model, case["seed"])
    return model.cuda()


def _spy(monkeypatch):
    calls = []
    orig = SL.expected_latency
    monkeypatch.setattr(SL, "expected_latency", lambda m, plan: calls.append(plan) or orig(m, plan))
    return calls


@pytest.mark.parametrize("case", mk.CASES, ids=IDS)
def test_kernel_matches_reference(case, monkeypatch):
    model = _model(case, monkeypatch)
    calls = _spy(monkeypatch)
    assert_matches(mkg.evaluate_grad(model, case), golden_of(case), IDS(case))
    assert len(calls) == 2 * len(mk.FLAGS)        # every call took the kernel


@pytest.mark.parametrize("case", mk.CASES, ids=IDS)
def test_kernel_matches_cuda_walk(case, monkeypatch):
    model = _model(case, monkeypatch)
    got = mkg.evaluate_grad(model, case)
    monkeypatch.setattr(SL, "ENABLED", False)
    calls = _spy(monkeypatch)
    walk = mkg.evaluate_grad(model, case)
    assert not calls
    assert_matches(got, walk, IDS(case))


def test_no_sync_and_one_launch_each(monkeypatch):
    model = _model(mk.CASES[-1], monkeypatch)
    model.arch_idx = 1
    for flags in ((True, False, False), (False, True, False), (False, False, True)):
        model.forward_latency((3, 1024, 2048), *flags).backward()      # plans built and copied to the device
    torch.cuda.synchronize()
    for flags in ((True, False, False), (False, True, False), (False, False, True)):
        with LaunchCounter() as fwd:
            torch.cuda.set_sync_debug_mode("error")
            try:
                lat = model.forward_latency((3, 1024, 2048), *flags)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        with LaunchCounter() as bwd:
            torch.cuda.set_sync_debug_mode("error")
            try:
                lat.backward()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        assert (fwd.n, dict(fwd.by_name)) == (1, {"fsb_supernet_latency_fwd": 1}), flags
        assert (bwd.n, dict(bwd.by_name)) == (1, {"fsb_supernet_latency_bwd": 1}), flags
    torch.cuda.synchronize()


def _architect_steps(model, n, seed):
    """the latency half of search/architect.py:45-79 (first order) with latency_weight = [0, 1e-2], restated"""
    opts = [torch.optim.Adam(p, lr=3e-4, betas=(0.5, 0.999)) for p in model._arch_parameters]
    weights = [0, 1e-2]
    torch.manual_seed(seed)
    np.random.seed(seed)
    for _ in range(n):
        for o in opts:
            o.zero_grad()
        loss_latency = 0
        model.prun_mode = None
        for idx in range(len(opts)):
            model.arch_idx = idx
            if weights[idx] > 0:
                latency = 1. / 500 * model.forward_latency((3, 1024, 2048), alpha=True, beta=False, ratio=False)
                latency = latency + 497. / 500 * model.forward_latency((3, 1024, 2048), alpha=False, beta=True, ratio=False)
                latency = latency + 2. / 500 * model.forward_latency((3, 1024, 2048), alpha=False, beta=False, ratio=True)
                loss_latency = loss_latency + latency * weights[idx]
        loss_latency.backward()
        for o in opts:
            o.step()
    return [p.detach().clone() for ps in model._arch_parameters for p in ps]


def test_architect_steps_match_walk(monkeypatch):
    case = mk.CASES[-1]
    got = _architect_steps(_model(case, monkeypatch), 3, 11)
    monkeypatch.setattr(SL, "ENABLED", False)
    want = _architect_steps(_model(case, monkeypatch), 3, 11)
    for g, w in zip(got, want):     # per tensor, relative to its largest entry
        assert (g - w).abs().max() <= 1e-5 * w.abs().max(), (g - w).abs().max()
    init = [p.detach() for ps in _model(case, monkeypatch)._arch_parameters for p in ps]
    assert any(not torch.equal(g, i.to(g.device)) for g, i in zip(got, init))      # the steps did move the student's arch parameters
