"""tests/golden/conv_fwd_census.json is what the networks run: regenerated on the CPU stand-in backend it must match, and it must
contain the geometries whose branches tests/test_conv_fwd_gpu.py relies on it for."""
import json

import pytest

from tests import conv_fwd_census as FC
from tests.conv_harness import STATS, X_DOWN2, Y_UP2, fwd_plan

H100_SMS = 132


@pytest.fixture(scope="module")
def fresh():
    return FC.generate()


def test_census_matches_a_fresh_recording(fresh):
    assert json.loads(FC.dumps(fresh)) == FC.load(), "the networks' forward conv calls changed: rerun python -m tests.conv_fwd_census"


def _plan(g):
    return fwd_plan(g["N"], g["H"], g["W"], g["Cin"], g["Cout"], g["k"], g["stride"], g["pad"], g["dil"], (g["off_h"], g["off_w"]),
                    g["x_cstride"], g["flags"], sms=H100_SMS)


def test_census_covers_the_kernels_branches(fresh):
    gs = FC.geometries(fresh)
    assert {g["run"] for g in gs} == set(FC.RUNS) and len(gs) > 100
    convs = [g for g in gs if g["op"] in ("conv", "unit")]
    s1k3 = [g for g in convs if g["k"] == 3 and g["stride"] == 1 and not _plan(g)["direct"]]
    assert any(_plan(g)["ctas"] > H100_SMS and _plan(g)["win"] for g in s1k3), "3x3 stride 1, window mode by default"
    assert any(not _plan(g)["win"] for g in s1k3), "3x3 stride 1, per-tap mode by default"
    assert any(g["flags"] & STATS and g["stats_off"] > 0 for g in convs), "statistics at stats_off > 0"
    # the student's latency network never folds both resizes into one conv at 1024 x 2048: the edge grid has that case
    for f in (X_DOWN2, Y_UP2):
        assert any(g["flags"] & (X_DOWN2 | Y_UP2) == f for g in convs), "X_DOWN2 / Y_UP2 flags %d" % f
    assert any(g["Cout"] % 8 for g in convs), "Cout % 8 != 0 (the class heads)"
    assert any(_plan(g)["Wo"] < 16 for g in convs), "Wo < 16"
    assert any(g["k"] == 3 and g["stride"] == 2 for g in convs), "3x3 stride 2"
    assert any(g["k"] == 1 and g["stride"] == 2 and (g["off_h"], g["off_w"]) == (1, 1) for g in convs), "1x1 stride 2, offset (1, 1)"
    assert any(g["w_stride_o"] > g["Cin"] * g["k"] ** 2 for g in convs), "sliced master weight"
    assert any(g["Cin"] % 64 for g in convs if not _plan(g)["direct"]), "Cin % 64 != 0 on conv_tc"
    assert any(g["y_coff"] > 0 for g in convs if g["op"] == "conv"), "y view at a channel offset (zero-copy concat)"
    assert any(_plan(g)["direct"] for g in convs), "direct kernel (Cin < 16)"
    assert {g["op"] for g in gs} >= {"conv", "unit", "stem_nchw"}
