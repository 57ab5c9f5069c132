"""tests/golden/conv_bwd_census.json is what the training steps run: regenerated on the CPU stand-in backend it must match, and it
must contain the geometries whose branches tests/test_conv_bwd_gpu.py relies on it for."""
import json

import pytest

from tests import conv_bwd_census as CC


@pytest.fixture(scope="module")
def fresh():
    return CC.generate()


def test_census_matches_a_fresh_recording(fresh):
    assert json.loads(CC.dumps(fresh)) == CC.load(), "the networks' backward conv calls changed: rerun python -m tests.conv_bwd_census"


def test_census_covers_the_kernels_branches(fresh):
    gs = CC.geometries(fresh)
    wg = [g for g in gs if g["op"] == "wgrad"]
    dg = [g for g in gs if g["op"] == "dgrad"]
    assert wg and dg and {g["run"] for g in gs} == set(CC.RUNS)
    for op in (wg, dg):
        assert any(g["k"] == 1 and g["stride"] == 2 and (g["off_h"], g["off_w"]) == (1, 1) for g in op), "1x1 stride 2, offset (1, 1)"
        assert any(g["k"] == 3 and g["stride"] == 2 for g in op), "3x3 stride 2"
        assert any((g["W"] - g["off_w"] + 2 * g["pad"] - g["k"]) // g["stride"] + 1 < 16 for g in op), "Wo < 16"
        assert any(g["w_stride_o"] > g["Cin"] * g["k"] ** 2 for g in op), "sliced master weight"
        assert any(g["Cin"] % 64 for g in op) and any(g["Cout"] % 64 for g in op), "channel counts off the 64-channel tiles"
    assert any(g["accumulate"] == 1 for g in wg), "accumulate = 1"
    assert {g["gscale"] for g in wg} == {1024.0}
