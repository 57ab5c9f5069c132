"""The latency/ deployment network variant (fasterseg_b200/latency_variant) without a GPU: checkpoint format against the reference
latency/ modules (tests/golden/latency_variant.npz, oracle/make_golden_latency_variant.py), latency-table keys, the launcher's
directory rule, the CPU oracle's nearest path against the goldens, the new wrappers' marshalling, and the inference-only guard."""
import json

import numpy as np
import pytest
import torch

from fasterseg_b200 import _lib, launch, zoo
from fasterseg_b200 import functional as F_
from fasterseg_b200 import operations as train_ops
from fasterseg_b200.latency_variant import operations as lat_ops
from oracle import fasterseg_oracle as orc
from oracle import latency_variant_oracle as lvo
from tests import helpers as H
from tests.test_marshalling_cpu import act, fake  # noqa: F401  (fixture)


def golden():
    g = H.load_npz("latency_variant.npz")
    return g, json.loads(bytes(g["meta"]).decode())


def shapes(module):
    return {k: list(v.shape) for k, v in module.state_dict().items() if not k.endswith("num_batches_tracked")}


@pytest.mark.parametrize("arch", [0, 1])
def test_state_dict_matches_reference_latency_network(arch):
    _, meta = golden()
    m = meta["arch%d" % arch]
    model = zoo.build_network(arch, lasts=m["lasts"], variant="latency")
    assert shapes(model) == m["shapes"]


def test_single_conv_stride2_factorized_reduce_matches_reference():
    _, meta = golden()
    fr = meta["factorized_reduce"]
    op = lat_ops.FactorizedReduce(fr["C_in"], fr["C_out"], 2, slimmable=False)
    assert shapes(op) == fr["shapes"] and "conv2.weight" not in op.state_dict()
    assert tuple(op.conv1.weight.shape) == (fr["C_out"], fr["C_in"], 1, 1)
    # the train variant's two-conv form is untouched, and so are the slimmable and stride-1 forms
    assert "conv2.weight" in train_ops.FactorizedReduce(fr["C_in"], fr["C_out"], 2, slimmable=False).state_dict()
    for args in ((32, 48, 2, True), (32, 48, 1, True), (32, 32, 1, False)):
        assert shapes(lat_ops.FactorizedReduce(*args)) == shapes(train_ops.FactorizedReduce(*args))


def test_public_surface_matches_train_operations():
    assert lat_ops.__all__ == train_ops.__all__
    assert lat_ops.OPS_name == train_ops.OPS_name and list(lat_ops.OPS_Class) == list(train_ops.OPS_Class)
    assert lat_ops.OPS_Class["conv_downup"] is lat_ops.BasicResidual_downup_1x
    assert lat_ops.OPS_Class["conv_2x_downup"].__name__ == "BasicResidual_downup_2x"


class _Table(dict):
    """latency table that has every key: value = a deterministic function of the key; records the lookups"""

    def __init__(self):
        super().__init__()
        self.seen = []

    def __contains__(self, k):
        return True

    def __getitem__(self, k):
        self.seen.append(k)
        return (hash(k) % 1000) / 1000.0


@pytest.mark.parametrize("arch", [0, 1])
def test_forward_latency_same_keys_and_totals_as_train(arch, monkeypatch):
    import zlib
    results = []
    for variant in ("train", "latency"):
        table = _Table()
        table.__class__.__getitem__ = lambda self, k: (self.seen.append(k), zlib.crc32(k.encode()) % 1000 / 1000.0)[1]
        monkeypatch.setattr(train_ops, "latency_lookup_table", table)
        model = zoo.build_network(arch, variant=variant)
        total, shape = model.forward_latency((3, 1024, 2048))
        results.append((table.seen, total, shape))
    assert results[0][0] == results[1][0] and len(results[0][0]) > 10
    assert results[0][1] == pytest.approx(results[1][1]) and results[0][2] == results[1][2]


def test_launcher_picks_variant_by_script_directory(tmp_path):
    lat = launch.shadow_module_names(str(tmp_path / "FasterSeg" / "latency" / "run_latency.py"))
    assert lat["operations"] == "fasterseg_b200.latency_variant.operations"
    assert lat["model_seg"] == "fasterseg_b200.latency_variant.model_seg"
    assert lat["slimmable_ops"] == "fasterseg_b200.slimmable_ops" and lat["seg_oprs"] == "fasterseg_b200.seg_oprs"
    for d in ("train", "search", "tools", "latency_old"):
        other = launch.shadow_module_names(str(tmp_path / d / "script.py"))
        assert other == {n: "fasterseg_b200." + n for n in launch.SHADOWED}
    assert launch.shadow_module_names(None) == {n: "fasterseg_b200." + n for n in launch.SHADOWED}


def test_zoo_variant_argument():
    assert type(zoo.build_network(1)).__module__ == "fasterseg_b200.model_seg"
    assert type(zoo.build_network(1, variant="latency")).__module__ == "fasterseg_b200.latency_variant.model_seg"
    with pytest.raises(ValueError):
        zoo.build_network(1, variant="nearest")


def test_nearest_index_rule_matches_torch():
    for n_in in (1, 2, 3, 5, 7, 9, 13, 64, 97, 128):
        for n_out in sorted({1, 2, 3, 4, 5, max(1, n_in // 2), 2 * n_in, 8 * n_in, 37}):
            x = torch.arange(n_in, dtype=torch.float32).view(1, 1, 1, n_in)
            ref = torch.nn.functional.interpolate(x, size=(1, n_out), mode="nearest").view(-1).long()
            assert torch.equal(lvo.nearest_index(n_in, n_out), ref), (n_in, n_out)


def test_resize_fold_decision():
    assert lat_ops.resize_fold((64, 128), (32, 64)) == "down2"
    assert lat_ops.resize_fold((32, 64), (64, 128)) == "up2"
    assert lat_ops.resize_fold((3, 5), (1, 2)) is None and lat_ops.resize_fold((1, 2), (3, 5)) is None
    assert lat_ops.resize_fold((6, 5), (3, 2)) is None and lat_ops.resize_fold((4, 4), (4, 4)) is None


@pytest.mark.parametrize("arch", [0, 1])
@pytest.mark.parametrize("hw", [(64, 128), (96, 160)])
def test_oracle_nearest_network_matches_golden(arch, hw):
    g, meta = golden()
    m = meta["arch%d" % arch]
    st, _ = H.student_structure(arch, lasts=m["lasts"])
    sd = orc.random_state_dict({k: tuple(v) for k, v in m["shapes"].items()}, seed=m["seed_weights"])
    x = orc.random_input((1, 3) + hw, seed=40 + hw[0] + hw[1])
    with torch.no_grad():
        out = lvo.student_forward(x, sd, st).numpy()
    want = g["arch%d/%dx%d/logits.s4" % (arch, hw[0], hw[1])]
    assert H.rel_err(out[:, :, ::4, ::4], want) < 2e-3       # fp16 storage rounding of the oracle vs the fp32 reference
    assert (out.argmax(1).astype(np.uint8) == g["arch%d/%dx%d/argmax" % (arch, hw[0], hw[1])]).mean() > 0.98


def test_oracle_single_conv_factorized_reduce_matches_golden():
    g, meta = golden()
    fr = meta["factorized_reduce"]
    sd = orc.random_state_dict({k: tuple(v) for k, v in fr["shapes"].items()}, seed=fr["seed_weights"])
    x = orc.random_input((2, fr["C_in"]) + tuple(fr["hw"]), seed=fr["seed_input"])
    out = lvo.factorized_reduce(x, orc.Params(sd), 2).numpy()
    assert H.rel_err(out, g["factorized_reduce/out"]) < 2e-3


def test_nearest_wrappers_marshalling(fake):
    x = act(2, 32, 6, 10, wide=16)
    out = act(2, 32, 3, 5, wide=8)
    assert F_.nearest(x, (3, 5), out=out) is out
    a = fake.last("fsb_nearest_fwd")
    assert a[:6] == [2, 32, 6, 10, 3, 5] and a[6] == x.data_ptr() and a[7] == 48 and a[8] == out.data_ptr() and a[9] == 40
    y = F_.nearest(x, (12, 20))
    assert tuple(y.shape) == (2, 32, 12, 20) and fake.last("fsb_nearest_fwd")[9] == 32
    logits = act(1, 19, 4, 6)
    o = F_.upsample_logits_nearest(logits, (32, 48), dtype=torch.float16)
    a = fake.last("fsb_upsample_logits_nearest_nchw")
    assert tuple(o.shape) == (1, 19, 32, 48) and o.is_contiguous() and a[:6] == [1, 19, 4, 6, 32, 48] and a[7] == 24 and a[9] == 0
    o = F_.upsample_logits_nearest(logits, (32, 48))
    assert o.dtype == torch.float32 and fake.last("fsb_upsample_logits_nearest_nchw")[9] == 1
    lab = F_.upsample_argmax_nearest(logits, (32, 48))
    a = fake.last("fsb_upsample_argmax_nearest")
    assert lab.dtype == torch.uint8 and tuple(lab.shape) == (1, 32, 48) and a[:6] == [1, 19, 4, 6, 32, 48] and a[8] == lab.data_ptr()


def test_conv_fold_flags_marshalling(fake):
    wp = torch.empty(4096, dtype=torch.float16)
    x = act(2, 32, 12, 20, wide=16)
    y = F_.conv_fwd(x, wp, 24, 3, 1, 1, relu=True, down2=True)
    d = fake.last("fsb_conv_fwd")[0]
    assert tuple(y.shape) == (2, 24, 6, 10)
    assert (d["H"], d["W"], d["Ho"], d["Wo"], d["x_cstride"]) == (6, 10, 6, 10, 48)
    assert d["flags"] == _lib.FSB_CONV_RELU | _lib.FSB_CONV_X_DOWN2
    out = act(2, 24, 24, 40, wide=8)
    assert F_.conv_fwd(x, wp, 24, 1, 1, 0, up2=True, out=out) is out
    d = fake.last("fsb_conv_fwd")[0]
    assert (d["H"], d["W"], d["Ho"], d["Wo"], d["y_cstride"]) == (12, 20, 12, 20, 32) and d["flags"] == _lib.FSB_CONV_Y_UP2
    y = F_.conv_fwd(x, wp, 24, 3, 1, 1, down2=True, up2=True)
    d = fake.last("fsb_conv_fwd")[0]
    assert tuple(y.shape) == (2, 24, 12, 20) and d["flags"] == _lib.FSB_CONV_X_DOWN2 | _lib.FSB_CONV_Y_UP2
    with pytest.raises(ValueError):
        F_.conv_fwd(act(1, 32, 7, 10), wp, 24, 3, 1, 1, down2=True)
    assert _lib.FSB_CONV_X_DOWN2 == 64 and _lib.FSB_CONV_Y_UP2 == 128


def test_training_or_grad_forward_raises(fake):
    model = zoo.build_network(1, variant="latency")
    x = torch.zeros(1, 3, 64, 128)
    model.train()
    with pytest.raises(NotImplementedError, match="inference only"):
        model(x)
    model.eval()
    with pytest.raises(NotImplementedError, match="inference only"):
        model(x)                      # grad mode: parameters require grad
    x.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="inference only"):
        model(x)
    op = lat_ops.BasicResidual_downup_1x(32, 32, slimmable=False)
    with pytest.raises(NotImplementedError, match="inference only"):
        op(torch.zeros(1, 32, 8, 8))
    fr = lat_ops.FactorizedReduce(32, 48, 2, slimmable=False)
    with pytest.raises(NotImplementedError, match="inference only"):
        fr(torch.zeros(1, 32, 8, 8))
    assert fake.calls == []           # no kernel ran, bilinear or otherwise


def test_latency_table_variant_builds_the_same_keys_from_its_operators():
    from tools import build_latency_table as blt
    keys = blt.table_keys()
    for key in keys:
        mt, st = blt.build_module(key)
        ml, sl = blt.build_module(key, "latency")
        assert st == sl and type(mt).__name__ == type(ml).__name__
        if key.startswith("BasicResidual_downup") or (key.startswith("FactorizedReduce") and key.endswith("stride2")):
            assert type(ml).__module__ == "fasterseg_b200.latency_variant.operations", key
    fr = blt.build_module("FactorizedReduce_H64_W128_Cin32_Cout64_stride2", "latency")[0]
    assert "conv2.weight" not in fr.state_dict()
    assert "conv2.weight" in blt.build_module("FactorizedReduce_H64_W128_Cin32_Cout64_stride2")[0].state_dict()
