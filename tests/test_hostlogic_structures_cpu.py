"""Wiring of the derived network for structures the shipped genotypes do not exercise -- three branches, a branch that ends
at 1/8 (its feature is copied straight into the fusion buffer), single-branch networks, eval and train builds -- on random
architectures: ours (CPU stand-in backend) against the UNMODIFIED reference network run in fp32 on the same state_dict and
input (tests/golden/random_structures.npz, oracle/make_golden_random_structures.py).  Random genotypes with random weights
are badly conditioned (zoomed operators on 4x8 feature maps: the reference's own logits move by up to 30 % when it is merely
run in torch fp16), so the gate is two-sided: our deviation from the fp32 reference must not exceed 1.5 x the deviation of
the reference run in fp16 -- a mis-wired branch or concat offset produces O(1) errors and is far outside that band for the
well-conditioned cases."""
import numpy as np
import pytest
import torch

from oracle import make_golden_random_structures as RS
from tests import cpu_backend
from tests import helpers as H


@pytest.fixture(scope="module")
def golden():
    return np.load(H.GOLDEN + "/random_structures.npz")


@pytest.mark.parametrize("seed,lasts", RS.EVAL_CASES)
def test_eval_logits_match_the_reference_on_random_structures(golden, seed, lasts):
    from fasterseg_b200.model_seg import Network_Multi_Path_Infer
    ours = RS.student(Network_Multi_Path_Infer, seed, lasts, train=False)
    x = RS.input_(seed, 1)
    with torch.no_grad():
        with cpu_backend.installed():
            got = ours(x)
            labels = ours.predict_labels(x)
    key = "eval.%d" % seed
    want = torch.from_numpy(golden[key + ".want"])
    assert got.shape == (1, 19, 128, 256)
    err = float((RS.sample(got) - want).norm() / want.norm())
    err16 = float(golden[key + ".err16"])
    print("seed %d lasts %s: norm-wise rel err ours %.3e | reference in fp16 %.3e" % (seed, lasts, err, err16))
    assert err <= 1.5 * err16 + 2e-3
    agree = float((RS.sample(labels.unsqueeze(1).float()).squeeze(1).long() == want.argmax(1)).float().mean())
    assert agree >= float(golden[key + ".agree16"]) - 0.02


@pytest.mark.parametrize("seed,lasts", RS.TRAIN_CASES)
def test_train_mode_auxiliary_heads_match_the_reference_on_random_structures(golden, seed, lasts):
    """Train-mode build (auxiliary 1/16 and 1/32 heads, model_seg.py:217-226,298-335) for `lasts` combinations the shipped
    genotypes do not cover: which features feed heads16 / heads32, in which order, and which predictions are None."""
    from fasterseg_b200.model_seg import Network_Multi_Path_Infer
    ours = RS.student(Network_Multi_Path_Infer, seed, lasts, train=True)
    x = RS.input_(seed, 2)
    with torch.no_grad():
        with cpu_backend.installed():
            got = ours(x)
    assert len(got) == 3
    for name, g in zip(("pred8", "pred16", "pred32"), got):
        key = "train.%d.%s" % (seed, name)
        assert (g is None) == (key + ".none" in golden.files), name
        if g is None:
            continue
        want = torch.from_numpy(golden[key + ".want"])
        gs = RS.sample(g)
        assert gs.shape == want.shape
        err = float((gs - want).norm() / want.norm())
        err16 = float(golden[key + ".err16"])
        print("seed %d lasts %s %s: ours %.3e | reference in fp16 %.3e" % (seed, lasts, name, err, err16))
        assert err <= 1.5 * err16 + 5e-3, name
