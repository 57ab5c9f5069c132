"""fsb_train_pre (csrc/trainpre.cu) on the GPU: bit-identical to the reference's TrainPre on every golden case, including the drivers'
two full-size geometries; one launch over a batch that mixes source sizes, scales, mirrors, crop positions and padding; and the
reference's recorded batches end to end through the launcher's wrap: with the reference's own get_train_loader where a copy of it
is available, and with a PNG dataset of the same item protocol everywhere."""
import random

import numpy as np
import pytest
import torch

from fasterseg_b200 import functional as F_
from oracle import make_golden_trainpre as G
from tests import trainpre_standin
from tests.test_trainpre_cpu import (FULL, GOLDEN, SMALL, bits_equal, case, check_e2e, device_inputs, e2e_batches,
                                     e2e_batches_standalone)

pytestmark = pytest.mark.gpu


def _run(pairs, cfg, draws):
    src, gt, geom, lut, crop, lab = device_inputs(pairs, cfg, draws)
    data, label = F_.train_pre(src.cuda(), gt.cuda(), geom.cuda(), lut.cuda(), crop, lab)
    torch.cuda.synchronize()
    return data.cpu(), label.cpu()


@pytest.mark.parametrize("name", SMALL)
def test_kernel_is_bit_identical_to_the_reference(name):
    pair, cfg, _, draws = case(name)
    data, label = _run([pair], cfg, [draws])
    assert bits_equal(data[0].numpy(), GOLDEN[name + "/data"])
    assert bits_equal(label[0].numpy(), GOLDEN[name + "/label"])


@pytest.mark.parametrize("name", FULL)
def test_kernel_full_size_digests(name):
    pair, cfg, _, draws = case(name)
    data, label = _run([pair], cfg, [draws])
    assert bits_equal(data[0].numpy().reshape(-1)[::G.STRIDE], GOLDEN[name + "/data_sample"])
    assert bits_equal(label[0].numpy().reshape(-1)[::G.STRIDE], GOLDEN[name + "/label_sample"])
    assert G.digest(data[0].numpy()) == str(GOLDEN[name + "/data_sha256"])
    assert G.digest(label[0].numpy()) == str(GOLDEN[name + "/label_sha256"])


@pytest.mark.parametrize("g", [1, 8])
def test_one_launch_over_mixed_geometries(g):
    """sources of different sizes, every scale, both mirrors, crops at 0, at the +1 edge and smaller than the crop (padding)"""
    cfg = G.config((40, 64), [0.75, 1, 1.25], g)
    sizes = [(37, 53), (64, 96), (33, 17), (48, 80), (41, 160), (96, 64), (1024, 2048)]
    rs = random.Random(11)
    pairs, draws = [], []
    for k, (H, W) in enumerate(sizes * 3):
        pairs.append(G.synthetic_pair(H, W, k))
        s = (0.75, 1, 1.25)[k % 3]
        sh, sw = int(H * s), int(W * s)
        ph = rs.choice([0, max(sh - 40 + 1, 0)]) if sh > 40 else 0
        pw = rs.randint(0, sw - 64 + 1) if sw > 64 else 0
        draws.append((k % 2, sh, sw, min(ph, sh - 1), pw))
    data, label = _run(pairs, cfg, draws)
    want_d, want_l = trainpre_standin.train_pre(*device_inputs(pairs, cfg, draws))
    assert bits_equal(data.numpy(), want_d.numpy()) and bits_equal(label.numpy(), want_l.numpy())


@pytest.mark.parametrize("source", ["reference", "standalone"])
def test_end_to_end_loader_on_the_device(tmp_path, source):
    """pinned worker batches, non_blocking copies and the kernel, against the reference's recorded batches: through the reference's
    own get_train_loader where a copy of it is available, and through tests/trainpre_dataset.py everywhere"""
    batches = (e2e_batches if source == "reference" else e2e_batches_standalone)(tmp_path)
    for b in batches:
        assert b["data"].is_cuda and b["label"].is_cuda and b["data"].device.index == torch.cuda.current_device()
    check_e2e(batches)
