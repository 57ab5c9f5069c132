"""Supernet wiring with RANDOM architecture parameters (the goldens use the constant 1e-3 initialisation): MixedOp weights,
beta mixing of the two cell invocations, width selection in every mode incl. gumbel-sampled `arch_ratio`, for several
depths -- ours on the CPU stand-in backend against the UNMODIFIED reference (CPU fp32) on the same state_dict and RNG seeds
(tests/golden/random_structures.npz, oracle/make_golden_random_structures.py), two-sided gate against the reference run in
torch fp16 (random supernets are ill-conditioned, see tests/test_hostlogic_structures_cpu.py)."""
import numpy as np
import pytest
import torch

from oracle import make_golden_random_structures as RS
from tests import cpu_backend
from tests import helpers as H


@pytest.mark.parametrize("layers,arch_idx,mode,seed", RS.SUPERNET_CASES)
def test_eval_forward_matches_reference_with_random_arch_parameters(layers, arch_idx, mode, seed):
    from fasterseg_b200.model_search import Network_Multi_Path
    golden = np.load(H.GOLDEN + "/random_structures.npz")
    ours = RS.supernet(Network_Multi_Path, layers, seed)
    x = RS.input_(seed, 1)
    with cpu_backend.installed():
        got = RS.run_supernet(ours, x, arch_idx, mode, seed)
    assert len(got) == 5
    for i, g in enumerate(got):
        key = "supernet.%d.%d" % (seed, i)
        want = torch.from_numpy(golden[key + ".want"])
        err = float((RS.sample(g) - want).norm() / want.norm())
        err16 = float(golden[key + ".err16"])
        print("layers %d arch %d mode %s pred%d: ours %.3e | reference in fp16 %.3e" % (layers, arch_idx, mode, i, err, err16))
        assert err <= 1.5 * err16 + 3e-3, i
