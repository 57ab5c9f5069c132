"""TEST INFRASTRUCTURE ONLY -- reference outputs for the random-structure wiring tests (tests/test_hostlogic_structures_cpu.py,
tests/test_hostlogic_supernet_fuzz_cpu.py).

Weights are drawn on OUR network (init_weights_, seeded; the same call in the tests reproduces them) and loaded into the
UNMODIFIED reference, which runs in fp32 and, for the two-sided gate, in torch fp16.  Stored per output: the reference's fp32
values on a fixed pixel sample (sample(): at most 8 rows x 16 columns of the map), and the reference's own fp16 deviation and
argmax agreement on that sample.  Run where the reference checkout is available (oracle/ref_harness.py REFERENCE_ROOT):
    python -m oracle.make_golden_random_structures   ->  tests/golden/random_structures.npz"""
import copy
import os

import numpy as np
import torch
import torch.nn as nn

from oracle import make_golden_decode as mk
from oracle import make_golden_latency as mkl

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "random_structures.npz")
EVAL_CASES = [(1003, [0, 1, 2]), (1010, [2, 0]), (1017, [1]), (1024, [0]), (1031, [1, 0]), (1038, [2]), (1045, [2, 1])]
TRAIN_CASES = [(1003, [0, 1, 2]), (1010, [2, 0]), (1017, [1]), (1045, [2, 1]), (1052, [1, 2])]
SUPERNET_CASES = [(5, 0, "max", 1), (5, 1, None, 2), (6, 1, "min", 3), (8, 1, None, 4), (8, 0, "random", 5)]


def sample(t):
    """fixed pixel sample of an N x C x H x W output: every s-th row and column, s = max(1, H // 8)"""
    s = max(1, t.shape[-2] // 8)
    return t[..., ::s, ::s].float()


def init_weights_(model, seed, bn_stats):
    """variance-preserving conv init (torch's default shrinks the signal into fp16 subnormals over 40 layers) and non-trivial
    BatchNorm affine (and, with bn_stats, running statistics), like a trained net; module order, seeded"""
    torch.manual_seed(seed)
    with torch.no_grad():
        for mod in model.modules():
            if isinstance(mod, nn.Conv2d):
                nn.init.kaiming_normal_(mod.weight, mode="fan_in", nonlinearity="relu")
            if isinstance(mod, nn.BatchNorm2d) and mod.running_mean is not None:
                if bn_stats:
                    mod.running_mean.normal_(0, 0.1)
                    mod.running_var.uniform_(0.5, 1.5)
                mod.weight.normal_(1.0, 0.1)
                mod.bias.normal_(0, 0.1)


def input_(seed, n):
    return torch.randn(n, 3, 128, 256, generator=torch.Generator().manual_seed(seed + 7))


def student(Net, seed, lasts, train):
    case = mk.draw_case(seed)
    alphas, betas, ratios = mk.clone_params(case)
    torch.manual_seed(seed)   # parameters the constructor draws and init_weights_ leaves alone (conv biases ...)
    m = Net(alphas, betas, ratios, num_classes=19, layers=case["layers"], Fch=12, width_mult_list=mk.WML,
            stem_head_width=case["stem_head_width"], ignore_skip=case["ignore_skip"])
    m.train(train)
    m.build_structure(list(lasts))
    init_weights_(m, seed, bn_stats=not train)
    return m


def supernet(Net, layers, seed):
    torch.manual_seed(seed)   # parameters the constructor draws and init_weights_ leaves alone
    m = mkl.build(Net, layers).eval()
    mkl.randomise_arch(m, 900 + seed)
    init_weights_(m, seed, bn_stats=True)
    return m


def run_supernet(model, inp, arch_idx, mode, seed):
    model.arch_idx, model.prun_mode = arch_idx, mode
    np.random.seed(seed)          # 'random' widths
    torch.manual_seed(100 + seed)  # gumbel noise of 'arch_ratio'
    with torch.no_grad():
        return model(inp)


def _store(out, key, want, half):
    w, h = sample(want), sample(half)
    out[key + ".want"] = w.numpy().astype(np.float32)
    out[key + ".err16"] = np.float64((h - w).norm() / w.norm())
    out[key + ".agree16"] = np.float64((h.argmax(1) == w.argmax(1)).float().mean())


def main():
    from oracle import ref_harness
    from fasterseg_b200.model_search import Network_Multi_Path
    from fasterseg_b200.model_seg import Network_Multi_Path_Infer
    ref_student = ref_harness.load_reference("train", "model_seg").model_seg.Network_Multi_Path_Infer
    out = {}
    for seed, lasts in EVAL_CASES:
        ours = student(Network_Multi_Path_Infer, seed, lasts, train=False)
        ref = student(ref_student, seed, lasts, train=False)
        assert list(ours.state_dict()) == list(ref.state_dict())
        ref.load_state_dict(ours.state_dict())
        x = input_(seed, 1)
        with torch.no_grad():
            _store(out, "eval.%d" % seed, ref(x), copy.deepcopy(ref).half()(x.half()).float())
    for seed, lasts in TRAIN_CASES:
        ours = student(Network_Multi_Path_Infer, seed, lasts, train=True)
        ref = student(ref_student, seed, lasts, train=True)
        ref.load_state_dict(ours.state_dict())
        half = copy.deepcopy(ref).half()
        x = input_(seed, 2)
        with torch.no_grad():
            want, got16 = ref(x), half(x.half())
        for name, w, h in zip(("pred8", "pred16", "pred32"), want, got16):
            if w is None:
                out["train.%d.%s.none" % (seed, name)] = np.int64(1)
            else:
                _store(out, "train.%d.%s" % (seed, name), w, h)
    ref_super = ref_harness.load_reference("search", "slimmable_ops", "operations", "seg_oprs", "genotypes", "model_search").model_search.Network_Multi_Path
    for layers, arch_idx, mode, seed in SUPERNET_CASES:
        ours = supernet(Network_Multi_Path, layers, seed)
        ref = mkl.build(ref_super, layers).eval()
        assert [k for k, _ in ours.named_parameters()] == [k for k, _ in ref.named_parameters()]
        ref.load_state_dict(ours.state_dict())
        half = copy.deepcopy(ref).half()
        x = input_(seed, 1)
        want = run_supernet(ref, x, arch_idx, mode, seed)
        got16 = run_supernet(half, x.half(), arch_idx, mode, seed)
        for i, (w, h) in enumerate(zip(want, got16)):
            _store(out, "supernet.%d.%d" % (seed, i), w, h)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays, %d bytes)" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
