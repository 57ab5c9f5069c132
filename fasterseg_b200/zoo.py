"""The two shipped FasterSeg genotypes (teacher arch_0, student arch_1) as data + builders.

`data/fasterseg_arch.json` holds the alpha/beta/ratio tensors and mIoU/latency scalars of the reference's
`train/fasterseg/arch_{0,1}.pt` (converted by oracle/make_golden.py; SURVEY section 2 row 15), so the benchmark
configuration "FasterSeg student (arch_1, F12.L16)" can be built where the reference tree is not mounted.
"""
import json
import math
import os

import torch

_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "fasterseg_arch.json")
WIDTH_MULT_LIST = [4. / 12, 6. / 12, 8. / 12, 10. / 12, 1.]   # train/config_train.py:82
STEM_HEAD_WIDTH = [(1, 1), (8. / 12, 8. / 12)]                 # train/config_train.py:96  [teacher, student]


def load_arch(arch_idx):
    """Equivalent of torch.load('fasterseg/arch_%d.pt') (train/train.py:93)."""
    with open(_DATA) as f:
        entry = json.load(f)["arch_%d" % arch_idx]["arch"]
    return {k: (torch.tensor(v, dtype=torch.float32) if isinstance(v, list) else v) for k, v in entry.items()}


def objective_acc_lat(acc, lat, lat_target=8.3, alpha=-0.07, beta=-0.07):
    """tools/utils/darts_utils.py:343-348."""
    return acc * math.pow(lat / lat_target, alpha if lat <= lat_target else beta)


def build_network(arch_idx=1, lasts=None, training=False, num_classes=19, layers=16, Fch=12, variant="train"):
    """Network_Multi_Path_Infer for a shipped genotype, constructed as train/train.py:95-105 does.
    variant: "train" (the train/ network: bilinear resizes) or "latency" (the latency/ deployment network: nearest resizes,
    single-conv stride-2 FactorizedReduce; inference only -- latency_variant/)."""
    if variant == "train":
        from .model_seg import Network_Multi_Path_Infer
    elif variant == "latency":
        from .latency_variant.model_seg import Network_Multi_Path_Infer
    else:
        raise ValueError("variant must be 'train' or 'latency', got %r" % (variant,))
    state = load_arch(arch_idx)
    model = Network_Multi_Path_Infer(
        [state["alpha_%d_0" % arch_idx], state["alpha_%d_1" % arch_idx], state["alpha_%d_2" % arch_idx]],
        [None, state["beta_%d_1" % arch_idx], state["beta_%d_2" % arch_idx]],
        [state["ratio_%d_0" % arch_idx], state["ratio_%d_1" % arch_idx], state["ratio_%d_2" % arch_idx]],
        num_classes=num_classes, layers=layers, Fch=Fch, width_mult_list=WIDTH_MULT_LIST,
        stem_head_width=STEM_HEAD_WIDTH[arch_idx], ignore_skip=(arch_idx == 0))
    if lasts is None:
        obj02 = objective_acc_lat(state["mIoU02"], state["latency02"])
        obj12 = objective_acc_lat(state["mIoU12"], state["latency12"])
        lasts = [2, 0] if obj02 > obj12 else [2, 1]
    model.train(training)
    model.build_structure(lasts)
    return model
