#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- goldens of the drivers' per-step training mIoU from the UNMODIFIED reference (train/seg_metrics.py:5-24
`Seg_Metrics`, :43-69 `batch_intersection_union`), for fasterseg_b200/train_metrics.py.  Inputs are regenerated from the seeds
(numpy MT19937): label maps drawn per case, the logits their one-hot encoding (so the argmax is unique), so the file only holds
the reference's outputs.  Written to tests/golden/seg_metrics.json.
Run in the build container:  python oracle/make_golden_seg_metrics.py"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_harness  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "seg_metrics.json")

# name -> (seed, n_classes, shape of one update, number of updates, fraction of 255, extra target values outside [0, n_classes),
#          classes absent from both prediction and target)
CASES = {
    "cityscapes_19": (1, 19, (2, 24, 40), 3, 0.10, (), ()),
    "out_of_range_labels": (2, 19, (2, 16, 32), 2, 0.05, (19, 20, 254, 256, -1, -5), ()),
    "absent_classes": (3, 19, (1, 32, 48), 2, 0.05, (), (0, 5, 18)),          # union 0: get_scores skips them
    "camvid_11": (4, 11, (3, 20, 24), 3, 0.10, (11, 12, 18, -1), (7,)),
    "all_ignored_update": (5, 11, (1, 8, 8), 2, 1.0, (), ()),                 # nothing valid in any update
}


def inputs(name):
    """[(logits float32 N x C x H x W, target int64 N x H x W)] for each update of the case"""
    seed, n, shape, updates, p_ign, extra, absent = CASES[name]
    rs = np.random.RandomState(seed)
    present = np.array([c for c in range(n) if c not in absent])
    out = []
    for _ in range(updates):
        target = present[rs.randint(0, len(present), size=shape)].astype(np.int64)
        pred = target.copy()
        flip = rs.uniform(size=shape) < 0.4
        pred[flip] = present[rs.randint(0, len(present), size=int(flip.sum()))]
        if extra:
            odd = rs.uniform(size=shape) < 0.15
            target[odd] = np.array(extra)[rs.randint(0, len(extra), size=int(odd.sum()))]
        target[rs.uniform(size=shape) < p_ign] = 255
        logits = np.eye(n, dtype=np.float32)[pred].transpose(0, 3, 1, 2).copy()
        out.append((logits, target))
    return out


def main():
    import torch
    ns = ref_harness.load_reference("train", "seg_metrics")
    out = {}
    for name, case in CASES.items():
        n = case[1]
        m = ns.seg_metrics.Seg_Metrics(n_classes=n)
        steps = []
        for logits, target in inputs(name):
            inter, union = ns.seg_metrics.batch_intersection_union(torch.from_numpy(logits), torch.from_numpy(target), n)
            m.update(torch.from_numpy(logits), torch.from_numpy(target))
            steps.append({"inter": np.asarray(inter).astype(np.int64).tolist(), "union": np.asarray(union).astype(np.int64).tolist(),
                          "total_inter": m.total_inter.tolist(), "total_union": m.total_union.tolist(),
                          "score": float(m.get_scores()) if (m.total_union > 0).any() else None})
        out[name] = steps
    with open(OUT, "w") as f:
        json.dump(out, f)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
