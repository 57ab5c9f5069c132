#!/usr/bin/env python
"""TEST INFRASTRUCTURE ONLY -- value AND gradients of the supernet's expected-latency model (`Network_Multi_Path.forward_latency`
followed by `.backward()`, search/model_search.py:361-475 and search/architect.py:60-75) from the UNMODIFIED reference on the CPU,
over the synthetic lookup table and the cases / seeds of oracle/make_golden_latency.py: 6 supernets x 2 architectures x 8
alpha / beta / ratio switch combinations.  For every combination the npz holds
  <seed>/a<idx>.<abr>/value          float64 [1]  the latency
  <seed>/a<idx>.<abr>/none           uint8 [8]    1 where the arch tensor's .grad stays None (alphas x3, betas x2, ratios x3)
  <seed>/a<idx>.<abr>/<tensor name>  float32      the gradient of every tensor whose .grad is not None
Written byte for byte reproducibly to tests/golden/supernet_latency_grad.npz.
Run in the build container:  python oracle/make_golden_latency_grad.py"""
import io
import os
import sys
import zipfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import make_golden_latency as mk  # noqa: E402
from oracle import ref_harness  # noqa: E402
from oracle.make_golden_decode import SyntheticLatencyTable  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "supernet_latency_grad.npz")
KINDS = (("alphas", 3), ("betas", 2), ("ratios", 3))


def arch_tensors(model, arch_idx):
    names = [model._arch_names[arch_idx][kind][i] for kind, n in KINDS for i in range(n)]
    return names, [getattr(model, n) for n in names]


def evaluate_grad(model, case):
    """{"<seed>/a<idx>.<abr>/...": array} -- called with the reference model here and with ours in the tests"""
    out = {}
    H, W = case["hw"]
    for arch_idx in (0, 1):
        for flags in mk.FLAGS:
            model.arch_idx, model.prun_mode = arch_idx, None
            names, params = arch_tensors(model, arch_idx)
            for p in model.parameters():
                p.grad = None
            torch.manual_seed(case["seed"] * 7 + arch_idx)     # same seeds as make_golden_latency.evaluate
            np.random.seed(case["seed"] * 11 + arch_idx)
            lat = model.forward_latency((3, H, W), alpha=flags[0], beta=flags[1], ratio=flags[2])
            if isinstance(lat, torch.Tensor) and lat.requires_grad:
                lat.backward()
            key = "%d/a%d.%d%d%d/" % ((case["seed"], arch_idx) + tuple(int(f) for f in flags))
            out[key + "value"] = np.array([float(lat)], np.float64)
            out[key + "none"] = np.array([p.grad is None for p in params], np.uint8)
            for n, p in zip(names, params):
                if p.grad is not None:
                    out[key + n] = p.grad.detach().cpu().numpy().astype(np.float32)
    return out


def savez_fixed(path, arrays):
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            z.writestr(info, buf.getvalue())


def main():
    ns = ref_harness.load_reference("search", "slimmable_ops", "operations", "seg_oprs", "genotypes", "model_search")
    for mod in (ns.operations, ns.seg_oprs):
        assert isinstance(mod.latency_lookup_table, dict)
        mod.latency_lookup_table = SyntheticLatencyTable()
    if not torch.cuda.is_available():
        torch.Tensor.cuda = lambda self, *a, **k: self      # model_search.py:373-384 hard-codes .cuda(); generator process only
    rec = {}
    for case in mk.CASES:
        model = mk.build(ns.model_search.Network_Multi_Path, case["layers"])
        mk.randomise_arch(model, case["seed"])
        rec.update(evaluate_grad(model, case))
        print(case)
    savez_fixed(OUT, rec)
    print("wrote %s (%d arrays, %d bytes)" % (OUT, len(rec), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
