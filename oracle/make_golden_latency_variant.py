"""TEST INFRASTRUCTURE ONLY -- golden outputs of the UNMODIFIED reference latency/ network (latency/operations.py,
latency/model_seg.py: nearest resizes, single-conv stride-2 FactorizedReduce), for tests/test_latency_variant_{cpu,gpu}.py.

Weights: fasterseg_oracle.random_state_dict over the reference model's own state_dict shapes, seeded per case (as make_golden.py
does).  Stored per case: the state_dict shapes, the fp32 logits at every 4th pixel and the full argmax map; for arch_1 at
1x3x1024x2048 a strided digest like baseline_sizes.npz.  96x160 makes the 1/32 map 3x5, whose /2 and x2 (3x5 -> 1x2 -> 3x5)
take the non-lattice index rule.  The single-conv stride-2 FactorizedReduce is pinned as an operator (shapes and output).  Entries are written with a fixed zip timestamp, so a rerun reproduces the file byte for
byte.  Run where the reference checkout is available (oracle/ref_harness.py REFERENCE_ROOT):
    python -m oracle.make_golden_latency_variant   ->  tests/golden/latency_variant.npz"""
import io
import json
import os
import zipfile

import numpy as np
import torch

from oracle import fasterseg_oracle as orc
from oracle import ref_harness as rh

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "latency_variant.npz")
SIZES = [(64, 128), (96, 160)]
FR_CASE = {"C_in": 32, "C_out": 48, "hw": [16, 24], "seed_weights": 7104, "seed_input": 7105}


def weight_seed(tag):
    return {"arch0": 7100, "arch1": 7101, "full": 7102}.get(tag, 7103)


def input_seed(h, w):
    return 40 + h + w


def shapes_of(model):
    return {k: tuple(v.shape) for k, v in model.state_dict().items() if not k.endswith("num_batches_tracked")}


def load(model, shapes, seed):
    """seeded weights; a cell shared by several branches has one key per branch -- the first key in sorted order wins (the
    oracle reads the cell under its lead branch's key, the smallest one)"""
    sd = orc.random_state_dict(shapes, seed=seed)
    own = model.state_dict()
    seen = set()
    with torch.no_grad():
        for k in sorted(sd):
            if own[k].data_ptr() not in seen:
                seen.add(own[k].data_ptr())
                own[k].copy_(sd[k])
    return sd


def run(model, x):
    with torch.no_grad():
        return model(x).float().numpy()


def savez_fixed(path, arrays):
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            z.writestr(info, buf.getvalue())


def main():
    torch.manual_seed(0)
    ns = rh.load_reference("latency", "operations", "seg_oprs", "model_seg")
    rec, meta = {}, {}
    for arch in (0, 1):
        model, _, lasts = rh.build_reference_student(ns, arch, train_mode=False)
        model.eval()
        shapes = shapes_of(model)
        load(model, shapes, weight_seed("arch%d" % arch))
        meta["arch%d" % arch] = {"lasts": list(lasts), "seed_weights": weight_seed("arch%d" % arch), "shapes": shapes}
        for h, w in SIZES:
            x = orc.random_input((1, 3, h, w), seed=input_seed(h, w))
            out = run(model, x)
            rec["arch%d/%dx%d/logits.s4" % (arch, h, w)] = np.ascontiguousarray(out[:, :, ::4, ::4])
            rec["arch%d/%dx%d/argmax" % (arch, h, w)] = out.argmax(1).astype(np.uint8)
    # The single-conv stride-2 FactorizedReduce, pinned as an operator: the decoder never keeps a skip as a cell's operator (a
    # skip is either dropped or replaced by the runner-up, decode.py select_ops), so no decoded structure contains one.
    fr = ns.operations.FactorizedReduce(FR_CASE["C_in"], FR_CASE["C_out"], 2, slimmable=False).eval()
    shapes = shapes_of(fr)
    load(fr, shapes, FR_CASE["seed_weights"])
    meta["factorized_reduce"] = dict(FR_CASE, shapes=shapes)
    x = orc.random_input((2, FR_CASE["C_in"]) + tuple(FR_CASE["hw"]), seed=FR_CASE["seed_input"])
    rec["factorized_reduce/out"] = run(fr, x)
    model, _, lasts = rh.build_reference_student(ns, 1, train_mode=False)
    model.eval()
    load(model, shapes_of(model), weight_seed("full"))
    out = run(model, orc.random_input((1, 3, 1024, 2048), seed=4242))
    lab = out.argmax(1).astype(np.uint8)
    srt = np.sort(out, axis=1)
    rec["full/logits.s32"] = np.ascontiguousarray(out[:, :, 3::32, 7::32])
    rec["full/argmax.s4"] = np.ascontiguousarray(lab[:, 1::4, 2::4])
    rec["full/margin.s4"] = np.ascontiguousarray((srt[:, -1] - srt[:, -2])[:, 1::4, 2::4]).astype(np.float32)
    rec["full/abs_max"] = np.float64(np.abs(out).max())
    meta["full"] = {"lasts": list(lasts), "seed_weights": weight_seed("full"), "seed_input": 4242, "hw": [1024, 2048]}
    rec["meta"] = np.frombuffer(json.dumps(meta, sort_keys=True).encode(), dtype=np.uint8)
    savez_fixed(OUT, rec)
    print("wrote %s (%d arrays, %d bytes)" % (OUT, len(rec), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
