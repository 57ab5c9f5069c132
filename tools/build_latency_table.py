#!/usr/bin/env python
"""Build `latency_lookup_table.npy` for THIS GPU with our kernels ("next" row N3 of SURVEY section 8f).

The search's latency regulariser (search/architect.py:60-74 -> forward_latency) and the latency of a decoded genotype
(train/model_seg.py:368-408) are sums of per-operator entries of a lookup table keyed by operator, input size and channel
counts; the reference ships a table measured with TensorRT on a 1080Ti.  This tool enumerates the same key space --
every searchable operator at every (scale, input width, output width, stride), the stems, arm / refine convs, feature
fusion and heads for Fch in {8, 12} at 1024x2048 -- builds each operator from `fasterseg_b200.operations / seg_oprs` and
times it on the current device (CUDA events, warm-up + fixed iterations; `--protocol reference` uses the reference's
doubling protocol of tools/utils/darts_utils.py:182-223 instead, ~7 s per entry).

  python tools/build_latency_table.py --out latency_lookup_table.npy            # one pass over the 667 operator shapes
  python tools/build_latency_table.py --list                                    # print the keys only (no GPU needed)
  python tools/build_latency_table.py --variant latency --out latency/latency_lookup_table.npy
                                    # the same keys measured on the latency/ deployment network's operators (nearest resizes,
                                    # single-conv stride-2 FactorizedReduce), from which the reference built its table

`table_keys()` is checked on the build machine against the key set of the reference's shipped table
(tests/test_latency_table_keys_cpu.py)."""
import argparse
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, W = 1024, 2048
WIDTHS = [4. / 12, 6. / 12, 8. / 12, 10. / 12, 1.]
CELL_OPS = ("BasicResidual1x", "BasicResidual_downup_1x", "BasicResidual2x", "BasicResidual_downup_2x", "FactorizedReduce")


def _cell_key(op, h, w, c_in, c_out, stride):
    if op == "FactorizedReduce":
        return "FactorizedReduce_H%d_W%d_Cin%d_Cout%d_stride%d" % (h, w, c_in, c_out, stride)
    return "%s_H%d_W%d_Cin%d_Cout%d_stride%d_dilation%d" % (op, h, w, c_in, c_out, stride, 1)


def _convnorm_key(h, w, c_in, c_out, k, stride):
    return "ConvNorm_H%d_W%d_Cin%d_Cout%d_kernel%d_stride%d" % (h, w, c_in, c_out, k, stride)


def table_keys(fch_cells=(12,), fch_decoder=(8, 12), fch_max=12):
    """Every key `forward_latency` can ask for at 1024x2048 (insertion order = build order)."""
    keys = []
    add = lambda k: keys.append(k) if k not in keys else None
    for fch in fch_cells:
        for scale in (8, 16, 32):
            h, w = H // scale, W // scale
            for w_in in WIDTHS:
                for w_out in WIDTHS:
                    c_in = int(fch * scale * w_in)
                    for op in CELL_OPS:
                        add(_cell_key(op, h, w, c_in, int(fch * scale * w_out), 1))
                        if scale < 32:   # the stride-2 variant doubles the channel count on the way down
                            add(_cell_key(op, h, w, c_in, int(fch * scale * 2 * w_out), 2))
    for fch in fch_decoder:
        # stem: ConvNorm 3 -> 4F (s2), then [ConvNorm | BasicResidual2x] 4F -> 8F (s2), BasicResidual2x 8F -> 8F... (s2)
        add(_convnorm_key(H, W, 3, 2 * fch * 2, 3, 2))
        add(_convnorm_key(H // 2, W // 2, 2 * fch * 2, 4 * fch * 2, 3, 2))
        add(_cell_key("BasicResidual2x", H // 2, W // 2, 2 * fch * 2, 4 * fch * 2, 2))
        add(_cell_key("BasicResidual2x", H // 4, W // 4, 4 * fch * 2, 8 * fch, 2))
    for fch in fch_decoder:
        # arms (1x1) and refines (3x3 over [upsampled arm | skip feature of any searched width])
        add(_convnorm_key(H // 32, W // 32, 32 * fch, 16 * fch, 1, 1))
        for w_skip in WIDTHS:
            add(_convnorm_key(H // 16, W // 16, 16 * fch + 16 * fch_max * w_skip, 16 * fch, 3, 1))
        add(_convnorm_key(H // 16, W // 16, 16 * fch, 8 * fch, 1, 1))
        for w_skip in WIDTHS:
            add(_convnorm_key(H // 8, W // 8, 8 * fch + 8 * fch_max * w_skip, 8 * fch, 3, 1))
        for branches in (1, 2, 3):
            add("ff_H%d_W%d_C%d" % (H // 8, W // 8, 8 * fch * branches))
    for fch in fch_decoder:
        for branches in (1, 2, 3):
            add("head_H%d_W%d_Cin%d_Cout%d" % (H // 8, W // 8, 8 * fch * branches, 19))
    return keys


_PATTERNS = (
    (re.compile(r"^(BasicResidual1x|BasicResidual_downup_1x|BasicResidual2x|BasicResidual_downup_2x)_H(\d+)_W(\d+)_Cin(\d+)_Cout(\d+)_stride(\d+)_dilation(\d+)$"), "cell"),
    (re.compile(r"^FactorizedReduce_H(\d+)_W(\d+)_Cin(\d+)_Cout(\d+)_stride(\d+)$"), "skip"),
    (re.compile(r"^ConvNorm_H(\d+)_W(\d+)_Cin(\d+)_Cout(\d+)_kernel(\d+)_stride(\d+)$"), "convnorm"),
    (re.compile(r"^ff_H(\d+)_W(\d+)_C(\d+)$"), "ff"),
    (re.compile(r"^head_H(\d+)_W(\d+)_Cin(\d+)_Cout(\d+)$"), "head"),
)


def operators(variant="train"):
    """the operator module a table is measured with: the train/ network's or the latency/ deployment network's"""
    if variant == "latency":
        from fasterseg_b200.latency_variant import operations as ops
    elif variant == "train":
        from fasterseg_b200 import operations as ops
    else:
        raise ValueError("variant must be 'train' or 'latency', got %r" % (variant,))
    return ops


def build_module(key, variant="train"):
    """-> (nn.Module in eval mode, input shape (1, C, H, W)) for a table key, built from `operators(variant)`"""
    ops = operators(variant)
    from fasterseg_b200.seg_oprs import FeatureFusion, Head
    for rx, kind in _PATTERNS:
        m = rx.match(key)
        if not m:
            continue
        if kind == "cell":
            cls = ops.OPS_Class[{v.__name__: k for k, v in ops.OPS_Class.items()}[m.group(1)]]
            h, w, ci, co, s = (int(m.group(i)) for i in (2, 3, 4, 5, 6))
            return cls(ci, co, kernel_size=3, stride=s, dilation=1, groups=1, slimmable=False), (1, ci, h, w)
        g = [int(v) for v in m.groups()]
        if kind == "skip":
            h, w, ci, co, s = g
            # like FactorizedReduce._latency (search/operations.py:503-507): the non-slimmable build, i.e. the identity for stride 1
            return ops.FactorizedReduce(ci, co, stride=s, slimmable=False), (1, ci, h, w)
        if kind == "convnorm":
            h, w, ci, co, k, s = g
            return ops.ConvNorm(ci, co, kernel_size=k, stride=s, padding=1 if k == 3 else None, slimmable=False), (1, ci, h, w)
        if kind == "ff":
            h, w, c = g
            return FeatureFusion(c, c), (1, c, h, w)
        h, w, ci, co = g
        return Head(ci, co), (1, ci, h, w)
    raise ValueError("unrecognised latency-table key: " + key)


def time_module(module, shape, protocol="fast", iters=30):
    import torch
    if protocol == "reference":
        from fasterseg_b200.latency import compute_latency_ms
        return compute_latency_ms(module, shape)
    module = module.cuda().eval()
    x = torch.randn(*shape, device="cuda")
    flush = torch.empty(160 << 20, dtype=torch.uint8, device="cuda")     # > 50 MB L2
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    with torch.no_grad():
        for _ in range(5):
            module(x)
        for _ in range(iters):
            flush.zero_()
            start.record()
            module(x)
            stop.record()
            stop.synchronize()
            total += start.elapsed_time(stop)
    return total / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="latency_lookup_table.npy")
    ap.add_argument("--list", action="store_true", help="print the keys and exit (no GPU)")
    ap.add_argument("--protocol", default="fast", choices=["fast", "reference"])
    ap.add_argument("--limit", type=int, default=0, help="only the first N keys (smoke test)")
    ap.add_argument("--variant", default="train", choices=["train", "latency"],
                    help="operators to measure: train/ (bilinear) or latency/ (nearest, single-conv stride-2 skip)")
    args = ap.parse_args()
    keys = table_keys()
    if args.limit:
        keys = keys[:args.limit]
    if args.list:
        print("\n".join(keys))
        print("# %d keys" % len(keys), file=sys.stderr)
        return
    table = {}
    for i, key in enumerate(keys):
        module, shape = build_module(key, args.variant)
        table[key] = float(time_module(module, shape, args.protocol))
        if i % 50 == 0:
            print("%4d/%d %-70s %.4f ms" % (i, len(keys), key, table[key]), flush=True)
    np.save(args.out, table)
    print("wrote %s (%d entries, sum %.1f ms)" % (args.out, len(table), sum(table.values())))


if __name__ == "__main__":
    main()
