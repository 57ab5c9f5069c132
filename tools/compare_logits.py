#!/usr/bin/env python
"""Compare two logits.npy files written by `bench.py --dump-outputs DIR` (e.g. one run per FSB_CONV_TC2 setting).
Prints the max-abs difference, the norm-wise relative difference ||a - b|| / ||b|| and the argmax agreement."""
import argparse

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a", help="logits.npy under test")
    ap.add_argument("b", help="logits.npy of the baseline")
    args = ap.parse_args()
    a = np.load(args.a).astype(np.float64)
    b = np.load(args.b).astype(np.float64)
    if a.shape != b.shape:
        raise SystemExit("shape mismatch: %s vs %s" % (a.shape, b.shape))
    d = a - b
    rel = np.linalg.norm(d) / max(np.linalg.norm(b), 1e-30)
    print("shape %s  max-abs %.3e  norm-wise rel %.3e  max|b| %.3e" % (a.shape, np.abs(d).max(), rel, np.abs(b).max()))
    if a.ndim == 4:
        agree = (a.argmax(1) == b.argmax(1)).mean()
        print("argmax agreement %.6f" % agree)


if __name__ == "__main__":
    main()
