"""TEST INFRASTRUCTURE ONLY -- store the facts about the reference tree that tests check against as data:
  * line counts of every reference Python file (tools/check_citations.py resolves our `dir/file.py:LINE` citations with them),
  * the reference's shipped latency lookup table (train/latency_lookup_table.npy: operator key -> ms).
Run where the reference checkout is available (oracle/ref_harness.py REFERENCE_ROOT):
    python -m oracle.make_golden_reference_tree   ->  tests/golden/reference_tree.json"""
import json
import os

import numpy as np

from oracle import ref_harness

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_tree.json")


def main():
    root = ref_harness.REFERENCE_ROOT
    assert ref_harness.reference_available(), "reference tree not available at %s" % root
    counts = {}
    for d, _, names in os.walk(root):
        for n in names:
            if n.endswith(".py"):
                full = os.path.join(d, n)
                counts[os.path.relpath(full, root)] = sum(1 for _ in open(full, errors="replace"))
    table = np.load(os.path.join(root, "train", "latency_lookup_table.npy"), allow_pickle=True).item()
    with open(OUT, "w") as f:
        json.dump({"py_line_counts": dict(sorted(counts.items())),
                   "latency_lookup_table": {k: float(v) for k, v in sorted(table.items())}}, f, indent=0, sort_keys=True)
    print("wrote %s: %d files, %d latency entries" % (OUT, len(counts), len(table)))


if __name__ == "__main__":
    main()
