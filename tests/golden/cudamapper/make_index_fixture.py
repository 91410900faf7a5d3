"""Stores the unmodified reference index's outputs on every seeded case (tests/index_libs.py cases()) as
reference_index_outputs.json.gz: full arrays for the small cases, counts plus SHA-256 of each array for the large ones, and
IndexDescriptor hashes. Run once on a GPU with oracle/_ref/libgwref_index.so built:

    python tests/golden/cudamapper/make_index_fixture.py [output path]
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import index_libs as il  # noqa: E402
from checker_lib import write_fixture  # noqa: E402

DESCRIPTORS = [(0, 0), (0, 1), (5, 10), (0xFFFFFFFF, 1), (123456, 0xFFFFFFFF), (7, 3000)]


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else il.FIXTURE
    out = {"cases": {}, "descriptor_hashes": []}
    for name, c in il.cases().items():
        res, _, _ = il.ref_run(c["reads"], c["first"], c["n"], c["k"], c["w"], c["hash"], c["F"])
        out["cases"][name] = il.to_json(res, c["small"])
        print(name, out["cases"][name]["sizes"], flush=True)
    for first, n in DESCRIPTORS:
        out["descriptor_hashes"].append([first, n, int(il.ref().ref_index_descriptor_hash(first, n))])
    write_fixture(path, out)


if __name__ == "__main__":
    main()
