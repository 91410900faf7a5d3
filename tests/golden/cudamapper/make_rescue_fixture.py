"""Stores the unmodified reference rescue's outputs (Overlapper::rescue_overlap_ends, or extend_overlap_by_sequence_similarity on
each overlap for the extend-once cases) on every seeded case of tests/rescue_libs.py cases() under each of its parameter sets as
reference_rescue_outputs.json.gz: full arrays for the small cases, the count plus a SHA-256 for the large ones. The rescue is host
code, so no GPU is needed; oracle/_ref/libgwref_rescue.so must be built:

    python tests/golden/cudamapper/make_rescue_fixture.py [output path]
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import rescue_libs as rl  # noqa: E402
from checker_lib import write_fixture  # noqa: E402


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else rl.FIXTURE
    out = {"cases": {}}
    for name, c in rl.cases().items():
        out["cases"][name] = {p: rl.to_json(rl.ref_run(c["overlaps"], c["query_reads"], c["target_reads"], e, thr, c["mode"])[0], c["small"])
                              for p, (e, thr) in c["params"].items()}
        print(name, len(c["overlaps"]), flush=True)
    write_fixture(path, out)


if __name__ == "__main__":
    main()
