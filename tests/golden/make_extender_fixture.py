"""Writes tests/golden/cudaextender/reference_extender_outputs.json.gz: the outputs of the UNMODIFIED reference extender
(oracle/_ref/libgwref_extender.so, built by build() from the reference sources) on the seeded synthetic cases of
tests/extender_libs.synthetic_cases(). Needs a CUDA device. Run from the repository root:

    python tests/golden/make_extender_fixture.py [output path]
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import extender_libs as xl  # noqa: E402
from checker_lib import write_fixture  # noqa: E402


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else xl.REF_OUTPUTS
    # the library reproduces the reference's own golden file before anything is recorded from it
    seq, seeds, golden = xl.sample()
    got, _ = xl.ref_run(seq, seq, xl.SAMPLE_MATRIX, xl.SAMPLE_XDROP, False, xl.SAMPLE_THRESHOLD, seeds)
    assert np.array_equal(got, golden), "reference library does not reproduce sample_scored_segment_pairs.csv"
    table = {}
    for c in xl.synthetic_cases():
        res, _ = xl.ref_run(c["query"], c["target"], c["matrix"], c["xdrop"], c["no_entropy"], c["threshold"], c["seeds"])
        table[c["name"]] = xl.ssp_rows(res)
        print(c["name"], len(c["seeds"]), "seeds ->", len(res), "segments")
    write_fixture(out_path, table)
    print("wrote", out_path)


if __name__ == "__main__":
    main()
