"""Stores the unmodified reference matcher's anchors on every seeded case (tests/matcher_libs.py cases()) as
reference_matcher_outputs.json.gz: full arrays for the small cases, the count plus a SHA-256 for the large ones. Run once on a
GPU with oracle/_ref/libgwref_matcher.so built:

    python tests/golden/cudamapper/make_matcher_fixture.py [output path]

Before it runs the reference on a case it asks the CPU oracle, and it refuses a case where both indices have unique
representations but no anchor: the reference launches a zero-block grid there and aborts (DESIGN.md section 11.3).
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import matcher_libs as ml  # noqa: E402
from checker_lib import write_fixture  # noqa: E402


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else ml.FIXTURE
    out = {"cases": {}}
    for name, c in ml.cases().items():
        q, t, _, _ = ml.sketches(c)
        if len(q["unique_representations"]) and len(t["unique_representations"]) and ml.oracle_count(q, t) == 0:
            raise SystemExit("%s: non-empty indices without a shared representation abort the reference" % name)
        (qf, qn), (tf, tn) = c["q"], c["t"]
        anchors, _, _ = ml.ref_run(c["reads"], qf, qn, tf, tn, c["k"], c["w"], c["hash"], c["F"])
        out["cases"][name] = ml.to_json(anchors, c["small"])
        print(name, len(anchors), flush=True)
    write_fixture(path, out)


if __name__ == "__main__":
    main()
