"""Stores the unmodified reference overlapper's outputs on every seeded case (tests/overlapper_libs.py cases() and matcher_cases())
and its post_process_overlaps on every list (post_lists(), with and without dropping the fused members) as
reference_overlapper_outputs.json.gz: full arrays for the small cases, the count plus a SHA-256 for the large ones. Run once on a
GPU with oracle/_ref/libgwref_overlapper.so built:

    python tests/golden/cudamapper/make_overlapper_fixture.py [output path]
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import overlapper_libs as ol  # noqa: E402
from checker_lib import write_fixture  # noqa: E402


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else ol.FIXTURE
    out = {"cases": {}, "post": {}}
    for name, c in {**ol.cases(), **ol.matcher_cases()}.items():
        out["cases"][name] = {p: ol.to_json(ol.ref_run(c["anchors"], params)[0], c["small"]) for p, params in c["params"].items()}
        print(name, len(c["anchors"]), {p: v["n"] for p, v in out["cases"][name].items()}, flush=True)
    for name, lst in ol.post_lists().items():
        src = ol.from_rows(lst)
        out["post"][name] = {"drop%d" % d: ol.rows(ol.ref_post_process(src, bool(d))) for d in (0, 1)}
    write_fixture(path, out)


if __name__ == "__main__":
    main()
