"""Stores the unmodified reference cudamapper tool's PAF output on every input of tests/mapper_libs.py write_inputs() under each
option set of mapper_libs.OPTIONS as reference_mapper_outputs.json.gz: the sorted lines, or their count and SHA-256 for large
outputs. Needs an H100 and oracle/_ref/cudamapper (built by build() where the reference sources exist):

    python tests/golden/cudamapper/make_mapper_fixture.py [output path]

"-a 2" is added to the sets of mapper_libs.ALIGN_BASES on the inputs of one tile where the output with -D equals the one without
(nothing fuses, so the reference's CIGARs, computed before fusion, sit on the right lines) and with at least two overlaps (with
fewer overlaps than engines the reference's alignment batch size is 0 and it never returns). Every run has a timeout.
"""
import os
import sys
import tempfile

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))
import mapper_libs as mp  # noqa: E402
from checker_lib import write_fixture  # noqa: E402


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else mp.FIXTURE
    out = {"cases": {}}
    with tempfile.TemporaryDirectory() as d:
        for name, (q, t) in mp.write_inputs(d).items():
            res, texts = {}, {}
            for opt, args in mp.OPTIONS.items():
                rc, text, err = mp.run(mp.REF_TOOL, args, q, t)
                assert rc == 0, (name, opt, rc, err[-2000:])
                texts[opt] = text
                res[opt] = mp.to_json(text)
                print(name, opt, len(mp.sorted_lines(text)), flush=True)
            single_tile = os.path.getsize(q) + (0 if q == t else os.path.getsize(t)) < 25000000
            for base in mp.ALIGN_BASES:
                if not single_tile or len(mp.sorted_lines(texts[base])) < 2:
                    continue
                rc, dropped, err = mp.run(mp.REF_TOOL, mp.OPTIONS[base] + ["-D"], q, t)
                assert rc == 0, (name, base, rc, err[-2000:])
                if mp.sorted_lines(dropped) != mp.sorted_lines(texts[base]):
                    continue
                rc, text, err = mp.run(mp.REF_TOOL, mp.options(base + "_a2"), q, t)
                assert rc == 0, (name, base, rc, err[-2000:])
                res[base + "_a2"] = mp.to_json(text)
                print(name, base + "_a2", len(mp.sorted_lines(text)), flush=True)
            out["cases"][name] = res
    write_fixture(path, out)


if __name__ == "__main__":
    main()
