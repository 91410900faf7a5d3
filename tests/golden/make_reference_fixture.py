"""Generates tests/golden/reference_kernel_outputs.json.gz: outputs of the UNMODIFIED reference cudapoa kernels (oracle/_ref/libgwref.so,
rebuilt for sm_90a) on deterministic synthetic windows, for every band mode. Run on a GPU box:
    python tests/golden/make_reference_fixture.py
The CPU test tests/test_oracle_poa.py::test_oracle_matches_reference_kernel_fixture re-creates the inputs from the recorded generator
parameters and checks the CPU oracle against these outputs, which pins the oracle to the reference itself (not only to its KATs)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle_lib as ol  # noqa: E402
import ref_lib  # noqa: E402
from checker_lib import GOLDEN, write_fixture  # noqa: E402
from genomeworks_b200 import synth  # noqa: E402

GEN = dict(n_windows=12, backbone=600, reads=10, mut=12, ins=6, dele=6, seed0=4242)
CASES = [dict(band_mode=0, band_width=256, max_pred=0), dict(band_mode=1, band_width=128, max_pred=0), dict(band_mode=2, band_width=128, max_pred=0),
         dict(band_mode=3, band_width=128, max_pred=0), dict(band_mode=4, band_width=128, max_pred=60)]
win_nseq, seq_len, data = synth.poa_windows(GEN["n_windows"], GEN["backbone"], GEN["reads"], GEN["mut"], GEN["ins"], GEN["dele"], seed0=GEN["seed0"])
windows = synth.split_windows(win_nseq, seq_len, data)
out = dict(generator=GEN, max_sequence_size=1024, max_sequences_per_poa=16, scores=dict(gap=-8, mismatch=-6, match=8), cases=[])
for c in CASES:
    ref = ref_lib.ref_poa_run(win_nseq, seq_len, data, 1024, 16, c["band_width"], c["band_mode"], max_pred_dist=c["max_pred"])
    cfg = ol.batch_config(1024, 16, c["band_width"], c["band_mode"], max_pred_dist=c["max_pred"])
    orc = ol.poa_run(windows, cfg)  # IEEE division for the band gradient (the device uses div.approx)
    same = list(orc["status"]) == list(ref["status"]) and list(orc["consensus"]) == list(ref["consensus"]) and \
        all(list(a) == list(b) for a, b in zip(orc["coverage"], ref["coverage"]))
    out["cases"].append(dict(c, status=[int(x) for x in ref["status"]], consensus=list(ref["consensus"]),
                             coverage=[[int(v) for v in cv] for cv in ref["coverage"]], oracle_with_ieee_division_identical=bool(same)))
    print(c, "reference ok windows:", int((np.array(ref["status"]) == 0).sum()), "oracle(ieee) identical:", same)
path = os.path.join(GOLDEN, "reference_kernel_outputs.json.gz")
write_fixture(path, out)
print("wrote", path)
