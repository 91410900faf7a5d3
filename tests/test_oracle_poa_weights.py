"""The POA's uint16_t edge weights at the polisher's depth limit, on the CPU oracle alone (DESIGN.md 15.5).

With qualities a piece's bases weigh 0 .. 93 and an edge adds w[r - 1] + w[r], at most 186 per piece; the draft window adds 2.
max_depth = 352 is the largest depth at which no edge can pass 65535. Here a draft, n Q93 copies of it and three Q93 copies with
one substitution: up to n = 352 the consensus is the majority, at 353 the majority's edges wrap to 124 and it flips to the
minority. The GPU test of the same window is tests/test_gpu_poa_weighted_windows.py; a change of the oracle's edge-weight type
fails here first."""
import numpy as np
import pytest

import oracle_lib as ol
import poa_window_libs as pw

MAX_DEPTH = 352  # DESIGN.md 15.5, the limit the polisher's argument checks enforce with qualities


def test_depth_limit_arithmetic():
    assert 2 + 186 * MAX_DEPTH == 65474 <= 0xFFFF
    assert 2 + 186 * (MAX_DEPTH + 1) == 65660 > 0xFFFF
    assert pw.edge_weight(MAX_DEPTH) == 65474
    assert pw.edge_weight(MAX_DEPTH + 1) == 124
    # the minority's three reads outweigh a wrapped majority edge, and no majority edge below the limit
    assert pw.edge_weight(MAX_DEPTH + 1) < 3 * 186 < pw.edge_weight(MAX_DEPTH)


@pytest.mark.parametrize("n", [351, 352, 353, 354])
def test_consensus_flips_past_the_limit(n):
    (seqs, weights), majority, minority = pw.flip_window(n)
    cfg = ol.batch_config(2 * len(seqs[0]), len(seqs), 256, 1)  # static band: no device division involved
    r = ol.poa_run([seqs], cfg, weights=[pw.explicit_weights(seqs, weights)])
    assert int(r["status"][0]) == 0
    assert r["consensus"][0] == (majority if n <= MAX_DEPTH else minority)


def test_flip_needs_the_weights():
    """Unit weights (no qualities) never wrap at these depths: the majority wins on both sides."""
    for n in (352, 353):
        (seqs, _), majority, _ = pw.flip_window(n)
        r = ol.poa_run([seqs], ol.batch_config(2 * len(seqs[0]), len(seqs), 256, 1))
        assert int(r["status"][0]) == 0 and r["consensus"][0] == majority


def test_admission_rules():
    """The restatement of the batch's admission that the GPU tests apply before the oracle."""
    cfg = type("Cfg", (), dict(max_sequence_size=10, max_sequences_per_poa=3))
    seqs = [b"ACGT", b"A" * 11, b"CCCC", b"GGGG", b"TTTT", b"ACGA"]
    weights = [None, None, np.zeros(4, np.int8), np.array([0, 0, 5, 0], np.int8), None, None]
    st, kept, kw = pw.admit(seqs, weights, cfg)
    assert st == [0, 2, 10, 0, 0, 3]
    assert kept == [b"ACGT", b"GGGG", b"TTTT"]
    assert [list(w) for w in kw] == [[1] * 4, [0, 0, 5, 0], [1] * 4]
    st, kept, _ = pw.admit([b"A" * 11, b"CC"], [None, np.zeros(2, np.int8)], cfg)
    assert st == [2, 10] and kept == []
