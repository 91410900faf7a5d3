"""The gapped extender's CPU oracle (oracle/gapped_extender_oracle.cpp) on hand-computed cases, against an unpruned numpy DP,
and its CIGARs re-scored by a separate function."""
import numpy as np
import pytest

import gapped_extender_libs as gl
from extender_libs import SAMPLE_MATRIX as SAMPLE, SIMPLE_MATRIX
from genomeworks_b200.cudaextender import encode_sequence

M10 = SIMPLE_MATRIX  # +10 / -10 among A/C/G/T


def anchors(*pairs):
    a = np.zeros(len(pairs), dtype=gl.ANCHOR_DTYPE)
    for k, (q, t) in enumerate(pairs):
        a[k] = (q, t)
    return a


def run(q, t, pairs, o=5, e=2, y=100, threshold=0, matrix=M10, budget=1 << 62):
    q = encode_sequence(q) if isinstance(q, str) else np.asarray(q, np.int8)
    t = encode_sequence(t) if isinstance(t, str) else np.asarray(t, np.int8)
    return gl.oracle_run(q, t, matrix, o, e, y, threshold, anchors(*pairs), budget)


def one(q, t, pair, **kw):
    rec, cig, _ = run(q, t, [pair], **kw)
    assert len(rec) == 1
    r = rec[0]
    return int(r["score"]), (int(r["query_begin"]), int(r["query_end"]), int(r["target_begin"]), int(r["target_end"])), cig[0]


def test_exact_match_and_one_mismatch():
    assert one("ACGTACGT", "ACGTACGT", (4, 4)) == (80, (0, 8, 0, 8), "8M")
    assert one("ACGTACGTAC", "ACGTACGAAC", (4, 4)) == (80, (0, 10, 0, 10), "10M")


T20 = "ACGTACGTAC" + "TTGCATGCAA"


def test_one_insertion_run_and_one_deletion_run():
    q = T20[:10] + "GG" + T20[10:]
    assert one(q, T20, (0, 0)) == (200 - (5 + 2 * 2), (0, 22, 0, 20), "10M2I10M")
    assert one(T20, q, (0, 0)) == (200 - (5 + 2 * 2), (0, 20, 0, 22), "10M2D10M")


def test_gap_through_the_anchor_is_charged_two_opens():
    q = T20[:10] + "GGGG" + T20[10:]
    # left side: 2I then 10M; right side: 2I then 10M; one 4-base gap would score 200 - 13
    assert one(q, T20, (12, 10)) == (200 - 2 * (5 + 2 * 2), (0, 24, 0, 20), "10M4I10M")


def test_cell_at_exactly_b_minus_y_stays_live():
    # every odd anti-diagonal of an exact match holds only gap cells at B - (o + e)
    assert one("ACGTACGT", "ACGTACGT", (0, 0), o=3, e=2, y=5) == (80, (0, 8, 0, 8), "8M")
    assert one("ACGTACGT", "ACGTACGT", (0, 0), o=3, e=2, y=4) == (0, (0, 0, 0, 0), "")
    side = gl.oracle_side(encode_sequence("ACGT"), encode_sequence("ACGT"), M10, 3, 2, 5, 0, 0, False)
    # anti-diagonals 0 .. 8: the diagonal cell on even ones, the two gap cells beside it on odd ones
    assert (side["best"], side["i"], side["d"], side["live"]) == (40, 4, 8, 5 + 4 * 2)


def test_anchors_at_position_zero_and_at_the_last_base():
    s = "ACGTACGT"
    assert one(s, s, (0, 0)) == (80, (0, 8, 0, 8), "8M")
    assert one(s, s, (7, 7)) == (80, (0, 8, 0, 8), "8M")
    l = gl.oracle_side(encode_sequence(s), encode_sequence(s), M10, 5, 2, 100, 7, 7, True)
    r = gl.oracle_side(encode_sequence(s), encode_sequence(s), M10, 5, 2, 100, 7, 7, False)
    assert (l["best"], l["i"], r["best"], r["i"]) == (70, 7, 10, 1)


def test_codes_4_to_7_and_bytes_above_7_are_read_modulo_8():
    mat = np.full(64, -8, dtype=np.int32)
    mat[::9] = 8
    q = np.array([4, 5, 6, 7], dtype=np.int8)
    t = np.array([12, 13, 14, -1], dtype=np.int8)  # 12, 13, 14 and 0xff are 4, 5, 6, 7 modulo 8
    assert one(q, t, (0, 0), matrix=mat) == (32, (0, 4, 0, 4), "4M")


def test_ydrop_zero():
    assert one("ACGT", "ACGT", (0, 0), o=0, e=0, y=0) == (40, (0, 4, 0, 4), "4M")
    # with gaps of positive cost nothing survives the first anti-diagonal
    assert one("ACGT", "ACGT", (0, 0), o=0, e=1, y=0) == (0, (0, 0, 0, 0), "")


def test_best_cell_ties_go_to_the_smallest_antidiagonal_then_the_smallest_i():
    # M M X M: 20 at anti-diagonal 4 and again at 8
    side = gl.oracle_side(encode_sequence("ACAT"), encode_sequence("ACGT"), M10, 20, 5, 100, 0, 0, False)
    assert (side["best"], side["i"], side["d"]) == (20, 2, 4)
    # (2, 1) and (1, 2) both score 8 on anti-diagonal 3: i = 1 wins
    assert one("CA", "AC", (0, 0), o=1, e=1) == (8, (0, 1, 0, 2), "1D1M")


def test_traceback_prefers_the_diagonal_then_i_then_d():
    # at (2, 1) the diagonal and the I value tie at 8
    assert one("AAC", "AC", (0, 0), o=1, e=1) == (18, (0, 3, 0, 2), "1I2M")
    assert one("AC", "AAC", (0, 0), o=1, e=1) == (18, (0, 2, 0, 3), "1D2M")


def test_duplicate_intervals_keep_the_first_anchor():
    rec, cig, _ = run("ACGTACGT", "ACGTACGT", [(0, 0), (7, 7), (3, 3)])
    assert [int(a) for a in rec["anchor"]] == [0] and cig == ["8M"]


def test_threshold():
    assert len(run("ACGTACGT", "ACGTACGT", [(4, 4)], threshold=80)[0]) == 1
    assert len(run("ACGTACGT", "ACGTACGT", [(4, 4)], threshold=81)[0]) == 0


def test_budget_decides_has_cigar_per_alignment():
    q = T20[:10] + "GG" + T20[10:]
    l = gl.oracle_side(encode_sequence(q), encode_sequence(T20), M10, 5, 2, 100, 0, 0, True)
    r = gl.oracle_side(encode_sequence(q), encode_sequence(T20), M10, 5, 2, 100, 0, 0, False)
    need = l["storage"] + r["storage"]
    rec, cig, _ = run(q, T20, [(0, 0)], budget=need)
    assert int(rec[0]["has_cigar"]) == 1 and cig == ["10M2I10M"]
    rec2, cig2, _ = run(q, T20, [(0, 0)], budget=need - 1)
    assert int(rec2[0]["has_cigar"]) == 0 and cig2 == [""]
    assert gl.rows(rec2)[0][:2] == gl.rows(rec)[0][:2] and gl.rows(rec2)[0][3:] == gl.rows(rec)[0][3:]


@pytest.mark.parametrize("seed", range(3))
def test_side_scores_equal_an_unpruned_numpy_dp(seed):
    rng = np.random.default_rng(seed)
    for _ in range(100):
        m, n = int(rng.integers(0, 30)), int(rng.integers(0, 30))
        a = rng.integers(-16, 16, m).astype(np.int8)
        b = rng.integers(-16, 16, n).astype(np.int8)
        mat = rng.integers(-12, 13, 64).astype(np.int32)
        o, e = int(rng.integers(0, 6)), int(rng.integers(0, 4))
        q = np.concatenate([[0], a]).astype(np.int8)
        t = np.concatenate([[0], b]).astype(np.int8)
        side = gl.oracle_side(q, t, mat, o, e, 1 << 28, 1, 1, False, trace=False)
        assert side["best"] == gl.numpy_best_prefix(a, b, mat, o, e)
        # the left side reads backwards from the anchor
        q2 = np.concatenate([a[::-1], [0]]).astype(np.int8)
        t2 = np.concatenate([b[::-1], [0]]).astype(np.int8)
        side = gl.oracle_side(q2, t2, mat, o, e, 1 << 28, m, n, True, trace=False)
        assert side["best"] == gl.numpy_best_prefix(a, b, mat, o, e)


@pytest.mark.parametrize("divergence", [0.0, 0.1, 0.3])
def test_every_cigar_consumes_its_intervals_and_rescores_to_its_score(divergence):
    from genomeworks_b200 import synth
    target, query, seeds = synth.extender_workload(3000, divergence, 60, 0.3, seed=5)
    for o, e, y in ((400, 30, 9400), (5, 2, 60), (0, 1, 30)):
        mat = SIMPLE_MATRIX if o < 100 else SAMPLE
        rec, cig, _ = gl.oracle_run(query, target, mat, o, e, y, -(1 << 40), seeds)
        assert len(rec) > 0
        for r, c in zip(rec, cig):
            assert int(r["has_cigar"]) == 1
            a = seeds[int(r["anchor"])]
            score, dq, dt = gl.rescore(c, query, target, mat, o, e, int(r["query_begin"]), int(r["target_begin"]),
                                       (int(a["query"]), int(a["target"])))
            assert (score, dq, dt) == (int(r["score"]), int(r["query_end"] - r["query_begin"]), int(r["target_end"] - r["target_begin"]))


def test_score_past_2_31():
    mat = np.full(64, -(1 << 20), dtype=np.int32)
    mat[::9] = 1 << 20
    rng = np.random.default_rng(3)
    s = rng.integers(0, 4, 4096).astype(np.int8)
    rec, cig, _ = gl.oracle_run(s, s, mat, 400, 30, 9400, 1 << 31, anchors((2048, 2048)))
    assert int(rec[0]["score"]) == 4096 << 20 > (1 << 31) and cig == ["4096M"]

