"""The checkers behind tests/test_gpu_extender_edges.py, pinned without a GPU: both extender oracles read the matrix as
sub[target * 8 + query] (a hand case only the right reading scores), the width cases reach exactly the widths they are built
for, the tie cases tie where they are meant to, and the parameter-limit cases equal the unpruned numpy DP."""
import numpy as np
import pytest

import extender_edges_libs as el
import extender_libs as xl
import gapped_extender_libs as gl

A, C = 0, 1


def test_hand_asymmetric_matrix_in_the_gapped_oracle():
    cs, as_ = np.full(10, C, np.int8), np.full(10, A, np.int8)
    anchor = np.array([(5, 5)], dtype=gl.ANCHOR_DTYPE)
    # query C against target A scores +5 per base: the whole diagonal
    rec, cig, _ = gl.oracle_run(cs, as_, el.HAND_MATRIX, 3, 1, 50, 0, anchor)
    assert gl.rows(rec) == [(50, 0, 1, 0, 10, 0, 10)] and cig == ["10M"]
    # query A against target C scores -7 per base: nothing beats the empty alignment at the anchor
    rec, cig, _ = gl.oracle_run(as_, cs, el.HAND_MATRIX, 3, 1, 50, 0, anchor)
    assert gl.rows(rec) == [(0, 0, 1, 5, 5, 5, 5)] and cig == [""]
    side = gl.oracle_side(cs, as_, el.HAND_MATRIX, 3, 1, 50, 5, 5, False)
    assert (side["best"], side["i"], side["d"], side["ops"]) == (25, 5, 10, "MMMMM")


def test_hand_asymmetric_matrix_in_the_ungapped_oracle():
    cs, as_ = np.full(10, C, np.int8), np.full(10, A, np.int8)
    got = xl.oracle_seed(cs, as_, el.HAND_MATRIX, 20, True, 1, 5, 5)
    assert (got["query"], got["target"], got["length"], got["score"], got["kept"]) == (0, 0, 9, 50, 1)
    got = xl.oracle_seed(as_, cs, el.HAND_MATRIX, 20, True, 1, 5, 5)
    assert (got["score"], got["kept"]) == (0, 0)


def test_width_cases_reach_their_widths():
    query, target, anchors, widths = el.width_case()
    seen = set()
    for a, (wl, wr) in zip(anchors, widths):
        for left, w in ((True, wl), (False, wr)):
            side = gl.oracle_side(query, target, *el.WIDTH_PARAMS, int(a["query"]), int(a["target"]), left, trace=False)
            assert side["width"] == w
            seen.add(w)
    assert set(el.WIDTH_EDGES) <= seen


def test_width_of_a_side_pruned_by_the_ydrop():
    # ACGT against itself, open 3, extend 2, y-drop 5: the diagonal cell and the two gap cells beside it (DESIGN.md 16.1), and
    # the range formed from them is three cells wide
    s = np.array([0, 1, 2, 3], dtype=np.int8)
    m10 = np.full(64, -10, dtype=np.int32)
    m10[::9] = 10
    assert gl.oracle_side(s, s, m10, 3, 2, 5, 0, 0, False)["width"] == 3
    # nothing pruned: min(m, n) + 1
    assert gl.oracle_side(s, s[:3], m10, 3, 2, 1 << 28, 0, 0, False)["width"] == 4


@pytest.mark.parametrize("p", el.TIE_PS)
def test_tie_cases_tie_across_the_boundary(p):
    query, target = el.tie_case(p)
    mat, o, e, y = el.TIE_PARAMS
    side = gl.oracle_side(query, target, mat, o, e, y, 0, 0, False)
    assert (side["best"], side["i"], side["d"]) == (10 * p + 8, p + 1, 2 * p + 3)
    # the tied cell one row further scores the same from the other gap
    assert gl.numpy_best_prefix(query[:p + 2], target[:p + 1], mat, o, e) == 10 * p + 8
    assert gl.numpy_best_prefix(query[:p + 1], target[:p + 2], mat, o, e) == 10 * p + 8


def test_limit_cases_equal_the_numpy_dp():
    for q, t, anchor, mat, o, e in el.limit_cases():
        rec, _, _ = gl.oracle_run(q, t, mat, o, e, 1 << 28, -(1 << 40), np.array([anchor], dtype=gl.ANCHOR_DTYPE))
        assert int(rec[0]["score"]) == el.numpy_score(q, t, anchor, mat, o, e)
