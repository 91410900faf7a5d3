"""The CPU oracle of the ungapped extender where its scores pass 2^31 (DESIGN.md 9.1): int64 sums, the X-drop test and the
entropy gate in int64, the score saturated at INT32_MAX. Each seed is compared with a plain numpy restatement
(tests/wide_score_libs.py); each call with that restatement's sort and unique rule."""
import numpy as np
import pytest

import extender_libs as xl
import wide_score_libs as wl

CASES = wl.cpu_cases(long=False)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_equals_the_numpy_reference(case):
    expected = wl.expected_run(case)
    got = xl.ssp_rows(xl.oracle_run(case["query"], case["target"], case["matrix"], case["xdrop"], case["no_entropy"], case["threshold"],
                                    case["seeds"]))
    assert got == expected


@pytest.mark.parametrize("n", [127, 128, 129, 255, 256, 257])
def test_identical_runs_give_their_exact_total(n):
    """An identical run of n bases at 2^24 a match: n * 2^24 from a seed in the middle, at the first base and at the last."""
    case = next(c for c in CASES if c["name"] == "identity_run_%d" % n)
    got = xl.oracle_run(case["query"], case["target"], case["matrix"], case["xdrop"], True, case["threshold"], case["seeds"])
    assert xl.ssp_rows(got) == [[40, 40, n - 1, min(n << 24, wl.INT32_MAX)]]
    for s in case["seeds"]:
        o = wl.oracle_seed(case["query"], case["target"], case["matrix"], case["xdrop"], True, case["threshold"], int(s["query"]),
                           int(s["target"]))
        assert (o["query"], o["target"], o["length"], o["total"], o["score"], o["kept"]) == (40, 40, n - 1, n << 24, n << 24, 1)


@pytest.mark.parametrize("case", wl.long_match_cases(), ids=lambda c: c["name"])
def test_long_identical_pairs_at_match_100(case):
    """22 Mb from its first base (one side past 2^31) and 25 Mb from its middle (each side below, the sum above)."""
    n = len(case["query"])
    got = xl.oracle_run(case["query"], case["target"], case["matrix"], case["xdrop"], True, case["threshold"], case["seeds"])
    assert xl.ssp_rows(got) == [[0, 0, n - 1, wl.INT32_MAX]]
    s = case["seeds"][0]
    o = wl.check_seed(case["query"], case["target"], case["matrix"], case["xdrop"], True, case["threshold"], int(s["query"]),
                      int(s["target"]))
    assert (o["query"], o["target"], o["length"], o["total"]) == (0, 0, n - 1, 100 * n)


def test_descents_at_the_xdrop_limit_stop_where_the_reference_says():
    """A descent of 2^31 - 1 does not pass X-drop 2^31 - 1 and one of 2^31 does: both occur in the descent cases."""
    case = next(c for c in CASES if c["name"] == "descents_xdrop_%d" % wl.INT32_MAX)
    m = np.asarray(case["matrix"], np.int64).reshape(8, 8)
    assert m[1, 0] == -wl.INT32_MAX and m[0, 1] == -(1 << 31)
    rng = np.random.default_rng(1)
    # "match, C/A, match" goes on past the descent; "match, A/C, match" stops at it
    for mis, through in (((1, 0), True), ((0, 1), False)):
        b = rng.integers(0, 4, 4).astype(np.int8)
        t = np.concatenate([b[:2], [mis[0]], b[2:]]).astype(np.int8)
        q = np.concatenate([b[:2], [mis[1]], b[2:]]).astype(np.int8)
        o = wl.check_seed(q, t, case["matrix"], wl.INT32_MAX, True, 1, 0, 0)
        assert o["length"] == (4 if through else 1), (mis, o)


@pytest.mark.parametrize("thr", [wl.GATE_WRAP - 1, wl.GATE_WRAP, wl.INT32_MAX])
def test_the_entropy_gate_runs_past_715827882(thr):
    """Every seed of the gate cases has a total inside [T, 3T]; the entropy rule applies to each, so no score equals its total
    and the scores are the oracle's, within 1 of numpy's entropy."""
    case = next(c for c in CASES if c["name"] == "entropy_gate_%d" % thr)
    for s in case["seeds"]:
        r = wl.reference_seed(case["query"], case["target"], case["matrix"], case["xdrop"], False, thr, int(s["query"]), int(s["target"]))
        assert r["gated"] and r["entropy_applies"], r
        o = wl.check_seed(case["query"], case["target"], case["matrix"], case["xdrop"], False, thr, int(s["query"]), int(s["target"]))
        assert o["score"] < o["total"]


def test_a_low_entropy_run_inside_the_gate_is_dropped():
    case = next(c for c in CASES if c["name"] == "entropy_gate_low_entropy")
    for s in case["seeds"]:
        o = wl.check_seed(case["query"], case["target"], case["matrix"], case["xdrop"], False, case["threshold"], int(s["query"]),
                          int(s["target"]))
        assert o["total"] == 100 << 24 and o["kept"] == 0, o
    assert len(xl.oracle_run(case["query"], case["target"], case["matrix"], case["xdrop"], False, case["threshold"], case["seeds"])) == 0


def test_saturated_records_tie_on_score_in_the_sort_and_unique_rule():
    case = next(c for c in CASES if c["name"] == "saturated_ties")
    expected = wl.expected_run(case)
    assert len(expected) >= 4 and all(r[3] == wl.INT32_MAX for r in expected)
    # every kept record, duplicates included, goes in; the rule leaves one per run
    kept = []
    for s in case["seeds"]:
        o = wl.oracle_seed(case["query"], case["target"], case["matrix"], case["xdrop"], True, case["threshold"], int(s["query"]),
                           int(s["target"]))
        kept.append(wl.reported(o))
    rng = np.random.default_rng(3)
    for _ in range(3):
        order = rng.permutation(len(kept))
        rows = np.array([kept[i] for i in order], dtype=np.int64)
        a = np.zeros(len(rows), dtype=xl.SSP_DTYPE)
        for k, f in enumerate(xl.SSP_DTYPE.names):
            a[f] = rows[:, k]
        assert xl.ssp_rows(xl.oracle_sort_unique(a)) == expected


def test_scores_below_2_31_are_unchanged():
    """A seed whose total stays below 2^31 reports its total as before, on the reference's sample matrix."""
    case = wl.case("sample", *wl.homologous(np.random.default_rng(9), 2000, 0.05), xl.SAMPLE_MATRIX, xl.SAMPLE_XDROP,
                   xl.SAMPLE_THRESHOLD, False, [(p, p) for p in range(0, 2000, 37)])
    assert wl.expected_run(case) == xl.ssp_rows(xl.oracle_run(case["query"], case["target"], case["matrix"], case["xdrop"], False,
                                                                case["threshold"], case["seeds"]))
