"""The skip-covered oracle (DESIGN.md section 18) against an independent Python restatement over the gapped extender's oracle,
on hand cases, SSP score ties, random cases and the golden sample. CPU only."""
import numpy as np
import pytest

import extender_libs as xl
import gapped_extender_libs as gl
import gapped_skip_libs as sk

SIMPLE = (xl.SIMPLE_MATRIX, 5, 2, 80)
LASTZ = (xl.SAMPLE_MATRIX, gl.LASTZ_OPEN, gl.LASTZ_EXTEND, gl.LASTZ_YDROP)


def anchors(*pairs):
    return np.array(list(pairs), dtype=gl.ANCHOR_DTYPE)


def both(query, target, params, threshold, a, order=None, budget=1 << 62):
    """The oracle's run, checked equal to the restatement's."""
    got = sk.skip_run(query, target, *params, threshold, a, order, budget)
    want = sk.python_skip(query, target, *params, threshold, a, order, budget)
    assert gl.rows(got[0]) == gl.rows(want[0])
    assert got[1] == want[1] and got[2] == want[2]
    assert got[3]["extended"] == want[3]["extended"] and got[3]["skipped"] == want[3]["skipped"]
    assert got[3]["extended"] + got[3]["skipped"] == len(a)
    return got, want[3]["skipped_anchors"]


def random_seq(rng, n):
    return rng.integers(0, 4, n).astype(np.int8)


def test_second_anchor_on_the_first_path_is_skipped():
    s = random_seq(np.random.default_rng(1), 400)
    (rec, cig, live, stats), skipped = both(s, s, SIMPLE, 0, anchors((100, 100), (200, 200), (300, 301)))
    assert cig[0] == "400M" and stats == {"extended": 2, "skipped": 1} and skipped == [1]
    # the default mode extends all three; the second and the third (which crosses the diagonal with a gap) are duplicates
    full = gl.oracle_run(s, s, *SIMPLE, 0, anchors((100, 100), (200, 200), (300, 301)))
    assert len(full[0]) == 1 and live < full[2]


def insertion_case():
    rng = np.random.default_rng(2)
    t = random_seq(rng, 400)
    q = np.concatenate([t[:200], np.array([0, 1, 2, 3, 3, 2], np.int8), t[200:]])
    rec, cig, _ = gl.oracle_run(q, t, *SIMPLE, 0, anchors((100, 100)))
    assert cig == ["200M6I200M"]
    return q, t


def test_anchor_on_an_insertion_or_deletion_cell_is_extended():
    q, t = insertion_case()
    # (203, 200): query 203 lies in the inserted run, opposite target 200; no M aligns them
    assert (203, 200) not in sk.m_cells(gl.oracle_run(q, t, *SIMPLE, 0, anchors((100, 100)))[0][0], "200M6I200M")
    (rec, _, _, stats), _ = both(q, t, SIMPLE, 0, anchors((100, 100), (203, 200)))
    assert stats == {"extended": 2, "skipped": 0}
    # the same for a deletion: swap the sequences
    (rec, cig, _, stats), _ = both(t, q, SIMPLE, 0, anchors((100, 100), (200, 203)))
    assert cig[0] == "200M6D200M" and stats == {"extended": 2, "skipped": 0}


def test_anchor_covered_only_by_a_below_threshold_alignment_is_extended():
    s = random_seq(np.random.default_rng(3), 400)
    (rec, _, _, stats), _ = both(s, s, SIMPLE, 5000, anchors((100, 100), (200, 200)))
    assert len(rec) == 0 and stats == {"extended": 2, "skipped": 0}


def test_anchor_covered_only_by_an_alignment_without_cigar_is_extended_and_its_duplicate_dropped():
    s = random_seq(np.random.default_rng(4), 400)
    (rec, cig, _, stats), _ = both(s, s, SIMPLE, 0, anchors((100, 100), (200, 200)), budget=0)
    assert len(rec) == 1 and cig == [""] and int(rec[0]["has_cigar"]) == 0 and stats == {"extended": 2, "skipped": 0}


def test_anchor_whose_alignment_duplicates_an_earlier_one_is_dropped():
    # the insertion-cell anchor is extended, and its alignment has the first one's ends
    q, t = insertion_case()
    (rec, _, _, stats), _ = both(q, t, SIMPLE, 0, anchors((100, 100), (203, 200)))
    assert len(rec) == 1 and int(rec[0]["anchor"]) == 0 and stats["extended"] == 2


def test_ssp_score_ties_go_to_the_smaller_index():
    ssps = np.zeros(6, dtype=xl.SSP_DTYPE)
    ssps["score"] = [5, 9, 5, 9, -3, 9]
    assert sk.ssp_order(ssps).tolist() == [1, 3, 5, 0, 2, 4]
    # equal scores on one diagonal: the smaller index is extended, the later ones lie on its path
    s = random_seq(np.random.default_rng(5), 500)
    ssps = np.zeros(4, dtype=ssps.dtype)
    ssps["query"] = ssps["target"] = [300, 100, 200, 50]
    ssps["length"] = 20
    ssps["score"] = [7, 9, 9, 7]
    order = sk.ssp_order(ssps)
    assert order.tolist() == [1, 2, 0, 3]
    (rec, _, _, stats), skipped = both(s, s, SIMPLE, 0, gl.ssp_anchors(ssps), order)
    assert [int(r["anchor"]) for r in rec] == [1] and skipped == [2, 0, 3]


def random_case(rng):
    n = int(rng.integers(60, 240))
    t = random_seq(rng, n)
    q = t.copy()
    q[rng.random(n) < rng.uniform(0, 0.3)] = rng.integers(0, 6)
    if rng.random() < 0.5:  # an indel
        at = int(rng.integers(1, n - 1))
        q = np.concatenate([q[:at], random_seq(rng, int(rng.integers(1, 6))), q[at:]]) if rng.random() < 0.5 else np.delete(q, range(at, min(n - 1, at + 3)))
    k = int(rng.integers(1, 13))
    a = np.zeros(k, dtype=gl.ANCHOR_DTYPE)
    a["query"] = rng.integers(0, len(q), k)
    # mostly near the diagonal, so that anchors share paths
    a["target"] = np.clip(a["query"].astype(np.int64) + rng.integers(-3, 4, k), 0, len(t) - 1)
    order = rng.permutation(k).astype(np.int32)
    return q, t, a, order


@pytest.mark.parametrize("seed", range(300))
def test_random_cases(seed):
    rng = np.random.default_rng(1000 + seed)
    q, t, a, order = random_case(rng)
    o, e, y = int(rng.integers(0, 12)), int(rng.integers(0, 5)), int(rng.integers(10, 120))
    threshold = int(rng.integers(-50, 200))
    budget = [1 << 62, int(rng.integers(0, 3000)), 0][int(rng.integers(0, 3))]
    both(q, t, (xl.SIMPLE_MATRIX, o, e, y), threshold, a, order, budget)


def test_golden_sample_subset_and_coverage_against_the_default_oracle():
    seq, _, golden = xl.sample()
    assert len(golden) == 1337
    a = gl.ssp_anchors(golden)
    order = sk.ssp_order(golden)
    rec, cig, live, stats = sk.skip_run(seq, seq, *LASTZ, gl.LASTZ_THRESHOLD, a, order)
    full_rec, full_cig, full_live = gl.oracle_run(seq, seq, *LASTZ, gl.LASTZ_THRESHOLD, a)
    assert stats["extended"] + stats["skipped"] == 1337 and stats["skipped"] > 0 and live < full_live
    # every skip-mode alignment's score and intervals are one of the default mode's; its CIGAR is the default mode's where both
    # kept the same anchor. (Anchors with equal ends can force different paths, e.g. 20I20D against 20D20I, and the duplicate
    # rule keeps the first in each mode's own order.)
    key = lambda r: (int(r["score"]), int(r["has_cigar"]), int(r["query_begin"]), int(r["query_end"]), int(r["target_begin"]),
                     int(r["target_end"]))
    full = {key(r): (int(r["anchor"]), c) for r, c in zip(full_rec, full_cig)}
    assert 0 < len(rec) <= len(full_rec) and all(key(r) in full for r in rec)
    same = [(c, full[key(r)][1]) for r, c in zip(rec, cig) if full[key(r)][0] == int(r["anchor"])]
    assert len(same) > len(rec) // 2 and all(a == b for a, b in same)
    # every skipped anchor lies on the path of a skip-mode alignment
    cells = set()
    for r, c in zip(rec, cig):
        cells |= sk.m_cells(r, c)
    on_path = [k for k in range(len(a)) if (int(a[k]["query"]), int(a[k]["target"])) in cells]
    assert len(on_path) >= stats["skipped"]
    # the skipped anchors themselves, from the restatement
    want = sk.python_skip(seq, seq, *LASTZ, gl.LASTZ_THRESHOLD, a, order)
    assert gl.rows(want[0]) == gl.rows(rec) and want[1] == cig and want[2] == live
    assert set(want[3]["skipped_anchors"]) <= set(on_path) and len(want[3]["skipped_anchors"]) == stats["skipped"]
