"""The chain oracle (oracle/chain_oracle.cpp) against the plain-Python restatement of DESIGN.md section 19: hand cases at every
edge of the contract, 300 random sets, and a permutation of a tie-free input. CPU only."""
import numpy as np
import pytest

import chain_libs as cl

TOP = (1 << 32) - 1


def check(rows, D=0, A=0):
    s = cl.ssps_of(rows) if not isinstance(rows, np.ndarray) else rows
    got = cl.oracle_run(s, D, A)
    want = cl.python_chain(s, D, A)
    assert cl.same(got, want), (got, want)
    return got


def test_empty_and_single():
    r = check([])
    assert len(r["chain"]) == 0 and r["score"] == 0
    r = check([(5, 9, 3, -7)])
    assert list(r["chain"]) == [0] and r["score"] == -7 and list(r["p"]) == [-1]


@pytest.mark.parametrize("axis", ["query", "target", "both"])
def test_touching_segments_do_not_chain(axis):
    # the first covers [10, 20]; the second starts at 21 (end + 1) in `axis` and well after in the other
    q2 = 21 if axis in ("query", "both") else 40
    t2 = 21 if axis in ("target", "both") else 40
    r = check([(10, 10, 10, 50), (q2, t2, 5, 50)])
    assert list(r["p"]) == [-1, 0] and r["score"] == 100
    # starting at 20, the end itself, they touch and do not chain
    q2 = 20 if axis in ("query", "both") else 40
    t2 = 20 if axis in ("target", "both") else 40
    r = check([(10, 10, 10, 50), (q2, t2, 5, 50)])
    assert list(r["p"]) == [-1, -1] and r["score"] == 50 and list(r["chain"]) == [0]


def test_overlapping_segments_do_not_chain():
    r = check([(0, 0, 100, 10), (50, 50, 100, 20), (80, 300, 10, 5)])
    assert list(r["p"]) == [-1, -1, -1] and list(r["chain"]) == [1]


def test_diagonal_shift_broken_by_a_large_diagonal_penalty():
    rows = [(0, 0, 10, 100), (20, 40, 10, 100)]  # dq = 9, dt = 29: |dt - dq| = 20
    assert check(rows)["score"] == 200
    assert check(rows, D=4)["score"] == 120
    r = check(rows, D=5)
    assert r["score"] == 100 and list(r["chain"]) == [0] and list(r["p"]) == [-1, -1]  # 100 - 100 = 0 is not > 0


def test_anti_diagonal_gap_broken_by_a_large_anti_penalty():
    rows = [(0, 0, 10, 100), (30, 30, 10, 100)]  # dq = dt = 19
    assert check(rows, A=2)["score"] == 200 - 76
    for A in (3, 1 << 20):  # 100 - 38 A <= 0
        r = check(rows, A=A)
        assert r["score"] == 100 and list(r["chain"]) == [0] and list(r["p"]) == [-1, -1]


def test_equal_f_ends_take_the_smallest_index():
    r = check([(100, 100, 5, 30), (0, 0, 5, 30), (200, 0, 5, 30)])
    assert list(r["f"]) == [60, 30, 30] and list(r["chain"]) == [0, 1]
    r = check([(200, 0, 5, 30), (0, 200, 5, 30), (400, 400, 5, 10), (500, 500, 5, 10)])
    assert r["score"] == 50 and list(r["chain"]) == [3, 2, 0]


def test_equal_value_predecessors_take_the_smallest_index():
    r = check([(0, 50, 5, 40), (50, 0, 5, 40), (0, 0, 5, 40), (100, 100, 5, 1)])
    assert r["p"][3] == 0 and list(r["chain"]) == [3, 0]
    r = check([(50, 0, 5, 40), (0, 50, 5, 40), (100, 100, 5, 1)])
    assert r["p"][2] == 0


def test_zero_and_negative_scores():
    r = check([(0, 0, 5, 0), (10, 10, 5, 0), (20, 20, 5, 0)])
    assert list(r["p"]) == [-1, -1, -1] and r["score"] == 0 and list(r["chain"]) == [0]
    r = check([(0, 0, 5, -5), (10, 10, 5, -1), (20, 20, 5, -3)])
    assert list(r["p"]) == [-1, -1, -1] and r["score"] == -1 and list(r["chain"]) == [1]
    # a negative SSP is chained through when what comes before it pays for it and the direct link costs more
    r = check([(0, 0, 5, 50), (10, 10, 20, -20), (40, 40, 5, 10)], A=1)
    assert list(r["p"]) == [-1, 0, 1] and list(r["f"]) == [50, 22, 14] and r["score"] == 50


def test_empty_segments():
    # L = -1 covers nothing: it precedes a segment that starts at its start, and follows one that ends just before it
    r = check([(10, 10, -1, 5), (10, 10, 4, 5)])
    assert list(r["p"]) == [-1, 0]
    r = check([(0, 0, 9, 5), (10, 10, -1, 5)])
    assert list(r["p"]) == [-1, 0]
    # two empty segments at one start: only the smaller index precedes
    r = check([(10, 10, -1, 5), (10, 10, -1, 7), (10, 10, -1, 1)])
    assert list(r["p"]) == [-1, 0, 1] and r["score"] == 13 and list(r["chain"]) == [2, 1, 0]
    with pytest.raises(ValueError):
        cl.oracle_run(cl.ssps_of([(0, 0, -2, 5)]))


def test_starts_near_the_top_of_uint32():
    rows = [(TOP - 100, TOP - 100, 20, 30), (TOP - 50, TOP - 60, 10, 30), (TOP - 1, TOP, 0, 30), (TOP, TOP, -1, 3), (TOP, TOP - 10, 5, 1)]
    for D, A in ((0, 0), (1, 1), (1 << 20, 1 << 20)):
        check(rows, D, A)
    r = check(rows)
    assert r["score"] == 90 and list(r["chain"]) == [2, 1, 0] and r["p"][3] == 1


@pytest.mark.parametrize("seed", range(300))
def test_random_sets(seed):
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(0, 60))
    D, A = [(0, 0), (1, 0), (0, 1), (3, 2), (1 << 20, 0), (0, 1 << 20)][seed % 6]
    base = TOP - 400 if seed % 10 == 9 else 0
    s = cl.random_ssps(rng, n, span=int(rng.integers(20, 400)), max_len=int(rng.integers(0, 40)), base=base)
    check(s, D, A)


def tie_free(rng, n):
    """A random set whose largest f is unique and whose every positive maximum over predecessors is attained once."""
    while True:
        s = cl.random_ssps(rng, n, span=5000, max_len=200, scores=(1, 10 ** 8))
        s["length"] = np.maximum(s["length"], 0)
        f = cl.python_chain(s, 1, 1)["f"]
        q, t, L = (s[x].astype(np.int64) for x in ("query", "target", "length"))
        ties = (f == f.max()).sum() > 1
        for j in range(n):
            dq, dt = q[j] - q - L - 1, t[j] - t - L - 1
            v = (f - np.abs(dt - dq) - (dq + dt))[(dq >= 0) & (dt >= 0)]
            ties |= len(v) > 0 and v.max() > 0 and (v == v.max()).sum() > 1
        if not ties:
            return s


def test_permutation_of_a_tie_free_input():
    rng = np.random.default_rng(77)
    s = tie_free(rng, 80)
    want = cl.oracle_run(s, 1, 1)
    assert len(want["chain"]) > 3
    for _ in range(5):
        perm = rng.permutation(len(s))
        got = cl.oracle_run(s[perm], 1, 1)
        assert sorted(perm[got["chain"]].tolist()) == sorted(want["chain"].tolist()) and got["score"] == want["score"]
        assert np.array_equal(got["f"], want["f"][perm])
