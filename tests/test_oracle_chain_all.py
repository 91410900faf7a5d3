"""The all-chains extract oracle (oracle/chain_extract_oracle.cpp) against the plain-Python restatement of DESIGN.md
section 20.1 by the subtree form: hand cases, 300 random sets at three minimum scores, and the contract's invariants. CPU only."""
import numpy as np
import pytest

import chain_all_libs as ca
import chain_libs as cl

LO = ca.INT64_MIN
HI = ca.INT64_MAX


def check(rows, S=LO, D=0, A=0):
    s = cl.ssps_of(rows) if not isinstance(rows, np.ndarray) else rows
    got = ca.oracle_all(s, D, A, S)
    want = ca.python_extract(s, got["f"], got["p"], S)
    assert ca.same_chains(got, want), (got, want)
    invariants(s, got, S)
    return got


def chains(res):
    o = res["offsets"]
    return [res["members"][o[c]:o[c + 1]].tolist() for c in range(len(res["scores"]))]


def invariants(s, res, S):
    """Chains are disjoint and ascending; each is one p-path (exactly one member's p leaves it, and exactly one member is no
    member's p); every score is >= S; at S = INT64_MIN the chains partition all n SSPs; the union and sum match the chains."""
    n, p = len(s), res["p"]
    seen = set()
    for ch, score in zip(chains(res), res["scores"]):
        assert ch == sorted(ch) and not seen & set(ch) and score >= S
        seen |= set(ch)
        assert sum(1 for k in ch if p[k] < 0 or p[k] not in ch) == 1
        assert sum(1 for k in ch if k not in p[ch]) == 1  # one head: the member no other member links to
    if S == LO:
        assert seen == set(range(n))
    assert np.array_equal(res["union"], np.sort(np.array(sorted(seen), dtype=np.int32))) and res["sum"] == int(res["scores"].sum())


def test_two_disjoint_ladders():
    rows = [(0, 1000, 10, 50), (20, 1020, 10, 50), (40, 1040, 10, 50), (1000, 0, 10, 40), (1020, 20, 10, 40)]
    r = check(rows)
    assert chains(r) == [[0, 1, 2], [3, 4]] and list(r["scores"]) == [150, 80]
    r = check(rows, S=100)
    assert chains(r) == [[0, 1, 2]] and list(r["union"]) == [0, 1, 2] and r["sum"] == 150


def test_overlapping_side_ssp_is_its_own_chain_and_is_dropped():
    rows = [(0, 0, 10, 50), (20, 20, 10, 50), (40, 40, 10, 50), (22, 22, 10, 30)]
    r = check(rows)
    assert r["p"][3] == 0 and r["f"][3] == 80
    assert chains(r) == [[0, 1, 2], [3]] and list(r["scores"]) == [150, 30]
    r = check(rows, S=100)
    assert chains(r) == [[0, 1, 2]]


def test_shared_prefix_second_chain_stops_there():
    rows = [(0, 0, 10, 50), (20, 20, 10, 60), (40, 40, 10, 60), (20, 100, 10, 40)]
    r = check(rows)
    assert r["p"][3] == 0 and r["f"][3] == 90
    assert chains(r) == [[0, 1, 2], [3]] and list(r["scores"]) == [170, 40]


def test_heads_with_equal_f_go_by_index():
    rows = [(98, 98, 5, 7), (100, 0, 5, 30), (0, 100, 5, 30)]
    r = check(rows)
    assert chains(r) == [[1], [2], [0]] and list(r["scores"]) == [30, 30, 7]


def test_truncated_chain_with_a_negative_score():
    rows = [(0, 0, 10, 50), (20, 20, 10, 60), (40, 40, 10, 60), (20, 100, 10, -5)]
    r = check(rows)
    assert r["p"][3] == 0 and r["f"][3] == 45
    assert chains(r) == [[0, 1, 2], [3]] and list(r["scores"]) == [170, -5]
    assert chains(check(rows, S=0)) == [[0, 1, 2]]
    assert chains(check(rows, S=-5)) == [[0, 1, 2], [3]]


def test_penalised_links_score_as_the_chain_alone():
    # the chain's score is its sum of s less its links' penalties, = f(h) - f(c_1) + s(c_1)
    rows = [(0, 0, 10, 100), (20, 25, 10, 100), (40, 50, 10, 100), (22, 200, 10, 90)]
    r = check(rows, D=2, A=1)
    assert list(r["p"]) == [-1, 0, 1, -1] and chains(r) == [[0, 1, 2], [3]] and list(r["scores"]) == [300 - 2 * 33, 90]


def test_empty_and_single():
    r = check([])
    assert len(r["scores"]) == 0 and list(r["offsets"]) == [0] and r["sum"] == 0
    r = check([(5, 9, 3, -7)])
    assert chains(r) == [[0]] and list(r["scores"]) == [-7]
    r = check([(5, 9, 3, -7)], S=-6)
    assert chains(r) == [] and list(r["offsets"]) == [0]


def test_lowest_and_highest_minimum():
    rng = np.random.default_rng(5)
    s = cl.random_ssps(rng, 50, span=300, max_len=30)
    r = check(s, S=LO)
    assert sorted(r["members"].tolist()) == list(range(50))
    r = check(s, S=HI)
    assert len(r["scores"]) == 0 and len(r["members"]) == 0
    top = int(check(s)["scores"].max())
    assert len(check(s, S=top + 1)["scores"]) == 0 and len(check(s, S=top)["scores"]) >= 1


@pytest.mark.parametrize("seed", range(300))
def test_random_sets(seed):
    rng = np.random.default_rng(3000 + seed)
    n = int(rng.integers(0, 60))
    D, A = [(0, 0), (1, 0), (0, 1), (3, 2), (1 << 20, 0)][seed % 5]
    s = cl.random_ssps(rng, n, span=int(rng.integers(20, 400)), max_len=int(rng.integers(0, 40)))
    for S in (LO, 0, 60):
        check(s, S, D, A)


@pytest.mark.parametrize("seed", range(20))
def test_first_candidate_is_the_best_chain(seed):
    rng = np.random.default_rng(7000 + seed)
    s = cl.random_ssps(rng, int(rng.integers(1, 60)), span=300, max_len=30)
    best = cl.oracle_run(s, 1, 1)
    r = check(s, LO, 1, 1)
    assert chains(r)[0] == cl.chain_indices(best).tolist() and r["scores"][0] == best["score"]
    r = check(s, best["score"], 1, 1)
    assert chains(r)[0] == cl.chain_indices(best).tolist()
