"""CPU checks of the seeder's oracle with any seed pattern and a word cap (oracle/seeder_pattern_oracle.cpp, DESIGN.md section
22): the golden seed file under the default pattern, the §17 oracle's results, and a brute-force restatement in Python for
every pattern, cap, transition variant and word records split across target records."""
import numpy as np
import pytest

import extender_libs as xl
import seed_pattern_libs as sp
import seeder_libs as sl

LAST = (249999, 249999)  # the hit at the sequence's last base, which the golden file omits (DESIGN.md section 17.2)


@pytest.fixture(scope="module")
def sample():
    seq, _, _ = xl.sample()
    return seq, sl.golden_seeds()


@pytest.mark.parametrize("seed", ["12of19", "1110100110010101111"])
@pytest.mark.parametrize("transition", [True, False])
def test_default_pattern_reproduces_the_golden_sample(sample, seed, transition):
    seq, golden = sample
    got = sp.oracle_run(seq, seq, seed, transition)
    want = sl.pair_set(golden)
    if not transition:
        want = {(t, q) for t, q in want if sl.care_codes(seq, t) == sl.care_codes(seq, q)}
    assert sl.pair_set(got) == want | {LAST} and len(got) == len(want) + 1
    # content and order of the section 17 oracle, and a cap above every count changes nothing
    assert sp.rows(got) == sp.rows(sl.oracle_run(seq, seq, transition))
    assert sp.rows(sp.oracle_run(seq, seq, seed, transition, max_word_count=len(seq))) == sp.rows(got)


def repeat_pair(seed, n_target=240, n_query=90):
    """A target and a query built from one short unit with scattered transitions, an N and a soft-masked base: many hits per
    query position, in several buckets, for every pattern."""
    rng = np.random.default_rng(seed)
    unit = rng.integers(0, 4, 24).astype(np.int8)
    target = np.tile(unit, n_target // 24)
    target[rng.integers(0, len(target), 12)] ^= 2
    target[rng.integers(0, len(target))] = 4
    query = np.tile(unit, n_query // 24 + 1)[:n_query]
    query[rng.integers(0, len(query), 3)] ^= 2
    query[rng.integers(0, len(query))] = 5
    return query, target


@pytest.mark.parametrize("transition", [True, False])
@pytest.mark.parametrize("seed", sp.PATTERNS)
def test_patterns_against_brute_force(seed, transition):
    for case in (1, 2):
        query, target = repeat_pair(case)
        want = sp.brute(query, target, seed, transition)
        assert rows_of(query, target, seed, transition) == want
    # random sequences, where most buckets are small
    rng = np.random.default_rng(7)
    query, target = rng.integers(0, 4, 300).astype(np.int8), rng.integers(0, 4, 400).astype(np.int8)
    assert rows_of(query, target, seed, transition) == sp.brute(query, target, seed, transition)


def rows_of(query, target, seed, transition=True, cap=0, word_records=None):
    return sp.rows(sp.oracle_run(query, target, seed, transition, cap, word_records))


@pytest.mark.parametrize("seed", ["12of19", "14of22", "match5", "101"])
@pytest.mark.parametrize("cap", [1, 2, 5, 10 ** 6])
def test_caps_against_brute_force(seed, cap):
    query, target = repeat_pair(3)
    want = sp.brute(query, target, seed, True, cap)
    assert rows_of(query, target, seed, True, cap) == want
    if cap == 10 ** 6:
        assert want == sp.brute(query, target, seed, True)
    elif cap == 1:
        assert len(want) < len(sp.brute(query, target, seed, True))


def variant_case():
    """A query word w whose exact copy occurs 3 times in the target and whose transition variant at care position 0 occurs
    once, under match4 (no other window of the target repeats it)."""
    w = np.array([0, 1, 2, 3], np.int8)
    v = w.copy()
    v[0] ^= 2
    gap = np.array([5], np.int8)
    target = np.concatenate([w, gap, w, gap, w, gap, v, gap])
    return w, v, target


def test_cap_skips_an_exact_bucket_over_the_cap_but_keeps_its_variant():
    w, _, target = variant_case()
    got = rows_of(w, target, "match4", True, 2)
    assert got == [(3, 18)]  # the variant's one copy, ending at 18
    assert got == sp.brute(w, target, "match4", True, 2)
    assert rows_of(w, target, "match4", True, 3) == [(3, 3), (3, 8), (3, 13), (3, 18)]


def test_cap_skips_a_variant_over_the_cap_but_keeps_its_exact_bucket():
    w, v, target = variant_case()
    # query the variant: its exact bucket is the single copy, its variant at care position 0 is w with 3 copies
    got = rows_of(v, target, "match4", True, 2)
    assert got == [(3, 18)] and got == sp.brute(v, target, "match4", True, 2)
    assert rows_of(v, target, "match4", True, 0) == [(3, 18), (3, 3), (3, 8), (3, 13)]


def test_words_are_counted_over_every_word_record():
    """Copies of one word split across records: each record alone stays under the cap, their total does not."""
    w = np.array([2, 0, 3, 1, 1], np.int8)
    records = [np.concatenate([w, np.array([5], np.int8)]) for _ in range(3)]
    target = records[1]
    assert rows_of(w, target, "match5", False, 2) == [(4, 4)]  # the target alone holds one copy
    assert rows_of(w, target, "match5", False, 2, records) == []
    assert rows_of(w, target, "match5", False, 3, records) == [(4, 4)]
    assert rows_of(w, target, "match5", False, 2, records) == sp.brute(w, target, "match5", False, 2, records)


def test_split_repeat_case_depends_on_counting_over_all_records():
    targets, queries, cap = sp.split_repeat_case()
    q = queries[0]
    whole = [rows_of(q, t, "12of19", True, cap, targets) for t in targets]
    alone = [rows_of(q, t, "12of19", True, cap) for t in targets]
    assert sum(map(len, whole)) < sum(map(len, alone))
    assert whole[0] == sp.brute(q, targets[0], "12of19", True, cap, targets)


def test_bad_patterns_and_caps_are_rejected():
    L = sp.oracle()
    import ctypes as C
    span, weight = C.c_int32(), C.c_int32()
    for bad in sp.BAD_PATTERNS:
        assert L.oracle_seed_pattern(bad.encode(), C.byref(span), C.byref(weight)) == 0, bad
    assert L.oracle_seed_pattern(None, C.byref(span), C.byref(weight)) == 0
    for good in sp.PATTERNS:
        assert L.oracle_seed_pattern(good.encode(), C.byref(span), C.byref(weight)) == 1, good
        assert (span.value, weight.value) == (len(sp.bits(good)), sp.bits(good).count("1"))
    s = np.zeros(30, np.int8)
    with pytest.raises(AssertionError):
        sp.oracle_run(s, s, "12of19", True, -1)
