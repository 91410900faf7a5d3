"""The seeder with any seed pattern and a word cap (DESIGN.md section 22) against its CPU oracle, in content and order: the
golden sample, random and reverse-complemented pairs, device sequences, block cuts, a key with 10^5 target positions at the
cap's edge, and one seeder reused across patterns of different weights with a stream and an allocator."""
import numpy as np
import pytest

import extender_libs as xl
import seed_pattern_libs as sp
import seeder_libs as sl
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu

# weight >= 8: few enough seeds on 10^4 to 10^5 codes for the oracle; the light patterns run on short sequences
HEAVY = ["12of19", "14of22", "match12", "match14", "11010010000000000000000000011011"]
LIGHT = ["match1", "match5", "1", "101"]


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def assert_same(got, want):
    assert len(got) == len(want)
    assert np.array_equal(got["query"], want["query"]) and np.array_equal(got["target"], want["target"])


def blocks(seeder, n, size, first=0):
    """Seeds [first, n) fetched in blocks of `size`, concatenated."""
    parts = [seeder.get_block(f, min(size, n - f)) for f in range(first, n, size)]
    seeder.sync()
    out = np.zeros(n - first, dtype=xl.SEED_DTYPE)
    if n > first:
        h = np.concatenate([p.cpu().numpy() for p in parts])
        out["query"], out["target"] = h[:, 0].view(np.uint32), h[:, 1].view(np.uint32)
    return out


def homologous_pair(seed, n=20000, divergence=0.1):
    from genomeworks_b200 import synth
    target, query, _ = synth.extender_workload(n, divergence, 0, 0.0, seed=seed)
    return query, target


@pytest.mark.parametrize("seed", HEAVY)
@pytest.mark.parametrize("transition", [True, False])
def test_golden_sample(ce, seed, transition):
    seq, _, _ = xl.sample()
    s = ce.create_seeder(transition, seed=seed)
    got = s.seed_pairs(seq, seq)
    assert_same(got, sp.oracle_run(seq, seq, seed, transition))
    s.close()


@pytest.mark.parametrize("seed", HEAVY + LIGHT)
@pytest.mark.parametrize("cap", [0, 1, 2, 1 << 40])
def test_random_and_reverse_complemented_pairs(ce, seed, cap):
    n = 20000 if seed in HEAVY else 1500
    query, target = homologous_pair(sp.PATTERNS.index(seed) + 1, n)
    rng = np.random.default_rng(5)
    query[rng.integers(0, len(query), 20)] = rng.choice(np.array([4, 5, 6], dtype=np.int8), 20)
    for transition in (True, False):
        s = ce.create_seeder(transition, seed=seed, max_word_count=cap)
        for q in (query, sl.reverse_complement(query)):
            want = sp.oracle_run(q, target, seed, transition, cap)
            assert_same(s.seed_pairs(q, target), want)
        s.close()


def repeat_pair():
    """A short repeat unit with scattered transitions: many hits per query position in several buckets, for every pattern."""
    rng = np.random.default_rng(3)
    unit = rng.integers(0, 4, 24).astype(np.int8)
    target = np.tile(unit, 40)
    target[rng.integers(0, len(target), 30)] ^= 2
    query = np.tile(unit, 8)
    query[rng.integers(0, len(query), 6)] ^= 2
    return query, target


@pytest.mark.parametrize("seed", HEAVY + LIGHT)
@pytest.mark.parametrize("cap", [0, 3, 20])
def test_repeats_against_brute_force(ce, seed, cap):
    query, target = repeat_pair()
    s = ce.create_seeder(True, seed=seed, max_word_count=cap)
    got = s.seed_pairs(query, target)
    assert sp.rows(got) == sp.brute(query, target, seed, True, cap)
    s.close()


# each cap drops some buckets and keeps most seeds
@pytest.mark.parametrize("seed, cap", [("14of22", 4), ("match5", 4), ("101", 140)])
def test_device_sequences(ce, seed, cap):
    import torch
    query, target = homologous_pair(13, 20000 if seed == "14of22" else 2000)
    s = ce.create_seeder(True, seed=seed, max_word_count=cap)
    s.index_target(torch.from_numpy(target).cuda())
    n = s.count(torch.from_numpy(query).cuda())
    assert n > 0
    assert_same(blocks(s, n, n), sp.oracle_run(query, target, seed, True, cap))
    s.close()


@pytest.mark.parametrize("size", [1, 7, 1000])
@pytest.mark.parametrize("seed, cap", [("14of22", 0), ("match5", 40), ("101", 0)])
def test_block_cuts(ce, size, seed, cap):
    query, target = repeat_pair()
    s = ce.create_seeder(True, seed=seed, max_word_count=cap)
    s.index_target(target)
    n = s.count(query)
    want = sp.oracle_run(query, target, seed, True, cap)
    assert n == len(want) and n > 3 * size
    # some block ends inside one query position's run of seeds
    q = want["query"]
    ends = np.arange(size, n, size)
    assert (q[ends - 1] == q[ends]).any()
    assert_same(blocks(s, n, size), want)
    assert_same(blocks(s, n, size, n // 3), want[n // 3:])
    s.close()


def test_a_key_with_ten_to_the_five_positions_at_the_cap(ce):
    """Key 0 of 12of19 (19 A's) ends at 10^5 target positions: capped at 99,999 its bucket is gone, at 10^5 it is kept."""
    rng = np.random.default_rng(77)
    rand = rng.integers(1, 4, 3000).astype(np.int8)
    target = np.concatenate([np.zeros(100000 + 18, dtype=np.int8), rand])
    query = np.concatenate([np.zeros(19, dtype=np.int8), np.full(1, 5, np.int8), rand[:500]])
    counts = {}
    for cap in (99_999, 100_000):
        s = ce.create_seeder(False, max_word_count=cap)
        got = s.seed_pairs(query, target)
        want = sp.oracle_run(query, target, "12of19", False, cap)
        assert_same(got, want)
        counts[cap] = int((got["query"] == 18).sum())
        s.close()
    assert counts == {99_999: 0, 100_000: 100_000}


def test_explicit_default_equals_no_set_seed(ce):
    query, target = homologous_pair(31)
    plain = ce.create_seeder(True)
    explicit = ce.create_seeder(True)
    explicit.set_seed("12of19", 0)
    assert_same(explicit.seed_pairs(query, target), plain.seed_pairs(query, target))
    assert_same(plain.seed_pairs(query, target), sl.oracle_run(query, target, True))
    plain.close()
    explicit.close()


def test_one_handle_across_patterns_with_a_stream_and_an_allocator(ce):
    import torch
    query, target = homologous_pair(41, 20000)
    small_q, small_t = query[:1500], target[:1500]
    stream = torch.cuda.Stream()
    alloc = CountingAllocator()
    for s in (ce.create_seeder(True, stream=stream), ce.create_seeder(True, allocator=alloc)):
        for seed, cap in [("14of22", 0), ("match5", 3), ("match14", 0), ("101", 0), ("12of19", 2), ("12of19", 0)]:
            q, t = (query, target) if seed not in LIGHT else (small_q, small_t)
            s.index_target(t)
            s.set_seed(seed, cap)
            # the new seed dropped the index
            with pytest.raises(RuntimeError):
                s.count(q)
            assert_same(s.seed_pairs(q, t), sp.oracle_run(q, t, seed, True, cap))
        s.close()
    assert alloc.calls > 0 and alloc.live == {}
