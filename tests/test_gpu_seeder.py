"""The seeder on the GPU against its CPU oracle, in content and order: the golden sample, random pairs, a key with 10^5 target
positions, block cuts, a reverse-complemented query, and one seeder reused across targets with a stream and an allocator."""
import numpy as np
import pytest

import extender_libs as xl
import seeder_libs as sl
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def assert_same(got, want):
    assert len(got) == len(want)
    assert np.array_equal(got["query"], want["query"]) and np.array_equal(got["target"], want["target"])


def blocks(seeder, n, size):
    """Seeds [0, n) fetched in blocks of `size`, concatenated."""
    parts = [seeder.get_block(first, min(size, n - first)) for first in range(0, n, size)]
    seeder.sync()
    out = np.zeros(n, dtype=xl.SEED_DTYPE)
    if n:
        h = np.concatenate([p.cpu().numpy() for p in parts])
        out["query"], out["target"] = h[:, 0].view(np.uint32), h[:, 1].view(np.uint32)
    return out


@pytest.mark.parametrize("transition", [True, False])
def test_golden_sample(ce, transition):
    seq, _, _ = xl.sample()
    s = ce.create_seeder(transition)
    got = s.seed_pairs(seq, seq)
    assert_same(got, sl.oracle_run(seq, seq, transition))
    assert len(got) == (143671 if transition else 129165)
    index_ms, count_ms, write_ms = s.last_ms()
    assert index_ms > 0 and count_ms > 0 and write_ms > 0
    s.close()


def homologous_pair(seed, n=20000, divergence=0.1):
    from genomeworks_b200 import synth
    target, query, _ = synth.extender_workload(n, divergence, 0, 0.0, seed=seed)
    return query, target


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_random_pairs(ce, seed):
    query, target = homologous_pair(seed)
    rng = np.random.default_rng(seed)
    query[rng.integers(0, len(query), 50)] = rng.choice(np.array([4, 5, 6], dtype=np.int8), 50)
    for transition in (True, False):
        s = ce.create_seeder(transition)
        assert_same(s.seed_pairs(query, target), sl.oracle_run(query, target, transition))
        s.close()


def repeat_case():
    """A target where key 0 (19 A's) ends at 10^5 positions, plus random sequence, and a query of A's and that sequence."""
    rng = np.random.default_rng(77)
    rand = rng.integers(0, 4, 3000).astype(np.int8)
    target = np.concatenate([np.zeros(100000 + 18, dtype=np.int8), rand])
    g = np.zeros(40, dtype=np.int8)
    g[20] = 2  # a G: windows one transition away from all-A
    query = np.concatenate([np.zeros(30, dtype=np.int8), g, rand[:500]])
    return query, target


def small_repeat_case():
    rng = np.random.default_rng(78)
    rand = rng.integers(0, 4, 2000).astype(np.int8)
    return np.concatenate([np.zeros(25, dtype=np.int8), rand[:300]]), np.concatenate([np.zeros(50, dtype=np.int8), rand])


def test_a_key_with_ten_to_the_five_positions(ce):
    query, target = repeat_case()
    s = ce.create_seeder(True)
    got = s.seed_pairs(query, target)
    want = sl.oracle_run(query, target, True)
    assert len(want) > 2_000_000
    assert_same(got, want)
    s.close()


@pytest.mark.parametrize("size", [1, 7, 1000])
def test_block_cuts(ce, size):
    query, target = repeat_case() if size > 1 else small_repeat_case()
    s = ce.create_seeder(True)
    s.index_target(target)
    n = s.count(query)
    want = sl.oracle_run(query, target, True)
    assert n == len(want)
    # some block ends inside one query position's run of seeds
    q = want["query"]
    ends = np.arange(size, n, size)
    assert ((q[ends - 1] == q[ends]).any())
    assert_same(blocks(s, n, size), want)
    # an arbitrary range and an empty one
    first = n // 3
    assert_same(blocks_from(s, first, 12345 if size > 1 else 5), want[first:first + (12345 if size > 1 else 5)])
    assert s.get_block(n, 0).numel() == 0
    with pytest.raises(ValueError):
        s.get_block(n - 1, 2)
    s.close()


def blocks_from(seeder, first, count):
    d = seeder.get_block(first, count)
    seeder.sync()
    h = d.cpu().numpy()
    out = np.zeros(count, dtype=xl.SEED_DTYPE)
    out["query"], out["target"] = h[:, 0].view(np.uint32), h[:, 1].view(np.uint32)
    return out


def test_reverse_complemented_query(ce):
    query, target = homologous_pair(12)
    rc = sl.reverse_complement(query)
    s = ce.create_seeder(True)
    got = s.seed_pairs(rc, target)
    assert_same(got, sl.oracle_run(rc, target, True))
    s.close()


def test_device_sequences(ce):
    import torch
    query, target = homologous_pair(13)
    s = ce.create_seeder(True)
    s.index_target(torch.from_numpy(target).cuda())
    n = s.count(torch.from_numpy(query).cuda())
    assert_same(blocks(s, n, n), sl.oracle_run(query, target, True))
    s.close()


def test_reused_across_targets_with_a_stream_and_an_allocator(ce):
    import torch
    pairs = [homologous_pair(s, 8000) for s in (21, 22, 23)]
    stream = torch.cuda.Stream()
    alloc = CountingAllocator()
    on_stream = ce.create_seeder(True, stream=stream)
    pooled = ce.create_seeder(True, allocator=alloc)
    for query, target in pairs + pairs[:1]:
        want = sl.oracle_run(query, target, True)
        assert_same(on_stream.seed_pairs(query, target), want)
        assert_same(pooled.seed_pairs(query, target), want)
        # one target, two queries
        other = pairs[0][0]
        assert_same(pooled.seed_pairs(other, target), sl.oracle_run(other, target, True))
    assert alloc.calls > 0 and alloc.live
    pooled.close()
    on_stream.close()
    assert alloc.live == {}


def test_call_order_errors(ce):
    s = ce.create_seeder(True)
    with pytest.raises(RuntimeError):
        s.count(np.zeros(30, dtype=np.int8))
    s.index_target(np.zeros(30, dtype=np.int8))
    with pytest.raises(RuntimeError):
        s.get_block(0, 0)
    assert s.count(np.zeros(30, dtype=np.int8)) == 12 * 12
    s.close()
