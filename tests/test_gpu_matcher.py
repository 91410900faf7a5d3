"""The anchor matcher (genomeworks_b200.cudamapper.create_matcher) on the GPU against the stored reference outputs and the CPU
oracle: seeded indices, synthetic array sets, every key width, the INT_MAX limit, launches, the allocator and streams."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import index_libs as il
import matcher_libs as ml
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu

ROOT = ml.ROOT


@pytest.fixture(scope="module")
def cm():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from genomeworks_b200 import cudamapper
    return cudamapper


def index(cm, reads, first, n, k, w, h=True, F=1.0, **kw):
    idx = cm.create_index(reads, first_read_id=first, number_of_reads=n, kmer_size=k, window_size=w, hash_representations=h,
                          filtering_parameter=F, **kw)
    idx.wait_to_be_ready()
    return idx


def run(cm, q, t, **kw):
    m = cm.create_matcher(q, t, **kw)
    out = ml.as_rows(m.anchors())
    assert m.number_of_anchors() == len(out)
    bits = m.key_bits()
    m.close()
    return out, bits


def same(a, b):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.array_equal(a, b)


class DeviceIndex:
    """IndexArrays over device copies of host arrays (any index: the role of the reference tests' MockIndex)."""

    def __init__(self, s, number_of_reads, smallest_read_id, longest):
        import torch
        from genomeworks_b200._lib import IndexArrays
        self.keep = []

        def dev(name, dt):
            a = np.ascontiguousarray(s[name], dtype=dt)
            t = torch.from_numpy(a.view(np.int64 if dt == np.uint64 else np.int32).copy()).cuda()
            self.keep.append(t)
            return t.data_ptr() if len(a) else None

        nu = len(s["unique_representations"])
        self.arrays = IndexArrays(unique_representations=dev("unique_representations", np.uint64),
                                  first_occurrence_of_representations=dev("first_occurrence_of_representations", np.uint32),
                                  read_ids=dev("read_ids", np.uint32), positions_in_reads=dev("positions_in_reads", np.uint32),
                                  number_of_sketch_elements=len(s["read_ids"]), number_of_unique_representations=nu,
                                  first_occurrence_size=nu + 1 if nu else 0, number_of_reads=number_of_reads,
                                  smallest_read_id=smallest_read_id, number_of_basepairs_in_longest_read=longest)


def random_sketch(rng, reps, n_reads, smallest, longest, max_run=6):
    """A sketch over the given unique representations: each gets 1..max_run elements with read ids in [smallest,
    smallest + n_reads] and positions in [0, longest] (the inclusive bounds the reference's compound keys allow)."""
    runs = rng.integers(1, max_run + 1, len(reps))
    first = np.concatenate([[0], np.cumsum(runs)]).astype(np.uint32)
    n = int(first[-1])
    return {"unique_representations": np.asarray(reps, np.uint64), "first_occurrence_of_representations": first,
            "read_ids": (smallest + rng.integers(0, n_reads + 1, n, dtype=np.int64)).astype(np.uint32),
            "positions_in_reads": rng.integers(0, longest + 1, n, dtype=np.int64).astype(np.uint32)}


def test_engine_equals_stored_reference_outputs(cm):
    stored = ml.load_fixture()["cases"]
    for name, c in ml.cases().items():
        (qf, qn), (tf, tn) = c["q"], c["t"]
        q = index(cm, c["reads"], qf, qn, c["k"], c["w"], c["hash"], c["F"])
        t = q if c["t"] == c["q"] else index(cm, c["reads"], tf, tn, c["k"], c["w"], c["hash"], c["F"])
        got, _ = run(cm, q, t)
        ren = ml.renumber(got, c["reads"][qf:qf + qn], qf, c["reads"][tf:tf + tn], tf, c["k"], c["w"])
        assert ml.matches(ren, stored[name]), name
        q.close()
        t.close()


def test_seeded_indices_against_oracle(cm):
    """Different first_read_ids on the two sides, the same Index object as query and target, and an index that has been
    through the host-copy round trip."""
    rng = np.random.default_rng(31)
    genome = il.random_reads(40, 1, 20000, 20000)[0]
    reads = []
    for _ in range(120):
        L = int(rng.integers(30, 2000))
        s = int(rng.integers(0, len(genome) - L))
        reads.append(genome[s:s + L])
    reads += [b"ACG", b"T"] + il.random_reads(41, 10, 50, 400)
    for k, w, h in ((15, 10, True), (11, 3, False), (5, 1, True)):
        q = index(cm, reads, 7, 60, k, w, h)
        t = index(cm, reads, 50, len(reads) - 50, k, w, h)
        qs = il.oracle_run(reads[7:67], 7, k, w, h)
        ts = il.oracle_run(reads[50:], 50, k, w, h)
        same(run(cm, q, t)[0], ml.oracle_run(qs, ts))
        same(run(cm, t, q)[0], ml.oracle_run(ts, qs))
        same(run(cm, q, q)[0], ml.oracle_run(qs, qs))
        hc = cm.IndexHostCopy(t)
        back = hc.copy_index_to_device()
        back.wait_to_be_ready()
        same(run(cm, q, back)[0], ml.oracle_run(qs, ts))
        for x in (back, hc, q, t):
            x.close()


def test_synthetic_arrays_against_oracle(cm):
    """Random array sets: disjoint representations (zero anchors), query representations beyond the last target one, read ids
    and positions at their inclusive bounds, and heavy runs."""
    rng = np.random.default_rng(32)
    for trial in range(24):
        pool = np.unique(rng.integers(0, 2**64 - 1, 400, dtype=np.uint64))
        if trial % 4 == 0:  # disjoint
            qr, tr = pool[:150], pool[150:300]
        elif trial % 4 == 1:  # every query representation beyond the last target one but a few
            qr, tr = pool[-120:], pool[:200].tolist() + pool[-120:-115].tolist()
        else:
            qr = np.sort(rng.choice(pool, 200, replace=False))
            tr = np.sort(rng.choice(pool, 200, replace=False))
        nq, nt = int(rng.integers(1, 5000)), int(rng.integers(1, 5000))
        lq, lt = int(rng.integers(1, 10**6)), int(rng.integers(1, 10**6))
        q_min, t_min = int(rng.integers(0, 10**6)), int(rng.integers(0, 10**6))
        qs = random_sketch(rng, np.sort(np.asarray(qr, np.uint64)), nq, q_min, lq, 3 + 20 * (trial % 3 == 2))
        ts = random_sketch(rng, np.sort(np.asarray(tr, np.uint64)), nt, t_min, lt, 3 + 20 * (trial % 3 == 2))
        qd, td = DeviceIndex(qs, nq, q_min, lq), DeviceIndex(ts, nt, t_min, lt)  # the device arrays live as long as these
        got, bits = run(cm, qd.arrays, td.arrays)
        want = ml.oracle_run(qs, ts)
        same(got, want)
        if trial % 4 == 0:
            assert len(got) == 0
        elif len(want):
            assert bits == ml.key_bits(nq, lq, nt, lt)


def reads_for_width(bits, longest):
    """The number of reads N (one of `longest` bases, N - 1 of one base) for which an all-vs-all key has exactly `bits` bits."""
    n = 1
    while ml.key_bits(n, longest, n, longest) < bits:
        n += 1
    assert ml.key_bits(n, longest, n, longest) == bits
    return n


@pytest.mark.parametrize("bits,longest", [(31, 500), (32, 500), (33, 500), (63, 100000), (64, 100000), (65, 100000), (67, 100000)])
def test_key_widths_against_oracle(cm, bits, longest):
    """Real indices whose key needs the given width: one-base reads (skipped, but counted in number_of_reads) inflate N, one long
    read sets L. 65 and 67 bits take the 128-bit key."""
    n = reads_for_width(bits, longest)
    long_read = il.random_reads(50 + bits, 1, longest, longest)[0]
    reads = [b"A"] * (n // 2) + [long_read] + [b"C"] * (n - 1 - n // 2)
    idx = index(cm, reads, 0, n, 15, 10)
    assert idx.number_of_reads() == n and idx.number_of_basepairs_in_longest_read() == longest
    got, got_bits = run(cm, idx, idx)
    s = il.oracle_run(reads, 0, 15, 10)
    assert got_bits == bits and len(got) > 0
    same(got, ml.oracle_run(s, s))
    idx.close()


def test_widest_key_against_oracle(cm):
    """Read ids and positions at the top of the 32-bit range: a 128-bit key."""
    rng = np.random.default_rng(33)
    reps = np.sort(rng.choice(2**40, 50, replace=False)).astype(np.uint64)
    top = 2**32 - 1
    qs = random_sketch(rng, reps, top - 5, 2, top - 1)
    ts = random_sketch(rng, reps[::2], top - 7, 4, top - 1)
    qd, td = DeviceIndex(qs, top - 5, 2, top - 1), DeviceIndex(ts, top - 7, 4, top - 1)
    got, bits = run(cm, qd.arrays, td.arrays)
    assert bits == ml.key_bits(top - 5, top - 1, top - 7, top - 1) > 120
    same(got, ml.oracle_run(qs, ts))


def test_more_than_int_max_anchors_rejected_before_allocating_them(cm):
    """One 46,355-base homopolymer per side: 2,147,488,281 anchors. The call raises after counting, and nothing it allocated is
    left outstanding; no buffer was anchor-sized."""
    q = index(cm, [b"A" * 46355], 0, 1, 15, 1, False)
    t = index(cm, [b"A" * 46355], 0, 1, 15, 1, False)
    al = CountingAllocator()
    sizes = []
    alloc = al.alloc
    al.alloc = lambda n: (sizes.append(n), alloc(n))[1]
    with pytest.raises(ValueError, match="INT_MAX"):
        cm.create_matcher(q, t, allocator=al)
    assert al.live == {} and sizes and max(sizes) < 2**20
    q.close()
    t.close()


def test_launch_count_independent_of_read_count(cm):
    from genomeworks_b200._lib import lib
    cv = il.covid()
    all_reads = index(cm, cv, 0, 3000, 15, 10)
    one = index(cm, cv, 0, 1, 15, 10)
    empty = index(cm, [b"ACG"], 0, 1, 15, 10)
    counts = []
    for q, t in ((one, all_reads), (all_reads, all_reads), (empty, all_reads), (all_reads, empty)):
        before = lib().gwb200_kernel_launch_count()
        m = cm.create_matcher(q, t)
        assert (m.number_of_anchors() > 0) == (q is not empty and t is not empty)
        counts.append(lib().gwb200_kernel_launch_count() - before)
        m.close()
    assert counts[0] == counts[1] > 0 and counts[2] == counts[3] == 0, counts
    for x in (all_reads, one, empty):
        x.close()


def test_allocator_holds_only_the_anchors(cm):
    cv = il.covid()[:300]
    idx = index(cm, cv, 0, 300, 15, 10)
    al = CountingAllocator()
    m = cm.create_matcher(idx, idx, allocator=al)
    n = m.number_of_anchors()
    assert n > 0 and al.calls > 1 and len(al.live) == 1 and list(al.live.values())[0] >= 16 * n
    same(ml.as_rows(m.anchors()), run(cm, idx, idx)[0])
    m.close()
    assert al.live == {}
    for refuse in range(1, al.calls + 1):
        bad = CountingAllocator(refuse)
        with pytest.raises(MemoryError):
            cm.create_matcher(idx, idx, allocator=bad)
        assert bad.live == {}, refuse
    idx.close()


def test_non_default_stream(cm):
    import torch
    s = torch.cuda.Stream()
    cv = il.covid()
    q = index(cm, cv, 0, 700, 15, 10, stream=s)
    t = index(cm, cv, 500, 900, 15, 10, stream=s)
    got, _ = run(cm, q, t, stream=s)
    same(got, ml.oracle_run(il.oracle_run(cv[:700], 0, 15, 10), il.oracle_run(cv[500:1400], 500, 15, 10)))
    q.close()
    t.close()


def test_cpp_matcher_api(cm):
    exe = os.path.join(ROOT, "build", "test_cpp_matcher")
    r = subprocess.run([exe, os.path.join(il.GOLDEN, "catcaag_aagcta.fasta")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ok" in r.stdout
