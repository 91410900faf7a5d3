"""The minimizer index (genomeworks_b200.cudamapper) on the GPU against the stored reference outputs and the CPU oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import index_libs as il
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu

ROOT = il.ROOT
TILE = 2048  # windows per tile (index_kernels.cuh kTileWindows)


@pytest.fixture(scope="module")
def cm():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from genomeworks_b200 import cudamapper
    return cudamapper


def engine(cm, reads, first, k, w, h=True, F=1.0, **kw):
    idx = cm.create_index(reads, first_read_id=first, number_of_reads=len(reads) - first if kw.get("n") is None else kw["n"], kmer_size=k,
                          window_size=w, hash_representations=h, filtering_parameter=F,
                          **{a: b for a, b in kw.items() if a != "n"})
    idx.wait_to_be_ready()
    out = idx.host_copy()
    out["number_of_reads"] = idx.number_of_reads()
    out["longest"] = idx.number_of_basepairs_in_longest_read()
    out["smallest"], out["largest"] = idx.smallest_read_id(), idx.largest_read_id()
    idx.close()
    return out


def same(a, b):
    for name in il.ARRAYS:
        assert len(a[name]) == len(b[name]), name
        assert np.array_equal(a[name].astype(np.uint64), b[name].astype(np.uint64)), name
    assert a["number_of_reads"] == b["number_of_reads"] and a["longest"] == b["longest"]


def test_engine_equals_stored_reference_outputs(cm):
    stored = il.load_fixture()["cases"]
    for name, c in il.cases().items():
        got = engine(cm, c["reads"], c["first"], c["k"], c["w"], c["hash"], c["F"], n=c["n"])
        if c["n"] > 0 and got["number_of_reads"] > 0:
            assert got["smallest"] == c["first"] and got["largest"] == c["first"] + c["n"] - 1, name
        else:
            assert got["smallest"] == 0 and got["largest"] == 0, name
        sub = c["reads"][c["first"]:c["first"] + c["n"]]
        # the only documented difference: the reference renumbers the reads after a skipped one
        assert il.matches(il.renumber(got, sub, c["first"], c["k"], c["w"]), stored[name], il.reference_directions_defined(c)), name


def test_engine_equals_oracle_at_tile_edges(cm):
    rng = np.random.default_rng(5)
    for k, w in ((15, 10), (5, 1), (21, 33), (32, 4), (2, 700)):
        reads = []
        for windows in (TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE + 1, 3 * TILE):
            length = windows + k - w  # a read of L bases has L - k + w windows
            if length >= w + k - 1:
                reads.append(bytes(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, length)]))
        # a final window ending at every residue of the tile width
        for res in range(0, TILE, 97):
            length = TILE * 2 + res + k - w
            reads.append(bytes(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, length)]))
        for h in (True, False):
            same(engine(cm, reads, 0, k, w, h), il.oracle_run(reads, 0, k, w, h))


def test_many_reads_of_exactly_one_window(cm):
    rng = np.random.default_rng(6)
    for k, w in ((15, 10), (3, 1), (32, 20)):
        reads = [bytes(np.frombuffer(b"ACGTN", np.uint8)[rng.integers(0, 5, w + k - 1)]) for _ in range(3000)]
        reads += [b"A" * (w + k - 2)]
        # create_index takes the whole read list and indexes reads[first:]; the oracle takes the indexed reads
        same(engine(cm, [b""] * 7 + reads, 7, k, w), il.oracle_run(reads, 7, k, w))


def test_stream_reuse_and_random_reads(cm):
    import torch
    s = torch.cuda.Stream()
    for seed in range(12):
        rng = np.random.default_rng(100 + seed)
        k, w = int(rng.integers(1, 33)), int(rng.integers(1, 60))
        reads = [bytes(rng.integers(0, 256, int(rng.integers(1, 6000)), dtype=np.uint8)) for _ in range(int(rng.integers(1, 40)))]
        F = float(rng.choice([1.0, 0.3, 1e-3, 0.0]))
        h = bool(seed % 2)
        same(engine(cm, [b""] * seed + reads, seed, k, w, h, F, stream=s), il.oracle_run(reads, seed, k, w, h, F))


def test_host_copy_round_trip_and_readiness(cm):
    reads = il.covid()[:400]
    idx = cm.create_index(reads, kmer_size=15, window_size=10)
    assert not idx.is_ready()
    with pytest.raises(RuntimeError):
        idx.number_of_reads()
    idx.wait_to_be_ready()
    assert idx.is_ready()
    hc = cm.IndexHostCopy(idx)
    a = hc.arrays()
    back = hc.copy_index_to_device()
    assert not back.is_ready()
    back.wait_to_be_ready()
    b = back.host_copy()
    for name in il.ARRAYS:
        assert np.array_equal(a[name], b[name]), name
    assert back.number_of_reads() == idx.number_of_reads() == 400
    assert back.number_of_basepairs_in_longest_read() == idx.number_of_basepairs_in_longest_read()
    back.close()
    hc.close()
    idx.close()


def test_launch_count_independent_of_read_count(cm):
    from genomeworks_b200._lib import lib
    counts = []
    for n in (1, 50, 3000):
        reads = il.covid()[:n]
        before = lib().gwb200_kernel_launch_count()
        idx = cm.create_index(reads, kmer_size=15, window_size=10, filtering_parameter=1e-5)
        idx.wait_to_be_ready()
        counts.append(lib().gwb200_kernel_launch_count() - before)
        idx.close()
    assert counts[0] == counts[1] == counts[2] > 0, counts


def test_all_device_memory_returns_to_the_allocator(cm):
    al = CountingAllocator()
    idx = cm.create_index(il.covid()[:300], kmer_size=15, window_size=10, filtering_parameter=0.5, allocator=al)
    idx.wait_to_be_ready()
    assert al.calls > 0 and al.live
    hc = cm.IndexHostCopy(idx)
    back = hc.copy_index_to_device(allocator=al)
    back.wait_to_be_ready()
    back.close()
    hc.close()
    idx.close()
    assert al.live == {}


def test_cpp_index_api(cm):
    exe = os.path.join(ROOT, "build", "test_cpp_index")
    r = subprocess.run([exe, os.path.join(il.GOLDEN, "catcaag_aagcta.fasta")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ok" in r.stdout
