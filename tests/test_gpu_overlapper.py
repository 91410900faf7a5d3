"""The overlapper (genomeworks_b200.cudamapper.create_overlapper) on the GPU against the stored reference outputs and the CPU
oracle with the device's division: seeded and synthetic anchor sets, chains and groups across the kernels' tile edges, the full
index -> matcher -> overlapper pipeline, launches, the allocator, the INT_MAX limit, streams and the C++ classes."""
import os
import subprocess

import numpy as np
import pytest

import index_libs as il
import matcher_libs as ml
import overlapper_libs as ol
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu

ROOT = ol.ROOT


@pytest.fixture(scope="module")
def cm():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from genomeworks_b200 import cudamapper
    return cudamapper


@pytest.fixture(scope="module")
def fdiv(cm):
    """The device's __fdividef as the oracle's division of the fraction filter (the reference's float division compiles to it
    under -use_fast_math)."""
    from genomeworks_b200 import cudapoa
    cache = {}

    def div(a, b):
        k = (a, b)
        if k not in cache:
            cache[k] = float(cudapoa.device_fdividef([a], [b])[0])
        return cache[k]

    return ol.DIV_T(div)


class DeviceAnchors:
    """A device copy of an (n, 4) anchor array, as the (pointer, count) pair get_overlaps takes."""

    def __init__(self, anchors):
        import torch
        a = ol.anchors_array(anchors)
        self.t = torch.from_numpy(a.view(np.int32).copy()).cuda() if len(a) else None
        self.arg = (self.t.data_ptr() if len(a) else 0, len(a))


def run(cm, anchors, params, overlapper=None, **kw):
    ov = overlapper or cm.create_overlapper(**kw)
    out = ov.get_overlaps(DeviceAnchors(anchors).arg, *params)
    if overlapper is None:
        ov.close()
    return out


def same(got, want):
    assert ol.rows(got) == ol.rows(want)


def test_engine_equals_stored_reference_outputs(cm):
    stored = ol.load_fixture()["cases"]
    ov = cm.create_overlapper()
    for name, c in {**ol.cases(), **ol.matcher_cases()}.items():
        d = DeviceAnchors(c["anchors"])
        for p, params in c["params"].items():
            assert ol.matches(ov.get_overlaps(d.arg, *params), stored[name][p]), (name, p)
    ov.close()


def test_engine_equals_oracle_with_the_device_division(cm, fdiv):
    ov = cm.create_overlapper()
    for name, c in ol.cases().items():
        d = DeviceAnchors(c["anchors"])
        for p, params in c["params"].items():
            same(ov.get_overlaps(d.arg, *params), ol.oracle_run(c["anchors"], params, fdiv))
    ov.close()


def tiled_anchors(rng, n, long_every):
    """n sorted anchors of few read pairs: mostly chains of random length 1..6, with a chain of long_every anchors now and then, so
    chains, kept chains and groups start and end at every offset of a tile, and some chains span many tiles."""
    out, q, t, pair = [], 0, 0, 0
    while len(out) < n:
        if rng.random() < 0.02:
            pair += 1
            q, t = 0, 0
        L = long_every if rng.random() < 0.01 else int(rng.integers(1, 7))
        for _ in range(L):
            out.append([pair // 7, pair % 7, q, t])
            q += int(rng.integers(1, 150))
            t += int(rng.integers(0, 150))
        q += int(rng.integers(150, 900))
        t += int(rng.integers(150, 900)) + int(rng.choice([0, 0, 400]))
    return ol.anchors_array(out[:n])


@pytest.mark.parametrize("n", [4, 255, 256, 257, 2047, 2048, 2049, 3 * 1920 + 1, 65536 + 7, 300001])
def test_tile_edges_against_oracle(cm, fdiv, n):
    rng = np.random.default_rng(n)
    a = tiled_anchors(rng, n, 5000)
    ov = cm.create_overlapper()
    d = DeviceAnchors(a)
    for p in ("cli_a2a", "negative_bases_per_residue", "triggered"):
        same(ov.get_overlaps(d.arg, *ol.PARAMS[p]), ol.oracle_run(a, ol.PARAMS[p], fdiv))
    ov.close()


def test_one_chain_across_many_tiles(cm, fdiv):
    a = ol.anchors_array(ol.chain(0, 1, 0, 0, [(100, 100)] * 200000))
    got = run(cm, a, ol.PARAMS["cli"])
    assert len(got) == 1 and int(got[0]["num_residues"]) == 200001
    same(got, ol.oracle_run(a, ol.PARAMS["cli"], fdiv))


def test_pipeline_on_covid_reads_against_oracle_chain(cm, fdiv):
    cv = il.covid()
    idx = cm.create_index(cv, kmer_size=15, window_size=10)
    idx.wait_to_be_ready()
    m = cm.create_matcher(idx, idx)
    s = il.oracle_run(cv, 0, 15, 10)
    anchors = ml.oracle_run(s, s)
    ov = cm.create_overlapper()
    for p in ("cli_a2a", "triggered_a2a"):
        got = ov.get_overlaps(m, *ol.PARAMS[p])
        same(got, ol.oracle_run(anchors, ol.PARAMS[p], fdiv))
    assert len(got) > 0
    for x in (ov, m, idx):
        x.close()


def test_pipeline_on_reads_of_one_genome_against_oracle_chain(cm, fdiv):
    rng = np.random.default_rng(61)
    genome = il.random_reads(61, 1, 100000, 100000)[0]
    reads = []
    for _ in range(200):
        L = int(rng.integers(2000, 8000))
        st = int(rng.integers(0, len(genome) - L))
        reads.append(genome[st:st + L])
    idx = cm.create_index(reads, kmer_size=15, window_size=10)
    idx.wait_to_be_ready()
    m = cm.create_matcher(idx, idx)
    s = il.oracle_run(reads, 0, 15, 10)
    anchors = ml.oracle_run(s, s)
    ov = cm.create_overlapper()
    got = ov.get_overlaps(m, *ol.PARAMS["cli_a2a"])
    assert len(got) > 100
    same(got, ol.oracle_run(anchors, ol.PARAMS["cli_a2a"], fdiv))
    fused = cm.post_process_overlaps(got)
    assert len(fused) >= len(got)
    for x in (ov, m, idx):
        x.close()


def test_launch_count_independent_of_anchor_count(cm):
    from genomeworks_b200._lib import lib
    ov = cm.create_overlapper()
    counts = []
    for n in (1, 3, 1000, 250000, 0):
        d = DeviceAnchors(tiled_anchors(np.random.default_rng(5), n, 100))
        before = lib().gwb200_kernel_launch_count()
        ov.get_overlaps(d.arg, *ol.PARAMS["cli"])
        counts.append(lib().gwb200_kernel_launch_count() - before)
    assert counts[:4] == [counts[0]] * 4 and counts[0] > 0 and counts[4] == 0, counts
    assert ov.last_kernel_ms() == -1.0  # nothing ran for n == 0
    ov.close()


def test_allocator_balance_and_refusal(cm):
    a = ol.synthetic_anchors(200, n_pairs=3000, max_chains=30)
    d = DeviceAnchors(a)
    al = CountingAllocator()
    ov = cm.create_overlapper(allocator=al)
    got = ov.get_overlaps(d.arg, *ol.PARAMS["cli"])
    assert al.calls > 1 and al.live == {}
    same(got, run(cm, a, ol.PARAMS["cli"]))
    ov.close()
    for refuse in range(1, al.calls + 1):
        bad = CountingAllocator(refuse)
        ovb = cm.create_overlapper(allocator=bad)
        with pytest.raises(MemoryError):
            ovb.get_overlaps(d.arg, *ol.PARAMS["cli"])
        assert bad.live == {}, refuse
        same(ovb.get_overlaps(d.arg, *ol.PARAMS["cli"]), got)  # the same overlapper works once memory is there again
        assert bad.live == {}
        ovb.close()


def test_more_than_int_max_anchors_rejected_before_device_work(cm):
    al = CountingAllocator()
    ov = cm.create_overlapper(allocator=al)
    with pytest.raises(ValueError, match="INT_MAX"):
        ov.get_overlaps((16, ol.INT_MAX + 1), True)  # a dummy pointer: nothing is read through it
    assert al.calls == 0
    ov.close()


def test_non_default_stream_and_reuse(cm, fdiv):
    import torch
    s = torch.cuda.Stream()
    ov = cm.create_overlapper(stream=s)
    for seed in range(4):
        a = ol.synthetic_anchors(400 + seed, n_pairs=200)
        with torch.cuda.stream(s):
            d = DeviceAnchors(a)
        s.synchronize()
        same(ov.get_overlaps(d.arg, *ol.PARAMS["cli"]), ol.oracle_run(a, ol.PARAMS["cli"], fdiv))
        assert ov.last_kernel_ms() > 0
    ov.close()


def test_cpp_overlapper_api(cm, fdiv, tmp_path):
    """The reference sample's sequence through the C++ classes on the covid reads (uncompressed: the FASTA parser reads plain
    text): the overlaps it prints equal the oracle chain's, and its post-processed list equals the library's
    post_process_overlaps of them."""
    exe = os.path.join(ROOT, "build", "test_cpp_overlapper")
    cv = il.covid()
    path = tmp_path / "covid.fasta"
    path.write_bytes(b"".join(b">read_%d\n%s\n" % (i, r) for i, r in enumerate(cv)))
    r = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr
    lines = r.stdout.split("\n")
    assert lines[-2] == "ok"
    got = [[int(v) for v in ln.split()[1:]] for ln in lines if ln.startswith("overlap ")]
    fused = [[int(v) for v in ln.split()[1:]] for ln in lines if ln.startswith("fused ")]
    s = il.oracle_run(cv, 0, 15, 10)
    want = ol.oracle_run(ml.oracle_run(s, s), ol.PARAMS["cli_a2a"], fdiv)
    assert got == ol.rows(want) and len(got) > 0
    assert fused == ol.rows(cm.post_process_overlaps(want))
