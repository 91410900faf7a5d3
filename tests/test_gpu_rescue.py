"""The overlap-end rescue (genomeworks_b200.cudamapper.rescue_overlap_ends) on the GPU against the stored reference outputs and
the CPU oracle: windows on each side of the kernels' path switches (the warp path up to 78 bases, the shared-memory table up to
2,062 and the global table past it, whole reads), three effective rounds, the index -> matcher -> overlapper -> rescue pipeline,
rejections, launches, the allocator, streams and the C++ API."""
import os
import subprocess

import numpy as np
import pytest

import index_libs as il
import rescue_libs as rl
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu

ROOT = rl.ROOT
WARP_WINDOW = 78     # rescue_kernels.cuh kWarpWindow
SMEM_WINDOW = 2062   # the largest window whose table (2 * 2,048 slots) fits kSmemSlots


@pytest.fixture(scope="module")
def cm():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from genomeworks_b200 import cudamapper
    return cudamapper


def engine(cm, c, e, thr, **kw):
    f = cm.rescue_overlap_ends if c["mode"] == rl.RESCUE else cm.extend_overlaps_by_sequence_similarity
    return f(c["overlaps"], c["query_reads"], c["target_reads"], e, thr, **kw)


def against_oracle(cm, c, e, thr, **kw):
    got = engine(cm, c, e, thr, **kw)
    rc, want = rl.oracle_run(c["overlaps"], c["query_reads"], c["target_reads"], e, thr, c["mode"])
    assert rc == 0 and rl.ol.rows(got) == rl.ol.rows(want)
    return got


def test_engine_equals_stored_reference_outputs(cm):
    stored = rl.load_fixture()["cases"]
    for name, c in rl.cases().items():
        for p, (e, thr) in c["params"].items():
            assert rl.matches(engine(cm, c, e, thr), stored[name][p]), (name, p)


def switch_case(length, margin, divergence, seed):
    q, t, o = rl.diagonal_case(seed, 12, length, divergence, margin)
    return dict(query_reads=q, target_reads=t, overlaps=o, mode=rl.RESCUE)


@pytest.mark.parametrize("ext", [WARP_WINDOW, WARP_WINDOW + 1, SMEM_WINDOW, SMEM_WINDOW + 1, -1])
@pytest.mark.parametrize("divergence", [0.0, 0.01, 0.05])
def test_windows_at_each_path_switch_against_oracle(cm, ext, divergence):
    """Both ends of every overlap start with a window of exactly `ext` bases (the reads leave more room than that), or with the
    rest of the read for -1, which takes the global table."""
    c = switch_case(6000, (2100, 2400), divergence, 70 + int(divergence * 100))
    got = None
    for thr in (0.5, 0.8, rl.THIRD):
        got = against_oracle(cm, c, ext, thr)
        against_oracle(cm, dict(c, mode=rl.EXTEND_ONCE), ext, thr)
    if divergence == 0.0 and 0 < ext <= WARP_WINDOW + 1:
        # identical reads: each end moves by three windows
        assert np.all(c["overlaps"]["query_start_position_in_read"] - got["query_start_position_in_read"] == 3 * ext)


def test_whole_reads_with_long_windows_against_oracle(cm):
    c = switch_case(20000, (5000, 9000), 0.01, 77)
    for thr in (0.5, 0.9):
        against_oracle(cm, c, -1, thr)
        against_oracle(cm, c, 3000, thr)


def test_three_effective_rounds_on_identical_reads(cm):
    reads = il.random_reads(81, 4, 1000, 1000)
    o = rl.overlaps_array([rl.ov(i, i, 400, 600, 400, 600) for i in range(4)] + [rl.ov(0, 0, 120, 880, 120, 880)])
    got = cm.rescue_overlap_ends(o, reads, reads, 50, 0.5)
    assert got["query_start_position_in_read"].tolist() == [250] * 4 + [0]
    assert got["query_end_position_in_read"].tolist() == [750] * 4 + [1000]
    assert got["target_start_position_in_read"].tolist() == [250] * 4 + [0]
    once = cm.extend_overlaps_by_sequence_similarity(o, reads, reads, 50, 0.5)
    assert once["query_start_position_in_read"].tolist() == [350] * 4 + [70]


def test_pipeline_index_matcher_overlapper_rescue_against_oracle_chain(cm):
    reads = rl.genome_reads(91, 0.01, n_reads=120, genome_len=60000, lo=2000, hi=6000)
    idx = cm.create_index(reads, kmer_size=15, window_size=10)
    idx.wait_to_be_ready()
    m = cm.create_matcher(idx, idx)
    ov = cm.create_overlapper()
    got = cm.post_process_overlaps(ov.get_overlaps(m, True, 3, 250, 1000, 0.8))
    assert len(got) > 100
    assert (got["relative_strand"] == rl.REVERSE).any() and (got["relative_strand"] == rl.FORWARD).any()
    c = dict(query_reads=reads, target_reads=reads, overlaps=got, mode=rl.RESCUE)
    for p in ("cli", "strict", "unlimited", "ext1000"):
        res = against_oracle(cm, c, *rl.PARAMS[p])
    assert rl.ol.rows(res) != rl.ol.rows(got)
    for x in (ov, m, idx):
        x.close()


def test_rejections_leave_the_overlaps_unchanged(cm):
    from test_oracle_rescue import rejected_cases
    for name, (q, t, rows, mode) in rejected_cases().items():
        src = rl.overlaps_array(rows)
        keep = src.copy()
        al = CountingAllocator()
        f = cm.rescue_overlap_ends if mode == rl.RESCUE else cm.extend_overlaps_by_sequence_similarity
        with pytest.raises(ValueError):
            f(src, q, t, 50, 0.5, allocator=al)
        assert al.calls == 0 and rl.ol.rows(src) == rl.ol.rows(keep), name


def test_launch_count_independent_of_overlap_count(cm):
    from genomeworks_b200._lib import lib
    counts = []
    for n in (1, 30, 1000, 0):
        reads = rl.genome_reads(5, 0.01)
        rng = np.random.default_rng(n)
        o = rl.random_overlaps(rng, reads, reads, n)
        before = lib().gwb200_kernel_launch_count()
        cm.rescue_overlap_ends(o, reads, reads, 2000, 0.5)
        counts.append(lib().gwb200_kernel_launch_count() - before)
        if n:
            assert cm.rescue_last_kernel_ms() > 0
    assert counts == [2, 2, 2, 0], counts
    assert cm.rescue_last_kernel_ms() == -1.0  # nothing ran for n == 0


def test_allocator_balance_and_refusal(cm):
    c = switch_case(6000, (2100, 2400), 0.01, 99)
    al = CountingAllocator()
    got = cm.rescue_overlap_ends(c["overlaps"], c["query_reads"], c["target_reads"], -1, 0.5, allocator=al)
    assert al.calls == 2 and al.live == {}  # the staged inputs and the global tables
    rc, want = rl.oracle_run(c["overlaps"], c["query_reads"], c["target_reads"], -1, 0.5)
    assert rl.ol.rows(got) == rl.ol.rows(want)
    for refuse in (1, 2):
        bad = CountingAllocator(refuse)
        with pytest.raises(MemoryError):
            cm.rescue_overlap_ends(c["overlaps"], c["query_reads"], c["target_reads"], -1, 0.5, allocator=bad)
        assert bad.live == {}


def test_non_default_stream(cm):
    import torch
    s = torch.cuda.Stream()
    for seed in range(3):
        c = switch_case(3000, (0, 1500), 0.02, 200 + seed)
        against_oracle(cm, c, 50, 0.5, stream=s)
        against_oracle(cm, c, -1, 0.5, stream=s)


def test_cpp_rescue_api(cm):
    """The reference-named C++ API over create_kseq_fasta_parser and an in-memory parser: the unit test's known answer, the
    rejections (checked in the program) and the rescued overlaps, which must equal the oracle's."""
    exe = os.path.join(ROOT, "build", "test_cpp_rescue")
    r = subprocess.run([exe, rl.UNIT_FASTA], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr
    lines = r.stdout.split("\n")
    assert lines[-2] == "ok"
    got = [[int(v) for v in ln.split()[1:]] for ln in lines if ln.startswith("rescued ")]
    q, t = rl.unit_reads()
    reads = q + t
    v = rl.overlaps_array([rl.ov(0, 1, 1, 636, 341, 976), rl.ov(1, 0, 345, 970, 5, 630), rl.ov(0, 1, 100, 600, 200, 700, rl.REVERSE),
                           rl.ov(0, 0, 10, 990, 10, 990)])
    w = rl.overlaps_array([rl.ov(1, 0, 100, 500, 100, 500, rl.REVERSE), rl.ov(0, 0, 1, 636, 341, 976)])
    rc1, want_v = rl.oracle_run(v, reads, reads, 50, 0.5)
    rc2, want_w = rl.oracle_run(w, [q[0], rl.revcomp(t[0][:600])], t, -1, 0.5)
    assert rc1 == 0 and rc2 == 0
    assert got == rl.ol.rows(want_v) + rl.ol.rows(want_w)
