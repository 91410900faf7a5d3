"""The SSP chainer (DESIGN.md section 19) on the GPU against its CPU oracle -- f, p, the chain and its score -- on the golden
sample's SSPs, random sets on both sides of the tile sizes, ladders, anti-diagonals, planted ties and the penalty limits; and the
genome aligner with chaining against the oracle composition (seeder -> ungapped -> chain -> gapped or skip-covered), in records,
CIGARs, PAF and chain stats."""
import ctypes as C

import numpy as np
import pytest

import chain_libs as cl
import extender_libs as xl
import genome_aligner_libs as ga
import seeder_libs as sl
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu
K = 1024  # chain_kernels.cuh kTile
TOP = 1 << 20
PENALTIES = [(0, 0), (1, 1), (TOP, TOP), (1, 0), (0, TOP)]


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


@pytest.fixture(scope="module")
def chainer(ce):
    c = ce.create_ssp_chainer()
    yield c
    c.close()


def run(c, ssps, D=0, A=0):
    idx, score = c.chain(ssps, diag_penalty=D, anti_penalty=A)
    f, p = c.get_dp()
    return {"f": f, "p": p, "chain": idx, "score": score}


def assert_oracle(got, ssps, D=0, A=0):
    want = cl.oracle_run(ssps, D, A)
    assert np.array_equal(got["f"], want["f"])
    assert np.array_equal(got["p"], want["p"])
    assert np.array_equal(got["chain"], cl.chain_indices(want))
    assert got["score"] == want["score"]
    return want


def golden_strands():
    seq, _, plus = xl.sample()
    rc = sl.reverse_complement(seq)
    minus = xl.oracle_run(rc, seq, xl.SAMPLE_MATRIX, xl.SAMPLE_XDROP, False, xl.SAMPLE_THRESHOLD, sl.oracle_run(rc, seq))
    return plus, minus


def test_golden_sample_ssps_both_strands(chainer):
    for ssps in golden_strands():
        for D, A in ((0, 0), (1, 1)):
            want = assert_oracle(run(chainer, ssps, D, A), ssps, D, A)
            assert len(want["chain"]) > 1


@pytest.mark.parametrize("n", [0, 1, 2, K - 1, K, K + 1, 2 * K + 1, 3 * K + 5])
def test_random_sets(chainer, n):
    rng = np.random.default_rng(500 + n)
    for D, A in PENALTIES:
        ssps = cl.random_ssps(rng, n, span=max(50, 4 * n), max_len=60)
        got = run(chainer, ssps, D, A)
        assert_oracle(got, ssps, D, A)
        assert (n == 0) == (len(got["chain"]) == 0)


def test_random_sets_of_10e5_against_the_contract(chainer):
    # the O(n^2) oracle needs about a minute per set here, so the contract's equations are checked on the device instead
    rng = np.random.default_rng(9)
    n = 10 ** 5
    for D, A in ((0, 0), (1, 1)):
        for ssps in (cl.backbone_set(rng, n, 2000), cl.random_ssps(rng, n, span=10 ** 5, max_len=100, scores=(-50, 500))):
            got = run(chainer, ssps, D, A)
            # 256 x 10^5 int64 per temporary, about 1.5 GB in all
            cl.check_contract_on_device(ssps, D, A, got["f"], got["p"], got["chain"], got["score"], rows_per_step=256)


def test_colinear_ladder_is_one_chain(chainer):
    ssps = cl.ladder(10 ** 4)
    got = run(chainer, ssps)
    assert np.array_equal(got["chain"], np.arange(10 ** 4)) and got["score"] == 100 * 10 ** 4
    assert_oracle(got, ssps)
    # a shuffled ladder chains the same SSPs
    perm = np.random.default_rng(4).permutation(10 ** 4)
    got = run(chainer, ssps[perm])
    assert np.array_equal(np.sort(perm[got["chain"]]), np.arange(10 ** 4)) and got["score"] == 100 * 10 ** 4


def test_anti_diagonal_is_one_ssp(chainer):
    ssps = cl.anti_diagonal(10 ** 4)
    got = run(chainer, ssps)
    assert list(got["chain"]) == [0] and got["score"] == 100 and (got["p"] == -1).all()
    assert_oracle(got, ssps)


def test_ties_planted_across_tile_boundaries(chainer):
    # a pool of 40 distinct SSPs, each repeated at indices spread over four tiles: equal f values and equal-value predecessors
    # at ranks on both sides of every tile and chunk boundary
    rng = np.random.default_rng(12)
    pool = cl.random_ssps(rng, 40, span=400, max_len=20, scores=(10, 12))
    ssps = pool[rng.integers(0, 40, 4 * K + 3)]
    for D, A in PENALTIES:
        want = assert_oracle(run(chainer, ssps, D, A), ssps, D, A)
        assert (want["p"] >= 0).any()
    # identical ladders in the two halves: every link has a twin of equal value one tile away
    half = cl.ladder(K + 7, step=20, length=5, score=9)
    ssps = np.concatenate([half, half])
    got = run(chainer, ssps)
    assert_oracle(got, ssps)
    assert np.array_equal(got["chain"], np.arange(K + 7))


def test_reuse_with_a_stream_and_an_allocator(ce):
    import torch
    from genomeworks_b200._lib import lib
    stream = torch.cuda.Stream()
    alloc = CountingAllocator()
    c = ce.create_ssp_chainer(stream=stream, allocator=alloc)
    rng = np.random.default_rng(3)
    for n in (5, 3 * K + 5, 0, 700, 2 * K):
        ssps = cl.random_ssps(rng, n, span=4 * n + 50)
        assert_oracle(run(c, ssps, 1, 2), ssps, 1, 2)
    # a CUDA tensor and a raw device address give the same result
    ssps = cl.random_ssps(rng, 900, span=3000)
    dev = xl.ssps_on_device(ssps)
    torch.cuda.synchronize()
    want = cl.oracle_run(ssps)
    assert np.array_equal(c.chain(dev)[0], cl.chain_indices(want))
    assert np.array_equal(c.chain(dev.data_ptr(), n=600)[0], cl.chain_indices(cl.oracle_run(ssps[:600])))
    # a second call while one is pending is invalid_operation; sync finishes the first
    L = lib()
    assert L.gwb200_ssp_chainer_chain_device(c._h, C.c_void_p(dev.data_ptr()), 900, 0, 0) == ce.success
    assert L.gwb200_ssp_chainer_chain_device(c._h, C.c_void_p(dev.data_ptr()), 900, 0, 0) == ce.invalid_operation
    assert L.gwb200_ssp_chainer_sync(c._h) == ce.success
    assert L.gwb200_ssp_chainer_sync(c._h) == ce.invalid_operation
    c._n = 900
    assert np.array_equal(c.get_dp()[0], want["f"]) and c.last_ms() >= 0
    # a length below -1 is refused at sync, and the handle stays usable
    bad = ssps.copy()
    bad["length"][17] = -2
    with pytest.raises(ValueError):
        c.chain(bad)
    with pytest.raises(RuntimeError):
        c.get_chain()
    with pytest.raises(ValueError):
        c.chain(ssps, diag_penalty=TOP + 1)
    assert_oracle(run(c, ssps), ssps)
    assert alloc.calls > 0 and len(alloc.live) > 0
    c.close()
    assert alloc.live == {}


def test_aligner_golden_sample(ce):
    seq, _, _ = xl.sample()
    default, _ = ce.align_genomes([seq], [seq])
    for chain in ((0, 0), (2, 1)):
        rec, _, _, stats = ga.check_aligner(ce, [seq], [seq], chain=chain)
        assert (rec["strand"] == 1).any() and stats["pairs"] == 2
        assert stats["ssps_chained"] < stats["ssps_in"] and len(rec) < len(default)


def test_aligner_inversion_pair_and_records(ce):
    target, query, _ = sl.rearranged_pair(5)
    rec = ga.check_aligner(ce, [target], [query], chain=(0, 0))[0]
    assert (rec["strand"] == 1).any()
    targets, queries = ga.records_case()
    want = ga.check_aligner(ce, targets, queries, chain=(0, 0))
    assert want[3]["pairs"] >= 3
    # blocks of 7 seeds give the same output
    got = ga.check_aligner(ce, targets, queries, chain=(0, 0), block_size=7)
    assert ga.engine_rows(got[0]) == ga.engine_rows(want[0]) and got[1] == want[1]


def test_aligner_chain_with_skip_covered(ce):
    targets, queries = ga.records_case()
    ga.check_aligner(ce, targets, queries, chain=(1, 1), skip=True)
    seq, _, _ = xl.sample()
    ga.check_aligner(ce, [seq], [seq], chain=(0, 0), skip=True)


def test_chained_run_then_default_run_on_one_handle(ce):
    targets, queries = ga.records_case()
    al = ce.GenomeAligner(chain=True)
    chained = al.run(targets, queries)
    al.set_chain(None)
    rec, cigars = al.run(targets, queries)
    assert al.last_chain_stats() == {"ssps_in": 0, "ssps_chained": 0, "pairs": 0, "chain_ms": 0.0}
    al.close()
    rows, want_cigars, _, _ = ga.aligner_oracle(targets, queries)
    assert ga.engine_rows(rec) == rows and cigars == want_cigars
    assert len(chained[0]) <= len(rec)


def test_tool_chain_prints_the_same_paf(ce, tmp_path):
    targets, queries = ga.records_case()
    for opt, chain in (("--chain", True), ("--chain=3,2", (3, 2))):
        rec, cigars = ce.align_genomes(targets, queries, chain=chain)
        want = ga.tool_paf(ce, rec, cigars, targets, queries)
        out = ga.run_tool(tmp_path, targets, queries, opt)
        assert out.returncode == 0, out.stderr
        assert out.stdout == want and want
