"""Every chain above a minimum score (DESIGN.md section 20) on the GPU: the chainer against the DP oracle and the extract oracle --
f, p, scores, offsets, members, union and score sum -- on the golden sample's SSPs, random sets around the tile size, a ladder,
an anti-diagonal, a comb and backbone sets up to 10^6; the handle's reuse, a C++ caller; and the genome aligner in this mode
against the oracle composition (seeder -> ungapped -> chain -> extract -> gapped or skip-covered)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import chain_all_libs as ca
import chain_libs as cl
import extender_libs as xl
import genome_aligner_libs as ga
import seeder_libs as sl
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 1024  # chain_kernels.cuh kTile
TOP = 1 << 20
LO, HI = ca.INT64_MIN, (1 << 63) - 1
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


def run_all(c, ssps, D=0, A=0, S=LO):
    scores, offsets, members = c.chain_all(ssps, diag_penalty=D, anti_penalty=A, min_score=S)
    f, p = c.get_dp()
    union, total = c.get_chain()
    return {"f": f, "p": p, "scores": scores, "offsets": offsets, "members": members, "union": union, "sum": total}


def assert_same(got, want):
    for k in ("f", "p", "scores", "offsets", "members", "union"):
        assert np.array_equal(got[k], want[k]), k
    assert got["sum"] == want["sum"]


def assert_oracle(got, ssps, D=0, A=0, S=LO):
    want = ca.oracle_all(ssps, D, A, S)
    assert_same(got, want)
    return want


def assert_extract_on_device_dp(got, ssps, D=0, A=0, S=LO):
    """The extract oracle on the device's own f and p, for sizes the O(n^2) DP oracle is too slow for."""
    want = ca.oracle_extract(ssps, D, A, got["f"], got["p"], S)
    want.update(f=got["f"], p=got["p"], union=ca.union(want), sum=int(want["scores"].sum()))
    assert_same(got, want)
    return want


def chains(res):
    o = res["offsets"]
    return [res["members"][o[c]:o[c + 1]] for c in range(len(res["scores"]))]


def golden_strands():
    seq, _, plus = xl.sample()
    rc = sl.reverse_complement(seq)
    minus = xl.oracle_run(rc, seq, xl.SAMPLE_MATRIX, xl.SAMPLE_XDROP, False, xl.SAMPLE_THRESHOLD, sl.oracle_run(rc, seq))
    return plus, minus


def test_golden_sample_ssps_both_strands(chainer):
    for ssps in golden_strands():
        for D, A in ((0, 0), (1, 1)):
            for S in (LO, 0, 10000, 30000, HI):
                want = assert_oracle(run_all(chainer, ssps, D, A, S), ssps, D, A, S)
                if S == LO:
                    assert len(want["scores"]) > 1 and len(want["union"]) == len(ssps)


@pytest.mark.parametrize("n", [0, 1, 2, K - 1, K, K + 1, 2 * K + 1, 3 * K + 5])
def test_random_sets(chainer, n):
    rng = np.random.default_rng(900 + n)
    for D, A in PENALTIES:
        ssps = cl.random_ssps(rng, n, span=max(50, 4 * n), max_len=60)
        for S in (LO, 0, 100):
            got = run_all(chainer, ssps, D, A, S)
            assert_oracle(got, ssps, D, A, S)
        # the first candidate is section 19's chain
        best = cl.oracle_run(ssps, D, A)
        got = run_all(chainer, ssps, D, A, best["score"] if n else 0)
        assert n == 0 or (np.array_equal(chains(got)[0], cl.chain_indices(best)) and got["scores"][0] == best["score"])


def test_ladder_is_one_chain(chainer):
    ssps = cl.ladder(10 ** 4)
    got = run_all(chainer, ssps)
    assert len(got["scores"]) == 1 and got["scores"][0] == 100 * 10 ** 4 and np.array_equal(got["members"], np.arange(10 ** 4))
    assert_oracle(got, ssps)


def test_anti_diagonal_is_single_chains_in_index_order(chainer):
    n = 10 ** 4
    ssps = cl.anti_diagonal(n)
    got = run_all(chainer, ssps)
    assert (got["scores"] == 100).all() and np.array_equal(got["offsets"], np.arange(n + 1)) and np.array_equal(got["members"], np.arange(n))
    assert_oracle(got, ssps)
    got = run_all(chainer, ssps, S=101)
    assert len(got["scores"]) == 0 and len(got["union"]) == 0 and got["sum"] == 0


def comb(n):
    """A trunk of n colinear SSPs (f rising by 100) and at every trunk SSP i a side SSP whose best predecessor is trunk SSP i and
    whose f beats trunk SSP i + 1: the last side SSP's chain takes the whole trunk, every other side SSP is a chain of one."""
    s = np.zeros(2 * n, dtype=xl.SSP_DTYPE)
    i = np.arange(n)
    s["query"][:n], s["target"][:n], s["length"][:n], s["score"][:n] = i * 100, i * 100, 30, 100
    s["query"][n:], s["target"][n:], s["length"][n:], s["score"][n:] = i * 100 + 40, 10 ** 7 - i * 100, 10, 150
    return s


def test_comb(chainer):
    n = 10 ** 4
    ssps = comb(n)
    got = run_all(chainer, ssps)
    want = assert_oracle(got, ssps)
    assert got["p"][n + 5] == 5 and len(want["scores"]) == n
    assert np.array_equal(chains(got)[0], np.concatenate([np.arange(n), [2 * n - 1]])) and got["scores"][0] == 100 * n + 150
    assert (got["scores"][1:] == 150).all()
    assert_oracle(run_all(chainer, ssps, S=151), ssps, S=151)


@pytest.mark.parametrize("n", [10 ** 5, 10 ** 6])
def test_backbone_sets(chainer, n):
    rng = np.random.default_rng(31)
    ssps = cl.backbone_set(rng, n, n // 10)
    for S in (LO, 30000):
        got = run_all(chainer, ssps, 0, 0, S)
        if n <= 10 ** 5 and S == LO:
            # f and p against the DP's equations on the device; the best chain is the first candidate
            order = np.argsort(-got["f"], kind="stable")
            walk = [int(order[0])]
            while got["p"][walk[-1]] >= 0:
                walk.append(int(got["p"][walk[-1]]))
            cl.check_contract_on_device(ssps, 0, 0, got["f"], got["p"], np.sort(walk).astype(np.int32), int(got["f"][order[0]]))
        want = assert_extract_on_device_dp(got, ssps, 0, 0, S)
        assert len(want["scores"]) > 1


def test_chain_after_chain_all_and_reuse(ce):
    import torch
    from genomeworks_b200._lib import lib
    stream = torch.cuda.Stream()
    alloc = CountingAllocator()
    c = ce.create_ssp_chainer(stream=stream, allocator=alloc)
    rng = np.random.default_rng(8)
    ssps = cl.random_ssps(rng, 2 * K + 9, span=5000, max_len=60)
    for _ in range(2):
        assert_oracle(run_all(c, ssps, 1, 2, 50), ssps, 1, 2, 50)
        # chain() on the same handle gives exactly section 19's result, and reports it as one chain
        idx, score = c.chain(ssps, diag_penalty=1, anti_penalty=2)
        want = cl.oracle_run(ssps, 1, 2)
        assert np.array_equal(idx, cl.chain_indices(want)) and score == want["score"]
        scores, offsets, members = c.get_chains()
        assert list(scores) == [score] and list(offsets) == [0, len(idx)] and np.array_equal(members, idx)
        assert np.array_equal(c.get_dp()[0], want["f"])
    # n = 0 after either call: no chain
    assert [len(x) for x in c.chain_all(ssps[:0])] == [0, 1, 0] and [len(x) for x in c.get_chains()] == [0, 1, 0]
    c.chain(ssps[:0])
    assert [len(x) for x in c.get_chains()] == [0, 1, 0]
    # a CUDA tensor and a raw device address give the host array's result
    dev = xl.ssps_on_device(ssps)
    torch.cuda.synchronize()
    want = ca.oracle_all(ssps, 0, 0, 40)
    assert_same(run_all(c, dev, 0, 0, 40), want)
    got = c.chain_all(dev.data_ptr(), n=700, min_score=40)
    want = ca.oracle_all(ssps[:700], 0, 0, 40)
    assert all(np.array_equal(g, want[k]) for g, k in zip(got, ("scores", "offsets", "members")))
    # a second call while one is pending is invalid_operation; sync finishes the first
    L = lib()
    assert L.gwb200_ssp_chainer_chain_all_device(c._h, C.c_void_p(dev.data_ptr()), len(ssps), 0, 0, LO) == ce.success
    assert L.gwb200_ssp_chainer_chain_all_device(c._h, C.c_void_p(dev.data_ptr()), len(ssps), 0, 0, LO) == ce.invalid_operation
    assert L.gwb200_ssp_chainer_chain_device(c._h, C.c_void_p(dev.data_ptr()), len(ssps), 0, 0) == ce.invalid_operation
    assert L.gwb200_ssp_chainer_sync(c._h) == ce.success
    c._n = len(ssps)
    want = ca.oracle_all(ssps)
    got = c.get_chains()
    assert np.array_equal(c.get_dp()[1], want["p"]) and all(np.array_equal(g, want[k]) for g, k in zip(got, ("scores", "offsets", "members")))
    # a bad length is refused at sync, and the handle stays usable
    bad = ssps.copy()
    bad["length"][17] = -2
    with pytest.raises(ValueError):
        c.chain_all(bad)
    with pytest.raises(RuntimeError):
        c.get_chains()
    with pytest.raises(TypeError):
        c.chain_all(ssps, min_score=1.5)
    with pytest.raises(ValueError):
        c.chain_all(ssps, min_score=HI + 1)
    assert_oracle(run_all(c, ssps, 0, 0, HI), ssps, 0, 0, HI)
    assert alloc.calls > 0 and len(alloc.live) > 0
    c.close()
    assert alloc.live == {}


CPP = r"""
#include <claraparabricks/genomeworks/cudaextender/chainer.hpp>
#include <claraparabricks/genomeworks/utils/allocator.hpp>
#include <cstdio>
#include <vector>
using namespace claraparabricks::genomeworks;
using namespace claraparabricks::genomeworks::cudaextender;
int main()
{
    // two disjoint ladders and a side SSP: chains {0, 1, 2} (150) and {3, 4} (80); {5} (30) is below the minimum
    const int rows[6][4] = {{0, 1000, 10, 50}, {20, 1020, 10, 50}, {40, 1040, 10, 50}, {1000, 0, 10, 40}, {1020, 20, 10, 40}, {22, 1022, 10, 30}};
    std::vector<ScoredSegmentPair> h(6);
    for (int k = 0; k < 6; ++k)
    {
        h[k].start_coord.query_position_in_read  = rows[k][0];
        h[k].start_coord.target_position_in_read = rows[k][1];
        h[k].length                              = rows[k][2];
        h[k].score                               = rows[k][3];
    }
    ScoredSegmentPair* d = nullptr;
    cudaMalloc(reinterpret_cast<void**>(&d), sizeof(ScoredSegmentPair) * 6);
    cudaMemcpy(d, h.data(), sizeof(ScoredSegmentPair) * 6, cudaMemcpyHostToDevice);
    DefaultDeviceAllocator alloc = create_default_device_allocator(1ull << 26);
    std::unique_ptr<SspChainer> c = create_ssp_chainer(nullptr, 0, alloc);
    if (c->chain_all_device(d, 6, 0, 0, 50) != success || c->sync() != success)
        return 1;
    std::vector<int64_t> scores, offsets;
    const std::vector<int32_t> members = c->get_chains(scores, offsets);
    int64_t total = 0;
    const std::vector<int32_t> all = c->get_chain(total);
    std::printf("%zu %lld %lld %lld %lld %lld %zu %lld\n", scores.size(), (long long)scores[0], (long long)scores[1], (long long)offsets[0],
                (long long)offsets[1], (long long)offsets[2], all.size(), (long long)total);
    for (int32_t m : members)
        std::printf("%d ", m);
    std::printf("\n");
    if (c->chain_device(d, 6, 0, 0) != success || c->sync() != success)
        return 1;
    c->get_chains(scores, offsets);
    std::printf("%zu %lld %lld\n", scores.size(), (long long)scores[0], (long long)offsets[1]);
    c.reset();
    cudaFree(d);
    std::printf("CHAIN_ALL_CPP_OK\n");
    return 0;
}
"""


def test_cpp_caller(ce, tmp_path):
    src, exe = tmp_path / "chain_all.cpp", str(tmp_path / "chain_all")
    src.write_text(CPP)
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src), "-o", exe,
                           "-L", os.path.join(ROOT, "genomeworks_b200"), "-lgwb200", "-L", "/usr/local/cuda/lib64", "-lcudart",
                           "-Wl,-rpath," + os.path.join(ROOT, "genomeworks_b200"), "-Wl,-rpath,/usr/local/cuda/lib64"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "CHAIN_ALL_CPP_OK" in out.stdout, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[0] == "2 150 80 0 3 5 5 230" and lines[1].split() == ["0", "1", "2", "3", "4"] and lines[2] == "1 150 3"


# ---- the genome aligner ----

def test_aligner_golden_sample(ce):
    seq, _, _ = xl.sample()
    best = ce.GenomeAligner(chain=True)
    best_rec, _ = best.run([seq], [seq])
    best_stats = best.last_chain_stats()
    best.close()
    for S in (30000, 10 ** 6):
        rec, _, _, stats = ca.check_aligner(ce, [seq], [seq], chain=(0, 0), min_chain_score=S)
        assert stats["pairs"] == 2
        if S == 30000:
            assert (rec["strand"] == 1).any() and stats["ssps_chained"] > best_stats["ssps_chained"] and len(rec) > len(best_rec)


def test_aligner_inversion_pair_and_records(ce):
    target, query, _ = sl.rearranged_pair(5)
    rec = ca.check_aligner(ce, [target], [query], chain=(0, 0), min_chain_score=30000)[0]
    assert (rec["strand"] == 1).any()
    targets, queries = ga.records_case()
    want = ca.check_aligner(ce, targets, queries, chain=(1, 1), min_chain_score=5000)
    assert want[3]["pairs"] >= 3
    # blocks of 7 seeds give the same output
    got = ca.check_aligner(ce, targets, queries, chain=(1, 1), min_chain_score=5000, block_size=7)
    assert ga.engine_rows(got[0]) == ga.engine_rows(want[0]) and got[1] == want[1]
    # with skip-covered mode too
    ca.check_aligner(ce, targets, queries, chain=(0, 0), skip=True, min_chain_score=5000)


def test_lowest_minimum_is_chaining_off(ce):
    targets, queries = ga.records_case()
    seq, _, _ = xl.sample()
    for t, q in ((targets, queries), ([seq], [seq])):
        off = ce.align_genomes(t, q)
        al = ce.GenomeAligner(chain=True, min_chain_score=LO)
        got = al.run(t, q)
        stats = al.last_chain_stats()
        al.close()
        assert ga.engine_rows(got[0]) == ga.engine_rows(off[0]) and got[1] == off[1]
        assert stats["ssps_chained"] == stats["ssps_in"] > 0


def test_all_chains_run_then_default_runs_on_one_handle(ce):
    targets, queries = ga.records_case()
    al = ce.GenomeAligner(chain=True, min_chain_score=5000)
    al.run(targets, queries)
    assert al.last_chain_count() >= 3
    al.set_chain(None)
    rec, cigars = al.run(targets, queries)
    assert al.last_chain_count() == 0 and al.last_chain_stats()["pairs"] == 0
    off = ce.align_genomes(targets, queries)
    assert ga.engine_rows(rec) == ga.engine_rows(off[0]) and cigars == off[1]
    al.set_chain(True)
    rec, cigars = al.run(targets, queries)
    one = ce.align_genomes(targets, queries, chain=True)
    assert ga.engine_rows(rec) == ga.engine_rows(one[0]) and cigars == one[1]
    assert al.last_chain_count() == al.last_chain_stats()["pairs"]
    al.close()


def repeat_case():
    """A 60 kb target holding eight copies of a 400-base repeat outside a 20 kb block; the query is the block diverged by 3 %,
    behind one more copy of the repeat."""
    rng = np.random.default_rng(41)
    target = rng.integers(0, 4, 60000).astype(np.int8)
    rep = rng.integers(0, 4, 400).astype(np.int8)
    spots = [1000 + 5000 * k for k in range(4)] + [42000 + 4000 * k for k in range(4)]
    for s in spots:
        target[s:s + 400] = rep
    block = (21000, 41000)
    query = np.concatenate([rng.integers(0, 4, 3000).astype(np.int8), rep, rng.integers(0, 4, 3000).astype(np.int8),
                            sl.mutate(target[block[0]:block[1]], 0.03, rng)])
    return target, query, spots, block


def test_block_survives_and_isolated_repeat_hits_do_not(ce):
    target, query, spots, block = repeat_case()

    def on_repeat(rec):
        return [r for r in rec if any(s - 1000 <= r["target_begin"] and r["target_end"] <= s + 1400 for s in spots)]

    def on_block(rec):
        return [r for r in rec if r["target_begin"] < block[1] and r["target_end"] > block[0] and r["target_end"] - r["target_begin"] > 10000]

    off, _ = ce.align_genomes([target], [query], strand="plus")
    assert len(on_repeat(off)) >= 6 and on_block(off)
    S = 100000
    rec, _, _, stats = ca.check_aligner(ce, [target], [query], strand="plus", chain=(0, 0), min_chain_score=S)
    assert on_block(rec) and len(on_repeat(rec)) <= 1
    assert stats["ssps_chained"] < stats["ssps_in"]


def test_tool_prints_the_same_paf(ce, tmp_path):
    targets, queries = ga.records_case()
    for opts, chain, S in ((["--chain", "--chain-min-score=5000"], True, 5000), (["--chain-min-score=-9223372036854775808", "--chain=3,2"], (3, 2), LO)):
        rec, cigars = ce.align_genomes(targets, queries, chain=chain, min_chain_score=S)
        want = ga.tool_paf(ce, rec, cigars, targets, queries)
        out = ga.run_tool(tmp_path, targets, queries, *opts)
        assert out.returncode == 0, out.stderr
        assert out.stdout == want and want
