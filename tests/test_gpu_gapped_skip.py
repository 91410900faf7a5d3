"""The skip-covered mode (DESIGN.md section 18) on the GPU against its CPU oracle: records, their order, CIGARs, has_cigar, live
cells and the extended / skipped counts, for the gapped extender and the genome aligner; round sizes, budgets and block sizes
do not change the output, and the mode does not leak into later default calls."""
import numpy as np
import pytest

import extender_libs as xl
import gapped_extender_libs as gl
import gapped_skip_libs as sk
import genome_aligner_libs as ga
import seeder_libs as sl
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu
LASTZ = (xl.SAMPLE_MATRIX, gl.LASTZ_OPEN, gl.LASTZ_EXTEND, gl.LASTZ_YDROP)


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def finish(x, ce):
    assert x.sync() == ce.success
    rec, cig = x.get_alignments()
    return rec, cig, x.last_live_cells(), x.last_skip_stats()


def run_host(ce, query, target, params, threshold, anchors, budget=1 << 30, round_anchors=0, ext=None):
    x = ext or ce.create_gapped_extender(*params, budget, skip_covered=True, round_anchors=round_anchors)
    assert x.extend_async(query, target, threshold, anchors) == ce.success
    out = finish(x, ce)
    if ext is None:
        x.close()
    return out


def run_ssps(ce, seq_q, seq_t, params, threshold, ssps, budget=1 << 30, round_anchors=0):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(seq_q, np.int8)).cuda()
    dt = torch.from_numpy(np.ascontiguousarray(seq_t, np.int8)).cuda()
    ds = xl.ssps_on_device(ssps)
    x = ce.create_gapped_extender(*params, budget, skip_covered=True, round_anchors=round_anchors)
    assert x.extend_ssps_device(dq, dt, threshold, ds, len(ssps)) == ce.success
    out = finish(x, ce)
    x.close()
    return out


def assert_equal(got, want, n):
    rec, cig, live, stats = got
    assert gl.rows(rec) == gl.rows(want[0])
    assert cig == want[1]
    assert live == want[2]
    assert (stats["extended"], stats["skipped"]) == (want[3]["extended"], want[3]["skipped"])
    assert stats["extended"] + stats["skipped"] == n and 0 <= stats["speculative"] <= stats["skipped"]
    assert stats["traced"] >= int(rec["has_cigar"].sum()) and (stats["rounds"] > 0) == (n > 0)


def golden():
    seq, _, ssps = xl.sample()
    return seq, ssps


def test_golden_sample_ssps_on_the_device(ce):
    seq, ssps = golden()
    want = sk.skip_run(seq, seq, *LASTZ, gl.LASTZ_THRESHOLD, gl.ssp_anchors(ssps), sk.ssp_order(ssps))
    assert want[3]["skipped"] > 0
    got = run_ssps(ce, seq, seq, LASTZ, gl.LASTZ_THRESHOLD, ssps)
    assert_equal(got, want, len(ssps))
    # the same call in rounds of 1 and 7 anchors
    for k in (1, 7):
        assert_equal(run_ssps(ce, seq, seq, LASTZ, gl.LASTZ_THRESHOLD, ssps, round_anchors=k), want, len(ssps))


def test_host_anchors_in_the_ssp_order_equal_the_device_call(ce):
    seq, ssps = golden()
    order = sk.ssp_order(ssps)
    dev = run_ssps(ce, seq, seq, LASTZ, gl.LASTZ_THRESHOLD, ssps)
    host = run_host(ce, seq, seq, LASTZ, gl.LASTZ_THRESHOLD, gl.ssp_anchors(ssps)[order])
    rec = host[0].copy()
    rec["anchor"] = order[rec["anchor"]]
    assert gl.rows(rec) == gl.rows(dev[0]) and host[1:] == dev[1:]


@pytest.mark.parametrize("n", [0, 1, 7, 1001])
@pytest.mark.parametrize("divergence", [0.0, 0.15, 0.3])
def test_synthetic_anchors_against_the_oracle(ce, n, divergence):
    from genomeworks_b200 import synth
    target, query, seeds = synth.extender_workload(5000, divergence, n, 0.3, seed=100 + n)
    for params, threshold in ((LASTZ, gl.LASTZ_THRESHOLD), ((xl.SIMPLE_MATRIX, 5, 2, 80), 0)):
        want = sk.skip_run(query, target, *params, threshold, seeds)
        assert_equal(run_host(ce, query, target, params, threshold, seeds), want, n)
        if n == 1001:
            assert want[3]["skipped"] > 0
            assert_equal(run_host(ce, query, target, params, threshold, seeds, round_anchors=7), want, n)


def test_range_wider_than_the_shared_ring(ce):
    rng = np.random.default_rng(8)
    s = rng.integers(0, 4, 6000).astype(np.int8)
    q = s.copy()
    q[rng.random(6000) < 0.1] = 4
    a = np.array([(3000, 3000), (0, 0), (5999, 5999), (1500, 1500)], dtype=gl.ANCHOR_DTYPE)
    params = (xl.SIMPLE_MATRIX, 1, 0, 3000)
    want = sk.skip_run(q, s, *params, -(1 << 40), a)
    assert want[2] > 10 ** 7
    assert_equal(run_host(ce, q, s, params, -(1 << 40), a), want, len(a))
    assert_equal(run_host(ce, q, s, params, -(1 << 40), a, round_anchors=1), want, len(a))


def test_budgets_that_force_many_trace_rounds_or_no_cigar(ce):
    target, query, seeds = gl.synthetic()
    full = sk.skip_run(query, target, *LASTZ, gl.LASTZ_THRESHOLD, seeds)
    sizes = [sum(gl.oracle_side(query, target, *LASTZ, int(seeds[k]["query"]), int(seeds[k]["target"]), side, trace=False)["storage"]
                 for side in (True, False)) for k in full[0]["anchor"]]
    for budget in (max(sizes), sorted(sizes)[len(sizes) // 2], 0):
        want = sk.skip_run(query, target, *LASTZ, gl.LASTZ_THRESHOLD, seeds, budget=budget)
        if budget == 0:
            assert int(want[0]["has_cigar"].sum()) == 0 and want[3]["skipped"] == 0
        for k in (0, 7):
            assert_equal(run_host(ce, query, target, LASTZ, gl.LASTZ_THRESHOLD, seeds, budget, round_anchors=k), want, len(seeds))


def test_mode_does_not_leak_and_allocator_balances(ce):
    target, query, seeds = gl.synthetic(400, 41)
    default = gl.oracle_run(query, target, *LASTZ, gl.LASTZ_THRESHOLD, seeds)
    alloc = CountingAllocator()
    x = ce.create_gapped_extender(*LASTZ, allocator=alloc, skip_covered=True, round_anchors=5)
    got = run_host(ce, query, target, LASTZ, gl.LASTZ_THRESHOLD, seeds, ext=x)
    assert_equal(got, sk.skip_run(query, target, *LASTZ, gl.LASTZ_THRESHOLD, seeds), len(seeds))
    x.set_skip_covered(False)
    assert x.extend_async(query, target, gl.LASTZ_THRESHOLD, seeds) == ce.success
    # the mode cannot change while a call is pending
    with pytest.raises(RuntimeError):
        x.set_skip_covered(True)
    rec, cig, live, stats = finish(x, ce)
    assert gl.rows(rec) == gl.rows(default[0]) and cig == default[1] and live == default[2]
    assert stats == {"extended": len(seeds), "skipped": 0, "speculative": 0, "traced": int(rec["has_cigar"].sum()), "rounds": 1}
    assert alloc.calls > 0 and len(alloc.live) > 0
    x.close()
    assert alloc.live == {}


def test_aligner_golden_sample_both_strands(ce):
    seq, _ = golden()
    rec, _, stats, _ = ga.check_aligner(ce, [seq], [seq], skip=True)
    assert (rec["strand"] == 1).any() and stats["skipped"] > 0
    default, _ = ce.align_genomes([seq], [seq])
    assert len(rec) <= len(default)


def test_aligner_inversion_pair_and_records(ce):
    target, query, _ = sl.rearranged_pair(5)
    rec, _, _, _ = ga.check_aligner(ce, [target], [query], skip=True)
    assert (rec["strand"] == 1).any()
    targets, queries = ga.records_case()
    want = ga.check_aligner(ce, targets, queries, skip=True)
    # blocks of 7 seeds and rounds of 7 anchors give the same output
    got = ga.check_aligner(ce, targets, queries, skip=True, block_size=7, round_anchors=7)
    assert ga.engine_rows(got[0]) == ga.engine_rows(want[0]) and got[1] == want[1]
    # the rule's counts do not depend on the rounds; speculative and rounds describe the grouping itself
    assert all(got[2][k] == want[2][k] for k in ("extended", "skipped", "traced"))


def test_tool_skip_covered_prints_the_same_paf(ce, tmp_path):
    targets, queries = ga.records_case()
    rec, cigars = ce.align_genomes(targets, queries, skip_covered=True)
    want = ga.tool_paf(ce, rec, cigars, targets, queries)
    out = ga.run_tool(tmp_path, targets, queries, "--skip-covered")
    assert out.returncode == 0, out.stderr
    assert out.stdout == want and want
