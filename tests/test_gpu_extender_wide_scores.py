"""The ungapped extender and the genome aligner on the GPU where scores pass 2^31 (DESIGN.md 9.1): both extender APIs against
the CPU oracle and the numpy restatement of tests/wide_score_libs.py on every CPU case, the 2^31 crossing placed at lane and
tile edges on both sides on the int32 and the int64 kernel, a mixed call of saturated and ordinary SSPs, one seed over two
identical records of 2^31 - 1 codes, the aligner in its three modes with a 2^24-scale matrix, and the chainer and the
skip-covered order on saturated scores."""
import time

import numpy as np
import pytest

import chain_all_libs as ca
import chain_libs as cl
import extender_libs as xl
import gapped_extender_libs as gl
import gapped_skip_libs as sk
import genome_aligner_libs as gal
import seeder_libs as sl
import wide_score_libs as wl

pytestmark = pytest.mark.gpu

INT32_MIN = -(1 << 31)
TOP = (1 << 32) - 1


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def run_both(ce, case):
    """(host-pointer result, device-pointer result) of one extender on a case, as SSP rows."""
    import torch
    ext = ce.create_extender(case["matrix"], case["xdrop"], no_entropy=case["no_entropy"])
    q, t, s = case["query"], case["target"], case["seeds"]
    assert ext.extend_async(q, t, case["threshold"], s) == ce.success and ext.sync() == ce.success
    host = xl.ssp_rows(ext.get_scored_segment_pairs())
    dq, dt = torch.from_numpy(q).cuda(), torch.from_numpy(t).cuda()
    ds = torch.from_numpy(np.ascontiguousarray(s).view(np.int32).reshape(-1, 2).copy()).cuda()
    out = torch.full((len(s), 4), -7, dtype=torch.int32, device="cuda")
    n = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    assert ext.extend_async_device(dq, dt, case["threshold"], ds, out, n) == ce.success
    torch.cuda.synchronize()
    dev = xl.ssp_rows(np.ascontiguousarray(out[:int(n.item())].cpu().numpy()).view(ce.SSP_DTYPE).reshape(-1))
    ext.close()
    return host, dev


def check_case(ce, case):
    want = wl.expected_run(case)
    oracle = xl.ssp_rows(xl.oracle_run(case["query"], case["target"], case["matrix"], case["xdrop"], case["no_entropy"],
                                       case["threshold"], case["seeds"]))
    assert oracle == want
    host, dev = run_both(ce, case)
    assert host == want, case["name"]
    assert dev == want, case["name"]
    return want


CPU_CASES = wl.cpu_cases()


@pytest.mark.parametrize("case", CPU_CASES, ids=[c["name"] for c in CPU_CASES])
def test_both_apis_equal_the_oracle_and_the_numpy_reference(ce, case):
    check_case(ce, case)


def crossing_case(v, side, xs):
    """One call whose seeds each see the running sum cross 2^31 at one of the offsets xs, on the right or the left side. Matrix:
    A/A scores 0, C/C, G/G and T/T score v, every mismatch -v; a block is mismatching flank, p zero-scoring A's and a run of
    C/G/T long enough to cross, placed so that the crossing falls on offset x."""
    rng = np.random.default_rng(v + len(side))
    m = wl.identity(v)
    m[0] = 0
    j = -(-(1 << 31) // v)  # the scoring positions that take the sum to 2^31 or past it
    q, t, pairs = [], [], []
    for x in xs:
        p = x - (j - 1) if side == "right" else x - j
        run = rng.integers(1, 4, j + 40).astype(np.int8)
        zeros = np.zeros(p, np.int8)
        fq = rng.integers(0, 4, 80).astype(np.int8)
        ft = ((fq + rng.integers(1, 4, 80)) % 4).astype(np.int8)
        at = sum(len(b) for b in q)
        if side == "right":  # the seed is the first A (or the run's first base); the left side mismatches at once
            body = np.concatenate([zeros, run])
            pairs.append((at + 40, at + 40))
        else:  # the seed mismatches; left of it come the A's, then the run
            body = np.concatenate([run, zeros])
            pairs.append((at + 40 + len(body), at + 40 + len(body)))
        q.append(np.concatenate([fq[:40], body, fq[40:]]))
        t.append(np.concatenate([ft[:40], body, ft[40:]]))
    return wl.case("cross_%s_%d" % (side, v), np.concatenate(q), np.concatenate(t), m, 910, 3000, True, pairs)


# v = 2^23 - 1 is the largest entry the int32 kernel takes (256 v <= INT32_MAX); 2^23 and 2^24 run on the int64 kernel
@pytest.mark.parametrize("v", [(1 << 23) - 1, 1 << 23, 1 << 24])
@pytest.mark.parametrize("side", ["right", "left"])
def test_crossing_at_lane_and_tile_edges(ce, v, side):
    j = -(-(1 << 31) // v)
    lo = j - 1 if side == "right" else j
    # right offsets: lanes start at 0 mod 4, steps at 0 mod 128; left offsets: at 1 mod 4 and 1 mod 128
    xs = [x for x in range(lo, lo + 300) if x % 4 in (0, 1, 3) and (x % 128 in (0, 1, 127) or x % 128 == 61 or x % 8 == 3)]
    case = crossing_case(v, side, xs)
    want = check_case(ce, case)
    assert len(want) == len(xs) and all(r[3] == wl.INT32_MAX for r in want)


@pytest.mark.parametrize("dip", [255, 256, 257])
def test_int32_kernel_carries_a_maximum_xdrop_above_the_sum_past_2_31(ce, dip):
    """v = 2^22, X-drop 2^30 (the int32 kernel): 600 matches (past 2^31), a dip of `dip` mismatches (255 v < 2^30 < 257 v;
    256 v = 2^30 is not more than it), then 300 matches that pass the first maximum when the dip did not stop the extension."""
    v = 1 << 22
    rng = np.random.default_rng(dip)
    a = rng.integers(0, 4, 600 + dip + 300).astype(np.int8)
    b = a.copy()
    b[600:600 + dip] = (b[600:600 + dip] + 1) % 4
    case = wl.case("dip_%d" % dip, b, a, wl.identity(v), 1 << 30, 3000, True, [(0, 0), (len(a) - 1, len(a) - 1)])
    want = check_case(ce, case)
    full = [0, 0, len(a) - 1, wl.INT32_MAX]
    assert (full in want) == (dip <= 256) and ([0, 0, 599, wl.INT32_MAX] in want) == (dip > 256)


def test_mixed_call_of_saturated_and_ordinary_ssps(ce):
    from genomeworks_b200 import synth
    target, query, seeds = synth.extender_workload(40000, 0.01, 4000, 0.3, seed=5)
    for xdrop in (910, 1 << 26):
        case = wl.case("mixed_%d" % xdrop, query, target, wl.identity(1 << 24), xdrop, 20 << 24, False, seeds)
        want = check_case(ce, case)
        scores = np.array([r[3] for r in want])
        assert (scores == wl.INT32_MAX).sum() >= 20 and (scores < wl.INT32_MAX).sum() >= 10


@pytest.mark.parametrize("v", [2, 1 << 24])
def test_one_seed_over_records_of_2_31_minus_1_codes(ce, v):
    """Query and target are one device buffer of 2^31 - 1 codes (ACGT repeated). A seed on the main diagonal extends over both
    whole records: total v (2^31 - 1), length 2^31 - 2, start 0. v = 2 runs the int32 kernel, 2^24 the int64 one."""
    import torch
    n = (1 << 31) - 1
    free, _ = torch.cuda.mem_get_info()
    if free < n + (512 << 20):
        pytest.skip("needs about %.1f GB of free device memory, the device has %.1f GB" % ((n + (512 << 20)) / 1e9, free / 1e9))
    seq = torch.arange(4, dtype=torch.int8, device="cuda").repeat(n // 4 + 1)[:n]
    ext = ce.create_extender(wl.identity(v), 910)
    ts = (1 << 30) + 12345
    ds = torch.tensor([[ts, ts]], dtype=torch.int32, device="cuda")
    out = torch.full((1, 4), -7, dtype=torch.int32, device="cuda")
    cnt = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    t0 = time.perf_counter()
    assert ext.extend_async_device(seq, seq, 3000, ds, out, cnt) == ce.success
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    assert int(cnt.item()) == 1
    assert out[0].tolist() == [0, 0, n - 1, min(v * n, wl.INT32_MAX)]
    assert ext.last_positions() == n
    print("one seed over 2 x (2^31 - 1) codes, v = %d: %.2f s" % (v, seconds))
    ext.close()
    del seq
    torch.cuda.empty_cache()


def aligner_records(n=3000):
    """One target; queries: the target itself and the reverse complement of a 1 %-diverged copy."""
    rng = np.random.default_rng(90)
    t = rng.integers(0, 4, n).astype(np.int8)
    hit = rng.random(n) < 0.01
    diverged = t.copy()
    diverged[hit] = (diverged[hit] + rng.integers(1, 4, int(hit.sum()))) % 4
    return [t], [t.copy(), sl.reverse_complement(diverged)]


class _AlignerTakingMatrix:
    """The cudaextender module as check_aligner uses it, with the aligner's score_matrix passed under the oracle's name, matrix."""

    def __init__(self, ce):
        self.format_paf = ce.format_paf
        self._ce = ce

    def GenomeAligner(self, strand, matrix, **kw):
        return self._ce.GenomeAligner(strand, score_matrix=matrix, **kw)


WIDE_ALIGNER = dict(matrix=wl.identity(1 << 24), ssp_threshold=wl.GATE_WRAP, gap_open=1 << 22, gap_extend=1 << 20, ydrop=1 << 28,
                    gapped_threshold=1 << 30)


@pytest.mark.parametrize("mode", ["default", "skip", "chain"])
def test_aligner_with_a_2_24_matrix(ce, mode):
    """An identical and a 1 %-diverged reverse-complement record of 3 kb, both strands, SSP threshold 715,827,883: the aligner
    equals its oracle composition, and the identical pair aligns over its whole length with score n * 2^24."""
    targets, queries = aligner_records()
    n = len(targets[0])
    rec = gal.check_aligner(_AlignerTakingMatrix(ce), targets, queries, "both", chain=(0, 0) if mode == "chain" else None,
                            skip=mode == "skip", **WIDE_ALIGNER)[0]
    whole = [r for r in rec if (int(r["query_record"]), int(r["strand"]), int(r["query_begin"]), int(r["query_end"]),
                                int(r["target_begin"]), int(r["target_end"])) == (0, 0, 0, n, 0, n)]
    assert len(whole) == 1 and int(whole[0]["score"]) == n << 24
    assert any(int(r["query_record"]) == 1 and int(r["strand"]) == 1 for r in rec)


def saturated_chain_set(rng, n, base):
    s = cl.random_ssps(rng, n, span=400, max_len=40, base=base)
    pick = rng.integers(0, 3, n)
    s["score"] = np.where(pick == 0, wl.INT32_MAX, np.where(pick == 1, INT32_MIN, s["score"]))
    return s


@pytest.mark.parametrize("n", [50, 700, 3000])
def test_chainer_on_saturated_scores_and_starts_near_the_top_of_uint32(ce, n):
    """The chaining DP and the all-chains extraction on the device against their oracles, with SSP scores at INT32_MAX and
    INT32_MIN and (for half the sets) starts within 400 of 2^32 - 1."""
    c = ce.create_ssp_chainer()
    rng = np.random.default_rng(n)
    for base in (0, TOP - 400):
        s = saturated_chain_set(rng, n, base)
        for D, A in ((0, 0), (1, 1), (1 << 20, 1 << 20)):
            idx, score = c.chain(s, diag_penalty=D, anti_penalty=A)
            f, p = c.get_dp()
            want = cl.oracle_run(s, D, A)
            assert np.array_equal(f, want["f"]) and np.array_equal(p, want["p"])
            assert np.array_equal(idx, cl.chain_indices(want)) and score == want["score"]
            for S in (ca.INT64_MIN, 0, wl.INT32_MAX):
                scores, offsets, members = c.chain_all(s, diag_penalty=D, anti_penalty=A, min_score=S)
                w = ca.oracle_all(s, D, A, S)
                assert np.array_equal(scores, w["scores"]) and np.array_equal(offsets, w["offsets"])
                assert np.array_equal(members, w["members"])
    c.close()


def test_skip_covered_order_falls_back_to_index_order_on_saturated_ties(ce):
    """SSPs of the 2^24 identity matrix on a 1 %-diverged pair, most of them at INT32_MAX: the device takes them in score order,
    ties in index order, as the skip-covered oracle does."""
    import torch
    from genomeworks_b200 import synth
    target, query, seeds = synth.extender_workload(20000, 0.01, 1500, 0.2, seed=8)
    case = wl.case("skip_ties", query, target, wl.identity(1 << 24), 910, 20 << 24, True, seeds)
    ssps = xl.oracle_run(case["query"], case["target"], case["matrix"], case["xdrop"], True, case["threshold"], case["seeds"])
    assert (ssps["score"] == wl.INT32_MAX).sum() >= 20 and (ssps["score"] < wl.INT32_MAX).sum() >= 5
    params = (case["matrix"], 1 << 22, 1 << 20, 1 << 28)
    want = sk.skip_run(query, target, *params, 1 << 30, gl.ssp_anchors(ssps), sk.ssp_order(ssps), 1 << 30)
    dq, dt = torch.from_numpy(np.ascontiguousarray(query, np.int8)).cuda(), torch.from_numpy(np.ascontiguousarray(target, np.int8)).cuda()
    x = ce.create_gapped_extender(*params, 1 << 30, skip_covered=True)
    assert x.extend_ssps_device(dq, dt, 1 << 30, xl.ssps_on_device(ssps), len(ssps)) == ce.success
    assert x.sync() == ce.success
    rec, cig = x.get_alignments()
    stats = x.last_skip_stats()
    x.close()
    assert gl.rows(rec) == gl.rows(want[0]) and cig == want[1]
    assert (stats["extended"], stats["skipped"]) == (want[3]["extended"], want[3]["skipped"]) and want[3]["skipped"] > 0
