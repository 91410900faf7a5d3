"""The extender stack on the GPU at the edges of its inputs, against the CPU oracles: asymmetric and random scoring schemes in
both extenders, an unpruned numpy DP for the gapped kernel, the parameter limits, ranges exactly at the chunk and ring widths,
best-cell and traceback ties across lane and chunk boundaries, anchors at the sequence ends, degenerate records in the seeder
and the genome aligner, and skip-covered anchors at the edges of a kept alignment. Every comparison is exact, and every CIGAR
re-scores to its score."""
import numpy as np
import pytest

import extender_edges_libs as el
import extender_libs as xl
import gapped_extender_libs as gl
import gapped_skip_libs as sk
import genome_aligner_libs as ga
import seeder_libs as sl

pytestmark = pytest.mark.gpu
NO_THRESHOLD = -(1 << 40)


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def gapped(ce, query, target, params, threshold, anchors, budget=1 << 30, ext=None):
    """(records, CIGARs, live cells) of one host-anchor call; params = (matrix, open, extend, y-drop)."""
    x = ext or ce.create_gapped_extender(*params, budget)
    assert x.extend_async(query, target, threshold, anchors) == ce.success
    assert x.sync() == ce.success
    rec, cig = x.get_alignments()
    out = rec, cig, x.last_live_cells()
    if ext is None:
        x.close()
    return out


def assert_gapped(got, want):
    assert gl.rows(got[0]) == gl.rows(want[0])
    assert got[1] == want[1]
    assert got[2] == want[2]


def assert_rescored(rec, cigars, query, target, params, anchors):
    mat, o, e, _ = params
    for r, cg in zip(rec, cigars):
        if not r["has_cigar"]:
            continue
        a = anchors[int(r["anchor"])]
        got = gl.rescore(cg, query, target, mat, o, e, int(r["query_begin"]), int(r["target_begin"]), (int(a["query"]), int(a["target"])))
        assert got == (int(r["score"]), int(r["query_end"] - r["query_begin"]), int(r["target_end"] - r["target_begin"]))


def check_gapped(ce, query, target, params, threshold, anchors, budget=1 << 30):
    """The engine equals the oracle, and every CIGAR re-scores; returns the engine's output."""
    got = gapped(ce, query, target, params, threshold, anchors, budget)
    assert_gapped(got, gl.oracle_run(query, target, *params, threshold, anchors, budget))
    assert_rescored(got[0], got[1], query, target, params, anchors)
    return got


def anchors_of(points):
    return np.array([tuple(int(v) for v in p) for p in points], dtype=gl.ANCHOR_DTYPE)


def ungapped_host(ce, ext, q, t, threshold, seeds):
    assert ext.extend_async(q, t, threshold, seeds) == ce.success and ext.sync() == ce.success
    return ext.get_scored_segment_pairs()


def ungapped_device(ce, ext, q, t, threshold, seeds):
    import torch
    dq = torch.from_numpy(np.ascontiguousarray(q, np.int8)).cuda()
    dt = torch.from_numpy(np.ascontiguousarray(t, np.int8)).cuda()
    s = np.ascontiguousarray(seeds, dtype=ce.SEED_DTYPE)
    ds = torch.from_numpy(np.concatenate([s, np.zeros(1, dtype=ce.SEED_DTYPE)]).view(np.int32).reshape(-1, 2).copy()).cuda()
    out = torch.full((len(s) + 1, 4), -7, dtype=torch.int32, device="cuda")
    n = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    assert ext.extend_async_device(dq, dt, threshold, ds, out, n, num_seed_pairs=len(s)) == ce.success
    torch.cuda.synchronize()
    return np.ascontiguousarray(out[:int(n.item())].cpu().numpy()).view(ce.SSP_DTYPE).reshape(-1)


# 1. Asymmetric and random scoring schemes

def test_hand_asymmetric_matrix_on_the_device(ce):
    cs, as_ = np.full(10, 1, np.int8), np.full(10, 0, np.int8)
    anchor = anchors_of([(5, 5)])
    params = (el.HAND_MATRIX, 3, 1, 50)
    assert gl.rows(gapped(ce, cs, as_, params, 0, anchor)[0]) == [(50, 0, 1, 0, 10, 0, 10)]
    assert gl.rows(gapped(ce, as_, cs, params, 0, anchor)[0]) == [(0, 0, 1, 5, 5, 5, 5)]
    ext = ce.create_extender(el.HAND_MATRIX, 20, no_entropy=True)
    for run in (ungapped_host, ungapped_device):
        assert xl.ssp_rows(run(ce, ext, cs, as_, 1, anchor)) == [[0, 0, 9, 50]]
        assert len(run(ce, ext, as_, cs, 1, anchor)) == 0
    ext.close()


def homologous(rng, n_target, n_query):
    """A random target and a query taken from it with substitutions, indels and bytes outside 0..3, of about n_query bases."""
    t = rng.integers(0, 4, n_target).astype(np.int8)
    q = sl.mutate(t[:n_query], 0.08, rng)
    return el.with_odd_bytes(q, rng), el.with_odd_bytes(t, rng)


def random_anchors(rng, qlen, tlen, n):
    k = rng.integers(0, min(qlen, tlen), n)
    pts = [(int(v), int(min(v + rng.integers(-3, 4), tlen - 1))) for v in k[: n // 2]]
    pts += [(int(rng.integers(0, qlen)), int(rng.integers(0, tlen))) for _ in range(n - n // 2)]
    return anchors_of([(q, max(t, 0)) for q, t in pts])


@pytest.mark.parametrize("seed", range(4))
def test_random_asymmetric_schemes_in_the_gapped_extender(ce, seed):
    rng = np.random.default_rng(1000 + seed)
    q, t = homologous(rng, 1300, 900)
    if seed == 3:  # the hand matrix, doubled, with matches among A/C/G/T
        mat = el.HAND_MATRIX * 2
        mat[[0, 9, 18, 27]] = 12
    else:
        mat = el.asymmetric_matrix(rng)
    assert (mat.reshape(8, 8) != mat.reshape(8, 8).T).any()
    for o, e in ((0, 3), (4, 0), (6, 2)):
        for y in (0, 1, 60, 400):
            for query, target in ((q, t), (t, q)):
                anchors = random_anchors(rng, len(query), len(target), 24)
                check_gapped(ce, query, target, (mat, o, e, y), NO_THRESHOLD, anchors)


@pytest.mark.parametrize("seed", range(3))
def test_random_asymmetric_schemes_in_the_ungapped_extender(ce, seed):
    rng = np.random.default_rng(2000 + seed)
    q, t = homologous(rng, 6000, 4000)
    mat = el.asymmetric_matrix(rng, scale=10)
    for query, target in ((q, t), (t, q)):
        seeds = random_anchors(rng, len(query), len(target), 2000)
        for xdrop, thr in ((0, 1), (1, 30), (300, 200)):
            for no_entropy in (False, True):
                ext = ce.create_extender(mat, xdrop, no_entropy=no_entropy)
                want = xl.ssp_rows(xl.oracle_run(query, target, mat, xdrop, no_entropy, thr, seeds))
                assert xl.ssp_rows(ungapped_host(ce, ext, query, target, thr, seeds)) == want
                assert xl.ssp_rows(ungapped_device(ce, ext, query, target, thr, seeds)) == want
                ext.close()


# 2. An independent reference: the unpruned numpy DP

def test_gapped_scores_equal_the_numpy_dp(ce):
    rng = np.random.default_rng(3000)
    cases = 0
    for _ in range(60):
        mat = el.asymmetric_matrix(rng)
        o, e = int(rng.integers(0, 8)), int(rng.integers(0, 4))
        params = (mat, o, e, 1 << 28)
        x = ce.create_gapped_extender(*params)
        for _ in range(5):
            ml, nl, mr, nr = (int(v) for v in rng.integers(0, 31, 4))
            q = rng.integers(-128, 128, ml + mr + 1).astype(np.int8)
            t = rng.integers(-128, 128, nl + nr + 1).astype(np.int8)
            anchor = anchors_of([(ml, nl)])
            rec, cig, _ = gapped(ce, q, t, params, NO_THRESHOLD, anchor, ext=x)
            assert int(rec[0]["score"]) == el.numpy_score(q, t, (ml, nl), mat, o, e)
            assert_rescored(rec, cig, q, t, params, anchor)
            cases += 1
        x.close()
    assert cases == 300


# 3. Parameter limits

def test_limit_cases_equal_the_numpy_dp_and_the_oracle(ce):
    for q, t, anchor, mat, o, e in el.limit_cases():
        a = anchors_of([anchor])
        got = check_gapped(ce, q, t, (mat, o, e, 1 << 28), NO_THRESHOLD, a)
        assert int(got[0][0]["score"]) == el.numpy_score(q, t, anchor, mat, o, e)


def test_scores_past_2_31_and_long_gap_runs_at_the_limits(ce):
    big = 1 << 24
    rng = np.random.default_rng(4000)
    s = rng.integers(0, 4, 4096).astype(np.int8)
    # a 10-base deletion and a 12-base insertion: gap runs of 11 and 13 times 2^24, within a y-drop of 2^28
    q = np.concatenate([s[:1000], s[1010:2000], rng.integers(0, 4, 12).astype(np.int8), s[2000:]])
    ident = np.where(np.eye(8, dtype=bool), big, -big).astype(np.int32).ravel()
    anchors = anchors_of([(500, 500), (3000, 2988), (0, 0), (len(q) - 1, len(s) - 1)])
    asym = rng.integers(-big, big // 4, 64).astype(np.int32)
    asym[[0, 9, 18, 27]] = big
    asym[[1, 8]] = big // 2, -big
    for mat in (ident, asym):
        for o, e, y in ((big, big, 1 << 28), (big, 0, 1 << 28), (0, big, 1 << 28), (400, 30, 1 << 28), (big, big, 3 * big)):
            got = check_gapped(ce, q, s, (mat, o, e, y), NO_THRESHOLD, anchors)
            if mat is ident and (o, e, y) == (big, big, 1 << 28):
                assert int(got[0]["score"].max()) > 1 << 31
                assert any("10D" in c and "12I" in c for c in got[1])


def test_parameters_at_the_limits_are_accepted_and_one_past_refused(ce):
    big = 1 << 24
    mat = np.full(64, big, dtype=np.int64)
    mat[::2] = -big
    ce.create_gapped_extender(mat, big, big, 1 << 28).close()
    for kw in (dict(gap_open=big + 1), dict(gap_extend=big + 1), dict(ydrop=(1 << 28) + 1), dict(gap_open=-1), dict(gap_extend=-1),
               dict(ydrop=-1)):
        args = dict(score_matrix=mat, gap_open=big, gap_extend=big, ydrop=1 << 28)
        args.update(kw)
        with pytest.raises(ValueError):
            ce.create_gapped_extender(**args)
    for v in (big + 1, -big - 1):
        m = mat.copy()
        m[17] = v
        with pytest.raises(ValueError):
            ce.create_gapped_extender(m, 1, 1, 1)


# 4. Widths at the chunk and ring edges

def test_widths_at_the_chunk_and_ring_edges_in_one_call(ce):
    query, target, anchors, widths = el.width_case()
    params = el.WIDTH_PARAMS
    sides = [gl.oracle_side(query, target, *params, int(a["query"]), int(a["target"]), left, trace=False)
             for a in anchors for left in (True, False)]
    assert [s["width"] for s in sides] == [w for pair in widths for w in pair]
    want = gl.oracle_run(query, target, *params, NO_THRESHOLD, anchors)
    got = gapped(ce, query, target, params, NO_THRESHOLD, anchors)
    assert_gapped(got, want)
    # anchors 0 and 1 give the same whole-diagonal alignment: the duplicate rule keeps the first
    assert len(got[0]) == len(anchors) - 1 and all(int(h) == 1 for h in got[0]["has_cigar"])
    assert_rescored(got[0], got[1], query, target, params, anchors)
    # a budget of the largest alignment: pass 2 in rounds of one or a few alignments, each with its own ring size
    budget = max(sides[2 * k]["storage"] + sides[2 * k + 1]["storage"] for k in range(len(anchors)))
    assert_gapped(gapped(ce, query, target, params, NO_THRESHOLD, anchors, budget=budget), want)


# 5. Ties

@pytest.mark.parametrize("p", el.TIE_PS)
def test_best_cell_ties_across_lane_and_chunk_boundaries(ce, p):
    query, target = el.tie_case(p)
    params = el.TIE_PARAMS
    got = check_gapped(ce, query, target, params, NO_THRESHOLD, anchors_of([(0, 0)]))
    assert gl.rows(got[0]) == [(10 * p + 8, 0, 1, 0, p + 1, 0, p + 2)]
    # the same tie on the left side of an anchor, and with the roles of query and target swapped
    q2, t2 = np.concatenate([query[::-1], [3]]).astype(np.int8), np.concatenate([target[::-1], [3]]).astype(np.int8)
    check_gapped(ce, q2, t2, params, NO_THRESHOLD, anchors_of([(len(query), len(target))]))
    check_gapped(ce, target, query, params, NO_THRESHOLD, anchors_of([(0, 0)]))


ASYMMETRIC_TIE_MATRIX = xl.SIMPLE_MATRIX.copy()
ASYMMETRIC_TIE_MATRIX[[2 * 8 + 0, 3 * 8 + 1, 1 * 8 + 3, 0 * 8 + 5]] = [-3, 4, -15, 2]


@pytest.mark.parametrize("case", el.periodic_cases(), ids=lambda c: c[0])
def test_low_complexity_repeats_tie_everywhere(ce, case):
    _, q, t, anchors = case
    for mat in (xl.SIMPLE_MATRIX, ASYMMETRIC_TIE_MATRIX):
        for o, e, y in ((1, 1, 3000), (0, 2, 100), (3, 0, 40)):
            check_gapped(ce, q, t, (mat, o, e, y), NO_THRESHOLD, anchors)
            check_gapped(ce, t, q, (mat, o, e, y), NO_THRESHOLD, anchors_of([(b, a) for a, b in anchors]))


# 6. Sequence-end geometry

def test_anchors_at_the_four_corners(ce):
    rng = np.random.default_rng(5000)
    q, t = homologous(rng, 530, 500)
    m, n = len(q), len(t)
    anchors = anchors_of([(0, 0), (0, n - 1), (m - 1, 0), (m - 1, n - 1)])
    for params in ((xl.SIMPLE_MATRIX, 5, 2, 80), (el.asymmetric_matrix(rng), 1, 0, 1000)):
        check_gapped(ce, q, t, params, NO_THRESHOLD, anchors)
        check_gapped(ce, t, q, params, NO_THRESHOLD, anchors_of([(b, a) for a, b in anchors]))


def test_one_base_against_a_hundred_thousand(ce):
    rng = np.random.default_rng(5001)
    long = rng.integers(0, 4, 100000).astype(np.int8)
    one = np.array([2], dtype=np.int8)
    # open 1, extend 0: a gap of any length costs 1, so every side runs to the far end of the long sequence
    for params in ((xl.SIMPLE_MATRIX, 1, 0, 50), (xl.SIMPLE_MATRIX, 5, 2, 80)):
        check_gapped(ce, one, long, params, NO_THRESHOLD, anchors_of([(0, 0), (0, 50000), (0, 99999)]))
        check_gapped(ce, long, one, params, NO_THRESHOLD, anchors_of([(0, 0), (50000, 0), (99999, 0)]))


def test_ssp_midpoints_on_the_last_base(ce):
    import torch
    rng = np.random.default_rng(5002)
    q, t = homologous(rng, 3001, 2999)
    m, n = len(q), len(t)
    ssps = np.array([(m - 5, n - 5, 9, 50), (m - 4, n - 4, 7, 40), (m - 1, n - 1, 1, 10), (m - 1, n - 1, 0, 5), (0, 0, 1, 10),
                     (0, n - 1, 0, 5), (m - 1, 0, 1, 5), (m - 9, n - 5, 8, 30)], dtype=xl.SSP_DTYPE)
    params = (xl.SIMPLE_MATRIX, 5, 2, 80)
    anchors = gl.ssp_anchors(ssps)
    assert (int(anchors["query"].max()), int(anchors["target"].max())) == (m - 1, n - 1)
    dq = torch.from_numpy(np.ascontiguousarray(q, np.int8)).cuda()
    dt = torch.from_numpy(np.ascontiguousarray(t, np.int8)).cuda()
    x = ce.create_gapped_extender(*params)
    assert x.extend_ssps_device(dq, dt, NO_THRESHOLD, xl.ssps_on_device(ssps), len(ssps)) == ce.success and x.sync() == ce.success
    got = x.get_alignments() + (x.last_live_cells(),)
    x.close()
    assert_gapped(got, gl.oracle_run(q, t, *params, NO_THRESHOLD, anchors))
    assert_rescored(got[0], got[1], q, t, params, anchors)


# 7. Seeder and genome aligner on degenerate records

def seeds_of(ce, seeder, query, target):
    return seeder.seed_pairs(np.ascontiguousarray(query, np.int8), np.ascontiguousarray(target, np.int8))


def assert_seeds(got, want):
    assert len(got) == len(want)
    assert np.array_equal(got["query"], want["query"]) and np.array_equal(got["target"], want["target"])


@pytest.mark.parametrize("transition", [True, False])
def test_seeder_on_short_and_all_n_records(ce, transition):
    rng = np.random.default_rng(6000)
    base = rng.integers(0, 4, 20).astype(np.int8)
    s = ce.create_seeder(transition)
    for lq in (0, 1, 18, 19, 20):
        for lt in (0, 1, 18, 19, 20):
            q, t = base[:lq], base[:lt]
            want = sl.oracle_run(q, t, transition)
            assert_seeds(seeds_of(ce, s, q, t), want)
            if lq >= 19 and lt >= 19:
                assert (18, 18) in set(zip(want["query"].tolist(), want["target"].tolist()))
    n = np.full(300, 5, dtype=np.int8)
    for q, t in ((n, n), (n, np.resize(base, 300)), (np.resize(base, 300), n)):
        assert len(seeds_of(ce, s, q, t)) == 0 == len(sl.oracle_run(q, t, transition))
    s.close()


@pytest.mark.parametrize("transition", [True, False])
def test_seeder_with_odd_bytes_in_every_seed_position(ce, transition):
    rng = np.random.default_rng(6001)
    base = rng.integers(0, 4, 60).astype(np.int8)
    s = ce.create_seeder(transition)
    bytes_ = np.array([4, 5, 6, 7, 8, 11, 12, 127, -1, -125, -128], dtype=np.int8)
    for pos in range(19):
        for k, b in enumerate(bytes_):
            q = base.copy()
            q[20 + pos] = b
            q[(45 + pos + k) % 60] = bytes_[(k + 3) % len(bytes_)]
            for query, target in ((q, base), (base, q)):
                want = sl.oracle_run(query, target, transition)
                assert_seeds(seeds_of(ce, s, query, target), want)
    s.close()


def degenerate_records(rng):
    shared = rng.integers(0, 4, 4000).astype(np.int8)
    targets = [shared[:3000].copy(), np.zeros(0, np.int8), rng.integers(0, 4, 1).astype(np.int8), shared[100:118].copy(),
               shared[200:219].copy(), np.full(300, 5, np.int8), rng.integers(0, 4, 2500).astype(np.int8),
               sl.reverse_complement(shared[1000:4000])]
    queries = [sl.mutate(shared[500:3500], 0.03, rng), np.zeros(0, np.int8), shared[100:101].copy(), shared[100:118].copy(),
               shared[200:219].copy(), np.full(257, 5, np.int8), rng.integers(0, 4, 1200).astype(np.int8)]
    return targets, queries


@pytest.mark.parametrize("strand", ["both", "plus", "minus"])
def test_aligner_on_degenerate_records(ce, strand):
    targets, queries = degenerate_records(np.random.default_rng(7000))
    rec = ga.check_aligner(ce, targets, queries, strand)[0]
    assert len(rec) > 0
    if strand == "both":
        assert {int(v) for v in rec["strand"]} == {0, 1}
        ga.check_aligner(ce, targets[:3], queries, strand, transition=False)


def test_aligner_on_forty_tiny_records_by_three(ce):
    rng = np.random.default_rng(7001)
    shared = rng.integers(0, 4, 600).astype(np.int8)
    targets = [shared, sl.reverse_complement(shared[:300]), np.full(25, 5, np.int8)]
    queries = [shared[k * 13:k * 13 + k].copy() for k in range(40)]
    rec = ga.check_aligner(ce, targets, queries, "both", ssp_threshold=100, gapped_threshold=100)[0]
    assert len(rec) > 0


def test_minus_strand_mapping_at_an_odd_length(ce):
    rng = np.random.default_rng(7002)
    t = rng.integers(0, 4, 5001).astype(np.int8)
    q = sl.reverse_complement(t[1000:3001])  # 2001 bases, the minus strand of target[1000, 3001)
    q[[0, 1, 2, 1000, 1001, 1997, 1998, 1999, 2000]] = [4, 5, 6, 7, 4, 5, 6, 7, 4]
    rec = ga.check_aligner(ce, [t], [q], "both")[0]
    assert len(q) % 2 == 1 and (rec["strand"] == 1).any()


# 8. Skip-covered mode at the edges of a run

def edge_anchors(rec, cigar):
    """Points on a kept alignment: its first and last M cells, one past its end, and cells inside its I and D runs."""
    q, t = int(rec["query_begin"]), int(rec["target_begin"])
    m_cells, gap_cells = [], []
    for n, op in gl.cigar_ops(cigar):
        if op == "M":
            m_cells += [(q + k, t + k) for k in range(n)]
        elif op == "I":
            gap_cells += [(q + k, t) for k in range(n)]
        else:
            gap_cells += [(q, t + k) for k in range(n)]
        q += 0 if op == "D" else n
        t += 0 if op == "I" else n
    return [m_cells[0], m_cells[-1], m_cells[len(m_cells) // 2], (q, t)] + gap_cells[:3] + gap_cells[-2:]


def skip_case():
    """Query and target with homologous pieces near the far positive extreme of the diagonals, on diagonal 0, on a positive and
    on a negative diagonal, and host anchors: each piece's anchor, then anchors on the edges of the alignment it gives, then
    the corners."""
    rng = np.random.default_rng(8000)
    t = rng.integers(0, 4, 5000).astype(np.int8)
    tlen = len(t)
    pieces = [t[-60:], t[60:400], rng.integers(0, 4, 300).astype(np.int8), sl.mutate(t[2000:2600], 0.04, rng),
              rng.integers(0, 4, 100).astype(np.int8), sl.mutate(t[300:900], 0.04, rng)]
    starts = np.cumsum([0] + [len(p) for p in pieces])
    q = np.concatenate(pieces)
    qlen = len(q)
    first = [(10, tlen - 50), (200, 200), (int(starts[3]) + 3, 2003), (int(starts[5]) + 3, 303)]
    params = (xl.SAMPLE_MATRIX, gl.LASTZ_OPEN, gl.LASTZ_EXTEND, gl.LASTZ_YDROP)
    pts = []
    for a in first:
        rec, cig, _ = gl.oracle_run(q, t, *params, gl.LASTZ_THRESHOLD, anchors_of([a]))
        assert len(rec) == 1 and "M" in cig[0]
        pts += [a] + [p for p in edge_anchors(rec[0], cig[0]) if p[0] < qlen and p[1] < tlen]
    pts += [(0, tlen - 1), (qlen - 1, 0), (0, 0)]
    return q, t, params, anchors_of(pts)


def test_skip_covered_at_the_edges_of_a_run(ce):
    q, t, params, anchors = skip_case()
    diags = {int(a["target"]) - int(a["query"]) for a in anchors}
    assert min(diags) < 0 and 0 in diags and max(diags) == len(t) - 1
    want = sk.skip_run(q, t, *params, gl.LASTZ_THRESHOLD, anchors)
    assert want[3]["skipped"] > 0
    for k in (1, 0):
        x = ce.create_gapped_extender(*params, skip_covered=True, round_anchors=k)
        assert x.extend_async(q, t, gl.LASTZ_THRESHOLD, anchors) == ce.success and x.sync() == ce.success
        rec, cig = x.get_alignments()
        stats = x.last_skip_stats()
        assert gl.rows(rec) == gl.rows(want[0]) and cig == want[1] and x.last_live_cells() == want[2]
        assert (stats["extended"], stats["skipped"]) == (want[3]["extended"], want[3]["skipped"])
        x.close()
