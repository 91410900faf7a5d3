"""The genome aligner with its records packed into groups (DESIGN.md section 21) on the GPU: against its oracle composition at
group sizes of 1, one that splits the record list and the default, identical output and stats across group sizes in every
mode, strand, seed setting and block size, homology that runs across a record boundary, boundary records, the group stats
against a restatement of the grouping rule, the tool's --group-bases, and a handle reused across group sizes with a stream
and an allocator."""
import ctypes as C

import numpy as np
import pytest

import genome_aligner_libs as ga
import extender_libs as xl
import seeder_libs as sl
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu

SPLIT = 4096  # splits every many-record case below into several groups per side
MODES = {"default": {}, "skip": dict(skip_covered=True), "chain": dict(chain=(0, 0)), "chains": dict(chain=(0, 0), min_chain_score=3000)}


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def slot(n):
    return (n + 16) & ~15


def groups(records, group_bases):
    """The grouping rule of DESIGN.md section 21.1: records in order, each in a slot of its length + 1 rounded up to 16; a
    group takes records while its slots total at most group_bases, and a record whose slot alone is larger forms its own."""
    out, used = [], 0
    for k, r in enumerate(records):
        if used > 0 and used + slot(len(r)) > group_bases:
            used = 0
        if used == 0:
            out.append([])
        out[-1].append(k)
        used += slot(len(r))
    return out


def gapped_pairs(targets, queries, strand, **params):
    """(record pair, strand)s whose unique SSPs are not empty in the oracle composition."""
    p = dict(ga.DEFAULTS, **params)
    n = 0
    for t in targets:
        for q in queries:
            for s in ga.STRANDS[strand]:
                q8 = np.asarray(q, np.int8)
                n += len(ga.ungapped_ssps(sl.reverse_complement(q8) if s else q8, np.asarray(t, np.int8), p)) > 0
    return n


def contigs(seed, n_targets=24, n_queries=9):
    """A genome cut into contigs as the target side, and diverged pieces of it, some reverse-complemented and some spanning
    contig ends, as the query side; plus unrelated records on both sides."""
    rng = np.random.default_rng(seed)
    genome = rng.integers(0, 4, 30000).astype(np.int8)
    cuts = np.sort(rng.choice(np.arange(200, 29800), n_targets - 1, replace=False))
    targets = [genome[a:b].copy() for a, b in zip(np.r_[0, cuts], np.r_[cuts, 30000])]
    queries = []
    for k in range(n_queries):
        n = int(rng.integers(800, 4000))
        s = int(rng.integers(0, 30000 - n))
        piece = sl.mutate(genome[s:s + n], 0.03, rng)
        queries.append(sl.reverse_complement(piece) if k % 3 == 1 else piece)
    targets.insert(5, rng.integers(0, 4, 1500).astype(np.int8))
    queries.insert(2, rng.integers(0, 4, 700).astype(np.int8))
    return targets, queries


def everything(ce, targets, queries, strand="both", group_bases=None, **kw):
    """(rows, CIGARs, counts, skip stats, chain stats without the time, chain count, group stats) of one aligner run."""
    extra = {} if group_bases is None else dict(group_bases=group_bases)
    al = ce.GenomeAligner(strand, **extra, **kw)
    rec, cigars = al.run(targets, queries)
    chain_stats = al.last_chain_stats()
    chain_stats.pop("chain_ms")
    out = (ga.engine_rows(rec), cigars, al.last_stats()[1], al.last_skip_stats(), chain_stats, al.last_chain_count(), al.last_group_stats())
    al.close()
    return out


def assert_same_at_every_group_size(ce, targets, queries, strand="both", sizes=(SPLIT, None), **kw):
    """Runs at group size 1 and at each of `sizes` (None: the default) and asserts every output and stat but the group stats
    equal. -> the runs."""
    runs = [everything(ce, targets, queries, strand, 1, **kw)] + [everything(ce, targets, queries, strand, g, **kw) for g in sizes]
    for r in runs[1:]:
        assert r[:-1] == runs[0][:-1]
        assert r[-1]["gapped_pairs"] == runs[0][-1]["gapped_pairs"]
    return runs


def assert_group_stats(ce, targets, queries, group_bases, strand="both", **params):
    al = ce.GenomeAligner(strand, group_bases=group_bases, **params)
    al.run(targets, queries)
    st = al.last_group_stats()
    al.close()
    assert st == dict(target_groups=len(groups(targets, group_bases)), query_groups=len(groups(queries, group_bases)),
                      gapped_pairs=gapped_pairs(targets, queries, strand, **params))


@pytest.mark.parametrize("group_bases", [1, SPLIT, None])
def test_records_case_against_the_oracle(ce, group_bases):
    targets, queries = ga.records_case()
    extra = {} if group_bases is None else dict(group_bases=group_bases)
    rec = ga.check_aligner(ce, targets, queries, **extra)[0]
    assert set(zip(rec["target_record"].tolist(), rec["query_record"].tolist())) >= {(0, 0), (2, 0), (1, 1)}
    assert_group_stats(ce, targets, queries, group_bases or ce.DEFAULT_GROUP_BASES)


def test_golden_sample_in_groups_of_one(ce):
    seq, _, _ = xl.sample()
    ga.check_aligner(ce, [seq], [seq], group_bases=1)


@pytest.mark.parametrize("group_bases", [1, SPLIT, 20000, None])
def test_contigs_against_the_oracle(ce, group_bases):
    targets, queries = contigs(11)
    assert len(groups(targets, SPLIT)) > 3 and len(groups(queries, SPLIT)) > 3 and len(groups(targets, 20000)) > 1
    extra = {} if group_bases is None else dict(group_bases=group_bases)
    rec = ga.check_aligner(ce, targets, queries, **extra)[0]
    assert {0, 1} <= set(rec["strand"].tolist()) and len({(int(r["target_record"]), int(r["query_record"])) for r in rec}) > 5
    assert_group_stats(ce, targets, queries, group_bases or ce.DEFAULT_GROUP_BASES)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("strand", ["both", "plus", "minus"])
def test_every_mode_and_strand_is_identical_across_group_sizes(ce, mode, strand):
    targets, queries = contigs(12)
    runs = assert_same_at_every_group_size(ce, targets, queries, strand, **MODES[mode])
    assert len(runs[0][0]) > 0
    if mode == "chain":
        ga.check_aligner(ce, targets, queries, strand, chain=(0, 0), group_bases=SPLIT)
    if mode == "skip":
        ga.check_aligner(ce, targets, queries, strand, skip=True, group_bases=SPLIT)


@pytest.mark.parametrize("kw", [dict(transition=False), dict(block_size=7), dict(block_size=1000)], ids=["exact", "B7", "B1000"])
def test_seed_setting_and_block_size_do_not_change_the_output(ce, kw):
    targets, queries = contigs(13, 12, 5)
    assert len(assert_same_at_every_group_size(ce, targets, queries, **kw)[0][0]) > 0


def boundary_case(rng, equal_cut):
    """Two homologous sequences, each cut into two records; the cut points are the same or 300 bases apart."""
    a = rng.integers(0, 4, 3000).astype(np.int8)
    b = sl.mutate(a, 0.02, rng)
    tcut, qcut = 1400, 1400 if equal_cut else 1700
    return [a[:tcut].copy(), a[tcut:].copy()], [b[:qcut].copy(), b[qcut:].copy()]


@pytest.mark.parametrize("equal_cut", [True, False])
def test_homology_across_a_record_boundary(ce, equal_cut):
    targets, queries = boundary_case(np.random.default_rng(21 + equal_cut), equal_cut)
    for g in (1, 64, None):
        extra = {} if g is None else dict(group_bases=g)
        rec = ga.check_aligner(ce, targets, queries, **extra)[0]
        assert len(rec) > 0
        # no alignment passes a record end
        for r in rec:
            assert r["target_end"] <= len(targets[r["target_record"]]) and r["query_end"] <= len(queries[r["query_record"]])


@pytest.mark.parametrize("equal_cut", [True, False])
def test_only_the_record_bounds_stop_a_matrix_that_scores_everything(ce, equal_cut):
    # every code pair, separators included, scores +100: an extension that ran past a record end would keep gaining
    targets, queries = boundary_case(np.random.default_rng(31 + equal_cut), equal_cut)
    targets = [t[:700] for t in targets]
    queries = [q[:600] for q in queries]
    params = dict(score_matrix=np.full(64, 100, np.int32), matrix=np.full(64, 100, np.int32), xdrop=1 << 30, ydrop=1 << 28)
    engine = {k: v for k, v in params.items() if k != "matrix"}
    runs = assert_same_at_every_group_size(ce, targets, queries, "plus", sizes=(64, None), **engine)
    rows, _, _, _ = ga.aligner_oracle(targets, queries, "plus", **{k: v for k, v in params.items() if k != "score_matrix"})
    assert runs[0][0] == rows and len(rows) > 0


def odd_byte_records(rng):
    """Records whose first and last bases are bytes 4-127 or negative, and records that are copies of one another, so the
    diagonals of different record pairs collide inside a group."""
    base = rng.integers(0, 4, 900).astype(np.int8)
    recs = []
    for k, v in enumerate((4, 5, 7, 8, 64, 127, -1, -128, -3)):
        r = base[k * 40:k * 40 + 500].copy()
        r[:2] = v
        r[-2:] = v
        recs.append(r)
    return recs + [base[:600].copy(), base[:600].copy(), base[:600].copy()]


def test_boundary_records(ce):
    rng = np.random.default_rng(41)
    shared = rng.integers(0, 4, 4000).astype(np.int8)
    targets = [shared[:3000].copy(), np.zeros(0, np.int8), rng.integers(0, 4, 1).astype(np.int8), shared[100:118].copy(),
               shared[200:219].copy(), shared[300:320].copy(), np.full(300, 5, np.int8), sl.reverse_complement(shared[1000:4000])]
    queries = [sl.mutate(shared[500:3500], 0.03, rng), np.zeros(0, np.int8), shared[100:101].copy(), shared[100:118].copy(),
               shared[200:219].copy(), shared[300:320].copy(), np.full(257, 5, np.int8)]
    for g in (1, 48, SPLIT, None):
        extra = {} if g is None else dict(group_bases=g)
        for strand in ("both", "minus"):
            assert len(ga.check_aligner(ce, targets, queries, strand, **extra)[0]) > 0
        assert_group_stats(ce, targets, queries, g or ce.DEFAULT_GROUP_BASES)
    odd = odd_byte_records(rng)
    for g in (1, 1024, None):
        extra = {} if g is None else dict(group_bases=g)
        ga.check_aligner(ce, odd, odd[::-1], **extra)
    assert_same_at_every_group_size(ce, odd, odd[::-1], sizes=(1024, None), skip_covered=True)


@pytest.mark.parametrize("threshold", [0, -50])
def test_ssp_threshold_at_or_below_zero(ce, threshold):
    # length -1 SSPs are kept; one may only be dropped as contained in an SSP of the same record pair
    rng = np.random.default_rng(51)
    shared = rng.integers(0, 4, 400).astype(np.int8)
    targets = [shared[:200].copy(), shared[:200].copy(), rng.integers(0, 4, 150).astype(np.int8), shared[150:400].copy()]
    queries = [sl.mutate(shared[50:300], 0.05, rng), shared[:200].copy(), shared[180:260].copy()]
    params = dict(ssp_threshold=threshold, gapped_threshold=1 << 40)
    for g in (1, 256, None):
        extra = {} if g is None else dict(group_bases=g)
        ga.check_aligner(ce, targets, queries, **extra, **params)
    runs = assert_same_at_every_group_size(ce, targets, queries, sizes=(256, None), **params)
    assert runs[0][2]["ssps"] > 0


def test_the_tool_prints_the_same_paf(ce, tmp_path):
    targets, queries = contigs(14, 10, 4)
    rec, cigars = ce.align_genomes(targets, queries)
    want = ga.tool_paf(ce, rec, cigars, targets, queries)
    assert want
    for g in ("1", str(SPLIT), "2147483647"):
        out = ga.run_tool(tmp_path, targets, queries, "--group-bases=" + g)
        assert out.returncode == 0 and out.stdout == want, (g, out.stderr)
    out = ga.run_tool(tmp_path, targets, queries, "-s", "minus", "--group-bases", "100", "--chain")
    rec, cigars = ce.align_genomes(targets, queries, strand="minus", chain=True)
    assert out.returncode == 0 and out.stdout == ga.tool_paf(ce, rec, cigars, targets, queries)


def test_a_handle_reused_across_group_sizes_with_a_stream_and_an_allocator(ce):
    import torch
    from genomeworks_b200._lib import lib
    targets, queries = contigs(15, 14, 6)
    small_t, small_q = ga.records_case()
    want = {k: everything(ce, t, q, group_bases=1) for k, (t, q) in enumerate(((targets, queries), (small_t, small_q)))}
    alloc = CountingAllocator()
    al = ce.GenomeAligner(stream=torch.cuda.Stream(), allocator=alloc, group_bases=SPLIT)
    for g in (SPLIT, 1, ce.DEFAULT_GROUP_BASES, 300, SPLIT):
        assert lib().gwb200_genome_aligner_set_group_bases(al._h, C.c_int64(g)) == ce.success
        for k, (t, q) in enumerate(((targets, queries), (small_t, small_q))):
            rec, cigars = al.run(t, q)
            assert (ga.engine_rows(rec), cigars, al.last_stats()[1]) == want[k][:3]
            st = al.last_group_stats()
            assert (st["target_groups"], st["query_groups"]) == (len(groups(t, g)), len(groups(q, g)))
            assert st["gapped_pairs"] == want[k][-1]["gapped_pairs"]
    ms, counts = al.last_stats()
    assert ms["index"] > 0 and ms["count"] > 0 and ms["write"] > 0 and ms["ungapped"] > 0 and ms["gapped_pass1"] > 0
    assert alloc.calls > 0 and len(alloc.live) > 0
    al.close()
    assert alloc.live == {}
