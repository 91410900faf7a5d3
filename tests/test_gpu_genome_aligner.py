"""The genome aligner on the GPU against its oracle composition (seeder, ungapped and gapped extender oracles, numpy reverse
complement and coordinate mapping, the PAF rules in Python): records, CIGARs and PAF, on the golden sample, a rearranged pair
and several records per side; every CIGAR re-scores to its score, the block size does not change the output, and the
cudaextender tool prints the same PAF."""
import numpy as np
import pytest

import extender_libs as xl
import genome_aligner_libs as ga
import seeder_libs as sl

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def test_golden_sample_both_strands(ce):
    seq, _, _ = xl.sample()
    rec = ga.check_aligner(ce, [seq], [seq])[0]
    assert (rec["strand"] == 0).sum() > 0


def test_rearranged_pair_finds_the_inversion_on_the_minus_strand(ce):
    target, query, (a, b) = sl.rearranged_pair(5)
    rec = ga.check_aligner(ce, [target], [query])[0]
    minus = rec[rec["strand"] == 1]
    # the inverted piece sits at about [a, b) in both: a minus-strand alignment covers most of it at forward coordinates
    hit = [r for r in minus if r["target_begin"] < b and r["target_end"] > a and abs(int(r["query_begin"]) - int(r["target_begin"])) < 500
           and min(int(r["target_end"]), b) - max(int(r["target_begin"]), a) > (b - a) // 2]
    assert hit, minus
    # the translocated pieces align on the plus strand off the main diagonal
    plus = rec[rec["strand"] == 0]
    assert (np.abs(plus["query_begin"].astype(np.int64) - plus["target_begin"].astype(np.int64)) > 2000).any()


def test_three_targets_by_two_queries(ce):
    targets, queries = ga.records_case()
    rec = ga.check_aligner(ce, targets, queries)[0]
    assert set(zip(rec["target_record"].tolist(), rec["query_record"].tolist())) >= {(0, 0), (2, 0), (1, 1)}
    order = [(int(r["target_record"]), int(r["query_record"]), int(r["strand"])) for r in rec]
    assert order == sorted(order)


def test_block_size_does_not_change_the_output(ce):
    seq, _, _ = xl.sample()
    targets, queries = ga.records_case()
    for t, q in (([seq], [seq]), (targets, queries)):
        want = ce.align_genomes(t, q)
        for b in (1000, 7):
            if b == 7 and len(t) == 1:
                continue  # 143,671 seeds in blocks of 7 is slow, not different
            got = ce.align_genomes(t, q, block_size=b)
            assert ga.engine_rows(got[0]) == ga.engine_rows(want[0]) and got[1] == want[1]


def test_one_strand_and_exact_seeds(ce):
    targets, queries = ga.records_case()
    for strand in ("plus", "minus"):
        ga.check_aligner(ce, targets, queries, strand=strand)
    ga.check_aligner(ce, targets[:1], queries[:1], transition=False)


def test_tool_prints_the_same_paf(ce, tmp_path):
    targets, queries = ga.records_case()
    rec, cigars = ce.align_genomes(targets, queries)
    want = ga.tool_paf(ce, rec, cigars, targets, queries)
    assert want == ga.paf_oracle(ga.engine_rows(rec), cigars, ga.names("t", targets), ga.lengths(targets), ga.names("q", queries),
                                 ga.lengths(queries))
    out = ga.run_tool(tmp_path, targets, queries, fastq=True)
    assert out.returncode == 0, out.stderr
    assert out.stdout == want and want
    out = ga.run_tool(tmp_path, targets, queries, "-s", "minus", "-B", "1000", fastq=True)
    rec, cigars = ce.align_genomes(targets, queries, strand="minus")
    assert out.returncode == 0 and out.stdout == ga.tool_paf(ce, rec, cigars, targets, queries)


def test_stats_and_a_stream(ce):
    import torch
    targets, queries = ga.records_case()
    want = ce.align_genomes(targets, queries)
    al = ce.GenomeAligner(stream=torch.cuda.Stream())
    got = al.run(targets, queries)
    assert ga.engine_rows(got[0]) == ga.engine_rows(want[0]) and got[1] == want[1]
    ms, counts = al.last_stats()
    assert ms["index"] > 0 and ms["count"] > 0 and ms["write"] > 0 and ms["ungapped"] > 0 and ms["gapped_pass1"] > 0
    assert counts["seeds"] > counts["ssps"] > 0 and counts["alignments"] == len(got[0])
    al.close()
