"""The genome aligner with other seed patterns and a word cap (DESIGN.md section 22) against its oracle composition: 14of22,
match12 and a capped 12of19 in every mode and strand at group sizes 1, splitting and default, with identical outputs across
group sizes; a repeated element whose copies lie in different target groups, which only a count over every target record
caps correctly; and the cudaextender tool's PAF with --seed and --max-word-count."""
import numpy as np
import pytest

import genome_aligner_libs as ga
import seed_pattern_libs as sp

pytestmark = pytest.mark.gpu

MODES = {"default": dict(chain=None, min_chain_score=None, skip=False), "skip": dict(chain=None, min_chain_score=None, skip=True),
         "chain": dict(chain=(0, 0), min_chain_score=None, skip=False), "chains": dict(chain=(0, 0), min_chain_score=5000, skip=False)}
SEEDS = [("14of22", 0), ("match12", 0), ("12of19", 1)]


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def run_everywhere(ce, targets, queries, mode, seed, cap, group_sizes):
    """check_aligner at every strand and group size; the outputs and counts of one strand are identical across group sizes."""
    for strand in ("plus", "minus", "both"):
        outs = []
        for gb in group_sizes:
            rec, cigars, counts = sp.check_aligner(ce, targets, queries, strand, seed=seed, max_word_count=cap, group_bases=gb,
                                                   **MODES[mode])
            outs.append((ga.engine_rows(rec), cigars, counts))
        assert all(o == outs[0] for o in outs[1:]), strand
        assert outs[0][2]["seeds"] == sp.seeds_of(targets, queries, strand, seed, cap)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("seed, cap", SEEDS)
def test_records_case_in_every_mode(ce, mode, seed, cap):
    targets, queries = ga.records_case()
    # 9000 puts target 0 on its own and targets 1 and 2 in one group
    run_everywhere(ce, targets, queries, mode, seed, cap, [1, 9000, ce.DEFAULT_GROUP_BASES])


@pytest.mark.parametrize("mode", list(MODES))
def test_a_word_cap_counts_every_target_group(ce, mode):
    targets, queries, cap = sp.split_repeat_case()
    whole = sp.seeds_of(targets, queries, "both", "12of19", cap)
    per_record = sum(len(sp.oracle_run(q_, t, "12of19", True, cap)) for t in targets for q in queries
                     for q_ in (np.asarray(q, np.int8), sp.sl.reverse_complement(q)))
    assert whole < per_record  # counting the words of one record or group at a time would keep more seeds
    # 7000 puts two target records in each group
    run_everywhere(ce, targets, queries, mode, "12of19", cap, [1, 7000, ce.DEFAULT_GROUP_BASES])
    rec, _ = ce.align_genomes(targets, queries, seed="12of19", max_word_count=cap)
    assert len(rec) > 0


def test_the_default_seed_set_explicitly(ce):
    targets, queries = ga.records_case()
    a = ce.align_genomes(targets, queries)
    b = ce.align_genomes(targets, queries, seed="12of19", max_word_count=0)
    assert ga.engine_rows(a[0]) == ga.engine_rows(b[0]) and a[1] == b[1]


def test_tool_seed_and_cap(ce, tmp_path):
    targets, queries, cap = sp.split_repeat_case()
    for options, kw in [(["--seed=14of22", "--max-word-count=%d" % cap], dict(seed="14of22", max_word_count=cap)),
                        (["--seed", "match12", "--no-transition", "--group-bases=7000"], dict(seed="match12", transition=False, group_bases=7000))]:
        r = ga.run_tool(tmp_path, targets, queries, *options)
        assert r.returncode == 0, r.stderr
        rec, cigars = ce.align_genomes(targets, queries, **kw)
        assert len(rec) > 0 and r.stdout == ga.tool_paf(ce, rec, cigars, targets, queries)
