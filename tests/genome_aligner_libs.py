"""Checkers of the genome aligner: its oracle composition -- seeder oracle, ungapped extender oracle, optional chain oracle,
gapped or skip-covered extender oracle, numpy reverse complement and coordinate mapping, and the PAF rules restated here -- one
check of an aligner run against it for every mode, and the inputs and tool runs the aligner's tests share. TEST INFRASTRUCTURE
ONLY."""
import os
import re
import subprocess

import numpy as np

import chain_libs as cl
import extender_libs as xl
import gapped_extender_libs as gl
import gapped_skip_libs as sk
import seeder_libs as sl
from checker_lib import ROOT

# the aligner's defaults (gwb200_genome_aligner_default_params)
DEFAULTS = dict(matrix=xl.SAMPLE_MATRIX, xdrop=xl.SAMPLE_XDROP, ssp_threshold=xl.SAMPLE_THRESHOLD, gap_open=gl.LASTZ_OPEN,
                gap_extend=gl.LASTZ_EXTEND, ydrop=gl.LASTZ_YDROP, gapped_threshold=gl.LASTZ_THRESHOLD, transition=True,
                traceback_budget=1 << 30)
# parameters that change how the engine groups its work, never its output
ENGINE_ONLY = ("block_size", "round_anchors")
STRANDS = {"plus": [0], "minus": [1], "both": [0, 1]}

_ungapped = {}


def ungapped_ssps(qs, target, p):
    """The unique SSPs of the seeder and ungapped oracles, kept for the process: the compositions of one test share them."""
    key = (qs.tobytes(), target.tobytes(), bool(p["transition"]), np.asarray(p["matrix"]).tobytes(), p["xdrop"], p["ssp_threshold"])
    if key not in _ungapped:
        seeds = sl.oracle_run(qs, target, p["transition"])
        _ungapped[key] = xl.oracle_run(qs, target, p["matrix"], p["xdrop"], False, p["ssp_threshold"], seeds)
    return _ungapped[key]


def _strand_records(ti, qi, strand, query, target, p, chain, skip):
    """(record tuples, CIGARs, anchors, stats) of one pair and strand. The rules run in the strand's own coordinates; minus-strand
    query intervals are then mapped to forward coordinates."""
    qs = sl.reverse_complement(query) if strand else query
    ssps = ungapped_ssps(qs, target, p)
    stats = dict(extended=0, skipped=0, ssps_in=0, ssps_chained=0, pairs=0)
    if len(ssps) == 0:
        return [], [], [], stats
    if chain is not None:
        stats.update(ssps_in=len(ssps), pairs=1)
        ssps = ssps[cl.chain_indices(cl.oracle_run(ssps, *chain))]
        stats["ssps_chained"] = len(ssps)
    anchors = gl.ssp_anchors(ssps)
    args = (qs, target, p["matrix"], p["gap_open"], p["gap_extend"], p["ydrop"], p["gapped_threshold"], anchors)
    if skip:
        rec, cigars, _, counts = sk.skip_run(*args, sk.ssp_order(ssps), p["traceback_budget"])
        stats.update(counts)
    else:
        rec, cigars, _ = gl.oracle_run(*args, p["traceback_budget"])
        stats["extended"] = len(anchors)
    rows, at, L = [], [], len(query)
    for r, cg in zip(rec, cigars):
        qb, qe = int(r["query_begin"]), int(r["query_end"])
        if strand:
            qb, qe = L - qe, L - qb
        tb, te = int(r["target_begin"]), int(r["target_end"])
        matches, block = paf_columns(cg, qs, target, int(r["query_begin"]), tb, bool(r["has_cigar"]), qe - qb, te - tb)
        rows.append((int(r["score"]), ti, qi, strand, int(r["has_cigar"]), qb, qe, tb, te, matches, block))
        a = anchors[int(r["anchor"])]
        at.append((int(a["query"]), int(a["target"])))
    return rows, cigars, at, stats


def aligner_oracle(targets, queries, strand="both", chain=None, skip=False, **params):
    """(record tuples in the engine's order, CIGARs, the anchor of each in its strand's coordinates, stats) of
    align_genomes(..., chain=chain, skip_covered=skip) over the records (int8 codes). chain is None or the (D, A) penalties; stats
    are {extended, skipped} of the gapped stage and {ssps_in, ssps_chained, pairs} of the chainer, summed over pairs and strands
    as the engine reports them."""
    p = dict(DEFAULTS)
    p.update(params)
    rows, cigars, anchors, stats = [], [], [], dict(extended=0, skipped=0, ssps_in=0, ssps_chained=0, pairs=0)
    for ti, t in enumerate(targets):
        for qi, q in enumerate(queries):
            for s in STRANDS[strand]:
                r, c, a, st = _strand_records(ti, qi, s, np.asarray(q, np.int8), np.asarray(t, np.int8), p, chain, skip)
                rows += r
                cigars += c
                anchors += a
                for k in stats:
                    stats[k] += st[k]
    return rows, cigars, anchors, stats


def paf_columns(cigar, qcodes, tcodes, qb, tb, has_cigar, qspan, tspan):
    """PAF columns 10 and 11: M positions with equal codes in 0..3, and the sum of M, I and D lengths; without a CIGAR 0 and the
    larger span."""
    if not has_cigar:
        return 0, max(qspan, tspan)
    matches = block = 0
    for n, op in re.findall(r"(\d+)([MID])", cigar):
        n = int(n)
        block += n
        if op == "M":
            a = np.asarray(qcodes[qb:qb + n])
            b = np.asarray(tcodes[tb:tb + n])
            matches += int(((a == b) & (a >= 0) & (a < 4)).sum())
            qb += n
            tb += n
        elif op == "I":
            qb += n
        else:
            tb += n
    return matches, block


def engine_rows(rec):
    return [tuple(int(r[f]) for f in ("score", "target_record", "query_record", "strand", "has_cigar", "query_begin", "query_end",
                                      "target_begin", "target_end", "matches", "block_length")) for r in rec]


def paf_oracle(rows, cigars, target_names, target_lengths, query_names, query_lengths):
    lines = []
    for r, cg in zip(rows, cigars):
        score, ti, qi, strand, has_cigar, qb, qe, tb, te, matches, block = r
        cols = [query_names[qi], query_lengths[qi], qb, qe, "-" if strand else "+", target_names[ti], target_lengths[ti], tb, te,
                matches, block, 255, "AS:i:%d" % score]
        if has_cigar:
            cols.append("cg:Z:" + cg)
        lines.append("\t".join(str(c) for c in cols) + "\n")
    return "".join(lines)


def names(prefix, records):
    return ["%s%d" % (prefix, k) for k in range(len(records))]


def lengths(records):
    return [len(s) for s in records]


def check_aligner(ce, targets, queries, strand="both", chain=None, skip=False, **params):
    """Runs a GenomeAligner and asserts that it equals the oracle composition: records and CIGARs, every CIGAR re-scored from its
    anchor, the PAF text, the gapped stage's extended and skipped counts, and the chain stats. -> (records, CIGARs, skip stats,
    chain stats)."""
    al = ce.GenomeAligner(strand, skip_covered=skip, chain=chain, **params)
    rec, cigars = al.run(targets, queries)
    skip_stats, chain_stats = al.last_skip_stats(), al.last_chain_stats()
    al.close()
    params = {k: v for k, v in params.items() if k not in ENGINE_ONLY}
    rows, want, anchors, stats = aligner_oracle(targets, queries, strand, chain, skip, **params)
    assert engine_rows(rec) == rows
    assert cigars == want
    p = dict(DEFAULTS, **params)
    # every CIGAR re-scores to its score, on its strand's query
    for r, cg, anchor in zip(rec, cigars, anchors):
        if not r["has_cigar"]:
            continue
        q = np.asarray(queries[r["query_record"]], np.int8)
        qs = sl.reverse_complement(q) if r["strand"] else q
        qb = len(q) - int(r["query_end"]) if r["strand"] else int(r["query_begin"])
        got = gl.rescore(cg, qs, targets[r["target_record"]], p["matrix"], p["gap_open"], p["gap_extend"], qb, int(r["target_begin"]),
                         anchor=anchor)
        assert got == (int(r["score"]), int(r["query_end"] - r["query_begin"]), int(r["target_end"] - r["target_begin"]))
    tn, tl, qn, ql = names("t", targets), lengths(targets), names("q", queries), lengths(queries)
    assert ce.format_paf(rec, cigars, tn, tl, qn, ql) == paf_oracle(rows, want, tn, tl, qn, ql)
    assert (skip_stats["extended"], skip_stats["skipped"]) == (stats["extended"], stats["skipped"])
    assert {k: chain_stats[k] for k in ("ssps_in", "ssps_chained", "pairs")} == {k: stats[k] for k in ("ssps_in", "ssps_chained", "pairs")}
    assert (chain_stats["chain_ms"] > 0) == (stats["pairs"] > 0)
    return rec, cigars, skip_stats, chain_stats


def records_case():
    """Three targets by two queries: a shared piece on the plus strand of target 0 and the minus strand of target 2, a
    diverged copy of target 1 behind 500 unrelated bases with a run of N, and record pairs with no hit."""
    rng = np.random.default_rng(17)
    shared = rng.integers(0, 4, 6000).astype(np.int8)
    targets = [np.concatenate([rng.integers(0, 4, 2000).astype(np.int8), shared[:3000]]),
               rng.integers(0, 4, 4000).astype(np.int8),
               np.concatenate([sl.reverse_complement(shared[2500:]), rng.integers(0, 4, 1000).astype(np.int8)])]
    queries = [sl.mutate(shared, 0.03, rng), np.concatenate([rng.integers(0, 4, 500).astype(np.int8), sl.mutate(targets[1][1000:3000], 0.05, rng)])]
    queries[1][100:140] = 5
    return targets, queries


def run_tool(tmp_path, targets, queries, *options, fastq=False):
    """build/cudaextender with `options` over the records written as FASTA named t0, t1, ... and q0, q1, ...; with fastq=True
    the queries are FASTQ and every target name carries extra words, which the tool drops. -> the completed process."""
    tfile, qfile = tmp_path / "t.fa", tmp_path / ("q.fq" if fastq else "q.fa")
    with open(tfile, "w") as f:
        for n, s in zip(names("t", targets), targets):
            f.write(">%s%s\n%s\n" % (n, " extra words" if fastq else "", sl.text(s)))
    with open(qfile, "w") as f:
        for n, s in zip(names("q", queries), queries):
            f.write("@%s\n%s\n+\n%s\n" % (n, sl.text(s), "I" * len(s)) if fastq else ">%s\n%s\n" % (n, sl.text(s)))
    return subprocess.run([os.path.join(ROOT, "build", "cudaextender"), *options, str(tfile), str(qfile)], capture_output=True,
                          text=True, timeout=600)


def tool_paf(ce, rec, cigars, targets, queries):
    """format_paf of an aligner run under the record names run_tool writes."""
    return ce.format_paf(rec, cigars, names("t", targets), lengths(targets), names("q", queries), lengths(queries))
