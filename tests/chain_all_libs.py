"""Checkers of the all-chains mode (DESIGN.md section 20): ctypes bindings for its extract oracle
(oracle/liboracle_chain_extract.so), a plain-Python restatement of section 20.1 by the subtree form that pins the oracle, and
the genome aligner's oracle composition in this mode -- the composition of genome_aligner_libs with the extract oracle between
the chain oracle and the gapped stage -- with one check of an aligner run against it. TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

import chain_libs as cl
import gapped_extender_libs as gl
import gapped_skip_libs as sk
import genome_aligner_libs as ga
import seeder_libs as sl
from checker_lib import load, ptr
from extender_libs import SSP_DTYPE

INT64_MIN = -(1 << 63)
INT64_MAX = (1 << 63) - 1


def oracle():
    return load("liboracle_chain_extract.so", {
        "oracle_chain_extract": (C.c_int64, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                             C.c_void_p, C.c_void_p])})


def oracle_extract(ssps, D, A, f, p, S):
    """{scores, offsets, members} of section 20.1 over a given f and p, as SspChainer.chain_all returns them."""
    s = np.ascontiguousarray(ssps, dtype=SSP_DTYPE)
    n = len(s)
    f = np.ascontiguousarray(f, dtype=np.int64)
    p = np.ascontiguousarray(p, dtype=np.int32)
    scores = np.zeros(max(n, 1), dtype=np.int64)
    offsets = np.zeros(n + 1, dtype=np.int64)
    members = np.zeros(max(n, 1), dtype=np.int32)
    m = oracle().oracle_chain_extract(ptr(s), n, D, A, ptr(f), ptr(p), S, ptr(scores), ptr(offsets), ptr(members))
    return {"scores": scores[:m].copy(), "offsets": offsets[:m + 1].copy(), "members": members[:offsets[m]].copy()}


def union(res):
    """The members of all reported chains in ascending index, as the engine gives them to the gapped stage."""
    return np.sort(res["members"]).astype(np.int32)


def oracle_all(ssps, D=0, A=0, S=INT64_MIN):
    """The DP oracle (chain_libs), then the extract oracle on its f and p: {f, p, scores, offsets, members, union, sum}."""
    dp = cl.oracle_run(ssps, D, A)
    out = oracle_extract(ssps, D, A, dp["f"], dp["p"], S)
    out.update(f=dp["f"], p=dp["p"], union=union(out), sum=int(out["scores"].sum()))
    return out


def python_extract(ssps, f, p, S):
    """Section 20.1 restated by the subtree form: the owner of x is the priority-best SSP among x's descendants in the p-forest
    (every j whose p-path passes through x, x included); a chain is the SSPs of one owner; its first member c_1 is the one whose
    p is -1 or owned by another, and its score is f(h) - f(c_1) + s(c_1). Owners are reported in priority order."""
    n = len(ssps)
    f = [int(v) for v in f]
    p = [int(v) for v in p]

    def prio(k):
        return (-f[k], k)

    owner = list(range(n))
    for j in range(n):
        x = j
        while x >= 0:
            if prio(j) < prio(owner[x]):
                owner[x] = j
            x = p[x]
    heads = sorted({owner[x] for x in range(n)}, key=prio)
    scores, offsets, members = [], [0], []
    for h in heads:
        mem = [x for x in range(n) if owner[x] == h]
        first = [x for x in mem if p[x] < 0 or owner[p[x]] != h]
        assert len(first) == 1
        c1 = first[0]
        score = f[h] - f[c1] + int(ssps[c1]["score"])
        if score >= S:
            scores.append(score)
            members += mem
            offsets.append(len(members))
    return {"scores": np.array(scores, dtype=np.int64), "offsets": np.array(offsets, dtype=np.int64),
            "members": np.array(members, dtype=np.int32)}


def same_chains(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("scores", "offsets", "members"))


# ---- the genome aligner with all chains ----

def _strand_records(ti, qi, strand, query, target, p, chain, S, skip):
    """(record tuples, CIGARs, anchors, stats) of one pair and strand: ga's ungapped SSPs, the chain oracle, the extract oracle's
    union, then ga's gapped or skip-covered stage and coordinate mapping."""
    qs = sl.reverse_complement(query) if strand else query
    ssps = ga.ungapped_ssps(qs, target, p)
    stats = dict(extended=0, skipped=0, ssps_in=0, ssps_chained=0, pairs=0, chains=0)
    if len(ssps) == 0:
        return [], [], [], stats
    res = oracle_all(ssps, *chain, S)
    stats.update(ssps_in=len(ssps), pairs=1, chains=len(res["scores"]))
    ssps = ssps[res["union"]]
    stats["ssps_chained"] = len(ssps)
    if len(ssps) == 0:
        return [], [], [], stats
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
        matches, block = ga.paf_columns(cg, qs, target, int(r["query_begin"]), tb, bool(r["has_cigar"]), qe - qb, te - tb)
        rows.append((int(r["score"]), ti, qi, strand, int(r["has_cigar"]), qb, qe, tb, te, matches, block))
        a = anchors[int(r["anchor"])]
        at.append((int(a["query"]), int(a["target"])))
    return rows, cigars, at, stats


def aligner_oracle(targets, queries, strand="both", chain=(0, 0), min_chain_score=INT64_MIN, skip=False, **params):
    """(record tuples in the engine's order, CIGARs, anchors, stats) of align_genomes(..., chain=chain,
    min_chain_score=min_chain_score, skip_covered=skip); stats as ga.aligner_oracle's plus the number of reported chains."""
    p = dict(ga.DEFAULTS)
    p.update(params)
    rows, cigars, anchors, stats = [], [], [], dict(extended=0, skipped=0, ssps_in=0, ssps_chained=0, pairs=0, chains=0)
    for ti, t in enumerate(targets):
        for qi, q in enumerate(queries):
            for s in ga.STRANDS[strand]:
                r, c, a, st = _strand_records(ti, qi, s, np.asarray(q, np.int8), np.asarray(t, np.int8), p, chain, min_chain_score, skip)
                rows += r
                cigars += c
                anchors += a
                for k in stats:
                    stats[k] += st[k]
    return rows, cigars, anchors, stats


def check_aligner(ce, targets, queries, strand="both", chain=(0, 0), min_chain_score=INT64_MIN, skip=False, **params):
    """Runs a GenomeAligner with all chains on and asserts what ga.check_aligner asserts -- records and CIGARs, every CIGAR
    re-scored from its anchor, the PAF text, the extended and skipped counts, the chain stats -- and the chain count. ->
    (records, CIGARs, skip stats, chain stats)."""
    al = ce.GenomeAligner(strand, skip_covered=skip, chain=chain, min_chain_score=min_chain_score, **params)
    rec, cigars = al.run(targets, queries)
    skip_stats, chain_stats, chain_count = al.last_skip_stats(), al.last_chain_stats(), al.last_chain_count()
    al.close()
    params = {k: v for k, v in params.items() if k not in ga.ENGINE_ONLY}
    rows, want, anchors, stats = aligner_oracle(targets, queries, strand, chain, min_chain_score, skip, **params)
    assert ga.engine_rows(rec) == rows
    assert cigars == want
    p = dict(ga.DEFAULTS, **params)
    for r, cg, anchor in zip(rec, cigars, anchors):
        if not r["has_cigar"]:
            continue
        q = np.asarray(queries[r["query_record"]], np.int8)
        qs = sl.reverse_complement(q) if r["strand"] else q
        qb = len(q) - int(r["query_end"]) if r["strand"] else int(r["query_begin"])
        got = gl.rescore(cg, qs, targets[r["target_record"]], p["matrix"], p["gap_open"], p["gap_extend"], qb, int(r["target_begin"]),
                         anchor=anchor)
        assert got == (int(r["score"]), int(r["query_end"] - r["query_begin"]), int(r["target_end"] - r["target_begin"]))
    tn, tl, qn, ql = ga.names("t", targets), ga.lengths(targets), ga.names("q", queries), ga.lengths(queries)
    assert ce.format_paf(rec, cigars, tn, tl, qn, ql) == ga.paf_oracle(rows, want, tn, tl, qn, ql)
    assert (skip_stats["extended"], skip_stats["skipped"]) == (stats["extended"], stats["skipped"])
    assert {k: chain_stats[k] for k in ("ssps_in", "ssps_chained", "pairs")} == {k: stats[k] for k in ("ssps_in", "ssps_chained", "pairs")}
    assert (chain_stats["chain_ms"] > 0) == (stats["pairs"] > 0)
    assert chain_count == stats["chains"]
    return rec, cigars, skip_stats, chain_stats
