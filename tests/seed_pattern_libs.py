"""Checkers of the seeding rule with any seed pattern and a word cap (DESIGN.md section 22): ctypes bindings for its CPU oracle
(oracle/liboracle_seeder_pattern.so), a brute-force restatement in Python, and the genome aligner's oracle composition and
check with a seed and a cap, in every mode (default, skip-covered, best chain, all chains). TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

import chain_all_libs as cal
import chain_libs as cl
import extender_libs as xl
import gapped_extender_libs as gl
import gapped_skip_libs as sk
import genome_aligner_libs as ga
import seeder_libs as sl
from checker_lib import load, ptr

NAMED = {"12of19": "1110100110010101111", "14of22": "1110101100110010101111"}
# the patterns the tests run: the named ones, match<N> at both ends of the weight range, and a span-1, a span-3 and a span-32
# pattern of 0/1 strings
PATTERNS = ["12of19", "14of22", "match1", "match5", "match12", "match14", "1", "101", "11010010000000000000000000011011"]
BAD_PATTERNS = ["", "0", "01", "10", "1x1", "T1", "match0", "match15", "1" * 15, "1" + "0" * 31 + "1"]


def bits(seed):
    """The 0/1 string of a valid pattern."""
    if seed.startswith("match"):
        return "1" * int(seed[5:])
    return NAMED.get(seed, seed)


def oracle():
    return load("liboracle_seeder_pattern.so", {
        "oracle_seed_pattern": (C.c_int32, [C.c_char_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
        "oracle_seeder_pattern_run": (C.c_int64, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_char_p, C.c_int32, C.c_int64, C.c_void_p,
                                                  C.c_void_p, C.c_int32, C.c_void_p, C.c_int64])})


def flat(records):
    """(codes, offsets) of a list of records."""
    codes = [np.ascontiguousarray(r, np.int8) for r in records]
    off = np.zeros(len(codes) + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(c) for c in codes]) if codes else []
    return (np.concatenate(codes) if codes else np.zeros(1, np.int8)), off


def oracle_run(query, target, seed="12of19", transition=True, max_word_count=0, word_records=None):
    """The seed pairs of query against target in the engine's global order (xl.SEED_DTYPE), the word cap counting the words of
    word_records (default: the target alone)."""
    q, t = np.ascontiguousarray(query, np.int8), np.ascontiguousarray(target, np.int8)
    w, woff = flat([t] if word_records is None else word_records)
    L = oracle()
    args = (ptr(q), len(q), ptr(t), len(t), seed.encode(), int(bool(transition)), int(max_word_count), ptr(w), ptr(woff), len(woff) - 1)
    n = L.oracle_seeder_pattern_run(*args, None, 0)
    assert n >= 0, "invalid pattern or cap"
    out = np.zeros(n, dtype=xl.SEED_DTYPE)
    L.oracle_seeder_pattern_run(*args, ptr(out), n)
    return out


def rows(seeds):
    return list(zip(seeds["query"].tolist(), seeds["target"].tolist()))


def window_keys(seq, pattern):
    """The key tuple (care codes in pattern order) of the window ending at every position, None where there is none."""
    span, care = len(pattern), [i for i, c in enumerate(pattern) if c == "1"]
    s = [int(c) for c in seq]
    return [tuple(s[p - span + 1 + c] for c in care) if p >= span - 1 and all(0 <= x <= 3 for x in s[p - span + 1:p + 1]) else None
            for p in range(len(s))]


def brute(query, target, seed, transition=True, max_word_count=0, word_records=None):
    """The rule restated: q ascending; the exact bucket, then the transition at care position 0 ... W - 1, each skipped when its
    word occurs more than max_word_count times over word_records (when > 0); t ascending. -> [(q, t)]."""
    pattern = bits(seed)
    tkeys = window_keys(target, pattern)
    counts = {}
    for r in ([target] if word_records is None else word_records):
        for k in window_keys(r, pattern):
            if k is not None:
                counts[k] = counts.get(k, 0) + 1
    out = []
    for q, k in enumerate(window_keys(query, pattern)):
        if k is None:
            continue
        variants = [k] + ([tuple(c ^ 2 if i == j else c for i, c in enumerate(k)) for j in range(len(k))] if transition else [])
        for v in variants:
            if max_word_count > 0 and counts.get(v, 0) > max_word_count:
                continue
            out += [(q, t) for t, tk in enumerate(tkeys) if tk == v]
    return out


# ---- the genome aligner with a seed pattern and a word cap ----

_ungapped = {}


def ungapped_ssps(qs, target, targets, p, seed, max_word_count):
    """ga.ungapped_ssps with this seeding rule; the cap counts the words of every target record."""
    key = (qs.tobytes(), target.tobytes(), seed, max_word_count, b"".join(np.asarray(t, np.int8).tobytes() + b"|" for t in targets) if max_word_count else b"",
           bool(p["transition"]), np.asarray(p["matrix"]).tobytes(), p["xdrop"], p["ssp_threshold"])
    if key not in _ungapped:
        seeds = oracle_run(qs, target, seed, p["transition"], max_word_count, targets)
        _ungapped[key] = xl.oracle_run(qs, target, p["matrix"], p["xdrop"], False, p["ssp_threshold"], seeds)
    return _ungapped[key]


def _strand_records(ti, qi, strand, query, target, targets, p, chain, min_chain_score, skip, seed, max_word_count):
    """(record tuples, CIGARs, anchors, stats) of one pair and strand: this rule's ungapped SSPs, then the modes' stages as the
    §19 and §20 compositions run them (ga and chain_all_libs)."""
    qs = sl.reverse_complement(query) if strand else query
    ssps = ungapped_ssps(qs, target, targets, p, seed, max_word_count)
    stats = dict(extended=0, skipped=0, ssps_in=0, ssps_chained=0, pairs=0, chains=0)
    if len(ssps) == 0:
        return [], [], [], stats
    if chain is not None:
        stats.update(ssps_in=len(ssps), pairs=1)
        if min_chain_score is None:
            ssps = ssps[cl.chain_indices(cl.oracle_run(ssps, *chain))]
            stats["chains"] = 1
        else:
            res = cal.oracle_all(ssps, *chain, min_chain_score)
            stats["chains"] = len(res["scores"])
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
    rows_, at, L = [], [], len(query)
    for r, cg in zip(rec, cigars):
        qb, qe = int(r["query_begin"]), int(r["query_end"])
        if strand:
            qb, qe = L - qe, L - qb
        tb, te = int(r["target_begin"]), int(r["target_end"])
        matches, block = ga.paf_columns(cg, qs, target, int(r["query_begin"]), tb, bool(r["has_cigar"]), qe - qb, te - tb)
        rows_.append((int(r["score"]), ti, qi, strand, int(r["has_cigar"]), qb, qe, tb, te, matches, block))
        a = anchors[int(r["anchor"])]
        at.append((int(a["query"]), int(a["target"])))
    return rows_, cigars, at, stats


def aligner_oracle(targets, queries, strand="both", chain=None, min_chain_score=None, skip=False, seed="12of19", max_word_count=0,
                   **params):
    """(record tuples in the engine's order, CIGARs, anchors, stats) of align_genomes(..., chain=chain,
    min_chain_score=min_chain_score, skip_covered=skip, seed=seed, max_word_count=max_word_count); stats as
    chain_all_libs.aligner_oracle's (chains: one per chained pair and strand with the best chain)."""
    p = dict(ga.DEFAULTS)
    p.update(params)
    targets = [np.asarray(t, np.int8) for t in targets]
    rows_, cigars, anchors, stats = [], [], [], dict(extended=0, skipped=0, ssps_in=0, ssps_chained=0, pairs=0, chains=0)
    for ti, t in enumerate(targets):
        for qi, q in enumerate(queries):
            for s in ga.STRANDS[strand]:
                r, c, a, st = _strand_records(ti, qi, s, np.asarray(q, np.int8), t, targets, p, chain, min_chain_score, skip, seed,
                                              max_word_count)
                rows_ += r
                cigars += c
                anchors += a
                for k in stats:
                    stats[k] += st[k]
    return rows_, cigars, anchors, stats


def check_aligner(ce, targets, queries, strand="both", chain=None, min_chain_score=None, skip=False, seed="12of19", max_word_count=0,
                  **params):
    """Runs a GenomeAligner with the seed and cap and asserts what ga.check_aligner and chain_all_libs.check_aligner assert:
    records and CIGARs, every CIGAR re-scored from its anchor, the PAF text, the extended and skipped counts, the chain stats
    and the chain count. -> (records, CIGARs, last_stats counts)."""
    al = ce.GenomeAligner(strand, skip_covered=skip, chain=chain, min_chain_score=min_chain_score, seed=seed, max_word_count=max_word_count,
                          **params)
    rec, cigars = al.run(targets, queries)
    skip_stats, chain_stats, chain_count = al.last_skip_stats(), al.last_chain_stats(), al.last_chain_count()
    counts = al.last_stats()[1]
    al.close()
    params = {k: v for k, v in params.items() if k not in ga.ENGINE_ONLY + ("group_bases",)}
    rows_, want, anchors, stats = aligner_oracle(targets, queries, strand, chain, min_chain_score, skip, seed, max_word_count, **params)
    assert ga.engine_rows(rec) == rows_
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
    assert ce.format_paf(rec, cigars, tn, tl, qn, ql) == ga.paf_oracle(rows_, want, tn, tl, qn, ql)
    assert (skip_stats["extended"], skip_stats["skipped"]) == (stats["extended"], stats["skipped"])
    assert {k: chain_stats[k] for k in ("ssps_in", "ssps_chained", "pairs")} == {k: stats[k] for k in ("ssps_in", "ssps_chained", "pairs")}
    assert chain_count == (stats["chains"] if chain is not None else 0)
    return rec, cigars, counts


def seeds_of(targets, queries, strand, seed, max_word_count, transition=True):
    """The seeds the aligner counts over every (target record, query record, strand), from the oracle."""
    targets = [np.asarray(t, np.int8) for t in targets]
    n = 0
    for t in targets:
        for q in queries:
            for s in ga.STRANDS[strand]:
                qs = sl.reverse_complement(np.asarray(q, np.int8)) if s else np.asarray(q, np.int8)
                n += len(oracle_run(qs, t, seed, transition, max_word_count, targets))
    return n


def split_repeat_case(seed=41, copies=6, unit_len=400):
    """Target contigs and a query where one element's copies, 1 % diverged, are spread over the target records, one per record:
    with the cap of 2 returned, a word the copies share occurs at most once in a record and up to `copies` times in all of
    them, so a cap counted per record or per group keeps seeds that the whole-target count drops. -> (targets, queries, cap)."""
    rng = np.random.default_rng(seed)
    unit = rng.integers(0, 4, unit_len).astype(np.int8)
    targets = []
    for k in range(copies):
        left, right = rng.integers(0, 4, 1500).astype(np.int8), rng.integers(0, 4, 1500).astype(np.int8)
        targets.append(np.concatenate([left, sl.mutate(unit, 0.01, rng), right]))
    queries = [np.concatenate([rng.integers(0, 4, 700).astype(np.int8), sl.mutate(unit, 0.01, rng), targets[2][:1500],
                               rng.integers(0, 4, 700).astype(np.int8)])]
    return targets, queries, 2
