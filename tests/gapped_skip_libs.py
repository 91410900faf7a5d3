"""Checkers of the skip-covered mode (DESIGN.md section 18): ctypes bindings for its CPU oracle (oracle/liboracle_gapped_skip.so),
an independent Python restatement over the gapped extender's oracle, the SSP processing order, the M cells of a CIGAR, and the
genome aligner's skip-mode composition. TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

import extender_libs as xl
import gapped_extender_libs as gl
import seeder_libs as sl
from checker_lib import load, ptr


def oracle():
    return load("liboracle_gapped_skip.so", {
        "oracle_gapped_run_skip": (C.c_void_p, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64,
                                                C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
        "oracle_gapped_count": (C.c_int64, [C.c_void_p]),
        "oracle_gapped_live": (C.c_int64, [C.c_void_p]),
        "oracle_gapped_text_bytes": (C.c_int64, [C.c_void_p]),
        "oracle_gapped_fetch": (None, [C.c_void_p, C.c_void_p, C.c_char_p, C.c_void_p]),
        "oracle_gapped_free": (None, [C.c_void_p])})


def skip_run(query, target, matrix, o, e, y, threshold, anchors, order=None, budget=1 << 62):
    """-> (GAPPED_DTYPE records, CIGARs, live cells, {extended, skipped}) of the sequential rule over `anchors` taken in
    `order` (default: the order given)."""
    q = np.ascontiguousarray(query, np.int8)
    t = np.ascontiguousarray(target, np.int8)
    m = np.ascontiguousarray(np.asarray(matrix).ravel(), np.int32)
    a = np.ascontiguousarray(anchors, dtype=gl.ANCHOR_DTYPE)
    order = np.arange(len(a), dtype=np.int32) if order is None else np.ascontiguousarray(order, dtype=np.int32)
    stats = np.zeros(2, dtype=np.int64)
    L = oracle()
    h = L.oracle_gapped_run_skip(ptr(q), len(q), ptr(t), len(t), ptr(m), o, e, y, threshold, ptr(a), len(a), ptr(order), budget,
                                 ptr(stats))
    try:
        n = L.oracle_gapped_count(h)
        rec = np.zeros(n, dtype=gl.GAPPED_DTYPE)
        size = L.oracle_gapped_text_bytes(h)
        text = C.create_string_buffer(max(size, 1))
        offsets = np.zeros(n + 1, dtype=np.int64)
        L.oracle_gapped_fetch(h, ptr(rec), text, ptr(offsets))
        raw = text.raw[:size].decode()
        return (rec, [raw[offsets[k]:offsets[k + 1]] for k in range(n)], L.oracle_gapped_live(h),
                {"extended": int(stats[0]), "skipped": int(stats[1])})
    finally:
        L.oracle_gapped_free(h)


def m_cells(record, cigar):
    """The (query, target) cells the M operations of a CIGAR laid at the record's begins align."""
    q, t = int(record["query_begin"]), int(record["target_begin"])
    cells = set()
    for n, op in gl.cigar_ops(cigar):
        if op == "M":
            cells.update((q + k, t + k) for k in range(n))
        if op != "D":
            q += n
        if op != "I":
            t += n
    return cells


def python_skip(query, target, matrix, o, e, y, threshold, anchors, order=None, budget=1 << 62):
    """The sequential rule restated over oracle_run: each anchor alone, with coverage and duplicates applied here. The stats
    also list the skipped anchors."""
    order = range(len(anchors)) if order is None else order
    rec_out, cig_out, live, ext, skipped = [], [], 0, 0, []
    covered, seen = set(), set()
    for k in order:
        k = int(k)
        a = anchors[k:k + 1]
        if (int(a["query"][0]), int(a["target"][0])) in covered:
            skipped.append(k)
            continue
        ext += 1
        rec, cig, lv = gl.oracle_run(query, target, matrix, o, e, y, threshold, a, budget)
        live += lv
        if len(rec) == 0:
            continue
        r = rec[0].copy()
        ends = (int(r["query_begin"]), int(r["query_end"]), int(r["target_begin"]), int(r["target_end"]))
        if ends in seen:
            continue
        seen.add(ends)
        r["anchor"] = k
        rec_out.append(r)
        cig_out.append(cig[0])
        if r["has_cigar"]:
            covered |= m_cells(r, cig[0])
    rec = np.array(rec_out, dtype=gl.GAPPED_DTYPE) if rec_out else np.zeros(0, dtype=gl.GAPPED_DTYPE)
    return rec, cig_out, live, {"extended": ext, "skipped": len(skipped), "skipped_anchors": skipped}


def ssp_order(ssps):
    """The processing order of scored segment pairs: score descending, ties by index."""
    return np.argsort(-np.asarray(ssps["score"], dtype=np.int64), kind="stable").astype(np.int32)


def ssp_anchors(ssps):
    a = np.zeros(len(ssps), dtype=gl.ANCHOR_DTYPE)
    a["query"] = ssps["query"] + ssps["length"] // 2
    a["target"] = ssps["target"] + ssps["length"] // 2
    return a


def _strand_records(ti, qi, strand, query, target, p):
    """(records as tuples, CIGARs) of one pair and strand in skip mode: seeder oracle, ungapped oracle, skip oracle in SSP order,
    minus-strand intervals mapped to forward coordinates after the rule ran in the strand's own."""
    qs = sl.reverse_complement(query) if strand else np.asarray(query, np.int8)
    seeds = sl.oracle_run(qs, target, p["transition"])
    ssps = xl.oracle_run(qs, target, p["matrix"], p["xdrop"], False, p["ssp_threshold"], seeds)
    if len(ssps) == 0:
        return [], [], {"extended": 0, "skipped": 0}
    rec, cigars, _, stats = skip_run(qs, target, p["matrix"], p["gap_open"], p["gap_extend"], p["ydrop"], p["gapped_threshold"],
                                     ssp_anchors(ssps), ssp_order(ssps), p.get("traceback_budget", 1 << 30))
    rows, L = [], len(query)
    for r, cg in zip(rec, cigars):
        qb, qe = int(r["query_begin"]), int(r["query_end"])
        if strand:
            qb, qe = L - qe, L - qb
        matches, block = sl.paf_columns(cg, qs, target, int(r["query_begin"]), int(r["target_begin"]), bool(r["has_cigar"]), qe - qb,
                                        int(r["target_end"]) - int(r["target_begin"]))
        rows.append((int(r["score"]), ti, qi, strand, int(r["has_cigar"]), qb, qe, int(r["target_begin"]), int(r["target_end"]),
                     matches, block))
    return rows, cigars, stats


def aligner_skip_oracle(targets, queries, strand="both", **params):
    """(record tuples in the engine's order, CIGARs, {extended, skipped} summed) of align_genomes(..., skip_covered=True)."""
    p = dict(sl.DEFAULTS)
    p.update(params)
    strands = {"plus": [0], "minus": [1], "both": [0, 1]}[strand]
    rows, cigars, stats = [], [], {"extended": 0, "skipped": 0}
    for ti, t in enumerate(targets):
        for qi, q in enumerate(queries):
            for s in strands:
                r, c, st = _strand_records(ti, qi, s, np.asarray(q, np.int8), np.asarray(t, np.int8), p)
                rows += r
                cigars += c
                for k in stats:
                    stats[k] += st[k]
    return rows, cigars, stats
