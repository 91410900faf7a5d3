"""Checkers of the skip-covered mode (DESIGN.md section 18): ctypes bindings for its CPU oracle (oracle/liboracle_gapped_skip.so),
an independent Python restatement over the gapped extender's oracle, the SSP processing order and the M cells of a CIGAR. TEST
INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

import gapped_extender_libs as gl
from checker_lib import load, ptr


def oracle():
    return load("liboracle_gapped_skip.so", {
        "oracle_gapped_run_skip": (C.c_void_p, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64,
                                                C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
        **gl.FETCH_SIGNATURES})


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
    return gl._fetch(L, h) + ({"extended": int(stats[0]), "skipped": int(stats[1])},)


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
