"""Checkers of the gapped extender: ctypes bindings for the CPU oracle (oracle/liboracle_gapped_extender.so), the anchor rule
for scored segment pairs, a separate CIGAR re-scorer, an unpruned numpy DP and the parameters and inputs the tests share. TEST
INFRASTRUCTURE ONLY."""
import ctypes as C
import re

import numpy as np

import extender_libs as xl
from checker_lib import load, ptr

ANCHOR_DTYPE = xl.SEED_DTYPE
GAPPED_DTYPE = np.dtype([("score", np.int64), ("anchor", np.int32), ("has_cigar", np.int32), ("query_begin", np.uint32),
                         ("query_end", np.uint32), ("target_begin", np.uint32), ("target_end", np.uint32)])
FIELDS = GAPPED_DTYPE.names

# LASTZ-style gapped parameters over the ungapped extender's sample matrix
LASTZ_OPEN, LASTZ_EXTEND, LASTZ_YDROP, LASTZ_THRESHOLD = 400, 30, 9400, 3000
# the functions that read a run's results out of its handle, in this oracle and in the skip-covered one built on it
FETCH_SIGNATURES = {
    "oracle_gapped_count": (C.c_int64, [C.c_void_p]),
    "oracle_gapped_live": (C.c_int64, [C.c_void_p]),
    "oracle_gapped_text_bytes": (C.c_int64, [C.c_void_p]),
    "oracle_gapped_fetch": (None, [C.c_void_p, C.c_void_p, C.c_char_p, C.c_void_p]),
    "oracle_gapped_free": (None, [C.c_void_p])}


def oracle():
    return load("liboracle_gapped_extender.so", {
        "oracle_gapped_side": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                         C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_char_p, C.c_int64]),
        "oracle_gapped_side_width": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64,
                                               C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_char_p, C.c_int64]),
        "oracle_gapped_run": (C.c_void_p, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                           C.c_int64, C.c_void_p, C.c_int64, C.c_int64]),
        **FETCH_SIGNATURES})


def _arrays(query, target, matrix):
    return (np.ascontiguousarray(query, np.int8), np.ascontiguousarray(target, np.int8),
            np.ascontiguousarray(np.asarray(matrix).ravel(), np.int32))


def oracle_side(query, target, matrix, o, e, y, q0, t0, left, trace=True):
    """-> dict(best, i, d, live, storage, width, ops) of one side; ops in traceback order (best cell back to (0, 0)); width is
    the widest cell range hi - lo + 1 of any anti-diagonal the side formed, as the device sizes its rings by it."""
    q, t, m = _arrays(query, target, matrix)
    out = np.zeros(6, dtype=np.int64)
    cap = len(q) + len(t) + 2
    buf = C.create_string_buffer(cap) if trace else None
    rc = oracle().oracle_gapped_side_width(ptr(q), len(q), ptr(t), len(t), ptr(m), o, e, y, q0, t0, int(left), ptr(out), buf, cap)
    assert rc == 0
    r = dict(zip(("best", "i", "d", "live", "storage", "width"), (int(v) for v in out)))
    r["ops"] = buf.value.decode() if trace else None
    return r


def oracle_run(query, target, matrix, o, e, y, threshold, anchors, budget=1 << 62):
    """-> (GAPPED_DTYPE records, CIGAR strings, live cells) of one call."""
    q, t, m = _arrays(query, target, matrix)
    a = np.ascontiguousarray(anchors, dtype=ANCHOR_DTYPE)
    L = oracle()
    return _fetch(L, L.oracle_gapped_run(ptr(q), len(q), ptr(t), len(t), ptr(m), o, e, y, threshold, ptr(a), len(a), budget))


def _fetch(L, h):
    """(GAPPED_DTYPE records, CIGAR strings, live cells) of the run handle h of library L, which is then freed."""
    try:
        n = L.oracle_gapped_count(h)
        rec = np.zeros(n, dtype=GAPPED_DTYPE)
        size = L.oracle_gapped_text_bytes(h)
        text = C.create_string_buffer(max(size, 1))
        offsets = np.zeros(n + 1, dtype=np.int64)
        L.oracle_gapped_fetch(h, ptr(rec), text, ptr(offsets))
        raw = text.raw[:size].decode()
        return rec, [raw[offsets[k]:offsets[k + 1]] for k in range(n)], L.oracle_gapped_live(h)
    finally:
        L.oracle_gapped_free(h)


def ssp_anchors(ssps):
    """The anchor of each scored segment pair (SSP_DTYPE): its midpoint, as the device takes it."""
    a = np.zeros(len(ssps), dtype=ANCHOR_DTYPE)
    a["query"] = ssps["query"] + ssps["length"] // 2
    a["target"] = ssps["target"] + ssps["length"] // 2
    return a


def synthetic(n=300, seed=21):
    """(target, query, seeds) of a 30 kb homologous pair at 15 % divergence with n seeds, 30 % of them spurious."""
    from genomeworks_b200 import synth
    return synth.extender_workload(30000, 0.15, n, 0.3, seed=seed)


def rows(rec):
    return [tuple(int(r[f]) for f in FIELDS) for r in rec]


def cigar_ops(cigar):
    return [(int(n), op) for n, op in re.findall(r"(\d+)([MID])", cigar)]


def rescore(cigar, query, target, matrix, o, e, q_begin, t_begin, anchor=None):
    """(score, query bases, target bases) of a CIGAR laid at (q_begin, t_begin): M scores matrix[t * 8 + q], a run of I or D
    of length L scores -(o + L * e). With anchor = (q0, t0), a run that passes through the anchor is charged a second open, as
    the two sides of an extension each open their own part of it."""
    mat = np.asarray(matrix).ravel()
    qi, tj, score = q_begin, t_begin, 0
    for n, op in cigar_ops(cigar):
        if op == "M":
            for k in range(n):
                score += int(mat[(int(target[tj + k]) & 7) * 8 + (int(query[qi + k]) & 7)])
            qi += n
            tj += n
        elif op == "I":
            score -= o + n * e
            if anchor is not None and tj == anchor[1] and qi < anchor[0] < qi + n:
                score -= o
            qi += n
        else:
            score -= o + n * e
            if anchor is not None and qi == anchor[0] and tj < anchor[1] < tj + n:
                score -= o
            tj += n
    return score, qi - q_begin, tj - t_begin


def numpy_best_prefix(a, b, matrix, o, e):
    """Best H over all prefix pairs of the unpruned Gotoh DP of a (query side) against b (target side), int64."""
    mat = np.asarray(matrix, dtype=np.int64).reshape(8, 8)
    m, n = len(a), len(b)
    neg = np.int64(-(1 << 60))
    a7 = np.asarray(a, dtype=np.int64) & 7
    b7 = np.asarray(b, dtype=np.int64) & 7
    H = np.full(n + 1, neg)
    D = np.full(n + 1, neg)
    H[0] = 0
    for j in range(1, n + 1):  # row i = 0: D gaps only
        D[j] = max(D[j - 1] - e, H[j - 1] - o - e)
        H[j] = D[j]
    best = int(H.max())
    I = np.full(n + 1, neg)
    for i in range(1, m + 1):
        diag = np.full(n + 1, neg)
        diag[1:] = H[:-1] + mat[b7, a7[i - 1]]
        I = np.maximum(I - e, H - o - e)
        Hn = np.maximum(diag, I)
        Dn = np.full(n + 1, neg)
        # D along the row: D[j] = max(D[j-1] - e, H[j-1] - o - e) with H the new row; a prefix max with the -e slope
        for j in range(1, n + 1):
            Dn[j] = max(Dn[j - 1] - e, Hn[j - 1] - o - e)
            if Dn[j] > Hn[j]:
                Hn[j] = Dn[j]
        H, D = Hn, Dn
        best = max(best, int(H.max()))
    return best
