"""ctypes bindings of read correction's CPU restatement (oracle/liboracle_correct.so, oracle/correct_oracle.cpp, built by build()),
a Python restatement of view B, and the composition of read correction from proven parts (DESIGN.md section 15.6).

- oracle_correct_groups: steps 1-3, in the shape cudapolish.correction_window_groups returns ("weights" with qualities);
- oracle_mirror / oracle_view: view B's CIGAR text, and one view's R and cut points;
- py_mirror / py_view: the same restated in Python;
- composition: map_reads(reads, align=True), oracle_correct_groups, the POA batch one group at a time, the oracle's stitching;
- correction_case: seeded reads of a truth with each read's true segment.
"""
import ctypes as C

import numpy as np

import polish_libs as pl
import polish_quality_libs as pq
from checker_lib import load, ptr


def oracle():
    return load("liboracle_correct.so", {
        "oracle_correct_groups": (C.c_int, [C.c_void_p, C.c_int64, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_char_p,
                                            C.c_double, C.c_int32, C.c_int32]),
        "oracle_correct_mirror": (C.c_int64, [C.c_char_p, C.c_int64, C.c_uint8, C.c_char_p, C.c_int64]),
        "oracle_correct_view": (C.c_int64, [C.c_void_p, C.c_char_p, C.c_int64, C.c_char_p, C.c_void_p, C.c_int32, C.c_int32, C.c_char_p,
                                            C.c_void_p]),
        "oracle_polish_view": (C.c_int, [C.POINTER(pl._View)]),
        "oracle_polish_weights": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64)])})


def oracle_correct_groups(overlaps, cigars, reads, window_length, max_depth, qualities=None, threshold=10.0):
    """(0, dict of pl.KEYS and "n_kept", plus "weights" with qualities) or (-1, None) for the arguments the contract rejects."""
    ov = np.ascontiguousarray(overlaps, dtype=pl.OVERLAP_DTYPE)
    text, toffs = pl.cigar_text(cigars)
    rb, roffs = pl._flat(reads)
    qb = None
    if qualities is not None:
        qb, qoffs = pl._flat(qualities)
        assert np.array_equal(roffs, qoffs), "one quality string per read, as long as the read"
    L = oracle()
    rc = L.oracle_correct_groups(ptr(ov), len(ov), text, ptr(toffs), rb,
                                 ptr(roffs), len(roffs) - 1, qb, threshold, window_length, max_depth)
    if rc != 0:
        return rc, None
    v = pl._View()
    L.oracle_polish_view(C.byref(v))
    out = {
        "draft_window_first": pl._array(v.draft_window_first, v.n_drafts + 1, np.int64),
        "candidates": pl._array(v.candidates, v.n_windows, np.int32),
        "used": pl._array(v.used, v.n_windows, np.int32),
        "group_draft": pl._array(v.group_draft, v.n_groups, np.int32),
        "group_window": pl._array(v.group_window, v.n_groups, np.int32),
        "win_nseq": pl._array(v.win_nseq, v.n_groups, np.int32),
        "seq_len": pl._array(v.seq_len, v.n_sequences, np.int32),
        "seq_data": pl._array(v.seq_data, v.n_bases, np.uint8),
        "n_kept": v.n_kept,
    }
    if qualities is not None:
        w, n = C.c_void_p(), C.c_int64()
        L.oracle_polish_weights(C.byref(w), C.byref(n))
        out["weights"] = pl._array(w.value, n.value, np.int8)
    return 0, out


def oracle_mirror(cigar, strand):
    c = cigar.encode() if isinstance(cigar, str) else bytes(cigar)
    buf = C.create_string_buffer(2 * len(c) + 16)
    n = oracle().oracle_correct_mirror(c, len(c), ord(strand), buf, len(buf))
    return None if n < 0 else buf.raw[:n].decode()


def oracle_view(overlap, cigar, reads, view, window_length):
    """(R, cut points) of view 0 (A) or 1 (B) of one overlap, or None for a CIGAR the contract rejects."""
    o = np.ascontiguousarray(np.asarray(overlap, dtype=pl.OVERLAP_DTYPE).reshape(1))
    c = cigar.encode() if isinstance(cigar, str) else bytes(cigar)
    rb, roffs = pl._flat(reads)
    r_len = int(o[0]["query_end_position_in_read"] - o[0]["query_start_position_in_read"]) if view else \
        int(o[0]["target_end_position_in_read"] - o[0]["target_start_position_in_read"])
    d_len = int(o[0]["target_end_position_in_read"] - o[0]["target_start_position_in_read"]) if view else \
        int(o[0]["query_end_position_in_read"] - o[0]["query_start_position_in_read"])
    rbuf = C.create_string_buffer(max(1, r_len))
    cuts = np.zeros(d_len // window_length + 3, dtype=np.int64)
    n = oracle().oracle_correct_view(ptr(o), c, len(c), rb, ptr(roffs), view, window_length, rbuf,
                                     ptr(cuts))
    if n < 0:
        return None
    return rbuf.raw[:r_len], cuts[:n]


# ---------------------------------------------------------------------------------------------------------------------------
# a Python restatement of view B

def _runs(cigar):
    out, num = [], ""
    for ch in cigar:
        if ch.isdigit():
            num += ch
        else:
            out.append((int(num), ch))
            num = ""
    return out


def py_mirror(cigar, strand):
    """View B's CIGAR: I and D swapped, the runs reversed for '-'."""
    runs = [(n, {"I": "D", "D": "I"}.get(op, op)) for n, op in _runs(cigar)]
    if strand == "-":
        runs = runs[::-1]
    return "".join("%d%s" % r for r in runs)


def py_view(o, cigar, reads, view, W):
    """(R, cut points) of one view, walking the (mirrored) CIGAR one run at a time."""
    a, b = int(o["query_read_id"]), int(o["target_read_id"])
    qs, qe, ts, te = (int(o[k]) for k in ("query_start_position_in_read", "query_end_position_in_read", "target_start_position_in_read",
                                          "target_end_position_in_read"))
    strand = chr(int(o["relative_strand"]))
    if view == 0:
        ds, de, R, cg = qs, qe, bytes(reads[b][ts:te]), cigar
    else:
        ds, de, R, cg = ts, te, bytes(reads[a][qs:qe]), py_mirror(cigar, strand)
    if strand == "-":
        R = bytes(b"TGAC"[(c >> 1) & 3] for c in R[::-1])
    starts = list(range((ds // W + 1) * W, de, W))
    J, p, r, k = {}, ds, 0, 0
    for n, op in _runs(cg):
        if op == "I":
            r += n
            continue
        # the window starts this run consumes: p .. p + n - 1
        while k < len(starts) and starts[k] < p + n:
            J[starts[k]] = r + (starts[k] - p if op == "M" else 0)
            k += 1
        p += n
        if op == "M":
            r += n
    return R, np.array([0] + [J[s] for s in starts] + [len(R)], dtype=np.int64)


# ---------------------------------------------------------------------------------------------------------------------------
# read correction from proven parts

def composition(reads, window_length=500, max_depth=30, qualities=None, threshold=10.0, **mapper_kwargs):
    """Read correction restated from proven parts -> (corrected reads, outcome array, status array, used, candidates)."""
    from genomeworks_b200 import cudamapper
    reads = list(reads)
    mapper_kwargs.setdefault("filtering_parameter", 1.0)
    if reads:
        ov, cigars, _ = cudamapper.map_reads(reads, align=True, **mapper_kwargs)
    else:
        ov, cigars = np.zeros(0, dtype=pl.OVERLAP_DTYPE), []
    rc, g = oracle_correct_groups(ov, cigars, reads, window_length, max_depth, qualities, threshold)
    assert rc == 0
    if qualities is None:
        status, cons = pl.poa_groups(pl.split_groups(g), window_length, max_depth)
    else:
        status, cons = pq.poa_groups_weighted(pl.split_groups(g), pq.split_weights(g), window_length, max_depth)
    corrected, outcome, st = pl.oracle_stitch(reads, window_length, g["used"], status, cons)
    return corrected, outcome, st, g["used"], g["candidates"]


def correction_case(seed, truth_len, coverage, read_lo, read_hi, read_rate):
    """(truth, reads, segments, starts): reads of read_lo .. read_hi bases cut from a random truth at `coverage`, each with
    read_rate edits, every other one reverse-complemented; segments[i] is read i's true sequence in the read's orientation, cut
    from the truth at starts[i]."""
    rng = np.random.default_rng(seed)
    truth = pl.random_seq(rng, truth_len)
    reads, segments, starts, total = [], [], [], 0
    while total < coverage * truth_len:
        ln = int(rng.integers(read_lo, read_hi + 1))
        st = int(rng.integers(0, max(1, truth_len - ln)))
        seg = truth[st:st + ln]
        r = pl.mutate(rng, seg, read_rate)
        if len(reads) % 2:
            r, seg = pl.revcomp(r), pl.revcomp(seg)
        reads.append(r)
        segments.append(seg)
        starts.append(st)
        total += ln
    return truth, reads, segments, starts


def true_pairs(segments, starts, min_overlap):
    """The unordered read pairs whose true segments share at least min_overlap bases."""
    ends = [s + len(g) for s, g in zip(starts, segments)]
    out = set()
    for i in range(len(starts)):
        for j in range(i + 1, len(starts)):
            if min(ends[i], ends[j]) - max(starts[i], starts[j]) >= min_overlap:
                out.add((i, j))
    return out


def edit_distances(seqs, segments, band=2048):
    """The CPU oracle's banded Myers edit distance of each sequence to its segment (asserting the band holds it)."""
    import oracle_lib as ol
    out = []
    for s, g in zip(seqs, segments):
        r = ol.myers_align(s, g, band)
        assert r["is_optimal"], "the band of %d does not hold the alignment" % band
        out.append(r["edit_distance"])
    return np.array(out)


def random_correction_overlaps(seed, n, n_reads, read_len, max_run, window_length):
    """n overlaps among n_reads random reads of read_len bases, with random CIGARs: (overlaps, cigars, reads). Intervals are drawn
    so that pieces cross many windows; both strands occur; one overlap in ten repeats an earlier one's pair as (b, a) with the
    mirrored CIGAR and equal spans (a tie), one in ten repeats it as (a, b) with other intervals, and one in fifty is a self
    overlap."""
    rng = np.random.default_rng(seed)
    reads = [pl.random_seq(rng, read_len) for _ in range(n_reads)]
    W = window_length
    ov = np.zeros(n, dtype=pl.OVERLAP_DTYPE)
    cigars = []
    for i in range(n):
        u = rng.random()
        if i > 0 and u < 0.1:  # (b, a) of an earlier overlap: the same alignment seen from the target
            j = int(rng.integers(0, i))
            o = ov[j]
            ov[i] = (o["target_read_id"], o["query_read_id"], o["target_start_position_in_read"], o["query_start_position_in_read"],
                     o["target_end_position_in_read"], o["query_end_position_in_read"], o["relative_strand"], 1, 1)
            cigars.append(py_mirror(cigars[j], chr(int(o["relative_strand"]))) if cigars[j] else "")
            continue
        a = int(rng.integers(0, n_reads))
        if i > 0 and u < 0.2:  # another overlap of an earlier pair
            j = int(rng.integers(0, i))
            a = int(ov[j]["query_read_id"])
            b = int(ov[j]["target_read_id"])
        elif u < 0.22:
            b = a
        else:
            b = int((a + rng.integers(1, n_reads)) % n_reads)
        qs = int(rng.integers(0, read_len))
        qe = int(rng.integers(qs, min(read_len, qs + 4 * W + 50) + 1))
        if rng.random() < 0.2:  # snap to window edges so that full pieces occur
            qs = qs // W * W
            qe = min(read_len, -(-qe // W) * W)
        ql = qe - qs
        tl = max(0, min(read_len, ql + int(rng.integers(-ql // 4 - 1, ql // 4 + 2))))
        ts = int(rng.integers(0, read_len - tl + 1))
        if rng.random() < 0.2:
            ts = ts // W * W
        ov[i] = (a, b, qs, ts, qe, ts + tl, ord("-") if rng.random() < 0.5 else ord("+"), 1, 1)
        cigars.append(pl.random_cigar(rng, ql, tl, max_run) if ql + tl > 0 else "")
    return ov, cigars, reads
