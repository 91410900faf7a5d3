"""ctypes bindings for the CPU oracle (oracle/liboracle.so). TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

from checker_lib import load, ptr

FDIV_T = C.CFUNCTYPE(C.c_float, C.c_float, C.c_float)


def lib():
    return load("liboracle.so", {"oracle_graph_create": (C.c_void_p, None), "oracle_set_fdiv": (C.c_int, [C.c_void_p])})


def batch_config(max_seq=1024, max_seq_per_poa=100, band_width=256, band_mode=0, adaptive_storage_factor=2.0,
                 graph_length_factor=3.0, max_pred_dist=0):
    out = np.zeros(8, dtype=np.int32)
    lib().oracle_poa_batch_config(C.c_int32(max_seq), C.c_int32(max_seq_per_poa), C.c_int32(band_width), C.c_int32(band_mode),
                                  C.c_float(adaptive_storage_factor), C.c_float(graph_length_factor), C.c_int32(max_pred_dist),
                                  ptr(out))
    return out


def flatten_windows(windows):
    """windows: list of list of bytes/str -> (win_nseq, seq_len, seq_data)"""
    win_nseq = np.array([len(w) for w in windows], dtype=np.int32)
    seqs = [s.encode() if isinstance(s, str) else bytes(s) for w in windows for s in w]
    seq_len = np.array([len(s) for s in seqs], dtype=np.int32)
    data = np.frombuffer(b"".join(seqs) + b"\0", dtype=np.uint8).copy()
    return win_nseq, seq_len, data


def poa_run(windows, cfg8, msa=False, gap=-8, mismatch=-6, match=8, weights=None):
    """Runs the oracle pipeline; returns dict(consensus=list[str], coverage=list[np.ndarray], status=np.ndarray, msa=..., cells=..., nodes=...)."""
    win_nseq, seq_len, data = flatten_windows(windows)
    n = len(windows)
    mc = int(cfg8[1])
    ms = int(cfg8[5])
    cons = np.zeros((n, mc), dtype=np.uint8)
    cov = np.zeros((n, mc), dtype=np.uint16)
    status = np.zeros(n, dtype=np.int32)
    msa_buf = np.zeros((n, ms, mc), dtype=np.uint8) if msa else None
    cells = np.zeros(n, dtype=np.int64)
    nodes = np.zeros(n, dtype=np.int32)
    w = None
    if weights is not None:
        w = np.ascontiguousarray(np.concatenate([np.asarray(x, dtype=np.int8) for win in weights for x in win] + [np.zeros(1, np.int8)]))
    cfg8 = np.ascontiguousarray(cfg8, dtype=np.int32)
    lib().oracle_poa_run(C.c_int32(n), ptr(win_nseq), ptr(seq_len), ptr(data), ptr(w),
                         ptr(cfg8), C.c_int32(1 if msa else 0), C.c_int32(gap), C.c_int32(mismatch), C.c_int32(match),
                         ptr(cons), ptr(cov), ptr(status), ptr(msa_buf) if msa else None,
                         ptr(cells), ptr(nodes))
    out_c, out_cov = [], []
    for i in range(n):
        s = bytes(cons[i]).split(b"\0", 1)[0].decode()
        out_c.append(s)
        out_cov.append(cov[i, :len(s)].copy())
    res = dict(consensus=out_c, coverage=out_cov, status=status, cells=cells, nodes=nodes)
    if msa:
        rows = []
        for i in range(n):
            if status[i] != 0:
                rows.append([])
                continue
            rows.append([bytes(msa_buf[i, r]).split(b"\0", 1)[0].decode() for r in range(int(win_nseq[i]))])
        res["msa"] = rows
    return res


def poa_row_stats(windows, cfg8, gap=-8, mismatch=-6, match=8):
    """Shape of the graphs the DP rows of each window run over, over all its alignments: an int64 array [n, 4] of the largest
    predecessor row distance, the largest in-degree, the rows with a predecessor >= 64 rows back, the rows with >= 3 predecessors."""
    win_nseq, seq_len, data = flatten_windows(windows)
    out = np.zeros((len(windows), 4), dtype=np.int64)
    cfg8 = np.ascontiguousarray(cfg8, dtype=np.int32)
    lib().oracle_poa_row_stats(C.c_int32(len(windows)), ptr(win_nseq), ptr(seq_len), ptr(data),
                               ptr(cfg8), C.c_int32(gap), C.c_int32(mismatch), C.c_int32(match), ptr(out))
    return out


class OGraph:
    """Single-stage oracle graph, mirroring cudapoa/tests/basic_graph.hpp + sorted_graph.hpp."""

    def __init__(self, nodes, out_edges, sorted_graph=None, in_w_raw=None, coverage=None, alignments=None, max_nodes=3072):
        n = len(nodes)
        self.n = n
        self.max_nodes = max_nodes
        nodes_a = np.frombuffer(bytes(nodes) if not isinstance(nodes, str) else nodes.encode(), dtype=np.uint8).copy()
        off = np.zeros(n + 1, dtype=np.int32)
        adj = []
        for i, e in enumerate(out_edges):
            adj.extend(e)
            off[i + 1] = len(adj)
        adj_a = np.array(adj + [0], dtype=np.int32)
        sg = np.array(sorted_graph, dtype=np.int32) if sorted_graph is not None else None
        iw = np.ascontiguousarray(in_w_raw, dtype=np.uint16) if in_w_raw is not None else None
        cv = np.array(coverage, dtype=np.uint16) if coverage is not None else None
        self.h = C.c_void_p(lib().oracle_graph_create(C.c_int32(n), C.c_int32(max_nodes), ptr(nodes_a), ptr(sg),
                                                      ptr(off), ptr(adj_a), ptr(iw), ptr(cv)))
        if alignments is not None:
            for i, a in enumerate(alignments):
                if len(a):
                    aa = np.array(a, dtype=np.int32)
                    lib().oracle_graph_set_alignments(self.h, C.c_int32(i), C.c_int32(len(a)), ptr(aa))

    def __del__(self):
        try:
            lib().oracle_graph_destroy(self.h)
        except Exception:
            pass

    def node_count(self):
        return lib().oracle_graph_node_count(self.h)

    def out_edges(self):
        res = []
        buf = np.zeros(64, dtype=np.int32)
        for i in range(self.node_count()):
            k = lib().oracle_graph_out_edges(self.h, C.c_int32(i), ptr(buf))
            res.append([int(x) for x in buf[:k]])
        return res

    def add_alignment(self, alignment_graph, alignment_read, read, base_weights):
        ag = np.array(alignment_graph, dtype=np.int32)
        ar = np.array(alignment_read, dtype=np.int32)
        rd = np.frombuffer(read.encode() if isinstance(read, str) else bytes(read), dtype=np.uint8).copy()
        bw = np.array(base_weights, dtype=np.int8)
        return lib().oracle_graph_add_alignment(self.h, C.c_int32(len(ag)), ptr(ag), ptr(ar), ptr(rd),
                                                ptr(bw))

    def nw(self, read, mode, band_width=128, max_nodes=3072, matrix_seq_dim=136, gap=-8, mismatch=-6, match=8):
        rd = np.frombuffer((read.encode() if isinstance(read, str) else bytes(read)) + b"\0\0\0\0\0\0\0\0", dtype=np.uint8).copy()
        L = len(rd) - 8
        ag = np.zeros(max_nodes * 2 + L + 16, dtype=np.int32)
        ar = np.zeros_like(ag)
        r = lib().oracle_graph_nw(self.h, ptr(rd), C.c_int32(L), C.c_int32(mode), C.c_int32(band_width), C.c_int32(max_nodes),
                                  C.c_int32(matrix_seq_dim), C.c_int32(gap), C.c_int32(mismatch), C.c_int32(match), ptr(ag),
                                  ptr(ar))
        if r < 0:
            return r, None, None
        return r, [int(x) for x in ag[:r]], [int(x) for x in ar[:r]]

    def consensus(self, max_consensus=2048):
        buf = np.zeros(max_consensus + 2, dtype=np.uint8)
        cov = np.zeros(max_consensus + 2, dtype=np.uint16)
        st = lib().oracle_graph_consensus(self.h, C.c_int32(max_consensus), ptr(buf), ptr(cov))
        s = bytes(buf).split(b"\0", 1)[0].decode()
        return st, s, cov[:len(s)].copy()


def topsort(out_edges):
    n = len(out_edges)
    off = np.zeros(n + 1, dtype=np.int32)
    adj = []
    for i, e in enumerate(out_edges):
        adj.extend(e)
        off[i + 1] = len(adj)
    adj_a = np.array(adj + [0], dtype=np.int32)
    out = np.zeros(n, dtype=np.int32)
    lib().oracle_topsort(C.c_int32(n), ptr(off), ptr(adj_a), ptr(out))
    return [int(x) for x in out]


# ---- banded Myers aligner oracle -------------------------------------------------------------------
ACTION_CHARS_BASIC = {0: "M", 1: "M", 2: "I", 3: "D"}
ACTION_CHARS_EXT = {0: "=", 1: "X", 2: "I", 3: "D"}


def cigar_from_runs(actions, runs, extended=False):
    """AlignmentImpl::convert_to_cigar on the RLE representation (cudaaligner/src/alignment_impl.cpp:99-153)."""
    tab = ACTION_CHARS_EXT if extended else ACTION_CHARS_BASIC
    out = []
    last, cnt = None, 0
    for a, r in zip(actions, runs):
        c = tab[int(a)]
        if extended:
            out.append("%d%s" % (int(r), c))
            continue
        if c == last:
            cnt += int(r)
        else:
            if last is not None:
                out.append("%d%s" % (cnt, last))
            last, cnt = c, int(r)
    if not extended and last is not None:
        out.append("%d%s" % (cnt, last))
    return "".join(out)


def edit_distance_from_runs(actions, runs):
    """AlignmentImpl::get_edit_distance (alignment_impl.cpp:218-234)."""
    return int(sum(int(r) for a, r in zip(actions, runs) if int(a) != 0))


def myers_align(query, target, max_bandwidth, max_elements_per_matrix=0):
    q = query.encode() if isinstance(query, str) else bytes(query)
    t = target.encode() if isinstance(target, str) else bytes(target)
    n = len(q) + len(t) + 4
    actions = np.zeros(n, dtype=np.int8)
    runs = np.zeros(n, dtype=np.int32)
    status = C.c_int32(0)
    opt = C.c_int32(0)
    cells = C.c_int64(0)
    k = lib().oracle_myers_banded_align(C.c_char_p(q), C.c_int32(len(q)), C.c_char_p(t), C.c_int32(len(t)), C.c_int32(max_bandwidth),
                                        C.c_int64(max_elements_per_matrix), C.byref(status), C.byref(opt), ptr(actions),
                                        ptr(runs), C.byref(cells))
    a, r = actions[:k].copy(), runs[:k].copy()
    return dict(status=status.value, is_optimal=opt.value, actions=a, runs=r, cigar=cigar_from_runs(a, r),
                cigar_extended=cigar_from_runs(a, r, True), edit_distance=edit_distance_from_runs(a, r), cells=cells.value)


def states_to_cigar(states, extended=False):
    """AlignmentImpl::convert_to_cigar (alignment_impl.cpp:99-153) for an expanded AlignmentState vector."""
    sym = "=XID" if extended else "MMID"
    out, prev, n = [], None, 0
    for s in states:
        c = sym[int(s)]
        if c == prev:
            n += 1
        else:
            if prev is not None:
                out.append("%d%s" % (n, prev))
            prev, n = c, 1
    if prev is not None:
        out.append("%d%s" % (n, prev))
    return "".join(out)


def hirschberg_myers_align(query, target, max_query_length=None):
    """AlignerGlobalHirschbergMyers as create_aligner(max_query_length, ...) builds it -> (states ndarray, failed)."""
    q = query.encode() if isinstance(query, str) else bytes(query)
    t = target.encode() if isinstance(target, str) else bytes(target)
    mq = len(q) if max_query_length is None else max_query_length
    out = np.zeros(len(q) + len(t) + 1, dtype=np.int8)
    failed = C.c_int32(0)
    n = lib().oracle_hirschberg_myers_align(q, C.c_int32(len(q)), t, C.c_int32(len(t)), C.c_int32(mq), ptr(out), C.byref(failed))
    return out[:n].copy(), bool(failed.value)


def myers_full_align(query, target):
    """AlignerGlobalMyers (unbanded) -> states ndarray."""
    q = query.encode() if isinstance(query, str) else bytes(query)
    t = target.encode() if isinstance(target, str) else bytes(target)
    out = np.zeros(len(q) + len(t) + 1, dtype=np.int8)
    n = lib().oracle_myers_full_align(q, C.c_int32(len(q)), t, C.c_int32(len(t)), ptr(out))
    return out[:n].copy()


GLOBAL_STATS = ("cells", "leaves", "splits", "short_splits", "single_char_long", "tied_splits", "lane_rule_splits")


def global_stats(algorithm, query, target, max_query_length=None):
    """What one alignment of a fixed-size global aligner ("hirschberg_myers" at max_query_length, "myers", "ukkonen") runs: the DP
    cells as the kernels count them (GlobalAligner.last_cells sums them over a batch) and, for Hirschberg-Myers, its leaf / split
    decisions and midpoint ties -> dict over GLOBAL_STATS plus "failed"."""
    q = query.encode() if isinstance(query, str) else bytes(query)
    t = target.encode() if isinstance(target, str) else bytes(target)
    mq = len(q) if max_query_length is None else max_query_length
    alg = {"hirschberg_myers": 0, "myers": 1, "ukkonen": 2}[algorithm]
    out = np.zeros(len(GLOBAL_STATS), dtype=np.int64)
    failed = lib().oracle_global_stats(C.c_int32(alg), q, C.c_int32(len(q)), t, C.c_int32(len(t)), C.c_int32(mq), ptr(out))
    res = {k: int(v) for k, v in zip(GLOBAL_STATS, out)}
    res["failed"] = bool(failed)
    return res


def ukkonen_align(query, target, p=100):
    """AlignerGlobalUkkonen (fixed p = 100) -> states ndarray."""
    q = query.encode() if isinstance(query, str) else bytes(query)
    t = target.encode() if isinstance(target, str) else bytes(target)
    out = np.zeros(len(q) + len(t) + 1, dtype=np.int8)
    n = lib().oracle_ukkonen_align(q, C.c_int32(len(q)), t, C.c_int32(len(t)), C.c_int32(p), ptr(out))
    return out[:n].copy()
