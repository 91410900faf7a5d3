"""ctypes bindings for the reference-as-oracle libraries under oracle/_ref/ (built by oracle/Makefile from the
unmodified reference sources), and the stored outputs of those libraries the tests compare against. TEST / BASELINE
INFRASTRUCTURE ONLY."""
import ctypes as C
import hashlib
import json
import os

import numpy as np

from checker_lib import GOLDEN, REF_DIR, ROOT, load, ptr, read_fixture, write_fixture  # noqa: F401

GOLDEN_OUTPUTS = os.path.join(GOLDEN, "reference_outputs.json.gz")
_golden = None


def digest(x):
    """Short content hash of a string, a byte string or a sequence of integers (consensus, coverage, CIGAR, MSA rows)."""
    if isinstance(x, str):
        x = x.encode()
    elif not isinstance(x, bytes):
        x = ",".join(str(int(v)) for v in x).encode()
    return hashlib.sha256(x).hexdigest()[:16]


def recorded(key, run):
    """The reference's output for the test case `key`, as stored in tests/golden/reference_outputs.json.gz.

    `run` computes it with the unmodified reference (oracle/_ref/) and returns a JSON-serialisable value. It is only called when
    GWB200_RECORD_REFERENCE names the file to write, which is how the stored outputs are produced; otherwise the stored value is
    returned, so the comparison needs neither the reference sources nor libraries built from them."""
    global _golden
    out = os.environ.get("GWB200_RECORD_REFERENCE")
    if out:
        value = json.loads(json.dumps(run()))
        table = read_fixture(out) if os.path.exists(out) else {}
        table[key] = value
        write_fixture(out, table)
        return value
    if _golden is None:
        _golden = read_fixture(GOLDEN_OUTPUTS)
    return _golden[key]


def have_gwref():
    return os.path.exists(os.path.join(REF_DIR, "libgwref.so"))


def have_spoa():
    return os.path.exists(os.path.join(REF_DIR, "libspoa_ref.so"))


def gwref():
    return load("_ref/libgwref.so", {})


def spoa():
    return load("_ref/libspoa_ref.so", {"spoa_consensus_run": (C.c_double, None)})


def ref_poa_run(win_nseq, seq_len, seq_data, max_seq_size, max_seq_per_poa, band_width, band_mode, adaptive_storage_factor=2.0,
                graph_length_factor=3.0, max_pred_dist=0, msa=False, gap=-8, mismatch=-6, match=8, mem_fraction=0.5,
                max_windows_per_batch=0, weights=None):
    """Runs the reference cudapoa; returns dict(consensus, coverage, status, msa, timings)."""
    win_nseq = np.ascontiguousarray(win_nseq, dtype=np.int32)
    seq_len = np.ascontiguousarray(seq_len, dtype=np.int32)
    seq_data = np.ascontiguousarray(seq_data, dtype=np.uint8)
    n = len(win_nseq)
    mc = 2 * max_seq_size
    cons = np.zeros((n, mc), dtype=np.uint8)
    cov = np.zeros((n, mc), dtype=np.uint16)
    status = np.full(n, -99, dtype=np.int32)
    msa_buf = np.zeros((n, max_seq_per_poa, mc), dtype=np.uint8) if msa else None
    mc_out = C.c_int32(0)
    timings = np.zeros(3, dtype=np.float64)
    err = C.create_string_buffer(1024)
    if weights is not None:
        weights = np.ascontiguousarray(weights, dtype=np.int8)
    rc = gwref().ref_poa_run(C.c_int32(n), ptr(win_nseq), ptr(seq_len), ptr(seq_data), ptr(weights), C.c_int32(max_seq_size), C.c_int32(max_seq_per_poa),
                             C.c_int32(band_width), C.c_int32(band_mode), C.c_float(adaptive_storage_factor), C.c_float(graph_length_factor),
                             C.c_int32(max_pred_dist), C.c_int32(2 if msa else 1), C.c_int32(gap), C.c_int32(mismatch), C.c_int32(match),
                             C.c_double(mem_fraction), C.c_int32(max_windows_per_batch), ptr(cons), ptr(cov), ptr(status), ptr(msa_buf),
                             C.byref(mc_out), ptr(timings), err, C.c_int32(1024))
    if rc != 0:
        raise RuntimeError("reference cudapoa failed: " + err.value.decode())
    assert mc_out.value == mc
    out_c, out_cov = [], []
    for i in range(n):
        s = bytes(cons[i]).split(b"\0", 1)[0].decode()
        out_c.append(s)
        out_cov.append(cov[i, :len(s)].copy())
    res = dict(consensus=out_c, coverage=out_cov, status=status, timings=timings)
    if msa:
        rows = []
        for i in range(n):
            if status[i] != 0:
                rows.append([])
            else:
                rows.append([bytes(msa_buf[i, r]).split(b"\0", 1)[0].decode() for r in range(int(win_nseq[i]))])
        res["msa"] = rows
    return res


def ref_aligner_run(q_len, q_data, t_len, t_data, max_bandwidth, max_device_memory=6 << 30, cigar_stride=None):
    q_len = np.ascontiguousarray(q_len, dtype=np.int32)
    t_len = np.ascontiguousarray(t_len, dtype=np.int32)
    q_data = np.ascontiguousarray(q_data, dtype=np.uint8)
    t_data = np.ascontiguousarray(t_data, dtype=np.uint8)
    n = len(q_len)
    if cigar_stride is None:
        cigar_stride = int(12 * (int(q_len.max(initial=1)) + int(t_len.max(initial=1))) + 64)
    status = np.full(n, -99, dtype=np.int32)
    opt = np.zeros(n, dtype=np.int32)
    ed = np.zeros(n, dtype=np.int32)
    cb = np.zeros((n, cigar_stride), dtype=np.uint8)
    ce = np.zeros((n, cigar_stride), dtype=np.uint8)
    timings = np.zeros(2, dtype=np.float64)
    err = C.create_string_buffer(1024)
    rc = gwref().ref_aligner_run(C.c_int32(n), ptr(q_len), ptr(q_data), ptr(t_len), ptr(t_data), C.c_int32(max_bandwidth),
                                 C.c_int64(max_device_memory), ptr(status), ptr(opt), ptr(ed), ptr(cb), ptr(ce), C.c_int32(cigar_stride),
                                 ptr(timings), err, C.c_int32(1024))
    if rc != 0:
        raise RuntimeError("reference cudaaligner failed: " + err.value.decode())
    return dict(status=status, is_optimal=opt, edit_distance=ed,
                cigar_basic=[bytes(cb[i]).split(b"\0", 1)[0].decode() for i in range(n)],
                cigar_extended=[bytes(ce[i]).split(b"\0", 1)[0].decode() for i in range(n)], timings=timings)


def spoa_consensus(win_nseq, seq_len, seq_data, n_threads=0, match=8, mismatch=-6, gap=-8, stride=4096, want_strings=True):
    win_nseq = np.ascontiguousarray(win_nseq, dtype=np.int32)
    seq_len = np.ascontiguousarray(seq_len, dtype=np.int32)
    seq_data = np.ascontiguousarray(seq_data, dtype=np.uint8)
    n = len(win_nseq)
    buf = np.zeros((n, stride), dtype=np.uint8) if want_strings else None
    cells = C.c_double(0)
    secs = spoa().spoa_consensus_run(C.c_int32(n), ptr(win_nseq), ptr(seq_len), ptr(seq_data), C.c_int32(match), C.c_int32(mismatch),
                                     C.c_int32(gap), C.c_int32(n_threads), ptr(buf), C.c_int32(stride), C.byref(cells))
    cons = [bytes(buf[i]).split(b"\0", 1)[0].decode() for i in range(n)] if want_strings else None
    return dict(seconds=secs, cells=cells.value, consensus=cons, threads=n_threads or spoa().spoa_hardware_threads())


def ref_global_aligner_run(q_len, q_data, t_len, t_data, algorithm, max_query_length, max_target_length, cigar_stride=None):
    """algorithm 0: the reference's deprecated factory (AlignerGlobalHirschbergMyers); 1: AlignerGlobalMyers; 2: AlignerGlobalUkkonen."""
    q_len = np.ascontiguousarray(q_len, dtype=np.int32)
    t_len = np.ascontiguousarray(t_len, dtype=np.int32)
    q_data = np.ascontiguousarray(q_data, dtype=np.uint8)
    t_data = np.ascontiguousarray(t_data, dtype=np.uint8)
    n = len(q_len)
    if cigar_stride is None:
        cigar_stride = int(12 * (int(q_len.max(initial=1)) + int(t_len.max(initial=1))) + 64)
    status = np.full(n, -99, dtype=np.int32)
    opt = np.zeros(n, dtype=np.int32)
    ed = np.zeros(n, dtype=np.int32)
    cb = np.zeros((n, cigar_stride), dtype=np.uint8)
    ce = np.zeros((n, cigar_stride), dtype=np.uint8)
    timings = np.zeros(2, dtype=np.float64)
    err = C.create_string_buffer(1024)
    rc = gwref().ref_global_aligner_run(C.c_int32(n), ptr(q_len), ptr(q_data), ptr(t_len), ptr(t_data), C.c_int32(algorithm),
                                        C.c_int32(max_query_length), C.c_int32(max_target_length), ptr(status), ptr(opt), ptr(ed), ptr(cb), ptr(ce),
                                        C.c_int32(cigar_stride), ptr(timings), err, C.c_int32(1024))
    if rc != 0:
        raise RuntimeError("reference global aligner failed: " + err.value.decode())
    return dict(status=status, is_optimal=opt, edit_distance=ed,
                cigar_basic=[bytes(cb[i]).split(b"\0", 1)[0].decode() for i in range(n)],
                cigar_extended=[bytes(ce[i]).split(b"\0", 1)[0].decode() for i in range(n)], timings=timings)


def spoa_msa(seqs, match=8, mismatch=-6, gap=-8, stride=8192):
    """3rdparty/spoa MSA of one window (list of str) -> list of rows."""
    lens = np.array([len(x) for x in seqs], dtype=np.int32)
    data = np.frombuffer(("".join(seqs) + "\0").encode(), dtype=np.uint8)
    out = np.zeros((len(seqs), stride), dtype=np.uint8)
    w = spoa().spoa_msa_run(C.c_int32(len(seqs)), ptr(lens), ptr(data), C.c_int32(match), C.c_int32(mismatch), C.c_int32(gap), ptr(out),
                            C.c_int32(stride))
    if w < 0:
        raise RuntimeError("stride too small")
    return [bytes(out[i]).split(b"\0", 1)[0].decode() for i in range(len(seqs))]
