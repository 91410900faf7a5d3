"""GPU: POA batches that stage more than 2^31 bases (DESIGN.md 15.5).

A batch counts the bases and reads it has staged, and each window's first base and first read length, in 64-bit integers. These
cases fill one batch with 1,094 windows of 2,048 reads of about 1 kb, so that base 2^31 falls inside a read in the middle of
one window and whole windows lie past it, and check every window against the same windows run in batches of at most 64 windows
(where every offset is small) and a sample of windows against the CPU oracle. Each window has its own template, so a window that
read another window's bases would give another consensus.

Cases: the v3 kernel with unit weights through add_poa_groups_flat (the threaded staging copies); the v3 kernel with weights
through one add_group call per window, the first weighted read in the first window past 2^31 (the unit-weight backfill of more
than 2^31 bytes); the traceback-mode kernel; the v3 kernel with MSA output (seq_path offsets past 4 GB).

Each case needs 8-15 GB of device memory and 7-14 GB of host memory (DESIGN.md 15.3 lists them); a machine with less skips it.
"""
import ctypes as C
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import oracle_lib as ol
import poa_window_libs as pw

pytestmark = pytest.mark.gpu

READS = 2048        # reads per window
MIN_LEN, MAX_LEN = 896, 1024
SITES = 16          # variant sites per window, one alternative base each
AFTER = 3           # whole windows past the one that holds base 2^31
SMALL = 64          # windows per batch of the small-batch runs
MAX_WEIGHT = 15     # 2 x 15 x 2048 = 61,440: no edge weight wraps in uint16_t (DESIGN.md 15.5)
TWO31 = 1 << 31
ACGT = np.frombuffer(b"ACGT", np.uint8)
KERNELS = {"tb": 0, "v3": 1}


def _a4(n):
    return (n + 3) // 4 * 4


def _plan(seed=2031):
    """Template lengths of the windows and the window k that holds base 2^31: the base lies strictly inside a read (not at its
    first byte, not in its padding) in the middle half of window k's reads, and AFTER whole windows follow window k."""
    for s in range(seed, seed + 100):
        rng = np.random.default_rng(s)
        lens = rng.integers(MIN_LEN, MAX_LEN + 1, TWO31 // (READS * MIN_LEN) + AFTER + 2)
        starts = np.concatenate([[0], np.cumsum(READS * _a4(lens))])
        k = int(np.searchsorted(starts, TWO31, side="right")) - 1
        read, inside = divmod(TWO31 - int(starts[k]), int(_a4(lens[k])))
        if READS // 4 <= read < 3 * READS // 4 and 0 < inside < lens[k]:
            return lens[:k + 1 + AFTER].astype(np.int64), k
    raise AssertionError("no plan found")


class Inputs:
    """The planned windows, flat: READS reads per window, each the window's template with the window's alternative base at each
    variant site drawn with that site's rate (0.1 .. 0.9, so the consensus takes the alternative at some sites)."""

    def __init__(self, seed=31):
        self.lens, self.k = _plan()
        n = len(self.lens)
        rng = np.random.default_rng(seed)
        self.win_nseq = np.full(n, READS, np.int32)
        self.seq_len = np.repeat(self.lens, READS).astype(np.int32)
        self.read_start = np.concatenate([[0], np.cumsum(self.seq_len.astype(np.int64))])  # in the unpadded input
        self.data = np.empty(int(self.read_start[-1]) + 1, np.uint8)
        self.data[-1] = 0
        o = 0
        for L in self.lens:
            L = int(L)
            t = rng.integers(0, 4, L, dtype=np.uint8)
            sites = rng.choice(L, SITES, replace=False)
            alt = (t[sites] + rng.integers(1, 4, SITES, dtype=np.uint8)) & 3
            take = rng.random((READS, SITES)) < rng.uniform(0.1, 0.9, SITES)
            reads = np.broadcast_to(t, (READS, L)).copy()
            reads[:, sites] = np.where(take, alt, t[sites])
            self.data[o:o + READS * L] = ACGT[reads].ravel()
            o += READS * L
        self.weights = None

    @property
    def n(self):
        return len(self.lens)

    def staged_bases(self):
        """Bases the batch stages: every read padded to 4."""
        return int((READS * _a4(self.lens)).sum())

    def add_weights(self, seed=32):
        """Weights 1 .. MAX_WEIGHT for every base of the windows past window k (the windows up to k pass NULL)."""
        if self.weights is None:
            first = int(self.read_start[(self.k + 1) * READS])
            self.weights = np.ones(len(self.data), np.int8)
            self.weights[first:-1] = np.random.default_rng(seed).integers(1, MAX_WEIGHT + 1, len(self.data) - 1 - first, dtype=np.int8)
        return self.weights

    def reads(self, w):
        """Window w as a list of bytes"""
        r0 = w * READS
        return [bytes(self.data[self.read_start[r]:self.read_start[r + 1]]) for r in range(r0, r0 + READS)]

    def read_weights(self, w):
        r0 = w * READS
        return [self.weights[self.read_start[r]:self.read_start[r + 1]] for r in range(r0, r0 + READS)]


_INPUTS = []


@pytest.fixture(scope="module")
def inputs():
    if not _INPUTS:
        _INPUTS.append(Inputs())
    return _INPUTS[0]


def _config(case):
    from genomeworks_b200 import cudapoa
    if case == "msa":
        # max_consensus_size just above the MSA width (the template length: reads differ from it by substitutions only)
        return cudapoa.make_config_explicit(MAX_LEN, MAX_LEN + 8, 3 * MAX_LEN, 256, READS, 256 + 8, "static_band")
    return cudapoa.make_config(MAX_LEN, READS, 256, "adaptive_band_traceback" if case == "traceback" else "static_band")


def _window_device_bytes(cfg, output):
    """Device bytes one window needs, from the batch's own refusal of a zero budget."""
    from genomeworks_b200 import cudapoa
    with pytest.raises(RuntimeError, match="Requires at least") as e:
        cudapoa.CudaPoaBatch(READS, MAX_LEN, 0, output_type=output, config=cfg)
    return int(str(e.value).split("Requires at least ")[1].split()[0])


def _window_host_bytes(cfg, output):
    """Pinned host bytes of one window, the large arrays of the batch's layout: sequences and weights, the read lengths, the
    consensus and coverage, the MSA rows."""
    ms, mc = cfg.max_sequences_per_poa, cfg.max_consensus_size
    return 2 * ms * _a4(cfg.max_sequence_size) + 4 * ms + 3 * mc + 256 + (ms * mc if output == "msa" else 0)


def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def _batch(cfg, output, n, stream=None):
    from genomeworks_b200 import cudapoa
    per = _window_device_bytes(cfg, output)
    b = cudapoa.CudaPoaBatch(READS, MAX_LEN, n * per + per // 2, output_type=output, config=cfg, stream=stream)
    assert b.max_poas == n
    return b


class Results:
    def __init__(self, n, cfg, output):
        mc = cfg.max_consensus_size
        self.status = np.full(n, -1, np.int32)
        if output == "msa":
            self.rows = np.zeros(n, np.int32)
            self.msa = np.zeros((n, cfg.max_sequences_per_poa, mc), np.uint8)
        else:
            self.cons = np.zeros((n, mc), np.uint8)
            self.cov = np.zeros((n, mc), np.uint16)
            self.lens = np.zeros(n, np.int32)
        self.cells = 0


def _add(batch, inp, lo, hi, how):
    """Windows lo .. hi - 1 into the batch: "flat" through add_poa_groups_flat, "groups" through one add_group call per window
    with per-read weight pointers (NULL for the windows up to k)."""
    from genomeworks_b200._lib import check, lib
    if how == "flat":
        r0, r1 = lo * READS, hi * READS
        a, z = int(inp.read_start[r0]), int(inp.read_start[r1])
        rc, added = batch.add_poa_groups_flat(inp.win_nseq[lo:hi], inp.seq_len[r0:r1], inp.data[a:z + 1])
        assert (rc, added) == (pw.SUCCESS, hi - lo)
        return
    base, wbase = inp.data.ctypes.data, inp.weights.ctypes.data
    lens = (C.c_int32 * READS)()
    for w in range(lo, hi):
        starts = inp.read_start[w * READS:(w + 1) * READS]
        seqs = (C.c_void_p * READS)(*(base + starts).tolist())
        wp = None
        if w > inp.k:
            wp = C.cast((C.c_void_p * READS)(*(wbase + starts).tolist()), C.c_void_p)
        lens[:] = inp.seq_len[w * READS:(w + 1) * READS].tolist()
        rc = check(lib().gwb200_poa_batch_add_group(batch._h, C.c_int32(READS), C.cast(seqs, C.POINTER(C.c_char_p)), wp, lens, None, None))
        assert rc == pw.SUCCESS, "window %d: add_group returned %d" % (w, rc)


def _collect(batch, res, lo, hi, output):
    from genomeworks_b200._lib import check, lib
    assert batch.total_poas == hi - lo
    if output == "msa":
        check(lib().gwb200_poa_batch_get_msa(batch._h, res.msa[lo:hi].ctypes.data, res.rows[lo:hi].ctypes.data, res.status[lo:hi].ctypes.data))
    else:
        check(lib().gwb200_poa_batch_get_consensus(batch._h, res.cons[lo:hi].ctypes.data, res.cov[lo:hi].ctypes.data, res.lens[lo:hi].ctypes.data,
                                                   res.status[lo:hi].ctypes.data))
    res.cells += batch.last_cells()


def _run_one_batch(inp, cfg, output, how):
    """Every window in one batch -> (results, kernel, score bytes)."""
    res = Results(inp.n, cfg, output)
    b = _batch(cfg, output, inp.n)
    try:
        _add(b, inp, 0, inp.n, how)
        assert b.total_poas == inp.n, "the batch split"
        b.generate_poa()
        _collect(b, res, 0, inp.n, output)
        return res, b.kernel, b.score_bytes
    finally:
        b.close()


def _run_small_batches(inp, cfg, output, how, kernel, score_bytes):
    """The same windows in batches of at most SMALL windows, each on its own stream so that they run side by side."""
    res = Results(inp.n, cfg, output)
    spans = [(lo, min(lo + SMALL, inp.n)) for lo in range(0, inp.n, SMALL)]
    batches = []
    try:
        for lo, hi in spans:
            b = _batch(cfg, output, hi - lo, stream=torch.cuda.Stream())
            batches.append(b)
            assert (b.kernel, b.score_bytes) == (kernel, score_bytes)
            _add(b, inp, lo, hi, how)
            b.generate_poa()
        for b, (lo, hi) in zip(batches, spans):
            _collect(b, res, lo, hi, output)
    finally:
        for b in batches:
            b.close()
    return res


def _first_difference(a, b):
    d = np.flatnonzero((a != b).reshape(len(a), -1).any(axis=1))
    return "%d windows differ, the first %s" % (len(d), d[:8].tolist())


def _assert_same(big, small, output):
    """Outputs first: a window that failed has an empty consensus and no MSA rows, so its status shows there too."""
    if output == "msa":
        assert np.array_equal(big.msa, small.msa), "MSA: " + _first_difference(big.msa, small.msa)
        assert np.array_equal(big.rows, small.rows), "MSA rows: " + _first_difference(big.rows, small.rows)
    else:
        assert np.array_equal(big.cons, small.cons), "consensus: " + _first_difference(big.cons, small.cons)
        assert np.array_equal(big.lens, small.lens), "consensus length: " + _first_difference(big.lens, small.lens)
        assert np.array_equal(big.cov, small.cov), "coverage: " + _first_difference(big.cov, small.cov)
    assert np.array_equal(big.status, small.status), "status: " + _first_difference(big.status, small.status)
    assert big.cells == small.cells, "DP cells: one batch %d, small batches %d" % (big.cells, small.cells)


def _sample(inp, seed=33, extra=4):
    """The first window, the one that holds base 2^31, the one after it, the last, and `extra` more."""
    must = [0, inp.k, inp.k + 1, inp.n - 1]
    rest = np.setdiff1d(np.arange(inp.n), must)
    return sorted(must + np.random.default_rng(seed).choice(rest, extra, replace=False).tolist())


def _assert_oracle(inp, cfg, output, weighted, res):
    """A sample of windows through the CPU oracle, one window per thread."""
    sample = _sample(inp)
    cfg8 = pw.cfg8(cfg)

    def one(w):
        seqs = inp.reads(w)
        wts = None
        if weighted:
            wts = [pw.explicit_weights(seqs, inp.read_weights(w) if w > inp.k else None)]
        return ol.poa_run([seqs], cfg8, msa=output == "msa", weights=wts)

    with ThreadPoolExecutor(max(1, min(len(sample), os.cpu_count() or 1))) as ex:
        orcs = list(ex.map(one, sample))
    for w, o in zip(sample, orcs):
        what = "window %d (k = %d)" % (w, inp.k)
        assert res.status[w] == int(o["status"][0]), what + ": status %d, oracle %d" % (res.status[w], int(o["status"][0]))
        if output == "msa":
            rows = [bytes(res.msa[w, r]).split(b"\0", 1)[0].decode() for r in range(res.rows[w])]
            assert rows == o["msa"][0], what + ": MSA differs from the oracle"
        else:
            assert bytes(res.cons[w, :res.lens[w]]).decode() == o["consensus"][0], what + ": consensus differs from the oracle"
            assert res.cov[w, :res.lens[w]].tolist() == o["coverage"][0].tolist(), what + ": coverage differs from the oracle"
    return sample


# case -> (output, how the windows are added, weights, kernel)
CASES = {
    "flat": ("consensus", "flat", False, "v3"),
    "weighted_groups": ("consensus", "groups", True, "v3"),
    "traceback": ("consensus", "flat", False, "tb"),
    "msa": ("msa", "flat", False, "v3"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_batch_past_2_31_bases(case, inputs, device_fdiv):
    output, how, weighted, kernel = CASES[case]
    inp = inputs
    t0 = time.time()
    staged = inp.staged_bases()
    assert staged > TWO31 and inp.n - inp.k - 1 == AFTER
    cfg = _config(case)
    # the one batch, or the small batches (each holds half a window of slack)
    per = _window_device_bytes(cfg, output)
    dev = (inp.n + inp.n // SMALL + 1) * per
    # the pinned blocks, the weights, and the MSA of both runs
    host = inp.n * _window_host_bytes(cfg, output)
    more = (inp.data.nbytes if weighted and inp.weights is None else 0) + (2 * inp.n * READS * cfg.max_consensus_size if output == "msa" else 0)
    free_dev = torch.cuda.mem_get_info()[0]
    if free_dev < dev * 1.05:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (dev / 1e9, free_dev / 1e9))
    if _mem_available() < host + more + (2 << 30):
        pytest.skip("needs %.1f GB more host memory, %.1f GB available" % ((host + more) / 1e9, _mem_available() / 1e9))
    if weighted:
        inp.add_weights()

    t1 = time.time()
    big, k_id, sb = _run_one_batch(inp, cfg, output, how)
    t2 = time.time()
    assert k_id == KERNELS[kernel]
    small = _run_small_batches(inp, cfg, output, how, k_id, sb)
    t3 = time.time()
    _assert_same(big, small, output)
    assert (big.status == 0).all(), "windows with a status: %s" % np.flatnonzero(big.status).tolist()[:8]
    sample = _assert_oracle(inp, cfg, output, weighted, big)
    t4 = time.time()
    read = (TWO31 - int((READS * _a4(inp.lens[:inp.k])).sum())) // int(_a4(inp.lens[inp.k]))
    print("%s: %d windows, %d staged bases (2^31 inside read %d of window %d), one batch's device block %.2f GB, its pinned host block about %.2f GB; "
          "one batch %.1f s, small batches %.1f s, oracle on windows %s %.1f s, whole case %.1f s" % (
              case, inp.n, staged, read, inp.k, inp.n * per / 1e9, host / 1e9, t2 - t1, t3 - t2, sample, t4 - t3, t4 - t0))
