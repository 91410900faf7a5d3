"""Checkers of the seed extender: ctypes bindings for the CPU oracle (oracle/liboracle_extender.so) and the reference extender
(oracle/_ref/libgwref_extender.so), the fixtures under tests/golden/cudaextender/ and the seeded synthetic cases whose
reference outputs tests/golden/make_extender_fixture.py stores. TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import gzip
import os

import numpy as np

import checker_lib
from checker_lib import load, ptr

GOLDEN = os.path.join(checker_lib.GOLDEN, "cudaextender")
REF_OUTPUTS = os.path.join(GOLDEN, "reference_extender_outputs.json.gz")
REF_LIB = os.path.join(checker_lib.REF_DIR, "libgwref_extender.so")

# the scoring matrix, X-drop and threshold of the reference's end-to-end test (cudaextender/tests/Test_CudaextenderEnd2End.cu)
SAMPLE_MATRIX = np.array([91, -114, -31, -123, -1000, -1000, -100, -9100,
                          -114, 100, -125, -31, -1000, -1000, -100, -9100,
                          -31, -125, 100, -114, -1000, -1000, -100, -9100,
                          -123, -31, -114, 91, -1000, -1000, -100, -9100,
                          -1000, -1000, -1000, -1000, -1000, -1000, -1000, -9100,
                          -1000, -1000, -1000, -1000, -1000, -1000, -1000, -9100,
                          -100, -100, -100, -100, -1000, -1000, -100, -9100,
                          -9100, -9100, -9100, -9100, -9100, -9100, -9100, -9100], dtype=np.int32)
SAMPLE_XDROP = 910
SAMPLE_THRESHOLD = 3000
# a small-score matrix: +10 match, -10 mismatch among A/C/G/T, -20 against the other codes
SIMPLE_MATRIX = np.full((8, 8), -20, dtype=np.int32)
SIMPLE_MATRIX[:4, :4] = -10
np.fill_diagonal(SIMPLE_MATRIX[:4, :4], 10)
SIMPLE_MATRIX = SIMPLE_MATRIX.ravel()

SEED_DTYPE = np.dtype([("query", np.uint32), ("target", np.uint32)])
SSP_DTYPE = np.dtype([("query", np.uint32), ("target", np.uint32), ("length", np.int32), ("score", np.int32)])

def oracle():
    return load("liboracle_extender.so", {
        "oracle_extender_seed": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                           C.c_uint32, C.c_uint32, C.c_void_p]),
        "oracle_extender_sort_unique": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
        "oracle_extender_run": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_int32, C.c_void_p])})


def oracle_seed(query, target, matrix, xdrop, no_entropy, threshold, qs, ts):
    """-> dict(query, target, length, score, kept, total) for one seed."""
    q, t, m = np.ascontiguousarray(query, np.int8), np.ascontiguousarray(target, np.int8), np.ascontiguousarray(matrix, np.int32)
    out = np.zeros(6, dtype=np.int32)
    oracle().oracle_extender_seed(ptr(q), len(q), ptr(t), len(t), ptr(m), xdrop, int(no_entropy), threshold, qs, ts, ptr(out))
    return dict(zip(("query", "target", "length", "score", "kept", "total"), (int(v) for v in out)))


def oracle_sort_unique(ssps):
    a = np.ascontiguousarray(ssps, dtype=SSP_DTYPE)
    out = np.zeros(len(a), dtype=SSP_DTYPE)
    n = oracle().oracle_extender_sort_unique(ptr(a), len(a), ptr(out))
    return out[:n]


def oracle_run(query, target, matrix, xdrop, no_entropy, threshold, seeds):
    q, t, m = np.ascontiguousarray(query, np.int8), np.ascontiguousarray(target, np.int8), np.ascontiguousarray(matrix, np.int32)
    s = np.ascontiguousarray(seeds, dtype=SEED_DTYPE)
    out = np.zeros(max(len(s), 1), dtype=SSP_DTYPE)
    n = oracle().oracle_extender_run(ptr(q), len(q), ptr(t), len(t), ptr(m), xdrop, int(no_entropy), threshold, ptr(s), len(s), ptr(out))
    return out[:n]


def ref_available():
    return os.path.exists(REF_LIB)


def ref_run(query, target, matrix, xdrop, no_entropy, threshold, seeds, reps=1, warmup=0):
    """The reference extender's device-pointer extend_async on cuda:0 -> (SSP array, ms of the `reps` calls that follow
    `warmup` untimed ones)."""
    L = load("_ref/libgwref_extender.so", {
        "ref_extender_run": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_int32, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_float), C.c_int32, C.c_int32])})
    q, t, m = np.ascontiguousarray(query, np.int8), np.ascontiguousarray(target, np.int8), np.ascontiguousarray(matrix, np.int32)
    s = np.ascontiguousarray(seeds, dtype=SEED_DTYPE)
    out = np.zeros(max(len(s), 1), dtype=SSP_DTYPE)
    n, ms = C.c_int32(0), C.c_float(0)
    rc = L.ref_extender_run(ptr(q), len(q), ptr(t), len(t), ptr(m), xdrop, int(no_entropy), threshold, ptr(s), len(s), ptr(out),
                               C.byref(n), C.byref(ms), reps, warmup)
    if rc != 0:
        raise RuntimeError("reference extender failed")
    return out[:n.value], ms.value


def sample():
    """(encoded sample.fa, seeds of sample_seed_pairs.csv, golden SSPs of sample_scored_segment_pairs.csv)."""
    from genomeworks_b200 import cudaextender as ce
    with gzip.open(os.path.join(GOLDEN, "sample.fa.gz"), "rt") as f:
        seq = "".join(line.strip() for line in f if not line.startswith(">"))
    with gzip.open(os.path.join(GOLDEN, "sample_seed_pairs.csv.gz"), "rt") as f:
        seeds = ce.parse_seed_pairs(f)
    with gzip.open(os.path.join(GOLDEN, "sample_scored_segment_pairs.csv.gz"), "rt") as f:
        golden = ce.parse_scored_segment_pairs(f)
    return ce.encode_sequence(seq), seeds, golden


def _case(name, seed, target_len, n_seeds, matrix, xdrop, threshold, no_entropy, divergence=0.15, spurious=0.5, query_prefix=0,
          masked=False, edge_seeds=False):
    from genomeworks_b200 import synth
    rng = np.random.default_rng(seed)
    target, query, seeds = synth.extender_workload(target_len, divergence, n_seeds, spurious, seed=seed)
    if query_prefix:  # unrelated bases in front of the query: homologous diagonals become negative
        query = np.concatenate([rng.integers(0, 4, query_prefix).astype(np.int8), query])
        seeds["query"] += query_prefix
    if masked:  # soft-masked / N / other codes over a homologous stretch
        a = target_len // 3
        target[a:a + 400] = rng.choice(np.array([4, 4, 4, 5, 6, 7], dtype=np.int8), 400)
        query[a:a + 300] = rng.choice(np.array([4, 4, 5, 5, 6, 7], dtype=np.int8), 300)
    if edge_seeds:
        extra = np.zeros(4, dtype=SEED_DTYPE)
        extra["query"] = [0, len(query) - 1, 0, len(query) - 1]
        extra["target"] = [0, target_len - 1, target_len - 1, 0]
        seeds = np.concatenate([seeds, extra])
    return dict(name=name, query=query, target=target, seeds=seeds, matrix=matrix, xdrop=xdrop, threshold=threshold, no_entropy=no_entropy)


def synthetic_cases():
    """The seeded cases of reference_extender_outputs.json.gz (inputs are regenerated here; only outputs are stored)."""
    return [
        _case("sample_settings", 11, 20000, 4000, SAMPLE_MATRIX, SAMPLE_XDROP, SAMPLE_THRESHOLD, False),
        _case("sample_settings_no_entropy", 11, 20000, 4000, SAMPLE_MATRIX, SAMPLE_XDROP, SAMPLE_THRESHOLD, True),
        _case("low_threshold_entropy", 12, 20000, 4000, SAMPLE_MATRIX, SAMPLE_XDROP, 1500, False, divergence=0.25),
        _case("simple_matrix_entropy_window", 13, 15000, 3000, SIMPLE_MATRIX, 60, 200, False, divergence=0.2),
        _case("xdrop_small", 14, 15000, 3000, SAMPLE_MATRIX, 200, 1000, False),
        _case("xdrop_large", 14, 15000, 3000, SAMPLE_MATRIX, 3000, 1000, False),
        _case("negative_diagonals", 15, 12000, 3000, SAMPLE_MATRIX, SAMPLE_XDROP, 2000, False, query_prefix=777),
        _case("sequence_ends", 16, 3000, 800, SIMPLE_MATRIX, 100, 100, False, divergence=0.05, edge_seeds=True),
        _case("masked_codes", 17, 15000, 3000, SAMPLE_MATRIX, SAMPLE_XDROP, 1000, False, masked=True),
        _case("masked_codes_no_entropy", 17, 15000, 3000, SIMPLE_MATRIX, 80, 150, True, masked=True, edge_seeds=True),
    ]


def ssps_on_device(ssps):
    """An SSP_DTYPE array as the n x 4 int32 CUDA tensor (query, target, length, score) the device-pointer calls take."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(ssps, dtype=SSP_DTYPE).view(np.int32).reshape(-1, 4).copy()).cuda()


def ssp_rows(a):
    return [[int(r["query"]), int(r["target"]), int(r["length"]), int(r["score"])] for r in a]


def recorded_outputs():
    return checker_lib.read_fixture(REF_OUTPUTS)
