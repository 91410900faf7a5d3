"""ctypes bindings of the minimizer-index checkers and the seeded cases they share.

- oracle/liboracle_index.so (this repo's CPU restatement, oracle/index_oracle.cpp): always built by build();
- oracle/_ref/libgwref_index.so (the unmodified reference cudamapper index + oracle/ref_index_capi.cu): built by build() where
  the reference sources exist; only the fixture generator and tools/bench_index.py load it.

A result is a dict with the six arrays (numpy), "number_of_reads" and "longest" (number_of_basepairs_in_longest_read).
"""
import ctypes as C
import hashlib
import os

import numpy as np

import checker_lib
from checker_lib import ROOT, load, ptr  # noqa: F401
from genomeworks_b200.cudamapper import read_fasta

GOLDEN = os.path.join(checker_lib.GOLDEN, "cudamapper")
FIXTURE = os.path.join(GOLDEN, "reference_index_outputs.json.gz")
ARRAYS = ("representations", "read_ids", "positions_in_reads", "directions_of_reads", "unique_representations",
          "first_occurrence_of_representations")
DTYPES = (np.uint64, np.uint32, np.uint32, np.uint32, np.uint64, np.uint32)


def flatten(reads):
    bs = [r.encode() if isinstance(r, str) else bytes(r) for r in reads]
    offsets = np.zeros(len(bs) + 1, dtype=np.int64)
    if bs:
        offsets[1:] = np.cumsum([len(b) for b in bs])
    bases = np.frombuffer(b"".join(bs) + b"\0", dtype=np.uint8).copy()
    return bases, offsets


def oracle():
    return load("liboracle_index.so", {
        "oracle_index_run": (C.c_void_p, [C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                          C.c_int32]),
        "oracle_index_sizes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
        "oracle_index_get": (C.c_int, [C.c_void_p] * 7),
        "oracle_index_free": (C.c_int, [C.c_void_p]),
        "oracle_index_hash": (C.c_uint64, [C.c_uint64])})


def ref():
    return load("_ref/libgwref_index.so", {
        "ref_index_run": (C.c_void_p, [C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_double, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
        "ref_index_sizes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
        "ref_index_get": (C.c_int, [C.c_void_p] * 7),
        "ref_index_free": (C.c_int, [C.c_void_p]),
        "ref_index_descriptor_hash": (C.c_uint64, [C.c_uint32, C.c_uint32])})


def _collect(L, prefix, h, nscalars):
    sizes = np.zeros(3, dtype=np.int64)
    scalars = np.zeros(nscalars, dtype=np.uint32)
    getattr(L, prefix + "_sizes")(h, ptr(sizes), ptr(scalars))
    ne, nu, nf = (int(x) for x in sizes)
    out = {name: np.zeros(n, dtype=dt) for name, n, dt in zip(ARRAYS, (ne, ne, ne, ne, nu, nf), DTYPES)}
    getattr(L, prefix + "_get")(h, *[ptr(out[a]) for a in ARRAYS])
    getattr(L, prefix + "_free")(h)
    return out, scalars


def oracle_run(reads, first_read_id, k, w, hash_representations=True, filtering_parameter=1.0, literal=False):
    """The oracle on the reads of the index (read i has id first_read_id + i)."""
    bases, offsets = flatten(reads)
    h = oracle().oracle_index_run(ptr(bases), ptr(offsets), len(reads), first_read_id, k, w,
                                  1 if hash_representations else 0, filtering_parameter, 1 if literal else 0)
    if not h:
        raise ValueError("invalid k or w")
    out, sc = _collect(oracle(), "oracle_index", h, 2)
    out["number_of_reads"], out["longest"] = int(sc[0]), int(sc[1])
    return out


def ref_run(all_reads, first_read, number_of_reads, k, w, hash_representations=True, filtering_parameter=1.0, reps=1, warmup=0):
    """The reference index over IndexDescriptor(first_read, number_of_reads) of a parser holding all_reads. Returns
    (result, device_ms, e2e_ms) for the reps timed calls."""
    bases, offsets = flatten(all_reads)
    dms, ems = C.c_float(), C.c_float()
    h = ref().ref_index_run(ptr(bases), ptr(offsets), len(all_reads), first_read, number_of_reads,
                            k, w, 1 if hash_representations else 0, filtering_parameter, reps, warmup, C.byref(dms), C.byref(ems))
    if not h:
        raise RuntimeError("reference index failed")
    out, sc = _collect(ref(), "ref_index", h, 4)
    out["number_of_reads"], out["longest"] = int(sc[0]), int(sc[3])
    return out, dms.value, ems.value


def reference_read_ids(reads, first_read_id, k, w):
    """The read ids the reference gives (compress_minimizers: first_read_id + the rank among the reads that were not skipped),
    indexed by the position of the read in `reads`; skipped reads map to their own id (they have no elements)."""
    ids = np.zeros(len(reads), dtype=np.uint32)
    rank = 0
    for i, r in enumerate(reads):
        if len(r) >= w + k - 1:
            ids[i] = first_read_id + rank
            rank += 1
        else:
            ids[i] = first_read_id + i
    return ids


def renumber(result, reads, first_read_id, k, w):
    """`result` with read ids mapped to the reference's numbering (the only documented difference)."""
    out = dict(result)
    ids = reference_read_ids(reads, first_read_id, k, w)
    out["read_ids"] = ids[result["read_ids"].astype(np.int64) - first_read_id] if len(result["read_ids"]) else result["read_ids"]
    return out


def digest(result):
    return {a: hashlib.sha256(np.ascontiguousarray(result[a], dtype=dt).astype(dt.newbyteorder("<")).tobytes()).hexdigest()
            for a, dt in zip(ARRAYS, (np.dtype(d) for d in DTYPES))}


# ---------------------------------------------------------------------------------------------------------------------------
# seeded cases

SMALL_FILES = {  # the (k, w) pairs the reference's own index tests use on each file
    "gatt.fasta": [(4, 1), (2, 3)],
    "cccatacc.fasta": [(2, 8), (3, 5)],
    "catcaag_aagcta.fasta": [(3, 5), (3, 2)],
    "aaaactgaa_gccaaag.fasta": [(2, 3)],
    "aagcta.fasta": [(3, 2)],
    "catcaag.fasta": [(3, 2)],
    "10_reads.fasta": [(4, 3), (15, 5)],
    "20_reads.fasta": [(4, 3), (15, 5)],
}


def random_reads(seed, n, lo, hi, alphabet=b"ACGT"):
    rng = np.random.default_rng(seed)
    al = np.frombuffer(alphabet, dtype=np.uint8)
    return [al[rng.integers(0, len(al), int(rng.integers(lo, hi + 1)))].tobytes() for _ in range(n)]


def covid():
    return read_fasta(os.path.join(GOLDEN, "covid-reads.fasta.gz"))


def cases():
    """name -> dict(reads (all reads of the parser), first, n, k, w, hash, F, small). The index covers reads[first:first+n]."""
    out = {}
    for fname, kws in SMALL_FILES.items():
        reads = read_fasta(os.path.join(GOLDEN, fname))
        for k, w in kws:
            for h in (False, True):
                out["%s_k%d_w%d_h%d" % (fname.split(".")[0], k, w, h)] = dict(reads=reads, first=0, n=len(reads), k=k, w=w, hash=h, F=1.0, small=True)
    aaa = read_fasta(os.path.join(GOLDEN, "aaaactgaa_gccaaag.fasta"))
    out["aaaactgaa_gccaaag_k2_w3_F0.5"] = dict(reads=aaa, first=0, n=len(aaa), k=2, w=3, hash=False, F=0.5, small=True)
    cv = covid()
    for h in (True, False):
        for F in (1.0, 1e-5, 0.5, 0.0):
            out["covid_k15_w10_h%d_F%g" % (h, F)] = dict(reads=cv, first=0, n=len(cv), k=15, w=10, hash=h, F=F, small=False)
    out["covid_first100_n500"] = dict(reads=cv, first=100, n=500, k=15, w=10, hash=True, F=1.0, small=False)
    every_byte = [bytes(np.random.default_rng(11 + i).integers(0, 256, 300 + 37 * i, dtype=np.uint8)) for i in range(6)]
    every_byte.append(bytes(range(256)) * 2)
    mixed = random_reads(12, 20, 50, 400, b"ACGTacgtNn")
    for h in (True, False):
        out["every_byte_h%d" % h] = dict(reads=every_byte, first=0, n=len(every_byte), k=15, w=10, hash=h, F=1.0, small=False)
        out["lower_n_h%d" % h] = dict(reads=mixed, first=0, n=len(mixed), k=11, w=7, hash=h, F=1.0, small=False)
    short_first = [b"ACGTACG"] + random_reads(13, 6, 200, 700) + [b"TTG"] + random_reads(14, 3, 200, 700)
    out["short_read_first"] = dict(reads=short_first, first=0, n=len(short_first), k=15, w=10, hash=True, F=1.0, small=False)
    out["all_short"] = dict(reads=random_reads(15, 5, 1, 20), first=0, n=5, k=15, w=10, hash=True, F=1.0, small=True)
    homo = [b"A" * 500, b"C" * 300, b"ACGT" * 100, b"AT" * 200, b"GC" * 150 + b"ACGTTGCA" * 30]
    for h in (True, False):
        out["homopolymer_palindrome_h%d" % h] = dict(reads=homo, first=0, n=len(homo), k=8, w=5, hash=h, F=1.0, small=False)
    rr = random_reads(16, 30, 100, 3000)
    out["k32_hashed"] = dict(reads=rr, first=0, n=len(rr), k=32, w=10, hash=True, F=1.0, small=False)
    out["k2_w1"] = dict(reads=rr[:5], first=0, n=5, k=2, w=1, hash=False, F=1.0, small=False)
    out["large_w300"] = dict(reads=rr, first=0, n=len(rr), k=15, w=300, hash=True, F=1.0, small=False)
    long1 = random_reads(17, 1, 50000, 50000) + random_reads(18, 4, 500, 3000)
    out["long_read"] = dict(reads=long1, first=0, n=len(long1), k=15, w=10, hash=True, F=1.0, small=False)
    return out


def load_fixture():
    return checker_lib.read_fixture(FIXTURE)


def to_json(result, small):
    d = {"number_of_reads": result["number_of_reads"], "longest": result["longest"], "sizes": [len(result[a]) for a in ARRAYS]}
    if small:
        d["arrays"] = {a: [int(v) for v in result[a]] for a in ARRAYS}
    else:
        d["sha256"] = digest(result)
    return d


def reference_directions_defined(case):
    """False when the reference reads some directions from overwritten shared memory: find_central_minimizers keeps one direction
    byte per window of its 512-base step (rounded up to 8) but writes one per k-mer, w - 1 more, into the positions array that
    the window pass then overwrites; a minimizer among the last k-mers of a step gets a byte of a window position as its
    direction. That happens once a read has more k-mers than that rounded window count."""
    k, w = case["k"], case["w"]
    reads = case["reads"][case["first"]:case["first"] + case["n"]]
    longest = max([len(r) for r in reads if len(r) >= w + k - 1], default=0)
    windows_per_step = 512 - (k - 1) - (w - 1)
    return longest - k + 1 <= (windows_per_step + 7) // 8 * 8


def matches(result, stored, directions=True):
    """True when `result` equals a stored reference output (full arrays or digests); directions_of_reads is left out of the
    comparison when `directions` is false."""
    if result["number_of_reads"] != stored["number_of_reads"] or result["longest"] != stored["longest"]:
        return False
    if [len(result[a]) for a in ARRAYS] != stored["sizes"]:
        return False
    names = [a for a in ARRAYS if directions or a != "directions_of_reads"]
    if "arrays" in stored:
        return all([int(v) for v in result[a]] == stored["arrays"][a] for a in names)
    d = digest(result)
    return all(d[a] == stored["sha256"][a] for a in names)
