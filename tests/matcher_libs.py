"""ctypes bindings of the anchor-matcher checkers and the seeded cases they share.

- oracle/liboracle_matcher.so (this repo's CPU restatement, oracle/matcher_oracle.cpp): always built by build();
- oracle/_ref/libgwref_matcher.so (the unmodified reference cudamapper index and matcher + oracle/ref_matcher_capi.cu): built by
  build() where the reference sources exist; only the fixture generator and tools/bench_matcher.py load it.

Anchors are (n, 4) uint32 arrays: query read id, target read id, query position, target position. Index sketches come from
index_libs (the index oracle), whose reads, renumbering and fixtures this module reuses.
"""
import ctypes as C
import hashlib
import os

import numpy as np

import index_libs as il
from checker_lib import load, ptr, read_fixture

ROOT = il.ROOT
FIXTURE = os.path.join(il.GOLDEN, "reference_matcher_outputs.json.gz")
INT_MAX = 2**31 - 1


def oracle():
    return load("liboracle_matcher.so", {
        "oracle_matcher_count": (C.c_int64, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
        "oracle_matcher_run": (C.c_int64, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64])})


def ref():
    return load("_ref/libgwref_matcher.so", {
        "ref_matcher_run": (C.c_void_p, [C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32,
                                         C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
        "ref_matcher_size": (C.c_int64, [C.c_void_p]),
        "ref_matcher_get": (C.c_int, [C.c_void_p, C.c_void_p]),
        "ref_matcher_free": (C.c_int, [C.c_void_p])})


def _index_arrays(s):
    return [np.ascontiguousarray(s[a]) for a in ("unique_representations", "first_occurrence_of_representations", "read_ids",
                                                 "positions_in_reads")]


def oracle_count(q, t):
    """Anchors of two sketches (dicts with the index arrays, as index_libs.oracle_run returns them), counted without building."""
    qu, qf, _, _ = _index_arrays(q)
    tu, tf, _, _ = _index_arrays(t)
    return int(oracle().oracle_matcher_count(ptr(qu), len(qu), ptr(qf), ptr(tu), len(tu), ptr(tf)))


def oracle_run(q, t):
    """The anchors of two sketches, sorted, as an (n, 4) uint32 array."""
    qu, qf, qr, qp = _index_arrays(q)
    tu, tf, tr, tp = _index_arrays(t)
    n = oracle_count(q, t)
    out = np.zeros((n, 4), dtype=np.uint32)
    got = oracle().oracle_matcher_run(ptr(qu), len(qu), ptr(qf), ptr(qr), ptr(qp), ptr(tu), len(tu), ptr(tf), ptr(tr), ptr(tp), ptr(out), n)
    assert got == n
    return out


def ref_run(all_reads, q_first, q_n, t_first, t_n, k, w, hash_representations=True, filtering_parameter=1.0, reps=1, warmup=0):
    """The reference matcher over IndexDescriptor(q_first, q_n) against IndexDescriptor(t_first, t_n) of a parser holding
    all_reads. Returns (anchors, device_ms, e2e_ms), the times summed over the reps timed calls. Never call it with two
    non-empty indices that share no representation (the reference aborts there)."""
    bases, offsets = il.flatten(all_reads)
    dms, ems = C.c_float(), C.c_float()
    h = ref().ref_matcher_run(ptr(bases), ptr(offsets), len(all_reads), q_first, q_n, t_first, t_n, k, w, 1 if hash_representations else 0,
                              filtering_parameter, reps, warmup, C.byref(dms), C.byref(ems))
    if not h:
        raise RuntimeError("reference matcher failed")
    out = np.zeros((ref().ref_matcher_size(h), 4), dtype=np.uint32)
    ref().ref_matcher_get(h, ptr(out))
    ref().ref_matcher_free(h)
    return out, dms.value, ems.value


def as_rows(anchors):
    """An (n, 4) uint32 array from a Matcher.anchors() structured array."""
    return np.stack([anchors[f].astype(np.uint32) for f in anchors.dtype.names], axis=1) if len(anchors) else np.zeros((0, 4), np.uint32)


def renumber(anchors, q_reads, q_first, t_reads, t_first, k, w):
    """Anchors with read ids mapped to the reference's numbering (index_libs.reference_read_ids); the map is monotone, so the
    order does not change."""
    out = anchors.copy()
    if len(out):
        out[:, 0] = il.reference_read_ids(q_reads, q_first, k, w)[anchors[:, 0].astype(np.int64) - q_first]
        out[:, 1] = il.reference_read_ids(t_reads, t_first, k, w)[anchors[:, 1].astype(np.int64) - t_first]
    return out


def digest(anchors):
    return hashlib.sha256(np.ascontiguousarray(anchors, dtype="<u4").tobytes()).hexdigest()


def key_bits(q_reads, q_longest, t_reads, t_longest):
    """Bits of the engine's sort key (DESIGN.md 11.2): the bit length of (N_q + 1)(N_t + 1)(L_q + 1)(L_t + 1) - 1."""
    return max(1, ((q_reads + 1) * (t_reads + 1) * (q_longest + 1) * (t_longest + 1) - 1).bit_length())


# ---------------------------------------------------------------------------------------------------------------------------
# seeded cases

def cases():
    """name -> dict(reads (all reads of the parser), q=(first, n), t=(first, n), k, w, hash, F, small)."""
    out = {}
    for fname, kws in il.SMALL_FILES.items():
        reads = il.read_fasta(os.path.join(il.GOLDEN, fname))
        for k, w in kws:
            for h in (False, True):
                out["%s_k%d_w%d_h%d" % (fname.split(".")[0], k, w, h)] = dict(reads=reads, q=(0, len(reads)), t=(0, len(reads)), k=k, w=w,
                                                                              hash=h, F=1.0, small=True)
    cat = il.read_fasta(os.path.join(il.GOLDEN, "catcaag_aagcta.fasta"))
    out["catcaag_vs_aagcta_k3_w2"] = dict(reads=cat, q=(0, 1), t=(1, 1), k=3, w=2, hash=False, F=1.0, small=True)
    cv = il.covid()
    for F in (1.0, 1e-5):
        out["covid_all_vs_all_F%g" % F] = dict(reads=cv, q=(0, 3000), t=(0, 3000), k=15, w=10, hash=True, F=F, small=False)
    # at F = 1e-5 an index of fewer reads than all 3,000 keeps no representation at all, so these run unfiltered
    out["covid_halves"] = dict(reads=cv, q=(0, 1500), t=(1500, 1500), k=15, w=10, hash=True, F=1.0, small=False)
    out["covid_first100_n500_vs_all"] = dict(reads=cv, q=(100, 500), t=(0, 3000), k=15, w=10, hash=True, F=1.0, small=False)
    ic = il.cases()
    for name in ("short_read_first", "homopolymer_palindrome_h0", "homopolymer_palindrome_h1", "every_byte_h0", "every_byte_h1",
                 "k32_hashed"):
        c = ic[name]
        out[name] = dict(reads=c["reads"], q=(c["first"], c["n"]), t=(c["first"], c["n"]), k=c["k"], w=c["w"], hash=c["hash"], F=c["F"],
                         small=False)
    short = ic["all_short"]["reads"]
    out["all_short_vs_covid"] = dict(reads=short + cv, q=(0, len(short)), t=(len(short), len(cv)), k=15, w=10, hash=True, F=1.0,
                                     small=False)
    return out


def sketches(c):
    """The index oracle's sketches of a case's query and target (read ids as this engine gives them), and their reads."""
    (qf, qn), (tf, tn) = c["q"], c["t"]
    q_reads, t_reads = c["reads"][qf:qf + qn], c["reads"][tf:tf + tn]
    q = il.oracle_run(q_reads, qf, c["k"], c["w"], c["hash"], c["F"])
    t = il.oracle_run(t_reads, tf, c["k"], c["w"], c["hash"], c["F"])
    return q, t, q_reads, t_reads


def load_fixture():
    return read_fixture(FIXTURE)


def to_json(anchors, small):
    d = {"n": int(len(anchors))}
    if small:
        d["anchors"] = anchors.astype(np.int64).tolist()
    else:
        d["sha256"] = digest(anchors)
    return d


def matches(anchors, stored):
    if len(anchors) != stored["n"]:
        return False
    if "anchors" in stored:
        return anchors.astype(np.int64).tolist() == stored["anchors"]
    return digest(anchors) == stored["sha256"]
