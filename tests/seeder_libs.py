"""Checkers of the seeder: ctypes bindings for its CPU oracle (oracle/liboracle_seeder.so), the golden seed file, and the
sequence helpers the seeder's and the genome aligner's tests share: reverse complement, mutation, a rearranged pair and FASTA
text. TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import gzip
import os

import numpy as np

import extender_libs as xl
from checker_lib import load, ptr

PATTERN = "1110100110010101111"
CARE = [i for i, c in enumerate(PATTERN) if c == "1"]


def oracle():
    return load("liboracle_seeder.so", {
        "oracle_seeder_run": (C.c_int64, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64])})


def oracle_run(query, target, transition=True):
    """The seed pairs of query against target in the engine's global order (xl.SEED_DTYPE)."""
    q, t = np.ascontiguousarray(query, np.int8), np.ascontiguousarray(target, np.int8)
    L = oracle()
    n = L.oracle_seeder_run(ptr(q), len(q), ptr(t), len(t), int(bool(transition)), None, 0)
    out = np.zeros(n, dtype=xl.SEED_DTYPE)
    L.oracle_seeder_run(ptr(q), len(q), ptr(t), len(t), int(bool(transition)), ptr(out), n)
    return out


def golden_seeds():
    """sample_seed_pairs.csv as SEED_DTYPE (the CSV's columns are target, query)."""
    from genomeworks_b200 import cudaextender as ce
    with gzip.open(os.path.join(xl.GOLDEN, "sample_seed_pairs.csv.gz"), "rt") as f:
        return ce.parse_seed_pairs(f)


def pair_set(seeds):
    return set(zip(seeds["target"].tolist(), seeds["query"].tolist()))


def care_codes(seq, p):
    return [int(seq[p - 18 + c]) for c in CARE]


def reverse_complement(codes):
    c = np.asarray(codes, dtype=np.int8)[::-1].copy()
    m = (c >= 0) & (c < 4)
    c[m] = 3 - c[m]
    return c


def mutate(codes, rate, rng):
    """codes with substitutions (80 % of `rate`) and 1-3 base insertions and deletions (10 % each)."""
    out = []
    i = 0
    n = len(codes)
    while i < n:
        u = rng.random()
        if u < rate * 0.8:
            out.append((int(codes[i]) + int(rng.integers(1, 4))) % 4)
            i += 1
        elif u < rate * 0.9:
            out += [int(v) for v in rng.integers(0, 4, int(rng.integers(1, 4)))]
        elif u < rate:
            i += int(rng.integers(1, 4))
        else:
            out.append(int(codes[i]))
            i += 1
    return np.array(out, dtype=np.int8)


def rearranged_pair(seed, n=30000, rate=0.04):
    """(target, query, inverted): a random target and a diverged query in which target[a:b] is reverse-complemented in place
    (`inverted` = (a, b)) and two later pieces swap places (a translocation)."""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, 4, n).astype(np.int8)
    a, b = n // 4, n // 4 + n // 5
    c, d, e = n // 2, n // 2 + n // 6, n // 2 + n // 3
    q = np.concatenate([t[:a], reverse_complement(t[a:b]), t[b:c], t[d:e], t[c:d], t[e:]])
    return t, mutate(q, rate, rng), (a, b)


def text(codes):
    """FASTA text that encode_sequence maps back to `codes` (0-3 ACGT, 4 lowercase a, 5 N)."""
    return "".join("ACGTaN"[int(c)] for c in codes)
