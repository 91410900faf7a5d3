"""ctypes bindings of the overlap-end rescue checkers and the seeded cases they share.

- oracle/liboracle_rescue.so (this repo's CPU restatement, oracle/rescue_oracle.cpp): always built by build();
- oracle/_ref/libgwref_rescue.so (the unmodified reference rescue + oracle/ref_rescue_capi.cu): built by build() where the
  reference sources exist; only the fixture generator and tools/bench_rescue.py load it. It runs on the host.

A case is a query read list, a target read list (the same list object for all-vs-all), an OVERLAP_DTYPE array, a mode (0: rescue,
1: extend once) and named (extension, required_similarity) parameter sets.
"""
import ctypes as C
import os

import numpy as np

import index_libs as il
import overlapper_libs as ol
from checker_lib import load, ptr, read_fixture

ROOT = il.ROOT
FIXTURE = os.path.join(il.GOLDEN, "reference_rescue_outputs.json.gz")
UNIT_FASTA = os.path.join(il.GOLDEN, "overlap_extension_unit.fasta")
RESCUE, EXTEND_ONCE = 0, 1
FORWARD, REVERSE = ol.FORWARD, ol.REVERSE
THIRD = float(np.float32(1 / 3))

# name -> (extension, required_similarity)
PARAMS = {
    "cli": (50, 0.5),
    "strict": (50, 0.8),
    "no_extension": (0, 0.5),
    "unlimited": (-1, 0.5),
    "ext1000": (1000, 0.5),
    "thr0": (50, 0.0),
    "thr_negative": (50, -1.0),
    "thr1": (50, 1.0),
    "thr1_5": (50, 1.5),
    "thr_nan": (50, float("nan")),
    "thr_third": (50, THIRD),
}

# overlaps, their count, query bases, offsets and count, target bases, offsets and count, extension, threshold, mode
_RUN_ARGS = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_int32]


def oracle():
    return load("liboracle_rescue.so", {"oracle_rescue_run": (C.c_int, _RUN_ARGS)})


def ref():
    return load("_ref/libgwref_rescue.so", {"ref_rescue_run": (C.c_int, _RUN_ARGS + [C.c_void_p])})


def flat(reads):
    from genomeworks_b200.cudamapper import flatten_reads
    bases, offsets = flatten_reads(reads)
    return np.ascontiguousarray(bases), np.ascontiguousarray(offsets)


def _args(overlaps, query_reads, target_reads):
    out = np.array(overlaps, dtype=ol.dtype(), copy=True).reshape(-1)
    qb, qo = flat(query_reads)
    tb, to = (qb, qo) if target_reads is query_reads else flat(target_reads)
    return out, (qb, qo, len(qo) - 1, tb, to, len(to) - 1)


def oracle_run(overlaps, query_reads, target_reads, extension, threshold, mode=RESCUE):
    """(0, updated overlaps) or (-1, the overlaps unchanged) for the arguments the contract rejects."""
    out, (qb, qo, nq, tb, to, nt) = _args(overlaps, query_reads, target_reads)
    rc = oracle().oracle_rescue_run(ptr(out), len(out), ptr(qb), ptr(qo), nq, ptr(tb), ptr(to), nt, extension, threshold, mode)
    return rc, out


def ref_run(overlaps, query_reads, target_reads, extension, threshold, mode=RESCUE):
    """(updated overlaps, the reference's host wall ms)."""
    out, (qb, qo, nq, tb, to, nt) = _args(overlaps, query_reads, target_reads)
    ms = C.c_float()
    rc = ref().ref_rescue_run(ptr(out), len(out), ptr(qb), ptr(qo), nq, ptr(tb), ptr(to), nt, extension, threshold, mode, C.byref(ms))
    if rc != 0:
        raise RuntimeError("the reference rescue threw")
    return out, ms.value


def load_fixture():
    return read_fixture(FIXTURE)


# ---------------------------------------------------------------------------------------------------------------------------
# reads and overlaps

_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def revcomp(r):
    return bytes(r).translate(_COMP)[::-1]


def reference_revcomp(r):
    """The reference's reverse complement: the middle base of an odd read is not complemented."""
    r = bytes(r)
    out = revcomp(r)
    if len(r) % 2:
        m = len(r) // 2
        out = out[:m] + r[m:m + 1] + out[m + 1:]
    return out


def ov(q, t, qs, qe, ts, te, strand=FORWARD):
    return [q, t, qs, ts, qe, te, strand, 7, 1]


def overlaps_array(rows):
    return ol.from_rows(rows)


def mutate(rng, r, divergence, alphabet=b"ACGT"):
    a = np.frombuffer(bytes(r), dtype=np.uint8).copy()
    sub = rng.random(len(a)) < divergence
    al = np.frombuffer(alphabet, dtype=np.uint8)
    a[sub] = al[rng.integers(0, len(al), int(sub.sum()))]
    return a.tobytes()


def unit_reads():
    seqs = il.read_fasta(UNIT_FASTA)
    return [seqs[0]], [seqs[1]]


def genome_reads(seed, divergence, n_reads=24, genome_len=12000, lo=1200, hi=3000):
    """Reads cut from one seeded genome, each with `divergence` of its bases substituted, every other one reverse-complemented."""
    rng = np.random.default_rng(seed)
    genome = il.random_reads(seed, 1, genome_len, genome_len)[0]
    reads = []
    for i in range(n_reads):
        L = int(rng.integers(lo, hi))
        s = int(rng.integers(0, genome_len - L))
        r = mutate(rng, genome[s:s + L], divergence)
        reads.append(revcomp(r) if i % 2 else r)
    return reads


def chain_overlaps(reads):
    """The oracle chain's all-vs-all overlaps of reads (index, matcher, overlapper with the CLI's thresholds), post-processed."""
    import matcher_libs as ml
    from genomeworks_b200.cudamapper import post_process_overlaps
    s = il.oracle_run(reads, 0, 15, 10)
    got = ol.oracle_run(ml.oracle_run(s, s), ol.PARAMS["cli_a2a"])
    return post_process_overlaps(got)


def random_overlaps(rng, q_reads, t_reads, n, strands=(FORWARD, REVERSE)):
    rows = []
    for _ in range(n):
        qi, ti = int(rng.integers(0, len(q_reads))), int(rng.integers(0, len(t_reads)))
        ql, tl = len(q_reads[qi]), len(t_reads[ti])
        qs, qe = sorted(int(x) for x in rng.integers(0, ql + 1, 2))
        ts, te = sorted(int(x) for x in rng.integers(0, tl + 1, 2))
        if rng.random() < 0.1:
            qs, qe = qe, qs  # start after end: still a valid window
        rows.append(ov(qi, ti, qs, qe, ts, te, int(rng.choice(strands))))
    return overlaps_array(rows)


def similar_pairs(seed, n, L, divergence, alphabet=b"ACGT"):
    """n read pairs (query i and target i) of length L: the target is the query with `divergence` substitutions."""
    rng = np.random.default_rng(seed)
    q = il.random_reads(seed, n, L, L, alphabet)
    t = [mutate(rng, r, divergence, alphabet) for r in q]
    return q, t


def diagonal_overlaps(rng, q_reads, t_reads, reverse, margin=(0, 120)):
    """For pair i an overlap of query i and target i on the main diagonal, with both ends `margin` bases from the reads' ends, so
    both ends have something to rescue. Where reverse[i], target i is taken as a reverse complement: the overlap is reverse and
    its positions are those of the diagonal in T' (position p of T' is position |T| - p of T)."""
    rows = []
    for i, (q, t) in enumerate(zip(q_reads, t_reads)):
        a = int(rng.integers(*margin))
        b = int(rng.integers(*margin))
        L = min(len(q), len(t))
        qs, qe = a, max(a, L - b)
        if reverse[i]:
            rows.append(ov(i, i, qs, qe, len(t) - qe, len(t) - qs, REVERSE))
        else:
            rows.append(ov(i, i, qs, qe, qs, qe))
    return overlaps_array(rows)


def diagonal_case(seed, n, L, divergence, margin=(0, 300)):
    """similar_pairs with every other target reverse-complemented, and their diagonal overlaps."""
    q, t = similar_pairs(seed, n, L, divergence)
    rev = [i % 2 == 1 for i in range(n)]
    t = [revcomp(r) if rv else r for r, rv in zip(t, rev)]
    return q, t, diagonal_overlaps(np.random.default_rng(seed), q, t, rev, margin)


def window_overlaps():
    """Windows of 0, 1, 14, 15 and 16 bases at each end, and overlaps touching either read end; identical and differing reads."""
    rng = np.random.default_rng(5)
    base = il.random_reads(5, 1, 200, 200)[0]
    q = [base, base, mutate(rng, base, 0.05)]
    t = [base, mutate(rng, base, 0.02), base[:150]]
    rows = []
    for w in (0, 1, 14, 15, 16):
        for ti in range(3):
            tl = len(t[ti])
            rows.append(ov(0, ti, w, 100, w, 100))                 # head window w
            rows.append(ov(1, ti, 40, 200 - w, 40, tl - w))       # tail window w (|T| - t_end = w)
            rows.append(ov(2, ti, w + 3, 120, tl - 120, tl - w, REVERSE))  # reverse: head window w in T' (t_end = |T| - w)
    rows += [ov(0, 0, 0, 200, 0, 200), ov(0, 2, 0, 150, 0, 150), ov(1, 1, 0, 0, 0, 0), ov(1, 1, 200, 200, 200, 200),
             ov(2, 2, 150, 150, 0, 0, REVERSE), ov(0, 0, 150, 50, 120, 60)]
    return q, t, overlaps_array(rows)


def middle_base_case():
    """Reverse overlaps where T'[|T| / 2] of an odd target is the uncomplemented middle base: a window of that one base decides
    the head, and the query holds the reference's T' (so only the reference's rule extends it). Even targets beside them."""
    rng = np.random.default_rng(9)
    rows, q, t = [], [], []
    for L in (41, 40, 101, 100):
        tgt = il.random_reads(int(rng.integers(0, 1000)), 1, L, L)[0]
        tgt = tgt[:L // 2] + b"A" + tgt[L // 2 + 1:]  # a middle base whose complement differs from it
        tp = reference_revcomp(tgt)
        m = L // 2
        q.append(tp[m:])
        t.append(tgt)
        i = len(q) - 1
        # in T': q [1, 1], t' [m + 1, m + 1]; the head window is Q[0, 1) against T'[m, m + 1)
        rows.append(ov(i, i, 1, 1, L - (m + 1), L - (m + 1), REVERSE))
        q.append(tp)
        t.append(tgt)
        j = len(q) - 1
        rows.append(ov(j, j - 1, m + 1, m + 1, L - (m + 1), L - (m + 1), REVERSE))  # a 15+ base window around the middle
        rows.append(ov(j, j - 1, m - 7, m + 8, L - (m + 8), L - (m - 7), REVERSE))
    return q, t, overlaps_array(rows)


def repeat_case():
    """Homopolymers and tandem repeats with different copy numbers: the multiset and set Jaccard similarities differ."""
    flank = il.random_reads(13, 1, 300, 300)[0]
    q, t, rows = [], [], []
    for unit, cq, ct in ((b"A", 50, 30), (b"A", 60, 60), (b"AC", 25, 12), (b"ACGTT", 10, 4), (b"ACGTT", 12, 11), (b"CAG", 20, 30)):
        rq = unit * cq
        rt = unit * ct
        # the repeat lies just before the overlap's start, and just after its end, on both reads
        qr = rq + flank[:100] + rq
        tr = rt + flank[:100] + rt
        q.append(qr)
        t.append(tr)
        i = len(q) - 1
        rows.append(ov(i, i, len(rq), len(rq) + 100, len(rt), len(rt) + 100))
        rows.append(ov(i, i, len(rq), len(rq) + 100, len(rt), len(rt) + 100, REVERSE))
    return q, t, overlaps_array(rows)


def alphabet_case():
    """N, IUPAC letters and lowercase in queries and forward targets; reverse overlaps whose targets hold uppercase IUPAC
    letters and N (complemented as themselves) and whose queries hold lowercase."""
    mixed = b"ACGTNacgtnRYKMSWBDHV"
    q, t = similar_pairs(17, 12, 400, 0.03, mixed)
    upper = [revcomp(r.upper()) for r in t[:6]]
    rng = np.random.default_rng(17)
    fw = diagonal_overlaps(rng, q, t, [False] * len(q))
    rv = diagonal_overlaps(rng, q[:6], upper, [True] * 6)
    q2 = q + q[:6]
    t2 = t + upper
    rv["query_read_id"] += 12
    rv["target_read_id"] += 12
    return q2, t2, np.concatenate([fw, rv])


def strand_byte_case():
    q, t = similar_pairs(19, 6, 300, 0.01)
    o = diagonal_overlaps(np.random.default_rng(19), q, t, [False] * 6)
    o["relative_strand"] = [0, ord("x"), 255, ord("+"), ord("F"), ord("R")]
    return q, t, o


def cases():
    """name -> dict(query_reads, target_reads, overlaps, mode, params (name -> (extension, threshold)), small)."""
    out = {}
    uq, ut = unit_reads()
    unit = overlaps_array([ov(0, 0, 1, 636, 341, 976)])
    out["unit_short_forward_head"] = dict(query_reads=uq, target_reads=ut, overlaps=unit, mode=EXTEND_ONCE,
                                          params={"unit": (50, 0.8), **PARAMS}, small=True)
    out["unit_short_forward_head_rescue"] = dict(query_reads=uq, target_reads=ut, overlaps=unit, mode=RESCUE, params=dict(PARAMS), small=True)
    for k, d in enumerate((0.0, 0.01, 0.05, 0.20)):
        reads = genome_reads(30 + k, d)
        o = chain_overlaps(reads)
        for mode, tag in ((RESCUE, ""), (EXTEND_ONCE, "_once")):
            out["chain_%g%s" % (d * 100, tag)] = dict(query_reads=reads, target_reads=reads, overlaps=o, mode=mode,
                                                      params={p: PARAMS[p] for p in ("cli", "strict", "unlimited", "ext1000", "thr_third")},
                                                      small=len(o) <= 200)
    rng = np.random.default_rng(3)
    q, t = similar_pairs(3, 10, 500, 0.02)
    out["random"] = dict(query_reads=q, target_reads=t, overlaps=random_overlaps(rng, q, t, 200), mode=RESCUE, params=dict(PARAMS),
                         small=True)
    out["random_once"] = dict(query_reads=q, target_reads=t, overlaps=random_overlaps(rng, q, t, 100), mode=EXTEND_ONCE, params=dict(PARAMS),
                              small=True)
    for d in (0.0, 0.02, 0.1):
        q, t, o = diagonal_case(int(d * 100) + 40, 16, 700, d)
        out["diagonal_%g" % (d * 100)] = dict(query_reads=q, target_reads=t, overlaps=o, mode=RESCUE, params=dict(PARAMS), small=True)
    for name, f in (("windows", window_overlaps), ("middle_base", middle_base_case), ("repeats", repeat_case), ("alphabet", alphabet_case),
                    ("strand_bytes", strand_byte_case)):
        q, t, o = f()
        out[name] = dict(query_reads=q, target_reads=t, overlaps=o, mode=RESCUE, params=dict(PARAMS), small=True)
        out[name + "_once"] = dict(query_reads=q, target_reads=t, overlaps=o, mode=EXTEND_ONCE, params=dict(PARAMS), small=True)
    q, t = similar_pairs(23, 2, 100, 0.0)
    out["n0"] = dict(query_reads=q, target_reads=t, overlaps=overlaps_array([]), mode=RESCUE, params={"cli": PARAMS["cli"]}, small=True)
    out["n1"] = dict(query_reads=q, target_reads=t, overlaps=overlaps_array([ov(1, 1, 30, 60, 30, 60)]), mode=RESCUE, params=dict(PARAMS),
                     small=True)
    return out


def to_json(overlaps, small):
    return ol.to_json(overlaps, small)


def matches(overlaps, stored):
    return ol.matches(overlaps, stored)
