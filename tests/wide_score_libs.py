"""Checkers of the ungapped extender where its scores pass 2^31: a plain numpy restatement of DESIGN.md 9.1 for one seed (int64
cumulative sums, the running maximum "strictly greater, earliest wins", the first X-drop, the int64 entropy gate and the
saturated score), the exact int64 output of the CPU oracle, and the cases the CPU and GPU tests share. TEST INFRASTRUCTURE
ONLY."""
import ctypes as C

import numpy as np

import extender_libs as xl
from checker_lib import ptr

INT32_MAX = (1 << 31) - 1
# the entropy gate T <= total <= 3T; 3T passes INT32_MAX from this threshold on
GATE_WRAP = 715_827_883


def identity(v, mismatch=None):
    """The 8 x 8 matrix with v on the diagonal and `mismatch` (default -v) elsewhere, flattened."""
    m = np.full((8, 8), -v if mismatch is None else mismatch, dtype=np.int64)
    np.fill_diagonal(m, v)
    return m.astype(np.int32).ravel()


def oracle_seed(query, target, matrix, xdrop, no_entropy, threshold, qs, ts):
    """The CPU oracle's exact result for one seed: dict(query, target, length, score, kept, total), score and total unsaturated."""
    L = xl.oracle()
    f = L.oracle_extender_seed_wide
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_uint32, C.c_uint32,
                  C.c_void_p]
    q, t, m = np.ascontiguousarray(query, np.int8), np.ascontiguousarray(target, np.int8), np.ascontiguousarray(matrix, np.int32)
    out = np.zeros(6, dtype=np.int64)
    f(ptr(q), len(q), ptr(t), len(t), ptr(m), xdrop, int(no_entropy), threshold, qs, ts, ptr(out))
    return dict(zip(("query", "target", "length", "score", "kept", "total"), (int(v) for v in out)))


def _side(scores, start_pos, first, xdrop):
    """(maximum, its offset) of one side whose position k (offset first + k) scores scores[k]."""
    if len(scores) == 0:
        return 0, start_pos
    s = np.cumsum(scores, dtype=np.int64)
    m = np.maximum.accumulate(np.maximum(s, 0))  # the maximum starts at 0
    drops = np.flatnonzero(m - s > xdrop)
    k = int(drops[0]) if len(drops) else len(s) - 1  # the last position the maximum may come from
    best = int(m[k])
    if best == 0:
        return 0, start_pos
    return best, first + int(np.argmax(s[:k + 1] == best))  # the first position that reaches it is the one strictly above


def reference_seed(query, target, matrix, xdrop, no_entropy, threshold, qs, ts):
    """DESIGN.md 9.1 for one seed inside both sequences: dict(query, target, length, total, gated, entropy_applies, score, kept).
    score is exact where the entropy rule does not apply, and None where it does (the fixed oracle gives it there)."""
    m = np.asarray(matrix, np.int64).reshape(8, 8)
    t = np.asarray(target, np.int8).view(np.uint8) & 7
    q = np.asarray(query, np.int8).view(np.uint8) & 7
    nr = min(len(t) - ts, len(q) - qs)
    rmax, rpos = _side(m[t[ts:ts + nr], q[qs:qs + nr]], -1, 0, xdrop)
    nl = min(ts, qs)
    lmax, lpos = _side(m[t[ts - nl:ts][::-1], q[qs - nl:qs][::-1]], 0, 1, xdrop)
    total, length = rmax + lmax, rpos + lpos
    t0, q0 = ts - lpos, qs - lpos
    gated = not no_entropy and threshold <= total <= 3 * threshold
    applies = False
    if gated:
        a, b = t[t0:t0 + length + 1], q[q0:q0 + length + 1]
        applies = int(np.count_nonzero((a == b) & (a < 4))) >= 20
    score = None if applies else total
    return dict(query=q0, target=t0, length=length, total=total, gated=gated, entropy_applies=applies, score=score,
                kept=None if applies else int(score >= threshold))


def numpy_entropy_score(query, target, r):
    """int64(total * entropy) of a reference_seed result where the entropy applies, with numpy's log and plain sums (not the
    oracle's fused multiply-add): within 1 of the oracle's score."""
    t = np.asarray(target, np.int8).view(np.uint8)[r["target"]:r["target"] + r["length"] + 1] & 7
    q = np.asarray(query, np.int8).view(np.uint8)[r["query"]:r["query"] + r["length"] + 1] & 7
    counts = np.bincount(t[(t == q) & (t < 4)], minlength=4)
    p = counts[counts > 0] / (r["length"] + 1)
    return int(r["total"] * float(-(p * np.log(p)).sum() / np.log(np.float32(4.0))))


def check_seed(query, target, matrix, xdrop, no_entropy, threshold, qs, ts):
    """Asserts that the oracle's exact result equals the reference for one seed; returns the oracle's result."""
    o = oracle_seed(query, target, matrix, xdrop, no_entropy, threshold, qs, ts)
    r = reference_seed(query, target, matrix, xdrop, no_entropy, threshold, qs, ts)
    where = (qs, ts, xdrop, threshold)
    assert (o["query"], o["target"], o["length"], o["total"]) == (r["query"], r["target"], r["length"], r["total"]), (where, o, r)
    if r["entropy_applies"]:
        assert abs(o["score"] - numpy_entropy_score(query, target, r)) <= 1, (where, o, r)
        assert 0 <= o["score"] <= o["total"] and o["kept"] == int(o["score"] >= threshold), (where, o)
    else:
        assert (o["score"], o["kept"]) == (r["score"], r["kept"]), (where, o, r)
    return o


def reported(o):
    """The SSP record of a kept oracle result: the score saturated at INT32_MAX."""
    return [o["query"], o["target"], o["length"], min(o["score"], INT32_MAX)]


def sort_unique(rows):
    """DESIGN.md 9.1's per-call rule over SSP rows in seed order: stable sort by (uint32 diagonal, target, length descending,
    score descending), then keep each row that is first or not contained in its immediate predecessor on the same diagonal."""
    diag = lambda r: (r[1] - r[0]) & 0xFFFFFFFF  # noqa: E731
    v = sorted(rows, key=lambda r: (diag(r), r[1], -r[2], -r[3]))

    def contains(a, b):
        return a[1] >= b[1] and (a[1] + a[2]) & 0xFFFFFFFF <= (b[1] + b[2]) & 0xFFFFFFFF

    return [r for i, r in enumerate(v) if i == 0 or diag(r) != diag(v[i - 1]) or not (contains(r, v[i - 1]) or contains(v[i - 1], r))]


def expected_run(case):
    """The result of one extend call on a case: every seed checked against the reference, then sorted and made unique."""
    rows = []
    for s in case["seeds"]:
        o = check_seed(case["query"], case["target"], case["matrix"], case["xdrop"], case["no_entropy"], case["threshold"],
                       int(s["query"]), int(s["target"]))
        if o["kept"]:
            rows.append(reported(o))
    return sort_unique(rows)


def seeds(pairs):
    a = np.zeros(len(pairs), dtype=xl.SEED_DTYPE)
    if len(pairs):
        a["query"], a["target"] = zip(*pairs)
    return a


def case(name, query, target, matrix, xdrop, threshold, no_entropy, seed_pairs):
    return dict(name=name, query=np.ascontiguousarray(query, np.int8), target=np.ascontiguousarray(target, np.int8),
                matrix=np.ascontiguousarray(matrix, np.int32), xdrop=int(xdrop), threshold=int(threshold), no_entropy=bool(no_entropy),
                seeds=seeds(seed_pairs))


def flanked_run(rng, n, flank=40):
    """(query, target): an identical random run of n bases between flanks that mismatch at every position."""
    run = rng.integers(0, 4, n).astype(np.int8)
    fq = rng.integers(0, 4, 2 * flank).astype(np.int8)
    ft = (fq + 1 + rng.integers(0, 3, 2 * flank)) % 4
    q = np.concatenate([fq[:flank], run, fq[flank:]])
    t = np.concatenate([ft[:flank].astype(np.int8), run, ft[flank:].astype(np.int8)])
    return q, t


def identity_run_cases():
    """+-2^24 identity matrix, identical runs of 127 ... 257 bases: the seed in the middle (each side below 2^31 up to 254
    bases, their sum above it from 128), at the run's first base (all on the right side) and at its last (all on the left)."""
    rng = np.random.default_rng(31)
    out = []
    for n in (127, 128, 129, 255, 256, 257):
        q, t = flanked_run(rng, n)
        pairs = [(40 + n // 2, 40 + n // 2), (40, 40), (40 + n - 1, 40 + n - 1)]
        out.append(case("identity_run_%d" % n, q, t, identity(1 << 24), 910, 3000, True, pairs))
    return out


def homologous(rng, n, divergence):
    target = rng.integers(0, 4, n).astype(np.int8)
    query = target.copy()
    hit = rng.random(n) < divergence
    query[hit] = (query[hit] + rng.integers(1, 4, int(hit.sum()))) % 4
    return query, target


def random_matrix_cases():
    """Random asymmetric matrices on 1 %-diverged pairs: entries in [-2^24, 2^24] and over the whole int32 range, the matches
    drawn from the upper part of the range so that homologous extensions run long."""
    out = []
    for k, (lo, hi) in enumerate([(-(1 << 24), 1 << 24), (-(1 << 31), INT32_MAX)]):
        rng = np.random.default_rng(40 + k)
        for rep in range(3):
            m = rng.integers(lo, hi + 1, (8, 8), dtype=np.int64)
            m[np.arange(4), np.arange(4)] = rng.integers(hi // 4, hi + 1, 4)
            query, target = homologous(rng, 3000, 0.01)
            pos = rng.integers(0, 3000, 60)
            pairs = [(int(p), int(p)) for p in pos] + [(int(a), int(b)) for a, b in rng.integers(0, 3000, (20, 2))]
            xdrop = int(rng.choice([0, 1, 1 << 24, 1 << 30, INT32_MAX]))
            out.append(case("random_matrix_%d_%d" % (k, rep), query, target, m.astype(np.int32).ravel(), xdrop, 3000, rep == 2, pairs))
    return out


def long_match_cases():
    """Match 100 / mismatch -100 on identical pairs of 22 and 25 Mb: one side past 2^31 (seed at 0), and each side below it
    with the sum above (seed in the middle)."""
    rng = np.random.default_rng(50)
    m = identity(100)
    out = []
    for n, s in ((22_000_000, 0), (25_000_000, 12_500_000)):
        seq = rng.integers(0, 4, n).astype(np.int8)
        out.append(case("match100_%d_at_%d" % (n, s), seq, seq, m, 910, 3000, True, [(s, s)]))
    return out


def descent_cases():
    """Runs of matches (2^30) broken by descents of 2^31 - 1, 2^31 and 2^31 + 2^30, with X-drops 0, 1 and 2^31 - 1. Each
    descent is one mismatch of the asymmetric matrix or two: A/C -2^31, C/A -(2^31 - 1), G/T and T/G -2^30."""
    m = np.full((8, 8), -(1 << 31), dtype=np.int64)
    np.fill_diagonal(m, 1 << 30)
    m[1, 0] = -INT32_MAX
    m[2, 3] = m[3, 2] = -(1 << 30)
    m = m.astype(np.int32).ravel()
    steps = [[(0, 1)], [(1, 0)], [(2, 3), (3, 2)], [(2, 3), (3, 2), (2, 3)], [(1, 0), (2, 3)], [(2, 3)]]  # (target, query) codes
    rng = np.random.default_rng(60)
    out = []
    for xdrop in (0, 1, INT32_MAX):
        t, q = [], []
        for _ in range(120):
            k = int(rng.integers(1, 6))
            b = rng.integers(0, 4, k)
            t += list(b)
            q += list(b)
            for a, c in steps[int(rng.integers(0, len(steps)))]:
                t.append(a)
                q.append(c)
        pos = rng.integers(0, len(t), 150)
        out.append(case("descents_xdrop_%d" % xdrop, q, t, m, xdrop, 1, True, [(int(p), int(p)) for p in pos]))
    return out


def entropy_gate_cases():
    """Thresholds 715,827,882 (3T fits int32), 715,827,883 and 2^31 - 1 (it does not), with the +-2^24 identity matrix and
    identical mixed-base runs whose totals lie in [T, 3T]: the entropy rule runs on them."""
    rng = np.random.default_rng(70)
    out = []
    for thr in (GATE_WRAP - 1, GATE_WRAP, INT32_MAX):
        pairs, qs, ts, at = [], [], [], 0
        for n in [n for n in (43, 60, 100, 127, 128, 129, 200, 300, 380) if thr <= n << 24 <= 3 * thr]:
            q, t = flanked_run(rng, n)
            qs.append(q)
            ts.append(t)
            pairs += [(at + 40 + n // 2, at + 40 + n // 2), (at + 40, at + 40)]
            at += len(q)
        out.append(case("entropy_gate_%d" % thr, np.concatenate(qs), np.concatenate(ts), identity(1 << 24), 910, thr, False, pairs))
    # a low-entropy run of 100 (all A but 20 C): its total, 100 * 2^24, is inside [T, 3T] and its score falls below T
    q, t = flanked_run(rng, 100)
    q[40:140] = 0
    q[40:140:5] = 1
    t[40:140] = q[40:140]
    out.append(case("entropy_gate_low_entropy", q, t, identity(1 << 24), 910, GATE_WRAP, False, [(90, 90), (40, 40)]))
    return out


def saturated_ties_case():
    """Several runs on a few diagonals whose totals all pass 2^31, many seeds per run, so that the sort and the unique rule meet
    records that tie on their saturated score; runs on one diagonal, one inside another's span on a second diagonal."""
    rng = np.random.default_rng(80)
    n = 6000
    target = rng.integers(0, 4, n).astype(np.int8)
    query = (target + 1 + rng.integers(0, 3, n)).astype(np.int8) % 4  # mismatches everywhere
    pairs = []
    for start, length, shift in ((100, 300, 0), (600, 200, 0), (900, 129, 0), (2000, 1000, 7), (2300, 150, 7), (4000, 500, -11)):
        qa = start + shift
        query[qa:qa + length] = target[start:start + length]
        pairs += [(qa + int(o), start + int(o)) for o in rng.integers(0, length, 12)]
    return case("saturated_ties", query, target, identity(1 << 24), 910, 3000, True, pairs)


def cpu_cases(long=True):
    """Every case of tests/test_oracle_extender_wide_scores.py; `long` adds the 22 and 25 Mb pairs."""
    out = identity_run_cases() + random_matrix_cases() + descent_cases() + entropy_gate_cases() + [saturated_ties_case()]
    return out + (long_match_cases() if long else [])
