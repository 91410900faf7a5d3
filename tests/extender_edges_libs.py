"""Inputs of the extender edge tests (tests/test_oracle_extender_edges.py on the CPU, tests/test_gpu_extender_edges.py on the
device): asymmetric scoring schemes, ranges of exact widths at the chunk and ring edges, and best-cell ties placed across a
lane or chunk boundary. TEST INFRASTRUCTURE ONLY."""
import numpy as np

import extender_libs as xl
import gapped_extender_libs as gl

# Only (target A, query C) scores positive: reading the matrix as sub[query * 8 + target] changes every result built on it.
HAND_MATRIX = np.full(64, -7, dtype=np.int32)
HAND_MATRIX[0 * 8 + 1] = 5

# Bytes the engines read modulo 8: codes 0-7, 8-127 and negative bytes.
ODD_BYTES = np.array([4, 5, 6, 7, 8, 9, 12, 15, 64, 127, -1, -2, -5, -8, -125, -128], dtype=np.int8)


def asymmetric_matrix(rng, lo=-12, hi=6, scale=1):
    """A random 8 x 8 matrix with M[t][q] != M[q][t] somewhere, positive matches among A/C/G/T and a few positive entries off
    the diagonal; entries times `scale`."""
    while True:
        m = rng.integers(lo, hi + 1, (8, 8)).astype(np.int64)
        m[np.arange(4), np.arange(4)] = rng.integers(5, 13, 4)
        m[rng.integers(0, 8, 3), rng.integers(0, 8, 3)] = rng.integers(1, 8, 3)
        if (m != m.T).any() and ((m > 0) & ~np.eye(8, dtype=bool)).any():
            return (m * scale).astype(np.int32).ravel()


def with_odd_bytes(codes, rng, rate=0.05):
    """codes with a fraction `rate` of positions replaced by bytes outside 0..3."""
    out = np.array(codes, dtype=np.int8)
    pick = rng.random(len(out)) < rate
    out[pick] = rng.choice(ODD_BYTES, int(pick.sum()))
    return out


# Widths at which the device changes path: one chunk (256) or two, the shared ring (512) or one rerun (C = 2048), one rerun
# or two (C = 8192), two reruns or three (C = 32768).
WIDTH_EDGES = (256, 257, 512, 513, 2048, 2049, 8192, 8193)
WIDTH_PARAMS = (xl.SIMPLE_MATRIX, 1, 1, 1 << 28)  # matrix, open, extend, y-drop: at this y-drop no cell is ever pruned
WIDTH_PAIRS = ((8193, 256), (257, 8192), (2049, 512), (513, 2048))  # (left width, right width) of one anchor each


def width_case(seed=61):
    """(query, target, anchors, widths): sequences of length L and anchors whose sides reach the sequence ends with every cell
    live, so a side of m query and n target bases has a widest range of exactly min(m, n) + 1. Anchor (a, L - b) has a left
    side of a x (L - b) cells and a right side of (L - a) x b. The last four anchors are small corner cases that share the
    launches with them. widths[k] = (left width, right width) of anchor k."""
    L = max(wl + wr for wl, wr in WIDTH_PAIRS)
    rng = np.random.default_rng(seed)
    target = rng.integers(0, 4, L).astype(np.int8)
    query = target.copy()
    flip = rng.random(L) < 0.05
    query[flip] = rng.integers(0, 8, int(flip.sum()))
    anchors = [(wl - 1, L - (wr - 1)) for wl, wr in WIDTH_PAIRS] + [(0, L - 1), (L - 1, 0), (2, L - 3), (L - 3, 2)]
    widths = [(min(q, t) + 1, min(L - q, L - t) + 1) for q, t in anchors]
    return query, target, np.array(anchors, dtype=gl.ANCHOR_DTYPE), widths


# Best-cell ties: query A^p C A against target A^(p+1) C G^(p+30) from anchor (0, 0), open 1, extend 1. Cells (p + 1, p + 2)
# and (p + 2, p + 1) of anti-diagonal 2p + 3 both score 10p + 8, the side's best; the range there is [0, p + 2], so the two
# lie on either side of a lane boundary (p = 6, 14), of a chunk boundary (p = 254) and of a chunk boundary past the shared
# ring (p = 510). The smaller i wins: query [0, p + 1), target [0, p + 2).
TIE_PS = (6, 14, 254, 510)
TIE_PARAMS = (xl.SIMPLE_MATRIX, 1, 1, 1 << 20)


def tie_case(p):
    query = np.array([0] * p + [1, 0], dtype=np.int8)
    target = np.array([0] * (p + 1) + [1] + [2] * (p + 30), dtype=np.int8)
    return query, target


def periodic_cases(seed=71, n=700):
    """(name, query, target, anchors) of low-complexity sequences against themselves and against copies with one inserted or
    one deleted base: poly-A, a dinucleotide, period 3 and period 8. Anchors sit on both sides of i = 8 and 256 and at the
    ends."""
    rng = np.random.default_rng(seed)
    units = {"polyA": [0], "dinucleotide": [0, 1], "period3": [0, 1, 2], "period8": list(rng.integers(0, 4, 8))}
    out = []
    for name, unit in units.items():
        s = np.resize(np.array(unit, dtype=np.int8), n)
        for kind, q in (("same", s), ("insertion", np.insert(s, 300, 3)), ("deletion", np.delete(s, 300))):
            pts = [(0, 0), (7, 7), (8, 8), (255, 255), (256, 256), (7, 9), (256, 255), (len(q) - 1, n - 1), (len(q) // 2, n // 2 + 1)]
            out.append(("%s_%s" % (name, kind), q.copy(), s, np.array(pts, dtype=gl.ANCHOR_DTYPE)))
    return out


def limit_cases(seed=81, n=40):
    """(query, target, anchor, matrix, open, extend) at the parameter limits: entries of +-2^24, open and extend 2^24, sides of
    at most 5 bases in each sequence, so that a y-drop of 2^28 prunes nothing and the unpruned DP is the reference."""
    rng = np.random.default_rng(seed)
    big = 1 << 24
    mats = [np.where(np.eye(8, dtype=bool), big, -big).astype(np.int32).ravel(),
            rng.choice(np.array([-big, big, -big + 1, big - 1, 0], dtype=np.int64), 64).astype(np.int32),
            HAND_MATRIX * (big // 8)]
    gaps = [(big, big), (0, big), (big, 0), (1, 1)]
    out = []
    for k in range(n):
        m_left, n_left, m_right, n_right = (int(v) for v in rng.integers(0, 5, 4))
        q = rng.integers(0, 8, m_left + m_right + 1).astype(np.int8)
        t = rng.integers(0, 8, n_left + n_right + 1).astype(np.int8)
        out.append((q, t, (m_left, n_left), mats[k % len(mats)], *gaps[k % len(gaps)]))
    return out


def numpy_score(q, t, anchor, mat, o, e):
    """The unpruned DP's best of the reversed left side plus that of the right side of `anchor` = (q0, t0)."""
    q0, t0 = anchor
    return gl.numpy_best_prefix(q[:q0][::-1], t[:t0][::-1], mat, o, e) + gl.numpy_best_prefix(q[q0:], t[t0:], mat, o, e)
