"""ctypes bindings of the overlapper checkers and the seeded cases they share.

- oracle/liboracle_overlapper.so (this repo's CPU restatement, oracle/overlapper_oracle.cpp): always built by build();
- oracle/_ref/libgwref_overlapper.so (the unmodified reference overlapper + oracle/ref_overlapper_capi.cu): built by build() where
  the reference sources exist; only the fixture generator and tools/bench_overlapper.py load it.

Anchors are (n, 4) uint32 arrays: query read id, target read id, query position, target position. Overlaps are
cudamapper.OVERLAP_DTYPE arrays. The cases are anchor sequences given to both sides as they are, so the index's read renumbering
plays no part.
"""
import ctypes as C
import hashlib
import os

import numpy as np

import index_libs as il
from checker_lib import load, ptr, read_fixture

ROOT = il.ROOT
FIXTURE = os.path.join(il.GOLDEN, "reference_overlapper_outputs.json.gz")
INT_MAX = 2**31 - 1
FIELDS = ("query_read_id", "target_read_id", "query_start_position_in_read", "target_start_position_in_read", "query_end_position_in_read",
          "target_end_position_in_read", "relative_strand", "num_residues", "overlap_complete")
FORWARD, REVERSE = ord("+"), ord("-")
DIV_T = C.CFUNCTYPE(C.c_float, C.c_float, C.c_float)

# name -> (all_to_all, min_residues, min_overlap_len, min_bases_per_residue, min_overlap_fraction)
PARAMS = {
    "cli_a2a": (True, 3, 250, 1000, 0.8),
    "cli": (False, 3, 250, 1000, 0.8),
    "triggered_a2a": (True, 20, 50, 50, 0.9),
    "triggered": (False, 20, 50, 50, 0.9),
    "zeros": (False, 0, 0, 0, 0.0),                        # min_bases_per_residue 0: len / residues < 0 holds for none
    "zeros_a2a": (True, 0, 0, 0, 0.0),
    "negative_bases_per_residue": (False, 0, 0, -1, 0.0),  # size_t(-1): every overlap passes the residue density test
    "negative_residues": (False, -3, 0, 1000, 0.0),       # size_t(-3): no overlap has that many residues
    "negative_length": (True, 3, -250, 1000, 0.0),        # size_t(-250): no overlap is that long
}

def dtype():
    from genomeworks_b200.cudamapper import OVERLAP_DTYPE
    return OVERLAP_DTYPE


def oracle():
    return load("liboracle_overlapper.so", {
        "oracle_overlapper_run": (C.c_int64, [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_float, C.c_void_p,
                                              C.c_void_p, C.c_int64])})


def ref():
    return load("_ref/libgwref_overlapper.so", {
        "ref_overlapper_run": (C.c_void_p, [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_float, C.c_int32,
                                            C.c_int32, C.c_void_p, C.c_void_p]),
        "ref_overlapper_size": (C.c_int64, [C.c_void_p]),
        "ref_overlapper_get": (C.c_int, [C.c_void_p, C.c_void_p]),
        "ref_overlapper_free": (C.c_int, [C.c_void_p]),
        "ref_post_process": (C.c_int64, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64])})


def anchors_array(rows):
    """An (n, 4) uint32 array; positions beyond 32 bits wrap, as uint32 arithmetic does."""
    a = np.asarray(rows)
    if a.dtype != np.uint32:
        a = (np.asarray(rows, dtype=np.int64) % 2**32).astype(np.uint32)
    return np.ascontiguousarray(a.reshape(-1, 4))


def oracle_run(anchors, params, div=None):
    """The oracle's overlaps of an (n, 4) anchor array. `div` is a DIV_T callback for the fraction filter (IEEE without one)."""
    a2a, mr, mol, mbpr, frac = params
    a = anchors_array(anchors)
    cap = max(len(a) // 3, 1)
    out = np.zeros(cap, dtype=dtype())
    n = oracle().oracle_overlapper_run(ptr(a), len(a), int(a2a), mr, mol, mbpr, frac, C.cast(div, C.c_void_p) if div else None, ptr(out), cap)
    assert n <= cap
    return out[:n].copy()


def ref_run(anchors, params, reps=1, warmup=0):
    """The reference's get_overlaps on the anchors: (overlaps, device_ms, e2e_ms), the times summed over the reps timed calls."""
    a2a, mr, mol, mbpr, frac = params
    a = anchors_array(anchors)
    dms, ems = C.c_float(), C.c_float()
    h = ref().ref_overlapper_run(ptr(a), len(a), int(a2a), mr, mol, mbpr, frac, reps, warmup, C.byref(dms), C.byref(ems))
    if not h:
        raise RuntimeError("reference overlapper failed")
    out = np.zeros(ref().ref_overlapper_size(h), dtype=dtype())
    ref().ref_overlapper_get(h, ptr(out))
    ref().ref_overlapper_free(h)
    return out, dms.value, ems.value


def ref_post_process(overlaps, drop):
    src = np.ascontiguousarray(overlaps, dtype=dtype())
    out = np.zeros(len(src) + len(src) // 2, dtype=dtype())
    n = ref().ref_post_process(ptr(src), len(src), int(drop), ptr(out), len(out))
    assert n <= len(out)
    return out[:n].copy()


def rows(overlaps):
    """Overlaps as lists of nine ints (FIELDS order)."""
    return fields(overlaps).astype(np.int64).tolist()


def from_rows(rs):
    out = np.zeros(len(rs), dtype=dtype())
    for i, r in enumerate(rs):
        for f, v in zip(FIELDS, r):
            out[i][f] = v
    return out


def fields(overlaps):
    """An (n, 9) uint32 array of the nine fields (FIELDS order): the records without their padding bytes."""
    return np.stack([np.asarray(overlaps[f]).astype(np.uint32) for f in FIELDS], axis=1) if len(overlaps) else np.zeros((0, 9), np.uint32)


def digest(overlaps):
    return hashlib.sha256(np.ascontiguousarray(fields(overlaps), dtype="<u4").tobytes()).hexdigest()


def to_json(overlaps, small):
    d = {"n": int(len(overlaps))}
    if small:
        d["overlaps"] = rows(overlaps)
    else:
        d["sha256"] = digest(overlaps)
    return d


def matches(overlaps, stored):
    if len(overlaps) != stored["n"]:
        return False
    if "overlaps" in stored:
        return rows(overlaps) == stored["overlaps"]
    return digest(overlaps) == stored["sha256"]


def load_fixture():
    return read_fixture(FIXTURE)


# ---------------------------------------------------------------------------------------------------------------------------
# anchor cases

def unit_cases():
    """The reference unit tests' anchor sets (Test_CudamapperOverlapperTriggered.cu): name -> (anchors, params, expected), where
    expected lists (query read, target read, query start, query end, target start, target end) per overlap. Their calls leave
    min_overlap_fraction at 0.9 and pass min_residues, min_overlap_len and min_bases_per_residue as given."""
    line = [[1, 2, 100, 1000], [1, 2, 200, 1100], [1, 2, 300, 1200], [1, 2, 400, 1300]]
    return {
        "one_anchor": ([[0, 0, 0, 0]], (False, 0, 50, 50, 0.9), []),
        "four_anchors_one_overlap": (line, (False, 0, 0, 1000, 0.9), [(1, 2, 100, 400, 1000, 1300)]),
        "four_anchors_no_overlap": ([[1, 2, 100, 1000], [3, 4, 200, 1100], [5, 6, 300, 1200], [8, 9, 400, 1300]], (False, 0, 1000, 50, 0.9), []),
        "four_colinear_anchors_no_overlap": ([[1, 2, 100, 1000], [1, 2, 2000, 11000], [1, 2, 3000, 12000], [1, 2, 4000, 13000]],
                                             (False, 0, 50, 50, 0.9), []),
        "four_anchors_last_not_in_overlap": (line[:3] + [[1, 2, 2400, 3300]], (False, 0, 0, 1000, 0.9), [(1, 2, 100, 300, 1000, 1200)]),
        "reverse_strand": ([[1, 2, 100, 1300], [1, 2, 200, 1200], [1, 2, 300, 1100], [1, 2, 400, 1000]], (False, 0, 0, 1000, 0.9),
                           [(1, 2, 100, 400, 1000, 1300)]),
    }


def chain(q_read, t_read, q0, t0, steps, reverse=False):
    """Anchors of one chain: `steps` is a list of (dq, dt) moves from (q0, t0); reverse walks the target backwards."""
    out, q, t = [[q_read, t_read, q0, t0]], q0, t0
    for dq, dt in steps:
        q += dq
        t = t - dt if reverse else t + dt
        out.append([q_read, t_read, q, t])
    return out


def synthetic_anchors(seed, n_pairs=40, max_chains=12):
    """Sorted anchors of n_pairs read pairs. Each pair holds runs of chains along one diagonal (forward or reverse) with chain
    lengths 1..8, steps up to 149 (so chains drift), gaps that break or keep fusion, and now and then a diagonal jump."""
    rng = np.random.default_rng(seed)
    out = []
    for p in range(n_pairs):
        qr, tr = int(rng.integers(0, 30)), int(rng.integers(0, 30))
        rev = bool(rng.integers(0, 2))
        q, t = int(rng.integers(0, 5000)), int(rng.integers(200000, 300000)) if rev else int(rng.integers(0, 5000))
        for _ in range(int(rng.integers(1, max_chains))):
            L = int(rng.choice([1, 2, 3, 3, 4, 6, 8, 20]))
            steps = [(int(rng.integers(1, 150)), int(rng.integers(0, 150))) for _ in range(L - 1)]
            c = chain(qr, tr, q, t, steps, rev)
            out += c
            q, t = c[-1][2], c[-1][3]
            gap = int(rng.integers(150, 2000))
            skew = int(rng.choice([0, 50, 290, 310, 1000]))
            q += gap
            t = t - (gap + skew) if rev else t + gap + skew
            t = max(t, 0)
    a = np.asarray(out, dtype=np.int64)
    a = a[np.lexsort((a[:, 3], a[:, 2], a[:, 1], a[:, 0]))]
    return anchors_array(a)


def drift_anchors():
    """One chain whose anchors step 149 in q and t: every step continues, so it spans far more than 150; then kept chains whose
    first anchors each lie within the fusion bound of the previous one, though the first and last are far apart."""
    c = chain(0, 1, 0, 0, [(149, 149)] * 200)
    fused, q, t = [], 100000, 100000
    for k in range(12):
        fused += chain(2, 3, q, t, [(10, 10), (10, 10)])
        q += 1000
        t += 1000 + 250  # |dq| and |dt| differ by 250 per pair: fused pairwise, 3,000 apart end to end
    return anchors_array(c + fused)


def edge_anchors():
    """Chains of length exactly 2 and 3, dropped chains inside a group, a uint32 wrap of the q step (q falls by one: the step is
    2^32 - 1), read ids changing inside a run, t steps of exactly 149 and 150, and positions near 2^32."""
    a = []
    a += chain(0, 0, 0, 0, [(5, 5)])                            # length 2: dropped
    a += chain(0, 0, 1000, 1000, [(5, 5), (5, 5)])              # length 3: kept
    a += chain(0, 0, 1200, 1200, [(5, 5)])                      # length 2 inside the group: spanned, not counted
    a += chain(0, 0, 1400, 1400, [(5, 5), (5, 5), (5, 5)])      # fuses with the first kept chain
    a += chain(0, 1, 10, 10, [(100, 149), (100, 150), (1, 1), (1, 1)])
    a += [[0, 2, 500, 500], [0, 2, 499, 501], [0, 2, 498, 502], [0, 2, 600, 600], [0, 2, 610, 610], [0, 2, 620, 620]]
    a += chain(1, 1, 2**32 - 400, 2**32 - 400, [(100, 100)] * 3)
    a += chain(1, 2, 2**31 - 50, 0, [(100, 100)] * 3)
    a += chain(1, 3, 0, 2**31 + 10, [(10, 2**31 + 20), (10, 10), (10, 10)])  # a t step of -2^31 + ... wraps in int
    a += chain(2, 2, 0, 0, [(10, 10)] * 5)                      # a read against itself: all_to_all drops it
    return anchors_array(a)


def fraction_anchors(q_len, t_len, copies=4):
    """copies read pairs, each one chain whose overlap has the given query and target lengths (steps below 150)."""
    out = []
    for r in range(copies):
        k = max(3, -(-max(q_len, t_len) // 140) + 1)
        qs = np.linspace(0, q_len, k).round().astype(np.int64)
        ts = np.linspace(0, t_len, k).round().astype(np.int64)
        out += [[r, r + 1, int(q) + 10, int(t) + 20] for q, t in zip(qs, ts)]
    return anchors_array(out)


FRACTION_SHAPES = [(997, 1000), (8999, 10000), (5001, 6251), (80000, 100003), (123457, 137174)]


def fraction_params(q_len, t_len):
    """Thresholds within an ulp or two of the smaller length ratio, where the device's approximate division and the IEEE one can
    disagree."""
    r = np.float32(min(q_len, t_len)) / np.float32(max(q_len, t_len))
    out = {}
    for k, f in enumerate([np.nextafter(np.nextafter(r, np.float32(0)), np.float32(0)), np.nextafter(r, np.float32(0)), r,
                           np.nextafter(r, np.float32(1))]):
        out["fraction_%d" % k] = (False, 0, 0, 10**6, float(f))
    return out


def cases():
    """name -> dict(anchors, params (name -> tuple), small (store full arrays), device_div (the parameter sets whose output may
    hinge on the device's approximate division: the CPU's IEEE division can differ there))."""
    out = {}
    for name, (a, p, _) in unit_cases().items():
        out["unit_" + name] = dict(anchors=anchors_array(a), params={"unit": p, **PARAMS}, small=True, device_div=set())
    std = dict(PARAMS)
    for s in range(6):
        a = synthetic_anchors(100 + s)
        out["synthetic_%d" % s] = dict(anchors=a, params=std, small=True, device_div=set())
    big = synthetic_anchors(200, n_pairs=3000, max_chains=30)
    out["synthetic_large"] = dict(anchors=big, params=std, small=False, device_div=set())
    rng = np.random.default_rng(7)
    a = synthetic_anchors(300)
    out["unsorted_shuffled"] = dict(anchors=a[rng.permutation(len(a))], params=std, small=True, device_div=set())
    b = a.copy()
    i = rng.choice(len(b) - 1, 25, replace=False)
    b[[*i, *(i + 1)]] = b[[*(i + 1), *i]]
    out["unsorted_swapped_neighbours"] = dict(anchors=b, params=std, small=True, device_div=set())
    out["unsorted_reversed"] = dict(anchors=a[::-1].copy(), params=std, small=True, device_div=set())
    out["drift"] = dict(anchors=drift_anchors(), params=std, small=True, device_div=set())
    out["edges"] = dict(anchors=edge_anchors(), params=std, small=True, device_div=set())
    line = unit_cases()["four_anchors_one_overlap"][0]
    for n in range(4):
        out["n%d" % n] = dict(anchors=anchors_array(line[:n]), params=std, small=True, device_div=set())
    for q_len, t_len in FRACTION_SHAPES:
        for swap in (False, True):
            ql, tl = (t_len, q_len) if swap else (q_len, t_len)
            fp = fraction_params(ql, tl)
            out["fraction_%d_%d" % (ql, tl)] = dict(anchors=fraction_anchors(ql, tl), params=fp, small=True, device_div=set(fp))
    return out


def matcher_cases():
    """Anchors of the matcher oracle on some of the matcher's seeded cases (covid all-vs-all among them): name -> dict as
    cases(). Slower to build (the index and matcher oracles run), so kept apart."""
    import matcher_libs as ml
    mc = ml.cases()
    out = {}
    for name in ("catcaag_aagcta_k3_w2_h0", "covid_all_vs_all_F1e-05", "covid_halves", "covid_first100_n500_vs_all", "short_read_first"):
        if name not in mc:
            continue
        q, t, _, _ = ml.sketches(mc[name])
        a = ml.oracle_run(q, t)
        # in these two, an overlap's length ratio lies within an ulp of 0.9, where the approximate division decides (found by
        # comparing the oracle with the IEEE division against the stored reference outputs)
        dd = {"triggered_a2a"} if name in ("covid_halves", "covid_first100_n500_vs_all") else set()
        out["matcher_" + name] = dict(anchors=a, params={k: PARAMS[k] for k in ("cli_a2a", "cli", "triggered_a2a", "zeros")},
                                      small=len(a) < 2000, device_div=dd)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# post_process_overlaps lists

def ov(q, t, qs, qe, ts, te, strand=FORWARD, res=10, complete=1):
    return [q, t, qs, ts, qe, te, strand, res, complete]


def post_unit_lists():
    """The reference unit tests' post-processing lists (forward pairs, one pair broken by a target id, one reverse pair)."""
    a = ov(20, 22, 1000, 2000, 4000, 5000)
    b = ov(20, 22, 2100, 3100, 5100, 6100)
    return {
        "two_forward_two_fusable": [a, b, ov(55, 90, 1000, 2000, 4000, 5000), ov(55, 90, 2100, 3100, 5100, 6100)],
        "two_forward_one_fusable": [a, b, ov(55, 90, 1000, 2000, 4000, 5000), ov(55, 91, 2100, 3100, 5100, 6100)],
        "forward_and_reverse_fusable": [a, b, ov(55, 90, 1000, 2000, 4000, 5000, REVERSE), ov(55, 90, 2100, 3100, 2900, 3900, REVERSE)],
    }


def post_lists():
    """name -> list of overlap rows: the unit lists and lists at each boundary of the mergeable test."""
    out = {"unit_" + k: v for k, v in post_unit_lists().items()}
    # short gap: 499 / 500 / 501 on each side
    for g in (499, 500, 501):
        out["gap_q%d" % g] = [ov(1, 2, 0, 1000, 0, 1000), ov(1, 2, 1000 + g, 2000 + g, 1000, 2000)]
        out["gap_t%d" % g] = [ov(1, 2, 0, 1000, 0, 1000), ov(1, 2, 1000, 2000, 1000 + g, 2000 + g)]
    # gap ratio around 0.8: gaps of 1000 and 800 +- 1
    for tg in (799, 800, 801):
        out["ratio_%d" % tg] = [ov(1, 2, 0, 100, 0, 100), ov(1, 2, 1100, 1200, 100 + tg, 200 + tg)]
    # gap proportions around 0.2: a 600-base query gap against long overlaps, target gap 2000 (ratio 0.3)
    for total in (2999, 3000, 3001):
        h = total // 2
        out["proportion_%d" % total] = [ov(1, 2, 0, h, 0, total * 4), ov(1, 2, h + 600, h + 600 + (total - h), total * 4 + 2000, total * 8)]
    # zero-length overlaps: totals of 0 give NaN or infinite proportions
    out["zero_lengths"] = [ov(1, 2, 100, 100, 100, 100), ov(1, 2, 1100, 1100, 100, 100), ov(1, 2, 1100, 1100, 2100, 2100)]
    # overlapping members (the start falls before the previous end: the uint32 difference wraps to a negative int)
    out["overlapping_members"] = [ov(3, 4, 0, 1000, 0, 1000), ov(3, 4, 900, 3000, 950, 3000), ov(3, 4, 2000, 5000, 2500, 5000)]
    # runs that end at the last element, with overlap_complete differing between its last two members
    out["run_to_the_end"] = [ov(1, 2, 0, 10, 0, 10), ov(5, 6, 0, 1000, 0, 1000, complete=1), ov(5, 6, 1100, 2000, 1100, 2000, complete=0),
                             ov(5, 6, 2100, 3000, 2100, 3000, complete=1)]
    out["run_to_the_end_reverse"] = [ov(5, 6, 0, 1000, 9000, 10000, REVERSE, complete=1), ov(5, 6, 1100, 2000, 8000, 8900, REVERSE, complete=0)]
    out["empty"] = []
    out["single"] = [ov(1, 2, 0, 10, 0, 10)]
    # random lists of runs: mixed strands and ids
    rng = np.random.default_rng(11)
    for s in range(4):
        lst = []
        for _ in range(60):
            q, t = int(rng.integers(0, 4)), int(rng.integers(0, 4))
            strand = int(rng.choice([FORWARD, REVERSE]))
            qs, ts = int(rng.integers(0, 20000)), int(rng.integers(0, 20000))
            ql, tl = int(rng.integers(0, 3000)), int(rng.integers(0, 3000))
            lst.append(ov(q, t, qs, qs + ql, ts, ts + tl, strand, int(rng.integers(3, 200)), int(rng.integers(0, 2))))
        out["random_%d" % s] = lst
    return out
