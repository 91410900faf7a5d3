"""The fixed-size global aligners (global_kernels.cuh: Hirschberg-Myers, unbanded Myers, int16 Ukkonen) on the code paths their
shapes select, against the CPU oracle and the stored outputs of the unmodified reference classes.

What a Hirschberg-Myers alignment runs depends on more than the pair it aligns:
  - the target midpoint of a split: the first minimum score sum per lane in stride-32 order, then a shuffle tree that keeps the
    lower lane on equal sums. The rule only shows when the minimum is tied, which near-equal lengths rarely give and skewed
    shapes (one sequence 5-20x the other), homopolymers and tandem repeats often do;
  - leaf or split: a query slice below 63 bases is solved with the full matrix when (target + 1) x words fits
    ceil(max_query_length / 32) x 64 words, so max_query_length moves the decision; otherwise the slice is split again, down to
    single query characters, whose closed form runs lane-parallel over the target slice;
  - the column state of a score pass lives in shared memory up to 4 096 words (queries of 131 072 bases), in global memory beyond;
  - a score pass walks the query in 32-word chunks (slices of 32/33/64/65 words sit on the chunk edges).
Unbanded Myers walks the same chunks over the whole query; Ukkonen runs one CTA of at most 1 024 threads over a band that can be
wider (max_target_length 20 000 allows a band of 1 101 slots) and keeps int16 scores, which wrap past 32 767.

Every GPU case checks each pair's extended CIGAR, status and is_optimal against the oracle, and the batch's executed DP cells
(GlobalAligner.last_cells) against the sum of oracle_lib.global_stats' cells, which pins every leaf / split decision. The tests
without the gpu mark check with the oracle alone that each builder reaches what its case is about."""
import ctypes as C
import functools
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle_lib as ol
import ref_lib

WORD = 32
FULL_MYERS_THRESHOLD = 63   # hirschberg_myers_switch_to_myers_size
COL_SMEM_WORDS = 4096       # column state words per pv / mv in shared memory at most (aligner_capi.cu)
UKKONEN_P = 100
UKKONEN_THREADS = 1024      # threads of the Ukkonen CTA at most
REF_ALGORITHM = {"hirschberg_myers": 0, "myers": 1, "ukkonen": 2}


def words(n):
    return (n + WORD - 1) // WORD


def leaf_elems(max_query_length):
    """Words of a Hirschberg leaf matrix: ceil(max_query_length / 32) x 64."""
    return words(max_query_length) * 64


def ukkonen_bw(q, t):
    m, n = min(q, t) + 1, max(q, t) + 1
    return (1 + n - m + 2 * UKKONEN_P + 1) // 2


def ukkonen_bw_max(max_target_length):
    """The widest band an aligner admits: lengths may differ by 10 % of max_target_length."""
    diff = int(np.float32(max_target_length) * np.float32(0.1))
    return (1 + diff + 2 * UKKONEN_P + 1) // 2


# ---------------------------------------------------------------------------------------------------------------------------
# sequence builders (seeded)
# ---------------------------------------------------------------------------------------------------------------------------
_RC ={"A": "T", "C": "G", "G": "C", "T": "A"}


def rand_seq(rng, n, alphabet="ACGT"):
    a = np.array(list(alphabet))
    return "".join(a[rng.randint(0, len(a), n)])


def mutate(rng, s, n):
    """n point edits (substitution, insertion or deletion) at random positions."""
    b = list(s)
    for _ in range(n):
        if not b:
            break
        p = rng.randint(len(b))
        op = rng.randint(3)
        if op == 0:
            b[p] = "ACGT"[("ACGT".index(b[p]) + 1 + rng.randint(3)) % 4]
        elif op == 1:
            b.insert(p, "ACGT"[rng.randint(4)])
        elif len(b) > 1:
            del b[p]
    return "".join(b)


def homopolymer_runs(rng, n):
    out = []
    while sum(len(x) for x in out) < n:
        out.append("ACGT"[rng.randint(4)] * int(rng.randint(1, 13)))
    return "".join(out)[:n]


def tandem(rng, unit, n):
    return mutate(rng, (unit * (n // len(unit) + 1))[:n], max(1, n // 100))


def revcomp(s):
    return "".join(_RC[c] for c in reversed(s))


@functools.lru_cache(maxsize=None)
def skewed_pairs():
    """One sequence 5-20x longer than the other (63 .. 4 000 bases), in both orientations: independent random sequences,
    homopolymer runs, tandem repeats of one unit (period 2-6), and the short sequence an exact substring of the long one."""
    rng = np.random.RandomState(31)
    pairs = []
    for kind in ("random", "homopolymer", "tandem", "substring"):
        for query_long in (True, False):
            for _ in range(3):
                ratio = int(rng.randint(5, 21))
                short = int(rng.randint(63, 4000 // ratio + 1))
                long_ = short * ratio
                if kind == "random":
                    a, b = rand_seq(rng, long_), rand_seq(rng, short)
                elif kind == "homopolymer":
                    a, b = homopolymer_runs(rng, long_), homopolymer_runs(rng, short)
                elif kind == "tandem":
                    unit = rand_seq(rng, int(rng.randint(2, 7)))
                    a, b = tandem(rng, unit, long_), tandem(rng, unit, short)
                else:
                    a = rand_seq(rng, long_)
                    x = int(rng.randint(0, long_ - short + 1))
                    b = a[x:x + short]
                pairs.append((a, b) if query_long else (b, a))
    return pairs


def embedded_target(rng, q, tl):
    """A target of tl bases holding a mutated copy of q at a random offset (random bases around it)."""
    core = mutate(rng, q, max(1, len(q) // 10))[:tl]
    x = int(rng.randint(0, tl - len(core) + 1))
    return rand_seq(rng, x) + core + rand_seq(rng, tl - len(core) - x)


@functools.lru_cache(maxsize=None)
def leaf_edge_cases():
    """name -> (max_query_length, pairs). For each small max_query_length, queries of max_query_length and about half of it
    against targets just inside and just outside the leaf matrix ((target + 1) x words against ceil(max_q / 32) x 64), and long
    targets that make the short slices split down to single characters over many lanes. large_max_q: query slices of 62
    (a leaf, up to a 19 999-base target) and 63 bases (split) at max_query_length 20 000."""
    rng = np.random.RandomState(43)
    out = {}
    for mq in (32, 33, 40, 62, 63, 64, 65):
        pairs = []
        for ql in sorted({mq, mq // 2 + 1}):
            edge = leaf_elems(mq) // words(ql) - 1  # longest target whose matrix fits
            for tl in (edge - 1, edge, edge + 1, edge + 2, 300, 2000):
                q = rand_seq(rng, ql)
                pairs.append((q, rand_seq(rng, tl)))
                pairs.append((q, embedded_target(rng, q, tl)))
        out["max_q_%d" % mq] = (mq, pairs)
    pairs = []
    for ql in (62, 63):
        for tl in (62, 63, 500, 2000, 19999, 20000):
            q = rand_seq(rng, ql)
            pairs.append((q, embedded_target(rng, q, tl)))
    out["large_max_q"] = (20000, pairs)
    return out


HIRSCHBERG_CHUNK_QUERIES = (2048, 2049, 2050, 4096, 4097, 4160)
MYERS_CHUNK_QUERIES = (1024, 1025, 2048, 2049)


@functools.lru_cache(maxsize=None)
def chunk_pairs(algorithm):
    """Queries whose first score passes (Hirschberg: the two query halves) or whose matrix (unbanded Myers) span 32, 33, 64 and
    65 words; targets with 2 % point edits, and one unrelated target per length."""
    rng = np.random.RandomState(47 if algorithm == "hirschberg_myers" else 53)
    pairs = []
    for L in (HIRSCHBERG_CHUNK_QUERIES if algorithm == "hirschberg_myers" else MYERS_CHUNK_QUERIES):
        q = rand_seq(rng, L)
        pairs.append((q, mutate(rng, q, L // 50)))
        pairs.append((q, rand_seq(rng, int(rng.randint(L // 2, L + 1)))))
    return pairs


@functools.lru_cache(maxsize=None)
def long_query_cases():
    """name -> (max_query_length, pairs). smem_full: a 131 072-base query at max_query_length 131 072, its column state fills
    the 4 096 shared-memory words to the last. col_ws: queries of 131 073 and 140 000 bases at max_query_length 140 000 (column
    state in global memory) next to short pairs of the same launch (column state in shared memory)."""
    rng = np.random.RandomState(57)

    def long_pair(L, tl):
        q = rand_seq(rng, L)
        x = int(rng.randint(0, L - tl))
        return q, mutate(rng, q[x:x + tl], tl // 50)

    out = {"smem_full": (131072, [long_pair(131072, 5000)])}
    short = [(lambda q: (q, mutate(rng, q, 10)))(rand_seq(rng, 500)), (rand_seq(rng, 3000), rand_seq(rng, 2900)),
             (rand_seq(rng, 200), rand_seq(rng, 900))]
    out["col_ws"] = (140000, [long_pair(131073, 5000), short[0], long_pair(140000, 4000), short[1], short[2]])
    return out


@functools.lru_cache(maxsize=None)
def ukkonen_cases():
    """name -> (max_query_length = max_target_length, pairs). wide_band: max 20 000 admits length differences up to 2 000, bands
    up to 1 101 slots on 1 024 threads, in both orientations, with a narrow pair in the same launch. long: a related 36 000-base
    pair, a pair over disjoint alphabets (every cell a mismatch: the distance passes the int16 range), and 40 000 against 36 100
    (band 2 051)."""
    rng = np.random.RandomState(61)
    wide = []
    t = rand_seq(rng, 20000)
    q = mutate(rng, t[:9000] + t[11000:], 60)          # a 2 000-base deletion
    wide.append((q, t))
    q = rand_seq(rng, 20000)
    wide.append((q, mutate(rng, q[:5000] + q[6950:], 60)))  # query longer: swapped orientation
    t = rand_seq(rng, 19500)
    wide.append((mutate(rng, t[:12000] + t[13870:], 200), t))
    q = rand_seq(rng, 1000)
    wide.append((q, mutate(rng, q, 30)))
    long_ = []
    q = rand_seq(rng, 36000)
    long_.append((q, mutate(rng, q, 300)))
    long_.append((rand_seq(rng, 36000, "AC"), rand_seq(rng, 36100, "GT")))
    t = rand_seq(rng, 40000)
    long_.append((t[:20000] + t[23900:], t))
    return {"wide_band": (20000, wide), "long": (40000, long_)}


@functools.lru_cache(maxsize=None)
def revcomp_pairs(algorithm):
    """(query as added, target as added, reverse_complement_query, reverse_complement_target): the aligned sequences are a base
    and its mutated copy, whichever strand is added."""
    rng = np.random.RandomState(67 + REF_ALGORITHM[algorithm])
    out = []
    for L in (5, 63, 200, 701):
        base = rand_seq(rng, L)
        other = mutate(rng, base, max(1, L // 30))
        out.append((revcomp(base), other, True, False))
        out.append((base, revcomp(other), False, True))
        out.append((revcomp(base), revcomp(other), True, True))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# oracle and GPU runners
# ---------------------------------------------------------------------------------------------------------------------------


@functools.lru_cache(maxsize=None)
def _oracle_one(algorithm, q, t, max_q):
    if algorithm == "hirschberg_myers":
        st, failed = ol.hirschberg_myers_align(q, t, max_query_length=max_q)
    elif algorithm == "myers":
        st, failed = ol.myers_full_align(q, t), False
    else:
        st, failed = ol.ukkonen_align(q, t), False
    stats = ol.global_stats(algorithm, q, t, max_q)
    assert stats["failed"] == failed
    return dict(stats, cigar=ol.states_to_cigar(st, extended=True))


def oracle(algorithm, pairs, max_q):
    """The oracle's CIGAR and statistics of every pair (the calls release the GIL: run them on threads)."""
    with ThreadPoolExecutor(8) as ex:
        return list(ex.map(lambda p: _oracle_one(algorithm, p[0], p[1], max_q), pairs))


def new_aligner(algorithm, max_q, max_t, n):
    from genomeworks_b200 import cudaaligner
    return cudaaligner.GlobalAligner(max_q, max_t, n, algorithm)


def run(al, pairs, flags=None):
    from genomeworks_b200 import cudaaligner
    for i, (q, t) in enumerate(pairs):
        rq, rt = flags[i] if flags else (False, False)
        assert al.add_alignment(q, t, reverse_complement_query=rq, reverse_complement_target=rt) == cudaaligner.success
    al.align_all()
    al.sync_alignments()
    return al.get_alignments(), al.last_cells()


def check(res, cells, expect):
    from genomeworks_b200 import cudaaligner
    assert len(res) == len(expect)
    for i, (r, o) in enumerate(zip(res, expect)):
        assert not o["failed"]
        assert r.status == cudaaligner.success and r.is_optimal, i
        assert r.convert_to_cigar(extended=True) == o["cigar"], i
    assert cells == sum(o["cells"] for o in expect)


def align_and_check(algorithm, pairs, max_q, max_t=None):
    max_t = max_t if max_t is not None else max(len(t) for _, t in pairs)
    expect = oracle(algorithm, pairs, max_q)
    al = new_aligner(algorithm, max_q, max_t, len(pairs))
    res, cells = run(al, pairs)
    al.close()
    check(res, cells, expect)
    return res


def reference(key, pairs, algorithm, max_q, max_t):
    """Status, edit distance and extended-CIGAR digest per pair from the unmodified reference class of `algorithm`."""
    def run_ref():
        q_len = np.array([len(q) for q, _ in pairs], dtype=np.int32)
        t_len = np.array([len(t) for _, t in pairs], dtype=np.int32)
        q_data = np.frombuffer(("".join(q for q, _ in pairs) + "\0").encode(), dtype=np.uint8)
        t_data = np.frombuffer(("".join(t for _, t in pairs) + "\0").encode(), dtype=np.uint8)
        ref = ref_lib.ref_global_aligner_run(q_len, q_data, t_len, t_data, REF_ALGORITHM[algorithm], max_q, max_t)
        return dict(status=[int(x) for x in ref["status"]], edit_distance=[int(x) for x in ref["edit_distance"]],
                    cigar_extended=[ref_lib.digest(c) for c in ref["cigar_extended"]])
    return ref_lib.recorded("global_paths/" + key, run_ref)


def check_reference(key, res, pairs, algorithm, max_q, max_t=None):
    max_t = max_t if max_t is not None else max(len(t) for _, t in pairs)
    ref = reference(key, pairs, algorithm, max_q, max_t)
    assert len(ref["status"]) == len(res)
    for i, a in enumerate(res):
        assert a.status == ref["status"][i], i
        assert ref_lib.digest(a.convert_to_cigar(extended=True)) == ref["cigar_extended"][i], (i, len(pairs[i][0]), len(pairs[i][1]))
        assert a.get_edit_distance() == ref["edit_distance"][i], i


class PoisonedGlobalAligner:
    """A GlobalAligner whose device buffers come from torch uint8 tensors (the alloc / free hooks of
    gwb200_global_aligner_create). Every buffer is filled with the current poison when it is handed out and again before each
    align_all: the kernels must never read a byte they did not write in the same launch."""

    def __init__(self, algorithm, max_q, max_t, n, poison):
        import torch
        from genomeworks_b200 import cudaaligner
        from genomeworks_b200._lib import check as lib_check, lib
        self.torch = torch
        self.live = []
        self.poison = poison
        self.gen = None
        if poison == "random":
            self.gen = torch.Generator(device="cuda")
            self.gen.manual_seed(4321)
        alloc_t = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_int64)
        free_t = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int64)

        def alloc(user, nbytes):
            x = torch.empty(int(nbytes), dtype=torch.uint8, device="cuda")
            self._fill(x)
            self.live.append(x)
            return x.data_ptr()

        def free(user, ptr, nbytes):
            pass

        self._cbs = (alloc_t(alloc), free_t(free))
        al = cudaaligner.GlobalAligner.__new__(cudaaligner.GlobalAligner)
        al._h, al._alignments, al._first_unsynced, al.stream = C.c_void_p(), [], 0, None
        lib_check(lib().gwb200_global_aligner_create(C.byref(al._h), C.c_int32(cudaaligner.GlobalAligner.ALGORITHMS[algorithm]),
                                                     C.c_int32(max_q), C.c_int32(max_t), C.c_int32(n), None, C.c_int32(0),
                                                     C.cast(self._cbs[0], C.c_void_p), C.cast(self._cbs[1], C.c_void_p), None))
        self.al = al

    def _fill(self, x):
        if self.poison == "random":
            x.random_(generator=self.gen)
        else:
            x.fill_(self.poison)

    def run(self, pairs):
        from genomeworks_b200 import cudaaligner
        for q, t in pairs:
            assert self.al.add_alignment(q, t) == cudaaligner.success
        for x in self.live:
            self._fill(x)
        self.torch.cuda.synchronize()
        self.al.align_all()
        self.al.sync_alignments()
        return self.al.get_alignments(), self.al.last_cells()

    def close(self):
        self.al.close()
        self.live.clear()
        self.torch.cuda.synchronize()
        self.torch.cuda.empty_cache()


@functools.lru_cache(maxsize=None)
def poison_batches(algorithm):
    """(max_q, max_t, long batch, shorter batch) for the poisoned-workspace case of `algorithm`."""
    rng = np.random.RandomState(71 + REF_ALGORITHM[algorithm])
    if algorithm == "ukkonen":
        long_ = []
        for L in (3000, 2500, 1800):
            q = rand_seq(rng, L)
            long_.append((q, mutate(rng, q[:L - L // 12], 40)))
        short = [(lambda q: (q, mutate(rng, q, 5)))(rand_seq(rng, L)) for L in (150, 400)]
        return 3000, 3000, long_, short
    long_ = [(rand_seq(rng, 2500), rand_seq(rng, 300)), (rand_seq(rng, 200), rand_seq(rng, 3000))]
    q = rand_seq(rng, 2049)
    long_.append((q, mutate(rng, q, 60)))
    short = [(lambda q: (q, mutate(rng, q, 4)))(rand_seq(rng, L)) for L in (40, 97)] + [(rand_seq(rng, 30), rand_seq(rng, 700))]
    return 2500, 3000, long_, short


POISONS = [0x00, 0xFF, "random"]

# ---------------------------------------------------------------------------------------------------------------------------
# CPU checks of the builders (oracle only)
# ---------------------------------------------------------------------------------------------------------------------------


def test_oracle_stats_count_what_the_kernels_count():
    """A x 50 against A x 400: at max_query_length 50 the 25-base halves do not fit a leaf and split down to single characters
    over more than 32 target bases; at 20 000 the whole query is one leaf."""
    st, failed = ol.hirschberg_myers_align("A" * 50, "A" * 400, max_query_length=50)
    assert not failed and ol.states_to_cigar(st, extended=True) == "25=7I12=20I6=26I3=29I2=61I1=207I1="
    s = ol.global_stats("hirschberg_myers", "A" * 50, "A" * 400, 50)
    assert s["short_splits"] > 0 and s["single_char_long"] > 0 and s["tied_splits"] > 0 and s["cells"] > 50 * 400
    s = ol.global_stats("hirschberg_myers", "A" * 50, "A" * 400, 20000)
    assert (s["cells"], s["leaves"], s["splits"]) == (50 * 400, 1, 0)
    assert ol.global_stats("myers", "ACGT" * 10, "ACG" * 7, 0)["cells"] == 40 * 21
    assert ol.global_stats("myers", "", "ACG", 0)["cells"] == 0
    assert ol.global_stats("ukkonen", "A" * 90, "A" * 100, 0)["cells"] == ukkonen_bw(90, 100) * (91 + 101)
    assert ol.global_stats("ukkonen", "A" * 100, "A" * 90, 0)["cells"] == ukkonen_bw(90, 100) * (91 + 101)
    # a leaf counts ql x tl, a split ql x tl, single characters nothing
    s = ol.global_stats("hirschberg_myers", "ACGTACGTAC", "ACGTTACGAC", 10)
    assert (s["cells"], s["leaves"], s["splits"]) == (100, 1, 0)
    # "AC" against A x 100 at max_query_length 2: the 2-base slice does not fit 64 words and splits; every midpoint 1 .. 99
    # sums to 99, lane 0 holds the first minimum of its stride (t = 32) and keeps it over the lanes holding t = 1 .. 31
    s = ol.global_stats("hirschberg_myers", "AC", "A" * 100, 2)
    assert (s["cells"], s["splits"], s["short_splits"], s["leaves"]) == (200, 1, 1, 0)
    assert (s["tied_splits"], s["lane_rule_splits"], s["single_char_long"]) == (1, 1, 1)
    st, _ = ol.hirschberg_myers_align("AC", "A" * 100, max_query_length=2)
    assert ol.states_to_cigar(st, extended=True) == "31I1=1X67I"


def test_skewed_pairs_reach_ties_the_lane_rule_decides():
    pairs = skewed_pairs()
    for q, t in pairs:
        lo, hi = sorted((len(q), len(t)))
        assert lo >= 63 and hi <= 4000 and 5 <= hi // lo <= 20
    assert sum(len(q) > len(t) for q, t in pairs) == sum(len(q) < len(t) for q, t in pairs)
    max_q = max(len(q) for q, _ in pairs)
    stats = [ol.global_stats("hirschberg_myers", q, t, max_q) for q, t in pairs]
    assert sum(s["tied_splits"] for s in stats) > 0
    assert sum(s["lane_rule_splits"] for s in stats) > 0
    # in both orientations
    assert any(s["lane_rule_splits"] for s, (q, t) in zip(stats, pairs) if len(q) > len(t))
    assert any(s["lane_rule_splits"] for s, (q, t) in zip(stats, pairs) if len(q) < len(t))


def test_leaf_edge_pairs_reach_short_splits_and_long_single_characters():
    cases = leaf_edge_cases()
    total = dict.fromkeys(ol.GLOBAL_STATS, 0)
    for name, (mq, pairs) in cases.items():
        for q, t in pairs:
            assert len(q) <= mq
            s = ol.global_stats("hirschberg_myers", q, t, mq)
            assert not s["failed"]
            for k in ol.GLOBAL_STATS:
                total[k] += s[k]
    assert total["short_splits"] > 0 and total["single_char_long"] > 0 and total["lane_rule_splits"] > 0
    # max_query_length 40, a 40-base query: targets of 62 / 63 are one leaf, 64 / 65 split
    mq, pairs = cases["max_q_40"]
    for tl in (62, 63, 64, 65):
        sel = [(q, t) for q, t in pairs if len(q) == 40 and len(t) == tl]
        assert sel
        for q, t in sel:
            s = ol.global_stats("hirschberg_myers", q, t, mq)
            if tl <= 63:
                assert (s["leaves"], s["splits"]) == (1, 0)
            else:
                assert s["short_splits"] > 0
    # at max_query_length 20 000 a 62-base slice is a leaf up to a 19 999-base target, a 63-base slice always splits
    mq, pairs = cases["large_max_q"]
    for q, t in pairs:
        s = ol.global_stats("hirschberg_myers", q, t, mq)
        top_leaf = len(q) < FULL_MYERS_THRESHOLD and (len(t) + 1) * words(len(q)) <= leaf_elems(mq)
        assert (s["splits"] == 0) == top_leaf, (len(q), len(t))
        assert top_leaf == (len(q) == 62 and len(t) <= 19999)


def test_chunk_edge_queries_span_32_33_64_65_words():
    half_words = set()
    for L in HIRSCHBERG_CHUNK_QUERIES:
        half_words |= {words(L // 2), words(L - L // 2)}
    assert {32, 33, 64, 65} <= half_words
    assert {words(L) for L in MYERS_CHUNK_QUERIES} == {32, 33, 64, 65}
    assert [len(q) for q, _ in chunk_pairs("myers")][::2] == list(MYERS_CHUNK_QUERIES)
    assert [len(q) for q, _ in chunk_pairs("hirschberg_myers")][::2] == list(HIRSCHBERG_CHUNK_QUERIES)


def test_long_queries_put_the_column_state_on_both_sides_of_shared_memory():
    cases = long_query_cases()
    mq, pairs = cases["smem_full"]
    col_smem = min(words(mq) + 1, COL_SMEM_WORDS)
    assert [words(len(q)) for q, _ in pairs] == [col_smem]       # in shared memory, to the last word
    mq, pairs = cases["col_ws"]
    col_smem = min(words(mq) + 1, COL_SMEM_WORDS)
    in_global = [words(len(q)) > col_smem for q, _ in pairs]
    assert in_global == [True, False, True, False, False]
    assert max(len(t) for _, t in pairs) <= 16000


def test_ukkonen_cases_put_two_slots_on_a_thread_and_pass_the_int16_range():
    cases = ukkonen_cases()
    mq, pairs = cases["wide_band"]
    threads = min(UKKONEN_THREADS, (ukkonen_bw_max(mq) + 31) // 32 * 32)
    assert ukkonen_bw_max(mq) > UKKONEN_THREADS and threads == UKKONEN_THREADS
    bws = [ukkonen_bw(len(q), len(t)) for q, t in pairs]
    assert all(abs(len(q) - len(t)) <= int(np.float32(mq) * np.float32(0.1)) for q, t in pairs)
    assert sum(bw > threads for bw in bws) >= 2 and min(bws) < threads
    assert any(len(q) > len(t) and ukkonen_bw(len(q), len(t)) > threads for q, t in pairs)
    mq, pairs = cases["long"]
    assert all(abs(len(q) - len(t)) <= int(np.float32(mq) * np.float32(0.1)) for q, t in pairs)
    assert max(ukkonen_bw(len(q), len(t)) for q, t in pairs) == 2051
    # every cell of the disjoint-alphabet pair is a mismatch: its distance does not fit an int16
    q, t = pairs[1]
    assert not set(q) & set(t) and max(len(q), len(t)) > 32767
    st = ol.ukkonen_align(q, t)
    assert int(np.count_nonzero(st != 2)) == len(q) and int(np.count_nonzero(st != 3)) == len(t)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU cases
# ---------------------------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("algorithm", ["hirschberg_myers", "myers"])
def test_skewed_shapes(algorithm):
    """Query 5-20x the target and target 5-20x the query: ties of the midpoint sum that the lane rule decides."""
    pairs = skewed_pairs()
    max_q = max(len(q) for q, _ in pairs)
    res = align_and_check(algorithm, pairs, max_q)
    check_reference("skewed_" + algorithm, res, pairs, algorithm, max_q)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(leaf_edge_cases()))
def test_leaf_edges_at_small_max_query_length(name):
    """Leaf against split on both sides of the leaf matrix size, the short-slice split and single characters over many lanes."""
    max_q, pairs = leaf_edge_cases()[name]
    res = align_and_check("hirschberg_myers", pairs, max_q)
    check_reference("leaf_" + name, res, pairs, "hirschberg_myers", max_q)


@pytest.mark.gpu
@pytest.mark.parametrize("algorithm", ["hirschberg_myers", "myers"])
def test_chunk_edges(algorithm):
    pairs = chunk_pairs(algorithm)
    align_and_check(algorithm, pairs, max(len(q) for q, _ in pairs))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["smem_full", "col_ws"])
def test_column_state_in_shared_and_global_memory(name):
    max_q, pairs = long_query_cases()[name]
    res = align_and_check("hirschberg_myers", pairs, max_q)
    check_reference("long_query_" + name, res, pairs, "hirschberg_myers", max_q)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["wide_band", "long"])
def test_ukkonen_wide_bands_and_long_pairs(name):
    max_len, pairs = ukkonen_cases()[name]
    res = align_and_check("ukkonen", pairs, max_len, max_len)
    check_reference("ukkonen_" + name, res, pairs, "ukkonen", max_len, max_len)


@pytest.mark.gpu
@pytest.mark.parametrize("algorithm", ["hirschberg_myers", "myers", "ukkonen"])
def test_reverse_complement_flags(algorithm):
    """reverse_complement_query / _target: the kernels align the complemented strands, as the oracle on those strings."""
    cases = revcomp_pairs(algorithm)
    aligned = [(revcomp(q) if rq else q, revcomp(t) if rt else t) for q, t, rq, rt in cases]
    max_q = max(len(q) for q, _ in aligned)
    max_t = max(len(t) for _, t in aligned)
    expect = oracle(algorithm, aligned, max_q)
    al = new_aligner(algorithm, max_q, max_t, len(cases))
    res, cells = run(al, [(q, t) for q, t, _, _ in cases], [(rq, rt) for _, _, rq, rt in cases])
    al.close()
    check(res, cells, expect)
    for r, (q, t) in zip(res, aligned):
        assert (r.get_query_sequence(), r.get_target_sequence()) == (q, t)


@pytest.mark.gpu
@pytest.mark.parametrize("algorithm", ["hirschberg_myers", "myers", "ukkonen"])
def test_poisoned_workspaces_and_reuse(algorithm):
    """Every device buffer filled with 0x00, 0xFF or random bytes before each launch: a long batch, then reset and a shorter
    batch on the same aligner. Both equal a fresh aligner's results and the oracle."""
    max_q, max_t, long_, short = poison_batches(algorithm)
    n = max(len(long_), len(short))
    fresh = {}
    for key, batch in (("long", long_), ("short", short)):
        al = new_aligner(algorithm, max_q, max_t, n)
        res, cells = run(al, batch)
        al.close()
        check(res, cells, oracle(algorithm, batch, max_q))
        fresh[key] = ([r.convert_to_cigar(extended=True) for r in res], cells)
    for poison in POISONS:
        pa = PoisonedGlobalAligner(algorithm, max_q, max_t, n, poison)
        res, cells = pa.run(long_)
        assert ([r.convert_to_cigar(extended=True) for r in res], cells) == fresh["long"], poison
        pa.al.reset()
        res, cells = pa.run(short)
        assert ([r.convert_to_cigar(extended=True) for r in res], cells) == fresh["short"], poison
        assert all(r.is_optimal for r in res)
        pa.close()
