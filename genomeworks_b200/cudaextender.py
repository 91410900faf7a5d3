"""Ungapped X-drop seed extension (GenomeWorks cudaextender) on this engine, through the C ABI (include/gwb200.h).

    ext = create_extender(score_matrix, xdrop_threshold)
    ext.extend_async(query, target, score_threshold, seed_pairs)    # host-pointer API
    ext.sync()
    ssp = ext.get_scored_segment_pairs()                            # structured array: query, target, length, score

Sequences are int8 arrays of codes or str (encoded with encode_sequence); seed pairs are a structured array with named
`query` and `target` fields (SEED_DTYPE), so the CSV's target-first column order cannot be confused with the record order.
create_gapped_extender (GappedXDrop) turns anchors into gapped alignments with CIGARs. create_seeder (Seeder) makes the seed
pairs of two sequences, create_ssp_chainer (SspChainer) finds the highest-scoring colinear chain of scored segment pairs, or
every chain above a minimum score, and align_genomes / format_paf run seeding, both extension stages and, optionally, chaining
over two sets of records.
There is no CPU fallback: without a CUDA device create_extender and create_gapped_extender raise.
"""
import ctypes as C
import re

import numpy as np

from ._lib import CallArgs, check, lib

success = 0
invalid_operation = 1
invalid_input = 2
generic_error = 3

# cudaextender/utils.hpp
A_NT, C_NT, G_NT, T_NT, L_NT, N_NT, X_NT, E_NT = range(8)
NUC = 8
NUC2 = 64

SEED_DTYPE = np.dtype([("query", np.uint32), ("target", np.uint32)])
SSP_DTYPE = np.dtype([("query", np.uint32), ("target", np.uint32), ("length", np.int32), ("score", np.int32)])

_ENCODE = np.full(256, X_NT, dtype=np.int8)
for _ch, _code in (("A", A_NT), ("C", C_NT), ("G", G_NT), ("T", T_NT), ("&", E_NT), ("n", N_NT), ("N", N_NT),
                   ("a", L_NT), ("c", L_NT), ("g", L_NT), ("t", L_NT)):
    _ENCODE[ord(_ch)] = _code


def encode_sequence(seq):
    """cudaextender::encode_sequence: A/C/G/T -> 0-3, lowercase acgt -> 4, n/N -> 5, '&' -> 7, anything else -> 6."""
    if isinstance(seq, str):
        seq = seq.encode()
    return _ENCODE[np.frombuffer(bytes(seq), dtype=np.uint8)]


def parse_seed_pairs(path):
    """cudaextender::parse_seed_pairs: CSV rows `target, query` -> SEED_DTYPE array."""
    rows = np.loadtxt(path, delimiter=",", dtype=np.int64, ndmin=2).reshape(-1, 2)
    out = np.zeros(len(rows), dtype=SEED_DTYPE)
    out["target"], out["query"] = rows[:, 0], rows[:, 1]
    return out


def parse_scored_segment_pairs(path):
    """cudaextender::parse_scored_segment_pairs: CSV rows `target, query, length, score` -> SSP_DTYPE array."""
    rows = np.loadtxt(path, delimiter=",", dtype=np.int64, ndmin=2).reshape(-1, 4)
    out = np.zeros(len(rows), dtype=SSP_DTYPE)
    out["target"], out["query"], out["length"], out["score"] = rows[:, 0], rows[:, 1], rows[:, 2], rows[:, 3]
    return out


def _codes(seq):
    if isinstance(seq, (str, bytes)):
        return encode_sequence(seq)
    return np.ascontiguousarray(seq, dtype=np.int8)


def _seeds(seed_pairs):
    s = np.asarray(seed_pairs)
    if s.dtype.names is None or "query" not in s.dtype.names or "target" not in s.dtype.names:
        raise TypeError("seed_pairs must be a structured array with 'query' and 'target' fields (SEED_DTYPE)")
    out = np.zeros(len(s), dtype=SEED_DTYPE)
    out["query"], out["target"] = s["query"], s["target"]
    return out


class UngappedXDrop:
    """cudaextender::Extender of type ungapped_xdrop (extender.hpp)."""

    def __init__(self, score_matrix, xdrop_threshold, no_entropy=False, stream=None, device_id=0):
        mat = np.ascontiguousarray(np.asarray(score_matrix, dtype=np.int32).ravel())
        self._h = C.c_void_p()
        check(lib().gwb200_extender_create(C.byref(self._h), mat.ctypes.data_as(C.c_void_p), C.c_int32(mat.size), C.c_int32(xdrop_threshold),
                                           C.c_int32(1 if no_entropy else 0), CallArgs(stream).stream, C.c_int32(device_id)))
        self._keep = ()

    def extend_async(self, query, target, score_threshold, seed_pairs):
        """Host-pointer extend_async; returns a StatusType. Inputs are kept alive until the next call."""
        q, t, s = _codes(query), _codes(target), _seeds(seed_pairs)
        self._keep = (q, t, s)
        return check(lib().gwb200_extender_extend_host(self._h, q.ctypes.data_as(C.c_void_p), C.c_int32(len(q)), t.ctypes.data_as(C.c_void_p),
                                                       C.c_int32(len(t)), C.c_int32(score_threshold), s.ctypes.data_as(C.c_void_p),
                                                       C.c_int32(len(s))))

    def extend_async_device(self, d_query, d_target, score_threshold, d_seed_pairs, d_scored_segment_pairs, d_num_scored_segment_pairs,
                            num_seed_pairs=None):
        """Device-pointer extend_async on torch CUDA tensors: int8 sequences, seeds as an int32 tensor of shape (n, 2) in
        (query, target) order, output int32 tensor with room for n x 4 values (query, target, length, score) and an int32
        count tensor of one element. num_seed_pairs defaults to the seed tensor's first dimension. Returns a StatusType;
        nothing waits for the device. A null (None or empty) tensor is invalid_input, as a null pointer is in the reference."""
        if num_seed_pairs is not None:
            n = num_seed_pairs
        else:
            n = d_seed_pairs.shape[0] if d_seed_pairs is not None else 0

        def ptr(x):
            return C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p(0)

        return check(lib().gwb200_extender_extend_device(self._h, ptr(d_query), C.c_int32(d_query.numel() if d_query is not None else 0),
                                                         ptr(d_target), C.c_int32(d_target.numel() if d_target is not None else 0),
                                                         C.c_int32(score_threshold), ptr(d_seed_pairs), C.c_int32(n),
                                                         ptr(d_scored_segment_pairs), ptr(d_num_scored_segment_pairs)))

    def sync(self):
        return check(lib().gwb200_extender_sync(self._h))

    def get_scored_segment_pairs(self):
        """Results of the last host-pointer call after sync(); raises RuntimeError otherwise (as the reference throws)."""
        n = check(lib().gwb200_extender_num_results(self._h))
        out = np.zeros(n, dtype=SSP_DTYPE)
        check(lib().gwb200_extender_get_results(self._h, out.ctypes.data_as(C.c_void_p), C.c_int32(n)))
        return out

    def reset(self):
        check(lib().gwb200_extender_reset(self._h))

    def last_kernel_ms(self):
        return lib().gwb200_extender_last_kernel_ms(self._h)

    def last_positions(self):
        return check(lib().gwb200_extender_last_positions(self._h))

    def close(self):
        if self._h:
            lib().gwb200_extender_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def create_extender(score_matrix, xdrop_threshold, no_entropy=False, stream=None, device_id=0):
    """cudaextender::create_extender(h_score_mat, 64, xdrop_threshold, no_entropy, stream, device_id): the 8 x 8 (or 64-entry)
    substitution matrix, row = target code, column = query code. Anything but 64 entries raises ValueError."""
    return UngappedXDrop(score_matrix, xdrop_threshold, no_entropy, stream, device_id)


# Gapped X-drop extension (DESIGN.md section 16): anchors to scored alignments with affine gaps and CIGARs.
ANCHOR_DTYPE = SEED_DTYPE
GAPPED_DTYPE = np.dtype([("score", np.int64), ("anchor", np.int32), ("has_cigar", np.int32), ("query_begin", np.uint32),
                         ("query_end", np.uint32), ("target_begin", np.uint32), ("target_end", np.uint32)])
DEFAULT_GAPPED_BUDGET = 1 << 30
SKIP_STATS = ("extended", "skipped", "speculative", "traced", "rounds")


def _skip_args(skip_covered, round_anchors):
    """Checks the skip-covered arguments (DESIGN.md section 18) before any device work; -> (on, round_anchors) as ints."""
    if not isinstance(skip_covered, (bool, np.bool_)):
        raise TypeError("skip_covered must be True or False")
    if isinstance(round_anchors, (bool, np.bool_)) or not isinstance(round_anchors, (int, np.integer)):
        raise TypeError("round_anchors must be an integer")
    if not 0 <= int(round_anchors) < (1 << 31):
        raise ValueError("round_anchors must lie in [0, 2^31 - 1]; 0 picks the device's default")
    return int(bool(skip_covered)), int(round_anchors)


class GappedXDrop:
    """Gapped X-drop extender: each anchor extended left and right by Gotoh DP with an anti-diagonal y-drop, the sides joined
    into one alignment with a CIGAR (M / I / D, I consuming the query)."""

    def __init__(self, score_matrix, gap_open, gap_extend, ydrop, budget_bytes=DEFAULT_GAPPED_BUDGET, stream=None, device_id=0,
                 allocator=None, skip_covered=False, round_anchors=0):
        mat = np.ascontiguousarray(np.asarray(score_matrix, dtype=np.int64).ravel())
        self._h = C.c_void_p()
        skip = _skip_args(skip_covered, round_anchors)
        for name, v, hi in (("gap_open", gap_open, 1 << 24), ("gap_extend", gap_extend, 1 << 24), ("ydrop", ydrop, 1 << 28)):
            if not 0 <= int(v) <= hi:
                raise ValueError("%s must lie in [0, %d]" % (name, hi))
        if mat.size != NUC2 or (mat.size and (mat.min() < -(1 << 24) or mat.max() > (1 << 24))):
            raise ValueError("the scoring matrix must have 64 entries (8 x 8 codes) in [-2^24, 2^24]")
        if int(budget_bytes) < 0:
            raise ValueError("budget_bytes must be >= 0")
        self._args = CallArgs(stream, allocator)
        mat = mat.astype(np.int32)
        rc = lib().gwb200_gapped_extender_create_with_allocator(C.byref(self._h), mat.ctypes.data_as(C.c_void_p), C.c_int32(mat.size),
                                                               C.c_int32(gap_open), C.c_int32(gap_extend), C.c_int32(ydrop),
                                                               C.c_int64(budget_bytes), self._args.stream, C.c_int32(device_id),
                                                               *self._args.mem)
        if rc == invalid_input:
            raise ValueError("invalid gapped extender parameters")
        check(rc)
        self._keep = ()
        if skip[0]:
            self.set_skip_covered(*skip)

    def set_skip_covered(self, on=True, round_anchors=0):
        """Skip-covered mode for later calls (DESIGN.md section 18): an anchor on the path of an alignment kept earlier in the
        same call is not extended. round_anchors (anchors per device round, 0 = the device's default) never changes an output.
        Raises RuntimeError while a call is pending."""
        on, round_anchors = _skip_args(bool(on), round_anchors)
        if check(lib().gwb200_gapped_extender_set_skip_covered(self._h, C.c_int32(on), C.c_int32(round_anchors))) == invalid_operation:
            raise RuntimeError("an extend call is pending: sync() it first")

    def extend_async(self, query, target, threshold, anchors):
        """Host-pointer extension of `anchors` (structured array with query / target fields); returns a StatusType
        (invalid_input for an anchor outside either sequence). Inputs are kept alive until the next call; sync() finishes it."""
        q, t, a = _codes(query), _codes(target), _seeds(anchors)
        self._keep = (q, t, a)
        return check(lib().gwb200_gapped_extender_extend_host(self._h, q.ctypes.data_as(C.c_void_p), C.c_int32(len(q)),
                                                              t.ctypes.data_as(C.c_void_p), C.c_int32(len(t)), C.c_int64(threshold),
                                                              a.ctypes.data_as(C.c_void_p), C.c_int32(len(a))))

    def extend_ssps_device(self, d_query, d_target, threshold, d_ssps, num_ssps=None):
        """Extension of scored segment pairs already on the device (torch CUDA tensors: int8 sequences, an int32 tensor of
        n x 4 values query, target, length, score as the ungapped extender writes them), each anchored at its middle.
        num_ssps (a host count) defaults to the tensor's first dimension. The tensors must stay alive until sync()."""
        n = num_ssps if num_ssps is not None else (d_ssps.shape[0] if d_ssps is not None else 0)

        def ptr(x):
            return C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p(0)

        self._keep = (d_query, d_target, d_ssps)
        return check(lib().gwb200_gapped_extender_extend_ssps_device(
            self._h, ptr(d_query), C.c_int32(d_query.numel() if d_query is not None else 0), ptr(d_target),
            C.c_int32(d_target.numel() if d_target is not None else 0), C.c_int64(threshold), ptr(d_ssps), C.c_int32(n)))

    def sync(self):
        return check(lib().gwb200_gapped_extender_sync(self._h))

    def get_alignments(self):
        """After sync(): (GAPPED_DTYPE array, list of CIGAR strings, '' where has_cigar is 0)."""
        n = check(lib().gwb200_gapped_extender_num_results(self._h))
        out = np.zeros(n, dtype=GAPPED_DTYPE)
        check(lib().gwb200_gapped_extender_get_results(self._h, out.ctypes.data_as(C.c_void_p), C.c_int32(n)))
        size = check(lib().gwb200_gapped_extender_cigar_bytes(self._h))
        text = C.create_string_buffer(max(size, 1))
        offsets = np.zeros(n + 1, dtype=np.int64)
        check(lib().gwb200_gapped_extender_get_cigars(self._h, text, C.c_int64(size), offsets.ctypes.data_as(C.c_void_p)))
        raw = text.raw[:size].decode()
        return out, [raw[offsets[k]:offsets[k + 1]] for k in range(n)]

    def reset(self):
        check(lib().gwb200_gapped_extender_reset(self._h))

    def last_pass_ms(self):
        """Device ms of pass 1 and pass 2 of the last finished call (-1 where a pass did not run)."""
        p1, p2 = C.c_float(), C.c_float()
        check(lib().gwb200_gapped_extender_last_ms(self._h, C.byref(p1), C.byref(p2)))
        return p1.value, p2.value

    def last_live_cells(self):
        return check(lib().gwb200_gapped_extender_last_live_cells(self._h))

    def last_skip_stats(self):
        """Of the last finished call: {extended, skipped, speculative, traced, rounds} (DESIGN.md section 18)."""
        out = np.zeros(len(SKIP_STATS), dtype=np.int64)
        check(lib().gwb200_gapped_extender_last_skip_stats(self._h, out.ctypes.data_as(C.c_void_p)))
        return dict(zip(SKIP_STATS, (int(v) for v in out)))

    def close(self):
        if self._h:
            lib().gwb200_gapped_extender_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def create_gapped_extender(score_matrix, gap_open, gap_extend, ydrop, budget_bytes=DEFAULT_GAPPED_BUDGET, stream=None, device_id=0,
                           allocator=None, skip_covered=False, round_anchors=0):
    """A GappedXDrop over the 8 x 8 (or 64-entry) substitution matrix, row = target code, column = query code. Parameters
    outside their ranges raise ValueError before any device work; without a CUDA device this raises RuntimeError.
    skip_covered=True starts it in skip-covered mode (GappedXDrop.set_skip_covered)."""
    return GappedXDrop(score_matrix, gap_open, gap_extend, ydrop, budget_bytes, stream, device_id, allocator, skip_covered, round_anchors)


# Seeding (DESIGN.md sections 17 and 22): the hits of a spaced seed (LASTZ's 12-of-19 by default), in the global order of
# include/gwb200.h.
DEFAULT_SEED = "12of19"
NAMED_SEEDS = {"12of19": "1110100110010101111", "14of22": "1110101100110010101111"}
MAX_SEED_SPAN, MAX_SEED_WEIGHT = 32, 14


def seed_pattern(seed):
    """The 0/1 string of a seed pattern (DESIGN.md section 22.1): "12of19", "14of22", "match<N>" (N ones, 1 <= N <= 14) or a
    string of 0 and 1 with a 1 at both ends, span 1 to 32 and 1 to 14 ones. TypeError for a non-string, ValueError otherwise."""
    if not isinstance(seed, str):
        raise TypeError("seed must be a string")
    bits = NAMED_SEEDS.get(seed, seed)
    m = re.fullmatch(r"match([1-9][0-9]?)", seed)
    if m:
        bits = "1" * int(m.group(1)) if int(m.group(1)) <= MAX_SEED_WEIGHT else ""
    if (not re.fullmatch(r"1([01]*1)?", bits) or len(bits) > MAX_SEED_SPAN or bits.count("1") > MAX_SEED_WEIGHT):
        raise ValueError("seed must be 12of19, 14of22, match<N> for N = 1 ... 14, or a string of 0 and 1 with a 1 at both ends, "
                         "of span 1 to 32 with 1 to 14 ones; got %r" % seed)
    return bits


def _seed_args(seed, max_word_count):
    """Checks a seed pattern and word cap before any device work; -> (seed bytes, cap)."""
    seed_pattern(seed)
    if isinstance(max_word_count, (bool, np.bool_)) or not isinstance(max_word_count, (int, np.integer)):
        raise TypeError("max_word_count must be an integer")
    if not 0 <= int(max_word_count) <= INT64_MAX:
        raise ValueError("max_word_count must lie in [0, 2^63 - 1] (0 turns the word cap off)")
    return seed.encode(), int(max_word_count)


def _seq_arg(seq):
    """(pointer, length, object to keep alive) of a sequence: a torch tensor (host or CUDA) is passed by address; anything else
    is encoded / converted to int8 codes on the host."""
    if hasattr(seq, "data_ptr"):
        return C.c_void_p(seq.data_ptr() if seq.numel() else 0), seq.numel(), seq
    s = _codes(seq)
    return s.ctypes.data_as(C.c_void_p), len(s), s


class Seeder:
    """Spaced-seed seeder: index_target(target) once, then count(query) and get_block(first, count) for any number of queries.
    Sequences are int8 codes (numpy, str, or torch tensors on the host or the device). seed and max_word_count as set_seed."""

    def __init__(self, transition=True, stream=None, device_id=0, allocator=None, seed=DEFAULT_SEED, max_word_count=0):
        seed_args = _seed_args(seed, max_word_count)
        self._args = CallArgs(stream, allocator)
        self._device = device_id
        self._h = C.c_void_p()
        check(lib().gwb200_seeder_create_with_allocator(C.byref(self._h), C.c_int32(1 if transition else 0), self._args.stream,
                                                        C.c_int32(device_id), *self._args.mem))
        if seed_args != (DEFAULT_SEED.encode(), 0):
            check(lib().gwb200_seeder_set_seed(self._h, *seed_args))

    def set_seed(self, seed=DEFAULT_SEED, max_word_count=0):
        """The seed pattern (seed_pattern) and word cap of later calls (DESIGN.md section 22): with max_word_count N > 0, the
        hits of a query word, exact or one transition variant, are dropped when the word occurs more than N times in the
        target. Drops the target index: index_target again before count."""
        check(lib().gwb200_seeder_set_seed(self._h, *_seed_args(seed, max_word_count)))

    def index_target(self, target):
        p, n, _ = _seq_arg(target)
        if check(lib().gwb200_seeder_index_target(self._h, p, C.c_int64(n))) == invalid_input:
            raise ValueError("a target must be a sequence of fewer than 2^31 codes")

    def count(self, query):
        """Counts the seeds of `query` against the indexed target; returns their total (blocking)."""
        p, n, _ = _seq_arg(query)
        return check(lib().gwb200_seeder_count(self._h, p, C.c_int64(n)))

    def get_block(self, first, count, d_out=None):
        """Seeds [first, first + count) of the last counted query, written to d_out (a CUDA tensor with room for count x 2 int32
        values, query then target) or to a new one; returns the tensor. Enqueued on the seeder's stream without waiting."""
        import torch
        if d_out is None:
            d_out = torch.empty((max(int(count), 0), 2), dtype=torch.int32, device="cuda:%d" % self._device)
        rc = check(lib().gwb200_seeder_get_block(self._h, C.c_int64(first), C.c_int64(count), C.c_void_p(d_out.data_ptr() if d_out.numel() else 0)))
        if rc == invalid_input:
            raise ValueError("block [%d, %d) lies outside the %d seeds" % (first, first + count, self.total()))
        if rc == invalid_operation:
            raise RuntimeError("no counted query: call count first")
        return d_out

    def total(self):
        return check(lib().gwb200_seeder_total(self._h))

    def sync(self):
        check(lib().gwb200_seeder_sync(self._h))

    def seed_pairs(self, query, target):
        """Every seed pair of query against target, in the global order, as a SEED_DTYPE array."""
        self.index_target(target)
        n = self.count(query)
        d = self.get_block(0, n)
        self.sync()
        out = np.zeros(n, dtype=SEED_DTYPE)
        if n:
            h = d.cpu().numpy()
            out["query"], out["target"] = h[:, 0].view(np.uint32), h[:, 1].view(np.uint32)
        return out

    def last_ms(self):
        """Device ms of the last index, count and get_block (-1 where none ran)."""
        v = [C.c_float(), C.c_float(), C.c_float()]
        check(lib().gwb200_seeder_last_ms(self._h, *(C.byref(x) for x in v)))
        return tuple(x.value for x in v)

    def close(self):
        if self._h:
            lib().gwb200_seeder_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def create_seeder(transition=True, stream=None, device_id=0, allocator=None, seed=DEFAULT_SEED, max_word_count=0):
    """A Seeder; transition=False keeps only the exact hits; seed and max_word_count as Seeder.set_seed. A bad seed or cap
    raises TypeError or ValueError before any device work; without a CUDA device this raises RuntimeError."""
    return Seeder(transition, stream, device_id, allocator, seed, max_word_count)


# Chaining (DESIGN.md section 19): the highest-scoring colinear chain of scored segment pairs.
MAX_CHAIN_PENALTY = 1 << 20
CHAIN_STATS = ("ssps_in", "ssps_chained", "pairs", "chain_ms")
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def _penalty(name, v):
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
        raise TypeError("%s must be an integer" % name)
    if not 0 <= int(v) <= MAX_CHAIN_PENALTY:
        raise ValueError("%s must lie in [0, 2^20]" % name)
    return int(v)


def _chain_arg(chain):
    """None or False: no chaining; True: penalties (0, 0); (D, A): those penalties, checked before any device work."""
    if chain is None or chain is False:
        return None
    if chain is True:
        return 0, 0
    if isinstance(chain, (tuple, list)) and len(chain) == 2:
        return _penalty("the diagonal penalty", chain[0]), _penalty("the anti-diagonal penalty", chain[1])
    raise TypeError("chain must be None, True or a (diag_penalty, anti_penalty) pair")


def _min_score(name, v):
    """A minimum chain score (DESIGN.md section 20): any int64, checked before any device work."""
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
        raise TypeError("%s must be an integer" % name)
    if not INT64_MIN <= int(v) <= INT64_MAX:
        raise ValueError("%s must lie in [-2^63, 2^63 - 1]" % name)
    return int(v)


def _chain_args(chain, min_chain_score):
    """(penalties or None, minimum chain score or None) of the aligner's chain arguments, checked before any device work."""
    penalties = _chain_arg(chain)
    if min_chain_score is None:
        return penalties, None
    min_score = _min_score("min_chain_score", min_chain_score)
    if penalties is None:
        raise ValueError("min_chain_score needs chain=True or (diag_penalty, anti_penalty)")
    return penalties, min_score


class SspChainer:
    """The chaining DP of DESIGN.md section 19 on the device: chain(ssps) returns the SSP indices of the highest-scoring colinear
    chain, in ascending order, and its score; chain_all(ssps, min_score=S) returns every chain scoring >= S (DESIGN.md section
    20); get_dp() returns f and p of every SSP."""

    def __init__(self, stream=None, device_id=0, allocator=None):
        self._args = CallArgs(stream, allocator)
        self._device = device_id
        self._h = C.c_void_p()
        self._n = 0
        check(lib().gwb200_ssp_chainer_create(C.byref(self._h), self._args.stream, C.c_int32(device_id), *self._args.mem))

    def chain(self, ssps, n=None, diag_penalty=0, anti_penalty=0):
        """ssps: an SSP_DTYPE array (copied to the device), a CUDA tensor of n x 4 int32 values (query, target, length, score) or
        a device address (then n is required). Blocking. Penalties outside [0, 2^20], n < 0 or a length below -1 raise
        ValueError."""
        D = _penalty("diag_penalty", diag_penalty)
        A = _penalty("anti_penalty", anti_penalty)
        self._call(ssps, n, lambda addr, m: lib().gwb200_ssp_chainer_chain_device(self._h, C.c_void_p(addr), C.c_int32(m), C.c_int32(D),
                                                                                  C.c_int32(A)))
        return self.get_chain()

    def chain_all(self, ssps, n=None, diag_penalty=0, anti_penalty=0, min_score=INT64_MIN):
        """Every chain scoring >= min_score (DESIGN.md section 20.1; the default reports every chain): (int64 scores, int64
        offsets of len(scores) + 1, int32 members), chain c being members[offsets[c]:offsets[c + 1]] in ascending index, the
        chains in their heads' priority order. Takes the inputs of chain(); min_score is any int64. get_chain() then gives the
        union of the chains' SSPs and the sum of their scores."""
        D = _penalty("diag_penalty", diag_penalty)
        A = _penalty("anti_penalty", anti_penalty)
        S = _min_score("min_score", min_score)
        self._call(ssps, n, lambda addr, m: lib().gwb200_ssp_chainer_chain_all_device(self._h, C.c_void_p(addr), C.c_int32(m), C.c_int32(D),
                                                                                      C.c_int32(A), C.c_int64(S)))
        return self.get_chains()

    def _call(self, ssps, n, enqueue):
        """Puts ssps (any form chain() takes) on the device, enqueues one call through enqueue(address, n) and finishes it."""
        keep = None
        if isinstance(ssps, np.ndarray):
            import torch
            rows = np.ascontiguousarray(ssps, dtype=SSP_DTYPE).view(np.int32).reshape(-1, 4)
            n = len(rows) if n is None else n
            if not 0 <= int(n) <= len(rows):
                raise ValueError("n must lie in [0, %d]" % len(rows))
            keep = torch.from_numpy(rows).to("cuda:%d" % self._device)
            addr = keep.data_ptr() if keep.numel() else 0
        elif hasattr(ssps, "data_ptr"):
            n = ssps.shape[0] if n is None else n
            addr = ssps.data_ptr() if ssps.numel() else 0
        else:
            if n is None:
                raise ValueError("n is required with a device address")
            addr = int(ssps or 0)
        if int(n) < 0:
            raise ValueError("n must be >= 0")
        rc = check(enqueue(addr, int(n)))
        if rc == invalid_input:
            raise ValueError("invalid chain arguments")
        if rc == invalid_operation:
            raise RuntimeError("a chain call is pending")
        rc = check(lib().gwb200_ssp_chainer_sync(self._h))
        del keep
        if rc == invalid_input:
            raise ValueError("an SSP length is below -1")
        self._n = int(n)

    def get_chain(self):
        """(int32 SSP indices of the chain in ascending order, score) of the last call."""
        m = check(lib().gwb200_ssp_chainer_num_chained(self._h))
        idx = np.zeros(m, dtype=np.int32)
        score = C.c_int64()
        check(lib().gwb200_ssp_chainer_get_chain(self._h, idx.ctypes.data_as(C.c_void_p), C.byref(score)))
        return idx, score.value

    def get_chains(self):
        """(scores, offsets, members) of the last call, as chain_all returns them; after chain() one chain, or none for n = 0."""
        m = check(lib().gwb200_ssp_chainer_num_chains(self._h))
        size = check(lib().gwb200_ssp_chainer_num_chained(self._h))
        scores = np.zeros(m, dtype=np.int64)
        offsets = np.zeros(m + 1, dtype=np.int64)
        members = np.zeros(size, dtype=np.int32)
        check(lib().gwb200_ssp_chainer_get_chains(self._h, scores.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                                  members.ctypes.data_as(C.c_void_p)))
        return scores, offsets, members

    def get_dp(self):
        """(f as int64, p as int32, -1 for none) of every SSP of the last call, by SSP index."""
        check(lib().gwb200_ssp_chainer_num_chained(self._h))
        f = np.zeros(self._n, dtype=np.int64)
        p = np.zeros(self._n, dtype=np.int32)
        check(lib().gwb200_ssp_chainer_get_dp(self._h, f.ctypes.data_as(C.c_void_p), p.ctypes.data_as(C.c_void_p)))
        return f, p

    def last_ms(self):
        """Device ms of the last call."""
        ms = C.c_float()
        check(lib().gwb200_ssp_chainer_last_ms(self._h, C.byref(ms)))
        return ms.value

    def close(self):
        if self._h:
            lib().gwb200_ssp_chainer_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def create_ssp_chainer(stream=None, device_id=0, allocator=None):
    """An SspChainer. Without a CUDA device this raises RuntimeError."""
    return SspChainer(stream, device_id, allocator)


# The genome-to-genome aligner (DESIGN.md section 17): seeds, blocked ungapped extension and gapped extension of every
# (target record, query record) pair on one or both strands.
GENOME_DTYPE = np.dtype([("score", np.int64), ("target_record", np.int32), ("query_record", np.int32), ("strand", np.int32),
                         ("has_cigar", np.int32), ("query_begin", np.uint32), ("query_end", np.uint32), ("target_begin", np.uint32),
                         ("target_end", np.uint32), ("matches", np.int64), ("block_length", np.int64)])
STRANDS = {"plus": 1, "minus": 2, "both": 3}
STAGES = ("index", "count", "write", "ungapped", "gapped_pass1", "gapped_pass2")
GROUP_STATS = ("target_groups", "query_groups", "gapped_pairs")
DEFAULT_GROUP_BASES = 1 << 28


def _group_bases(group_bases):
    """Checks group_bases (DESIGN.md section 21) before any device work; -> int."""
    if isinstance(group_bases, (bool, np.bool_)) or not isinstance(group_bases, (int, np.integer)):
        raise TypeError("group_bases must be an integer")
    if not 1 <= int(group_bases) < (1 << 31):
        raise ValueError("group_bases must lie in [1, 2^31 - 1]")
    return int(group_bases)


def default_genome_params():
    """gwb200_genome_aligner_default_params as a dict (score_matrix as a 64-entry int32 array)."""
    from ._lib import GenomeAlignerParams
    p = GenomeAlignerParams()
    lib().gwb200_genome_aligner_default_params(C.byref(p))
    out = {name: getattr(p, name) for name, _ in GenomeAlignerParams._fields_}
    out["score_matrix"] = np.array(list(p.score_matrix), dtype=np.int32)
    return out


def _records(seqs):
    codes = [_codes(s) for s in seqs]
    offsets = np.zeros(len(codes) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(c) for c in codes]) if codes else []
    flat = np.concatenate(codes) if codes else np.zeros(0, dtype=np.int8)
    return np.ascontiguousarray(flat, dtype=np.int8), offsets


class GenomeAligner:
    """The aligner with fixed parameters; run(targets, queries) aligns every query record against every target record."""

    def __init__(self, strand="both", stream=None, device_id=0, allocator=None, skip_covered=False, round_anchors=0, chain=None,
                 min_chain_score=None, group_bases=DEFAULT_GROUP_BASES, seed=DEFAULT_SEED, max_word_count=0, **params):
        """group_bases: the most codes of one side's records the aligner seeds and extends together (DESIGN.md section 21). It
        bounds the seeding stage's device memory and never changes the output; 1 runs every record on its own. seed and
        max_word_count: the seed pattern and word cap (Seeder.set_seed, DESIGN.md section 22); a word is counted over every
        target record together."""
        from ._lib import GenomeAlignerParams
        if strand not in STRANDS:
            raise ValueError("strand must be one of %s" % ", ".join(STRANDS))
        skip = _skip_args(skip_covered, round_anchors)
        group_bases = _group_bases(group_bases)
        seed_args = _seed_args(seed, max_word_count)
        penalties, min_score = _chain_args(chain, min_chain_score)
        p = default_genome_params()
        unknown = set(params) - set(p)
        if unknown:
            raise TypeError("unknown parameters: %s" % ", ".join(sorted(unknown)))
        p.update(params)
        p["strand"] = STRANDS[strand]
        p["transition"] = 1 if p["transition"] else 0
        mat = np.asarray(p.pop("score_matrix"), dtype=np.int64).ravel()
        if mat.size != NUC2 or mat.min() < -(1 << 24) or mat.max() > (1 << 24):
            raise ValueError("the scoring matrix must have 64 entries (8 x 8 codes) in [-2^24, 2^24]")
        cp = GenomeAlignerParams()
        cp.score_matrix[:] = [int(v) for v in mat]
        for name, v in p.items():
            setattr(cp, name, int(v))
            if getattr(cp, name) != int(v):  # a value that does not fit its C field
                raise ValueError("%s = %d is out of range" % (name, int(v)))
        self._args = CallArgs(stream, allocator)
        self._h = C.c_void_p()
        rc = lib().gwb200_genome_aligner_create(C.byref(self._h), C.byref(cp), self._args.stream, C.c_int32(device_id), *self._args.mem)
        if rc == invalid_input:
            raise ValueError("invalid genome aligner parameters")
        check(rc)
        check(lib().gwb200_genome_aligner_set_group_bases(self._h, C.c_int64(group_bases)))
        if seed_args != (DEFAULT_SEED.encode(), 0):
            check(lib().gwb200_genome_aligner_set_seed(self._h, *seed_args))
        if skip[0]:
            check(lib().gwb200_genome_aligner_set_skip_covered(self._h, C.c_int32(skip[0]), C.c_int32(skip[1])))
        if penalties is not None:
            self.set_chain(penalties, min_score)

    def set_chain(self, chain, min_chain_score=None):
        """Chaining for later runs (DESIGN.md section 19): None or False turns it off, True or (D, A) turns it on. With
        min_chain_score=S (any int64; it needs chain) every chain scoring >= S goes to the gapped stage instead of the best one
        (DESIGN.md section 20)."""
        penalties, min_score = _chain_args(chain, min_chain_score)
        check(lib().gwb200_genome_aligner_set_chain(self._h, int(penalties is not None), *(C.c_int32(v) for v in penalties or (0, 0))))
        check(lib().gwb200_genome_aligner_set_chain_min_score(self._h, int(min_score is not None), C.c_int64(min_score or 0)))

    def run(self, targets, queries):
        """-> (GENOME_DTYPE records, CIGAR strings, '' where has_cigar is 0). Blocking."""
        t, toff = _records(targets)
        q, qoff = _records(queries)
        rc = check(lib().gwb200_genome_aligner_run(self._h, t.ctypes.data_as(C.c_void_p), toff.ctypes.data_as(C.c_void_p), C.c_int32(len(toff) - 1),
                                                   q.ctypes.data_as(C.c_void_p), qoff.ctypes.data_as(C.c_void_p), C.c_int32(len(qoff) - 1)))
        if rc == invalid_input:
            raise ValueError("a record must be a sequence of fewer than 2^31 codes")
        n = check(lib().gwb200_genome_aligner_num_results(self._h))
        out = np.zeros(n, dtype=GENOME_DTYPE)
        check(lib().gwb200_genome_aligner_get_results(self._h, out.ctypes.data_as(C.c_void_p), C.c_int32(n)))
        size = check(lib().gwb200_genome_aligner_cigar_bytes(self._h))
        text = C.create_string_buffer(max(size, 1))
        offsets = np.zeros(n + 1, dtype=np.int64)
        check(lib().gwb200_genome_aligner_get_cigars(self._h, text, C.c_int64(size), offsets.ctypes.data_as(C.c_void_p)))
        raw = text.raw[:size].decode()
        return out, [raw[offsets[k]:offsets[k + 1]] for k in range(n)]

    def last_stats(self):
        """Of the last run: {stage: device ms} and the seeds, unique segments and alignments. Index, count, write and ungapped
        ms are summed over every pair of record groups and strand (index over target groups), the gapped passes over every
        record pair and strand."""
        ms = np.zeros(len(STAGES), dtype=np.float32)
        counts = np.zeros(3, dtype=np.int64)
        check(lib().gwb200_genome_aligner_last_stats(self._h, ms.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p)))
        return dict(zip(STAGES, (float(v) for v in ms))), dict(zip(("seeds", "ssps", "alignments"), (int(v) for v in counts)))

    def last_skip_stats(self):
        """Of the last run, summed over every pair and strand: {extended, skipped, speculative, traced, rounds} of the gapped
        stage (DESIGN.md section 18)."""
        out = np.zeros(len(SKIP_STATS), dtype=np.int64)
        check(lib().gwb200_genome_aligner_last_skip_stats(self._h, out.ctypes.data_as(C.c_void_p)))
        return dict(zip(SKIP_STATS, (int(v) for v in out)))

    def last_chain_stats(self):
        """Of the last run, summed over every pair and strand: {ssps_in, ssps_chained, pairs, chain_ms} (all zero without
        chaining; DESIGN.md section 19)."""
        from ._lib import ChainStats
        st = ChainStats()
        check(lib().gwb200_genome_aligner_last_chain_stats(self._h, C.byref(st)))
        return {name: getattr(st, name) for name in CHAIN_STATS}

    def last_chain_count(self):
        """The number of chains the last run reported, summed over every pair and strand (DESIGN.md section 20)."""
        n = C.c_int64()
        check(lib().gwb200_genome_aligner_last_chain_count(self._h, C.byref(n)))
        return n.value

    def last_group_stats(self):
        """Of the last run: {target_groups, query_groups, gapped_pairs}, the last being the (record pair, strand)s that had SSPs
        and went to the gapped stage (DESIGN.md section 21)."""
        out = np.zeros(len(GROUP_STATS), dtype=np.int64)
        check(lib().gwb200_genome_aligner_last_group_stats(self._h, out.ctypes.data_as(C.c_void_p)))
        return dict(zip(GROUP_STATS, (int(v) for v in out)))

    def close(self):
        if self._h:
            lib().gwb200_genome_aligner_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def align_genomes(targets, queries, strand="both", stream=None, device_id=0, allocator=None, skip_covered=False, chain=None,
                  min_chain_score=None, group_bases=DEFAULT_GROUP_BASES, seed=DEFAULT_SEED, max_word_count=0, **params):
    """Aligns every query record against every target record on the plus strand, the minus strand or both. targets and queries
    are lists of sequences (str or int8 codes). Keyword parameters override gwb200_genome_aligner_default_params: score_matrix,
    xdrop, ssp_threshold, gap_open, gap_extend, ydrop, gapped_threshold, transition, block_size, traceback_budget. Returns
    (GENOME_DTYPE records, CIGAR strings); query coordinates are forward for both strands and minus-strand CIGARs read the
    target forward. Bad parameters raise ValueError before any device work. skip_covered=True does not extend the anchors that
    lie on an alignment kept earlier for the same pair and strand (DESIGN.md section 18). chain=True or (D, A) extends only the
    SSPs of the highest-scoring colinear chain of each pair and strand (DESIGN.md section 19); with min_chain_score=S as well,
    those of every chain scoring >= S (DESIGN.md section 20). group_bases (1 to 2^31 - 1) is the most codes of one side's
    records seeded and extended together (DESIGN.md section 21); it bounds device memory and never changes the output. seed
    ("12of19", "14of22", "match<N>" or a 0/1 pattern) and max_word_count N (0 = off) choose the seed and drop the hits of words
    that occur more than N times over all target records (DESIGN.md section 22)."""
    al = GenomeAligner(strand, stream, device_id, allocator, skip_covered, chain=chain, min_chain_score=min_chain_score,
                       group_bases=group_bases, seed=seed, max_word_count=max_word_count, **params)
    try:
        return al.run(targets, queries)
    finally:
        al.close()


def format_paf(records, cigars, target_names, target_lengths, query_names, query_lengths):
    """PAF text of align_genomes' output: 12 columns (matches = M positions with equal codes in 0..3, block = M + I + D lengths,
    mapq 255), then AS:i:score and, where the alignment has a CIGAR, cg:Z:cigar."""
    lines = []
    for r, cg in zip(records, cigars):
        ti, qi = int(r["target_record"]), int(r["query_record"])
        line = "%s\t%d\t%d\t%d\t%s\t%s\t%d\t%d\t%d\t%d\t%d\t255\tAS:i:%d" % (
            query_names[qi], query_lengths[qi], r["query_begin"], r["query_end"], "-" if r["strand"] else "+", target_names[ti],
            target_lengths[ti], r["target_begin"], r["target_end"], r["matches"], r["block_length"], r["score"])
        if r["has_cigar"]:
            line += "\tcg:Z:" + cg
        lines.append(line + "\n")
    return "".join(lines)
