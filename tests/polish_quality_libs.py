"""ctypes bindings of the polisher's CPU restatement with base qualities (oracle/liboracle_polish_q.so,
oracle/polish_quality_oracle.cpp, built by build()), seeded phred strings, and the composition of the polisher with qualities
from proven parts (DESIGN.md section 15.5).

- oracle_groups_q: steps 2-4 with qualities, in the shape cudapolish.window_groups returns, "weights" included;
- composition_q: map_reads(drafts, reads, align=True), oracle_groups_q, CudaPoaBatch.add_poa_groups_flat one group at a time
  with its weights, the oracle's stitching.
"""
import ctypes as C

import numpy as np

import polish_libs as pl
from checker_lib import load, ptr


def oracle():
    return load("liboracle_polish_q.so", {
        "oracle_polish_groups_q": (C.c_int, [C.c_void_p, C.c_int64, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_char_p,
                                             C.c_void_p, C.c_int64, C.c_char_p, C.c_double, C.c_int32, C.c_int32]),
        "oracle_polish_view": (C.c_int, [C.POINTER(pl._View)]),
        "oracle_polish_weights": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64)])})


def oracle_groups_q(overlaps, cigars, drafts, reads, qualities, threshold, window_length, max_depth):
    """(0, dict of pl.KEYS, "weights" and "n_kept") or (-1, None) for the arguments the contract rejects."""
    ov = np.ascontiguousarray(overlaps, dtype=pl.OVERLAP_DTYPE)
    text, toffs = pl.cigar_text(cigars)
    db, doffs = pl._flat(drafts)
    rb, roffs = pl._flat(reads)
    qb, qoffs = pl._flat(qualities)
    assert np.array_equal(roffs, qoffs), "one quality string per read, as long as the read"
    L = oracle()
    rc = L.oracle_polish_groups_q(ptr(ov), len(ov), text, ptr(toffs), db,
                                  ptr(doffs), len(doffs) - 1, rb, ptr(roffs), len(roffs) - 1, qb,
                                  threshold, window_length, max_depth)
    if rc != 0:
        return rc, None
    v = pl._View()
    L.oracle_polish_view(C.byref(v))
    w, n = C.c_void_p(), C.c_int64()
    L.oracle_polish_weights(C.byref(w), C.byref(n))
    return 0, {
        "draft_window_first": pl._array(v.draft_window_first, v.n_drafts + 1, np.int64),
        "candidates": pl._array(v.candidates, v.n_windows, np.int32),
        "used": pl._array(v.used, v.n_windows, np.int32),
        "group_draft": pl._array(v.group_draft, v.n_groups, np.int32),
        "group_window": pl._array(v.group_window, v.n_groups, np.int32),
        "win_nseq": pl._array(v.win_nseq, v.n_groups, np.int32),
        "seq_len": pl._array(v.seq_len, v.n_sequences, np.int32),
        "seq_data": pl._array(v.seq_data, v.n_bases, np.uint8),
        "weights": pl._array(w.value, n.value, np.int8),
        "n_kept": v.n_kept,
    }


def split_weights(g):
    """The weights of a window-groups dict as one int8 array per sequence, grouped like pl.split_groups."""
    out, s, off = [], 0, 0
    for ns in g["win_nseq"]:
        grp = []
        for k in range(int(ns)):
            ln = int(g["seq_len"][s + k])
            grp.append(g["weights"][off:off + ln])
            off += ln
        s += int(ns)
        out.append(grp)
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# qualities

def random_qualities(seed, reads, lo=0, hi=40, spread=8):
    """One phred+33 string per read: a level drawn per read in lo .. hi, each base within `spread` of it (clipped to 0 .. 93), so
    that mean-quality thresholds inside lo .. hi drop some reads' pieces and keep others'."""
    rng = np.random.default_rng(seed)
    out = []
    for r in reads:
        m = int(rng.integers(lo, hi + 1))
        out.append(bytes((np.clip(rng.integers(m - spread, m + spread + 1, len(r)), 0, 93) + 33).astype(np.uint8)))
    return out


# ---------------------------------------------------------------------------------------------------------------------------
# the polisher with qualities from proven parts

def poa_groups_weighted(groups, weights, window_length, max_depth, max_gpu_mem=2 << 30):
    """(status, consensus bytes) of each group through CudaPoaBatch.add_poa_groups_flat with its weights, one group at a time, the
    batch generated and reset whenever it reports exceeded_maximum_poas."""
    from genomeworks_b200 import cudapoa
    cfg = cudapoa.make_config(2 * window_length, max_depth + 1, 256, "adaptive_band")
    batch = cudapoa.CudaPoaBatch(max_depth + 1, 2 * window_length, max_gpu_mem, output_type="consensus", config=cfg)
    status, cons = [cudapoa.generic_error] * len(groups), [b""] * len(groups)
    pending = []

    def flush():
        if not pending:
            return
        batch.generate_poa()
        c, _, st = batch.get_consensus()
        for i, gi in enumerate(pending):
            status[gi] = st[i]
            if st[i] == cudapoa.success:
                cons[gi] = c[i].encode("latin-1")
        pending.clear()
        batch.reset()

    for gi, (grp, wts) in enumerate(zip(groups, weights)):
        args = ([len(grp)], [len(s) for s in grp], np.frombuffer(b"".join(grp), dtype=np.uint8), np.concatenate(wts))
        st, added = batch.add_poa_groups_flat(*args)
        if st == cudapoa.exceeded_maximum_poas:
            flush()
            st, added = batch.add_poa_groups_flat(*args)
        if st in (cudapoa.success, cudapoa.empty_poa_group):
            assert added == 1
            pending.append(gi)
        else:
            status[gi] = st
    flush()
    batch.close()
    return status, cons


def composition_q(drafts, reads, qualities, threshold, window_length=500, max_depth=30, **mapper_kwargs):
    """The polisher with qualities restated from proven parts -> (polished drafts, outcome array, status array, used,
    candidates)."""
    from genomeworks_b200 import cudamapper
    drafts, reads = list(drafts), list(reads)
    mapper_kwargs.setdefault("filtering_parameter", 1.0)
    if drafts and reads:
        ov, cigars, _ = cudamapper.map_reads(drafts, reads, align=True, **mapper_kwargs)
    else:
        ov, cigars = np.zeros(0, dtype=pl.OVERLAP_DTYPE), []
    rc, g = oracle_groups_q(ov, cigars, drafts, reads, qualities, threshold, window_length, max_depth)
    assert rc == 0
    status, cons = poa_groups_weighted(pl.split_groups(g), split_weights(g), window_length, max_depth)
    polished, outcome, st = pl.oracle_stitch(drafts, window_length, g["used"], status, cons)
    return polished, outcome, st, g["used"], g["candidates"]


def quality_case(seed, truth_len, draft_rate, coverage, read_lo, read_hi, read_rate, q_edit=8.0, q_good=25.0):
    """(truth, draft, reads, qualities): pl.polishing_case's reads with simulated phred strings, the edited bases drawn around
    q_edit and the others around q_good. Each read is simulated forward from the truth, its qualities follow its bases, and
    every other read is reverse-complemented with its qualities reversed."""
    rng = np.random.default_rng(seed)
    truth = pl.random_seq(rng, truth_len)
    draft = pl.mutate(rng, truth, draft_rate)
    reads, quals, total = [], [], 0
    acgt = b"ACGT"
    while total < coverage * truth_len:
        ln = int(rng.integers(read_lo, read_hi + 1))
        st = int(rng.integers(0, max(1, truth_len - ln)))
        out, low = bytearray(), []
        u, kind = rng.random(ln), rng.random(ln)
        for i, c in enumerate(truth[st:st + ln]):
            if u[i] >= read_rate:
                out.append(c)
                low.append(False)
            elif kind[i] < 0.5:
                out.append(acgt[(acgt.index(c) + int(rng.integers(1, 4))) % 4])
                low.append(True)
            elif kind[i] < 0.75:
                out += bytes([c, acgt[int(rng.integers(0, 4))]])
                low += [False, True]
        low = np.array(low, dtype=bool)
        q = np.clip(np.rint(np.where(low, rng.normal(q_edit, 2.0, len(low)), rng.normal(q_good, 4.0, len(low)))), 0, 93).astype(np.uint8) + 33
        r = bytes(out)
        if len(reads) % 2:
            r, q = pl.revcomp(r), q[::-1]
        reads.append(r)
        quals.append(bytes(q))
        total += ln
    return truth, draft, reads, quals
