"""ctypes bindings of the polisher's CPU restatement (oracle/liboracle_polish.so, oracle/polish_oracle.cpp, built by build()) and
the seeded inputs the polisher's tests share.

- oracle_groups: steps 2-4 of DESIGN.md 15.1 (the window groups), in the shape cudapolish.window_groups returns;
- oracle_stitch: step 6 given each group's POA status and consensus;
- composition: the polisher restated from proven parts: map_reads(drafts, reads, align=True), oracle_groups,
  CudaPoaBatch.add_poa_group per group, oracle_stitch.
"""
import ctypes as C

import numpy as np

from checker_lib import ROOT, load, ptr  # noqa: F401

KEYS = ("draft_window_first", "candidates", "used", "group_draft", "group_window", "win_nseq", "seq_len", "seq_data")
OVERLAP_DTYPE = np.dtype({"names": ["query_read_id", "target_read_id", "query_start_position_in_read", "target_start_position_in_read",
                                    "query_end_position_in_read", "target_end_position_in_read", "relative_strand", "num_residues",
                                    "overlap_complete"],
                          "formats": ["<u4", "<u4", "<u4", "<u4", "<u4", "<u4", "u1", "<u4", "u1"],
                          "offsets": [0, 4, 8, 12, 16, 20, 24, 28, 32], "itemsize": 36})

class _View(C.Structure):
    _fields_ = [("n_drafts", C.c_int64), ("n_windows", C.c_int64), ("draft_window_first", C.c_void_p), ("candidates", C.c_void_p),
                ("used", C.c_void_p), ("n_groups", C.c_int64), ("group_draft", C.c_void_p), ("group_window", C.c_void_p),
                ("win_nseq", C.c_void_p), ("n_sequences", C.c_int64), ("seq_len", C.c_void_p), ("n_bases", C.c_int64),
                ("seq_data", C.c_void_p), ("n_kept", C.c_int64)]


def oracle():
    return load("liboracle_polish.so", {
        "oracle_polish_groups": (C.c_int, [C.c_void_p, C.c_int64, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_char_p,
                                           C.c_void_p, C.c_int64, C.c_int32, C.c_int32]),
        "oracle_polish_view": (C.c_int, [C.POINTER(_View)]),
        "oracle_polish_stitch": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_char_p, C.c_void_p]),
        "oracle_polish_stitched": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                             C.POINTER(C.c_int64)])})


def _array(ptr, n, dtype):
    dtype = np.dtype(dtype)
    if n <= 0:
        return np.zeros(0, dtype=dtype)
    return np.frombuffer(C.string_at(ptr, n * dtype.itemsize), dtype=dtype).copy()


def _flat(seqs):
    bs = [s.encode() if isinstance(s, str) else bytes(s) for s in seqs]
    offs = np.zeros(len(bs) + 1, dtype=np.int64)
    if bs:
        offs[1:] = np.cumsum([len(b) for b in bs])
    return b"".join(bs), offs


def cigar_text(cigars):
    cg = [c.encode() if isinstance(c, str) else bytes(c) for c in cigars]
    offs = np.zeros(len(cg) + 1, dtype=np.int64)
    if cg:
        offs[1:] = np.cumsum([len(c) for c in cg])
    return b"".join(cg), offs


def oracle_groups(overlaps, cigars, drafts, reads, window_length, max_depth):
    """(0, dict of KEYS and "n_kept") or (-1, None) for the arguments the contract rejects."""
    ov = np.ascontiguousarray(overlaps, dtype=OVERLAP_DTYPE)
    text, toffs = cigar_text(cigars)
    db, doffs = _flat(drafts)
    rb, roffs = _flat(reads)
    rc = oracle().oracle_polish_groups(ptr(ov), len(ov), text, ptr(toffs), db,
                                       ptr(doffs), len(doffs) - 1, rb, ptr(roffs), len(roffs) - 1,
                                       window_length, max_depth)
    if rc != 0:
        return rc, None
    v = _View()
    oracle().oracle_polish_view(C.byref(v))
    return 0, {
        "draft_window_first": _array(v.draft_window_first, v.n_drafts + 1, np.int64),
        "candidates": _array(v.candidates, v.n_windows, np.int32),
        "used": _array(v.used, v.n_windows, np.int32),
        "group_draft": _array(v.group_draft, v.n_groups, np.int32),
        "group_window": _array(v.group_window, v.n_groups, np.int32),
        "win_nseq": _array(v.win_nseq, v.n_groups, np.int32),
        "seq_len": _array(v.seq_len, v.n_sequences, np.int32),
        "seq_data": _array(v.seq_data, v.n_bases, np.uint8),
        "n_kept": v.n_kept,
    }


def oracle_stitch(drafts, window_length, used, group_status, consensus):
    """(polished drafts as bytes, outcome array, status array) of step 6."""
    db, doffs = _flat(drafts)
    used = np.ascontiguousarray(used, dtype=np.int32)
    st = np.ascontiguousarray(group_status, dtype=np.int32)
    ctext, coffs = _flat(consensus)
    oracle().oracle_polish_stitch(db, ptr(doffs), len(doffs) - 1, window_length, ptr(used),
                                  ptr(st), ctext, ptr(coffs))
    text, offs, outcome, status, n = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_int64()
    oracle().oracle_polish_stitched(C.byref(text), C.byref(offs), C.byref(outcome), C.byref(status), C.byref(n))
    o = _array(offs.value, len(doffs), np.int64)
    t = C.string_at(text.value, int(o[-1])) if len(o) and o[-1] else b""
    return [t[o[i]:o[i + 1]] for i in range(len(o) - 1)], _array(outcome.value, n.value, np.int32), _array(status.value, n.value, np.int32)


def split_groups(g):
    """The groups of a window-groups dict as lists of bytes."""
    out, s, off = [], 0, 0
    data = bytes(g["seq_data"])
    for ns in g["win_nseq"]:
        grp = []
        for k in range(int(ns)):
            ln = int(g["seq_len"][s + k])
            grp.append(data[off:off + ln])
            off += ln
        s += int(ns)
        out.append(grp)
    return out


def poa_groups(groups, window_length, max_depth, max_gpu_mem=2 << 30):
    """(status, consensus bytes) of each group through CudaPoaBatch.add_poa_group with the polisher's configuration, the batch
    generated and reset whenever it reports exceeded_maximum_poas."""
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

    for gi, grp in enumerate(groups):
        st, _ = batch.add_poa_group(list(grp))
        if st == cudapoa.exceeded_maximum_poas:
            flush()
            st, _ = batch.add_poa_group(list(grp))
        if st in (cudapoa.success, cudapoa.empty_poa_group):
            pending.append(gi)
        else:
            status[gi] = st
    flush()
    batch.close()
    return status, cons


def composition(drafts, reads, window_length=500, max_depth=30, **mapper_kwargs):
    """The polisher restated from proven parts -> (polished drafts, outcome array, status array, used, candidates)."""
    from genomeworks_b200 import cudamapper
    drafts, reads = list(drafts), list(reads)
    mapper_kwargs.setdefault("filtering_parameter", 1.0)  # the polisher's default
    if drafts and reads:
        ov, cigars, _ = cudamapper.map_reads(drafts, reads, align=True, **mapper_kwargs)
    else:
        ov, cigars = np.zeros(0, dtype=OVERLAP_DTYPE), []
    rc, g = oracle_groups(ov, cigars, drafts, reads, window_length, max_depth)
    assert rc == 0
    status, cons = poa_groups(split_groups(g), window_length, max_depth)
    polished, outcome, st = oracle_stitch(drafts, window_length, g["used"], status, cons)
    return polished, outcome, st, g["used"], g["candidates"]


# ---------------------------------------------------------------------------------------------------------------------------
# inputs

_COMP = bytes.maketrans(b"ACGT", b"TGCA")


def revcomp(s):
    return bytes(s).translate(_COMP)[::-1]


def random_seq(rng, n):
    return bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), n).astype(np.uint8))


def mutate(rng, s, rate, sub=0.5, ins=0.25):
    """s with about `rate` edits per base: a `sub` share substitutions, an `ins` share insertions, the rest deletions."""
    out = bytearray()
    acgt = b"ACGT"
    u = rng.random(len(s))
    kind = rng.random(len(s))
    for i, c in enumerate(s):
        if u[i] >= rate:
            out.append(c)
        elif kind[i] < sub:
            out.append(acgt[(acgt.index(c) + int(rng.integers(1, 4))) % 4] if c in acgt else c)
        elif kind[i] < sub + ins:
            out.append(c)
            out.append(acgt[int(rng.integers(0, 4))])
    return bytes(out)


def polishing_case(seed, truth_len, draft_rate, coverage, read_lo, read_hi, read_rate):
    """(truth, draft, reads): the draft is the truth with draft_rate edits; reads of read_lo .. read_hi bases cut from the truth at
    `coverage`, each with read_rate edits, every other one reverse-complemented."""
    rng = np.random.default_rng(seed)
    truth = random_seq(rng, truth_len)
    draft = mutate(rng, truth, draft_rate)
    reads, total = [], 0
    while total < coverage * truth_len:
        ln = int(rng.integers(read_lo, read_hi + 1))
        st = int(rng.integers(0, max(1, truth_len - ln)))
        r = mutate(rng, truth[st:st + ln], read_rate)
        reads.append(revcomp(r) if len(reads) % 2 else r)
        total += ln
    return truth, draft, reads


def random_cigar(rng, q_span, t_span, max_run):
    """A random M/I/D CIGAR consuming exactly q_span draft and t_span read bases, with runs up to max_run."""
    ops = []
    q, t = q_span, t_span
    while q > 0 or t > 0:
        choices = []
        if q > 0 and t > 0:
            choices.append("M")
        if t > 0:
            choices.append("I")
        if q > 0:
            choices.append("D")
        op = choices[int(rng.integers(0, len(choices)))]
        cap = min(q if op == "D" else t if op == "I" else min(q, t), max_run)
        n = int(rng.integers(1, cap + 1))
        if ops and ops[-1][0] == op:
            ops[-1][1] += n
        else:
            ops.append([op, n])
        if op != "I":
            q -= n
        if op != "D":
            t -= n
    return "".join("%d%s" % (n, op) for op, n in ops)


def random_overlaps(seed, n, draft_lengths, n_reads, read_len, max_run, window_length):
    """n overlaps over random drafts and reads (read i is always read i % n_reads) with random CIGARs: (overlaps, cigars, drafts,
    reads). Intervals and runs are drawn so that pieces cross many windows and both strands occur."""
    rng = np.random.default_rng(seed)
    drafts = [random_seq(rng, int(d)) for d in draft_lengths]
    reads = [random_seq(rng, read_len) for _ in range(n_reads)]
    ov = np.zeros(n, dtype=OVERLAP_DTYPE)
    cigars = []
    for i in range(n):
        d = int(rng.integers(0, len(drafts)))
        D = len(drafts[d])
        qs = int(rng.integers(0, D))
        qe = int(rng.integers(qs, min(D, qs + 4 * window_length + 50) + 1))
        if rng.random() < 0.2:  # snap to window edges so that full pieces occur
            qs = qs // window_length * window_length
            qe = min(D, -(-qe // window_length) * window_length)
        ql = qe - qs
        tl = max(0, min(read_len, ql + int(rng.integers(-ql // 4 - 1, ql // 4 + 2))))
        ts = int(rng.integers(0, read_len - tl + 1))
        ov[i] = (d, i % n_reads, qs, ts, qe, ts + tl, ord("-") if rng.random() < 0.5 else ord("+"), 1, 1)
        cigars.append(random_cigar(rng, ql, tl, max_run) if ql + tl > 0 else "")
    return ov, cigars, drafts, reads
