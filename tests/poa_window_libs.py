"""Weighted POA windows shaped like the polisher's (DESIGN.md sections 15.1 and 15.5), run through the POA batch and through the
CPU oracle, and compared window by window.

A window is (sequences, weights): a list of bytes and either None (every weight pointer NULL) or one entry per sequence, an int8
array or None (that sequence's pointer NULL, unit weights in the batch). The polisher passes the draft window as None and each
piece's phred weights q - 33.

- run_batch: the windows through gwb200_poa_batch_add_group, one group per call with per-sequence weight pointers; the batch is
  generated, read and reset whenever it reports exceeded_maximum_poas, as the polisher does;
- admit: the batch's admission rules restated, since the oracle does not apply them;
- run_oracle: the admitted windows through oracle_lib.poa_run with explicit weights (ones for NULL);
- assert_same: status, consensus, coverage and the executed DP cells, which pin every band width and rerun of the adaptive band;
- polisher_windows: synthetic windows of the polisher's shape."""
import ctypes as C

import numpy as np

import oracle_lib as ol

SUCCESS = 0
EXCEEDED_MAXIMUM_POAS = 1
EXCEEDED_MAXIMUM_SEQUENCE_SIZE = 2
EXCEEDED_MAXIMUM_SEQUENCES_PER_POA = 3
ZERO_WEIGHTED_POA_SEQUENCE = 10
EMPTY_POA_GROUP = 11


def polisher_config(window_length, max_depth):
    """The polisher's batch configuration for W = window_length and c = max_depth: BatchConfig(2W, c + 1, 256, adaptive_band)."""
    from genomeworks_b200 import cudapoa
    return cudapoa.make_config(2 * window_length, max_depth + 1, 256, "adaptive_band")


def cfg8(cfg):
    return np.array([cfg.max_sequence_size, cfg.max_consensus_size, cfg.max_nodes_per_graph, cfg.matrix_sequence_dimension,
                     cfg.alignment_band_width, cfg.max_sequences_per_poa, cfg.band_mode, cfg.max_banded_pred_distance], dtype=np.int32)


def index_bytes(cfg):
    """sizeof(SizeT) the config selects: int32 node and read indices once any of these dimensions passes INT16_MAX."""
    return 4 if max(cfg.max_consensus_size, cfg.max_nodes_per_graph, cfg.matrix_sequence_dimension) > 32767 else 2


def explicit_weights(seqs, weights):
    """The weights of a window with every NULL pointer replaced by unit weights, as the batch reads them."""
    if weights is None:
        weights = [None] * len(seqs)
    return [np.ones(len(s), np.int8) if w is None else np.asarray(w, dtype=np.int8) for s, w in zip(seqs, weights)]


def admit(seqs, weights, cfg):
    """(per-sequence status, admitted sequences, their explicit weights) under the batch's rules, in this order: a sequence longer
    than max_sequence_size is dropped; an all-zero-weight one is dropped; one past max_sequences_per_poa admitted ones is
    dropped. A group that keeps nothing still occupies a window (empty_poa_group)."""
    status, kept, kept_w = [], [], []
    for s, w in zip(seqs, explicit_weights(seqs, weights)):
        if len(s) > cfg.max_sequence_size:
            status.append(EXCEEDED_MAXIMUM_SEQUENCE_SIZE)
        elif not (w > 0).any():
            status.append(ZERO_WEIGHTED_POA_SEQUENCE)
        elif len(kept) >= cfg.max_sequences_per_poa:
            status.append(EXCEEDED_MAXIMUM_SEQUENCES_PER_POA)
        else:
            status.append(SUCCESS)
            kept.append(bytes(s))
            kept_w.append(w)
    return status, kept, kept_w


def add_group(batch, seqs, weights):
    """gwb200_poa_batch_add_group with per-sequence weight pointers -> (status, per-sequence statuses)."""
    from genomeworks_b200._lib import check, lib
    n = len(seqs)
    seqs = [bytes(s) for s in seqs]
    arr = (C.c_char_p * n)(*seqs)
    lens = (C.c_int32 * n)(*[len(s) for s in seqs])
    wp, keep = None, None
    if weights is not None:
        keep = [None if w is None else np.ascontiguousarray(w, dtype=np.int8) for w in weights]
        ptrs = (C.c_void_p * n)(*[None if w is None else w.ctypes.data for w in keep])
        wp = C.cast(ptrs, C.c_void_p)
    per = (C.c_int32 * n)()
    nper = C.c_int32(0)
    rc = check(lib().gwb200_poa_batch_add_group(batch._h, C.c_int32(n), arr, wp, lens, per, C.byref(nper)))
    del keep
    return rc, [int(per[i]) for i in range(nper.value)]


def run_batch(windows, cfg, max_gpu_mem=2 << 30, batch=None):
    """The windows through the POA batch in order, generated and reset at every exceeded_maximum_poas. Returns a dict: per window
    "status", "consensus", "coverage" and "per_seq" (add_group's per-sequence statuses); "cells" summed over the batches run,
    "batches", and the batch's "kernel", "score_bytes", "pool_bytes" and "max_poas". A given batch is used as it is and left
    open."""
    from genomeworks_b200 import cudapoa
    own = batch is None
    if own:
        batch = cudapoa.CudaPoaBatch(cfg.max_sequences_per_poa, cfg.max_sequence_size, max_gpu_mem, output_type="consensus", config=cfg)
    n = len(windows)
    out = dict(status=[None] * n, consensus=[None] * n, coverage=[None] * n, per_seq=[None] * n, cells=0, batches=0, kernel=batch.kernel,
               score_bytes=batch.score_bytes, pool_bytes=batch.pool_bytes, max_poas=batch.max_poas)
    pending = []

    def flush():
        if not pending:
            return
        batch.generate_poa()
        cons, cov, st = batch.get_consensus()
        assert len(st) == len(pending)
        for i, wi in enumerate(pending):
            out["status"][wi], out["consensus"][wi], out["coverage"][wi] = int(st[i]), cons[i], [int(x) for x in cov[i]]
        out["cells"] += batch.last_cells()
        out["batches"] += 1
        pending.clear()
        batch.reset()

    try:
        for wi, (seqs, weights) in enumerate(windows):
            rc, per = add_group(batch, seqs, weights)
            if rc == EXCEEDED_MAXIMUM_POAS:
                assert pending, "window %d does not fit an empty batch" % wi
                flush()
                rc, per = add_group(batch, seqs, weights)
            assert rc in (SUCCESS, EMPTY_POA_GROUP), "window %d: add_group returned %d" % (wi, rc)
            out["per_seq"][wi] = per
            pending.append(wi)
        flush()
    finally:
        if own:
            batch.close()
    return out


def run_oracle(windows, cfg, gap=-8, mismatch=-6, match=8):
    """The oracle on the admitted part of every window, in the shape run_batch returns. A window that admits nothing is
    empty_poa_group with an empty consensus and no cells."""
    adm = [admit(seqs, weights, cfg) for seqs, weights in windows]
    live = [i for i, a in enumerate(adm) if a[1]]
    n = len(windows)
    out = dict(status=[EMPTY_POA_GROUP] * n, consensus=[""] * n, coverage=[[]] * n, per_seq=[a[0] for a in adm], cells_per_window=[0] * n)
    if live:
        r = ol.poa_run([adm[i][1] for i in live], cfg8(cfg), gap=gap, mismatch=mismatch, match=match, weights=[adm[i][2] for i in live])
        for k, i in enumerate(live):
            out["status"][i] = int(r["status"][k])
            out["consensus"][i] = r["consensus"][k]
            out["coverage"][i] = [int(x) for x in r["coverage"][k]]
            out["cells_per_window"][i] = int(r["cells"][k])
    out["cells"] = sum(out["cells_per_window"])
    return out


def assert_same(ours, orc, what):
    """Every window's per-sequence admission, status, consensus and coverage, and the cells summed over all windows."""
    assert len(ours["status"]) == len(orc["status"])
    for w in range(len(orc["status"])):
        wn = "%s, window %d" % (what, w)
        assert ours["per_seq"][w] == orc["per_seq"][w], wn + ": per-sequence admission differs"
        assert ours["status"][w] == orc["status"][w], wn + ": status %d, oracle %d" % (ours["status"][w], orc["status"][w])
        assert ours["consensus"][w] == orc["consensus"][w], wn + ": consensus differs"
        assert ours["coverage"][w] == orc["coverage"][w], wn + ": coverage differs"
    assert ours["cells"] == orc["cells"], what + ": executed DP cells %d, oracle %d (a band width or a rerun differs)" % (
        ours["cells"], orc["cells"])


# ---------------------------------------------------------------------------------------------------------------------------
# synthetic windows of the polisher's shape

ACGT = b"ACGT"


def random_seq(rng, n):
    return bytes(rng.choice(np.frombuffer(ACGT, dtype=np.uint8), n).astype(np.uint8))


def mutate(rng, s, rate):
    """s with about `rate` edits per base: half substitutions, a quarter insertions, a quarter deletions."""
    out = bytearray()
    u, kind = rng.random(len(s)), rng.random(len(s))
    for i, c in enumerate(s):
        if u[i] >= rate:
            out.append(c)
        elif kind[i] < 0.5:
            out.append(ACGT[(ACGT.index(c) + int(rng.integers(1, 4))) % 4])
        elif kind[i] < 0.75:
            out += bytes([c, ACGT[int(rng.integers(0, 4))]])
    return bytes(out)


def phred_weights(rng, n, lo=0, hi=93, zero_runs=True):
    """n weights: a level drawn per sequence in lo .. hi, each base within 10 of it (clipped to 0 .. 93), with runs of 0 of 1 - 12
    bases over about a tenth of the sequence when zero_runs is set."""
    level = int(rng.integers(lo, hi + 1))
    w = np.clip(rng.integers(level - 10, level + 11, n), 0, 93).astype(np.int8)
    if zero_runs and n > 1:
        for _ in range(max(1, n // 60)):
            a = int(rng.integers(0, n))
            w[a:a + int(rng.integers(1, 13))] = 0
    return w


def polisher_windows(seed, n_windows, window_length, n_pieces, rate, lo=0, hi=93, zero_runs=True, all_zero=False, draft_null=True):
    """n_windows windows as the polisher builds them: a draft window of W bases with unit weights (a NULL pointer when
    draft_null), then n_pieces pieces of about W +- indels (1 .. 2W bases), each the window's truth with `rate` edits, with phred
    weights (phred_weights). With all_zero, the second piece of every window weighs 0 throughout."""
    rng = np.random.default_rng(seed)
    W = window_length
    out = []
    for _ in range(n_windows):
        truth = random_seq(rng, W)
        draft = mutate(rng, truth, rate)[:W] or truth[:1]
        draft = draft + truth[len(draft):W]
        seqs, weights = [draft], [None if draft_null else np.ones(W, np.int8)]
        for k in range(n_pieces):
            p = mutate(rng, truth, rate)[:2 * W] or truth[:1]
            seqs.append(p)
            weights.append(np.zeros(len(p), np.int8) if all_zero and k == 1 else phred_weights(rng, len(p), lo, hi, zero_runs))
        out.append((seqs, weights))
    return out


def flip_window(n_majority, n_minority=3, length=60, seed=1):
    """The edge-weight bound case (DESIGN.md 15.5): a draft, n_majority copies of it at Q93 and n_minority copies at Q93 with one
    substitution in the middle -> (window, majority, minority). Where the two paths part, the majority's edges weigh
    2 + 186 n_majority, which wraps in uint16_t from n_majority = 353 on."""
    rng = np.random.default_rng(seed)
    base = random_seq(rng, length)
    m = length // 2
    alt = base[:m] + bytes([ACGT[(ACGT.index(base[m]) + 1) % 4]]) + base[m + 1:]
    seqs = [base] + [base] * n_majority + [alt] * n_minority
    weights = [None] + [np.full(length, 93, np.int8)] * (n_majority + n_minority)
    return (seqs, weights), base.decode(), alt.decode()


def edge_weight(n_reads, draft_weight=1, q=93):
    """The weight of an edge every sequence of a window takes: the draft's 2 * draft_weight plus 2q per read, in uint16_t."""
    return (2 * draft_weight + 2 * q * n_reads) & 0xFFFF
