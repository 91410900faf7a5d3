"""The POA kernels on weighted windows of the polisher's and the corrector's shape, against the CPU oracle (DESIGN.md 15.3, 15.5).

The polisher's own GPU tests compare it with a composition that runs the same POA batch, so a POA fault would appear on both
sides. Here every window goes through the batch (tests/poa_window_libs.py: gwb200_poa_batch_add_group with per-sequence weight
pointers, the draft's NULL) and through oracle_lib.poa_run with explicit weights, after the batch's admission rules restated in
Python. Each case compares per-sequence admission, status, consensus, coverage and the executed DP cells, and asserts the path it
is meant to reach: the kernel, the score and index widths, the number of batches, or the consensus flip at the edge-weight bound.
"""
import numpy as np
import pytest

import poa_window_libs as pw
import polish_libs as pl
import polish_quality_libs as pq
import correct_libs as cl
import ref_lib
from test_gpu_poa import assert_same_as_reference, poa_digests

pytestmark = pytest.mark.gpu

KERNELS = {"tb": 0, "v3": 1, "v1": 2}


def _groups_as_windows(g):
    """A window-groups dict as polisher windows: the draft window's weight pointer NULL, each piece's weights its own. The draft
    windows' weights in the dict are ones, which the NULL pointer gives too."""
    out = []
    for seqs, wts in zip(pl.split_groups(g), pq.split_weights(g)):
        assert (wts[0] == 1).all()
        out.append((seqs, [None] + list(wts[1:])))
    return out


_REAL = {}


def _real_windows():
    """Every group of 2 or more used pieces the cutting stage gives at W = 500, c = 30: the polisher's on quality_case reads at
    t = 0 and t = 10, the corrector's on a 10 %-error correction_case with qualities. Computed once, with their oracle results."""
    if not _REAL:
        from genomeworks_b200 import cudamapper, cudapolish
        windows = []
        truth, draft, reads, quals = pq.quality_case(21, 12000, 0.01, 12, 1500, 4000, 0.10)
        ov, cigars, _ = cudamapper.map_reads([draft], reads, align=True, filtering_parameter=1.0)
        for t in (0.0, 10.0):
            g = cudapolish.window_groups(ov, cigars, [draft], reads, 500, 30, read_qualities=quals, quality_threshold=t)
            assert len(g["win_nseq"]) >= 20 and (g["win_nseq"] >= 3).all()
            windows += _groups_as_windows(g)
        _, creads, _, _ = cl.correction_case(22, 8000, 10, 1000, 3000, 0.10)
        cquals = pq.random_qualities(22, creads, 5, 40)
        ov, cigars, _ = cudamapper.map_reads(creads, align=True, filtering_parameter=1.0)
        g = cudapolish.correction_window_groups(ov, cigars, creads, 500, 30, read_qualities=cquals, quality_threshold=10.0)
        assert len(g["win_nseq"]) >= 20
        windows += _groups_as_windows(g)
        cfg = pw.polisher_config(500, 30)
        _REAL.update(windows=windows, cfg=cfg, oracle=pw.run_oracle(windows, cfg))
    return _REAL


@pytest.mark.parametrize("batches", ["one", "several"])
def test_real_windows_vs_oracle(batches, device_fdiv):
    from genomeworks_b200 import cudapoa
    real = _real_windows()
    windows, cfg = real["windows"], real["cfg"]
    mem = 2 << 30
    if batches == "several":
        b = cudapoa.CudaPoaBatch(cfg.max_sequences_per_poa, cfg.max_sequence_size, mem, config=cfg)
        per_gb = b.max_poas / 2.0
        b.close()
        mem = int((1 << 30) * (len(windows) / 4.0) / per_gb)
    ours = pw.run_batch(windows, cfg, mem)
    assert ours["kernel"] == KERNELS["v3"] and ours["score_bytes"] == 2
    if batches == "one":
        assert ours["batches"] == 1
        _REAL["pool_one"] = ours["pool_bytes"]
    else:
        assert ours["batches"] >= 3, ours["batches"]
        # fewer windows per SM: a larger shared-memory pool per window, so a deeper ring of score rows in the v3 kernel
        if "pool_one" in _REAL:
            assert ours["pool_bytes"] > _REAL["pool_one"]
    pw.assert_same(ours, real["oracle"], "real windows, %s batch(es)" % batches)
    assert sum(s == 0 for s in ours["status"]) >= 0.9 * len(windows)


# W -> (kernel, score bytes, index bytes, windows, pieces)
GRID = {
    1: ("v3", 2, 2, 40, 30),
    7: ("v3", 2, 2, 40, 30),
    744: ("v3", 2, 2, 4, 8),
    745: ("v3", 4, 2, 4, 8),
    5460: ("v3", 4, 2, 2, 3),
    5461: ("v3", 4, 4, 2, 3),
    32768: ("v1", 4, 4, 1, 3),
}


@pytest.mark.parametrize("window_length", sorted(GRID))
def test_window_length_grid(window_length, device_fdiv):
    """The polisher's config at the window lengths where its instantiation changes: int32 scores from W = 745 (44 W > 32768),
    int32 indices from W = 5461 (align_up(6 W, 4) = 32768), the first-generation kernel at W = 32768 (reads of 65536)."""
    W = window_length
    kernel, sb, ib, n_windows, n_pieces = GRID[W]
    cfg = pw.polisher_config(W, 30)
    assert pw.index_bytes(cfg) == ib
    windows = pw.polisher_windows(100 + W % 1000, n_windows, W, n_pieces, 0.2 if W < 8 else (0.03 if W < 1000 else 0.01))
    ours = pw.run_batch(windows, cfg, 8 << 30)
    assert ours["kernel"] == KERNELS[kernel] and ours["score_bytes"] == sb
    pw.assert_same(ours, pw.run_oracle(windows, cfg), "W = %d" % W)
    assert all(s == 0 for s in ours["status"])


@pytest.mark.parametrize("rate", [0.01, 0.10])
@pytest.mark.parametrize("depth", [31, 100, 352])
def test_depth(depth, rate, device_fdiv):
    """W = 500 at the depths the polisher allows with qualities, weights 0 .. 93; each window also offers two pieces more than
    the batch takes, so the last are refused as exceeded_maximum_sequences_per_poa."""
    n_windows = {31: 6, 100: 3, 352: 2}[depth]
    windows = pw.polisher_windows(depth + int(rate * 100), n_windows, 500, depth + 2, rate)
    cfg = pw.polisher_config(500, depth)
    ours = pw.run_batch(windows, cfg, 8 << 30)
    assert ours["kernel"] == KERNELS["v3"] and ours["score_bytes"] == 2
    orc = pw.run_oracle(windows, cfg)
    for per in orc["per_seq"]:
        assert per[-1] == pw.EXCEEDED_MAXIMUM_SEQUENCES_PER_POA and per.count(0) == depth + 1
    pw.assert_same(ours, orc, "depth %d, %g divergence" % (depth, rate))
    print("depth %d, rate %g: statuses %s" % (depth, rate, sorted(set(ours["status"]))))


@pytest.mark.parametrize("mode", ["adaptive_band", "static_band", "adaptive_band_traceback"])
def test_edge_weights_at_their_bound(mode, device_fdiv):
    """The 352 / 353 case of DESIGN.md 15.5 through the kernels: the majority's edges weigh 65474 at 352 and wrap to 124 at 353,
    where the three minority reads (558) win. The kernel must wrap as the oracle does."""
    from genomeworks_b200 import cudapoa
    cases = [pw.flip_window(n) for n in (352, 353)]
    windows = [c[0] for c in cases]
    cfg = cudapoa.make_config(120, 360, 256, mode)
    ours = pw.run_batch(windows, cfg, 4 << 30)
    assert ours["kernel"] == KERNELS["tb" if "traceback" in mode else "v3"]
    pw.assert_same(ours, pw.run_oracle(windows, cfg), "edge weights, " + mode)
    assert ours["status"] == [0, 0]
    assert ours["consensus"] == [cases[0][1], cases[1][2]], "majority at 352, minority at 353"


def _oracle_polish(drafts, reads, quals, threshold, window_length, max_depth):
    """The polisher from the oracle alone after the mapper: the oracle's groups and weights, the batch's admission restated, the
    oracle's POA with the polisher's config and the oracle's stitching -> (polished, outcome, status, groups dict, windows)."""
    from genomeworks_b200 import cudamapper
    ov, cigars, _ = cudamapper.map_reads(drafts, reads, align=True, filtering_parameter=1.0)
    rc, g = pq.oracle_groups_q(ov, cigars, drafts, reads, quals, threshold, window_length, max_depth)
    assert rc == 0
    windows = _groups_as_windows(g)
    orc = pw.run_oracle(windows, pw.polisher_config(window_length, max_depth))
    cons = [c.encode() if s == 0 else b"" for c, s in zip(orc["consensus"], orc["status"])]
    polished, outcome, status = pl.oracle_stitch(drafts, window_length, g["used"], orc["status"], cons)
    return polished, outcome, status, g, windows


def test_polish_at_max_depth_352_q93(device_fdiv):
    """polish() with every read Q93 and max_depth = 352, 360 reads over every window: the draft edge weighs 2 + 352 x 186 = 65474."""
    from genomeworks_b200 import cudapolish
    rng = np.random.default_rng(352)
    truth = pl.random_seq(rng, 2500)
    draft = pl.mutate(rng, truth, 0.01)
    reads = [pl.mutate(rng, truth, 0.01) for _ in range(360)]
    reads = [pl.revcomp(r) if i % 2 else r for i, r in enumerate(reads)]
    quals = [b"~" * len(r) for r in reads]
    got, outcomes = cudapolish.polish([draft], reads, max_depth=352, read_qualities=quals, quality_threshold=10)
    want, outcome, status, g, _ = _oracle_polish([draft], reads, quals, 10.0, 500, 352)
    assert np.array_equal(outcomes["used"], g["used"]) and np.array_equal(outcomes["candidates"], g["candidates"])
    assert np.array_equal(outcomes["outcome"], outcome) and np.array_equal(outcomes["status"], status)
    # the interior windows, which every read covers from end to end, run at the full depth
    assert (outcomes["used"][1:-1] == 352).all() and (outcome[1:-1] == cudapolish.POLISHED).all()
    assert got == want


def test_zero_weight_piece_is_dropped_but_counted(device_fdiv):
    """polish() at t = 0 with one read all '!': its pieces pass the filter (0 >= 0), count in `used`, and the batch drops them as
    zero_weighted_poa_sequence, so each window's POA is the oracle's on the group without that piece (DESIGN.md 15.5)."""
    from genomeworks_b200 import cudapolish
    rng = np.random.default_rng(77)
    truth = pl.random_seq(rng, 3500)
    draft = pl.mutate(rng, truth, 0.01)
    reads = [pl.mutate(rng, truth, 0.05) for _ in range(9)]
    reads = [pl.revcomp(r) if i % 2 else r for i, r in enumerate(reads)]
    quals = pq.random_qualities(77, reads, 10, 40)
    quals[4] = b"!" * len(reads[4])
    got, outcomes = cudapolish.polish([draft], reads, read_qualities=quals, quality_threshold=0.0)
    want, outcome, status, g, windows = _oracle_polish([draft], reads, quals, 0.0, 500, 30)
    zero = [sum(1 for w in wts[1:] if not (w > 0).any()) for _, wts in windows]
    assert len(windows) >= 3 and max(zero) == 1 and sum(zero) >= 2, "windows hold the all-'!' read's piece"
    assert np.array_equal(outcomes["used"], g["used"])
    for k, (seqs, _) in enumerate(windows):
        assert outcomes["used"][g["group_window"][k]] == len(seqs) - 1  # the zero-weight piece included
    assert np.array_equal(outcomes["outcome"], outcome) and np.array_equal(outcomes["status"], status)
    assert got == want
    # and the batch's own admission of the same windows
    cfg = pw.polisher_config(500, 30)
    ours = pw.run_batch(windows, cfg)
    assert all(per.count(pw.ZERO_WEIGHTED_POA_SEQUENCE) == 1 for per in ours["per_seq"])
    pw.assert_same(ours, pw.run_oracle(windows, cfg), "all-'!' piece")


# ---------------------------------------------------------------------------------------------------------------------------
# weights on every kernel, against the oracle and the stored outputs of the reference kernels

# name -> (max_sequence_size, max_sequences_per_poa, band, band mode, kernel, score bytes, index bytes, window length, windows)
MATRIX = {
    "v3_static_int16": (1000, 12, 256, "static_band", "v3", 2, 2, 300, 8),
    "v3_adaptive_int16": (1000, 12, 256, "adaptive_band", "v3", 2, 2, 300, 8),
    "v3_adaptive_int32_scores": (1490, 12, 256, "adaptive_band", "v3", 4, 2, 600, 6),
    "v3_adaptive_int32_indices": (10922, 6, 256, "adaptive_band", "v3", 4, 4, 5000, 2),
    "static_band_traceback": (1000, 12, 256, "static_band_traceback", "tb", 2, 2, 300, 8),
    "adaptive_band_traceback": (1000, 12, 256, "adaptive_band_traceback", "tb", 2, 2, 300, 8),
    "v1_static_2048": (1000, 12, 2048, "static_band", "v1", 2, 2, 300, 8),
}


def _flat(windows):
    win_nseq = np.array([len(s) for s, _ in windows], dtype=np.int32)
    seq_len = np.array([len(x) for s, _ in windows for x in s], dtype=np.int32)
    data = np.frombuffer(b"".join(x for s, _ in windows for x in s) + b"\0", dtype=np.uint8)
    weights = np.concatenate([w for s, wts in windows for w in pw.explicit_weights(s, wts)] + [np.zeros(1, np.int8)])
    return win_nseq, seq_len, data, weights


@pytest.mark.parametrize("name", sorted(MATRIX))
def test_weights_on_every_kernel(name, device_fdiv):
    """Small windows with weights 0 .. 93, runs of 0 and one all-zero piece per window, on each kernel and instantiation."""
    from genomeworks_b200 import cudapoa
    max_seq, nseq, band, mode, kernel, sb, ib, W, n = MATRIX[name]
    windows = pw.polisher_windows(500 + len(name), n, W, nseq - 3, 0.05, all_zero=True, draft_null=False)
    cfg = cudapoa.make_config(max_seq, nseq, band, mode)
    assert pw.index_bytes(cfg) == ib
    ours = pw.run_batch(windows, cfg, 8 << 30)
    assert ours["kernel"] == KERNELS[kernel] and ours["score_bytes"] == sb
    for per in ours["per_seq"]:
        assert per.count(pw.ZERO_WEIGHTED_POA_SEQUENCE) == 1
    pw.assert_same(ours, pw.run_oracle(windows, cfg), name)
    assert all(s == 0 for s in ours["status"])
    win_nseq, seq_len, data, weights = _flat(windows)
    ref = ref_lib.recorded("poa/weights_matrix/" + name, lambda: poa_digests(ref_lib.ref_poa_run(
        win_nseq, seq_len, data, max_seq, nseq, band, cfg.band_mode, weights=weights)))
    assert_same_as_reference(dict(consensus=ours["consensus"], coverage=ours["coverage"], status=np.array(ours["status"])), ref,
                             "reference " + name)


# ---------------------------------------------------------------------------------------------------------------------------
# NULL weight pointers

def _null_cases(seed):
    """(unweighted windows, weighted windows with some NULL pointers, the polisher's window): an unweighted window passes no
    weight array at all; a weighted one has per-sequence pointers, a NULL among them."""
    plain = [(s, None) for s, _ in pw.polisher_windows(seed, 3, 200, 5, 0.05)]
    weighted = pw.polisher_windows(seed + 1, 3, 200, 5, 0.05, draft_null=False)
    for i, (s, w) in enumerate(weighted):
        w[1 + i % 5] = None
    polisher = pw.polisher_windows(seed + 2, 2, 200, 5, 0.05)  # the draft NULL, the pieces weighted
    return plain, weighted, polisher


def test_null_weight_pointers(device_fdiv):
    """gwb200_poa_batch_add_group with NULL weight pointers in every order the host handles differently: unweighted groups
    before the batch's first weighted read (their unit weights written then), NULL reads after it, reset() clearing the weighted
    state before the opposite order, a batch with no weights at all (unit weights set on the device), and the polisher's draft
    NULL with weighted pieces as the first group of a batch. Each against the oracle given explicit ones."""
    from genomeworks_b200 import cudapoa
    plain, weighted, polisher = _null_cases(900)
    cfg = pw.polisher_config(200, 10)
    orders = [
        ("unweighted then weighted", plain + weighted),
        ("weighted then NULL", weighted + plain),
        ("polisher's window first", polisher + plain + weighted),
        ("no weights at all", plain),
        ("NULL pointers only", [(s, [None] * len(s)) for s, _ in plain]),
    ]
    b = cudapoa.CudaPoaBatch(cfg.max_sequences_per_poa, cfg.max_sequence_size, 2 << 30, config=cfg)
    try:
        # each order after reset() of a batch that ran the one before it, then the first two again in the opposite sequence
        for name, windows in orders + orders[1::-1]:
            ours = pw.run_batch(windows, cfg, batch=b)
            assert ours["batches"] == 1
            pw.assert_same(ours, pw.run_oracle(windows, cfg), name)
            assert all(s == 0 for s in ours["status"])
    finally:
        b.close()
    # the weights matter here: with unit weights the weighted windows' consensus differs somewhere
    unit = pw.run_oracle([(s, None) for s, _ in weighted + polisher], cfg)
    assert unit["consensus"] != pw.run_oracle(weighted + polisher, cfg)["consensus"]
