"""The POA kernels on the code paths their config and inputs select, against the CPU oracle.

v3 (poa_nw_v3.cuh) runs every non-traceback batch with a band of at most 1536 and reads shorter than 65 536 bases. Its DP
rows take different code depending on:
  - the chunks per row, ceil(band / 256) (int16 rows in groups of two chunks, int32 rows one at a time, a half chunk at the end);
  - the depth R of the shared-memory ring of score rows, min(pool_bytes / row_bytes, 64), where the pool per CTA shrinks as more
    windows share an SM (v3_pool_bytes in poa_capi.cu);
  - "fast" rows (at most two predecessors, both within R rows) against "general" rows (more predecessors, or one that left the
    ring and is read back from global memory behind a bulk-copy wait);
  - the adaptive band, widened from the read / graph length ratio and doubled on a rerun.
The windows here are built to reach each of these, and each case asserts through CudaPoaBatch.kernel / .pool_bytes that it ran
the kernel and ring depth it was meant for. Every GPU case compares consensus, coverage (or MSA rows), status and the executed
DP cells (which pin the band width of every alignment and every rerun) bit-exactly with oracle_lib.poa_run.

The tests without the gpu mark check, with the oracle alone, that the window builders produce what the GPU cases rely on:
read-1 band widths, reruns, predecessors 64 or more rows back and in-degrees of 3 or more."""
import functools

import numpy as np
import pytest

import oracle_lib as ol

KERNELS = {"tb": 0, "v3": 1, "v1": 2}
MAX_ADAPTIVE_BW = 1536
STRETCH_FLANK = 40

# ---------------------------------------------------------------------------------------------------------------------------
# window builders: plain Python, seeded; a window is a tuple of reads (str), read 0 is the backbone
# ---------------------------------------------------------------------------------------------------------------------------


def _rand(rng, n, alphabet="ACGT"):
    return "".join(alphabet[i] for i in rng.randint(0, len(alphabet), n))


def _substitute(rng, s, n, alphabet="ACGT"):
    """n point substitutions at distinct positions (each to a different base)."""
    b = list(s)
    for p in rng.choice(len(b), size=min(n, len(b)), replace=False):
        b[p] = alphabet[(alphabet.index(b[p]) + rng.randint(1, len(alphabet))) % len(alphabet)] if b[p] in alphabet else "A"
    return "".join(b)


def _with_ns(rng, s, n):
    b = list(s)
    for p in rng.choice(len(b), size=min(n, len(b)), replace=False):
        b[p] = "N"
    return "".join(b)


def planted_backbone(rng, length, stretches):
    """A random backbone with, for each (pos, d) in stretches, d bases drawn from {A, C} at pos, flanked by STRETCH_FLANK bases
    drawn from {G, T} on both sides. A read that deletes such a stretch cannot align its neighbouring bases inside it, so the
    deletion becomes one graph edge that skips d nodes: a predecessor d + 1 rows back. (With random sequence and linear gaps,
    the alignment scatters a long deletion into short ones at no cost.)"""
    out, at = [], 0
    for pos, d in sorted(stretches):
        out.append(_rand(rng, pos - STRETCH_FLANK - at))
        out.append(_rand(rng, STRETCH_FLANK, "GT") + _rand(rng, d, "AC") + _rand(rng, STRETCH_FLANK, "GT"))
        at = pos + d + STRETCH_FLANK
    out.append(_rand(rng, max(0, length - at)))
    return "".join(out)


def build_window(seed, backbone_len, n_reads, subs=0.01, far=(), hub=0, hub_ins=0, long_ins=(), frag=None, ext=0, ext_side="both",
                 ns=0):
    """One window:
      far      -- deletion lengths (70-400); read i (from 1) deletes planted stretch i-1 (predecessors that far back)
      hub      -- k: reads 1..k delete the last 4j (j = 1..k) bases of a planted stretch ending at the hub node, each joining the hub
                  from another node (in-degree up to k + 1)
      hub_ins  -- k: reads carry distinct short insertions (1-4 bases) at one site (another source of in-degree >= 3)
      long_ins -- insertion lengths, carried by the last reads (clear of the far deletions)
      frag     -- ("prefix" | "suffix" | "interior", fraction): reads 1.. are that fragment of the backbone (gradient < 0.8)
      ext      -- reads 1.. extend past the backbone by ext bases (gradient > 1.1), on "both" sides or the "left" one; the
                  extensions are shared between reads, so only read 1 sees the short graph
      ns       -- N bases per read (reads 1..)"""
    rng = np.random.RandomState(seed)
    stretches = []
    if far or hub:
        slots = list(far) + ([4 * hub + 12] if hub else [])
        span = sum(d + 2 * STRETCH_FLANK + 10 for d in slots)
        assert span < backbone_len, "backbone too short for the planted stretches"
        at = (backbone_len - span) // 2 + STRETCH_FLANK
        for d in slots:
            stretches.append((at, d))
            at += d + 2 * STRETCH_FLANK + 10
    bb = planted_backbone(rng, backbone_len, stretches)
    ins_site = backbone_len // 3
    left = _rand(rng, ext)
    right = _rand(rng, ext if ext_side == "both" else 0)
    reads = [bb]
    for i in range(1, n_reads):
        edits = []  # (start, end, replacement) on backbone coordinates, applied right to left
        if i - 1 < len(far):
            p, d = stretches[i - 1]
            edits.append((p, p + d, ""))
        if hub and i <= hub:
            p, d = stretches[-1]
            edits.append((p + d - 4 * i, p + d, ""))
        if hub_ins and i <= hub_ins:
            edits.append((ins_site, ins_site, _rand(rng, 1 + (i - 1) % 4)))
        if n_reads - 1 - i < len(long_ins):  # the last reads, clear of the far deletions
            q = (2 * backbone_len) // 3
            edits.append((q, q, _rand(rng, long_ins[n_reads - 1 - i])))
        r = bb
        for a, b, rep in sorted(edits, reverse=True):
            r = r[:a] + rep + r[b:]
        if frag is not None:
            kind, f = frag
            n = max(1, int(len(r) * f))
            r = r[:n] if kind == "prefix" else (r[len(r) - n:] if kind == "suffix" else r[(len(r) - n) // 2:(len(r) - n) // 2 + n])
        if ext:
            r = _substitute(rng, left, int(len(left) * subs)) + r + _substitute(rng, right, int(len(right) * subs))
        if subs:
            r = _substitute(rng, r, int(len(r) * subs))
        if ns:
            r = _with_ns(rng, r, ns)
        reads.append(r)
    return tuple(reads)


def flat(windows):
    return ol.flatten_windows([list(w) for w in windows])


# ---------------------------------------------------------------------------------------------------------------------------
# the adaptive band of nw_banded_v3 (widen_band and set_band in poa_common.cuh) and the ring depth of dp_rows_v3
# ---------------------------------------------------------------------------------------------------------------------------


def adaptive_width(read_len, graph_len, band=256):
    """Band width of an adaptive-band alignment before any rerun. The gradient is a float32 division (IEEE here; the device
    uses __fdividef, which agrees at these sizes), compared and scaled in double precision."""
    gradient = float(np.float32(read_len + 1) / np.float32(graph_len + 1))
    max_column = read_len + 1
    if gradient > 1.1:
        band = max(band, (int(max_column * 0.08 * gradient) + 127) & ~127)
    if gradient < 0.8:
        band = max(band, (int(max_column * 0.1 / gradient) + 127) & ~127)
    return min(band, MAX_ADAPTIVE_BW)


def ring_depth(pool_bytes, band, score_bytes):
    return min(pool_bytes // ((band + 8) * score_bytes), 64)


# ---------------------------------------------------------------------------------------------------------------------------
# configs, the oracle (cached per distinct window) and the GPU run
# ---------------------------------------------------------------------------------------------------------------------------


def config(max_seq, max_nodes, band, mode, msd=None, nseq=16, max_pred=0):
    """BatchConfig's explicit constructor; msd defaults to what the band mode needs (2x the band in adaptive mode)."""
    from genomeworks_b200 import cudapoa
    if msd is None:
        msd = band + 8 if "static" in mode else 2 * (band + 8)
    return cudapoa.make_config_explicit(max_seq, 2 * max_seq, max_nodes, band, nseq, msd, mode, max_pred)


def cfg8(cfg):
    return (cfg.max_sequence_size, cfg.max_consensus_size, cfg.max_nodes_per_graph, cfg.matrix_sequence_dimension, cfg.alignment_band_width,
            cfg.max_sequences_per_poa, cfg.band_mode, cfg.max_banded_pred_distance)


@functools.lru_cache(maxsize=None)
def _oracle_one(window, c8, match, msa):
    r = ol.poa_run([list(window)], np.array(c8, dtype=np.int32), msa=msa, match=match)
    return dict(consensus=r["consensus"][0], coverage=r["coverage"][0], status=int(r["status"][0]), cells=int(r["cells"][0]),
                msa=r["msa"][0] if msa else None)


def oracle(windows, cfg, match=8, msa=False):
    return [_oracle_one(w, cfg8(cfg), match, msa) for w in windows]


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


TABLE = []


def run_and_check(name, windows, cfg, mem, kernel, match=8, msa=False, ring=None, widths=None, min_ok=1):
    """Runs windows on the GPU, asserts the kernel (and for v3 the ring depth R at the configured band), and compares every
    window with the oracle. Returns the batch facts for the caller's own assertions."""
    from genomeworks_b200 import cudapoa
    b = cudapoa.CudaPoaBatch(cfg.max_sequences_per_poa, cfg.max_sequence_size, mem, output_type="msa" if msa else "consensus", config=cfg,
                             match_score=match)
    try:
        k, pool, sb, max_poas = b.kernel, b.pool_bytes, b.score_bytes, b.max_poas
        R = ring_depth(pool, cfg.alignment_band_width, sb) if k == KERNELS["v3"] else None
        where = "%s [kernel %s, R %s, pool %d B, max_poas %d, int%d scores]" % (name, cudapoa.KERNEL_NAMES.get(k, k), R, pool, max_poas, 8 * sb)
        assert k == KERNELS[kernel], where + ": expected the %s kernel" % kernel
        if ring is not None:
            assert R == ring, where + ": expected ring depth R = %d" % ring
        rc, added = b.add_poa_groups_flat(*flat(windows))
        assert rc == 0 and added == len(windows), (where, rc, added)
        b.generate_poa()
        if msa:
            rows, st = b.get_msa()
            ours = [dict(status=int(s), msa=[r.decode() for r in w]) for w, s in zip(rows, st)]
        else:
            cons, cov, st = b.get_consensus()
            ours = [dict(status=int(s), consensus=c, coverage=list(v)) for c, v, s in zip(cons, cov, st)]
        cells = b.last_cells()
    finally:
        b.close()
    orc = oracle(windows, cfg, match, msa)
    for w, (x, y) in enumerate(zip(ours, orc)):
        wn = "%s, window %d" % (where, w)
        assert x["status"] == y["status"], wn + ": status %d, oracle %d" % (x["status"], y["status"])
        if msa:
            assert x["msa"] == (y["msa"] if y["status"] == 0 else []), wn + ": MSA differs"
        else:
            assert x["consensus"] == y["consensus"], wn + ": consensus differs"
            assert x["coverage"] == [int(v) for v in y["coverage"]], wn + ": coverage differs"
    assert cells == sum(y["cells"] for y in orc), where + ": executed DP cells differ (a band width or a rerun differs)"
    ok = sum(1 for y in orc if y["status"] == 0)
    assert ok >= min_ok, where + ": only %d windows succeed in the oracle" % ok
    if widths is not None and k == KERNELS["v3"]:
        R = "/".join(str(ring_depth(pool, w, sb)) for w in widths)  # the adaptive alignments run at the R of their own band
    TABLE.append((name, cudapoa.KERNEL_NAMES.get(k, k), R, 8 * sb, widths if widths is not None else cfg.alignment_band_width))
    print("PATH | %-34s | %-2s | R %-4s | int%d | band %s" % TABLE[-1])
    return dict(kernel=k, R=R, pool=pool, score_bytes=sb, statuses=[x["status"] for x in ours])


def mem_for_max_poas(cfg, target, match=8, probe_mem=2 << 30):
    """Device memory that sizes a batch of cfg for `target` windows: capacity is linear in memory, so it is scaled from a probe."""
    from genomeworks_b200 import cudapoa
    b = cudapoa.CudaPoaBatch(cfg.max_sequences_per_poa, cfg.max_sequence_size, probe_mem, config=cfg, match_score=match)
    p0 = b.max_poas
    b.close()
    assert p0 > 8, "probe batch too small"
    return int(probe_mem * target / p0)


def tiled(windows, n):
    return [windows[i % len(windows)] for i in range(n)]


# ---------------------------------------------------------------------------------------------------------------------------
# inputs of the cases
# ---------------------------------------------------------------------------------------------------------------------------


def far_hub_windows(seed, backbone_len, n=6, n_reads=8):
    """Windows with predecessors 70-400 rows back and hubs of in-degree up to 13, plus plain ones."""
    out = []
    for i in range(n):
        kind = i % 3
        if kind == 0:
            hub = min(12, n_reads - 1)
            dels, span = [], 4 * hub + 12 + 2 * STRETCH_FLANK + 10
            for d in (70, 130, 250, 400):
                if len(dels) < 3 and span + d + 2 * STRETCH_FLANK + 10 < backbone_len:
                    dels.append(d)
                    span += d + 2 * STRETCH_FLANK + 10
            out.append(build_window(seed + i, backbone_len, n_reads, far=tuple(dels), hub=hub))
        elif kind == 1:
            out.append(build_window(seed + i, backbone_len, n_reads, far=(min(90, backbone_len // 5),), hub_ins=n_reads - 1, long_ins=(40, 80)))
        else:
            out.append(build_window(seed + i, backbone_len, n_reads, subs=0.03))
    return out


# (target width of read 1, backbone length, read-1 length): reads extend the backbone (gradient > 1.1) or are fragments of it
# (gradient < 0.8, width 0.1 x backbone). adaptive_width gives the widths; test_builders_reach_adaptive_widths checks them.
EXT_WIDTHS = [(640, 1200, 3000), (768, 1028, 3000), (896, 867, 3000), (1024, 750, 3000), (1152, 654, 3000), (1280, 585, 3000),
              (1408, 533, 3000), (1536, 479, 3000)]
FRAG_WIDTHS = [(640, 6000, None), (768, 7000, None)]


def ext_window(seed, target, bb, rl, n_reads=4, side="both"):
    return build_window(seed, bb, n_reads, ext=(rl - bb) // (2 if side == "both" else 1), ext_side=side, subs=0.01)


def adaptive_windows(seed):
    ws = [ext_window(seed + i, t, bb, rl) for i, (t, bb, rl) in enumerate(EXT_WIDTHS)]
    ws += [build_window(seed + 20 + i, bb, 4, frag=("interior", 0.5)) for i, (t, bb, _) in enumerate(FRAG_WIDTHS)]
    ws += [build_window(seed + 30, 3500, 4, frag=("prefix", 0.5)), build_window(seed + 31, 3500, 4, frag=("suffix", 0.5))]
    ws += threshold_windows() + rerun_windows()
    ws += [build_window(seed + 40, 900, 6)]  # neighbour with the configured band only
    return ws


def threshold_windows():
    """Read 1 on either side of the widening thresholds, long enough that widening changes the band: gradient 1.138 (384),
    1.097 (256), 0.78 (384) and 0.81 (256). A threshold moved by a few hundredths changes the band of one of them."""
    return [build_window(950, 2900, 4, ext=200), build_window(951, 3000, 4, ext=145), build_window(952, 3400, 4, frag=("interior", 0.78)),
            build_window(953, 3400, 4, frag=("interior", 0.81))]


def rerun_windows():
    """Read 1 reruns from a 512 band (doubled to 1024), from 768 (doubled to the 1536 cap) and from 1408 (shifted, not widened).
    The last window starts at 1536 and drifts out of its band, but a band of 1536 never asks for a rerun (the band check of the
    traceback is off at the cap), so it runs once."""
    return [ext_window(906, 512, 1500, 3000), ext_window(907, 768, 1028, 3000), build_window(909, 520, 4, ext=2480, ext_side="left", subs=0.0),
            build_window(910, 480, 4, ext=2520, ext_side="left", subs=0.0)]


# ---------------------------------------------------------------------------------------------------------------------------
# CPU: the builders produce what the GPU cases rely on
# ---------------------------------------------------------------------------------------------------------------------------


def test_adaptive_width_formula_edges():
    assert adaptive_width(999, 999) == 256  # gradient 1
    assert adaptive_width(8000, 4000) == 1280
    assert adaptive_width(3000, 6000) == 640
    assert adaptive_width(20000, 1000) == MAX_ADAPTIVE_BW
    # gradient just above / below the thresholds
    assert adaptive_width(3301, 3000) == 384 and adaptive_width(3300, 3000) == 256
    assert adaptive_width(2998, 3749) == 384 and adaptive_width(2999, 3749) == 256


@pytest.mark.parametrize("target,bb,rl", EXT_WIDTHS + FRAG_WIDTHS)
def test_builders_reach_adaptive_widths(target, bb, rl):
    w = ext_window(1, target, bb, rl) if rl is not None else build_window(1, bb, 2, frag=("interior", 0.5))
    assert len(w[0]) == bb
    assert adaptive_width(len(w[1]), len(w[0])) == target


def test_builders_rerun_widened_bands():
    """Read 1 of each rerun window, in the oracle: the executed cells over the backbone length give the band of the first pass
    plus that of the rerun."""
    cfg = (16384, 32768, 16384, 3088, 256, 16, 2, 0)
    seen = []
    for w in rerun_windows():
        r = ol.poa_run([list(w[:2])], np.array(cfg, dtype=np.int32))
        assert int(r["status"][0]) == 0 and int(r["cells"][0]) % len(w[0]) == 0
        w0 = adaptive_width(len(w[1]), len(w[0]))
        seen.append((w0, int(r["cells"][0]) // len(w[0]) - w0))
    assert seen == [(512, 1024), (768, 1536), (1408, 1408), (1536, 0)]


def test_builders_straddle_widening_thresholds():
    gradients, widths = [], []
    for w in threshold_windows():
        gradients.append(float(np.float32(len(w[1]) + 1) / np.float32(len(w[0]) + 1)))
        widths.append(adaptive_width(len(w[1]), len(w[0])))
    assert 1.1 < gradients[0] < 1.15 and 1.05 < gradients[1] < 1.1, gradients
    assert 0.75 < gradients[2] < 0.8 and 0.8 < gradients[3] < 0.85, gradients
    assert widths == [384, 256, 384, 256]
    # the oracle runs read 1 at those widths (plus a doubled rerun where the path leaves the band)
    cfg = np.array((4000, 8000, 4096, 3088, 256, 16, 2, 0), dtype=np.int32)
    for w, width in zip(threshold_windows(), widths):
        r = ol.poa_run([list(w[:2])], cfg)
        assert int(r["status"][0]) == 0 and int(r["cells"][0]) in (len(w[0]) * width, 3 * len(w[0]) * width)


def test_builders_reach_far_predecessors_and_hubs():
    """Predecessors at least 64 rows back (beyond the ring at every R) and in-degrees of 3 or more, in the graphs the DP rows
    run over."""
    for bb in (700, 1400, 2400):
        ws = far_hub_windows(7, bb, n=3)
        st = ol.poa_row_stats([list(w) for w in ws], np.array((3072, 6144, 4096, 1544, 1536, 16, 1, 0), dtype=np.int32))
        assert st[0, 0] >= (250 if bb > 1000 else 64) and st[0, 2] >= 3, (bb, st)  # far deletions
        assert st[0, 1] >= 4 and st[0, 3] >= 3, (bb, st)                           # deletion hub
        assert st[1, 0] >= 64 and st[1, 1] >= 3, (bb, st)                          # insertion hub + one far deletion


def edge_limit_window():
    """55 reads that each drop a different number of bases after one node: that node gets a 51st out-edge."""
    rng = np.random.RandomState(51)
    K, h = 60, 150
    bb = _rand(rng, h - K - 30) + _rand(rng, 30, "GT") + _rand(rng, K, "AC") + _rand(rng, 30, "GT") + _rand(rng, 100)
    return tuple([bb] + [bb[:h - K] + bb[h - K + j:] for j in range(1, 56)])


def wide_hub_window():
    """A hub of 37 predecessors, inside the 50-edge limit: 60 reads join it from different nodes of a planted stretch, 40 more
    through insertions. (Reads that do this converge on shared nodes; 51 distinct in-edges are not reached this way.)"""
    rng = np.random.RandomState(3)
    K, h = 240, 330
    bb = _rand(rng, h - K - 40) + _rand(rng, 40, "GT") + _rand(rng, K, "AC") + _rand(rng, 40, "GT") + _rand(rng, 200)
    return tuple([bb] + [bb[:h - 4 * j] + bb[h:] for j in range(1, 61)] + [bb[:h] + _rand(rng, 1 + j % 4) + bb[h:] for j in range(40)])


def test_builders_edge_and_node_limits():
    st = ol.poa_row_stats([list(wide_hub_window())], np.array((1024, 2048, 4096, 264, 256, 128, 1, 0), dtype=np.int32))
    assert 30 <= st[0, 1] <= 50, st
    cfg = np.array((1024, 2048, 2048, 264, 256, 64, 1, 0), dtype=np.int32)
    r = ol.poa_run([list(edge_limit_window())], cfg)
    assert int(r["status"][0]) == 5  # edge_count_exceeded_maximum_graph_size
    r = ol.poa_run([list(node_limit_window())], np.array((1024, 2048, 1100, 264, 256, 16, 1, 0), dtype=np.int32))
    assert int(r["status"][0]) == 4  # node_count_exceeded_maximum_graph_size
    r = ol.poa_run([list(node_limit_window(1400, 200))], np.array((1664, 3328, 1664, 1672, 1664, 16, 1, 0), dtype=np.int32))
    assert int(r["status"][0]) == 4


def node_limit_window(backbone=800, insertion=100):
    """Reads (at most backbone + insertion bases) with long insertions: the graph passes 1100 nodes (1664 with a backbone of 1400
    and insertions of 200) after a few reads."""
    return build_window(44, backbone, 10, long_ins=(insertion,) * 9, subs=0.05)


# ---------------------------------------------------------------------------------------------------------------------------
# GPU cases
# ---------------------------------------------------------------------------------------------------------------------------

STATIC_BANDS = [640, 768, 1024, 1280, 1408, 1536]


@pytest.mark.gpu
@pytest.mark.parametrize("score", [16, 32])
@pytest.mark.parametrize("band", STATIC_BANDS)
def test_v3_static_band_sweep(band, score, device_fdiv):
    """Bands of 3-6 chunks per row on v3, int16 and int32 rows, with reads narrower than the band (band start stays 0) and wider
    (the band moves), far predecessors and hubs."""
    match = 8 if score == 16 else 40  # 40: max_sequence_size x match > INT16_MAX -> int32 scores
    cfg = config(3072, 4096, band, "static_band")
    ws = far_hub_windows(100 + band, int(0.6 * band), n=3, n_reads=6) + far_hub_windows(200 + band, int(1.6 * band), n=3, n_reads=6)
    f = run_and_check("static %d int%d" % (band, score), ws, cfg, 4 << 30, "v3", match=match)
    assert f["score_bytes"] * 8 == score


@pytest.mark.gpu
def test_v3_static_band_1536_msa(device_fdiv):
    cfg = config(3072, 4096, 1536, "static_band")
    ws = far_hub_windows(31, 900, n=2, n_reads=6) + far_hub_windows(32, 2400, n=2, n_reads=6)
    run_and_check("static 1536 MSA", ws, cfg, 4 << 30, "v3", msa=True)


# (name, band, score bits, CTAs per SM the batch capacity gives, R that gives on an H100: 228 KB of shared memory per SM)
RING_CASES = [("R2 int32 1536", 1536, 32, 12, 2), ("R3 int32 1536", 1536, 32, 10, 3), ("R3 int16 1536", 1536, 16, 16, 3),
              ("R4 int32 1024", 1024, 32, 12, 4), ("R4 int16 1536", 1536, 16, 15, 4), ("R5 int16 1536", 1536, 16, 13, 5),
              ("R6 int16 1536", 1536, 16, 11, 6), ("R7 int16 1536", 1536, 16, 9, 7), ("R8 int16 1536", 1536, 16, 8, 8),
              ("R64 int16 640", 640, 16, 2, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,band,score,ctas,R", RING_CASES, ids=[c[0].replace(" ", "-") for c in RING_CASES])
def test_v3_ring_depth_sweep(name, band, score, ctas, R, device_fdiv):
    """Far predecessors and hubs at each ring depth: the row records pick the ring slot of fast rows and send every row with
    a predecessor R or more rows back through the bulk-copy wait and global memory. Batch capacity sets the CTAs per SM and so
    the pool per CTA; two windows per SM keep every SM busy."""
    match = 8 if score == 16 else 40
    cfg = config(max(band, 1024), max(band, 1024), band, "static_band", nseq=10)
    sms = _sms()
    mem = mem_for_max_poas(cfg, int((ctas - 0.5) * sms), match=match)
    assert mem <= 24 << 30
    distinct = far_hub_windows(300 + band, min(900, band // 2 + 300), n=6, n_reads=8)
    run_and_check(name, tiled(distinct, min(2 * sms, int((ctas - 0.5) * sms) - 8)), cfg, mem, "v3", match=match, ring=R)


@pytest.mark.gpu
@pytest.mark.parametrize("score", [16, 32])
def test_v3_adaptive_widening(score, device_fdiv):
    """Read 1 widened to every band from 640 to 1536, reruns from 512 and 768, a shifted rerun at 1408, next to a window that keeps
    the configured band. The cells pin every band width."""
    match = 8 if score == 16 else 40
    ws = adaptive_windows(500)
    cfg = config(7200 if score == 32 else 4000, 8192 if score == 32 else 4096, 256, "adaptive_band", msd=2 * 1544)
    if score == 16:
        ws = [w for w in ws if max(len(r) for r in w) <= 4000 and len(w[0]) < 4000]
    widths = sorted({adaptive_width(len(w[1]), len(w[0])) for w in ws if len(w) > 1})
    run_and_check("adaptive int%d" % score, ws, cfg, 8 << 30, "v3", match=match, widths=widths)


@pytest.mark.gpu
def test_v3_adaptive_widening_msa(device_fdiv):
    ws = [ext_window(600 + i, t, bb, rl) for i, (t, bb, rl) in enumerate(EXT_WIDTHS[::3])]
    cfg = config(4000, 4096, 256, "adaptive_band", msd=2 * 264)
    run_and_check("adaptive MSA", ws, cfg, 8 << 30, "v3", msa=True, widths=sorted({t for t, _, _ in EXT_WIDTHS[::3]}))


@pytest.mark.gpu
def test_v3_adaptive_widening_exceeds_matrix(device_fdiv):
    """A matrix sized for the configured band: a widened read 1 gives exceeded_adaptive_banded_matrix_size, windows that keep
    the configured band succeed."""
    from genomeworks_b200 import cudapoa
    ws = [build_window(70, 900, 5), ext_window(71, 640, 1200, 3000), build_window(72, 1000, 5), ext_window(73, 1024, 750, 3000),
          build_window(74, 600, 5)]
    cfg = config(4000, 4096, 256, "adaptive_band", msd=128)
    f = run_and_check("adaptive, small matrix", ws, cfg, 2 << 30, "v3", widths=[256, 640, 1024])
    assert f["statuses"] == [0, cudapoa.exceeded_adaptive_banded_matrix_size, 0, cudapoa.exceeded_adaptive_banded_matrix_size, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("score", [16, 32])
def test_kernel_selection_band_1536_vs_1664(score, device_fdiv):
    match = 8 if score == 16 else 40
    ws = far_hub_windows(800, 1100, n=3, n_reads=6)
    run_and_check("static 1536 int%d (selection)" % score, ws, config(2048, 4096, 1536, "static_band"), 4 << 30, "v3", match=match)
    run_and_check("static 1664 int%d (selection)" % score, ws, config(2048, 4096, 1664, "static_band"), 4 << 30, "v1", match=match)
    run_and_check("static 1664 int%d MSA (selection)" % score, ws, config(2048, 4096, 1664, "static_band"), 4 << 30, "v1", match=match, msa=True)


@pytest.mark.gpu
def test_kernel_selection_adaptive_band_2048_runs_static(device_fdiv):
    """An adaptive band above the widest adaptive band is not widened: the first-generation kernel runs it as a static band."""
    ws = far_hub_windows(810, 1100, n=2, n_reads=5) + [ext_window(811, 1024, 750, 3000)]
    run_and_check("adaptive 2048 (selection)", ws, config(4000, 4096, 2048, "adaptive_band", msd=2 * 2056), 4 << 30, "v1")


@pytest.mark.gpu
@pytest.mark.parametrize("max_seq,kernel", [(65535, "v3"), (65536, "v1")])
def test_kernel_selection_max_sequence_size_65535(max_seq, kernel, device_fdiv):
    """Reads of 60-65 kb: v3 packs band starts in 16 bits, so near 0xFFFF at max_sequence_size 65 535 (int32 sizes); 65 536
    selects the first-generation kernel."""
    ws = [build_window(820, 64000, 3, subs=0.002), build_window(821, 60000, 3, subs=0.002, far=(300,))]
    rng = np.random.RandomState(822)
    full = _rand(rng, 65535)
    ws.append((full, _substitute(rng, full, 100), _substitute(rng, full, 100)))
    run_and_check("max_seq %d (selection)" % max_seq, ws, config(max_seq, 66560, 256, "static_band", nseq=4), 8 << 30, kernel)


@pytest.mark.gpu
@pytest.mark.parametrize("score", [16, 32])
@pytest.mark.parametrize("mode", ["static_band_traceback", "adaptive_band_traceback"])
@pytest.mark.parametrize("band", [768, 1536])
def test_traceback_kernel_wide_bands(band, mode, score, device_fdiv):
    match = 8 if score == 16 else 40
    ws = far_hub_windows(830 + band, 1200, n=3, n_reads=6)
    if mode == "adaptive_band_traceback":
        ws.append(ext_window(831, 1024, 750, 3000))
    cfg = config(3072, 4096, band, mode, max_pred=2 * band)
    run_and_check("%s %d int%d" % (mode, band, score), ws, cfg, 8 << 30, "tb", match=match)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["v3", "tb", "v1"])
@pytest.mark.parametrize("mode", ["static_band", "adaptive_band"])
@pytest.mark.parametrize("score", [16, 32])
def test_shape_and_status_edges(kernel, mode, score, device_fdiv):
    """Windows of one read, reads of 1-5 and 31-33 bases and of exactly max_sequence_size, backbones of 31/32/33/64/65 bases
    (either side of v3's 32-row record groups), N bases, a 51st edge and a graph that outgrows max_nodes, each between ordinary
    windows of the same batch, on each kernel: tb runs the traceback counterpart of the band mode, v1 a band of 1664 (which
    needs reads and graphs of 1664)."""
    from genomeworks_b200 import cudapoa
    match = 8 if score == 16 else 40
    max_seq, max_nodes, band = (1664, 1664, 1664) if kernel == "v1" else (1024, 1100, 256)
    rng = np.random.RandomState(900)
    plain = [build_window(910 + i, 500 + 37 * i, 5) for i in range(12)]
    edges = [(_rand(rng, 300),)]  # one read
    for n in (1, 2, 3, 4, 5, 31, 32, 33):
        bb = _rand(rng, max(n, 40))
        edges.append((bb,) + tuple(_substitute(rng, bb[:n], 1 if n > 2 else 0) for _ in range(3)))  # short reads, long backbone
        edges.append(tuple([_rand(rng, n)] + [_substitute(rng, _rand(rng, n), 0) for _ in range(3)]))  # all reads short
    for n in (31, 32, 33, 64, 65):
        edges.append(build_window(930 + n, n, 6, subs=0.05))
    edges.append(build_window(940, max_seq, 4, subs=0.01))  # reads of exactly max_sequence_size (backbone) ...
    edges[-1] = tuple(r[:max_seq] if len(r) > max_seq else r + "A" * (max_seq - len(r)) for r in edges[-1])
    edges.append(build_window(941, 700, 6, ns=12))
    edges.append(build_window(942, 300, 6, ns=300, subs=0.0))
    edges.append(edge_limit_window())
    edges.append(wide_hub_window())
    edges.append(node_limit_window(1400, 200) if kernel == "v1" else node_limit_window())
    ws = []
    for i, e in enumerate(edges):
        ws += [e, plain[i % len(plain)]]
    cfg = config(max_seq, max_nodes, band, mode + ("_traceback" if kernel == "tb" else ""), nseq=128, max_pred=2 * band)
    f = run_and_check("edges %s %s int%d" % (kernel, mode, score), ws, cfg, 8 << 30, kernel, match=match)
    st = f["statuses"]
    assert cudapoa.edge_count_exceeded_maximum_graph_size in st and cudapoa.node_count_exceeded_maximum_graph_size in st
    assert all(s == 0 for s in st[1::2]), "a neighbouring window failed"
