"""Genome aligner benchmark: one JSON line per workload, with the aligner's defaults (both strands, transitions, the sample
matrix, LASTZ-style gapped parameters, blocks of 2^25 seeds).

    python tools/bench_genome_aligner.py [--steps K] [--warmup W] [--workloads sample,assembly,contigs,repeats]
                                         [--modes default,skip,chain,chain+skip,chains,chains+skip] [--skip-covered]
                                         [--min-chain-score 30000] [--group-bases N] [--contigs 2000]
                                         [--seed 12of19] [--max-word-count N] [--repeat-copies 300]

Workloads:
  sample    the golden sample (one 250 kb record) against itself;
  assembly  a 10 Mb random target against a query assembled from 5-50 kb pieces of it, each diverged by 2-10 % (80 %
            substitutions, 10 % each 1-3 base insertions and deletions), about a third of them reverse-complemented, in a
            shuffled order. Every homologous gapped side ends within its piece.
  contigs   the assembly workload's target cut at random points into --contigs records (a draft assembly). First against
            the 80 pieces as separate query records, run grouped (--group-bases) and with every record on its own
            (group_bases=1), alternating in one process, with identical outputs asserted; then grouped alone against the
            query cut into --contigs records as well. The per-record run pays an index build per target record and the
            launches and host synchronisations of every (target record, query record, strand), which is what grouping
            (DESIGN.md section 21) removes; that is why this workload is many short records on both sides.
  repeats   a repeat-rich pair that is not soft-masked: a 2 Mb random target and a 1 Mb random query, each carrying
            --repeat-copies copies of one 300 bp element, every copy 5 % diverged from it. The seeds of the element grow with
            the product of the copy counts, which is what the word cap (--max-word-count, DESIGN.md section 22) bounds.

--seed (12of19, 14of22, match<N> or a 0/1 pattern) and --max-word-count (0 = no cap) set the seeding stage of every run
(DESIGN.md section 22); every line reports them.

Each line: the per-stage device ms of the last run (CUDA events summed over pairs and strands: index, count, write, ungapped,
gapped pass 1 and pass 2), the seeds, unique segments and alignments, seeds/s of the seeding stage (count + write) and of the
write pass alone with its bytes/s (8 bytes written per seed), and the wall time of a whole run (host clock, mean of `steps` runs
after `warmup`). The card name and power limit are read in the same run. Writes nothing to the tree. Every line reports
the group size and the aligner's group stats (target groups, query groups, record pairs and strands given to the gapped
stage).

--modes default,skip runs each workload in both modes in the same process, the runs alternating between them, and prints one
line per mode; skip is the skip-covered mode (DESIGN.md section 18). A skip line adds the skip stats of the gapped stage and
whether every skip-mode alignment's score, records, strand and intervals are among the default mode's (subset_of_default,
when both modes ran). --skip-covered is --modes skip. chain is chaining with zero penalties (DESIGN.md section 19) and
chain+skip chaining in skip-covered mode; their lines add the chain stats (SSPs in, SSPs chained, pairs, chain ms). chains is
every chain scoring >= --min-chain-score (DESIGN.md section 20; default 30,000, ten times the SSP threshold) and chains+skip
that in skip-covered mode; their lines add the chain stats and the number of chains. On the assembly workload every line
reports pieces_found: the pieces that one alignment on their strand overlaps for at least half of their length in both
sequences, and the pieces it misses.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def assembly(seed=2026, target_len=10_000_000, pieces=80):
    """([target], [query], counts, placements): each placement is (query begin, query end, target begin, target end, strand)
    of one piece, strand 1 for a reverse-complemented piece."""
    import seeder_libs as sl
    rng = np.random.default_rng(seed)
    target = rng.integers(0, 4, target_len).astype(np.int8)
    parts, rc, placed, at = [], 0, [], 0
    for _ in range(pieces):
        n = int(rng.integers(5000, 50001))
        s = int(rng.integers(0, target_len - n))
        piece = sl.mutate(target[s:s + n], float(rng.uniform(0.02, 0.10)), rng)
        strand = 0
        if rng.random() < 1 / 3:
            piece = sl.reverse_complement(piece)
            rc += 1
            strand = 1
        parts.append(piece)
        placed.append((at, at + len(piece), s, s + n, strand))
        at += len(piece)
    return [target], [np.concatenate(parts)], dict(pieces=pieces, reverse_complemented=rc), placed


def pieces_found(rec, placed):
    """Indices of the pieces that one alignment on their strand overlaps for at least half of their length in both sequences."""
    found = []
    for k, (qb, qe, tb, te, strand) in enumerate(placed):
        mine = rec[rec["strand"] == strand]
        oq = np.minimum(mine["query_end"].astype(np.int64), qe) - np.maximum(mine["query_begin"].astype(np.int64), qb)
        ot = np.minimum(mine["target_end"].astype(np.int64), te) - np.maximum(mine["target_begin"].astype(np.int64), tb)
        if ((2 * oq >= qe - qb) & (2 * ot >= te - tb)).any():
            found.append(k)
    return found


def key(r):
    return tuple(int(r[f]) for f in ("score", "target_record", "query_record", "strand", "query_begin", "query_end", "target_begin",
                                     "target_end"))


def cut(seq, n, rng):
    """seq cut at n - 1 distinct random points into n records."""
    points = np.sort(rng.choice(np.arange(1, len(seq)), n - 1, replace=False))
    return [seq[a:b] for a, b in zip(np.r_[0, points], np.r_[points, len(seq)])]


def repeats(copies, seed=2027, element=300, divergence=0.05):
    """([target], [query], counts): 2 Mb and 1 Mb of random codes with `copies` diverged copies of one element inserted into
    each at random points."""
    import seeder_libs as sl
    rng = np.random.default_rng(seed)
    unit = rng.integers(0, 4, element).astype(np.int8)

    def carrier(n):
        base = rng.integers(0, 4, n).astype(np.int8)
        points = np.sort(rng.choice(np.arange(1, n), copies, replace=False))
        parts = [base[a:b] for a, b in zip(np.r_[0, points], np.r_[points, n])]
        out = [parts[0]]
        for p in parts[1:]:
            out += [sl.mutate(unit, divergence, rng), p]
        return np.concatenate(out)
    return [carrier(2_000_000)], [carrier(1_000_000)], dict(repeat_copies=copies, element=element, divergence=divergence)


def run_group_sizes(name, targets, queries, steps, warmup, extra, sizes, seed="12of19", max_word_count=0):
    """Default mode at each group size in `sizes`, the runs alternating; asserts that every size gives the first's output."""
    from genomeworks_b200 import cudaextender as ce
    aligners = {g: ce.GenomeAligner(group_bases=g, seed=seed, max_word_count=max_word_count) for g in sizes}
    for _ in range(warmup):
        for al in aligners.values():
            al.run(targets, queries)
    wall = dict.fromkeys(sizes, 0.0)
    out = {}
    for _ in range(steps):
        for g, al in aligners.items():
            t0 = time.perf_counter()
            out[g] = al.run(targets, queries)
            wall[g] += (time.perf_counter() - t0) / steps
    first = out[sizes[0]]
    for g, al in aligners.items():
        same = bool(np.array_equal(out[g][0], first[0]) and out[g][1] == first[1])
        assert same, "group_bases %d changed the output" % g
        ms, counts = al.last_stats()
        more = dict(extra, mode="default", group_bases=g, seed=seed, max_word_count=max_word_count, group_stats=al.last_group_stats(),
                    target_records=len(targets),
                    query_records=len(queries), same_output_as_group_bases=sizes[0] if len(sizes) > 1 else None)
        al.close()
        line(name, targets, queries, steps, warmup, out[g][0], wall[g], ms, counts, more)


def run(name, targets, queries, steps, warmup, extra, modes=("default",), min_chain_score=30000, placed=None, group_bases=1 << 28,
        seed="12of19", max_word_count=0):
    from genomeworks_b200 import cudaextender as ce
    aligners = {m: ce.GenomeAligner(skip_covered=m.endswith("skip"), chain=m.startswith("chain"),
                                    min_chain_score=min_chain_score if m.startswith("chains") else None, group_bases=group_bases,
                                    seed=seed, max_word_count=max_word_count)
                for m in modes}
    for _ in range(warmup):
        for al in aligners.values():
            al.run(targets, queries)
    wall = dict.fromkeys(modes, 0.0)
    out = {}
    for _ in range(steps):
        for m, al in aligners.items():
            t0 = time.perf_counter()
            out[m] = al.run(targets, queries)[0]
            wall[m] += (time.perf_counter() - t0) / steps
    for m, al in aligners.items():
        ms, counts = al.last_stats()
        more = dict(extra, mode=m, group_bases=group_bases, seed=seed, max_word_count=max_word_count, group_stats=al.last_group_stats())
        if m.startswith("chain"):
            more["chain_stats"] = al.last_chain_stats()
            more["chains"] = al.last_chain_count()
        if m.startswith("chains"):
            more["min_chain_score"] = min_chain_score
        if placed is not None:
            found = pieces_found(out[m], placed)
            more["pieces_found"] = len(found)
            more["pieces_missed"] = [k for k in range(len(placed)) if k not in found]
        if m == "skip":
            more["skip_stats"] = al.last_skip_stats()
            if "default" in out:
                default = {key(r) for r in out["default"]}
                more["subset_of_default"] = all(key(r) in default for r in out["skip"])
        al.close()
        line(name, targets, queries, steps, warmup, out[m], wall[m], ms, counts, more)


def line(name, targets, queries, steps, warmup, rec, wall, ms, counts, extra):
    gpu, power = card()
    seeding = ms["count"] + ms["write"]
    line = dict(workload=name, target_bases=int(sum(len(t) for t in targets)), query_bases=int(sum(len(q) for q in queries)),
                stage_ms={k: round(v, 3) for k, v in ms.items()}, **counts,
                seeds_per_s_seeding=counts["seeds"] / (seeding / 1e3) if seeding > 0 else None,
                seeds_per_s_write=counts["seeds"] / (ms["write"] / 1e3) if ms["write"] > 0 else None,
                write_bytes_per_s=8 * counts["seeds"] / (ms["write"] / 1e3) if ms["write"] > 0 else None,
                wall_s=round(wall, 4), steps=steps, warmup=warmup, minus_strand_alignments=int((rec["strand"] == 1).sum()),
                card=gpu, power_limit=power, **extra)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="sample,assembly")
    ap.add_argument("--modes", default="default")
    ap.add_argument("--skip-covered", action="store_true")
    ap.add_argument("--min-chain-score", type=int, default=30000)
    ap.add_argument("--group-bases", type=int, default=1 << 28)
    ap.add_argument("--contigs", type=int, default=2000)
    ap.add_argument("--seed", default="12of19")
    ap.add_argument("--max-word-count", type=int, default=0)
    ap.add_argument("--repeat-copies", type=int, default=300)
    a = ap.parse_args()
    modes = ["skip"] if a.skip_covered else a.modes.split(",")
    if set(modes) - {"default", "skip", "chain", "chain+skip", "chains", "chains+skip"}:
        sys.exit("modes are default, skip, chain, chain+skip, chains and chains+skip")
    from genomeworks_b200 import cudaextender as ce
    ce._seed_args(a.seed, a.max_word_count)
    seeding = dict(seed=a.seed, max_word_count=a.max_word_count)
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_genome_aligner.py needs a CUDA device")
    for w in a.workloads.split(","):
        if w == "sample":
            import extender_libs as xl
            seq, _, _ = xl.sample()
            run("sample", [seq], [seq], a.steps, a.warmup, {}, modes, a.min_chain_score, group_bases=a.group_bases, **seeding)
        elif w == "assembly":
            t, q, extra, placed = assembly()
            run("assembly", t, q, a.steps, a.warmup, extra, modes, a.min_chain_score, placed, a.group_bases, **seeding)
        elif w == "contigs":
            t, q, extra, placed = assembly()
            rng = np.random.default_rng(7)
            targets = cut(t[0], a.contigs, rng)
            pieces = [q[0][qb:qe] for qb, qe, _, _, _ in placed]
            run_group_sizes("contigs_x_pieces", targets, pieces, a.steps, a.warmup, extra, [a.group_bases, 1], **seeding)
            run_group_sizes("contigs_x_contigs", targets, cut(q[0], a.contigs, rng), a.steps, a.warmup, extra, [a.group_bases], **seeding)
        elif w == "repeats":
            t, q, extra = repeats(a.repeat_copies)
            run("repeats", t, q, a.steps, a.warmup, extra, modes, a.min_chain_score, group_bases=a.group_bases, **seeding)
        else:
            sys.exit("unknown workload " + w)


if __name__ == "__main__":
    main()
