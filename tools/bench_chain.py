"""SSP chainer benchmark (DESIGN.md section 19): one JSON line per size.

    python tools/bench_chain.py [--sizes 10000,100000,1000000] [--steps K] [--warmup W] [--oracle-max 20000]
                                [--min-chain-score 30000]

Each set is a colinear backbone of n / 10 SSPs with jittered gaps and diagonals over 10^8 positions, plus n - n / 10 random
off-chain SSPs over the same span, shuffled (chain_libs.backbone_set, seed 2026). Zero penalties, as LASTZ's bare --chain.
Each line: the device ms of one chain call (CUDA events around it, mean of `steps` calls after `warmup`), the pair tests the
external kernel makes (n(n-1)/2 minus the in-tile pairs) and their rate, the sequential in-tile steps (n), the chain's length
and score, and, for n <= --oracle-max, whether f, p, the chain and the score equal the CPU oracle's. The card name and power
limit are read in the same run. Writes nothing to the tree.

Each line also times chain_all (every chain scoring >= --min-chain-score, DESIGN.md section 20) on the same set, the two calls
alternating in one process: its device ms, the ms it adds to chain (the extraction after the same DP), the number of candidate
chains (at the lowest minimum) and of reported chains, and whether its first chain is chain's.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

TILE = 1024  # chain_kernels.cuh kTile


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10000,100000,1000000")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--oracle-max", type=int, default=20000)
    ap.add_argument("--min-chain-score", type=int, default=30000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_chain.py needs a CUDA device")
    import chain_libs as cl
    from genomeworks_b200 import cudaextender as ce
    gpu, power = card()
    c = ce.create_ssp_chainer()
    for n in (int(x) for x in a.sizes.split(",")):
        ssps = cl.backbone_set(np.random.default_rng(2026), n, n // 10)
        dev = torch.from_numpy(ssps.view(np.int32).reshape(-1, 4).copy()).cuda()
        torch.cuda.synchronize()
        for _ in range(a.warmup):
            c.chain(dev)
            c.chain_all(dev, min_score=a.min_chain_score)
        ms = ms_all = 0.0
        for _ in range(a.steps):
            idx, score = c.chain(dev)
            ms += c.last_ms() / a.steps
            scores, offsets, members = c.chain_all(dev, min_score=a.min_chain_score)
            ms_all += c.last_ms() / a.steps
        candidates = len(c.chain_all(dev)[0])
        in_tile = sum(m * (m - 1) // 2 for m in [TILE] * (n // TILE) + [n % TILE])
        pairs = n * (n - 1) // 2 - in_tile
        line = dict(n=n, backbone=n // 10, chain_ms=round(ms, 3), external_pair_tests=pairs,
                    pair_tests_per_s=pairs / (ms / 1e3) if ms > 0 else None, in_tile_steps=n, chain_length=int(len(idx)), score=int(score),
                    all_chains_ms=round(ms_all, 3), extract_added_ms=round(ms_all - ms, 3), min_chain_score=a.min_chain_score,
                    candidate_chains=candidates, reported_chains=int(len(scores)), union=int(len(members)),
                    first_chain_is_best=bool(len(scores) > 0 and np.array_equal(members[offsets[0]:offsets[1]], idx) and scores[0] == score),
                    steps=a.steps, warmup=a.warmup, card=gpu, power_limit=power)
        if n <= a.oracle_max:
            f, p = c.get_dp()
            want = cl.oracle_run(ssps)
            line["equals_oracle"] = bool(np.array_equal(f, want["f"]) and np.array_equal(p, want["p"]) and
                                         np.array_equal(idx, cl.chain_indices(want)) and score == want["score"])
        print(json.dumps(line), flush=True)
    c.close()


if __name__ == "__main__":
    main()
