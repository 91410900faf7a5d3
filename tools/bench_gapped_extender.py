"""Gapped-extender benchmark: one JSON line per workload, LASTZ-style parameters (gap open 400, extend 30, y-drop 9400,
threshold 3000) over the ungapped extender's sample matrix.

    python tools/bench_gapped_extender.py [--steps K] [--warmup W] [--workloads sample,synth] [--no-oracle] [--modes default,skip]
                                          [--skip-covered]

Workloads:
  sample  the golden sample pipeline: its seeds through the ungapped extender on the device, then the gapped stage on the
          resulting scored segment pairs through the device-pointer call. The anchors on diagonal 0 (the record against
          itself) and the others are also run and reported apart, as host-pointer calls;
  synth   synth.extender_workload(2 Mb, 15 % divergence, 16 seeds, half spurious): long homologous extensions.

Each line: anchors/s and live cells/s of the whole call (host clock around extend + sync, after `warmup` calls, mean of
`steps`), the per-pass device ms of the last call (CUDA events), and the oracle's CPU wall clock on the same anchors on one
thread and on all threads (anchors split across threads), with an identical_outputs flag. The card name and power limit are
read in the same run. Writes nothing to the tree.

--modes runs every workload in each listed mode: default, or skip (skip-covered, DESIGN.md section 18), which adds the skip stats
and compares against the skip oracle. --skip-covered is --modes skip.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

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


def oracle_times(q, t, anchors, threads, order=None):
    import extender_libs as xl
    import gapped_extender_libs as gl
    import gapped_skip_libs as sk
    args = (xl.SAMPLE_MATRIX, gl.LASTZ_OPEN, gl.LASTZ_EXTEND, gl.LASTZ_YDROP, gl.LASTZ_THRESHOLD)
    t0 = time.perf_counter()
    # skip mode: the skip oracle in the call's processing order (it has no threaded form)
    want = gl.oracle_run(q, t, *args, anchors) if order is None else sk.skip_run(q, t, *args, anchors, order)
    one = time.perf_counter() - t0
    if order is not None:
        return want, one, None
    parts = np.array_split(anchors, min(threads, max(1, len(anchors))))
    t0 = time.perf_counter()
    with ThreadPoolExecutor(len(parts)) as pool:
        list(pool.map(lambda p: gl.oracle_run(q, t, *args, p), parts))
    return want, one, time.perf_counter() - t0


def timed(call, steps, warmup):
    for _ in range(warmup):
        call()
    t0 = time.perf_counter()
    for _ in range(steps):
        out = call()
    return out, (time.perf_counter() - t0) / steps


def measure(name, gx, q, t, anchors, call, steps, warmup, oracle, skip=False, order=None):
    import gapped_extender_libs as gl
    from genomeworks_b200 import cudaextender as ce

    def once():
        assert call() == ce.success and gx.sync() == ce.success
        return gx.get_alignments()

    (rec, cig), sec = timed(once, steps, warmup)
    live = gx.last_live_cells()
    p1, p2 = gx.last_pass_ms()
    gpu, power = card()
    row = dict(workload=name, anchors=len(anchors), alignments=len(rec), with_cigar=int(rec["has_cigar"].sum()) if len(rec) else 0,
               live_cells=live, anchors_per_s=len(anchors) / sec, live_cells_per_s=live / sec, call_ms=sec * 1e3, pass1_ms=p1, pass2_ms=p2,
               gpu=gpu, power_limit=power, mode="skip" if skip else "default")
    if skip:
        row.update(gx.last_skip_stats())
    if oracle:
        want, one, many = oracle_times(q, t, anchors, os.cpu_count() or 1,
                                       (np.arange(len(anchors), dtype=np.int32) if order is None else order) if skip else None)
        row.update(oracle_ms_1_thread=one * 1e3, oracle_ms_all_threads=many * 1e3 if many is not None else None, oracle_threads=os.cpu_count(),
                   identical_outputs=gl.rows(rec) == gl.rows(want[0]) and cig == want[1] and live == want[2])
    print(json.dumps(row), flush=True)


def run_sample(steps, warmup, oracle, skip=False):
    import torch
    import extender_libs as xl
    import gapped_extender_libs as gl
    from genomeworks_b200 import cudaextender as ce
    seq, seeds, _ = xl.sample()
    ext = ce.create_extender(xl.SAMPLE_MATRIX, xl.SAMPLE_XDROP)
    dq = torch.from_numpy(seq).cuda()
    ds = torch.from_numpy(np.ascontiguousarray(seeds).view(np.int32).reshape(-1, 2).copy()).cuda()
    out = torch.empty((len(seeds), 4), dtype=torch.int32, device="cuda")
    cnt = torch.empty(1, dtype=torch.int32, device="cuda")
    assert ext.extend_async_device(dq, dq, xl.SAMPLE_THRESHOLD, ds, out, cnt) == ce.success
    torch.cuda.synchronize()
    n = int(cnt.item())
    ssps = out[:n].cpu().numpy()
    anchors = np.zeros(n, dtype=gl.ANCHOR_DTYPE)
    anchors["query"] = ssps[:, 0] + ssps[:, 2] // 2
    anchors["target"] = ssps[:, 1] + ssps[:, 2] // 2
    gx = ce.create_gapped_extender(xl.SAMPLE_MATRIX, gl.LASTZ_OPEN, gl.LASTZ_EXTEND, gl.LASTZ_YDROP, skip_covered=skip)
    order = np.argsort(-ssps[:, 3].astype(np.int64), kind="stable").astype(np.int32)
    measure("sample_pipeline", gx, seq, seq, anchors, lambda: gx.extend_ssps_device(dq, dq, gl.LASTZ_THRESHOLD, out, n), steps, warmup,
            oracle, skip, order)
    diag0 = anchors["query"] == anchors["target"]
    for label, part in (("sample_diagonal0", anchors[diag0]), ("sample_off_diagonal", anchors[~diag0])):
        measure(label, gx, seq, seq, part, lambda: gx.extend_async(seq, seq, gl.LASTZ_THRESHOLD, part), steps, warmup, oracle, skip)
    gx.close()
    ext.close()


def run_synth(steps, warmup, oracle, skip=False):
    import extender_libs as xl
    import gapped_extender_libs as gl
    from genomeworks_b200 import cudaextender as ce
    from genomeworks_b200 import synth
    t, q, seeds = synth.extender_workload(2_000_000, 0.15, 16, 0.5, seed=2025)
    gx = ce.create_gapped_extender(xl.SAMPLE_MATRIX, gl.LASTZ_OPEN, gl.LASTZ_EXTEND, gl.LASTZ_YDROP, skip_covered=skip)
    measure("synth_2mb_15pct", gx, q, t, seeds, lambda: gx.extend_async(q, t, gl.LASTZ_THRESHOLD, seeds), steps, warmup, oracle, skip)
    gx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="sample,synth")
    ap.add_argument("--no-oracle", action="store_true")
    ap.add_argument("--modes", default="default")
    ap.add_argument("--skip-covered", action="store_true")
    a = ap.parse_args()
    modes = ["skip"] if a.skip_covered else a.modes.split(",")
    for w in a.workloads.split(","):
        for m in modes:
            {"sample": run_sample, "synth": run_synth}[w](a.steps, a.warmup, not a.no_oracle, {"default": False, "skip": True}[m])


if __name__ == "__main__":
    main()
