"""Where the POA kernel spends its time: C3 of bench.py (640 windows of 10 kb x 32 reads, seeds 1000 + i, adaptive band 256,
int32 scores, adaptive_storage_factor 3.0) with the device phase timers, plus the kernel time of static bands 512 / 1024 / 1536
with int16 and int32 scores on v3, of static band 2048 on the first-generation kernel and of static_band_traceback 256 / 1536 on
the traceback-mode kernel.

usage: poa_phase_split.py [--reps N] [--no-static] [--no-c3]
Prints the card, the C3 kernel time (timers off, best of N), each phase's share of the summed phase cycles (timers on), and the
dp_rows cycles per executed DP cell. Kernel times are CUDA-event times of one launch of the whole batch."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from genomeworks_b200 import cudapoa, synth

REPS = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 3


def kernel_ms(b, reps):
    """Best-of-reps kernel time of the uploaded batch, timers off."""
    b.enable_timers(False)
    best = float("inf")
    for _ in range(reps):
        b.launch()
        b.sync()
        best = min(best, b.last_kernel_ms())
    return best


def c3():
    cfg = cudapoa.make_config(10240, 32, 256, "adaptive_band", adaptive_storage_factor=3.0)
    free_b, _ = torch.cuda.mem_get_info()
    b = cudapoa.CudaPoaBatch(32, 10240, int(free_b * 0.95), config=cfg)
    n = 640
    assert b.max_poas >= n, b.max_poas
    rc, added = b.add_poa_groups_flat(*synth.poa_windows(n, 10000, 32, 200, 100, 100, seed0=1000, max_read_len=10240))
    assert rc == 0 and added == n
    b.upload()
    b.sync()
    b.launch()  # warm-up
    b.sync()
    ms = kernel_ms(b, REPS)
    b.enable_timers(True)
    b.launch()
    b.sync()
    tm = b.get_timers()
    cells = b.last_cells()
    st = b.get_consensus_arrays()[3]
    print("C3: %d windows, resident %d, kernel %.1f ms (timers off, best of %d) -> %.0f windows/s, %d ok" % (
        n, b.resident_windows, ms, REPS, n / (ms / 1e3), int((st == 0).sum())))
    tot = max(1, sum(tm.values()))
    print("C3 phase shares: " + ", ".join("%s %.1f%%" % (k, 100.0 * v / tot) for k, v in tm.items()))
    print("C3 cycles per window %.3e; dp_rows cycles per executed DP cell %.3f (%d cells)" % (tot / n, tm["dp_rows"] / cells, cells))
    b.close()


def static_band(band, score, mode="static_band", kernel="v3"):
    # config of the static-band cases of test_gpu_poa_kernel_paths.py: match 8 keeps int16 scores, 40 needs int32
    match = 8 if score == 16 else 40
    cfg = cudapoa.make_config_explicit(3072, 6144, 4096, band, 16, band + 8, mode, 2 * band if "traceback" in mode else 0)
    free_b, _ = torch.cuda.mem_get_info()
    b = cudapoa.CudaPoaBatch(16, 3072, int(free_b * 0.9), config=cfg, match_score=match)
    assert b.score_bytes * 8 == score and cudapoa.KERNEL_NAMES[b.kernel] == kernel
    n = min(b.max_poas, 4 * max(b.resident_windows, 1))
    rc, added = b.add_poa_groups_flat(*synth.poa_windows(n, 2500, 16, 50, 25, 25, seed0=5000, max_read_len=3072))
    assert rc == 0 and added == n
    b.upload()
    b.sync()
    b.launch()
    b.sync()
    ms = kernel_ms(b, REPS)
    print("%s %s %4d int%d: %d windows, resident %d, kernel %.2f ms, cells %.3e" % (kernel, mode, band, score, n, b.resident_windows, ms, b.last_cells()))
    b.close()


if __name__ == "__main__":
    p = torch.cuda.get_device_properties(0)
    print("device:", p.name, p.multi_processor_count, "SMs")
    if "--no-c3" not in sys.argv:
        c3()
    if "--no-static" not in sys.argv:
        for band in (512, 1024, 1536):
            for score in (16, 32):
                static_band(band, score)
    for score in (16, 32):
        static_band(2048, score, kernel="v1")
        for band in (256, 1536):
            static_band(band, score, "static_band_traceback", "tb")
    torch.cuda.empty_cache()
