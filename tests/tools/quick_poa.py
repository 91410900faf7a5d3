"""Development aid: time a POA config, print per-phase cycle shares and a digest of the consensus.
usage: quick_poa.py {c2|c3} [n_windows] [--ref] [--factor F] [--len L] [--msa] [--band-mode NAME (c2 only)]"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from genomeworks_b200 import cudapoa, synth
import ref_lib

which = sys.argv[1] if len(sys.argv) > 1 else "c2"
n = int(sys.argv[2]) if len(sys.argv) > 2 and not sys.argv[2].startswith("--") else (1024 if which == "c2" else 132)
if which == "c2":
    win_nseq, seq_len, data = synth.poa_windows(n, 1000, 16, 20, 10, 10, seed0=1000, max_read_len=1024)
    bm = sys.argv[sys.argv.index("--band-mode") + 1] if "--band-mode" in sys.argv else "static_band"  # e.g. static_band_traceback
    cfg = cudapoa.make_config(1024, 16, 256, bm)
    mem = 16 << 30
    ref_args = (1024, 16, 256, cfg.band_mode)
    factor = 2.0
else:
    factor = float(sys.argv[sys.argv.index("--factor") + 1]) if "--factor" in sys.argv else 6.0
    L = int(sys.argv[sys.argv.index("--len") + 1]) if "--len" in sys.argv else 10000  # window length (C3: 10 kb)
    mseq = (L + 1023) // 1024 * 1024
    win_nseq, seq_len, data = synth.poa_windows(n, L, 32, L // 50, L // 100, L // 100, seed0=1000, max_read_len=mseq)
    cfg = cudapoa.make_config(mseq, 32, 256, "adaptive_band", adaptive_storage_factor=factor)
    mem = int(n * (factor * 32.5e6 + 20e6) * mseq / 10240) + (2 << 30)
    if "--allmem" in sys.argv:
        mem = -1
    ref_args = (mseq, 32, 256, 2)
MSA = "--msa" in sys.argv
if MSA and which != "c2":
    mem += int(n * 1.2e6 * 32)  # MSA rows + per-read node paths
b = cudapoa.CudaPoaBatch(cfg.max_sequences_per_poa, cfg.max_sequence_size, mem, output_type="msa" if MSA else "consensus", config=cfg)
kernel = "tb" if cfg.band_mode in (cudapoa.BAND_MODES["static_band_traceback"], cudapoa.BAND_MODES["adaptive_band_traceback"]) else "v3"
print("kernel", kernel, "max_poas", b.max_poas, "resident", b.resident_windows, flush=True)
for it in range(3):
    b.reset()
    b.add_poa_groups_flat(win_nseq, seq_len, data)
    b.enable_timers(it == 2)
    t1 = time.time()
    b.generate_poa()
    if MSA:
        msa, st_list = b.get_msa()
        st = np.array(st_list)
        c = cov = lens = None
    else:
        c, cov, lens, st = b.get_consensus_arrays()
    t2 = time.time()
    print("ours: generate+get %.1f ms, kernel %.2f ms, cells %.3e, ok=%d  -> %.0f windows/s" % ((t2 - t1) * 1e3, b.last_kernel_ms(), b.last_cells(),
                                                                                             int((st == 0).sum()), n / (b.last_kernel_ms() / 1e3)), flush=True)
tm = b.get_timers()
tot = max(1, sum(tm.values()))
print("phase shares:", {k: "%.1f%%" % (100.0 * v / tot) for k, v in tm.items()}, "cycles/window %.3e" % (tot / n), flush=True)
if MSA:
    print("msa: rows of window 0:", len(msa[0]), "columns:", len(msa[0][0]) if msa[0] else 0)
    b.close()
    sys.exit(0)
ours = [bytes(c[i, :lens[i]]).decode() for i in range(n)]
import hashlib
print("digest", hashlib.sha1(("|".join(ours) + str(list(st))).encode()).hexdigest()[:16], "cov", hashlib.sha1(cov.tobytes()).hexdigest()[:12], flush=True)
b.close()
if "--ref" in sys.argv and ref_lib.have_gwref():
    r = ref_lib.ref_poa_run(win_nseq, seq_len, data, *ref_args, adaptive_storage_factor=factor, mem_fraction=0.5, max_windows_per_batch=n)
    r = ref_lib.ref_poa_run(win_nseq, seq_len, data, *ref_args, adaptive_storage_factor=factor, mem_fraction=0.5, max_windows_per_batch=n)
    print("ref : generate+get %.1f ms -> %.0f windows/s; identical=%s" % (r["timings"][1], n / (r["timings"][1] / 1e3),
                                                                        r["consensus"] == ours and list(r["status"]) == list(st)), flush=True)
