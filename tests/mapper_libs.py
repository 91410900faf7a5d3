"""Inputs, option sets and runners shared by the cudamapper tool's tests, its fixture generator and tools/bench_mapper.py.

- build/cudamapper: this engine's tool (built by build());
- oracle/_ref/cudamapper: the unmodified reference tool, built by build() where the reference sources exist (oracle/Makefile);
  only the fixture generator and the benchmark run it;
- oracle/_ref/libgwref_mapper_utils.so: the reference's print_paf, group_reads_into_indices and parser order (host code), used
  by the CPU tests where it exists.

An input is one FASTA file (all-to-all) or two (query != target), written into a directory: the data files under
tests/golden/cudamapper (the gzipped covid reads decompressed, as the tool reads plain text only) and seeded synthetic reads of
one genome with every other read reverse-complemented.
"""
import ctypes as C
import gzip
import hashlib
import os
import subprocess
import sys

import numpy as np

import index_libs as il
from checker_lib import REF_DIR, load, ptr, read_fixture

ROOT = il.ROOT
GOLDEN = il.GOLDEN
TOOL = os.path.join(ROOT, "build", "cudamapper")
REF_TOOL = os.path.join(REF_DIR, "cudamapper")
REF_UTILS = os.path.join(REF_DIR, "libgwref_mapper_utils.so")
FIXTURE = os.path.join(GOLDEN, "reference_mapper_outputs.json.gz")
SMALL = 3000  # outputs of at most this many lines are stored line by line, larger ones as a count and a SHA-256
MEMORY = ["-m", "4"]  # an explicit pool of 4 GiB: the GPU machines are shared

sys.path.insert(0, os.path.join(ROOT, "tools"))

_RC = bytes.maketrans(b"ACGT", b"TGCA")


def synthetic(seed, total, divergence, genome_len=1000000):
    """Reads of 5-20 kb from one genome with `divergence` of their bases substituted; every other read reverse-complemented."""
    from bench_index import synthetic_reads
    reads = synthetic_reads(seed, genome_len, total, lo=5000, hi=20000, divergence=divergence)
    return [r[::-1].translate(_RC) if i % 2 else r for i, r in enumerate(reads)]


def write_fasta(path, reads, prefix="read"):
    with open(path, "wb") as f:
        for i, r in enumerate(reads):
            f.write(b">%s_%d some description\n" % (prefix.encode(), i))
            for k in range(0, len(r), 80):
                f.write(r[k:k + 80] + b"\n")


def write_inputs(d):
    """name -> (query path, target path) of every fixture input, written into directory d."""
    out = {}
    for name in ("10_reads", "20_reads"):
        p = os.path.join(GOLDEN, name + ".fasta")
        out[name] = (p, p)
    cov = os.path.join(d, "covid-reads.fasta")
    with gzip.open(os.path.join(GOLDEN, "covid-reads.fasta.gz"), "rb") as f, open(cov, "wb") as g:
        g.write(f.read())
    out["covid"] = (cov, cov)
    # genome length, total read length and divergence: a coverage of 2 to 3, where the default filter (1e-5) still leaves anchors
    for name, seed, genome, total, div in (("syn_1pct", 11, 1000000, 2000000, 0.01), ("syn_3pct", 12, 300000, 600000, 0.03),
                                           ("syn_small", 13, 100000, 300000, 0.02)):
        reads = synthetic(seed, total, div, genome)
        p = os.path.join(d, name + ".fasta")
        write_fasta(p, reads)
        out[name] = (p, p)
        if name == "syn_small":
            h = len(reads) // 2
            qp, tp = os.path.join(d, name + "_q.fasta"), os.path.join(d, name + "_t.fasta")
            write_fasta(qp, reads[:h], "q")
            write_fasta(tp, reads[h:], "t")
            out["syn_small_halves"] = (qp, tp)
    return out


# option set name -> arguments
OPTIONS = {
    "default": [],
    "tiles": ["-i", "1", "-t", "1"],
    "rescue": ["-R"],
    "drop": ["-D"],
    "thresholds": ["-r", "5", "-l", "500", "-b", "500", "-z", "0.5"],
    "k19w5": ["-k", "19", "-w", "5"],
    "filter": ["-F", "0.0002"],
}
# "-a 2" is added to these sets where nothing fuses (the output with -D is the same), so that the reference's CIGARs, which it
# computes before fusion, sit on the right lines; stored as "<set>_a2"
ALIGN_BASES = ("default", "k19w5", "filter")


def options(name):
    """The arguments of a stored option set."""
    if name.endswith("_a2"):
        return OPTIONS[name[:-3]] + ["-a", "2"]
    return OPTIONS[name]


def run(tool, args, query, target, timeout=900):
    """(exit code, stdout bytes, stderr text) of one run."""
    r = subprocess.run([tool] + MEMORY + args + [query, target], capture_output=True, timeout=timeout)
    return r.returncode, r.stdout, r.stderr.decode(errors="replace")


def sorted_lines(text):
    return sorted(text.decode().splitlines())


def to_json(text):
    lines = sorted_lines(text)
    if len(lines) <= SMALL:
        return {"lines": lines}
    return {"count": len(lines), "sha256": hashlib.sha256("\n".join(lines).encode()).hexdigest()}


def matches(text, stored):
    return to_json(text) == stored


def load_fixture():
    return read_fixture(FIXTURE)


def cigar_lengths(cigar):
    """(query bases, target bases) a basic CIGAR consumes: in cudaaligner's AlignmentState an insertion is a target base the query
    lacks and a deletion a query base the target lacks."""
    q = t = 0
    num = ""
    for c in cigar:
        if c.isdigit():
            num += c
            continue
        n, num = int(num), ""
        if c == "M":
            q, t = q + n, t + n
        elif c == "I":
            t += n
        elif c == "D":
            q += n
    return q, t


def ref_utils():
    return load("_ref/libgwref_mapper_utils.so", {
        "ref_print_paf": (C.c_int64, [C.c_char_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]),
        "ref_group_reads_into_indices": (C.c_int64, [C.c_char_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_int64]),
        "ref_parser_names": (C.c_int64, [C.c_char_p, C.c_uint32, C.c_void_p, C.c_int64])})


def ref_print_paf(query_path, target_path, overlaps, cigars, kmer_size):
    L = ref_utils()
    ov = np.ascontiguousarray(overlaps)
    cg = None
    if cigars is not None:
        bufs = [C.create_string_buffer(c.encode()) for c in cigars]
        cg = (C.c_char_p * max(1, len(bufs)))(*[C.cast(b, C.c_char_p) for b in bufs])
    args = (query_path.encode(), target_path.encode(), ptr(ov), len(ov), C.cast(cg, C.c_void_p) if cg is not None else None,
            kmer_size)
    n = L.ref_print_paf(*args, None, 0)
    out = C.create_string_buffer(max(1, n))
    L.ref_print_paf(*args, out, n)
    return out.raw[:n]


def ref_group_reads_into_indices(path, max_basepairs):
    L = ref_utils()
    cap = 1 << 16
    first = np.zeros(cap, dtype=np.uint32)
    count = np.zeros(cap, dtype=np.uint32)
    k = L.ref_group_reads_into_indices(path.encode(), max_basepairs, ptr(first), ptr(count), cap)
    return [(int(first[i]), int(count[i])) for i in range(k)]


def ref_parser_names(path, min_length):
    L = ref_utils()
    n = L.ref_parser_names(path.encode(), min_length, None, 0)
    out = C.create_string_buffer(max(1, n))
    L.ref_parser_names(path.encode(), min_length, out, n)
    return out.raw[:n].split(b"\n")[:-1]


def _i32(x):
    x = int(x) & 0xFFFFFFFF
    return x - (1 << 32) if x >= 1 << 31 else x


def paf_oracle(overlaps, query_names, query_lengths, target_names, target_lengths, kmer_size, cigars=None):
    """print_paf restated in Python: "%s\\t%lu\\t%i\\t%i\\t%c\\t%s\\t%lu\\t%i\\t%i\\t%i\\t%ld\\t%i" (the %i columns as int32, column 10 the
    uint32 product num_residues * kmer_size), then "\\tcg:Z:<cigar>" with CIGARs, then a newline."""
    out = []
    for i, o in enumerate(overlaps):
        qs, qe = int(o["query_start_position_in_read"]), int(o["query_end_position_in_read"])
        ts, te = int(o["target_start_position_in_read"]), int(o["target_end_position_in_read"])
        qn, tn = query_names[o["query_read_id"]], target_names[o["target_read_id"]]
        qn = qn.decode() if isinstance(qn, bytes) else qn
        tn = tn.decode() if isinstance(tn, bytes) else tn
        line = "%s\t%d\t%d\t%d\t%c\t%s\t%d\t%d\t%d\t%d\t%d\t255" % (
            qn, query_lengths[o["query_read_id"]], _i32(qs), _i32(qe), chr(o["relative_strand"]), tn, target_lengths[o["target_read_id"]],
            _i32(ts), _i32(te), _i32(int(o["num_residues"]) * kmer_size), max(abs(ts - te), abs(qs - qe)))
        if cigars is not None:
            line += "\tcg:Z:" + cigars[i]
        out.append(line + "\n")
    return "".join(out).encode()
