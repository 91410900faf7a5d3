"""CPU checks of the genome aligner's host side: parameter and record checks of the C ABI and of Python (all before any device
work), the PAF formatting with minus-strand coordinates, and the cudaextender tool's option errors."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import genome_aligner_libs as ga
import seeder_libs as sl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "build", "cudaextender")


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def test_defaults_are_the_tests_parameters(ce):
    p = ce.default_genome_params()
    assert np.array_equal(p["score_matrix"], ga.DEFAULTS["matrix"])
    assert (p["xdrop"], p["ssp_threshold"], p["gap_open"], p["gap_extend"], p["ydrop"], p["gapped_threshold"], p["transition"]) == (
        ga.DEFAULTS["xdrop"], ga.DEFAULTS["ssp_threshold"], ga.DEFAULTS["gap_open"], ga.DEFAULTS["gap_extend"], ga.DEFAULTS["ydrop"],
        ga.DEFAULTS["gapped_threshold"], 1)
    assert p["block_size"] == 1 << 25 and p["strand"] == 3 and p["traceback_budget"] == 1 << 30


@pytest.mark.parametrize("bad", [dict(gap_open=-1), dict(gap_extend=(1 << 24) + 1), dict(ydrop=-5), dict(ydrop=(1 << 28) + 1),
                                 dict(block_size=0), dict(traceback_budget=-1), dict(block_size=1 << 31)])
def test_bad_parameters_raise_before_device_work(ce, bad):
    with pytest.raises(ValueError):
        ce.align_genomes(["ACGT"], ["ACGT"], **bad)


def test_bad_matrix_strand_and_names(ce):
    m = np.array(ga.DEFAULTS["matrix"]).copy()
    m[3] = (1 << 24) + 1
    with pytest.raises(ValueError):
        ce.align_genomes(["A"], ["A"], score_matrix=m)
    with pytest.raises(ValueError):
        ce.align_genomes(["A"], ["A"], score_matrix=m[:63])
    with pytest.raises(ValueError):
        ce.align_genomes(["A"], ["A"], strand="forward")
    with pytest.raises(TypeError):
        ce.align_genomes(["A"], ["A"], x_drop=3)


def test_c_abi_checks(ce):
    from genomeworks_b200._lib import GenomeAlignerParams, lib
    L = lib()
    p = GenomeAlignerParams()
    L.gwb200_genome_aligner_default_params(C.byref(p))
    h = C.c_void_p()
    for field, value in (("strand", 0), ("strand", 4), ("block_size", -3), ("gap_open", 1 << 25)):
        q = GenomeAlignerParams()
        C.pointer(q)[0] = p
        setattr(q, field, value)
        assert L.gwb200_genome_aligner_create(C.byref(h), C.byref(q), None, 0, None, None, None) == ce.invalid_input
    assert L.gwb200_genome_aligner_create(C.byref(h), None, None, 0, None, None, None) == ce.invalid_input
    codes = np.zeros(10, dtype=np.int8)

    def run(offsets, n, data=codes):
        off = np.asarray(offsets, dtype=np.int64)
        return L.gwb200_genome_aligner_run(None, data.ctypes.data_as(C.c_void_p) if data is not None else None, off.ctypes.data_as(C.c_void_p),
                                           n, codes.ctypes.data_as(C.c_void_p), np.array([0, 10], np.int64).ctypes.data_as(C.c_void_p), 1)
    assert run([0, 10], -1) == ce.invalid_input
    assert run([1, 10], 1) == ce.invalid_input                # offsets start at 0
    assert run([0, 6, 4], 2) == ce.invalid_input              # decreasing
    assert run([0, 1 << 31], 1) == ce.invalid_input           # a record of 2^31 codes
    assert run([0, 10], 1, None) == ce.invalid_input          # no codes
    assert run([0, 10], 1) == -1                              # good input, null handle: GWB200_E_INVALID_ARGUMENT
    assert run([0, 0], 1, None) == -1                         # an empty record needs no codes
    # the seeder: a bad length before the handle, then the null handle
    assert L.gwb200_seeder_index_target(None, None, 5) == ce.invalid_input
    assert L.gwb200_seeder_index_target(None, codes.ctypes.data_as(C.c_void_p), 1 << 31) == ce.invalid_input
    assert L.gwb200_seeder_count(None, None, 5) == -1
    assert L.gwb200_seeder_get_block(None, 0, 0, None) == -1


def test_format_paf_minus_strand(ce):
    rec = np.zeros(3, dtype=ce.GENOME_DTYPE)
    # query [L - end, L - begin) of the reverse complement's [begin, end): L = 100, rc interval [10, 40) -> [60, 90)
    rec[0] = (4500, 1, 0, 1, 1, 60, 90, 200, 229, 27, 31)
    rec[1] = (3100, 0, 1, 0, 1, 5, 40, 7, 42, 35, 35)
    rec[2] = (9000, 0, 0, 1, 0, 0, 100, 300, 380, 0, 100)
    cigars = ["10M1I9M2D10M", "35M", ""]
    got = ce.format_paf(rec, cigars, ["chrA", "chrB"], [1000, 2000], ["read1", "read2"], [100, 50])
    assert got.splitlines() == [
        "read1\t100\t60\t90\t-\tchrB\t2000\t200\t229\t27\t31\t255\tAS:i:4500\tcg:Z:10M1I9M2D10M",
        "read2\t50\t5\t40\t+\tchrA\t1000\t7\t42\t35\t35\t255\tAS:i:3100\tcg:Z:35M",
        "read1\t100\t0\t100\t-\tchrA\t1000\t300\t380\t0\t100\t255\tAS:i:9000"]
    assert got == ga.paf_oracle(ga.engine_rows(rec), cigars, ["chrA", "chrB"], [1000, 2000], ["read1", "read2"], [100, 50])


def test_paf_columns_on_the_reverse_complement():
    q = np.array([0, 1, 2, 3, 4, 0, 0, 1], dtype=np.int8)  # ACGTaAAC
    rc = sl.reverse_complement(q)                            # GTTaACGT
    assert rc.tolist() == [2, 3, 3, 4, 0, 1, 2, 3]
    t = np.array([2, 3, 3, 4, 0, 1, 2, 2], dtype=np.int8)
    # 8M over rc: equal at 0, 1, 2, 4, 5, 6 (4 equals 4 but is not in 0..3)
    assert ga.paf_columns("8M", rc, t, 0, 0, True, 8, 8) == (6, 8)
    assert ga.paf_columns("3M1I2M1D2M", rc, t, 0, 0, True, 8, 8) == (4, 9)
    assert ga.paf_columns("", rc, t, 0, 0, False, 8, 6) == (0, 8)


def cli(args):
    return subprocess.run([CLI] + args, capture_output=True, text=True, timeout=120)


def test_cli_help_and_option_errors(ce, tmp_path):
    r = cli(["--help"])
    assert r.returncode == 0 and "Usage: cudaextender" in r.stderr and "--strand" in r.stderr and "--block-size" in r.stderr
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    for args, msg in ((["-s", "forward"], "strand must be plus, minus or both"), (["-B", "0"], "block-size takes an integer"),
                      (["-x", "ten"], "xdrop takes an integer"), (["-o", "-1"], "gap-open takes an integer"),
                      (["-y", str((1 << 28) + 1)], "ydrop takes an integer"), (["-b", "-2"], "traceback-budget takes an integer"),
                      (["-e", "1.5"], "gap-extend takes an integer")):
        r = cli(args + [str(fa), str(fa)])
        assert r.returncode == 1 and msg in r.stderr and r.stdout == "", (args, r.stderr)
    r = cli([str(fa)])
    assert r.returncode == 1 and "takes a target file and a query file" in r.stderr
    r = cli([str(fa), str(tmp_path / "missing.fa")])
    assert r.returncode == 1 and "cannot open" in r.stderr
    gz = tmp_path / "a.fa.gz"
    gz.write_bytes(b"\x1f\x8b\x08\x00")
    assert "gzip-compressed" in cli([str(gz), str(fa)]).stderr


def test_cli_without_gpu_fails_loudly(ce, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    r = cli([str(fa), str(fa)])
    assert r.returncode != 0 and r.stdout == "" and "CUDA device" in r.stderr
