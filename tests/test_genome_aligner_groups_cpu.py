"""Argument checks of the genome aligner's record groups (DESIGN.md section 21): the C entry points on NULL handles and out of
range sizes, the Python arguments before any device work, and the cudaextender tool's --group-bases option. CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "build", "cudaextender")
TOP = (1 << 31) - 1


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def test_entry_points_on_null_handles(ce):
    from genomeworks_b200._lib import lib
    L = lib()
    # the range check comes before the handle is looked at
    for n in (0, -1, TOP + 1, 1 << 40, -(1 << 63)):
        assert L.gwb200_genome_aligner_set_group_bases(None, C.c_int64(n)) == ce.invalid_input, n
        assert L.gwb200_genome_aligner_set_group_bases(C.c_void_p(16), C.c_int64(n)) == ce.invalid_input, n
    for n in (1, 4096, 1 << 28, TOP):
        assert L.gwb200_genome_aligner_set_group_bases(None, C.c_int64(n)) == -1, n
    out = np.zeros(3, dtype=np.int64)
    assert L.gwb200_genome_aligner_last_group_stats(None, out.ctypes.data_as(C.c_void_p)) == -1
    assert L.gwb200_genome_aligner_last_group_stats(None, None) == -1


@pytest.mark.parametrize("value, err", [(0, ValueError), (-5, ValueError), (TOP + 1, ValueError), (1 << 40, ValueError),
                                        (True, TypeError), (np.bool_(True), TypeError), (4096.0, TypeError), ("4096", TypeError),
                                        (None, TypeError), (np.float32(2), TypeError)])
def test_python_group_bases_is_checked_before_device_work(ce, value, err):
    # without a device a valid call raises RuntimeError; these raise their own error first
    with pytest.raises(err):
        ce.GenomeAligner("both", group_bases=value)
    with pytest.raises(err):
        ce.align_genomes(["ACGT"], ["ACGT"], group_bases=value)


def test_python_group_bases_forms(ce):
    assert ce._group_bases(1) == 1 and ce._group_bases(np.int64(TOP)) == TOP and ce._group_bases(np.uint8(7)) == 7
    assert ce.DEFAULT_GROUP_BASES == 1 << 28


def cli(args):
    return subprocess.run([CLI] + args, capture_output=True, text=True, timeout=120)


def test_cli_group_bases_option(ce, tmp_path):
    r = cli(["--help"])
    assert r.returncode == 0 and "--group-bases=N" in r.stderr
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    for value in ("", "a", "0", "-1", "1.5", "5x", "2147483648", "9223372036854775808"):
        r = cli(["--group-bases=" + value, str(fa), str(fa)])
        assert r.returncode == 1 and "group-bases takes an integer in [1, 2147483647]" in r.stderr and r.stdout == "", (value, r.stderr)
    r = cli(["--group-bases", str(fa), str(fa)])  # the option takes the first file as its value
    assert r.returncode == 1 and r.stdout == ""
    # good values parse; the files are looked at next
    for value in ("1", "16", "2147483647", "268435456"):
        for order in (["--group-bases=" + value], ["--group-bases", value, "-s", "minus"]):
            r = cli(order + [str(fa), str(tmp_path / "missing.fa")])
            assert r.returncode == 1 and "cannot open" in r.stderr, (order, r.stderr)


def test_cli_group_bases_without_gpu_fails_loudly(ce, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    r = cli(["--group-bases=64", str(fa), str(fa)])
    assert r.returncode != 0 and r.stdout == "" and "CUDA device" in r.stderr
