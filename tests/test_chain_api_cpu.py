"""Argument checks of the SSP chainer and of chaining in the genome aligner (DESIGN.md section 19): the C entry points on NULL
handles and out-of-range penalties, the Python arguments before any device work, and the cudaextender tool's --chain option.
CPU only."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "build", "cudaextender")
TOP = 1 << 20


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def test_chainer_entry_points_on_null_handles(ce):
    from genomeworks_b200._lib import ChainStats, lib
    L = lib()
    assert L.gwb200_ssp_chainer_create(None, None, 0, None, None, None) == -1
    dummy = C.c_void_p(16)  # never dereferenced: the argument checks come first
    # penalties outside [0, 2^20], n < 0 and NULL data with n > 0 are invalid_input before the handle is looked at
    for args in ((dummy, 1, -1, 0), (dummy, 1, 0, -1), (dummy, 1, TOP + 1, 0), (dummy, 1, 0, TOP + 1), (dummy, -1, 0, 0),
                 (None, 1, 0, 0), (None, -5, 0, 0)):
        assert L.gwb200_ssp_chainer_chain_device(None, *args) == ce.invalid_input, args
    # valid arguments on a NULL handle
    for args in ((dummy, 1, 0, 0), (None, 0, TOP, TOP), (dummy, 7, TOP, 0)):
        assert L.gwb200_ssp_chainer_chain_device(None, *args) == -1, args
    assert L.gwb200_ssp_chainer_sync(None) == -1
    assert L.gwb200_ssp_chainer_num_chained(None) == -1
    score = C.c_int64()
    assert L.gwb200_ssp_chainer_get_chain(None, None, C.byref(score)) == -1
    assert L.gwb200_ssp_chainer_get_dp(None, None, None) == -1
    ms = C.c_float()
    assert L.gwb200_ssp_chainer_last_ms(None, C.byref(ms)) == -1
    L.gwb200_ssp_chainer_destroy(None)
    # the aligner's setter checks the penalties first, then the handle
    for D, A in ((-1, 0), (0, -1), (TOP + 1, 0), (0, TOP + 1)):
        assert L.gwb200_genome_aligner_set_chain(None, 1, D, A) == ce.invalid_input
        assert L.gwb200_genome_aligner_set_chain(None, 0, D, A) == ce.invalid_input
    assert L.gwb200_genome_aligner_set_chain(None, 1, TOP, TOP) == -1
    assert L.gwb200_genome_aligner_set_chain(None, 0, 0, 0) == -1
    st = ChainStats()
    assert L.gwb200_genome_aligner_last_chain_stats(None, C.byref(st)) == -1
    assert L.gwb200_genome_aligner_last_chain_stats(None, None) == -1


def test_chainer_without_gpu_fails_loudly(ce):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    from genomeworks_b200._lib import lib
    h = C.c_void_p()
    assert lib().gwb200_ssp_chainer_create(C.byref(h), None, 0, None, None, None) < 0 and not h
    with pytest.raises(RuntimeError):
        ce.create_ssp_chainer()


@pytest.mark.parametrize("chain, err", [((-1, 0), ValueError), ((0, TOP + 1), ValueError), ((TOP + 1, TOP), ValueError),
                                        ("yes", TypeError), (1, TypeError), ((1,), TypeError), ((1, 2, 3), TypeError),
                                        ((1.5, 0), TypeError), ((True, 0), TypeError), ((0, None), TypeError)])
def test_python_chain_argument_is_checked_before_device_work(ce, chain, err):
    # without a device a valid call raises RuntimeError; these raise their own error first
    with pytest.raises(err):
        ce.GenomeAligner("both", chain=chain)
    with pytest.raises(err):
        ce.align_genomes(["ACGT"], ["ACGT"], chain=chain)


def test_python_chain_argument_forms(ce):
    assert ce._chain_arg(None) is None and ce._chain_arg(False) is None
    assert ce._chain_arg(True) == (0, 0)
    assert ce._chain_arg((3, 4)) == (3, 4) and ce._chain_arg([0, TOP]) == (0, TOP)
    assert ce.CHAIN_STATS == ("ssps_in", "ssps_chained", "pairs", "chain_ms")
    # the existing stats keep their keys
    assert ce.STAGES == ("index", "count", "write", "ungapped", "gapped_pass1", "gapped_pass2")


def test_params_struct_is_unchanged():
    from genomeworks_b200._lib import GenomeAlignerParams
    assert C.sizeof(GenomeAlignerParams) == 64 * 4 + 8 * 4 + 2 * 8
    assert [n for n, _ in GenomeAlignerParams._fields_] == ["score_matrix", "xdrop", "ssp_threshold", "gap_open", "gap_extend", "ydrop",
                                                            "transition", "strand", "block_size", "gapped_threshold", "traceback_budget"]


def cli(args):
    return subprocess.run([CLI] + args, capture_output=True, text=True, timeout=120)


def test_cli_chain_option(ce, tmp_path):
    r = cli(["--help"])
    assert r.returncode == 0 and "--chain[=D,A]" in r.stderr and "--skip-covered" in r.stderr
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    for value, what in (("5", "chain takes D,A"), ("", "chain takes D,A"), ("-1,0", "diagonal penalty takes an integer"),
                        ("0,-1", "anti-diagonal penalty takes an integer"), ("1048577,0", "diagonal penalty takes an integer"),
                        ("0,1048577", "anti-diagonal penalty takes an integer"), ("a,b", "diagonal penalty takes an integer"),
                        ("1,2,3", "anti-diagonal penalty takes an integer"), (",4", "diagonal penalty takes an integer")):
        r = cli(["--chain=" + value, str(fa), str(fa)])
        assert r.returncode == 1 and what in r.stderr and r.stdout == "", (value, r.stderr)
    # a long option only, whose value follows '='
    r = cli(["-c", str(fa), str(fa)])
    assert r.returncode == 1 and r.stdout == ""
    r = cli(["--chain", "3,4", str(fa), str(fa)])
    assert r.returncode == 1 and "takes a target file and a query file" in r.stderr
    r = cli(["--chain=3,4", str(fa), str(tmp_path / "missing.fa")])
    assert r.returncode == 1 and "cannot open" in r.stderr


def test_cli_chain_without_gpu_fails_loudly(ce, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    for opt in ("--chain", "--chain=1048576,0"):
        r = cli([opt, str(fa), str(fa)])
        assert r.returncode != 0 and r.stdout == "" and "CUDA device" in r.stderr
