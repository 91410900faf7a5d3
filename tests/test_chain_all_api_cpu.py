"""Argument checks of the all-chains mode (DESIGN.md section 20): the C entry points on NULL handles, the Python arguments before
any device work, and the cudaextender tool's --chain-min-score option. CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "build", "cudaextender")
TOP = 1 << 20
LO, HI = -(1 << 63), (1 << 63) - 1


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def test_entry_points_on_null_handles(ce):
    from genomeworks_b200._lib import lib
    L = lib()
    dummy = C.c_void_p(16)  # never dereferenced: the argument checks come first
    # the checks of chain_device, before the handle; every minimum score is valid
    for args in ((dummy, 1, -1, 0), (dummy, 1, 0, TOP + 1), (dummy, -1, 0, 0), (None, 1, 0, 0)):
        for S in (LO, 0, HI):
            assert L.gwb200_ssp_chainer_chain_all_device(None, *args, S) == ce.invalid_input, (args, S)
    for args in ((dummy, 1, 0, 0), (None, 0, TOP, TOP)):
        for S in (LO, -1, 0, HI):
            assert L.gwb200_ssp_chainer_chain_all_device(None, *args, S) == -1, (args, S)
    assert L.gwb200_ssp_chainer_num_chains(None) == -1
    scores, offsets, members = (np.zeros(4, dtype=t) for t in (np.int64, np.int64, np.int32))
    assert L.gwb200_ssp_chainer_get_chains(None, scores.ctypes.data_as(C.c_void_p), offsets.ctypes.data_as(C.c_void_p),
                                           members.ctypes.data_as(C.c_void_p)) == -1
    assert L.gwb200_ssp_chainer_get_chains(None, None, None, None) == -1
    for on in (0, 1):
        for S in (LO, 0, HI):
            assert L.gwb200_genome_aligner_set_chain_min_score(None, on, S) == -1
    n = C.c_int64()
    assert L.gwb200_genome_aligner_last_chain_count(None, C.byref(n)) == -1
    assert L.gwb200_genome_aligner_last_chain_count(None, None) == -1


@pytest.mark.parametrize("chain, score, err", [
    (None, 0, ValueError), (False, 5, ValueError), (None, LO, ValueError),
    (True, True, TypeError), ((0, 0), False, TypeError), (True, 1.0, TypeError), (True, "5", TypeError), (True, np.float64(3), TypeError),
    (True, HI + 1, ValueError), ((1, 2), LO - 1, ValueError), ((-1, 0), 0, ValueError)])
def test_python_min_chain_score_is_checked_before_device_work(ce, chain, score, err):
    # without a device a valid call raises RuntimeError; these raise their own error first
    with pytest.raises(err):
        ce.GenomeAligner("both", chain=chain, min_chain_score=score)
    with pytest.raises(err):
        ce.align_genomes(["ACGT"], ["ACGT"], chain=chain, min_chain_score=score)


def test_python_min_chain_score_forms(ce):
    assert ce._chain_args(True, None) == ((0, 0), None) and ce._chain_args(None, None) == (None, None)
    assert ce._chain_args((3, 4), LO) == ((3, 4), LO) and ce._chain_args(True, np.int64(HI)) == ((0, 0), HI)
    assert ce._min_score("min_score", np.int32(-7)) == -7
    for bad in (True, np.bool_(False), 2.5, None):
        with pytest.raises(TypeError):
            ce._min_score("min_score", bad)


def cli(args):
    return subprocess.run([CLI] + args, capture_output=True, text=True, timeout=120)


def test_cli_chain_min_score_option(ce, tmp_path):
    r = cli(["--help"])
    assert r.returncode == 0 and "--chain-min-score=S" in r.stderr and "--chain[=D,A]" in r.stderr
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    # without --chain
    for args in (["--chain-min-score=5"], ["--chain-min-score=-9223372036854775808"]):
        r = cli(args + [str(fa), str(fa)])
        assert r.returncode == 1 and "needs --chain" in r.stderr and r.stdout == "", args
    # bad values
    for value in ("", "a", "1.5", "5x", "9223372036854775808", "-9223372036854775809"):
        r = cli(["--chain", "--chain-min-score=" + value, str(fa), str(fa)])
        assert r.returncode == 1 and "chain-min-score takes an integer" in r.stderr and r.stdout == "", (value, r.stderr)
    # good values parse; the files are looked at next
    for value in ("0", "-9223372036854775808", "9223372036854775807", "30000"):
        for order in (["--chain=1,2", "--chain-min-score=" + value], ["--chain-min-score=" + value, "--chain"]):
            r = cli(order + [str(fa), str(tmp_path / "missing.fa")])
            assert r.returncode == 1 and "cannot open" in r.stderr, (order, r.stderr)


def test_cli_chain_min_score_without_gpu_fails_loudly(ce, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    r = cli(["--chain", "--chain-min-score=100", str(fa), str(fa)])
    assert r.returncode != 0 and r.stdout == "" and "CUDA device" in r.stderr
