"""Argument checks of the skip-covered mode (DESIGN.md section 18): the C entry points on NULL handles, the Python arguments
before any device work, and the cudaextender tool's --skip-covered option. CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import extender_libs as xl
import gapped_extender_libs as gl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "build", "cudaextender")


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def test_c_entry_points_on_null_handles(ce):
    from genomeworks_b200._lib import lib
    L = lib()
    out = np.zeros(5, dtype=np.int64)
    for name in ("gapped_extender", "genome_aligner"):
        assert getattr(L, "gwb200_%s_set_skip_covered" % name)(None, 1, 0) == -1
        assert getattr(L, "gwb200_%s_set_skip_covered" % name)(None, 0, 7) == -1
        # a negative round size is invalid_input, before the handle is looked at
        assert getattr(L, "gwb200_%s_set_skip_covered" % name)(None, 1, -1) == ce.invalid_input
        assert getattr(L, "gwb200_%s_last_skip_stats" % name)(None, out.ctypes.data_as(C.c_void_p)) == -1
        assert getattr(L, "gwb200_%s_last_skip_stats" % name)(None, None) == -1


@pytest.mark.parametrize("kw, err", [(dict(skip_covered="yes"), TypeError), (dict(skip_covered=1), TypeError),
                                     (dict(skip_covered=True, round_anchors=-1), ValueError),
                                     (dict(skip_covered=True, round_anchors=1 << 31), ValueError),
                                     (dict(skip_covered=True, round_anchors=2.5), TypeError),
                                     (dict(round_anchors=True), TypeError)])
def test_python_arguments_are_checked_before_device_work(ce, kw, err):
    # without a device a valid call raises RuntimeError; these raise their own error first
    with pytest.raises(err):
        ce.create_gapped_extender(xl.SAMPLE_MATRIX, gl.LASTZ_OPEN, gl.LASTZ_EXTEND, gl.LASTZ_YDROP, **kw)
    with pytest.raises(err):
        ce.GenomeAligner("both", **kw)
    if "skip_covered" in kw and "round_anchors" not in kw:
        with pytest.raises(err):
            ce.align_genomes(["ACGT"], ["ACGT"], skip_covered=kw["skip_covered"])
    else:
        with pytest.raises(err):
            ce.align_genomes(["ACGT"], ["ACGT"], **kw)


def test_last_stats_keys_are_unchanged(ce):
    assert ce.STAGES == ("index", "count", "write", "ungapped", "gapped_pass1", "gapped_pass2")
    assert ce.SKIP_STATS == ("extended", "skipped", "speculative", "traced", "rounds")


def cli(args):
    return subprocess.run([CLI] + args, capture_output=True, text=True, timeout=120)


def test_cli_skip_covered_option(ce, tmp_path):
    r = cli(["--help"])
    assert r.returncode == 0 and "--skip-covered" in r.stderr and "--block-size" in r.stderr
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    # a long option only, and it takes no value
    r = cli(["--skip-covered=1", str(fa), str(fa)])
    assert r.returncode == 1 and "skip-covered" in r.stderr and r.stdout == ""
    r = cli(["--skip", str(fa)])
    assert r.returncode == 1 and "takes a target file and a query file" in r.stderr
    r = cli(["--skip-covered", str(fa), str(tmp_path / "missing.fa")])
    assert r.returncode == 1 and "cannot open" in r.stderr
    r = cli(["--skip-covered", "-B", "0", str(fa), str(fa)])
    assert r.returncode == 1 and "block-size takes an integer" in r.stderr


def test_cli_skip_covered_without_gpu_fails_loudly(ce, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    r = cli(["--skip-covered", str(fa), str(fa)])
    assert r.returncode != 0 and r.stdout == "" and "CUDA device" in r.stderr
