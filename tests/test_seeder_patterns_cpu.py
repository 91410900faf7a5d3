"""Argument checks of the seed pattern and the word cap (DESIGN.md section 22): the C entry points on NULL handles, bad patterns
and negative caps, the Python arguments before any device work, and the cudaextender tool's --seed and --max-word-count
options. CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import seed_pattern_libs as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "build", "cudaextender")
INT64_MAX = (1 << 63) - 1


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


SETTERS = ("gwb200_seeder_set_seed", "gwb200_genome_aligner_set_seed")


@pytest.mark.parametrize("setter", SETTERS)
def test_entry_points_check_the_pattern_and_cap_before_the_handle(ce, setter):
    from genomeworks_b200._lib import lib
    f = getattr(lib(), setter)
    for bad in sp.BAD_PATTERNS:
        assert f(None, bad.encode(), C.c_int64(0)) == ce.invalid_input, bad
        assert f(C.c_void_p(16), bad.encode(), C.c_int64(0)) == ce.invalid_input, bad
    assert f(None, None, C.c_int64(0)) == ce.invalid_input
    for cap in (-1, -(1 << 63)):
        assert f(None, b"12of19", C.c_int64(cap)) == ce.invalid_input
        assert f(C.c_void_p(16), b"12of19", C.c_int64(cap)) == ce.invalid_input
    # valid arguments reach the handle: NULL is GWB200_E_INVALID_ARGUMENT
    for good in sp.PATTERNS:
        for cap in (0, 1, INT64_MAX):
            assert f(None, good.encode(), C.c_int64(cap)) == -1, (good, cap)


@pytest.mark.parametrize("seed, err", [(s, ValueError) for s in sp.BAD_PATTERNS] +
                         [("match01", ValueError), ("match", ValueError), ("half12", ValueError), ("12OF19", ValueError),
                          (None, TypeError), (12, TypeError), (b"12of19", TypeError), (["1"], TypeError)])
def test_python_seed_is_checked_before_device_work(ce, seed, err):
    # without a device a valid call raises RuntimeError; these raise their own error first
    for call in (lambda: ce.Seeder(seed=seed), lambda: ce.create_seeder(seed=seed), lambda: ce.GenomeAligner("both", seed=seed),
                 lambda: ce.align_genomes(["ACGT"], ["ACGT"], seed=seed)):
        with pytest.raises(err):
            call()


@pytest.mark.parametrize("cap, err", [(-1, ValueError), (1 << 63, ValueError), (True, TypeError), (np.bool_(False), TypeError),
                                      (1.0, TypeError), ("5", TypeError), (None, TypeError)])
def test_python_cap_is_checked_before_device_work(ce, cap, err):
    for call in (lambda: ce.Seeder(max_word_count=cap), lambda: ce.create_seeder(max_word_count=cap),
                 lambda: ce.GenomeAligner("both", max_word_count=cap), lambda: ce.align_genomes(["ACGT"], ["ACGT"], max_word_count=cap)):
        with pytest.raises(err):
            call()


def test_python_seed_forms(ce):
    for good in sp.PATTERNS:
        assert ce.seed_pattern(good) == sp.bits(good)
    assert ce._seed_args("match14", np.int64(5)) == (b"match14", 5) and ce._seed_args("1", INT64_MAX) == (b"1", INT64_MAX)
    assert ce.DEFAULT_SEED == "12of19"


def cli(args):
    return subprocess.run([CLI] + args, capture_output=True, text=True, timeout=120)


def test_cli_seed_options(ce, tmp_path):
    r = cli(["--help"])
    assert r.returncode == 0 and "--seed" in r.stderr and "--max-word-count=N" in r.stderr
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    for bad in sp.BAD_PATTERNS + ["match01", "half12"]:
        r = cli(["--seed=" + bad, str(fa), str(fa)])
        assert r.returncode == 1 and "seed must be 12of19, 14of22, match<N>" in r.stderr and r.stdout == "", (bad, r.stderr)
    for value in ("", "a", "-1", "1.5", "5x", "9223372036854775808"):
        r = cli(["--max-word-count=" + value, str(fa), str(fa)])
        assert r.returncode == 1 and "max-word-count takes an integer in [0, 9223372036854775807]" in r.stderr and r.stdout == "", value
    # good values parse, with and without --no-transition; the files are looked at next
    for good in sp.PATTERNS:
        for extra in ([], ["--no-transition"], ["--max-word-count=0"], ["--max-word-count", "9223372036854775807"]):
            r = cli(["--seed", good] + extra + [str(fa), str(tmp_path / "missing.fa")])
            assert r.returncode == 1 and "cannot open" in r.stderr, (good, extra, r.stderr)


def test_cli_seed_without_gpu_fails_loudly(ce, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    fa = tmp_path / "a.fa"
    fa.write_text(">a\nACGTACGTACGTACGTACGTAC\n")
    r = cli(["--seed=14of22", "--max-word-count=3", str(fa), str(fa)])
    assert r.returncode != 0 and r.stdout == "" and "CUDA device" in r.stderr
