"""GPU: how many windows a POA batch holds. For a grid of batch shapes that reaches every branch of the sizing (16/32-bit scores
and indices, full / static / adaptive band, both traceback modes with 8- and 16-bit trace, consensus and MSA, SPOA_ACCURATE, each
of the three window kernels) this pins the bytes one window needs, `max_poas` at fixed budgets, the score pool left over after the
device block is carved, and the smallest caller block that `gwb200_poa_batch_create_in_block` accepts. These numbers decide
`batch_capacity_windows` in bench.py and how get_multi_batch_sizes bins windows, so a change to the arena layout shows here.
Recorded on an NVIDIA H100 80GB HBM3; every number except estimate_max_poas's is independent of the card's free memory."""
import ctypes as C
import re

import pytest
import torch

from genomeworks_b200 import cudapoa
from genomeworks_b200._lib import PoaConfig, check, lib

pytestmark = pytest.mark.gpu

MIB = 1 << 20
BUDGET = 512 * MIB

# name -> (make_config arguments, (gap, mismatch, match))
SHAPES = {
    "static256_1k": (dict(max_sequence_size=1024, max_sequences_per_poa=32, band_width=256, band_mode="static_band"), (-8, -6, 8)),
    "static256_1k_match40": (dict(max_sequence_size=1024, max_sequences_per_poa=32, band_width=256, band_mode="static_band"), (-8, -6, 40)),
    "full_1k": (dict(max_sequence_size=1024, max_sequences_per_poa=32, band_width=256, band_mode="full_band"), (-8, -6, 8)),
    "adaptive_10k_f3": (dict(max_sequence_size=10240, max_sequences_per_poa=32, band_width=256, band_mode="adaptive_band",
                             adaptive_storage_factor=3.0), (-8, -6, 8)),
    "adaptive_12k": (dict(max_sequence_size=12000, max_sequences_per_poa=32, band_width=256, band_mode="adaptive_band"), (-8, -6, 8)),
    "static2048_4k": (dict(max_sequence_size=4096, max_sequences_per_poa=32, band_width=2048, band_mode="static_band"), (-8, -6, 8)),
    "static_tb_pd100": (dict(max_sequence_size=1024, max_sequences_per_poa=32, band_width=256, band_mode="static_band_traceback",
                             max_pred_dist=100), (-8, -6, 8)),
    "adaptive_tb": (dict(max_sequence_size=1024, max_sequences_per_poa=32, band_width=256, band_mode="adaptive_band_traceback"), (-8, -6, 8)),
}

# each shape as consensus and as MSA, and two of them again with SPOA_ACCURATE on
CASES = ["%s/%s" % (s, o) for s in SHAPES for o in ("consensus", "msa")] + ["static256_1k/consensus/accurate", "full_1k/consensus/accurate"]

# case -> (per-window bytes N, max_poas at 512 MiB, score bytes, kernel: 0 traceback-mode, 1 v3, 2 first-generation)
EXPECTED = {
    "static256_1k/consensus": (3064148, 175, 2, 1),
    "static256_1k/msa": (3232116, 166, 2, 1),
    "static256_1k_match40/consensus": (4686164, 114, 4, 1),
    "static256_1k_match40/msa": (4854132, 110, 4, 1),
    "full_1k/consensus": (7733588, 69, 2, 1),
    "full_1k/msa": (7901556, 67, 2, 1),
    "adaptive_10k_f3/consensus": (111656276, 4, 4, 1),
    "adaptive_10k_f3/msa": (113335668, 4, 4, 1),
    "adaptive_12k/consensus": (104061636, 5, 4, 1),
    "adaptive_12k/msa": (107157700, 5, 4, 1),
    "static2048_4k/consensus": (106796372, 5, 4, 2),
    "static2048_4k/msa": (107468148, 4, 4, 2),
    "static_tb_pd100/consensus": (2306196, 232, 2, 0),
    "static_tb_pd100/msa": (2474164, 216, 2, 0),
    "adaptive_tb/consensus": (5227092, 102, 2, 0),
    "adaptive_tb/msa": (5395060, 99, 2, 0),
    "static256_1k/consensus/accurate": (3094900, 173, 2, 1),
    "full_1k/consensus/accurate": (7764340, 69, 2, 1),
}


def _split(case):
    parts = case.split("/")
    return parts[0], parts[1], len(parts) > 2


@pytest.fixture
def spoa_accurate(request):
    """Sets the library-wide SPOA_ACCURATE switch for one case and restores what it was."""
    before = lib().gwb200_poa_get_spoa_accurate()
    lib().gwb200_poa_set_spoa_accurate(C.c_int32(1 if _split(request.param)[2] else 0))
    yield request.param
    lib().gwb200_poa_set_spoa_accurate(C.c_int32(before))


def _config(shape):
    return cudapoa.make_config(**SHAPES[shape][0])


def _batch(shape, output, max_gpu_mem):
    gap, mismatch, match = SHAPES[shape][1]
    cfg = _config(shape)
    return cudapoa.CudaPoaBatch(cfg.max_sequences_per_poa, cfg.max_sequence_size, max_gpu_mem, output_type=output, gap_score=gap,
                                mismatch_score=mismatch, match_score=match, config=cfg)


def _required_bytes(shape, output, max_gpu_mem):
    with pytest.raises(RuntimeError, match="Requires at least") as e:
        _batch(shape, output, max_gpu_mem)
    return int(re.search(r"Requires at least (\d+) bytes", str(e.value)).group(1))


@pytest.mark.parametrize("spoa_accurate", CASES, indirect=True)
def test_window_bytes_and_max_poas(spoa_accurate):
    shape, output, _ = _split(spoa_accurate)
    n_bytes, max_poas, score_bytes, kernel = EXPECTED[spoa_accurate]
    assert _required_bytes(shape, output, 0) == n_bytes
    b = _batch(shape, output, BUDGET)
    assert (b.max_poas, b.score_bytes, b.kernel) == (max_poas, score_bytes, kernel)
    b.close()
    b = _batch(shape, output, n_bytes)
    assert b.max_poas == 1
    b.close()
    if SHAPES[shape][0]["band_mode"] == "full_band":
        # full band admits a window without its score matrix: the scores of a window are sized by its longest read
        b = _batch(shape, output, n_bytes - 1)
        assert b.max_poas == 1
        b.close()
    else:
        assert _required_bytes(shape, output, n_bytes - 1) == n_bytes


# shape -> (read length, one-read groups accepted at 512 MiB). Full band sizes a window's scores by its longest read, and a read of
# max_sequence_size needs a little more than the matrix the batch reserved per window, so the pool runs out before max_poas (69).
# A banded window takes one matrix of the pool, so there max_poas is the limit.
POOL = {
    "full_1k": (1024, 68),
    "static256_1k": (1024, 175),
}


@pytest.mark.parametrize("shape", list(POOL))
def test_score_pool_admits(shape):
    length, accepted = POOL[shape]
    b = _batch(shape, "consensus", BUDGET)
    read = "ACGT" * (length // 4)
    n = 0
    while n <= b.max_poas:
        status, _ = b.add_poa_group([read])
        if status == cudapoa.exceeded_maximum_poas:
            break
        assert status == cudapoa.success
        n += 1
    b.close()
    assert n == accepted


def _create_in_block(shape, block_bytes):
    L = lib()
    L.gwb200_poa_batch_create_in_block.argtypes = [C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int8,
                                                   C.POINTER(PoaConfig), C.c_int16, C.c_int16, C.c_int16]
    gap, mismatch, match = SHAPES[shape][1]
    cfg = _config(shape)
    block = torch.empty(block_bytes, dtype=torch.uint8, device="cuda")
    h = C.c_void_p()
    try:
        check(L.gwb200_poa_batch_create_in_block(C.byref(h), 0, None, C.c_void_p(block.data_ptr()), block_bytes,
                                                 cudapoa.OUTPUT_TYPES["consensus"], C.byref(cfg), gap, mismatch, match))
        return L.gwb200_poa_batch_max_poas(h)
    finally:
        if h.value:
            L.gwb200_poa_batch_destroy(h)


# shape -> (smallest block accepted, a larger block, max_poas in the larger block)
IN_BLOCK = {
    "static256_1k": (3088724, 12356560, 4),
    "full_1k": (7758164, 31034320, 4),
}


@pytest.mark.parametrize("shape", list(IN_BLOCK))
def test_create_in_block(shape):
    smallest, larger, max_poas = IN_BLOCK[shape]
    assert _create_in_block(shape, smallest) == 1
    with pytest.raises(RuntimeError, match="Requires at least"):
        _create_in_block(shape, smallest - 1)
    assert _create_in_block(shape, larger) == max_poas


@pytest.mark.parametrize("spoa_accurate", CASES, indirect=True)
def test_estimate_max_poas(spoa_accurate):
    """estimate_max_poas reads the free memory of a shared card, so it is checked against its formula: quota x free / N."""
    shape, output, _ = _split(spoa_accurate)
    gap, mismatch, match = SHAPES[shape][1]
    L = lib()
    L.gwb200_poa_estimate_max_poas.argtypes = [C.POINTER(PoaConfig), C.c_int32, C.c_float, C.c_int16, C.c_int16, C.c_int16]
    L.gwb200_poa_estimate_max_poas.restype = C.c_int64
    cfg = _config(shape)
    quota = 0.5
    free_b, _ = torch.cuda.mem_get_info()
    got = L.gwb200_poa_estimate_max_poas(C.byref(cfg), 1 if output == "msa" else 0, quota, mismatch, gap, match)
    want = int(quota * free_b) // EXPECTED[spoa_accurate][0]
    assert got == pytest.approx(want, rel=0.01)
