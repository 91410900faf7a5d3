"""The gapped extender's public surface without a GPU: every argument check of the C ABI and of Python happens before any
device work, and the C++ header compiles."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import extender_libs as xl
import gapped_extender_libs as gl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_INPUT, INVALID_OPERATION = 2, 1


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200._lib import lib
    return lib()


def create(L, mat=None, dim=64, o=400, e=30, y=9400, budget=1 << 20):
    m = np.ascontiguousarray(xl.SIMPLE_MATRIX if mat is None else mat, dtype=np.int32)
    h = C.c_void_p()
    rc = L.gwb200_gapped_extender_create(C.byref(h), m.ctypes.data_as(C.c_void_p), dim, o, e, y, budget, None, 0)
    return rc, h


@pytest.mark.parametrize("kw", [dict(dim=63), dict(o=-1), dict(o=(1 << 24) + 1), dict(e=-1), dict(e=(1 << 24) + 1), dict(y=-1),
                                dict(y=(1 << 28) + 1), dict(budget=-1)])
def test_create_rejects_parameters_out_of_range(L, kw):
    assert create(L, **kw)[0] == INVALID_INPUT


@pytest.mark.parametrize("v", [-(1 << 24) - 1, (1 << 24) + 1])
def test_create_rejects_matrix_entries_out_of_range(L, v):
    m = xl.SIMPLE_MATRIX.copy()
    m[9] = v
    assert create(L, mat=m)[0] == INVALID_INPUT


def test_create_rejects_a_null_matrix_and_a_null_handle(L):
    h = C.c_void_p()
    assert L.gwb200_gapped_extender_create(C.byref(h), None, 64, 1, 1, 1, 0, None, 0) == INVALID_INPUT
    m = np.ascontiguousarray(xl.SIMPLE_MATRIX)
    assert L.gwb200_gapped_extender_create(None, m.ctypes.data_as(C.c_void_p), 64, 1, 1, 1, 0, None, 0) == -1


def test_create_at_the_range_limits_gets_past_the_checks(L):
    m = np.full(64, 1 << 24, dtype=np.int32)
    m[::2] = -(1 << 24)
    rc, h = create(L, mat=m, o=1 << 24, e=1 << 24, y=1 << 28, budget=0)
    if rc == 0:  # on a machine with a device
        L.gwb200_gapped_extender_destroy(h)
    else:
        assert rc == -3  # no device: GWB200_E_CUDA


def test_extend_checks_the_input_before_the_handle(L):
    q = np.zeros(10, dtype=np.int8)
    t = np.zeros(8, dtype=np.int8)

    def ext(qlen=10, tlen=8, anchors=((0, 0),), qp=q, tp=t, n=None):
        a = np.array([tuple(x) for x in anchors], dtype=gl.ANCHOR_DTYPE)
        return L.gwb200_gapped_extender_extend_host(None, qp.ctypes.data_as(C.c_void_p) if qp is not None else None, qlen,
                                                    tp.ctypes.data_as(C.c_void_p) if tp is not None else None, tlen, 0,
                                                    a.ctypes.data_as(C.c_void_p), len(a) if n is None else n)
    assert ext(qlen=-1) == INVALID_INPUT
    assert ext(tlen=-1) == INVALID_INPUT
    assert ext(n=-1) == INVALID_INPUT
    assert ext(qp=None) == INVALID_INPUT
    assert ext(tp=None) == INVALID_INPUT
    assert ext(anchors=((10, 0),)) == INVALID_INPUT
    assert ext(anchors=((0, 8),)) == INVALID_INPUT
    assert ext(anchors=((9, 7), (0, 0xffffffff))) == INVALID_INPUT
    assert ext(anchors=((9, 7),)) == -1  # valid input, null handle
    assert L.gwb200_gapped_extender_extend_ssps_device(None, None, 10, None, 8, 0, None, 0) == INVALID_INPUT
    assert L.gwb200_gapped_extender_extend_ssps_device(None, q.ctypes.data_as(C.c_void_p), -1, t.ctypes.data_as(C.c_void_p), 8, 0,
                                                       None, 0) == INVALID_INPUT
    assert L.gwb200_gapped_extender_extend_ssps_device(None, q.ctypes.data_as(C.c_void_p), 10, t.ctypes.data_as(C.c_void_p), 8, 0,
                                                       None, 3) == INVALID_INPUT


def test_null_handle_calls(L):
    assert L.gwb200_gapped_extender_sync(None) == -1
    assert L.gwb200_gapped_extender_num_results(None) == -1
    assert L.gwb200_gapped_extender_get_results(None, None, 0) == -1
    assert L.gwb200_gapped_extender_cigar_bytes(None) == -1
    assert L.gwb200_gapped_extender_get_cigars(None, None, 0, None) == -1
    assert L.gwb200_gapped_extender_reset(None) == -1
    assert L.gwb200_gapped_extender_last_live_cells(None) == -1
    p1, p2 = C.c_float(), C.c_float()
    assert L.gwb200_gapped_extender_last_ms(None, C.byref(p1), C.byref(p2)) == -1
    L.gwb200_gapped_extender_destroy(None)


@pytest.mark.parametrize("kw", [dict(gap_open=-1), dict(gap_extend=1 << 25), dict(ydrop=-5), dict(ydrop=(1 << 28) + 1),
                                dict(budget_bytes=-1), dict(score_matrix=np.zeros(63, dtype=np.int32)),
                                dict(score_matrix=np.full(64, 1 << 25, dtype=np.int64))])
def test_python_rejects_parameters_before_any_device_work(L, kw):
    from genomeworks_b200 import cudaextender as ce
    args = dict(score_matrix=xl.SIMPLE_MATRIX, gap_open=400, gap_extend=30, ydrop=9400)
    args.update(kw)
    with pytest.raises(ValueError):
        ce.create_gapped_extender(**args)


def test_python_without_a_device_raises(L):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    from genomeworks_b200 import cudaextender as ce
    with pytest.raises(RuntimeError):
        ce.create_gapped_extender(xl.SIMPLE_MATRIX, 400, 30, 9400)


def test_header_compiles_warning_free_as_cpp14(tmp_path):
    tu = tmp_path / "tu.cpp"
    tu.write_text("#include <claraparabricks/genomeworks/cudaextender/gapped_extender.hpp>\n"
                  "static_assert(sizeof(gwb200_gapped_alignment) == 32, \"record layout\");\n"
                  "int main() { return 0; }\n")
    r = subprocess.run(["g++", "-std=c++14", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-I",
                        "/usr/local/cuda/include", str(tu)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
