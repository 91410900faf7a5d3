"""The gapped extender on the GPU against the CPU oracle: records, CIGARs, has_cigar and the live-cell count."""
import os
import subprocess

import numpy as np
import pytest

import extender_libs as xl
import gapped_extender_libs as gl
from checker_lib import CountingAllocator

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LASTZ = (gl.LASTZ_OPEN, gl.LASTZ_EXTEND, gl.LASTZ_YDROP)


@pytest.fixture(scope="module")
def ce():
    import __graft_entry__ as g
    g.build()
    from genomeworks_b200 import cudaextender
    return cudaextender


def run_engine(ce, query, target, matrix, o, e, y, threshold, anchors, budget=1 << 30, ext=None, **kw):
    x = ext or ce.create_gapped_extender(matrix, o, e, y, budget, **kw)
    assert x.extend_async(query, target, threshold, anchors) == ce.success
    assert x.sync() == ce.success
    rec, cig = x.get_alignments()
    live = x.last_live_cells()
    if ext is None:
        x.close()
    return rec, cig, live


def assert_equal(got, want):
    assert gl.rows(got[0]) == gl.rows(want[0])
    assert got[1] == want[1]
    assert got[2] == want[2]


def sample_anchors():
    seq, _, golden = xl.sample()
    return seq, gl.ssp_anchors(golden), golden["query"] == golden["target"]


def test_golden_sample_anchors_against_the_oracle(ce):
    seq, a, diag0 = sample_anchors()
    assert diag0.sum() == 1035 and (~diag0).sum() == 302
    for part in (a[~diag0], a[diag0]):
        want = gl.oracle_run(seq, seq, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, part)
        got = run_engine(ce, seq, seq, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, part)
        assert len(want[0]) > 0
        assert_equal(got, want)


@pytest.mark.parametrize("n", [0, 1, 7, 1001])
@pytest.mark.parametrize("divergence", [0.0, 0.15, 0.3])
def test_synthetic_anchors_against_the_oracle(ce, n, divergence):
    from genomeworks_b200 import synth
    target, query, seeds = synth.extender_workload(5000, divergence, n, 0.3, seed=100 + n)
    for matrix, o, e, y, threshold in ((xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD), (xl.SIMPLE_MATRIX, 5, 2, 80, 0)):
        want = gl.oracle_run(query, target, matrix, o, e, y, threshold, seeds)
        assert_equal(run_engine(ce, query, target, matrix, o, e, y, threshold, seeds), want)


def test_range_wider_than_the_shared_ring(ce):
    # small gap extension and a large y-drop keep thousands of cells of every anti-diagonal live
    rng = np.random.default_rng(8)
    s = rng.integers(0, 4, 6000).astype(np.int8)
    q = s.copy()
    q[rng.random(6000) < 0.1] = 4
    a = np.array([(0, 0), (3000, 3000), (5999, 5999)], dtype=gl.ANCHOR_DTYPE)
    want = gl.oracle_run(q, s, xl.SIMPLE_MATRIX, 1, 0, 3000, -(1 << 40), a)
    # about 6000 x 6000 live cells per anchor: ranges of thousands of cells
    assert want[2] > 10 ** 7
    assert_equal(run_engine(ce, q, s, xl.SIMPLE_MATRIX, 1, 0, 3000, -(1 << 40), a), want)


def test_side_of_about_one_megabase(ce):
    from genomeworks_b200 import synth
    target, query, _ = synth.extender_workload(1 << 20, 0.02, 0, 0.0, seed=9)
    a = np.array([(0, 0)], dtype=gl.ANCHOR_DTYPE)
    want = gl.oracle_run(query, target, xl.SAMPLE_MATRIX, *LASTZ, 0, a)
    assert int(want[0]["query_end"][0]) > 900000
    assert_equal(run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, 0, a), want)


def test_score_past_2_31(ce):
    mat = np.full(64, -(1 << 20), dtype=np.int32)
    mat[::9] = 1 << 20
    s = np.random.default_rng(3).integers(0, 4, 4096).astype(np.int8)
    a = np.array([(2048, 2048)], dtype=gl.ANCHOR_DTYPE)
    want = gl.oracle_run(s, s, mat, *LASTZ, 1 << 31, a)
    got = run_engine(ce, s, s, mat, *LASTZ, 1 << 31, a)
    assert int(got[0]["score"][0]) == 4096 << 20 and got[1] == ["4096M"]
    assert_equal(got, want)


def test_many_rounds_equal_one_round(ce):
    target, query, seeds = gl.synthetic()
    one = run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds)
    # the largest alignment's storage: every round holds one or two alignments
    sizes = [gl.oracle_side(query, target, xl.SAMPLE_MATRIX, *LASTZ, int(s["query"]), int(s["target"]), side, trace=False)["storage"]
             for s in seeds[one[0]["anchor"]] for side in (True, False)]
    budget = max(a + b for a, b in zip(sizes[::2], sizes[1::2]))
    many = run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds, budget=budget)
    assert_equal(many, one)
    assert all(int(h) == 1 for h in many[0]["has_cigar"])
    assert_equal(many, gl.oracle_run(query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds, budget))


def test_budget_below_one_alignment_gives_exact_intervals_without_cigar(ce):
    # the golden sample's off-diagonal anchors: alignments of many sizes; a budget between the smallest and the largest
    seq, a, diag0 = sample_anchors()
    a = a[~diag0]
    full = gl.oracle_run(seq, seq, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, a)
    sizes = sorted(sum(gl.oracle_side(seq, seq, xl.SAMPLE_MATRIX, *LASTZ, int(a[k]["query"]), int(a[k]["target"]), side,
                                      trace=False)["storage"] for side in (True, False)) for k in full[0]["anchor"])
    budget = sizes[len(sizes) // 2]
    want = gl.oracle_run(seq, seq, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, a, budget)
    assert 0 < int((want[0]["has_cigar"] == 0).sum()) < len(want[0])
    # the same alignments, scores and intervals as with room for every CIGAR
    assert [r[:2] + r[3:] for r in gl.rows(want[0])] == [r[:2] + r[3:] for r in gl.rows(full[0])]
    assert_equal(run_engine(ce, seq, seq, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, a, budget=budget), want)


def test_device_pointer_api_equals_the_host_api(ce):
    import torch
    target, query, seeds = gl.synthetic(400, 23)
    ext = ce.create_extender(xl.SAMPLE_MATRIX, xl.SAMPLE_XDROP)
    dq = torch.from_numpy(query).cuda()
    dt = torch.from_numpy(target).cuda()
    ds = torch.from_numpy(np.stack([seeds["query"], seeds["target"]], 1).astype(np.int32)).cuda()
    dout = torch.zeros((len(seeds), 4), dtype=torch.int32, device="cuda")
    dn = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert ext.extend_async_device(dq, dt, 1500, ds, dout, dn) == ce.success
    torch.cuda.synchronize()
    n = int(dn.item())
    ssps = dout[:n].cpu().numpy()
    assert n > 0
    g = ce.create_gapped_extender(xl.SAMPLE_MATRIX, *LASTZ)
    assert g.extend_ssps_device(dq, dt, gl.LASTZ_THRESHOLD, dout, n) == ce.success and g.sync() == ce.success
    got = g.get_alignments() + (g.last_live_cells(),)
    a = gl.ssp_anchors(np.ascontiguousarray(ssps).view(xl.SSP_DTYPE).reshape(-1))
    assert_equal(got, run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, a))
    # an anchor outside the sequences is invalid_input at sync
    bad = dout[:1].clone()
    bad[0, 0] = len(query)
    assert g.extend_ssps_device(dq, dt, 0, bad, 1) == ce.success and g.sync() == ce.invalid_input
    ext.close()
    g.close()


def test_reused_extender_equals_fresh_ones_and_a_stream(ce):
    import torch
    cases = [gl.synthetic(200, s) for s in (31, 32, 33)]
    ext = ce.create_gapped_extender(xl.SAMPLE_MATRIX, *LASTZ)
    stream = torch.cuda.Stream()
    on_stream = ce.create_gapped_extender(xl.SAMPLE_MATRIX, *LASTZ, stream=stream)
    for target, query, seeds in cases + cases[:1]:
        fresh = run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds)
        assert_equal(run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds, ext=ext), fresh)
        assert_equal(run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds, ext=on_stream), fresh)
    p1, p2 = ext.last_pass_ms()
    assert p1 > 0 and p2 > 0
    ext.close()
    on_stream.close()


def test_allocator_balance(ce):
    target, query, seeds = gl.synthetic(200, 41)
    alloc = CountingAllocator()
    ext = ce.create_gapped_extender(xl.SAMPLE_MATRIX, *LASTZ, allocator=alloc)
    got = run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds, ext=ext)
    assert alloc.calls > 0 and len(alloc.live) > 0
    ext.close()
    assert alloc.live == {}
    assert_equal(got, run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds))


def test_cpp_program_agrees_with_python(ce, tmp_path):
    exe = os.path.join(ROOT, "build", "test_cpp_gapped_extender")
    target, query, seeds = gl.synthetic(150, 51)
    query.tofile(tmp_path / "q.bin")
    target.tofile(tmp_path / "t.bin")
    seeds.tofile(tmp_path / "a.bin")
    out = subprocess.run([exe, str(tmp_path / "q.bin"), str(tmp_path / "t.bin"), str(tmp_path / "a.bin")], capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 0 and "CPP_GAPPED_OK" in out.stdout, out.stdout + out.stderr
    rec, cig, _ = run_engine(ce, query, target, xl.SAMPLE_MATRIX, *LASTZ, gl.LASTZ_THRESHOLD, seeds)
    lines = [l for l in out.stdout.splitlines() if l.startswith("ALN ")]
    assert lines == ["ALN %d %d %d %d %d %d %d %s" % (r["score"], r["anchor"], r["has_cigar"], r["query_begin"], r["query_end"],
                                                    r["target_begin"], r["target_end"], c) for r, c in zip(rec, cig)]
