"""Every block-matching kernel instantiation against the float64 brute force (tests/bm_reference.py), bit for bit on all
three channels, with the kernels that ran observed through torch.profiler: each case must run exactly the hot
instantiation the restated dispatch predicts, its merge pass exactly when the geometry splits the disparity range (J > 1,
nchunks > 1), and K1 screen's seeding k1_fast pass exactly when the raster is large enough for it."""
import numpy as np
import pytest

from bm_reference import CASES, VIEW_CASES, brute_calc_disparity, float_raster, view_expect
from kernel_trace import inst_key, trace  # noqa: F401  (trace: the profiler fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device"
    return v


def _assert_same(got, ref, what):
    assert got.shape == ref.shape, what
    bad = ~np.all(got == ref, axis=-1)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} pixels differ, first at {np.argwhere(bad)[0]}"


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_kernel_matrix(vwb, trace, monkeypatch, case):
    left, right = case.inputs()
    exp = case.expect()
    if case.zone_int:
        monkeypatch.setenv("VWB200_K1_ZONE_INT", "1")
    got = trace.run(lambda: vwb.calc_disparity(case.cost, left, right, case.search, case.kernel))
    _assert_same(got, brute_calc_disparity(case.cost, left, right, case.search, case.kernel), case.id)
    want_hot = {inst_key(exp.family, exp.args)} | ({inst_key("k1_fast_abs_kernel", exp.seed)} if exp.seed else set())
    assert trace.hot() == want_hot, f"{case.id}: ran {sorted(trace.hot())}, expected {sorted(want_hot)} ({exp.geom})"
    want_merge = ([inst_key(*exp.merge)] if exp.merge else []) + ([inst_key("k1_fast_merge_kernel", ())] if exp.seed_merge else [])
    assert sorted(trace.merges()) == sorted(want_merge), f"{case.id}: merges {trace.merges()}, expected {want_merge} ({exp.geom})"


@pytest.mark.parametrize("case", VIEW_CASES, ids=[c[0] for c in VIEW_CASES])
def test_view_clamped_generic(vwb, oracle, trace, case):
    """a single-level view on float imagery with the consistency check on: the right-to-left zone reads left of the raster
    and its split search cannot be staged, so the generic kernel runs clamped and unstaged (bm_reference.VIEW_CASES)"""
    what, cost, (W, H), search, kernel = case
    m, shift = 40, (37, 1)
    base = float_raster(H + 2 * m, W + 2 * m, seed=950 + cost)
    left = np.ascontiguousarray(base[m:m + H, m:m + W], np.float32)
    right = np.ascontiguousarray(base[m - shift[1]:m - shift[1] + H, m - shift[0]:m - shift[0] + W], np.float32)
    mask = np.full((H, W), 255, np.uint8)
    got = trace.run(lambda: vwb.pyramid_correlate(left, right, mask, mask, vwb.PREFILTER_NONE, 0.0, search, kernel, cost, 0, 0.0,
                                                  2.0, 0, 0, 0).rasterize())
    p = oracle.make_params(search, kernel, cost=cost, consistency_threshold=2.0, filter_half_kernel=0, max_pyramid_levels=0)
    ref = oracle.pyramid_correlate(p, left, right, mask, mask)
    _assert_same(got, ref, what)
    exp = view_expect(cost)
    assert inst_key(exp.family, exp.args) in trace.hot(), f"{what}: ran {sorted(trace.hot())}"
    assert {k[0] for k in trace.hot()} == {"k1_generic_kernel"} and {k[1][0] for k in trace.hot()} == {cost}, what
    assert (ref[..., 2] == 1).mean() > 0.5
