"""K1 fast periods: the 12 warps of a CTA run the (dy, octet) passes of a period of up to sd = 3 dy rows, dealt to them
statically, with one barrier per period and the next period's right rows prefetched into a ring.  Partial periods,
fewer work units than warps, partial octets and the largest ring must stay bit-identical to the oracle, and so must
ties between warps that work on different dy of one period (the first disparity in raster order wins)."""
import numpy as np
import pytest

from kernel_trace import inst_key, trace  # noqa: F401  (trace: the profiler fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vwb():
    import visionworkbench_b200 as v
    assert v.device_count() > 0, "GPU tests need a CUDA device"
    return v


def _check(vwb, oracle, trace, cost, left, right, search, kernel, what):
    got = trace.run(lambda: vwb.calc_disparity(cost, left, right, search, kernel))
    assert vwb.last_k1_stats()["path"] == "exact-int", what
    assert inst_key("k1_fast_abs_kernel", (kernel[0], cost == 1)) in trace.hot(), f"{what}: ran {sorted(trace.hot())}"
    ref = oracle.calc_disparity(cost, left, right, search, kernel)
    assert got.shape == ref.shape, what
    bad = ~np.all(got == ref, axis=-1)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} pixels differ, first at {np.argwhere(bad)[0]}"
    return ref


@pytest.mark.parametrize("shape", [
    ((120, 60), (64, 1), (7, 7)),          # one dy: a one-row ring period
    ((120, 60), (64, 2), (7, 7)),          # two dy: periods of 2
    ((120, 60), (64, 4), (7, 7)),          # a full period of 3, then a period of 1
    ((120, 60), (64, 5), (7, 7)),          # a full period of 3, then a period of 2
    ((300, 70), (16, 41), (7, 7)),         # J = 5 dy chunks of 9 rows and a last one of 5: every chunk ends in a partial period
    ((300, 40), (8, 16), (5, 5)),          # one octet: 3 work units per period for 12 warps (J = 2)
    ((250, 40), (77, 5), (9, 5)),          # partial last octet (octet 9 of 10)
    ((100, 80), (512, 8), (3, 41)),        # widest search and tallest kernel: the largest ring, wrapped several times
])
def test_fast_periods_match_oracle(vwb, oracle, trace, shape):
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=17 + W + H + search[1])
    _check(vwb, oracle, trace, 0, left, right, search, kernel, f"abs {shape}")


@pytest.mark.parametrize("shape", [((300, 90), (40, 7), (9, 9)), ((120, 60), (64, 5), (7, 7))])
def test_fast_periods_squared(vwb, oracle, trace, shape):
    """SquaredCost (the SQ variant of the kernel) on the same periods"""
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=29 + W + H)
    _check(vwb, oracle, trace, 1, left, right, search, kernel, f"sq {shape}")


def test_fast_periods_ties_across_dy(vwb, oracle, trace):
    """Imagery constant along y: every dy of a period has the same cost at every dx, so the warps that run dy 0, 1, 2 of
    the first period offer equal costs, and dy 0 (the first in raster order) must win however they are timed."""
    rng = np.random.default_rng(43)
    W, H, (sx, sy), (kx, ky) = 280, 70, (32, 7), (7, 5)
    row = np.floor(rng.random(W + kx - 1 + sx - 1) * 8).astype(np.float32)
    right = np.ascontiguousarray(np.broadcast_to(row, (H + ky - 1 + sy - 1, row.size)))
    left = np.ascontiguousarray(right[:H + ky - 1, 5:5 + W + kx - 1])
    ref = _check(vwb, oracle, trace, 0, left, right, (sx, sy), (kx, ky), "stripes")
    valid = ref[..., 2] == 1
    assert valid.any() and (ref[..., 1][valid] == 0).all()


def test_fast_periods_constant(vwb, oracle, trace):
    """Constant imagery: every disparity has the same cost, so every pixel is invalid (the all-equal fix-up)"""
    W, H, (sx, sy), (kx, ky) = 260, 50, (24, 9), (5, 5)
    left = np.full((H + ky - 1, W + kx - 1), 7.0, np.float32)
    right = np.full((H + ky - 1 + sy - 1, W + kx - 1 + sx - 1), 7.0, np.float32)
    ref = _check(vwb, oracle, trace, 0, left, right, (sx, sy), (kx, ky), "constant")
    assert (ref[..., 2] == 0).all()
