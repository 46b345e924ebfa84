"""K1 fast band geometry: the band height comes from the shared-memory budget and the raster size, the 8 warps of a
CTA sweep disjoint dx octets over the whole band and meet in one shared plane of 64-bit (cost, raster index) keys.
Every case must stay bit-identical to the oracle, ties included (first disparity in raster order wins)."""
import numpy as np
import pytest

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


def _check(vwb, oracle, cost, left, right, search, kernel, what):
    got = vwb.calc_disparity(cost, left, right, search, kernel)
    assert vwb.last_k1_stats()["path"] == "exact-int"
    _assert_same(got, oracle.calc_disparity(cost, left, right, search, kernel), what)


@pytest.mark.parametrize("shape", [
    ((1200, 1500), (8, 8), (3, 3)),        # enough work items for tall bands (58 rows); 1500 is not a multiple of the height
    ((300, 20), (16, 8), (21, 21)),        # H smaller than one band
    ((300, 70), (16, 64), (7, 7)),         # few work items: the dy range is split into chunks (J > 1)
    ((100, 80), (512, 1), (3, 41)),        # widest search and tallest kernel: the largest shared-memory footprint
    ((250, 40), (77, 3), (9, 5)),          # partial last octet, owned by warp 1 (octet 9)
])
def test_fast_band_geometry_matches_oracle(vwb, oracle, shape):
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=3 + W + H)
    _check(vwb, oracle, 0, left, right, search, kernel, f"abs {shape}")


@pytest.mark.parametrize("search", [(72, 4), (64, 3)])
def test_fast_ties_across_warps(vwb, oracle, search):
    """2-bit imagery: exact cost ties between octets that different warps own (sx >= 64 gives every warp an octet, 72
    gives warp 0 two); the lowest raster index must win whichever warp reaches the cost first."""
    rng = np.random.default_rng(91)
    sx, sy = search
    W, H, kx, ky = 280, 70, 7, 7
    right = np.floor(rng.random((H + ky - 1 + sy - 1, W + kx - 1 + sx - 1)) * 4).astype(np.float32)
    right[20:60, 40:200] = 1.0                                                # flat block: all-equal costs
    left = np.ascontiguousarray(right[1:1 + H + ky - 1, 9:9 + W + kx - 1])
    ref = oracle.calc_disparity(0, left, right, search, (kx, ky))
    assert (ref[..., 2] == 0).any() and (ref[..., 2] == 1).any()
    _check(vwb, oracle, 0, left, right, search, (kx, ky), f"ties {search}")


@pytest.mark.parametrize("shape", [((300, 90), (40, 8), (9, 9)), ((1200, 1500), (8, 8), (3, 3)), ((300, 70), (16, 64), (7, 7))])
def test_fast_squared_band_geometry(vwb, oracle, shape):
    """SquaredCost on K1 fast (12-bit imagery, window sums within uint32): same bands, same key plane."""
    from visionworkbench_b200.synth import make_rasters
    (W, H), search, kernel = shape
    left, right = make_rasters(W, H, search, kernel, seed=5 + W + H)
    _check(vwb, oracle, 1, left, right, search, kernel, f"sq {shape}")
