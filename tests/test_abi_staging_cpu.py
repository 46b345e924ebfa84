"""The C ABI entry points that take `on_device`, without a GPU: each refuses an invalid call with its error code before it
looks for a device, and a valid call fails with VWB200_ENODEVICE when there is none."""
import ctypes as C

import numpy as np
import pytest

EARG, ENODEVICE = -1, -6


@pytest.fixture(scope="module")
def L():
    from visionworkbench_b200 import build
    build.build()
    import visionworkbench_b200 as v
    return v.lib()


def sgm_params():
    import visionworkbench_b200 as v
    return v.api._sgm_params((8, 8), 5, subpixel_mode=2)


def calls(L, f, d, u8, i32, bad):
    """one call per entry point; `bad` makes each one invalid"""
    n = 0 if bad else 8
    ow, oh = C.c_int(0), C.c_int(0)
    sp = sgm_params()
    return {
        "calc_disparity": lambda: L.vwb200_calc_disparity(0, f, 8, 8, 8, f, 8, 8, 8, 1, 1, 3 + bad, 3, i32, 8, 0, None),
        "pyramid_down": lambda: L.vwb200_pyramid_down(f, n, 8, 8, f, 8, 0, None),
        "prefilter": lambda: L.vwb200_prefilter(f, n, 8, 8, 1, C.c_float(1.4), f, 8, 0, None),
        "subsample_mask_by_two": lambda: L.vwb200_subsample_mask_by_two(u8, n, 8, 8, u8, 8, 0, None),
        "sgm_calc_disparity": lambda: L.vwb200_sgm_calc_disparity(f, 20, 20, 20, f, 28, 28, 28, 8, 8, 5 - bad, 0, 0, i32, 16,
                                                                  C.byref(ow), C.byref(oh), 0, None),
        "sgm_calc_disparity_subpixel": lambda: L.vwb200_sgm_calc_disparity_subpixel(f, 20, 20, 20, f, 28, 28, 28, 8, 8, 5, 0, 0, 2 + 9 * bad, i32,
                                                                                    16, f, 16, C.byref(ow), C.byref(oh), 0, None),
        "sgm_calc_disparity_ex": lambda: L.vwb200_sgm_calc_disparity_ex(C.byref(sp), f, 20, 20, 20, f, 28, 28, 28, None, 0, None, 0, 0, 0, None, 0, 0,
                                                                        0, None, i32, 16 - 8 * bad, f, 16, None, C.byref(ow), C.byref(oh), 0, None),
        "sgm_disp_bounds": lambda: L.vwb200_sgm_disp_bounds(C.byref(sp), None, 0, 0, 0, None, 0, None, 0, 0, 0, n, 8, i32, 0, None),
        "parabola_subpixel": lambda: L.vwb200_parabola_subpixel(d, 8, 8, f, 8, f, 8, 8, 8, 3, 3, 0, C.c_float(0), 0, 0, 8 + bad, 8, d, 8, 0, None),
        "disparity_median_filter": lambda: L.vwb200_disparity_median_filter(d, 8, 8, 8 - bad, 3, 0, None),
        "texture_measure": lambda: L.vwb200_texture_measure(f, 8, 8, 8, 3 - 3 * bad, C.c_double(0.5), C.c_double(0.5), f, 8, 0, None),
        "texture_preserving_disparity_filter": lambda: L.vwb200_texture_preserving_disparity_filter(d, 8, 8, 8, f, 8 - bad, C.c_float(0.15), 11, 0,
                                                                                                    None),
        "cross_corr_consistency_check": lambda: L.vwb200_cross_corr_consistency_check(i32, 8, 8, 8, None if bad else i32, 8, 8, 8, C.c_float(1), 0,
                                                                                      None),
        "rm_outliers_using_thresh": lambda: L.vwb200_rm_outliers_using_thresh(i32, n, 8, 1, 1, C.c_double(3), C.c_double(0.5), i32, 0, None),
        "disparity_cleanup_using_thresh": lambda: L.vwb200_disparity_cleanup_using_thresh(i32, n, 8, 1, 1, C.c_double(3), C.c_double(0.5), i32, 0,
                                                                                          None),
        "disparity_mask": lambda: L.vwb200_disparity_mask(i32, 8, 8, None if bad else u8, u8, 8, 8, i32, 0, None),
        "corr_set_inputs": lambda: L.vwb200_corr_set_inputs(None if bad else C.c_void_p(1), f, 8, 8, 8, f, 8, 8, 8, u8, 8, u8, 8, 0),
        "corr_set_lr_disp_diff": lambda: L.vwb200_corr_set_lr_disp_diff(None, f, 8, 8, 8 - 5 * bad, 0),
    }


@pytest.fixture
def buffers():
    f = np.zeros((40, 40), np.float32)
    return f, np.zeros((8, 8, 3), np.float32), np.full((40, 40), 255, np.uint8), np.zeros((40, 40, 4), np.int32)


def test_invalid_calls_are_refused_first(L, buffers):
    f, d, u8, i32 = buffers
    got = {k: fn() for k, fn in calls(L, f.ctypes.data, d.ctypes.data, u8.ctypes.data, i32.ctypes.data, 1).items()}
    assert got == {k: EARG for k in got}


def test_valid_calls_without_a_device(L, buffers):
    import visionworkbench_b200 as v
    if v.device_count() > 0:
        pytest.skip("a CUDA device is present")
    f, d, u8, i32 = buffers
    todo = calls(L, f.ctypes.data, d.ctypes.data, u8.ctypes.data, i32.ctypes.data, 0)
    del todo["corr_set_inputs"], todo["corr_set_lr_disp_diff"]      # need a view handle: covered by test_abi_cpu.py
    got = {k: fn() for k, fn in todo.items()}
    assert got == {k: ENODEVICE for k in got}
