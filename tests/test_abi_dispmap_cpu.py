"""The disparity resampling, range and transform calls without a GPU: every invalid call returns VWB200_EARG (with the
reference's message for a subregion of the wrong size) before the library looks for a device, and a valid call returns
VWB200_ENODEVICE when there is none."""
import ctypes as C

import numpy as np
import pytest

EARG, ENODEVICE = -1, -6


@pytest.fixture(scope="module")
def v():
    from visionworkbench_b200 import build
    build.build()
    import visionworkbench_b200 as v
    return v


def buffers(w=8, h=6, pitch=8):
    return np.zeros((max(h, 1), max(pitch, 1), 3), np.float32), np.zeros((2 * max(h, 1), 2 * max(pitch, 1), 3), np.float32)


def calls(v, pt=1, w=8, h=6, pitch=8, opitch=None, null_in=False, null_out=False, mode=0, matrix=True, box=None, same_buffer=False):
    L = v.lib()
    a, b = buffers(w, h, pitch)
    src = None if null_in else a.ctypes.data
    dst = None if null_out else (a.ctypes.data if same_buffer else b.ctypes.data)
    m = np.eye(3).reshape(9)
    mn, mx = np.zeros(2, np.float32), np.full(2, 9, np.float32)
    r = (C.c_float * 4)()
    sub = (C.c_int32 * 4)(*(box if box is not None else (0, 0, w, h)))
    return {
        "subsample": lambda: L.vwb200_disparity_subsample(pt, src, w, h, pitch, dst, opitch if opitch is not None else max((w + 1) // 2, 1), 0, None),
        "upsample": lambda: L.vwb200_disparity_upsample(pt, src, w, h, pitch, dst, opitch if opitch is not None else 2 * w, 0, None),
        "range": lambda: L.vwb200_get_disparity_range(pt, src, w, h, pitch, None if null_out else r, None, 0, None),
        "range_mask": lambda: L.vwb200_disparity_range_mask(pt, src, w, h, pitch, mn.ctypes.data, mx.ctypes.data, dst,
                                                            opitch if opitch is not None else pitch, 0, None),
        "transform": lambda: L.vwb200_transform_disparities(pt, mode, m.ctypes.data if matrix else None, 0, sub, src, w, h, pitch, dst,
                                                            opitch if opitch is not None else pitch, 0, None),
    }


def test_invalid_calls_return_earg_before_the_device(v):
    for name in ("subsample", "upsample", "range", "range_mask", "transform"):
        for what, kw in (("pixel type 2", dict(pt=2)), ("pixel type -1", dict(pt=-1)), ("null input", dict(null_in=True)),
                         ("null output", dict(null_out=True)), ("negative width", dict(w=-1)), ("pitch below width", dict(pitch=7))):
            assert calls(v, **kw)[name]() == EARG, (name, what)
        if name != "range":
            assert calls(v, opitch=1)[name]() == EARG, (name, "opitch below the output width")
    for name in ("subsample", "upsample"):                               # the resampling calls never run in place
        assert calls(v, same_buffer=True)[name]() == EARG, name
    assert calls(v, mode=2)["transform"]() == EARG
    assert calls(v, matrix=False)["transform"]() == EARG
    assert calls(v, mode=1, box=(0, 0, 7, 6))["transform"]() == EARG
    assert v.lib().vwb200_last_error() == b"transform_disparities: The sizes of subregion and disparity don't match.\n"
    assert calls(v, mode=1, box=(3, 2, 11, 7))["transform"]() == EARG


def test_valid_calls_need_a_device(v):
    if v.device_count() > 0:
        pytest.skip("device present: the GPU tests cover valid calls")
    for pt in (0, 1):
        c = calls(v, pt=pt)
        for name in ("subsample", "upsample", "range", "range_mask"):
            assert c[name]() == ENODEVICE, name
        for mode in (0, 1):
            assert calls(v, pt=pt, mode=mode, box=(3, 2, 11, 8))["transform"]() == ENODEVICE
        assert calls(v, pt=pt, same_buffer=True)["range_mask"]() == ENODEVICE         # out == in is allowed
    d = np.zeros((4, 5, 3), np.float32)
    for fn in (v.disparity_subsample, v.disparity_upsample, v.get_disparity_range, lambda x: v.disparity_range_mask(x, (0, 0), (5, 4)),
               lambda x: v.transform_disparities(x, np.eye(3)), lambda x: v.transform_disparities_explicit(False, (0, 0, 5, 4), np.eye(3), x)):
        with pytest.raises(v.NoDeviceErr):
            fn(d)


def test_python_refuses_other_dtypes_and_shapes(v):
    for bad in (np.zeros((4, 5, 3), np.float64), np.zeros((4, 5, 3), np.int64), np.zeros((4, 5, 2), np.float32), np.zeros((4, 5), np.int32)):
        for fn in (v.disparity_subsample, v.get_disparity_range, lambda x: v.transform_disparities(x, np.eye(3))):
            with pytest.raises(v.ArgumentErr):
                fn(bad)
    d = np.zeros((4, 5, 3), np.float32)
    with pytest.raises(v.ArgumentErr):
        v.disparity_range_mask(d, (0, 0), (5, 4), out=d.copy())        # out: None or the disparity itself
    with pytest.raises(v.ArgumentErr, match="subregion"):
        v.transform_disparities_explicit(False, (0, 0, 4, 4), np.eye(3), d)


def test_python_checks_the_matrix_as_the_reference_does(v):
    """HomographyTransform(T) needs a 3 x 3 T (ArgumentErr) and inverts it at construction (MathErr when singular)"""
    d = np.zeros((4, 5, 3), np.float32)
    for fn in (lambda m: v.transform_disparities(d, m), lambda m: v.transform_disparities_explicit(False, (0, 0, 5, 4), m, d)):
        with pytest.raises(v.ArgumentErr, match="3x3"):
            fn(np.eye(2))
        with pytest.raises(v.MathErr, match="singular"):
            fn(np.array([[1, 2, 3], [2, 4, 6], [0, 0, 1.0]]))
