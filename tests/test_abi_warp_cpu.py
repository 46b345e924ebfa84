"""vwb200_transform_image without a GPU: every invalid call returns VWB200_EARG before the library looks for a device, and a
valid call returns VWB200_ENODEVICE when there is none; the Python mirror checks its arguments as the reference does."""
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


def call(v, kind=0, interp=0, edge=0, null_params=False, null_in=False, null_out=False, null_disp=False, w=8, h=6, pitch=8,
         dw=8, dh=6, dpitch=8, x0=0, y0=0, ow=8, oh=6, opitch=8, out_is=None):
    L = v.lib()
    img = np.zeros((6, 8), np.float32)
    disp = np.zeros((6, 8, 3), np.float32)
    out = np.zeros((max(oh, 1), max(opitch, 1)), np.float32)
    p = v.WarpParams(kind, interp, edge)
    p.matrix[:] = list(np.eye(3).reshape(9))
    dst = {"in": img.ctypes.data, "in_row1": img[1:].ctypes.data, "disp": disp.ctypes.data, "disp_end": disp[5, 7:].ctypes.data,
           None: out.ctypes.data}[out_is]
    return L.vwb200_transform_image(None if null_params else C.byref(p), None if null_in else img.ctypes.data, w, h, pitch,
                                    None if null_disp else disp.ctypes.data, dw, dh, dpitch, x0, y0, None if null_out else dst, ow, oh, opitch,
                                    0, None)


INVALID = [
    ("null params", dict(null_params=True)), ("null input", dict(null_in=True)), ("null output", dict(null_out=True)),
    ("kind 2", dict(kind=2)), ("kind -1", dict(kind=-1)), ("interp 3", dict(interp=3)), ("interp -1", dict(interp=-1)),
    ("edge 2", dict(edge=2)), ("edge -1", dict(edge=-1)),
    ("width 0", dict(w=0)), ("height 0", dict(h=0)), ("negative width", dict(w=-1)), ("pitch below width", dict(pitch=7)),
    ("output width 0", dict(ow=0)), ("output height 0", dict(oh=0)), ("negative output height", dict(oh=-2)),
    ("output pitch below width", dict(opitch=7)),
    ("window beyond int32 x", dict(x0=2 ** 31 - 5)), ("window beyond int32 y", dict(y0=2 ** 31 - 3)),
    ("out is in", dict(out_is="in")), ("out overlaps in", dict(out_is="in_row1")),
    ("disparity kind, null disparity", dict(kind=1, null_disp=True)), ("disparity kind, dw 0", dict(kind=1, dw=0)),
    ("disparity kind, dh 0", dict(kind=1, dh=0)), ("disparity kind, dpitch below dw", dict(kind=1, dpitch=7)),
    ("out is the disparity", dict(kind=1, out_is="disp")), ("out overlaps the disparity's last pixel", dict(kind=1, out_is="disp_end")),
]


@pytest.mark.parametrize("what,kw", INVALID, ids=[w for w, _ in INVALID])
def test_invalid_calls_return_earg_before_the_device(v, what, kw):
    assert call(v, **kw) == EARG, what
    assert v.lib().vwb200_last_error().startswith(b"transform_image:")


def test_valid_calls_need_a_device(v):
    if v.device_count() > 0:
        pytest.skip("device present: the GPU tests cover valid calls")
    for kind in (0, 1):
        for interp in (0, 1, 2):
            for edge in (0, 1):
                assert call(v, kind=kind, interp=interp, edge=edge) == ENODEVICE
    # a homography ignores the disparity arguments; windows may start anywhere in int32 and end at 2^31 - 1
    assert call(v, null_disp=True, dw=0, dh=0, dpitch=0) == ENODEVICE
    assert call(v, x0=-2 ** 31, y0=2 ** 31 - 6) == ENODEVICE
    img = np.zeros((4, 5), np.float32)
    for tx in (v.HomographyTransform(np.eye(3)), v.DisparityTransform(np.zeros((4, 5, 3), np.float32))):
        with pytest.raises(v.NoDeviceErr):
            v.transform(img, tx)
        with pytest.raises(v.NoDeviceErr):
            v.transform(img, tx, (-2, -3, 7, 9), v.EDGE_CONSTANT, v.INTERP_BICUBIC)


def test_python_checks_as_the_reference_does(v):
    """HomographyTransform(H) needs a 3 x 3 H (ArgumentErr) and inverts it at construction (MathErr when singular)"""
    with pytest.raises(v.ArgumentErr, match="3x3"):
        v.HomographyTransform(np.eye(2))
    with pytest.raises(v.MathErr, match="singular"):
        v.HomographyTransform(np.array([[1, 2, 3], [2, 4, 6], [0, 0, 1.0]]))
    with pytest.raises(v.ArgumentErr):
        v.DisparityTransform(np.zeros((4, 5, 2), np.float32))
    img = np.zeros((4, 5), np.float32)
    with pytest.raises(v.ArgumentErr):
        v.transform(np.zeros((4, 5, 3), np.float32), v.HomographyTransform(np.eye(3)))
    with pytest.raises(v.ArgumentErr):
        v.transform(img, np.eye(3))                                      # a bare matrix is not a transform
    with pytest.raises(v.ArgumentErr):
        v.transform(img, v.HomographyTransform(np.eye(3)), (3, 0, 3, 4))    # an empty window
    with pytest.raises(v.ArgumentErr):
        v.transform(img, v.HomographyTransform(np.eye(3)), interp=5)
