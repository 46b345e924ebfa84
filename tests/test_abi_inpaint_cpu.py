"""vwb200_fill_holes_grass refuses bad arguments before it looks for a device, so these run without one."""
import numpy as np
import pytest

EARG = -1
F32 = 1


@pytest.fixture(scope="module")
def L():
    import visionworkbench_b200 as v
    return v.lib()


def call(L, *, ptype=F32, inp=None, w=8, h=8, pitch=8, length=2, x0=0, y0=0, out=None, ow=8, oh=8, opitch=8):
    d = np.zeros((16, 16, 3), np.float32)
    o = np.zeros((16, 16, 3), np.float32)
    inp = d.ctypes.data if inp is None else inp
    out = o.ctypes.data if out is None else out
    return L.vwb200_fill_holes_grass(ptype, inp, w, h, pitch, length, x0, y0, out, ow, oh, opitch, 0, None)


@pytest.mark.parametrize("kw", [dict(ptype=2), dict(length=-1), dict(length=46341), dict(length=2 ** 31 - 1), dict(w=0), dict(h=-1),
                                dict(pitch=7), dict(ow=0), dict(oh=0), dict(opitch=7), dict(x0=-1), dict(y0=-1), dict(x0=1),
                                dict(y0=1), dict(ow=9), dict(x0=4, ow=5)],
                         ids=lambda k: ",".join(f"{a}={b}" for a, b in k.items()))
def test_rejects(L, kw):
    assert call(L, **kw) == EARG
    assert L.vwb200_last_error()


def test_rejects_null_and_overlap(L):
    d = np.zeros((8, 8, 3), np.float32)
    assert L.vwb200_fill_holes_grass(F32, None, 8, 8, 8, 2, 0, 0, d.ctypes.data, 8, 8, 8, 0, None) == EARG
    assert L.vwb200_fill_holes_grass(F32, d.ctypes.data, 8, 8, 8, 2, 0, 0, None, 8, 8, 8, 0, None) == EARG
    # out inside in: the last rows of the input
    assert L.vwb200_fill_holes_grass(F32, d.ctypes.data, 8, 8, 8, 2, 0, 0, d[6:].ctypes.data, 8, 2, 8, 0, None) == EARG
    assert b"overlaps" in L.vwb200_last_error()
