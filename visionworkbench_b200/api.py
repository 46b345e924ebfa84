"""Python host-side mirror of the reference operator interface, over the C ABI (include/vwb200.h).

Names, argument order and error behaviour follow Vision Workbench:
  * calc_disparity            -- src/vw/Stereo/Correlation.h:50-57
  * PyramidCorrelationView    -- src/vw/Stereo/CorrelationView.h:35-193 (cols/rows/planes,
                                 prerasterize(bbox), rasterize(dest, bbox), operator() throws NoImplErr)
  * pyramid_correlate         -- src/vw/Stereo/CorrelationView.h:195-230
  * cross_corr_consistency_check, rm_outliers_using_thresh, disparity_cleanup_using_thresh,
    disparity_mask            -- src/vw/Stereo/Correlate.h:52-58, DisparityMap.h:318-442,97-253
  * rm_outliers_using_mean, disparity_cleanup_using_mean, rm_outliers_using_stddev, disparity_cleanup_using_stddev
    (int32 or float32 disparities; outlier_filter reaches all six filters on both)
                              -- src/vw/Stereo/DisparityMap.h:444-767
  * disparity_median_filter, texture_measure, texture_preserving_disparity_filter
                              -- src/vw/Stereo/Algorithms.cc:26-67, Algorithms.h:144-281
  * disparity_subsample, disparity_upsample, get_disparity_range, disparity_range_mask, transform_disparities,
    transform_disparities_explicit (int32 or float32 disparities)
                              -- src/vw/Stereo/DisparityMap.h:48-66, 255-300, 1016-1057, 1190-1224, 1251-1358
  * transform with HomographyTransform / DisparityTransform (float32 images; bilinear, bicubic, nearest; zero or
    constant edges)           -- src/vw/Image/Transform.h:485-601, Math/Transform.h:369-389, Stereo/DisparityMap.h:1164-1187
  * fill_holes_grass (int32 or float32 disparities)
                              -- src/vw/Image/InpaintView.h:239-311
  * PinholeModel (NULL or TSAI lens), stereo_triangulate, stereo_model_points (StereoModel::operator() on an image),
    universe_radius           -- src/vw/Camera/PinholeModel.cc:79-116, Stereo/StereoView.h:74-186, StereoModel.cc:254-309
  * epipolar, resize_epipolar_cameras_to_fit, camera_transform, epipolar_transformed_images (float32 or PixelMask<float>
    images)                   -- src/vw/Camera/PinholeModel.cc:351-397, 679-732, EpipolarUtils.cc:37-144, CameraTransform.h
  * ip_match (InterestPointMatcherSimple, L2 or Hamming), remove_duplicates, read/write_binary_ip_file,
    read/write_binary_match_file
                              -- src/vw/InterestPoint/Matcher.h:415-509, Matcher.cc:33-195, MatcherIO.cc:248-366

There is no CPU path: every call goes to libvwb200.so (hand-written sm_90a kernels) and raises if
the library or a CUDA device is missing.  Inputs may be numpy arrays (staged through HBM by the
library) or torch CUDA tensors (used in place, results returned as torch CUDA tensors).
"""
import ctypes as C
import math
import os
import re

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libvwb200.so")
_LIB = None

# vw::stereo::CostFunctionType (Stereo/CostFunctions.h:143-149)
ABSOLUTE_DIFFERENCE, SQUARED_DIFFERENCE, CROSS_CORRELATION, CENSUS_TRANSFORM, TERNARY_CENSUS_TRANSFORM = 0, 1, 2, 3, 4
# vw::stereo::PrefilterModeType (Stereo/PrefilterEnum.h:24-28)
PREFILTER_NONE, PREFILTER_LOG, PREFILTER_MEANSUB = 0, 1, 2
# vw::stereo::CorrelationAlgorithm (Stereo/CorrelationAlgorithms.h:29-35)
VW_CORRELATION_BM, VW_CORRELATION_SGM, VW_CORRELATION_MGM, VW_CORRELATION_FINAL_MGM = 0, 1, 2, 3
# SemiGlobalMatcher::SgmSubpixelMode (Stereo/SGM.h:93-99)
SUBPIXEL_NONE, SUBPIXEL_PARABOLA, SUBPIXEL_LINEAR, SUBPIXEL_POLY4, SUBPIXEL_COSINE, SUBPIXEL_LC_BLEND = 0, 1, 2, 3, 4, 5


class VwError(RuntimeError):
    """Base of the vw::Exception mirror (Core/Exception.h:201-253)."""


class ArgumentErr(VwError):
    pass


class MathErr(VwError):
    pass


class LogicErr(VwError):
    pass


class NoImplErr(VwError):
    pass


class CudaErr(VwError):
    pass


class NoDeviceErr(VwError):
    pass


class PointToPixelErr(VwError):
    """vw::camera::PointToPixelErr: point_to_pixel's round-trip check failed (VWB200_EPROJECT)"""


class IOErr(VwError):
    """vw::IOErr: a camera file could not be read"""


_ERR = {-1: ArgumentErr, -2: MathErr, -3: LogicErr, -4: NoImplErr, -5: CudaErr, -6: NoDeviceErr, -7: MemoryError, -8: PointToPixelErr}


class CorrParams(C.Structure):
    _fields_ = [("search_x0", C.c_int32), ("search_y0", C.c_int32), ("search_x1", C.c_int32), ("search_y1", C.c_int32),
                ("kernel_x", C.c_int32), ("kernel_y", C.c_int32), ("cost_type", C.c_int32),
                ("prefilter_mode", C.c_int32), ("prefilter_width", C.c_float),
                ("consistency_threshold", C.c_float), ("min_consistency_level", C.c_int32),
                ("filter_half_kernel", C.c_int32), ("max_pyramid_levels", C.c_int32), ("collar_size", C.c_int32),
                ("corr_timeout", C.c_int32), ("seconds_per_op", C.c_double),
                ("algorithm", C.c_int32), ("blob_filter_area", C.c_int32),
                ("sgm_subpixel_mode", C.c_int32), ("sgm_search_buffer_x", C.c_int32), ("sgm_search_buffer_y", C.c_int32),
                ("region_ul_x", C.c_int32), ("region_ul_y", C.c_int32), ("write_debug_images", C.c_int32),
                ("sgm_threads", C.c_int32), ("memory_limit_mb", C.c_double)]


class SgmParams(C.Structure):
    _fields_ = [("search_x", C.c_int32), ("search_y", C.c_int32), ("kernel_size", C.c_int32), ("cost_type", C.c_int32),
                ("ternary_threshold", C.c_int32), ("p1", C.c_int32), ("p2", C.c_int32), ("use_mgm", C.c_int32),
                ("subpixel_mode", C.c_int32), ("search_buffer_x", C.c_int32), ("search_buffer_y", C.c_int32),
                ("conserve_level", C.c_int32), ("memory_limit_mb", C.c_double), ("assumed_threads", C.c_int32),
                ("reserved", C.c_int32)]


class K1Stats(C.Structure):
    _fields_ = [("path", C.c_int32), ("launches", C.c_int32), ("kernel_ms", C.c_float), ("reserved", C.c_int32)]


def lib():
    """Load libvwb200.so.  Fails loudly if it has not been built (python -m visionworkbench_b200.build)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            raise ImportError(f"{_SO} is missing: build it with `python visionworkbench_b200/build.py` "
                              "(the engine has no CPU or PyTorch fallback)")
        L = C.CDLL(_SO)
        L.vwb200_last_error.restype = C.c_char_p
        L.vwb200_version.restype = C.c_char_p
        L.vwb200_kernel_launches.restype = C.c_longlong
        P, I, Z, F, D = C.c_void_p, C.c_int, C.c_ssize_t, C.c_float, C.c_double
        L.vwb200_calc_disparity.argtypes = [I, P, I, I, Z, P, I, I, Z, I, I, I, I, P, Z, I, P]
        L.vwb200_pyramid_down.argtypes = [P, I, I, Z, P, Z, I, P]
        L.vwb200_subsample_mask_by_two.argtypes = [P, I, I, Z, P, Z, I, P]
        L.vwb200_prefilter.argtypes = [P, I, I, Z, I, F, P, Z, I, P]
        L.vwb200_sgm_calc_disparity.argtypes = [P, I, I, Z, P, I, I, Z, I, I, I, I, I, P, Z, C.POINTER(I), C.POINTER(I), I, P]
        L.vwb200_sgm_calc_disparity_subpixel.argtypes = [P, I, I, Z, P, I, I, Z, I, I, I, I, I, I, P, Z, P, Z, C.POINTER(I), C.POINTER(I), I, P]
        L.vwb200_sgm_calc_disparity_ex.argtypes = [C.POINTER(SgmParams), P, I, I, Z, P, I, I, Z, P, Z, P, I, I, Z, P, I, I, Z, P, P, Z, P, Z, P,
                                                   C.POINTER(I), C.POINTER(I), I, P]
        L.vwb200_sgm_disp_bounds.argtypes = [C.POINTER(SgmParams), P, I, I, Z, P, Z, P, I, I, Z, I, I, P, I, P]
        L.vwb200_parabola_subpixel.argtypes = [P, I, I, P, Z, P, I, I, Z, I, I, I, F, I, I, I, I, P, Z, I, P]
        L.vwb200_disparity_median_filter.argtypes = [P, I, I, Z, I, I, P]
        L.vwb200_texture_measure.argtypes = [P, I, I, Z, I, D, D, P, Z, I, P]
        L.vwb200_texture_preserving_disparity_filter.argtypes = [P, I, I, Z, P, Z, F, I, I, P]
        L.vwb200_cross_corr_consistency_check.argtypes = [P, I, I, Z, P, I, I, Z, F, I, P]
        L.vwb200_rm_outliers_using_thresh.argtypes = [P, I, I, I, I, D, D, P, I, P]
        L.vwb200_disparity_cleanup_using_thresh.argtypes = [P, I, I, I, I, D, D, P, I, P]
        L.vwb200_disparity_mask.argtypes = [P, I, I, P, P, I, I, P, I, P]
        L.vwb200_outlier_filter.argtypes = [C.POINTER(OutlierParams), I, P, I, I, Z, P, Z, I, P]
        L.vwb200_disparity_subsample.argtypes = [I, P, I, I, Z, P, Z, I, P]
        L.vwb200_disparity_upsample.argtypes = [I, P, I, I, Z, P, Z, I, P]
        L.vwb200_get_disparity_range.argtypes = [I, P, I, I, Z, P, P, I, P]
        L.vwb200_disparity_range_mask.argtypes = [I, P, I, I, Z, P, P, P, Z, I, P]
        L.vwb200_transform_disparities.argtypes = [I, I, P, I, P, P, I, I, Z, P, Z, I, P]
        L.vwb200_transform_image.argtypes = [C.POINTER(WarpParams), P, I, I, Z, P, I, I, Z, I, I, P, I, I, Z, I, P]
        L.vwb200_fill_holes_grass.argtypes = [I, P, I, I, Z, I, I, I, P, I, I, Z, I, P]
        L.vwb200_last_fill_stats.argtypes = [C.POINTER(FillStats)]
        L.vwb200_stereo_triangulate.argtypes = [I, P, I, I, Z, I, I, I, I, C.POINTER(Pinhole), C.POINTER(Pinhole), D, P, Z, I, P]
        L.vwb200_stereo_model_points.argtypes = [P, I, I, Z, C.POINTER(Pinhole), C.POINTER(Pinhole), D, P, Z, P, Z, I, P]
        L.vwb200_last_triangulation_stats.argtypes = [C.POINTER(TriangulationStats)]
        L.vwb200_universe_radius.argtypes = [P, I, I, Z, P, D, D, P, Z, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), I, P]
        PH = C.POINTER(Pinhole)
        L.vwb200_pinhole_epipolar.argtypes = [PH, PH, PH, PH]
        L.vwb200_resize_epipolar_cameras_to_fit.argtypes = [PH, PH, PH, PH, P, P, P, P, P]
        L.vwb200_camera_transform.argtypes = [PH, PH, I, I, I, P, P, I, I, Z, I, I, P, I, I, Z, I, P]
        CH = C.POINTER(Cahv)
        L.vwb200_cahv_epipolar.argtypes = [CH, CH, CH, CH]
        L.vwb200_linearize_camera.argtypes = [CH, P, P, CH]
        L.vwb200_pinhole_to_cahv.argtypes = [PH, CH]
        L.vwb200_cahv_camera_transform.argtypes = [CH, CH, I, I, I, P, P, I, I, Z, I, I, P, I, I, Z, I, P]
        L.vwb200_cahv_stereo_triangulate.argtypes = [I, P, I, I, Z, I, I, I, I, CH, CH, D, P, Z, I, P]
        L.vwb200_cahv_stereo_model_points.argtypes = [P, I, I, Z, CH, CH, D, P, Z, P, Z, I, P]
        L.vwb200_ip_match.argtypes = [I, P, P, I, P, P, I, I, Z, Z, D, P, P, P, I, P]
        L.vwb200_last_ipmatch_stats.argtypes = [C.POINTER(IpMatchStats)]
        L.vwb200_remove_duplicate_matches.argtypes = [P, P, I, P, C.POINTER(I)]
        L.vwb200_corr_create.argtypes = [C.POINTER(CorrParams), C.POINTER(P)]
        L.vwb200_corr_set_inputs.argtypes = [P, P, I, I, Z, P, I, I, Z, P, Z, P, Z, I]
        L.vwb200_corr_rasterize.argtypes = [P, I, I, I, I, P, Z, I, P]
        L.vwb200_corr_prerasterize.argtypes = [P, I, I, I, I, P, Z, I, P]
        L.vwb200_corr_set_lr_disp_diff.argtypes = [P, P, I, I, Z, I]
        L.vwb200_corr_num_levels.argtypes = [P, I, I]
        L.vwb200_corr_cols.argtypes = [P]
        L.vwb200_corr_rows.argtypes = [P]
        L.vwb200_corr_destroy.argtypes = [P]
        L.vwb200_corr_destroy.restype = None
        L.vwb200_last_k1_stats.argtypes = [C.POINTER(K1Stats)]
        _LIB = L
    return _LIB


def _check(rc):
    if rc != 0:
        msg = lib().vwb200_last_error().decode("utf-8", "replace")
        raise _ERR.get(rc, VwError)(msg)


def device_count():
    return lib().vwb200_device_count()


def kernel_launches():
    return lib().vwb200_kernel_launches()


def last_k1_stats():
    s = K1Stats()
    lib().vwb200_last_k1_stats(C.byref(s))
    return {"path": "exact-int" if s.path == 0 else "general-fp64", "launches": s.launches, "kernel_ms": s.kernel_ms}


def _is_torch(x):
    return type(x).__module__.startswith("torch")


def _stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _np(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def _ptr(x):
    return x.data_ptr() if _is_torch(x) else x.ctypes.data


def _raster(x, dtype, channels=1, on_device=None):
    """(keep-alive, pointer, cols, rows, pitch in pixels, on_device) of an input raster (rows, cols[, channels]): a numpy array,
    made C-contiguous `dtype`, or a torch CUDA tensor, converted to `dtype` and copied only when its rows are not dense.
    on_device: where the call's other rasters are; a raster elsewhere is refused."""
    if _is_torch(x):
        import torch
        t = x.to(getattr(torch, np.dtype(dtype).name))
        if t.dim() < 2 or t.shape[0] == 0 or not t[0].is_contiguous() or t.stride(0) < t[0].numel():
            t = t.contiguous()
        r = (t, t.data_ptr(), t.shape[1], t.shape[0], t.stride(0) // channels, 1)
    else:
        a = _np(x, dtype)
        r = (a, a.ctypes.data, a.shape[1], a.shape[0], a.shape[1], 0)
    if on_device is not None and r[5] != on_device:
        raise ArgumentErr("the inputs must all be numpy arrays or all be CUDA tensors")
    return r


def _optional(x, dtype):
    """(keep-alive, pointer, cols, rows, pitch in pixels) of an optional host raster; (None, None, 0, 0, 0) without one"""
    return (None, None, 0, 0, 0) if x is None else _raster(_np(x, dtype), dtype)[:5]


def _output(beside, shape, dtype):
    """an uninitialised output where `beside` lives: a CUDA tensor on its device, or a numpy array"""
    if _is_torch(beside):
        import torch
        return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), device=beside.device)
    return np.empty(shape, dtype)


def _in_place(x, channels, what):
    """(pointer, cols, rows, pitch in pixels, on_device) of a float32 (rows, cols, channels) raster the library writes
    (a CUDA tensor, or a writeable numpy array) with dense pixels; ArgumentErr(what(on_device)) otherwise"""
    if _is_torch(x):
        import torch
        ok = x.is_cuda and x.dtype == torch.float32 and x.dim() == 3 and x.shape[2] == channels and x.stride(2) == 1 and x.stride(1) == channels
        r = (x.data_ptr(), x.shape[1], x.shape[0], x.stride(0) // channels, 1) if ok else None
    else:
        px = 4 * channels
        ok = (isinstance(x, np.ndarray) and x.dtype == np.float32 and x.ndim == 3 and x.shape[2] == channels and x.strides[2] == 4
              and x.strides[1] == px and x.strides[0] % px == 0 and x.flags.writeable)
        r = (x.ctypes.data, x.shape[1], x.shape[0], x.strides[0] // px, 0) if ok else None
    if not ok:
        raise ArgumentErr(what(_is_torch(x)))
    return r


def calc_disparity(cost_type, left_in, right_in, search_volume, kernel_size):
    """vw::stereo::calc_disparity (Stereo/Correlation.h:50-57) on already-cropped rasters.

    left_in : (H+ky-1, W+kx-1) float32;  right_in: at least (H+ky-1+sy-1, W+kx-1+sx-1).
    search_volume = (sx, sy), kernel_size = (kx, ky).
    Returns int32 (H, W, 3) {dx, dy, valid} -- PixelMask<Vector2i>.
    """
    sx, sy = search_volume
    kx, ky = kernel_size
    l, lp, lw, lh, lpitch, dev = _raster(left_in, np.float32)
    r, rp, rw, rh, rpitch, _ = _raster(right_in, np.float32, on_device=dev)
    H, W = lh - ky + 1, lw - kx + 1
    if H <= 0 or W <= 0:
        raise ArgumentErr("calc_disparity: Kernel size too large of active region.")
    out = _output(l, (H, W, 3), np.int32)
    _check(lib().vwb200_calc_disparity(cost_type, lp, lw, lh, lpitch, rp, rw, rh, rpitch, sx, sy, kx, ky, _ptr(out), W, dev,
                                       _stream_ptr() if dev else None))
    return out


def calc_disparity_sgm(left_in, right_in, search_volume, kernel_size, p1=0, p2=0):
    """vw::stereo::calc_disparity_sgm (Stereo/SGM.cc:167-230) for CENSUS_TRANSFORM / SGM on the cropped left_region and
    right_region rasters: the search box is [0, search_volume] (inclusive) for every pixel.  kernel_size 3, 5, 7 or 9.
    Returns int32 (out_h, out_w, 3) {dx, dy, valid} (the raster of SGM.cc:2397-2420: the borders the kernel and the search
    cannot cover are cropped)."""
    sx, sy = search_volume
    ow, oh = C.c_int(0), C.c_int(0)
    l, lp, lw, lh, lpitch, dev = _raster(left_in, np.float32)
    r, rp, rw, rh, rpitch, _ = _raster(right_in, np.float32, on_device=dev)
    args = (lp, lw, lh, lpitch, rp, rw, rh, rpitch, sx, sy, kernel_size, p1, p2)
    _check(lib().vwb200_sgm_calc_disparity(*args, None, 0, C.byref(ow), C.byref(oh), dev, None))
    out = _output(l, (max(oh.value, 0), max(ow.value, 0), 3), np.int32)
    if ow.value > 0 and oh.value > 0:
        _check(lib().vwb200_sgm_calc_disparity(*args, _ptr(out), ow.value, C.byref(ow), C.byref(oh), dev, _stream_ptr() if dev else None))
    return out


def calc_disparity_sgm_subpixel(left_in, right_in, search_volume, kernel_size, subpixel_mode=5, p1=0, p2=0):
    """calc_disparity_sgm followed by SemiGlobalMatcher::create_disparity_view_subpixel (Stereo/SGM.cc:1497-1614).
    subpixel_mode: SgmSubpixelMode (SGM.h:93-99), default SUBPIXEL_LC_BLEND.  Returns (int32 (h, w, 3), float32 (h, w, 3))."""
    sx, sy = search_volume
    ow, oh = C.c_int(0), C.c_int(0)
    l, r = _np(left_in, np.float32), _np(right_in, np.float32)
    args = (l.ctypes.data, l.shape[1], l.shape[0], l.shape[1], r.ctypes.data, r.shape[1], r.shape[0], r.shape[1], sx, sy, kernel_size, p1, p2,
            subpixel_mode)
    _check(lib().vwb200_sgm_calc_disparity_subpixel(*args, None, 0, None, 0, C.byref(ow), C.byref(oh), 0, None))
    out = np.empty((max(oh.value, 0), max(ow.value, 0), 3), np.int32)
    sub = np.empty((max(oh.value, 0), max(ow.value, 0), 3), np.float32)
    if out.size:
        _check(lib().vwb200_sgm_calc_disparity_subpixel(*args, out.ctypes.data, ow.value, sub.ctypes.data, ow.value, C.byref(ow), C.byref(oh), 0, None))
    return out, sub


def _sgm_params(search_volume, kernel_size, cost_type=CENSUS_TRANSFORM, use_mgm=False, subpixel_mode=SUBPIXEL_NONE, search_buffer=(2, 2),
                memory_limit_mb=6000, p1=0, p2=0, ternary_threshold=5, conserve_level=-1, assumed_threads=4):
    return SgmParams(int(search_volume[0]), int(search_volume[1]), int(kernel_size), int(cost_type), int(ternary_threshold), int(p1), int(p2),
                     int(bool(use_mgm)), int(subpixel_mode), int(search_buffer[0]), int(search_buffer[1]), int(conserve_level),
                     float(memory_limit_mb), int(assumed_threads), 0)


def calc_disparity_sgm_ex(cost_type, left_in, right_in, search_volume, kernel_size, use_mgm=False, subpixel_mode=SUBPIXEL_NONE,
                          search_buffer=(2, 2), memory_limit_mb=6000, left_mask=None, right_mask=None, prev_disparity=None,
                          bounds=None, p1=0, p2=0, ternary_threshold=5, conserve_level=-1, assumed_threads=4, return_bounds=False):
    """vw::stereo::calc_disparity_sgm with all its arguments (Stereo/SGM.h:361-376, SGM.cc:167-230): cost type
    (CENSUS_TRANSFORM / TERNARY_CENSUS_TRANSFORM), SGM or MGM, sub-pixel mode, search buffer, memory limit, masks and the
    previous pyramid level's disparity (which give every pixel its own search box).  `bounds` (h, w, 4) overrides the boxes.
    Returns (int32 (h, w, 3), float32 (h, w, 3) sub-pixel disparity[, int32 (h, w, 4) boxes])."""
    sp = _sgm_params(search_volume, kernel_size, cost_type, use_mgm, subpixel_mode, search_buffer, memory_limit_mb, p1, p2, ternary_threshold,
                     conserve_level, assumed_threads)
    l, r = _np(left_in, np.float32), _np(right_in, np.float32)
    ow, oh = C.c_int(0), C.c_int(0)
    head = (C.byref(sp), l.ctypes.data, l.shape[1], l.shape[0], l.shape[1], r.ctypes.data, r.shape[1], r.shape[0], r.shape[1])
    _check(lib().vwb200_sgm_calc_disparity_ex(*head, None, 0, None, 0, 0, 0, None, 0, 0, 0, None, None, 0, None, 0, None, C.byref(ow), C.byref(oh), 0, None))
    h, w = max(oh.value, 0), max(ow.value, 0)
    out = np.zeros((h, w, 3), np.int32)
    sub = np.zeros((h, w, 3), np.float32)
    bo = np.zeros((h, w, 4), np.int32)
    if out.size:
        lm, rm, pv, bd = _optional(left_mask, np.uint8), _optional(right_mask, np.uint8), _optional(prev_disparity, np.int32), \
            _optional(bounds, np.int32)
        if lm[0] is not None and lm[0].shape != (h, w):
            raise LogicErr("Left mask size does not match the output size.")
        if bd[0] is not None and bd[0].shape != (h, w, 4):
            raise ArgumentErr("sgm: bounds must be (out_h, out_w, 4)")
        _check(lib().vwb200_sgm_calc_disparity_ex(*head, lm[1], w, *rm[1:], *pv[1:], bd[1], out.ctypes.data, w, sub.ctypes.data, w,
                                                  bo.ctypes.data if return_bounds else None, C.byref(ow), C.byref(oh), 0, None))
    return (out, sub, bo) if return_bounds else (out, sub)


def sgm_disp_bounds(shape, search_volume, search_buffer=(2, 2), prev_disparity=None, left_mask=None, right_mask=None, conserve_level=0,
                    use_mgm=False, memory_limit_mb=6000, assumed_threads=4):
    """SemiGlobalMatcher::populate_disp_bound_image + constrain_disp_bound_image (Stereo/SGM.cc:241-668): the search box
    {min_x, min_y, max_x, max_y} of every pixel of an (h, w) output."""
    h, w = int(shape[0]), int(shape[1])
    sp = _sgm_params(search_volume, 5, CENSUS_TRANSFORM, use_mgm, 0, search_buffer, memory_limit_mb, conserve_level=conserve_level,
                     assumed_threads=assumed_threads)
    lm, rm, pv = _optional(left_mask, np.uint8), _optional(right_mask, np.uint8), _optional(prev_disparity, np.int32)
    if lm[0] is not None and lm[0].shape != (h, w):
        raise LogicErr("Left mask size does not match the output size.")
    out = np.zeros((h, w, 4), np.int32)
    _check(lib().vwb200_sgm_disp_bounds(C.byref(sp), *pv[1:], lm[1], w, *rm[1:], w, h, out.ctypes.data, 0, None))
    return out


def pyramid_down(img):
    """subsample(separable_convolution_filter(img, k, k), 2) with k = [1,4,6,4,1]/16
    (Stereo/CorrelationView.cc:210-214)."""
    a = _np(img, np.float32)
    h, w = a.shape
    out = np.empty((1 + (h - 1) // 2, 1 + (w - 1) // 2), np.float32)
    _check(lib().vwb200_pyramid_down(a.ctypes.data, w, h, w, out.ctypes.data, out.shape[1], 0, None))
    return out


def prefilter_image(image, prefilter_mode, prefilter_width):
    """vw::stereo::prefilter_image (Stereo/PreFilter.h:75-95)."""
    a = _np(image, np.float32)
    h, w = a.shape
    out = np.empty_like(a)
    _check(lib().vwb200_prefilter(a.ctypes.data, w, h, w, int(prefilter_mode), float(prefilter_width), out.ctypes.data, w, 0, None))
    return out


def subsample_mask_by_two(mask):
    a = _np(mask, np.uint8)
    h, w = a.shape
    out = np.empty((1 + (h - 1) // 2, 1 + (w - 1) // 2), np.uint8)
    _check(lib().vwb200_subsample_mask_by_two(a.ctypes.data, w, h, w, out.ctypes.data, out.shape[1], 0, None))
    return out


def cross_corr_consistency_check(l2r, r2l, cross_corr_threshold):
    """Stereo/Correlate.h:52-58; returns the checked copy of l2r."""
    a = _np(l2r, np.int32).copy()
    b = _np(r2l, np.int32)
    _check(lib().vwb200_cross_corr_consistency_check(a.ctypes.data, a.shape[1], a.shape[0], a.shape[1],
                                                     b.ctypes.data, b.shape[1], b.shape[0], b.shape[1],
                                                     float(cross_corr_threshold), 0, None))
    return a


def rm_outliers_using_thresh(disparity_map, half_h_kernel, half_v_kernel, pixel_threshold, rejection_threshold):
    a = _np(disparity_map, np.int32)
    out = np.empty_like(a)
    _check(lib().vwb200_rm_outliers_using_thresh(a.ctypes.data, a.shape[1], a.shape[0], half_h_kernel, half_v_kernel,
                                                 pixel_threshold, rejection_threshold, out.ctypes.data, 0, None))
    return out


def disparity_cleanup_using_thresh(disparity_map, h_half_kernel, v_half_kernel, pixel_threshold, rejection_threshold):
    a = _np(disparity_map, np.int32)
    out = np.empty_like(a)
    _check(lib().vwb200_disparity_cleanup_using_thresh(a.ctypes.data, a.shape[1], a.shape[0], h_half_kernel, v_half_kernel,
                                                       pixel_threshold, rejection_threshold, out.ctypes.data, 0, None))
    return out


def disparity_mask(disparity_map, left_mask, right_mask):
    a = _np(disparity_map, np.int32)
    lm, rm = _np(left_mask, np.uint8), _np(right_mask, np.uint8)
    if lm.shape != a.shape[:2]:
        raise ArgumentErr("disparity_mask: input and left mask are not same dimensions.")
    out = np.empty_like(a)
    _check(lib().vwb200_disparity_mask(a.ctypes.data, a.shape[1], a.shape[0], lm.ctypes.data, rm.ctypes.data,
                                       rm.shape[1], rm.shape[0], out.ctypes.data, 0, None))
    return out


class OutlierParams(C.Structure):
    _fields_ = [("method", C.c_int32), ("cleanup", C.c_int32), ("half_h", C.c_int32), ("half_v", C.c_int32),
                ("pixel_threshold", C.c_double), ("rejection_threshold", C.c_double), ("max_mean_diff", C.c_double)]


# vwb200_outlier_filter's methods and pixel types (include/vwb200.h)
OUTLIERS_THRESH, OUTLIERS_MEAN, OUTLIERS_STDDEV = 0, 1, 2
DISP_I32, DISP_F32 = 0, 1


def outlier_filter(method, cleanup, disparity_map, half_h, half_v, pixel_threshold=0.0, rejection_threshold=0.0, max_mean_diff=0.0):
    """vwb200_outlier_filter: one of the six neighbourhood outlier filters of Stereo/DisparityMap.h on an int32
    (PixelMask<Vector2i>) or float32 (PixelMask<Vector2f>) (rows, cols, 3) {dx, dy, valid} disparity, a numpy array or a
    CUDA tensor on the current stream.  Returns a new array or tensor of the same type; the input is not changed."""
    if _is_torch(disparity_map):
        import torch
        dt = {torch.int32: np.int32, torch.float32: np.float32}.get(disparity_map.dtype)
    else:
        dt = np.asarray(disparity_map).dtype.type
    if dt not in (np.int32, np.float32) or len(disparity_map.shape) != 3 or disparity_map.shape[2] != 3:
        raise ArgumentErr("the disparity must be an int32 or float32 (rows, cols, 3) array or CUDA tensor")
    t, ptr, cols, rows, pitch, dev = _raster(disparity_map, dt, channels=3)
    out = _output(t, (rows, cols, 3), dt)
    p = OutlierParams(int(method), int(bool(cleanup)), int(half_h), int(half_v), float(pixel_threshold), float(rejection_threshold),
                      float(max_mean_diff))
    _check(lib().vwb200_outlier_filter(C.byref(p), DISP_I32 if dt == np.int32 else DISP_F32, ptr, cols, rows, pitch, _ptr(out), cols, dev,
                                       _stream_ptr() if dev else None))
    return out


def rm_outliers_using_mean(disparity_map, half_h_kernel, half_v_kernel, max_mean_diff):
    """rm_outliers_using_mean (Stereo/DisparityMap.h:444-578): a valid pixel further than max_mean_diff from the mean of
    its window's valid pixels is rejected.  Pixels longer (|dx| + |dy|) than twice the window's 75th-percentile length end
    their window row, as in the reference.  int32 or float32 (rows, cols, 3), numpy or CUDA; returns a new raster."""
    return outlier_filter(OUTLIERS_MEAN, 0, disparity_map, half_h_kernel, half_v_kernel, max_mean_diff=max_mean_diff)


def disparity_cleanup_using_mean(disparity_map, h_half_kernel, v_half_kernel, max_mean_diff):
    """disparity_cleanup_using_mean (Stereo/DisparityMap.h:580-598): rm_outliers_using_mean, then the isolated-pixel pass
    RmOutliersUsingThreshFunc(1, 1, 3.0, 0.2)."""
    return outlier_filter(OUTLIERS_MEAN, 1, disparity_map, h_half_kernel, v_half_kernel, max_mean_diff=max_mean_diff)


def rm_outliers_using_stddev(disparity_map, half_h_kernel, half_v_kernel, pixel_threshold, rejection_threshold):
    """rm_outliers_using_stddev (Stereo/DisparityMap.h:600-748): a valid pixel further than pixel_threshold standard
    deviations (at least rejection_threshold) from its window's mean, on either axis, is rejected.  int32 or float32
    (rows, cols, 3), numpy or CUDA; returns a new raster."""
    return outlier_filter(OUTLIERS_STDDEV, 0, disparity_map, half_h_kernel, half_v_kernel, pixel_threshold, rejection_threshold)


def disparity_cleanup_using_stddev(disparity_map, h_half_kernel, v_half_kernel, pixel_threshold, rejection_threshold):
    """disparity_cleanup_using_stddev (Stereo/DisparityMap.h:750-767): rm_outliers_using_stddev, then the isolated-pixel
    pass RmOutliersUsingThreshFunc(1, 1, 3.0, 0.2)."""
    return outlier_filter(OUTLIERS_STDDEV, 1, disparity_map, h_half_kernel, v_half_kernel, pixel_threshold, rejection_threshold)


# vwb200_transform_disparities' modes (include/vwb200.h)
TRANSFORM_LAZY, TRANSFORM_EXPLICIT = 0, 1


def _disparity_in(disparity_map):
    """(keep-alive, pointer, cols, rows, pitch in pixels, on_device, numpy dtype) of an int32 or float32 (rows, cols, 3)
    disparity, a numpy array or a CUDA tensor"""
    if _is_torch(disparity_map):
        import torch
        dt = {torch.int32: np.int32, torch.float32: np.float32}.get(disparity_map.dtype)
    else:
        dt = np.asarray(disparity_map).dtype.type
    if dt not in (np.int32, np.float32) or len(disparity_map.shape) != 3 or disparity_map.shape[2] != 3:
        raise ArgumentErr("the disparity must be an int32 or float32 (rows, cols, 3) array or CUDA tensor")
    return _raster(disparity_map, dt, channels=3) + (dt,)


def _ptype(dt):
    return DISP_I32 if dt == np.int32 else DISP_F32


def disparity_subsample(disparity_map):
    """disparity_subsample (Stereo/DisparityMap.h:1251-1322): the 10 / 5 / 2 weighted mean of the valid pixels of each
    3 x 3 neighbourhood at stride 2 (clamped at the border), an image of 1 + (cols-1)/2 x 1 + (rows-1)/2 pixels.  int32 or
    float32 (rows, cols, 3), numpy or CUDA; returns a new raster of the same kind."""
    t, ptr, cols, rows, pitch, dev, dt = _disparity_in(disparity_map)
    ow, oh = (1 + (cols - 1) // 2, 1 + (rows - 1) // 2) if cols and rows else (0, 0)
    out = _output(t, (oh, ow, 3), dt)
    _check(lib().vwb200_disparity_subsample(_ptype(dt), ptr, cols, rows, pitch, _ptr(out), ow, dev, _stream_ptr() if dev else None))
    return out


def disparity_upsample(disparity_map):
    """disparity_upsample (Stereo/DisparityMap.h:1324-1358): each pixel doubled into a 2 x 2 block of a 2 cols x 2 rows
    image, validity carried from the pixel.  int32 or float32 (rows, cols, 3), numpy or CUDA; returns a new raster."""
    t, ptr, cols, rows, pitch, dev, dt = _disparity_in(disparity_map)
    out = _output(t, (2 * rows, 2 * cols, 3), dt)
    _check(lib().vwb200_disparity_upsample(_ptype(dt), ptr, cols, rows, pitch, _ptr(out), 2 * cols, dev, _stream_ptr() if dev else None))
    return out


def get_disparity_range(disparity_map):
    """get_disparity_range (Stereo/DisparityMap.h:48-66): BBox2f(min, max) of the valid pixels' children as a BBox2f-like
    tuple (min dx, min dy, max dx, max dy) of Python floats holding float32 values; (0, 0, 0, 0) without a valid pixel."""
    t, ptr, cols, rows, pitch, dev, dt = _disparity_in(disparity_map)
    r = (C.c_float * 4)()
    _check(lib().vwb200_get_disparity_range(_ptype(dt), ptr, cols, rows, pitch, r, None, dev, _stream_ptr() if dev else None))
    return tuple(r)


def _pixel_out(t, rows, cols, dt, out):
    if out is None:
        return _output(t, (rows, cols, 3), dt), cols
    if out is not t:
        raise ArgumentErr("out must be None or the disparity itself")
    return out, cols


def disparity_range_mask(disparity_map, min, max, out=None):
    """disparity_range_mask (Stereo/DisparityMap.h:255-300): a valid pixel that points outside [min, max - 1) of the
    secondary image becomes {0, 0, 0} (the y coordinate is compared against min[0], as in the reference).  min / max: the
    (dx, dy) children of the reference's min / max pixels.  out=None gives a new raster; out=disparity_map writes it in
    place (a CUDA tensor or a C-contiguous numpy array)."""
    t, ptr, cols, rows, pitch, dev, dt = _disparity_in(disparity_map)
    o, op = _pixel_out(t, rows, cols, dt, out)
    mn, mx = np.asarray(min, dt).reshape(2).copy(), np.asarray(max, dt).reshape(2).copy()
    _check(lib().vwb200_disparity_range_mask(_ptype(dt), ptr, cols, rows, pitch, mn.ctypes.data, mx.ctypes.data, _ptr(o), pitch if out is not None else op,
                                             dev, _stream_ptr() if dev else None))
    return o


def _homography(matrix):
    """the 3 x 3 float64 matrix and its inverse, refused as HomographyTransform's constructor refuses it (Math/Matrix.h)"""
    m = np.asarray(matrix, np.float64)
    if m.shape != (3, 3):
        raise ArgumentErr("Matrix must have dimensions 3x3.")
    try:
        return m, np.linalg.inv(m)
    except np.linalg.LinAlgError:
        raise MathErr("Matrix is singular in inverse()") from None


def transform_disparities(disparity_map, homography, out=None):
    """transform_disparities(disparity, HomographyTransform(H)) (Stereo/DisparityMap.h:1016-1057): each pixel becomes
    reverse(loc + d) - loc with reverse() applying inverse(H), computed here with numpy; it agrees with vw::math::inverse to
    rounding (pass the reference's inverse to vwb200_transform_disparities for its exact matrix).  Invalid pixels stay invalid
    and receive the transformed values.  out: as in disparity_range_mask."""
    return _transform(TRANSFORM_LAZY, _homography(homography)[1], False, None, disparity_map, out)


def transform_disparities_explicit(do_round, subregion, T, disparity, out=None):
    """transform_disparities(do_round, subregion, T, disparity) (Stereo/DisparityMap.h:1190-1224): each valid pixel becomes
    T(beg + d) - beg with beg = subregion.min() + loc, rounded when do_round; invalid pixels give {0, 0, 0}.  subregion:
    (x0, y0, x1, y1) or a BBox2i of the disparity's size (ArgumentErr otherwise).  T must be 3 x 3 (ArgumentErr) and
    invertible (MathErr), as for the reference's HomographyTransform(T)."""
    b = (subregion.x0, subregion.y0, subregion.x1, subregion.y1) if isinstance(subregion, BBox2i) else tuple(subregion)
    if len(disparity.shape) == 3 and (b[2] - b[0] != disparity.shape[1] or b[3] - b[1] != disparity.shape[0]):   # checked first, as there
        raise ArgumentErr("transform_disparities: The sizes of subregion and disparity don't match.\n")
    return _transform(TRANSFORM_EXPLICIT, _homography(T)[0], do_round, b, disparity, out)


def _transform(mode, matrix, do_round, box, disparity_map, out):
    t, ptr, cols, rows, pitch, dev, dt = _disparity_in(disparity_map)
    o, op = _pixel_out(t, rows, cols, dt, out)
    m = np.ascontiguousarray(np.asarray(matrix, np.float64).reshape(9))
    sub = (C.c_int32 * 4)(*[int(v) for v in box]) if box is not None else None
    _check(lib().vwb200_transform_disparities(_ptype(dt), mode, m.ctypes.data, int(bool(do_round)), sub, ptr, cols, rows, pitch, _ptr(o),
                                              pitch if out is not None else op, dev, _stream_ptr() if dev else None))
    return o


# vwb200_transform_image's transform kinds, interpolations and edge extensions (include/vwb200.h)
WARP_HOMOGRAPHY, WARP_DISPARITY = 0, 1
INTERP_BILINEAR, INTERP_BICUBIC, INTERP_NEAREST = 0, 1, 2
EDGE_ZERO, EDGE_CONSTANT, EDGE_VALUE = 0, 1, 2   # EDGE_VALUE: ValueEdgeExtension, camera_transform of PixelMask<float> images


class WarpParams(C.Structure):
    _fields_ = [("kind", C.c_int32), ("interp", C.c_int32), ("edge", C.c_int32), ("matrix", C.c_double * 9)]


class HomographyTransform:
    """vw::HomographyTransform(H) (Math/Transform.h:369-389): reverse() applies inverse(H), computed here with numpy (it agrees
    with vw::math::inverse to rounding).  H must be 3 x 3 (ArgumentErr) and invertible (MathErr), as in the reference."""

    def __init__(self, H):
        self.H, self.H_inverse = _homography(H)


class DisparityTransform:
    """vw::stereo::DisparityTransform(disparity) (Stereo/DisparityMap.h:1164-1187) on a float32 (rows, cols, 3) {dx, dy, valid}
    disparity, a numpy array or a CUDA tensor (the image it warps must be of the same kind): reverse(p) = p + (dx, dy) where
    the pixel at p is valid, and (-1, p.y) elsewhere, outside the disparity included."""

    def __init__(self, disparity):
        if len(disparity.shape) != 3 or disparity.shape[2] != 3:
            raise ArgumentErr("DisparityTransform: the disparity must be a float32 (rows, cols, 3) array or CUDA tensor")
        self.disparity = disparity


def transform(image, tx, bbox=None, edge=EDGE_ZERO, interp=INTERP_BILINEAR):
    """vw::transform(image, tx[, bbox], edge, interp) (Image/Transform.h:485-601), rasterised: the float32 image (rows, cols),
    numpy or CUDA, warped by a HomographyTransform or a DisparityTransform, over bbox (x0, y0, x1, y1) or a BBox2i of the
    transformed image; None gives the image's own extent (0, 0, cols, rows).  The width / height form is
    bbox=(0, 0, width, height).  Bit for bit the reference's where both reversed coordinates are finite with |c| < 2^30;
    0.0 elsewhere.  Returns a new (y1 - y0, x1 - x0) float32 raster where the image lives."""
    if not _is_torch(image) and _np(image, np.float32).ndim != 2:
        raise ArgumentErr("transform: the image must be 2-D")
    t, ptr, cols, rows, pitch, dev = _raster(image, np.float32)
    x0, y0, x1, y1 = _bbox(bbox) if bbox is not None else (0, 0, cols, rows)
    p = WarpParams(0, int(interp), int(edge))
    keep, dptr, dw, dh, dpitch = None, None, 0, 0, 0
    if isinstance(tx, HomographyTransform):
        p.kind = WARP_HOMOGRAPHY
        p.matrix[:] = [float(v) for v in np.asarray(tx.H_inverse, np.float64).reshape(9)]
    elif isinstance(tx, DisparityTransform):
        p.kind = WARP_DISPARITY
        keep, dptr, dw, dh, dpitch, _ = _raster(tx.disparity, np.float32, channels=3, on_device=dev)
    else:
        raise ArgumentErr("transform: tx must be a HomographyTransform or a DisparityTransform")
    out = _output(t, (max(y1 - y0, 0), max(x1 - x0, 0)), np.float32)
    _check(lib().vwb200_transform_image(C.byref(p), ptr, cols, rows, pitch, dptr, dw, dh, dpitch, x0, y0, _ptr(out), x1 - x0, y1 - y0,
                                        x1 - x0, dev, _stream_ptr() if dev else None))
    return out


class FillStats(C.Structure):
    _fields_ = [("holes", C.c_longlong), ("filled", C.c_longlong), ("max_sweeps", C.c_longlong), ("max_levels", C.c_longlong),
                ("critical_steps", C.c_longlong)]


def fill_holes_grass(disparity_map, hole_fill_len, bbox=None):
    """fill_holes_grass(img, hole_fill_len) (Image/InpaintView.h:239-311), rasterised over bbox (x0, y0, x1, y1) or a BBox2i
    inside the image; None is the whole image, the `ImageView<PixelT> result = fill_holes_grass(...)` form.  The holes (8-connected
    invalid pixels) at most hole_fill_len wide and tall are filled by the grassfire-ordered Gauss-Seidel inpainting of the
    reference; the result depends on bbox as the reference's does.  int32 or float32 (rows, cols, 3), numpy or CUDA; returns
    a new (y1 - y0, x1 - x0, 3) raster of the same kind.  ArgumentErr for hole_fill_len < 0 or with hole_fill_len^2 beyond
    int32, and for a bbox that is empty or leaves the image."""
    t, ptr, cols, rows, pitch, dev, dt = _disparity_in(disparity_map)
    x0, y0, x1, y1 = _bbox(bbox) if bbox is not None else (0, 0, cols, rows)
    out = _output(t, (max(y1 - y0, 0), max(x1 - x0, 0), 3), dt)
    _check(lib().vwb200_fill_holes_grass(_ptype(dt), ptr, cols, rows, pitch, int(hole_fill_len), x0, y0, _ptr(out), x1 - x0, y1 - y0,
                                         x1 - x0, dev, _stream_ptr() if dev else None))
    return out


def last_fill_stats():
    """what the last fill_holes_grass on this thread did: holes found in its tile, holes filled, the largest
    10 * max_distance^2, the most levels of one hole, and the longest chain of synchronised steps (sweeps x levels)"""
    s = FillStats()
    lib().vwb200_last_fill_stats(C.byref(s))
    return {k: int(getattr(s, k)) for k, _ in FillStats._fields_}


LENS_NULL, LENS_TSAI = 0, 1
DBL_MAX = float(np.finfo(np.float64).max)


class Pinhole(C.Structure):
    _fields_ = [("center", C.c_double * 3), ("rotation", C.c_double * 9), ("fu", C.c_double), ("fv", C.c_double), ("cu", C.c_double),
                ("cv", C.c_double), ("u_direction", C.c_double * 3), ("v_direction", C.c_double * 3), ("w_direction", C.c_double * 3),
                ("pixel_pitch", C.c_double), ("lens", C.c_int), ("num_lens_params", C.c_int), ("lens_params", C.c_double * 5)]


class TsaiLensDistortion:
    """TsaiLensDistortion(params) (Camera/LensDistortion.h): k1, k2, p1, p2, k3"""

    def __init__(self, params):
        self.params = tuple(float(p) for p in params)
        if len(self.params) != 5:
            raise ArgumentErr("TsaiLensDistortion: Incorrect number of parameters was passed in.")

    def name(self):
        return "TSAI"


class NullLensDistortion:
    def name(self):
        return "NULL"


class PinholeModel:
    """camera::PinholeModel(camera_center, rotation, f_u, f_v, c_u, c_v[, u_direction, v_direction, w_direction],
    distortion_model=None, pixel_pitch=1.0) (Camera/PinholeModel.cc:79-116): the parameters only; the engine builds the inverse
    camera transform of each call from them, as rebuild_camera_matrix does.  distortion_model: None / NullLensDistortion() or
    TsaiLensDistortion(k1, k2, p1, p2, k3)."""

    def __init__(self, camera_center, rotation, f_u, f_v, c_u, c_v, u_direction=(1, 0, 0), v_direction=(0, 1, 0), w_direction=(0, 0, 1),
                 distortion_model=None, pixel_pitch=1.0):
        self.camera_center = tuple(float(x) for x in camera_center)
        self.rotation = np.asarray(rotation, np.float64).reshape(3, 3).copy()
        self.fu, self.fv, self.cu, self.cv = float(f_u), float(f_v), float(c_u), float(c_v)
        self.frame = tuple(tuple(float(x) for x in d) for d in (u_direction, v_direction, w_direction))
        self.distortion = distortion_model if distortion_model is not None else NullLensDistortion()
        self.pixel_pitch = float(pixel_pitch)

    def _struct(self):
        p = Pinhole()
        p.center[:] = self.camera_center
        p.rotation[:] = [float(x) for x in self.rotation.reshape(9)]
        p.fu, p.fv, p.cu, p.cv = self.fu, self.fv, self.cu, self.cv
        p.u_direction[:], p.v_direction[:], p.w_direction[:] = self.frame
        p.pixel_pitch = self.pixel_pitch
        if isinstance(self.distortion, TsaiLensDistortion):
            p.lens, p.num_lens_params = LENS_TSAI, 5
            p.lens_params[:] = self.distortion.params
        elif not isinstance(self.distortion, NullLensDistortion):
            raise NoImplErr(f"lens distortion {self.distortion.name()} has no device form (NULL and TSAI do)")
        return p

    @classmethod
    def _from_struct(cls, p):
        lens = TsaiLensDistortion(p.lens_params[:]) if p.lens == LENS_TSAI else None
        return cls(p.center[:], np.array(p.rotation[:]).reshape(3, 3), p.fu, p.fv, p.cu, p.cv, p.u_direction[:], p.v_direction[:],
                   p.w_direction[:], lens, p.pixel_pitch)


def stereo_triangulate(disparity, cam1, cam2, bbox=None, angle_tol=0.0):
    """stereo_triangulate(disparity, cam1, cam2) (Stereo/StereoView.h:74-130) rasterised over bbox (x0, y0, x1, y1) or a BBox2i
    inside the image (None: the whole image).  Pixel (i, j) triangulates (i, j) against (i, j) + (double)disparity through
    StereoModel(cam1, cam2, angle_tol); invalid pixels give (0, 0, 0).  The cameras are both PinholeModels, or each a CAHVModel or
    a CAHVORModel (a pinhole with a CAHV-family camera is NoImplErr).  int32 or float32 (rows, cols, 3), numpy or CUDA;
    returns a (y1 - y0, x1 - x0, 3) float64 raster of the same kind."""
    t, ptr, cols, rows, pitch, dev, dt = _disparity_in(disparity)
    x0, y0, x1, y1 = _bbox(bbox) if bbox is not None else (0, 0, cols, rows)
    out = _output(t, (max(y1 - y0, 0), max(x1 - x0, 0), 3), np.float64)
    fn = lib().vwb200_cahv_stereo_triangulate if _family("stereo_triangulate", cam1, cam2) == "cahv" else lib().vwb200_stereo_triangulate
    c1, c2 = cam1._struct(), cam2._struct()
    _check(fn(_ptype(dt), ptr, cols, rows, pitch, x0, y0, x1 - x0, y1 - y0, C.byref(c1), C.byref(c2), float(angle_tol), _ptr(out), x1 - x0,
              dev, _stream_ptr() if dev else None))
    return out


def stereo_model_points(disparity, cam1, cam2, angle_tol=0.0):
    """StereoModel(cam1, cam2, angle_tol)(disparity_map, error) (Stereo/StereoModel.cc:254-309) of a float32 (rows, cols, 3)
    disparity, numpy or CUDA: (xyz float64 (rows, cols, 3), error float64 (rows, cols)).  last_triangulation_stats() gives
    what the reference prints."""
    t, ptr, cols, rows, pitch, dev, dt = _disparity_in(disparity)
    if dt != np.float32:
        raise ArgumentErr("StereoModel takes a float32 (PixelMask<Vector2f>) disparity")
    xyz, err = _output(t, (rows, cols, 3), np.float64), _output(t, (rows, cols), np.float64)
    fn = lib().vwb200_cahv_stereo_model_points if _family("StereoModel", cam1, cam2) == "cahv" else lib().vwb200_stereo_model_points
    c1, c2 = cam1._struct(), cam2._struct()
    _check(fn(ptr, cols, rows, pitch, C.byref(c1), C.byref(c2), float(angle_tol), _ptr(xyz), cols, _ptr(err), cols, dev,
              _stream_ptr() if dev else None))
    return xyz, err


class TriangulationStats(C.Structure):
    _fields_ = [("points", C.c_longlong), ("divergent", C.c_longlong), ("max_error", C.c_double), ("error_sum", C.c_double),
                ("tsai_iterations", C.c_longlong), ("cahvor_iterations", C.c_longlong)]


def last_triangulation_stats():
    """what the last stereo_model_points on this thread reports: points, divergent, max_error, error_sum (mean error =
    error_sum / points), and the Tsai Newton-Raphson (pinhole cameras) or CAHVOR Newton (CAHV cameras) iterations of the last
    stereo_triangulate or stereo_model_points"""
    s = TriangulationStats()
    lib().vwb200_last_triangulation_stats(C.byref(s))
    return {k: getattr(s, k) for k, _ in TriangulationStats._fields_}


def universe_radius(points, origin, near=0.0, far=DBL_MAX, out=None):
    """UniverseRadiusFunc(origin, near, far) (Stereo/StereoView.h:139-186) applied to a float64 (rows, cols, 3) point image,
    numpy or CUDA: (points, rejected, total).  out: None (a new raster) or points itself (in place).  ArgumentErr for
    radii that are not >= 0 and for near > far, as the reference's asserts."""
    t, ptr, cols, rows, pitch, dev = _raster(points, np.float64, channels=3)
    if out is None:
        out = _output(t, (rows, cols, 3), np.float64)
        opitch = cols
    elif out is points and t is points:
        opitch = pitch
    else:
        raise ArgumentErr("out must be None or the points themselves (a dense float64 raster)")
    o = np.ascontiguousarray(origin, np.float64)
    rej, tot = C.c_longlong(), C.c_longlong()
    _check(lib().vwb200_universe_radius(ptr, cols, rows, pitch, o.ctypes.data, float(near), float(far), _ptr(out), opitch, C.byref(rej),
                                        C.byref(tot), dev, _stream_ptr() if dev else None))
    return out, rej.value, tot.value


def _disparity_arg(disparity):
    """(pointer, cols, rows, pitch in pixels, on_device) of a float32 (rows, cols, 3) disparity that is filtered in place"""
    return _in_place(disparity, 3, lambda dev: "disparity must be a float32 CUDA tensor (rows, cols, 3) with dense pixels" if dev else
                     "disparity must be a writeable float32 (rows, cols, 3) array with dense pixels (it is filtered in place)")


def disparity_median_filter(disparity, kernel_size):
    """vw::stereo::disparity_median_filter (Stereo/Algorithms.cc:26-67).  Filters `disparity` (float32 (rows, cols, 3)
    {dx, dy, valid}: a numpy array, or a CUDA tensor on the current stream) IN PLACE, in raster order, as the reference's
    shallow `disparity_out = disparity_in` makes it do, and returns it."""
    ptr, cols, rows, pitch, dev = _disparity_arg(disparity)
    _check(lib().vwb200_disparity_median_filter(ptr, cols, rows, pitch, int(kernel_size), dev, _stream_ptr() if dev else None))
    return disparity


def texture_measure(image, kernel_size=9, gradient_weight=0.5, stddev_weight=0.5):
    """vw::stereo::texture_measure (Stereo/Algorithms.h:144-209) of a float image (numpy, or a CUDA tensor on the current
    stream): a new float32 image of the same size."""
    if not _is_torch(image) and _np(image, np.float32).ndim != 2:
        raise ArgumentErr("texture_measure: the image must be 2-D")
    t, ptr, cols, rows, pitch, dev = _raster(image, np.float32)
    out = _output(t, t.shape, np.float32)
    _check(lib().vwb200_texture_measure(ptr, cols, rows, pitch, int(kernel_size), float(gradient_weight), float(stddev_weight), _ptr(out),
                                        cols, dev, _stream_ptr() if dev else None))
    return out


def texture_preserving_disparity_filter(disparity, texture_image, texture_max=0.15, max_kernel_size=11):
    """vw::stereo::texture_preserving_disparity_filter<float> (Stereo/Algorithms.h:213-281): smooths `disparity` (as in
    disparity_median_filter: numpy or a CUDA tensor, filtered IN PLACE and returned) with a mean whose window shrinks as
    the texture grows.  A pixel whose kernel would exceed max_kernel_size is skipped silently."""
    ptr, cols, rows, pitch, dev = _disparity_arg(disparity)
    if dev and not (_is_torch(texture_image) and texture_image.is_cuda):
        raise ArgumentErr("the texture image must be a CUDA tensor when the disparity is one")
    keep, tptr, tcols, trows, tpitch, _ = _raster(texture_image if dev else _np(texture_image, np.float32), np.float32)
    if tuple(keep.shape) != (rows, cols):
        raise ArgumentErr("the texture image must have the disparity's size")
    _check(lib().vwb200_texture_preserving_disparity_filter(ptr, cols, rows, pitch, tptr, tpitch, float(texture_max), int(max_kernel_size),
                                                            dev, _stream_ptr() if dev else None))
    return disparity


class ParabolaSubpixelView:
    """vw::stereo::ParabolaSubpixelView (Stereo/ParabolaSubpixelView.h:27-117): lazy view refining an integer
    disparity (PixelMask<Vector2f> triples, same size as the left image) by a 2-D parabola fit."""

    def __init__(self, disparity, left_image, right_image, prefilter_mode, prefilter_width, kernel_size):
        self._d = _np(disparity, np.float32)
        self._l, self._r = _np(left_image, np.float32), _np(right_image, np.float32)
        if self._d.shape[:2] != self._l.shape:
            raise ArgumentErr("SubpixelView: Disparity image must match left image.")
        self._mode, self._width, self._k = int(prefilter_mode), float(prefilter_width), (int(kernel_size[0]), int(kernel_size[1]))

    def cols(self):
        return self._l.shape[1]

    def rows(self):
        return self._l.shape[0]

    def planes(self):
        return 1

    def __call__(self, i, j, p=0):
        raise NoImplErr("SubpixelView:operator() has not been implemented.")

    def rasterize(self, dest=None, bbox=None):
        b = _bbox(bbox) if bbox is not None else (0, 0, self.cols(), self.rows())
        w, h = b[2] - b[0], b[3] - b[1]
        if dest is None:
            dest = np.empty((h, w, 3), np.float32)
        _check(lib().vwb200_parabola_subpixel(self._d.ctypes.data, self.cols(), self.rows(), self._l.ctypes.data, self._l.shape[1],
                                              self._r.ctypes.data, self._r.shape[1], self._r.shape[0], self._r.shape[1],
                                              self._k[0], self._k[1], self._mode, self._width, b[0], b[1], b[2], b[3],
                                              dest.ctypes.data, dest.strides[0] // 12, 0, None))
        return dest

    prerasterize = rasterize


def parabola_subpixel(disparity, left_image, right_image, prefilter_mode, prefilter_width, kernel_size):
    """vw::stereo::parabola_subpixel (Stereo/ParabolaSubpixelView.h:111-117)."""
    return ParabolaSubpixelView(disparity, left_image, right_image, prefilter_mode, prefilter_width, kernel_size)


class BBox2i:
    """vw::BBox2i: half-open [min, max).  BBox2i(x, y, w, h) like Math/BBox.tcc:55-59."""

    def __init__(self, x=0, y=0, w=0, h=0):
        self.x0, self.y0, self.x1, self.y1 = x, y, x + w, y + h

    @classmethod
    def from_corners(cls, x0, y0, x1, y1):
        return cls(x0, y0, x1 - x0, y1 - y0)

    def width(self):
        return max(self.x1 - self.x0, 0)

    def height(self):
        return max(self.y1 - self.y0, 0)

    def __repr__(self):
        return f"BBox2i(({self.x0},{self.y0})-({self.x1},{self.y1}))"


class PyramidCorrelationView:
    """vw::stereo::PyramidCorrelationView (Stereo/CorrelationView.h:35-193) rasterised on an H100.

    Lazy like the reference: construction only records parameters and places the inputs in HBM;
    work happens in rasterize()/prerasterize(), one call per tile bbox, from any number of threads.
    """

    def __init__(self, left, right, left_mask, right_mask, prefilter_mode, prefilter_width,
                 search_region, kernel_size, cost_type, corr_timeout, seconds_per_op,
                 consistency_threshold, min_consistency_level, filter_half_kernel, max_pyramid_levels,
                 algorithm=VW_CORRELATION_BM, collar_size=0, sgm_subpixel_mode=SUBPIXEL_LC_BLEND, sgm_search_buffer=(2, 2),
                 memory_limit_mb=6000, blob_filter_area=0, lr_disp_diff=None, region_ul=(0, 0),
                 write_debug_images=False, sgm_threads=4, streamed=False):
        """Argument order = the reference constructor (Stereo/CorrelationView.h:48-69); sgm_threads stands for
        vw_settings().default_num_threads(), which SGM's memory estimate reads (SGM.cc:715-716).
        lr_disp_diff: float32 (rows, cols, 2) PixelMask<float> array whose pixel (0, 0) is image pixel region_ul; updated in place."""
        if isinstance(search_region, BBox2i):
            s = (search_region.x0, search_region.y0, search_region.x1, search_region.y1)
        else:
            s = tuple(int(v) for v in search_region)
        self._p = CorrParams(s[0], s[1], s[2], s[3], int(kernel_size[0]), int(kernel_size[1]), int(cost_type),
                             int(prefilter_mode), float(prefilter_width), float(consistency_threshold),
                             int(min_consistency_level), int(filter_half_kernel), int(max_pyramid_levels),
                             int(collar_size), int(corr_timeout), float(seconds_per_op), int(algorithm),
                             int(blob_filter_area), int(sgm_subpixel_mode), int(sgm_search_buffer[0]), int(sgm_search_buffer[1]),
                             int(region_ul[0]), int(region_ul[1]), int(bool(write_debug_images)), int(sgm_threads), float(memory_limit_mb))
        self._h = C.c_void_p()
        _check(lib().vwb200_corr_create(C.byref(self._p), C.byref(self._h)))
        self._diff = lr_disp_diff
        if lr_disp_diff is not None:
            ptr, cols, rows, pitch, dev = _in_place(lr_disp_diff, 2, lambda dev: "lr_disp_diff must be a float32 (rows, cols, 2) array")
            _check(lib().vwb200_corr_set_lr_disp_diff(self._h, ptr, cols, rows, pitch, dev))
        self._device = _is_torch(left)
        if self._device:
            import torch
            left_mask, right_mask = [m if m.dtype == torch.uint8 else m != 0 for m in (left_mask, right_mask)]
        l = _raster(left, np.float32)
        r, lm, rm = _raster(right, np.float32, on_device=l[5]), _raster(left_mask, np.uint8, on_device=l[5]), _raster(right_mask, np.uint8, on_device=l[5])
        if tuple(lm[0].shape) != tuple(l[0].shape) or tuple(rm[0].shape) != tuple(r[0].shape):
            raise ArgumentErr("masks must have the size of their images")
        # the library copies host rasters into HBM, except streamed ones: each rasterize() uploads its tile's region of interest
        self._keep = tuple(x[0] for x in (l, r, lm, rm)) if self._device or streamed else None
        _check(lib().vwb200_corr_set_inputs(self._h, *l[1:5], *r[1:5], lm[1], lm[4], rm[1], rm[4], 1 if self._device else 2 if streamed else 0))

    def __del__(self):
        try:
            if self._h:
                lib().vwb200_corr_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # --- standard ImageView interface (CorrelationView.h:109-117) ---
    def cols(self):
        return lib().vwb200_corr_cols(self._h)

    def rows(self):
        return lib().vwb200_corr_rows(self._h)

    def planes(self):
        return 1

    def __call__(self, i, j, p=0):
        raise NoImplErr("NewCorrelationView::operator() is not implemented.")

    def num_levels(self, bbox):
        b = _bbox(bbox)
        return lib().vwb200_corr_num_levels(self._h, b[2] - b[0], b[3] - b[1])

    def rasterize(self, dest=None, bbox=None):
        """rasterize(dest, bbox) (CorrelationView.h:123-133).  dest: float32 (h, w, 3) numpy array (or torch
        CUDA tensor) already sized to bbox, or None to allocate.  Pixels are {dx, dy, valid}."""
        return self._run(lib().vwb200_corr_rasterize, dest, bbox)

    def _run(self, fn, dest, bbox):
        b = _bbox(bbox) if bbox is not None else (0, 0, self.cols(), self.rows())
        w, h = b[2] - b[0], b[3] - b[1]
        if dest is None:
            dest = _output(self._keep[0] if self._device else None, (h, w, 3), np.float32)
        assert tuple(dest.shape) == (h, w, 3)
        ptr, _, _, pitch, dev = _in_place(dest, 3, lambda dev: "dest must be a float32 (h, w, 3) raster with dense pixels")
        _check(fn(self._h, b[0], b[1], b[2], b[3], ptr, pitch, dev, _stream_ptr() if dev else None))
        return dest

    def prerasterize(self, bbox):
        """prerasterize(bbox): an owning buffer of bbox size (CorrelationView.cc:880-884); processes exactly bbox --
        unlike rasterize() no collar is added (CorrelationView.h:123-133)."""
        return self._run(lib().vwb200_corr_prerasterize, None, bbox)


def _bbox(b):
    if isinstance(b, BBox2i):
        return (b.x0, b.y0, b.x1, b.y1)
    return tuple(int(v) for v in b)


def pyramid_correlate(left, right, left_mask, right_mask, prefilter_mode, prefilter_width, search_region, kernel_size,
                      cost_type, corr_timeout, seconds_per_op, consistency_threshold, min_consistency_level,
                      filter_half_kernel, max_pyramid_levels, algorithm=VW_CORRELATION_BM, collar_size=0,
                      sgm_subpixel_mode=SUBPIXEL_LC_BLEND, sgm_search_buffer=(2, 2), memory_limit_mb=6000, blob_filter_area=0,
                      lr_disp_diff=None, region_ul=(0, 0), write_debug_images=False, **kw):
    """vw::stereo::pyramid_correlate (Stereo/CorrelationView.h:195-230), same positional order."""
    return PyramidCorrelationView(left, right, left_mask, right_mask, prefilter_mode, prefilter_width, search_region,
                                  kernel_size, cost_type, corr_timeout, seconds_per_op, consistency_threshold,
                                  min_consistency_level, filter_half_kernel, max_pyramid_levels, algorithm,
                                  collar_size, sgm_subpixel_mode, sgm_search_buffer, memory_limit_mb, blob_filter_area,
                                  lr_disp_diff, region_ul, write_debug_images, **kw)


PIXEL_GRAY_F32, PIXEL_MASK_F32 = 0, 1


def epipolar(cam0, cam1):
    """epipolar(cam0, cam1, epi0, epi1) (Camera/PinholeModel.cc:679-732): two rectified PinholeModels at the sources' centers,
    sharing one rotation (baseline as u), the mean focal length, point offset and pixel pitch, the NULL lens and the default
    u, v, w frame.  Host arithmetic, bit for bit the reference's; coincident centers give NaN cameras.  For two CAHVModels,
    epipolar(CAHVModel, CAHVModel) (Camera/CAHVModel.cc:297-337): two CAHVModels at the sources' centers sharing A, H and V."""
    if _family("epipolar", cam0, cam1) == "cahv":
        a, b = Cahv(), Cahv()
        _check(lib().vwb200_cahv_epipolar(C.byref(cam0._struct()), C.byref(cam1._struct()), C.byref(a), C.byref(b)))
        return _cahv_from_struct(a), _cahv_from_struct(b)
    a, b = Pinhole(), Pinhole()
    _check(lib().vwb200_pinhole_epipolar(C.byref(cam0._struct()), C.byref(cam1._struct()), C.byref(a), C.byref(b)))
    return PinholeModel._from_struct(a), PinholeModel._from_struct(b)


def _roi(r):
    return (C.c_int32 * 4)(*_bbox(r))


def resize_epipolar_cameras_to_fit(cam1, cam2, epi1, epi2, roi1, roi2):
    """resize_epipolar_cameras_to_fit (Camera/EpipolarUtils.cc:37-76): (epi1, epi2, size1, size2) -- new epipolar cameras whose
    point offsets put both transformed ROIs (x0, y0, x1, y1) or BBox2i at (0, 0), and the (width, height) that holds each.
    The ROI perimeters go through CameraTransform(cam, epi)::forward on the device.  PointToPixelErr where the reference throws,
    LogicErr for a camera and its epipolar camera at different centers."""
    e1, e2 = epi1._struct(), epi2._struct()
    s1, s2 = (C.c_int32 * 2)(), (C.c_int32 * 2)()
    _check(lib().vwb200_resize_epipolar_cameras_to_fit(C.byref(cam1._struct()), C.byref(cam2._struct()), C.byref(e1), C.byref(e2), _roi(roi1),
                                                      _roi(roi2), s1, s2, None))
    return PinholeModel._from_struct(e1), PinholeModel._from_struct(e2), (s1[0], s1[1]), (s2[0], s2[1])


def camera_transform(image, src_camera, dst_camera, bbox=None, size=None, edge=EDGE_ZERO, interp=INTERP_BILINEAR, edge_value=None):
    """camera_transform(image, src_camera, dst_camera[, size | bbox], edge, interp) (Camera/CameraTransform.h:125-183),
    rasterised: the image resampled from src_camera into dst_camera (both at one center, else LogicErr) through
    reverse(p) = src.point_to_pixel(dst.pixel_to_vector(p) + C).  The output covers bbox (x0, y0, x1, y1) or a BBox2i, or
    (0, 0, width, height) for size=(width, height); with neither, the image's own extent.  image: float32 (rows, cols) -- any
    interpolation, zero or constant edges -- or PixelMask<float> (rows, cols, 2) {value, valid} -- bilinear, with zero,
    constant or value edges (edge_value {value, valid}, default PixelMask<float>() = (0, 0)); numpy or CUDA.  Bit for bit the
    reference's where both reversed coordinates are finite with |c| < 2^30; 0 ({0, 0}) elsewhere.  PointToPixelErr, naming the
    first failing pixel, where the reference throws.  Returns a new raster where the image lives.  The cameras are both
    PinholeModels, or a CAHVModel / CAHVORModel src and a CAHVModel dst (no check, so no PointToPixelErr); a pinhole with a
    CAHV-family camera is NoImplErr."""
    masked = len(image.shape) == 3
    if masked and image.shape[2] != 2 or len(image.shape) not in (2, 3):
        raise ArgumentErr("camera_transform: the image must be float32 (rows, cols) or PixelMask<float> (rows, cols, 2)")
    t, ptr, cols, rows, pitch, dev = _raster(image, np.float32, channels=2 if masked else 1)
    if size is not None:
        x0, y0, x1, y1 = 0, 0, int(size[0]), int(size[1])
    else:
        x0, y0, x1, y1 = _bbox(bbox) if bbox is not None else (0, 0, cols, rows)
    ev = (C.c_float * 2)(*(edge_value if edge_value is not None else (0.0, 0.0)))
    out = _output(t, (max(y1 - y0, 0), max(x1 - x0, 0)) + ((2,) if masked else ()), np.float32)
    fn = lib().vwb200_cahv_camera_transform if _family("camera_transform", src_camera, dst_camera) == "cahv" else lib().vwb200_camera_transform
    _check(fn(C.byref(src_camera._struct()), C.byref(dst_camera._struct()), PIXEL_MASK_F32 if masked else PIXEL_GRAY_F32, int(interp), int(edge),
              ev, ptr, cols, rows, pitch, x0, y0, _ptr(out), x1 - x0, y1 - y0, x1 - x0, dev, _stream_ptr() if dev else None))
    return out


def epipolar_transformed_images(left_camera, right_camera, left_epi_camera, right_epi_camera, left_image, right_image, left_size, right_size,
                                edge_value=(0.0, 0.0), left_roi=None, right_roi=None):
    """epipolar_transformed_images (Camera/EpipolarUtils.cc:79-144) for PinholeModels with NULL or TSAI lenses (fitPinholeModel
    returns those unchanged): both PixelMask<float> (rows, cols, 2) images resampled into their epipolar cameras at
    left_size / right_size (width, height), bilinear, ValueEdgeExtension(edge_value).  A ROI whose origin is not (0, 0) (the
    AdjustedCameraModel branch) is NoImplErr."""
    for roi in (left_roi, right_roi):
        if roi is not None and tuple(_bbox(roi)[:2]) != (0, 0):
            raise NoImplErr("epipolar_transformed_images: a ROI whose origin is not (0, 0) has no device form")
    return (camera_transform(left_image, left_camera, left_epi_camera, size=left_size, edge=EDGE_VALUE, edge_value=edge_value),
            camera_transform(right_image, right_camera, right_epi_camera, size=right_size, edge=EDGE_VALUE, edge_value=edge_value))


# ---- CAHV / CAHVOR cameras (Camera/CAHVModel.cc, CAHVORModel.cc, CameraTransform.h:185-225, EpipolarUtils.cc:148-222) ---------
CAMERA_CAHV, CAMERA_CAHVOR = 1, 2


class Cahv(C.Structure):
    _fields_ = [("model", C.c_int), ("C", C.c_double * 3), ("A", C.c_double * 3), ("H", C.c_double * 3), ("V", C.c_double * 3),
                ("O", C.c_double * 3), ("R", C.c_double * 3)]


def _vec3(v):
    return tuple(float(x) for x in v)


_WS = " \t\n\v\f\r"
_DOUBLE = re.compile(r"[+-]?(\d*)(?:\.(\d*))?")
_EXPONENT = re.compile(r"[eE][+-]?(\d*)")


class _TextIn:
    """the std::istream reads of the reference's camera readers (C locale): ignore(n, delim), >> char and >> double.  A double
    is what num_get accumulates -- sign, digits, a decimal point, an exponent -- converted as a whole, so "nan", "inf", hex,
    a bare "." or "1e" and a value that overflows fail; any failure is IOErr, as the reference's failbit exception is."""

    def __init__(self, text, what):
        self.t, self.p, self.what = text, 0, what

    def fail(self, msg="Could not read file"):
        raise IOErr(f"{self.what}: {msg}")

    def ignore(self, n, delim):
        k = self.t.find(delim, self.p, self.p + n)
        self.p = min(len(self.t), self.p + n) if k < 0 else k + 1

    def _skip(self):
        while self.p < len(self.t) and self.t[self.p] in _WS:
            self.p += 1
        if self.p >= len(self.t):
            self.fail()

    def char(self):
        self._skip()
        self.p += 1
        return self.t[self.p - 1]

    def double(self):
        self._skip()
        m = _DOUBLE.match(self.t, self.p)
        end, digits = m.end(), (m.group(1) or "") + (m.group(2) or "")
        if digits:
            e = _EXPONENT.match(self.t, end)
            if e:
                end = e.end()
                if not e.group(1):
                    self.fail()
        if not digits:
            self.fail()
        v = float(self.t[self.p:end])
        if v in (float("inf"), float("-inf")):
            self.fail()
        self.p = end
        return v


def _read_vectors(path, names, what):
    """the readers of CAHVModel.cc:194-231 and CAHVORModel.cc:30-80: skip to "C" followed by "=", then the vectors, each after
    its letter and "="""
    with open(path) as f:
        s = _TextIn(f.read(), what)
    while True:
        s.ignore(1024, "C")
        if s.char() == "=":
            break
    out = [tuple(s.double() for _ in range(3))]
    for name in names[1:]:
        if s.char() != name or s.char() != "=":
            s.fail(f"Could not read {name} vector")
        out.append(tuple(s.double() for _ in range(3)))
    return out


def _write_vectors(path, pairs):
    with open(path, "w") as f:
        for name, v in pairs:
            f.write(f"{name} = " + " ".join(format(x, ".20g") for x in v) + "\n")


class CAHVModel:
    """camera::CAHVModel(C, A, H, V) (Camera/CAHVModel.h): the four vectors as public fields.  read() / write() use the
    reference's text format (any leading text is skipped up to "C ="; written with 20 significant digits)."""
    type_name = "CAHV"

    def __init__(self, C=(0, 0, 0), A=(0, 0, 0), H=(0, 0, 0), V=(0, 0, 0)):
        self.C, self.A, self.H, self.V = _vec3(C), _vec3(A), _vec3(H), _vec3(V)

    def camera_center(self, pix=None):
        return self.C

    def type(self):
        return self.type_name

    @classmethod
    def read(cls, path):
        return cls(*_read_vectors(path, "CAHV", "CAHVModel"))

    def write(self, path):
        _write_vectors(path, zip("CAHV", (self.C, self.A, self.H, self.V)))

    @classmethod
    def from_pinhole(cls, pinhole):
        """CAHVModel = PinholeModel (CAHVModel.cc:64-99) of a NULL-lens pinhole, on the host"""
        out = Cahv()
        _check(lib().vwb200_pinhole_to_cahv(C.byref(pinhole._struct()), C.byref(out)))
        return _cahv_from_struct(out)

    def _struct(self):
        s = Cahv()
        s.model = CAMERA_CAHV
        s.C[:], s.A[:], s.H[:], s.V[:] = self.C, self.A, self.H, self.V
        return s

    def __repr__(self):
        return f"{type(self).__name__}(C={self.C}, A={self.A}, H={self.H}, V={self.V})"


class CAHVORModel(CAHVModel):
    """camera::CAHVORModel(C, A, H, V, O, R) (Camera/CAHVORModel.h): CAHV plus the optical axis O and the radial distortion
    terms R"""
    type_name = "CAHVOR"

    def __init__(self, C=(0, 0, 0), A=(0, 0, 0), H=(0, 0, 0), V=(0, 0, 0), O=(0, 0, 0), R=(0, 0, 0)):
        super().__init__(C, A, H, V)
        self.O, self.R = _vec3(O), _vec3(R)

    @classmethod
    def read(cls, path):
        return cls(*_read_vectors(path, "CAHVOR", "CAHVORModel"))

    def write(self, path):
        _write_vectors(path, zip("CAHVOR", (self.C, self.A, self.H, self.V, self.O, self.R)))

    def _struct(self):
        s = super()._struct()
        s.model = CAMERA_CAHVOR
        s.O[:], s.R[:] = self.O, self.R
        return s

    def __repr__(self):
        return f"CAHVORModel(C={self.C}, A={self.A}, H={self.H}, V={self.V}, O={self.O}, R={self.R})"


def _cahv_from_struct(s):
    if s.model == CAMERA_CAHVOR:
        return CAHVORModel(s.C[:], s.A[:], s.H[:], s.V[:], s.O[:], s.R[:])
    return CAHVModel(s.C[:], s.A[:], s.H[:], s.V[:])


def _family(what, *cams):
    """"pinhole" when every camera is a PinholeModel, "cahv" when every one is a CAHVModel / CAHVORModel; NoImplErr for a mix"""
    if all(isinstance(c, PinholeModel) for c in cams):
        return "pinhole"
    if all(isinstance(c, CAHVModel) for c in cams):
        return "cahv"
    raise NoImplErr(f"{what}: pinhole and CAHV-family cameras in one call have no device form")


def linearize_camera(camera_model, cahvor_image_size, cahv_image_size):
    """linearize_camera(CAHVORModel, cahvor_image_size, cahv_image_size) (Camera/CAHVORModel.cc:460-547), on the host: the
    CAHVModel at the same center with A the normalised sum of 12 perimeter rays and H, V spanning the smaller field of view.
    Sizes are (width, height)."""
    if not isinstance(camera_model, CAHVORModel):
        raise ArgumentErr("linearize_camera takes a CAHVORModel")
    out = Cahv()
    _check(lib().vwb200_linearize_camera(C.byref(camera_model._struct()), (C.c_int32 * 2)(*cahvor_image_size), (C.c_int32 * 2)(*cahv_image_size),
                                         C.byref(out)))
    return _cahv_from_struct(out)


def linearize_camera_transform(image, camera_model, edge=EDGE_ZERO, interp=INTERP_BILINEAR, edge_value=None):
    """linearize_camera_transform(image, cahvor[, edge, interp]) (Camera/CameraTransform.h:185-225): the image resampled from
    camera_model into linearize_camera(camera_model, size, size) of its own size (cols, rows)"""
    rows, cols = image.shape[0], image.shape[1]
    lin = linearize_camera(camera_model, (cols, rows), (cols, rows))
    return camera_transform(image, camera_model, lin, edge=edge, interp=interp, edge_value=edge_value)


def epipolar_transformed_cahv_images(left_camera, right_camera, left_epi_camera, right_epi_camera, left_image, right_image,
                                     edge_value=(0.0, 0.0)):
    """the CAHV and CAHVOR branches of epipolar_transformed_cahv_images (Camera/EpipolarUtils.cc:148-222): both PixelMask<float>
    (rows, cols, 2) images resampled from their CAHV / CAHVOR cameras into the epipolar CAHV cameras at their own size,
    bilinear, ValueEdgeExtension(edge_value)"""
    for c in (left_epi_camera, right_epi_camera):
        if type(c) is not CAHVModel:
            raise ArgumentErr("epipolar_transformed_cahv_images: the epipolar cameras must be CAHVModels")
    return (camera_transform(left_image, left_camera, left_epi_camera, edge=EDGE_VALUE, edge_value=edge_value),
            camera_transform(right_image, right_camera, right_epi_camera, edge=EDGE_VALUE, edge_value=edge_value))


# ---- exact interest point matching (InterestPoint/Matcher.h:415-509, Matcher.cc:33-195, MatcherIO.cc:248-365) --------------
METRIC_L2, METRIC_HAMMING = 0, 1
_METRICS = {"l2": METRIC_L2, "hamming": METRIC_HAMMING}


class IpMatchStats(C.Structure):
    _fields_ = [("pairs", C.c_longlong), ("matches", C.c_longlong), ("metric", C.c_int32), ("splits", C.c_int32)]


def _points(desc, pol, what, on_device=None):
    """(keep-alive, descriptor pointer, n, dim, pitch, polarity pointer, on_device) of an (n, dim) float32 descriptor list and
    its n polarities"""
    if len(desc.shape) != 2:
        raise ArgumentErr(f"ip_match: {what} descriptors must be (n, dim), not {tuple(desc.shape)}")
    if _is_torch(desc):
        import torch
        d = desc.to(torch.float32)
        if d.stride(1) != 1 or d.shape[0] > 1 and d.stride(0) < d.shape[1]:
            d = d.contiguous()
        p = (pol if _is_torch(pol) else torch.as_tensor(np.asarray(pol))).to(device=d.device, dtype=torch.bool).to(torch.uint8).contiguous()
        r = ((d, p), d.data_ptr(), d.shape[0], d.shape[1], max(d.stride(0), d.shape[1]), p.data_ptr(), 1)
    else:
        d = _np(desc, np.float32)
        p = np.ascontiguousarray(np.asarray(pol).astype(bool), np.uint8)
        r = ((d, p), d.ctypes.data, d.shape[0], d.shape[1], d.shape[1], p.ctypes.data, 0)
    if tuple(p.shape) != (r[2],):
        raise ArgumentErr(f"ip_match: {what} has {r[2]} descriptors but polarities of shape {tuple(p.shape)}")
    if on_device is not None and r[6] != on_device:
        raise ArgumentErr("ip_match: the inputs must all be numpy arrays or all be CUDA tensors")
    return r


def ip_match(desc1, pol1, desc2, pol2, threshold=0.5, metric="l2", distances=False):
    """InterestPointMatcherSimple<L2NormMetric | HammingMetric, NullConstraint>(threshold) over two interest point lists given
    as (n, dim) float32 descriptors and n polarities each (numpy arrays, or CUDA tensors on the current stream).  Returns the
    int32 match index of every ip1 (-1: no match) where the inputs live; with distances=True also the reference's float64
    first_pick / second_pick per ip1 (1e100 where none).  The matched pairs are (i, index[i]) for index[i] >= 0, in the
    reference's order.  metric "hamming" compares the bytes static_cast<uint8>(value): a value outside (-1, 256) or NaN is
    ArgumentErr, a dim above 2^21 NoImplErr.  Descriptors of unequal length are ArgumentErr."""
    if metric not in _METRICS:
        raise ArgumentErr(f"ip_match: unknown metric {metric!r} (l2 or hamming)")
    k1, d1, n1, dim1, p1, q1, dev = _points(desc1, pol1, "ip1")
    k2, d2, n2, dim2, p2, q2, _ = _points(desc2, pol2, "ip2", on_device=dev)
    if dim1 != dim2 and n1 and n2:
        raise ArgumentErr(f"ip_match: descriptors of unequal length ({dim1} and {dim2})")
    dim = dim1 if n1 else dim2
    index = _output(k1[0], (n1,), np.int32)
    first = _output(k1[0], (n1,), np.float64) if distances else None
    second = _output(k1[0], (n1,), np.float64) if distances else None
    _check(lib().vwb200_ip_match(_METRICS[metric], d1, q1, n1, d2, q2, n2, dim, max(p1, dim), max(p2, dim), float(threshold), _ptr(index),
                                 _ptr(first) if distances else None, _ptr(second) if distances else None, dev, _stream_ptr() if dev else None))
    return (index, first, second) if distances else index


def last_ipmatch_stats():
    """what the last ip_match on this thread did: descriptor pairs scanned, the metric, the CTAs its candidate range was split
    over (1: not split, 0: no candidates) and the matches kept"""
    s = IpMatchStats()
    lib().vwb200_last_ipmatch_stats(C.byref(s))
    return {"pairs": int(s.pairs), "matches": int(s.matches), "metric": "hamming" if s.metric == METRIC_HAMMING else "l2",
            "splits": int(s.splits)}


def remove_duplicates(xy1, xy2):
    """remove_duplicates(ip1, ip2) (Matcher.cc:151-195) on the (n, 2) float32 (x, y) of matched pairs: the int32 indices of the
    pairs kept, in order.  Walking from the last pair to the first, a pair is dropped when its ip1 or its ip2 position was
    already kept (-0.0 equals 0.0).  A NaN coordinate is ArgumentErr."""
    a = _np(np.asarray(xy1.cpu() if _is_torch(xy1) else xy1), np.float32).reshape(-1, 2)
    b = _np(np.asarray(xy2.cpu() if _is_torch(xy2) else xy2), np.float32).reshape(-1, 2)
    if a.shape != b.shape:
        raise ArgumentErr("remove_duplicates: Input vectors are not the same size.")
    keep = np.empty(len(a), np.int32)
    n = C.c_int()
    _check(lib().vwb200_remove_duplicate_matches(a.ctypes.data, b.ctypes.data, len(a), keep.ctypes.data, C.byref(n)))
    return keep[:n.value].copy()


# the packed little-endian record of write_ip_record (MatcherIO.cc:248-263) ahead of its dim descriptor floats
_IP_FIELDS = [("x", "<f4"), ("y", "<f4"), ("ix", "<i4"), ("iy", "<i4"), ("orientation", "<f4"), ("scale", "<f4"), ("interest", "<f4"),
              ("polarity", "u1"), ("octave", "<u4"), ("scale_lvl", "<u4"), ("size", "<u8")]
_IP_HEAD = np.dtype(_IP_FIELDS)          # 45 bytes, unaligned


def _ip_dtype(dim):
    return np.dtype(_IP_FIELDS + [("descriptor", "<f4", (dim,))])


def interest_points(x, y, descriptor, polarity=None, scale=None, interest=None, orientation=None, octave=None, scale_lvl=None,
                    ix=None, iy=None):
    """an interest point list as the .vwip record array: InterestPoint(x, y, scale=1, interest=0, ori=0, pol=false, octave=0,
    scale_lvl=0)'s defaults (ix, iy = int32(x), int32(y)) for the fields not given; descriptor is (n, dim)"""
    d = np.asarray(descriptor, np.float32)
    n = len(d)
    rec = np.zeros(n, _ip_dtype(d.shape[1] if d.ndim == 2 else 0))
    rec["x"], rec["y"] = x, y
    rec["ix"] = np.asarray(x, np.float32).astype(np.int32) if ix is None else ix
    rec["iy"] = np.asarray(y, np.float32).astype(np.int32) if iy is None else iy
    rec["scale"] = 1.0 if scale is None else scale
    for name, v in (("interest", interest), ("orientation", orientation), ("polarity", polarity), ("octave", octave), ("scale_lvl", scale_lvl)):
        if v is not None:
            rec[name] = v
    rec["size"] = rec.dtype["descriptor"].shape[0]
    rec["descriptor"] = d.reshape(n, -1)
    return rec


def _read_records(buf, offset, n):
    if n == 0:
        return np.zeros(0, _ip_dtype(0)), offset
    if len(buf) < offset + _IP_HEAD.itemsize:
        raise IOError("Failed to read interest point from file.")
    dim = int(np.frombuffer(buf, "<u8", 1, offset + _IP_HEAD.itemsize - 8)[0])
    dt = _ip_dtype(dim)
    if len(buf) < offset + n * dt.itemsize:
        raise IOError("Failed to read interest point from file.")
    rec = np.frombuffer(buf, dt, n, offset).copy()
    if np.any(rec["size"] != dim):
        raise ValueError("interest point records with descriptors of different lengths are not supported")
    return rec, offset + n * dt.itemsize


def write_binary_ip_file(path, points):
    """write_binary_ip_file (MatcherIO.cc:292-303): a u64 count, then the packed records of an interest_points() array"""
    rec = np.asarray(points)
    with open(path, "wb") as f:
        f.write(np.uint64(len(rec)).astype("<u8").tobytes())
        f.write(rec.tobytes())


def read_binary_ip_file(path):
    """read_binary_ip_file (MatcherIO.cc:305-322) as an interest_points() record array (every descriptor of one length)"""
    with open(path, "rb") as f:
        buf = f.read()
    if len(buf) < 8:
        return np.zeros(0, _ip_dtype(0))
    return _read_records(buf, 8, int(np.frombuffer(buf, "<u8", 1, 0)[0]))[0]


def write_binary_match_file(path, ip1, ip2):
    """write_binary_match_file (MatcherIO.cc:344-366): the two u64 counts, the ip1 records, then the ip2 records"""
    a, b = np.asarray(ip1), np.asarray(ip2)
    if len(a) != len(b):
        raise IOError("The vectors of matching interest points must have the same size.")
    with open(path, "wb") as f:
        f.write(np.array([len(a), len(b)], "<u8").tobytes())
        f.write(a.tobytes())
        f.write(b.tobytes())


def read_binary_match_file(path):
    """read_binary_match_file: (ip1, ip2) record arrays of a .match file"""
    with open(path, "rb") as f:
        buf = f.read()
    if len(buf) < 16:
        raise IOError(f"Failed to read {path} as a match file.")
    n1, n2 = (int(v) for v in np.frombuffer(buf, "<u8", 2, 0))
    ip1, off = _read_records(buf, 16, n1)
    ip2, _ = _read_records(buf, off, n2)
    return ip1, ip2


# ---- a20 / K12: interest point detection and description (ipfind --interest-operator iagd, sgrad descriptor) ----------
class IpPoint(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("ix", C.c_int32), ("iy", C.c_int32), ("scale", C.c_float),
                ("interest", C.c_float), ("orientation", C.c_float)]


class IpfindStats(C.Structure):
    _fields_ = [("tiles", C.c_longlong), ("extrema", C.c_longlong), ("kept", C.c_longlong), ("culled_tiles", C.c_longlong),
                ("described", C.c_longlong)]


_IPF_POINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("ix", "<i4"), ("iy", "<i4"), ("scale", "<f4"), ("interest", "<f4"),
                       ("orientation", "<f4")])
_IPF_READY = False
_IPF_EARG = -1                                  # vwb200_ipfind_detect: more points than cap (*n holds the count)
SGRAD_SIZE = 180


def _ipf():
    global _IPF_READY
    L = lib()
    if not _IPF_READY:
        P, I, Z, LL = C.c_void_p, C.c_int, C.c_ssize_t, C.c_longlong
        L.vwb200_ipfind_normalize.argtypes = [P, I, I, Z, I, C.c_double, P, Z, I, P]
        L.vwb200_ipfind_detect.argtypes = [P, I, I, Z, I, I, P, LL, C.POINTER(LL), I, P]
        L.vwb200_ipfind_remove_near_nodata.argtypes = [P, I, I, Z, C.c_double, I, P, C.POINTER(LL), I, P]
        L.vwb200_ipfind_describe.argtypes = [P, I, I, Z, I, P, LL, P, I, P]
        L.vwb200_ipfind_gaussian_taps.argtypes = [P]
        L.vwb200_last_ipfind_stats.argtypes = [C.POINTER(IpfindStats)]
        _IPF_READY = True
    return L


def _image2d(image, what):
    if not _is_torch(image) and _np(image, np.float32).ndim != 2:
        raise ArgumentErr(f"{what}: the image must be 2-D")
    return _raster(image, np.float32)


def _ipf_points(points):
    """the vwb200_ip_point array of an interest_points() record array (or of any array with x, y fields)"""
    rec = np.asarray(points)
    p = np.zeros(len(rec), _IPF_POINT)
    names = rec.dtype.names or ()
    if "x" not in names or "y" not in names:
        raise ArgumentErr("points need x and y fields")
    p["x"], p["y"] = rec["x"], rec["y"]
    p["ix"] = rec["ix"] if "ix" in names else rec["x"].astype(np.float32).astype(np.int32)
    p["iy"] = rec["iy"] if "iy" in names else rec["y"].astype(np.float32).astype(np.int32)
    p["scale"] = rec["scale"] if "scale" in names else 1.0
    for f in ("interest", "orientation"):
        if f in names:
            p[f] = rec[f]
    return p


def _ipf_records(p, descriptor=None, base=None):
    """an interest_points() record array of vwb200_ip_point p (the other fields from `base`, in p's order, or their defaults)"""
    d = np.zeros((len(p), 0), np.float32) if descriptor is None else np.asarray(descriptor, np.float32)
    rec = np.zeros(len(p), _ip_dtype(d.shape[1]))
    for f in ("x", "y", "ix", "iy", "scale", "interest", "orientation"):
        rec[f] = p[f]
    rec["size"] = d.shape[1]
    rec["descriptor"] = d
    if base is not None:
        for f in ("polarity", "octave", "scale_lvl"):
            rec[f] = base[f]
    return rec


def normalize(image, nodata=None):
    """normalize(image) to [0, 1] (Image/AutoNormalize.h:76-86), or with nodata apply_mask(normalize(create_mask(image,
    nodata))): the min / max are those of the pixels != float32(nodata), which become 0.  NaN / inf anywhere, or no valid
    pixel, is ArgumentErr.  Returns a new float32 raster where the image lives."""
    t, ptr, cols, rows, pitch, dev = _image2d(image, "normalize")
    out = _output(t, (rows, cols), np.float32)
    _check(_ipf().vwb200_ipfind_normalize(ptr, cols, rows, pitch, nodata is not None, 0.0 if nodata is None else float(nodata), _ptr(out),
                                          cols, dev, _stream_ptr() if dev else None))
    return out


def ipfind_gaussian_taps():
    """generate_gaussian_kernel(k, 2, 9): the nine Harris taps of the detector (float64)"""
    k = np.zeros(9, np.float64)
    _check(_ipf().vwb200_ipfind_gaussian_taps(k.ctypes.data))
    return k


def detection_tile_count(cols, rows, tile_size=1024):
    ts = max(1024, int(tile_size))
    return (-(-cols // ts)) * (-(-rows // ts)) if cols > 0 and rows > 0 else 0


def tile_num_ip(tile_w, tile_h, ip_per_tile, tile_size=1024):
    """InterestDetectionQueue's per-tile count (DetectorBase.h:276-290): clamp(ceil(area / tile^2 * desired), 1, desired);
    0 (keep every point) when ip_per_tile is 0"""
    if ip_per_tile <= 0:
        return 0
    ts = max(1024, int(tile_size))
    return max(1, min(int(math.ceil(float(tile_w) * tile_h / (float(ts) * ts) * float(ip_per_tile))), int(ip_per_tile)))


def ip_per_tile_for_image(ip_per_image, cols, rows, tile_size=1024):
    """ipfind.cc:255-262: max(1, ceil(ip_per_image / (cols * rows / tile_size^2))) with the unclamped tile_size"""
    num_tiles = cols * rows / float(tile_size * tile_size)
    return max(1, int(math.ceil(ip_per_image / num_tiles)))


def detect_interest_points_iagd(image, ip_per_tile=250, tile_size=1024):
    """detect_interest_points(image, IntegralAutoGainDetector(ip_per_tile), ip_per_tile) (InterestPoint/DetectorBase.h:250-328,
    IntegralDetector.cc:264-370) on a float32 image, numpy or CUDA, usually normalize()'s output.  tile_size is the default
    tile size (tiles are max(1024, tile_size) square); ip_per_tile 0 keeps every point.  Returns an interest_points() array
    with empty descriptors, in the reference's order."""
    if ip_per_tile < 0:
        raise ArgumentErr("detect_interest_points_iagd: ip_per_tile must be >= 0")
    t, ptr, cols, rows, pitch, dev = _image2d(image, "detect_interest_points_iagd")
    ntiles = detection_tile_count(cols, rows, tile_size)
    cap = ntiles * int(ip_per_tile) if ip_per_tile > 0 else max(4096, cols * rows // 64)
    n = C.c_longlong()
    while True:
        p = np.zeros(max(cap, 1), _IPF_POINT)
        rc = _ipf().vwb200_ipfind_detect(ptr, cols, rows, pitch, int(tile_size), int(ip_per_tile), p.ctypes.data, cap, C.byref(n), dev,
                                         _stream_ptr() if dev else None)
        if rc == _IPF_EARG and n.value > cap:
            cap = n.value
            continue
        _check(rc)
        break
    return _ipf_records(p[:n.value])



def remove_ip_near_nodata(raw_image, points, nodata=0.0, radius=1):
    """remove_ip_near_nodata(raw, nodata, list, radius) (InterestPoint/InterestPointUtils.h:45-82): drops the points whose
    (ix, iy) lies within radius of the image border or whose (2 radius + 1)^2 window holds a pixel equal to nodata (compared
    in double).  Returns the kept records of `points`, in order."""
    rec = np.asarray(points)
    p = _ipf_points(rec)
    t, ptr, cols, rows, pitch, dev = _image2d(raw_image, "remove_ip_near_nodata")
    n = C.c_longlong(len(p))
    idx = np.arange(len(p), dtype=np.int32)
    p["interest"] = idx.view(np.float32)          # carry each point's index through the compaction
    _check(_ipf().vwb200_ipfind_remove_near_nodata(ptr, cols, rows, pitch, float(nodata), int(radius), p.ctypes.data, C.byref(n), dev,
                                                   _stream_ptr() if dev else None))
    return rec[p["interest"][:n.value].view(np.int32)].copy()


def describe_sgrad(image, points, tile_size=1024):
    """describe_interest_points(image, SGradDescriptorGenerator, list) (InterestPoint/Descriptor.h:202-355, 414-471) on a
    float32 image, numpy or CUDA: the list is reordered as the reference's per-tile std::partition does, x / y take its crop
    round trip's float rounding, and each point gets the 180-float SGrad descriptor.  Returns a new interest_points() array."""
    rec = np.asarray(points)
    p = _ipf_points(rec)
    p_idx = np.arange(len(p), dtype=np.int32)
    t, ptr, cols, rows, pitch, dev = _image2d(image, "describe_sgrad")
    desc = np.zeros((len(p), SGRAD_SIZE), np.float32)
    # the partition moves whole points: order the extra fields by matching each output point back by its index
    q = p.copy()
    q["ix"] = p_idx
    _check(_ipf().vwb200_ipfind_describe(ptr, cols, rows, pitch, int(tile_size), q.ctypes.data, len(q), desc.ctypes.data, dev,
                                         _stream_ptr() if dev else None))
    order = q["ix"].copy()
    q["ix"] = p["ix"][order]
    base = rec[order] if rec.dtype.names and "polarity" in rec.dtype.names else None
    return _ipf_records(q, desc, base)


def last_ipfind_stats():
    """what the last detect_interest_points_iagd / describe_sgrad on this thread did: tiles, raw extrema, points kept after
    the auto-gain and Harris thresholds, tiles culled to their num_ip, points described"""
    s = IpfindStats()
    _ipf().vwb200_last_ipfind_stats(C.byref(s))
    return {f: int(getattr(s, f)) for f, _ in IpfindStats._fields_}


def ipfind(image, ip_per_tile=250, ip_per_image=0, nodata=None, nodata_radius=1, tile_size=1024, no_orientation=False):
    """ipfind --interest-operator iagd (tools/ipfind.cc:253-401): normalize, detect, remove the points near nodata (0 when
    nodata is None, as ipfind does) when nodata_radius > 0, then the sgrad descriptor.  Returns an interest_points() array
    whose write_binary_ip_file bytes are ipfind's .vwip."""
    t, ptr, cols, rows, pitch, dev = _image2d(image, "ipfind")
    if ip_per_image > 0:
        ip_per_tile = ip_per_tile_for_image(ip_per_image, cols, rows, tile_size)
    img = normalize(image, nodata)
    pts = detect_interest_points_iagd(img, ip_per_tile, tile_size)
    if len(pts) == 0:
        return _ipf_records(np.zeros(0, _IPF_POINT), np.zeros((0, SGRAD_SIZE), np.float32))
    if nodata_radius > 0:
        pts = remove_ip_near_nodata(image, pts, 0.0 if nodata is None else nodata, nodata_radius)
    if no_orientation:
        pts["orientation"] = 0
    return describe_sgrad(img, pts, tile_size)
