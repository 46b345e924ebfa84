/*
 * vwb200.h -- C ABI of the H100-native stereo-correlation engine.
 *
 * This is the drop-in boundary for Vision Workbench's dense block-matching path.  VW has no
 * FFI: its "operator API" is the compile-time ImageViewBase<> concept
 * (src/vw/Image/ImageViewBase.h:57-122).  The C++ shim include/vwb200/PyramidCorrelationView.h
 * keeps that concept (prerasterize()/rasterize()) and calls the functions below; no C++ or
 * torch types cross this boundary -- plain pointers, sizes and POD structs only.
 *
 * Conventions
 *  - images are row-major, one plane, pitch in ELEMENTS (vw::ImageView, Image/ImageView.h:226-227)
 *  - boxes are half-open [x0,x1) x [y0,y1) (vw::BBox2i, Math/BBox.tcc)
 *  - integer disparity pixel = {int32 dx, int32 dy, int32 valid(0/1)}   (PixelMask<Vector2i>)
 *  - float   disparity pixel = {float dx, float dy, float valid(0/1)}   (PixelMask<Vector2f>,
 *    Image/PixelMask.h:52-54: 12 bytes)
 *  - every function returns 0 on success or a negative VWB200_E* code; vwb200_last_error()
 *    gives the message of the calling thread's last failure.  The shim maps codes to
 *    vw::ArgumentErr / MathErr / LogicErr (Core/Exception.h:225-253).
 *  - "on_device" != 0 means the pointers are CUDA device pointers on the current device;
 *    otherwise they are host pointers and the call stages them through HBM itself.
 *  - `stream` is a cudaStream_t (or NULL for the library's own per-call stream).  All calls
 *    block until their result is complete unless stated otherwise.
 *  - all entry points are thread-safe (VW calls prerasterize() concurrently from its tile
 *    thread pool, Image/ImageIO.h:228-235).
 *  - there is NO CPU fallback: without a CUDA device every compute call fails with
 *    VWB200_ENODEVICE.
 */
#ifndef VWB200_H
#define VWB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VWB200_OK          0
#define VWB200_EARG       -1   /* -> vw::ArgumentErr */
#define VWB200_EMATH      -2   /* -> vw::MathErr     */
#define VWB200_ELOGIC     -3   /* -> vw::LogicErr    */
#define VWB200_ENOIMPL    -4   /* -> vw::NoImplErr   */
#define VWB200_ECUDA      -5   /* CUDA runtime failure */
#define VWB200_ENODEVICE  -6   /* no CUDA device: the engine has no CPU path */
#define VWB200_ENOMEM     -7
#define VWB200_EPROJECT   -8   /* -> vw::camera::PointToPixelErr */

/* vw::stereo::CostFunctionType, src/vw/Stereo/CostFunctions.h:143-149 */
enum { VWB200_ABSOLUTE_DIFFERENCE = 0, VWB200_SQUARED_DIFFERENCE = 1, VWB200_CROSS_CORRELATION = 2,
       VWB200_CENSUS_TRANSFORM = 3, VWB200_TERNARY_CENSUS_TRANSFORM = 4 };
/* vw::stereo::CorrelationAlgorithm, src/vw/Stereo/CorrelationAlgorithms.h:29-35 */
enum { VWB200_CORRELATION_BM = 0, VWB200_CORRELATION_SGM = 1, VWB200_CORRELATION_MGM = 2, VWB200_CORRELATION_FINAL_MGM = 3 };
/* vw::stereo::SemiGlobalMatcher::SgmSubpixelMode, src/vw/Stereo/SGM.h:93-99 */
enum { VWB200_SUBPIXEL_NONE = 0, VWB200_SUBPIXEL_PARABOLA = 1, VWB200_SUBPIXEL_LINEAR = 2, VWB200_SUBPIXEL_POLY4 = 3,
       VWB200_SUBPIXEL_COSINE = 4, VWB200_SUBPIXEL_LC_BLEND = 5 };
/* vw::stereo::PrefilterModeType, src/vw/Stereo/PrefilterEnum.h:24-28 */
enum { VWB200_PREFILTER_NONE = 0, VWB200_PREFILTER_LOG = 1, VWB200_PREFILTER_MEANSUB = 2 };

typedef struct { int32_t dx, dy, valid; } vwb200_dispi;

const char* vwb200_last_error(void);
int vwb200_device_count(void);          /* number of visible CUDA devices (0 if none) */
const char* vwb200_version(void);

/* ---------------------------------------------------------------------------------------------
 * K1: vw::stereo::calc_disparity (src/vw/Stereo/Correlation.h:50-57, Correlation.cc:330-375)
 * -> best_of_search_convolution (Correlation.cc:33-137).
 * left  : (W+kx-1) x (H+ky-1) float; right: at least (W+kx-1+sx-1) x (H+ky-1+sy-1) float.
 * out   : W x H vwb200_dispi, disparities in [0,sx) x [0,sy), first-in-raster-order wins ties,
 *         pixel invalid iff every disparity gave the same cost (Correlation.cc:121-133).
 * ------------------------------------------------------------------------------------------- */
int vwb200_calc_disparity(int cost_type,
                          const float* left,  int lw, int lh, ptrdiff_t lpitch,
                          const float* right, int rw, int rh, ptrdiff_t rpitch,
                          int sx, int sy, int kx, int ky,
                          vwb200_dispi* out, ptrdiff_t opitch,
                          int on_device, void* stream);

/* Statistics of the last vwb200_calc_disparity on this thread: which kernel path ran
 * (0 = exact-integer fast path, 1 = general fp64 path), kernel launches issued, and the device time of
 * the dominant (fused cost-volume + arg-best) kernel measured with CUDA events on its stream. */
typedef struct { int32_t path; int32_t launches; float kernel_ms; int32_t reserved; } vwb200_k1_stats;
int vwb200_last_k1_stats(vwb200_k1_stats* out);

/* ---------------------------------------------------------------------------------------------
 * K2: one Gaussian-pyramid level = subsample(separable_convolution_filter(in,{1,4,6,4,1}/16),2)
 * (src/vw/Stereo/CorrelationView.cc:210-214; Image/Convolution.h:275-328; Image/Filter.h:89-99;
 *  Image/Manipulation.h:238-251).  out is (1+(w-1)/2) x (1+(h-1)/2).  Bit-exact in float.
 * ------------------------------------------------------------------------------------------- */
int vwb200_pyramid_down(const float* in, int w, int h, ptrdiff_t pitch,
                        float* out, ptrdiff_t opitch, int on_device, void* stream);
/* vw::stereo::prefilter_image (src/vw/Stereo/PreFilter.h:75-95): NONE / LaplacianOfGaussian(width) /
 * SubtractedMean(width); gaussian_filter + laplacian_filter of src/vw/Image/Filter.h:204-237,318-335. */
int vwb200_prefilter(const float* in, int w, int h, ptrdiff_t pitch, int mode, float width,
                     float* out, ptrdiff_t opitch, int on_device, void* stream);
/* SubsampleMaskByTwoFunc, src/vw/Stereo/CorrelationView.cc:38-63 */
int vwb200_subsample_mask_by_two(const uint8_t* in, int w, int h, ptrdiff_t pitch,
                                 uint8_t* out, ptrdiff_t opitch, int on_device, void* stream);

/* K3: vw::stereo::cross_corr_consistency_check (src/vw/Stereo/Correlate.cc:1441-1502), in place */
int vwb200_cross_corr_consistency_check(vwb200_dispi* l2r, int lw, int lh, ptrdiff_t lpitch,
                                        const vwb200_dispi* r2l, int rw, int rh, ptrdiff_t rpitch,
                                        float threshold, int on_device, void* stream);

/* K4: rm_outliers_using_thresh / disparity_cleanup_using_thresh / disparity_mask
 * (src/vw/Stereo/DisparityMap.h:318-442, :97-253).  in/out are w x h, dense pitch. */
int vwb200_rm_outliers_using_thresh(const vwb200_dispi* in, int w, int h, int half_h, int half_v,
                                    double pixel_threshold, double rejection_threshold,
                                    vwb200_dispi* out, int on_device, void* stream);
int vwb200_disparity_cleanup_using_thresh(const vwb200_dispi* in, int w, int h, int half_h, int half_v,
                                          double pixel_threshold, double rejection_threshold,
                                          vwb200_dispi* out, int on_device, void* stream);
int vwb200_disparity_mask(const vwb200_dispi* in, int w, int h,
                          const uint8_t* left_mask, const uint8_t* right_mask, int rmw, int rmh,
                          vwb200_dispi* out, int on_device, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The outlier filters of src/vw/Stereo/DisparityMap.h on integer or float disparities:
 *   method THRESH, cleanup 0 / 1: rm_outliers_using_thresh / disparity_cleanup_using_thresh  (:318-442)
 *   method MEAN,   cleanup 0 / 1: rm_outliers_using_mean   / disparity_cleanup_using_mean    (:444-598)
 *   method STDDEV, cleanup 0 / 1: rm_outliers_using_stddev / disparity_cleanup_using_stddev  (:600-767)
 * THRESH and STDDEV read pixel_threshold and rejection_threshold, MEAN reads max_mean_diff.  The cleanup composites add
 * the reference's second RmOutliersUsingThreshFunc(1, 1, 3.0, 0.2) pass, which reads the first pass at the image's
 * border without a second edge extension.  Each output pixel is computed from the input, so out must not overlap in
 * (VWB200_EARG).  A rejected pixel becomes {0, 0, 0}; every other pixel is copied unchanged.  Results are bit for bit
 * the reference's for finite disparities with |dx|, |dy| < 2^30.  rm_outliers_using_stddev uses every valid window pixel;
 * the reference writes past its (2 * half_v + 1)^2 value vector when half_h > half_v and more pixels than that are valid.
 * in / out: w x h pixels of pixel_type, row pitches in pixels.  half_h or half_v <= 0, an unknown method, cleanup or
 * pixel type: VWB200_EARG.  A window whose tile and halo exceed the kernel's shared memory: VWB200_ENOIMPL.
 * ------------------------------------------------------------------------------------------- */
enum { VWB200_DISP_I32 = 0, VWB200_DISP_F32 = 1 };                 /* {int32 x3} / {float x3} pixels */
enum { VWB200_OUTLIERS_THRESH = 0, VWB200_OUTLIERS_MEAN = 1, VWB200_OUTLIERS_STDDEV = 2 };
typedef struct { int32_t method, cleanup, half_h, half_v;
                 double pixel_threshold, rejection_threshold, max_mean_diff; } vwb200_outlier_params;
int vwb200_outlier_filter(const vwb200_outlier_params* p, int pixel_type, const void* in, int w, int h, ptrdiff_t pitch,
                          void* out, ptrdiff_t opitch, int on_device, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Resampling, range and transforms of a disparity image (src/vw/Stereo/DisparityMap.h) on either pixel type
 * (VWB200_DISP_I32 / VWB200_DISP_F32); in / out are row-major, row pitches in pixels.  A pixel is valid when valid != 0.
 * Pixels the engine creates get valid = 1 (or 1.0f), invalid ones {0, 0, 0} unless stated otherwise; pixels the reference
 * passes through are copied unchanged, valid word included.  Results are bit for bit the reference's (floats as raw bits;
 * NaN payloads are not kept) inside the value limits given per call.
 *
 * disparity_subsample (:1251-1322): out is (1 + (w-1)/2) x (1 + (h-1)/2).  The 10 / 5 / 2 weighted mean of the valid
 * pixels of each 3 x 3 neighbourhood at stride 2, clamped reads at the border, summed in double (float pixels) or int64
 * (int32 pixels, then truncating division) in the reference's order.  int32: |dx|, |dy| < 2^28 (the reference multiplies
 * six of the nine terms in int32).  out must not overlap in.
 * disparity_upsample (:1324-1358): out is 2w x 2h, each pixel child(x >> 1, y >> 1) * 2 with the child's validity (invalid
 * pixels keep their doubled values and valid = 0).  int32: |dx|, |dy| < 2^30.  out must not overlap in.
 * ------------------------------------------------------------------------------------------- */
int vwb200_disparity_subsample(int pixel_type, const void* in, int w, int h, ptrdiff_t pitch, void* out, ptrdiff_t opitch,
                               int on_device, void* stream);
int vwb200_disparity_upsample(int pixel_type, const void* in, int w, int h, ptrdiff_t pitch, void* out, ptrdiff_t opitch,
                              int on_device, void* stream);
/* get_disparity_range (:48-66, PixelAccumulator<EWMinMaxAccumulator>, Image/Statistics.h:193-223): range (host, 4 floats)
 * receives BBox2f(min, max) = {min dx, min dy, max dx, max dy} over the valid pixels in raster order, integers converted to
 * float; (0, 0, 0, 0) when no pixel is valid.  Among equal values (-0.0 / +0.0) the first in raster order is kept; a NaN of
 * the first valid pixel sticks, later NaNs are skipped.  any_valid (may be NULL) receives 1 or 0.  w * h < 2^32. */
int vwb200_get_disparity_range(int pixel_type, const void* in, int w, int h, ptrdiff_t pitch, float* range, int* any_valid,
                               int on_device, void* stream);
/* disparity_range_mask (:255-300): min / max (host) point at two int32 or two floats, the children of the reference's
 * min / max pixels.  A valid pixel with x + dx < min[0], x + dx >= max[0] - 1, y + dy < min[0] (sic, :279) or
 * y + dy >= max[1] - 1 (in double; max - 1 in the channel type) becomes {0, 0, 0}; every other pixel is copied.
 * out may be in (same pitch) but must not overlap it otherwise. */
int vwb200_disparity_range_mask(int pixel_type, const void* in, int w, int h, ptrdiff_t pitch, const void* min, const void* max,
                                void* out, ptrdiff_t opitch, int on_device, void* stream);
/* transform_disparities.  matrix: the 3 x 3 matrix (row-major doubles) that is applied, p -> (m p) / w in homogeneous
 * coordinates, in the order of HomographyTransform (Math/Transform.h:377-387).
 *   VWB200_TRANSFORM_LAZY: transform_disparities(disparity, HomographyTransform(H)) (:1016-1057) with matrix = inverse(H),
 *     the matrix HomographyTransform::reverse applies: out = m(loc + d) - loc.  Invalid pixels stay invalid (valid = 0)
 *     and receive the transformed values.  do_round and the subregion are not used.
 *   VWB200_TRANSFORM_EXPLICIT: transform_disparities(do_round, subregion, matrix, disparity) (:1190-1224) with
 *     beg = subregion.min() + loc: out = m(beg + d) - beg, rounded half away from zero (std::round) when do_round.
 *     Invalid pixels give {0, 0, 0}.  The subregion {x0, y0, x1, y1} must be w x h (VWB200_EARG, the reference's message).
 * The matrix is applied as given; a singular one is not refused here (the C++ shim and the Python mirror refuse it as the
 * reference's HomographyTransform constructor does).
 * int32 pixels take the results truncated toward zero; a NaN or out-of-range result gives INT32_MIN, as x86-64 builds of the
 * reference give (the C++ conversion is undefined there).
 * out may be in (same pitch) but must not overlap it otherwise. */
enum { VWB200_TRANSFORM_LAZY = 0, VWB200_TRANSFORM_EXPLICIT = 1 };
int vwb200_transform_disparities(int pixel_type, int mode, const double* matrix, int do_round, const int32_t* subregion,
                                 const void* in, int w, int h, ptrdiff_t pitch, void* out, ptrdiff_t opitch, int on_device,
                                 void* stream);

/* ---------------------------------------------------------------------------------------------
 * transform(image, tx, edge, interp) (src/vw/Image/Transform.h:485-601) of a float image (PixelGray<float>), rasterised over
 * the output window (x0, y0, ow, oh): out pixel (i, j) is the TransformView pixel (x0 + i, y0 + j).  The plain form is the
 * window (0, 0, w, h), the width / height form (0, 0, width, height), the bbox form the bbox itself.
 *   kind VWB200_WARP_HOMOGRAPHY: HomographyTransform(H) (Math/Transform.h:369-389); matrix is the 3 x 3 matrix (row-major
 *     doubles) that reverse() applies, i.e. inverse(H), as VWB200_TRANSFORM_LAZY takes it.  The disparity is not used.
 *   kind VWB200_WARP_DISPARITY: DisparityTransform(disparity) (Stereo/DisparityMap.h:1164-1187) on a dw x dh float
 *     disparity ({dx, dy, valid} pixels, row pitch dpitch in pixels).  reverse(p) is p + (dx, dy) in double for a valid
 *     pixel at p, and (-1, p.y) for an invalid one or a p outside the disparity.  The matrix is not used.
 *   interp: VWB200_INTERP_BILINEAR (in float, Image/Interpolation.h:76-110), _BICUBIC (in double, :138-186) or _NEAREST
 *     (math::impl::_round, ties away from zero, :209-225).  Bilinear and bicubic return the pixel itself when the reversed
 *     point is integral, so NaN neighbours do not leak in there.
 *   edge: VWB200_EDGE_ZERO (+0.0f outside the image) or VWB200_EDGE_CONSTANT (each axis clamped) (Image/EdgeExtension.tcc).
 * Exactness: every pixel is bit for bit the reference's (floats as raw bits, NaN payloads not kept) when both reversed
 * coordinates are finite with |c| < 2^30.  Elsewhere (including w == 0 of a homography inside the window, giving inf or NaN)
 * the reference converts the coordinate out of int32 range, which is undefined; the engine writes 0.0f there.
 * in: w x h floats, row pitch `pitch`; out: ow x oh floats, row pitch `opitch`; x0 + ow and y0 + oh must not exceed 2^31 - 1.
 * VWB200_EARG, before the device is looked up, for a NULL params / in / out, a disparity kind without a disparity, an
 * unknown enum, w, h, ow, oh (or dw, dh) <= 0, a pitch below its width, or an out that overlaps in or the disparity.
 * ------------------------------------------------------------------------------------------- */
enum { VWB200_WARP_HOMOGRAPHY = 0, VWB200_WARP_DISPARITY = 1 };
enum { VWB200_INTERP_BILINEAR = 0, VWB200_INTERP_BICUBIC = 1, VWB200_INTERP_NEAREST = 2 };
enum { VWB200_EDGE_ZERO = 0, VWB200_EDGE_CONSTANT = 1 };
typedef struct { int32_t kind, interp, edge; double matrix[9]; } vwb200_warp_params;
int vwb200_transform_image(const vwb200_warp_params* p, const float* in, int w, int h, ptrdiff_t pitch, const void* disparity, int dw,
                           int dh, ptrdiff_t dpitch, int x0, int y0, float* out, int ow, int oh, ptrdiff_t opitch, int on_device,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * fill_holes_grass(img, hole_fill_len) (src/vw/Image/InpaintView.h:239-311) of a disparity (VWB200_DISP_I32 /
 * VWB200_DISP_F32), rasterised over the output window (x0, y0, ow, oh), which must lie inside the w x h input.  As in the
 * reference, the result depends on the window: the holes are looked for in the window grown by hole_fill_len (and cropped to
 * the image).  A hole is an 8-connected component of invalid pixels; it is filled when its bounding box is at most
 * hole_fill_len wide and tall, and its bounding box grown by one pixel lies inside that tile with its last column / row below
 * cols - 1 / rows - 1 (InpaintView.h:76-80 tests max >= cols on a half-open box, so a hole reaching column cols - 2 is
 * skipped too).  Its pixels are then ordered by their city-block distance to the nearest non-hole pixel, then column-major,
 * and given 10 * max_distance^2 in-place sweeps of the 8-neighbour stencil (.176765 corners, .073235 edges; each product in
 * double, each sum rounded to float; int32 stores truncate).  The first sweep reads the holes' invalid children as they are.
 * Filled pixels get valid = 1; every other pixel is copied, valid word included.  hole_fill_len = 0 fills nothing.
 * Exactness: bit for bit the reference's (floats as raw bits, NaN payloads not kept); int32 children need |dx|, |dy| < 2^30.
 * VWB200_EARG, before the device is looked up, for a NULL in / out, an unknown pixel type, w, h, ow, oh <= 0, a pitch below its
 * width, a window outside the input, and, where the reference does not check, for hole_fill_len < 0, a hole_fill_len^2 that
 * overflows int32, and an out that overlaps in.  VWB200_ENOIMPL for a tile of 2^30 pixels or more.
 * vwb200_last_fill_stats reports the last call on this thread: holes found in the tile, holes filled (those that meet the
 * window), the largest 10 * max_distance^2, the most levels of one hole and the longest chain of synchronised steps
 * (sweeps x levels) of one hole.
 * ------------------------------------------------------------------------------------------- */
int vwb200_fill_holes_grass(int pixel_type, const void* in, int w, int h, ptrdiff_t pitch, int hole_fill_len, int x0, int y0, void* out,
                            int ow, int oh, ptrdiff_t opitch, int on_device, void* stream);
typedef struct { long long holes, filled, max_sweeps, max_levels, critical_steps; } vwb200_fill_stats;
int vwb200_last_fill_stats(vwb200_fill_stats* out);

/* ---------------------------------------------------------------------------------------------
 * Dense two-camera triangulation through pinhole cameras (src/vw/Stereo/StereoView.h, StereoModel.cc:35-309,
 * Camera/PinholeModel.cc:79-116, 422-434, 553-605, Camera/LensDistortion.cc:258-400, Math/NewtonRaphson.cc).
 * A camera is the parameter list of the PinholeModel constructors: center C, rotation R (row-major), fu, fv, cu, cv, the
 * u, v, w frame vectors (the unit axes by default), pixel_pitch and a lens distortion: VWB200_LENS_NULL (num_lens_params 0)
 * or VWB200_LENS_TSAI (num_lens_params 5: k1, k2, p1, p2, k3).  Per call the host builds the inverse camera transform
 * inverse(uvw * transpose(R)) * inverse(K) exactly as rebuild_camera_matrix does (LU with partial pivoting, Math/Matrix.h:
 * 2218-2281); a u, v, w frame that fails its orthonormality asserts is VWB200_ELOGIC, a singular matrix VWB200_EMATH.
 * Per pixel: pixel_to_vector of both pixels (undistort pix * pixel_pitch -- Tsai by Newton-Raphson, tol 1e-9, at most 19
 * iterations --, inv * (u, v, 1), normalised), the nearly-parallel test 1 - dot(d0, d1) >= tol (tol = angle_tol when
 * angle_tol > 0, else 1e-4; NaN directions count as parallel), the closest-point midpoint and its reflection through cam1's center
 * when it falls behind either camera.  A pixel with a NaN component or equal to (-1e8, -1e8) is skipped; with a ray skipped or
 * parallel rays the point is (0, 0, 0).  Exactness: every double bit for bit the reference's (NaN payloads not kept).
 * Points are {x, y, z} doubles (24 bytes), pitches in pixels.  VWB200_EARG, before the device is looked up, for a NULL
 * pointer, an unknown pixel type or lens, w, h, ow, oh <= 0, a pitch below its width, a window outside the input, a Tsai lens
 * without num_lens_params == 5, a NULL lens with parameters, and an output that overlaps an input.
 * ------------------------------------------------------------------------------------------- */
enum { VWB200_LENS_NULL = 0, VWB200_LENS_TSAI = 1 };
typedef struct {
  double center[3];
  double rotation[9];
  double fu, fv, cu, cv;
  double u_direction[3], v_direction[3], w_direction[3];
  double pixel_pitch;
  int lens;                 /* VWB200_LENS_* */
  int num_lens_params;      /* 0 for NULL, 5 for TSAI */
  double lens_params[5];    /* TSAI: k1, k2, p1, p2, k3 */
} vwb200_pinhole;

/* stereo_triangulate(disparity, cam1, cam2) (StereoView.h:74-130) rasterised over the window (x0, y0, ow, oh) of a w x h
 * disparity (VWB200_DISP_I32 / VWB200_DISP_F32): pixel (i, j) triangulates (i, j) against (i, j) + (double)disparity;
 * an invalid pixel (valid == 0) gives (0, 0, 0).  xyz is ow x oh. */
int vwb200_stereo_triangulate(int pixel_type, const void* disparity, int w, int h, ptrdiff_t pitch, int x0, int y0, int ow, int oh,
                              const vwb200_pinhole* cam1, const vwb200_pinhole* cam2, double angle_tol, double* xyz, ptrdiff_t xyz_pitch,
                              int on_device, void* stream);
/* StereoModel::operator()(ImageView<PixelMask<Vector2f>>, ImageView<double>& error) (StereoModel.cc:254-309) over a whole
 * w x h float disparity: pixel (x, y) triangulates (x, y) against (x + dx, y + dy) summed in float; error = norm_2 of the
 * closest points' difference.  An invalid pixel gives xyz 0 and error 0; a NaN error gives xyz 0, keeps the NaN and counts
 * as divergent. */
int vwb200_stereo_model_points(const float* disparity, int w, int h, ptrdiff_t pitch, const vwb200_pinhole* cam1,
                               const vwb200_pinhole* cam2, double angle_tol, double* xyz, ptrdiff_t xyz_pitch, double* error,
                               ptrdiff_t error_pitch, int on_device, void* stream);
/* what the last vwb200_stereo_model_points on this thread reports (StereoModel.cc:301-307): points with error >= 0, divergent
 * points, the largest error (exact) and the sum of the errors (summed in another order than the reference's raster order:
 * within 1e-12 relative); the mean error is error_sum / points.  tsai_iterations: the Newton-Raphson iterations of the last
 * vwb200_stereo_triangulate or vwb200_stereo_model_points (both rays of every triangulated pixel). */
typedef struct { long long points, divergent; double max_error, error_sum; long long tsai_iterations;
                 long long cahvor_iterations;   /* the CAHVOR Newton passes of the last vwb200_cahv_stereo_* call */
} vwb200_triangulation_stats;
int vwb200_last_triangulation_stats(vwb200_triangulation_stats* out);
/* UniverseRadiusFunc(origin, near_radius, far_radius) applied to a w x h Vector3 image (StereoView.h:139-186): a point equal to
 * (0, 0, 0) (-0.0 included) becomes +0 and is not rejected; otherwise dist = norm_2(p - origin), and the point becomes +0
 * and is rejected when (near != 0 && dist < near) || (far != 0 && dist > far); a NaN point passes unchanged.  out may be in
 * (same pitch).  *rejected / *total (may be NULL) receive the counts.  VWB200_EARG also for radii that are not >= 0 or
 * near > far (the reference's asserts); far = DBL_MAX is the reference's default. */
int vwb200_universe_radius(const double* in, int w, int h, ptrdiff_t pitch, const double origin[3], double near_radius, double far_radius,
                           double* out, ptrdiff_t out_pitch, long long* rejected, long long* total, int on_device, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Epipolar rectification of a pinhole stereo pair (Camera/PinholeModel.cc:351-397, 679-732, Camera/EpipolarUtils.cc:37-76,
 * Camera/CameraTransform.h:43-183, Image/Transform.h:271-315).  Cameras are vwb200_pinhole as above, NULL or TSAI lens.
 * point_to_pixel is the reference's with its check on (m_do_point_to_pixel_check): P * (X, 1) de-homogenised, the lens's
 * distorted_coordinates (TSAI in closed form; HUGE_VAL for fu or fv < 1e-300), / pixel_pitch, then pixel_to_vector of that
 * pixel against normalize(X - C), retried with their sum; a difference still >= 0.01 or NaN is PointToPixelErr, returned as
 * VWB200_EPROJECT with the reference's message and the first failing pixel.  Exactness: every double and float bit for bit the
 * reference's (NaN payloads not kept).  VWB200_EARG comes before the device is looked up; a u, v, w frame that fails the
 * orthonormality asserts is VWB200_ELOGIC, as are a camera transform's cameras at different centers (the VW_ASSERT of
 * CameraTransform.h:53).
 * ------------------------------------------------------------------------------------------- */
/* epipolar(cam0, cam1, epi0, epi1) on the host: camera_pose() rotations through the quaternion round trip, the baseline as u,
 * w from the mean look vector, v = w x u, the mean focal length, point offset and pixel pitch, NULL lens and the default
 * u, v, w frame.  Coincident centers give NaN cameras, as in the reference. */
int vwb200_pinhole_epipolar(const vwb200_pinhole* cam0, const vwb200_pinhole* cam1, vwb200_pinhole* epi0, vwb200_pinhole* epi1);
/* resize_epipolar_cameras_to_fit(cam1, cam2, epi1, epi2, roi1, roi2, size1, size2): the BBox2f of each ROI's perimeter
 * (x0, y0, x1, y1) through CameraTransform(cam, epi)::forward, on the device; both epipolar point offsets shifted by the
 * smaller minimum corner times epi1's pixel pitch (epi1, epi2 are updated in place); the second pass's bbox maxima truncated
 * to int32 are the sizes (width, height).  A bound that rounds to zero may carry the other sign of zero than the reference's
 * order-dependent one; that changes a size or an offset only where the offset itself is +-0. */
int vwb200_resize_epipolar_cameras_to_fit(const vwb200_pinhole* cam1, const vwb200_pinhole* cam2, vwb200_pinhole* epi1, vwb200_pinhole* epi2,
                                          const int32_t roi1[4], const int32_t roi2[4], int32_t size1[2], int32_t size2[2], void* stream);
/* camera_transform(image, src, dst, edge, interp) rasterised over the output window (x0, y0, ow, oh) as vwb200_transform_image
 * does: out pixel (i, j) is the image interpolated at src.point_to_pixel(dst.pixel_to_vector(p) + C), p = (x0 + i, y0 + j),
 * with the same interpolations, edges and |c| < 2^30 domain rule.  pixel_type VWB200_PIXEL_GRAY_F32: float pixels, every
 * interpolation, zero and constant edges.  VWB200_PIXEL_MASK_F32: PixelMask<float> {float value, float valid} pixels (pitches in
 * pixels), bilinear only, zero ({0, 0}), constant and value edges (VWB200_EDGE_VALUE: ValueEdgeExtension(edge_value
 * {value, valid})).  The masked arithmetic is the reference's: an integral point returns {value, valid != 0}, an interpolated
 * one the float value with valid 1 when all four neighbours have valid != 0 (NaN counts as valid) and 0 otherwise; outside the
 * domain {0, 0}.  Other combinations are VWB200_ENOIMPL.  On VWB200_EPROJECT the contents of out are unspecified. */
enum { VWB200_PIXEL_GRAY_F32 = 0, VWB200_PIXEL_MASK_F32 = 1 };
enum { VWB200_EDGE_VALUE = 2 };
int vwb200_camera_transform(const vwb200_pinhole* src, const vwb200_pinhole* dst, int pixel_type, int interp, int edge, const float edge_value[2],
                            const void* in, int w, int h, ptrdiff_t pitch, int x0, int y0, void* out, int ow, int oh, ptrdiff_t opitch,
                            int on_device, void* stream);

/* ---------------------------------------------------------------------------------------------
 * JPL CAHV and CAHVOR cameras (Camera/CAHVModel.cc, CAHVORModel.cc, CameraTransform.h, StereoModel.cc:121-122).
 * pixel_to_vector is normalize(cross(V - y*A, H - x*A)), negated when dot(cross(V, H), A) < 0; CAHVOR then removes the radial
 * distortion with the reference's Newton loop (at most 20 passes, stopping when deriv <= 0 or after a step |du| < 1e-6).
 * point_to_pixel is (dot(p, H), dot(p, V)) / dot(p, A) of p = point - C (CAHVOR: p + mu * lambda); it has no round-trip check,
 * so these calls never return VWB200_EPROJECT.  Exactness: every double and float bit for bit the reference's (NaN payloads
 * not kept).  VWB200_EARG, before the device is looked up, for a NULL pointer or an unknown model; the other arguments are
 * checked as for the pinhole calls above.  CAHVORE is not supported.
 * ------------------------------------------------------------------------------------------- */
enum { VWB200_CAMERA_CAHV = 1, VWB200_CAMERA_CAHVOR = 2 };
typedef struct {
  int model;                                 /* VWB200_CAMERA_CAHV or VWB200_CAMERA_CAHVOR */
  double C[3], A[3], H[3], V[3], O[3], R[3]; /* O and R are ignored for CAHV */
} vwb200_cahv;
/* epipolar(CAHVModel, CAHVModel) (CAHVModel.cc:297-337) on the host: both outputs share A, H, V and keep their source's C.
 * The sources must be CAHV cameras (a CAHVOR camera is VWB200_EARG: linearize it first). */
int vwb200_cahv_epipolar(const vwb200_cahv* cam0, const vwb200_cahv* cam1, vwb200_cahv* epi0, vwb200_cahv* epi1);
/* linearize_camera(CAHVORModel, cahvor_image_size, cahv_image_size) (CAHVORModel.cc:460-547) on the host: the CAHV camera at
 * the same C whose A is the normalised sum of 12 perimeter rays and whose H, V span the smallest field of view.  Sizes are
 * (width, height).  cam must be a CAHVOR camera. */
int vwb200_linearize_camera(const vwb200_cahv* cam, const int32_t cahvor_size[2], const int32_t cahv_size[2], vwb200_cahv* out);
/* CAHVModel = PinholeModel (CAHVModel.cc:64-99) for a NULL-lens pinhole: VWB200_EARG for a Tsai lens (the conversion would drop
 * it) and for a zero pixel pitch (the reference's ArgumentErr); the frame asserts and a singular matrix as for the pinhole
 * calls. */
int vwb200_pinhole_to_cahv(const vwb200_pinhole* pin, vwb200_cahv* out);
/* camera_transform(image, src, dst, edge, interp) as vwb200_camera_transform, from a CAHV or CAHVOR src into a CAHV dst
 * (a CAHVOR dst is VWB200_ENOIMPL); the same pixel types, interpolations, edges and window.  Cameras at different centers are
 * VWB200_ELOGIC. */
int vwb200_cahv_camera_transform(const vwb200_cahv* src, const vwb200_cahv* dst, int pixel_type, int interp, int edge, const float edge_value[2],
                                 const void* in, int w, int h, ptrdiff_t pitch, int x0, int y0, void* out, int ow, int oh, ptrdiff_t opitch,
                                 int on_device, void* stream);
/* vwb200_stereo_triangulate and vwb200_stereo_model_points through CAHV or CAHVOR cameras (each may be either); the
 * statistics are those of vwb200_last_triangulation_stats, with cahvor_iterations in place of tsai_iterations. */
int vwb200_cahv_stereo_triangulate(int pixel_type, const void* disparity, int w, int h, ptrdiff_t pitch, int x0, int y0, int ow, int oh,
                                   const vwb200_cahv* cam1, const vwb200_cahv* cam2, double angle_tol, double* xyz, ptrdiff_t xyz_pitch,
                                   int on_device, void* stream);
int vwb200_cahv_stereo_model_points(const float* disparity, int w, int h, ptrdiff_t pitch, const vwb200_cahv* cam1, const vwb200_cahv* cam2,
                                    double angle_tol, double* xyz, ptrdiff_t xyz_pitch, double* error, ptrdiff_t error_pitch, int on_device,
                                    void* stream);

/* ---------------------------------------------------------------------------------------------
 * Exact interest point matching: InterestPointMatcherSimple<L2NormMetric | HammingMetric, NullConstraint>::operator()
 * (src/vw/InterestPoint/Matcher.h:415-509, Matcher.cc:33-100) and remove_duplicates (Matcher.cc:151-195).
 * desc1 is n1 x dim floats (row pitch pitch1 floats), desc2 n2 x dim (pitch2); pol1 / pol2 hold one polarity byte per point
 * (compared as bools).  For each query i the candidates j = 0..n2-1 of equal polarity are scanned; the distance is the
 * reference's float metric:
 *   VWB200_METRIC_L2       sum over k in order of (a - b) * (a - b), each sub, mul and add rounded to float (no FMA);
 *   VWB200_METRIC_HAMMING  the popcount of the XOR of the bytes static_cast<uint8>(value) (truncation), exact for 8 dim <= 2^24
 *                          (larger dim: VWB200_ENOIMPL).  A value outside (-1, 256) or NaN, undefined in the reference, is
 *                          VWB200_EARG naming the first such element.
 * first / second are the reference's double first_pick / second_pick (1e100 when none: an inf or NaN distance is never
 * picked; among equal minima the lowest j wins; a distance equal to first becomes second), and match_index[i] is the picked
 * j, or -1 when none was picked or first > threshold * second in double (threshold may be any double).  n2 == 0 gives -1
 * everywhere (the reference's empty-list early return).  match_index is int32; first / second may be NULL.  Exactness: every
 * index and double bit for bit the reference's.  VWB200_EARG, before the device is looked up, for a NULL pointer with n > 0,
 * n1, n2, dim < 0, a pitch below dim, an unknown metric, and outputs that overlap each other or an input.
 * ------------------------------------------------------------------------------------------- */
enum { VWB200_METRIC_L2 = 0, VWB200_METRIC_HAMMING = 1 };
int vwb200_ip_match(int metric, const float* desc1, const uint8_t* pol1, int n1, const float* desc2, const uint8_t* pol2, int n2,
                    int dim, ptrdiff_t pitch1, ptrdiff_t pitch2, double threshold, int32_t* match_index, double* first, double* second,
                    int on_device, void* stream);
/* the last vwb200_ip_match on this thread: descriptor pairs scanned (n1 * n2), the metric, the CTAs the candidate range was
 * split over (1: not split; 0: no candidates) and the matches kept */
typedef struct { long long pairs, matches; int32_t metric, splits; } vwb200_ipmatch_stats;
int vwb200_last_ipmatch_stats(vwb200_ipmatch_stats* out);
/* remove_duplicates on the host: pairs are walked from last to first; a pair is dropped when its (x1, y1) or its (x2, y2) was
 * already kept (compared as std::pair<float, float>, so -0.0 equals 0.0), and kept otherwise.  xy1 / xy2 hold n (x, y)
 * float pairs; keep receives the kept indices in ascending order, *n_kept their count.  A NaN coordinate, which breaks the
 * reference's std::set ordering, is VWB200_EARG. */
int vwb200_remove_duplicate_matches(const float* xy1, const float* xy2, int n, int32_t* keep, int* n_kept);

/* ---------------------------------------------------------------------------------------------
 * vw::stereo::ParabolaSubpixelView::rasterize(dest, bbox) (src/vw/Stereo/ParabolaSubpixelView.h:27-117,
 * .cc:31-330): 3x3 AbsoluteCost patch around the integer disparity, 6x9 pseudo-inverse parabola fit,
 * offset kept when its norm is below 5.  disparity: cols x rows PixelMask<Vector2f> triples (same size as
 * the left image); dest: (x1-x0) x (y1-y0) triples.  Floats agree with the reference within 1e-5.
 * ------------------------------------------------------------------------------------------- */
int vwb200_parabola_subpixel(const float* disparity, int cols, int rows, const float* left, ptrdiff_t lpitch,
                             const float* right, int rcols, int rrows, ptrdiff_t rpitch, int kx, int ky,
                             int prefilter_mode, float prefilter_width, int x0, int y0, int x1, int y1,
                             float* dest, ptrdiff_t dest_pitch, int on_device, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Disparity smoothing: vw::stereo::disparity_median_filter (src/vw/Stereo/Algorithms.cc:26-67), texture_measure
 * (Algorithms.h:144-209) and texture_preserving_disparity_filter<float> (Algorithms.h:213-281).  Results are bit for bit
 * the reference's (a zero may come out as -0.0 where the reference gives +0.0 or the reverse: its std::sort does not order
 * them).  Disparities are cols x rows {dx, dy, valid} float triples, pitch in pixels; a pixel is valid when valid != 0.
 *
 * IN PLACE: the two disparity filters overwrite `disparity`.  The reference's `disparity_out = disparity_in` is ImageView's
 * shallow copy, so there too the output shares the input's buffer, and each pixel's window sees the already filtered
 * pixels above and to its left (raster order).  The engine computes exactly that order.  Processed pixels get valid = 1;
 * every other pixel keeps all three floats.  The kernels take kernel_size / max_kernel_size up to 31 (VWB200_ENOIMPL
 * above) and pitches up to INT_MAX / 93 pixels.  An in-place sweep that makes no progress for 10 s returns VWB200_ELOGIC
 * ("wavefront stalled").
 * ------------------------------------------------------------------------------------------- */
/* kernel_size < 3: nothing changes.  Even sizes use the odd window below them (4 -> 3 x 3), as the reference does. */
int vwb200_disparity_median_filter(float* disparity, int cols, int rows, ptrdiff_t pitch, int kernel_size, int on_device, void* stream);
/* image: a plain float image (every pixel valid); out: cols x rows floats, row pitch opitch.  kernel_size < 1 ->
 * VWB200_EARG (the reference leaves its output uninitialised there). */
int vwb200_texture_measure(const float* image, int cols, int rows, ptrdiff_t pitch, int kernel_size, double gradient_weight,
                           double stddev_weight, float* out, ptrdiff_t opitch, int on_device, void* stream);
/* texture: cols x rows floats, row pitch tpitch.  max_kernel_size < 3 or texture_max <= 0: nothing changes.  A pixel whose
 * texture gives a kernel above max_kernel_size is skipped silently (the reference prints a message to stdout there). */
int vwb200_texture_preserving_disparity_filter(float* disparity, int cols, int rows, ptrdiff_t pitch, const float* texture,
                                               ptrdiff_t tpitch, float texture_max, int max_kernel_size, int on_device, void* stream);

/* ---------------------------------------------------------------------------------------------
 * vw::stereo::calc_disparity_sgm (src/vw/Stereo/SGM.cc:167-230, SGM.h:361-376) ->
 * SemiGlobalMatcher::semi_global_matching_func (:2387-2448): u8_convert, (ternary) census costs for kernel 3/5/7/9,
 * per-pixel search boxes, SGM or MGM accumulation along 8 directions, integer winner with the reference's tie
 * smoothing, optional sub-pixel stage.  left / right are the cropped left_region / right_region rasters (any float
 * range).  Disparities lie in [0, search_x] x [0, search_y] (inclusive = search_volume of the reference).
 * out receives out_w x out_h pixels (row pitch opitch elements; the size is (:2397-2420) and can be queried first
 * with all outputs NULL).
 * Penalties: after the defaults are applied (p1 / p2 <= 0), every entry point needs p1 <= p2 <= 30000 and returns
 * VWB200_ENOIMPL otherwise, with both values in vwb200_last_error().  This is stricter than the reference, which takes
 * any uint16 pair (SGM.cc:77-160): a given p2 below the default p1 (census 7 with p1 = 0, p2 = 29) is refused too.
 * Inside the range, accumulated costs above 65535 wrap around in uint16 exactly as the reference's do.
 * ------------------------------------------------------------------------------------------- */
/* the simple form: the same search box for every pixel (populate_constant_disp_bound_image, :231-239), plain
 * census costs, no masks, no previous disparity; p1 / p2 <= 0 select the reference's defaults (:108-157) */
int vwb200_sgm_calc_disparity(const float* left, int lw, int lh, ptrdiff_t lpitch,
                              const float* right, int rw, int rh, ptrdiff_t rpitch,
                              int search_x, int search_y, int kernel_size, int p1, int p2,
                              vwb200_dispi* out, ptrdiff_t opitch, int* out_w, int* out_h, int on_device, void* stream);
/* ... followed by SemiGlobalMatcher::create_disparity_view_subpixel (SGM.cc:1497-1614) on the integer result:
 * subpixel_mode = SgmSubpixelMode.  out (may be NULL) gets the integer disparity, out_sub the float
 * {dx, dy, valid} pixels (sub_pitch in pixels).  Floats agree with the reference's double arithmetic within 1e-5. */
int vwb200_sgm_calc_disparity_subpixel(const float* left, int lw, int lh, ptrdiff_t lpitch,
                                       const float* right, int rw, int rh, ptrdiff_t rpitch,
                                       int search_x, int search_y, int kernel_size, int p1, int p2, int subpixel_mode,
                                       vwb200_dispi* out, ptrdiff_t opitch, float* out_sub, ptrdiff_t sub_pitch,
                                       int* out_w, int* out_h, int on_device, void* stream);

/* the full form.  vwb200_sgm_params mirrors the SemiGlobalMatcher constructor (SGM.h:104-121). */
typedef struct {
  int32_t search_x, search_y;            /* max disparity, inclusive (min is 0) */
  int32_t kernel_size;                   /* 3, 5, 7 or 9 */
  int32_t cost_type;                     /* VWB200_CENSUS_TRANSFORM or VWB200_TERNARY_CENSUS_TRANSFORM; anything else:
                                            VWB200_ENOIMPL like SGM.cc:1888-1892 */
  int32_t ternary_threshold;             /* ternary_census_threshold (default 5) */
  int32_t p1, p2;                        /* <= 0: the reference's defaults for the cost type and kernel; then
                                            p1 <= p2 <= 30000, else VWB200_ENOIMPL */
  int32_t use_mgm;
  int32_t subpixel_mode;
  int32_t search_buffer_x, search_buffer_y;   /* sgm_search_buffer, applied around the doubled previous disparity */
  int32_t conserve_level;                /* -1: the reference's retry loop (SGM.cc:476-497): levels 0..3 until the buffers
                                            fit memory_limit_mb; 0..3: exactly that level of constrain_disp_bound_image */
  double  memory_limit_mb;               /* <= 0: 6000 (CorrelationView.h:65) */
  int32_t assumed_threads;               /* vw_settings().default_num_threads() of the size estimate (:715-716); <= 0: 4 */
  int32_t reserved;
} vwb200_sgm_params;
/* lmask (out_w x out_h, the size of the output, :250-256) / rmask (at least output + search, :262-268) / prev (the
 * half-resolution integer disparity of the previous pyramid level) may each be NULL.  bounds != NULL: use these
 * out_w * out_h boxes {min_x, min_y, max_x, max_y} (inclusive; max < min = no search area) instead of deriving them.
 * bounds_out (may be NULL) receives the boxes that were used. */
int vwb200_sgm_calc_disparity_ex(const vwb200_sgm_params* params,
                                 const float* left, int lw, int lh, ptrdiff_t lpitch,
                                 const float* right, int rw, int rh, ptrdiff_t rpitch,
                                 const uint8_t* lmask, ptrdiff_t lmpitch,
                                 const uint8_t* rmask, int rmw, int rmh, ptrdiff_t rmpitch,
                                 const vwb200_dispi* prev, int pw, int ph, ptrdiff_t ppitch,
                                 const int32_t* bounds,
                                 vwb200_dispi* out, ptrdiff_t opitch, float* out_sub, ptrdiff_t sub_pitch,
                                 int32_t* bounds_out, int* out_w, int* out_h, int on_device, void* stream);
/* only SemiGlobalMatcher::populate_disp_bound_image + constrain_disp_bound_image (SGM.cc:241-668) for an
 * ow x oh output: bounds receives ow * oh boxes */
int vwb200_sgm_disp_bounds(const vwb200_sgm_params* params, const vwb200_dispi* prev, int pw, int ph, ptrdiff_t ppitch,
                           const uint8_t* lmask, ptrdiff_t lmpitch, const uint8_t* rmask, int rmw, int rmh, ptrdiff_t rmpitch,
                           int ow, int oh, int32_t* bounds, int on_device, void* stream);

/* ---------------------------------------------------------------------------------------------
 * The lazy view: vw::stereo::PyramidCorrelationView (src/vw/Stereo/CorrelationView.h:35-193,
 * CorrelationView.cc:273-886) behind a handle.  vwb200_corr_params mirrors the constructor
 * arguments (CorrelationView.h:48-69) that the block-matching algorithm uses.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t search_x0, search_y0, search_x1, search_y1;   /* BBox2i search_region */
  int32_t kernel_x, kernel_y;                           /* Vector2i kernel_size (odd) */
  int32_t cost_type;                                    /* CostFunctionType */
  int32_t prefilter_mode; float prefilter_width;
  float   consistency_threshold;                        /* < 0: no L/R check */
  int32_t min_consistency_level;
  int32_t filter_half_kernel;
  int32_t max_pyramid_levels;
  int32_t collar_size;
  int32_t corr_timeout; double seconds_per_op;          /* accepted; timeouts never trigger on the GPU */
  int32_t algorithm;                                    /* CorrelationAlgorithm: BM, SGM, MGM, FINAL_MGM */
  int32_t blob_filter_area;                             /* > 0: disparity_blob_filter (CorrelationView.cc:242-271) */
  /* the remaining constructor arguments (CorrelationView.h:61-69) */
  int32_t sgm_subpixel_mode;                            /* SgmSubpixelMode, default SUBPIXEL_LC_BLEND = 5 */
  int32_t sgm_search_buffer_x, sgm_search_buffer_y;     /* default (2, 2) */
  int32_t region_ul_x, region_ul_y;                     /* image position of lr_disp_diff's pixel (0, 0) */
  int32_t write_debug_images;                           /* accepted, ignored: the engine writes no files */
  int32_t sgm_threads;                                  /* vw_settings().default_num_threads() of SGM's memory estimate; <= 0: 4 */
  double  memory_limit_mb;                              /* <= 0: 6000 */
} vwb200_corr_params;

typedef struct vwb200_corr vwb200_corr;

int  vwb200_corr_create(const vwb200_corr_params* p, vwb200_corr** out);
/* on_device == 0: host rasters, copied to HBM once.  on_device == 1: device rasters, referenced in place.
 * on_device == VWB200_INPUTS_STREAMED: host rasters that STAY on the host -- every rasterize() uploads just its tile's
 * region of interest (left box + kernel padding, right box + search window; CorrelationView.cc:89-97), so rasters larger
 * than HBM work and nothing is resident between calls (the tile feeder; caller pattern Image/ImageIO.h:150-314).
 * Referenced rasters must outlive the handle.  Masks are uint8, nonzero = valid, same size as their image. */
#define VWB200_INPUTS_STREAMED 2
int  vwb200_corr_set_inputs(vwb200_corr* h,
                            const float* left,  int lcols, int lrows, ptrdiff_t lpitch,
                            const float* right, int rcols, int rrows, ptrdiff_t rpitch,
                            const uint8_t* lmask, ptrdiff_t lmpitch,
                            const uint8_t* rmask, ptrdiff_t rmpitch, int on_device);
/* the optional lr_disp_diff output (CorrelationView.h:67-68, .cc:276-283,848-857): a caller-owned cols x rows image of
 * PixelMask<float> = {value, valid} float pairs (row pitch in pixels) whose pixel (0, 0) sits at params.region_ul.
 * rasterize() writes max(|dx_lr + dx_rl|, |dy_lr + dy_rl|) where the L/R check passes (level 0) and invalidates where the
 * final disparity is invalid; other pixels keep their content.  A processed box outside the image -> VWB200_EARG.
 * diff == NULL switches the output off. */
int  vwb200_corr_set_lr_disp_diff(vwb200_corr* h, float* diff, int cols, int rows, ptrdiff_t pitch, int on_device);
int  vwb200_corr_cols(const vwb200_corr* h);
int  vwb200_corr_rows(const vwb200_corr* h);
/* rasterize(dest, bbox): dest receives (x1-x0) x (y1-y0) float disparity pixels (3 floats each),
 * row pitch dest_pitch in PIXELS.  Collar handling as in CorrelationView.h:123-133. */
int  vwb200_corr_rasterize(vwb200_corr* h, int x0, int y0, int x1, int y1,
                           float* dest, ptrdiff_t dest_pitch, int dest_on_device, void* stream);
/* prerasterize(bbox) (CorrelationView.cc:273-886): like rasterize() but processes exactly bbox, without the collar */
int  vwb200_corr_prerasterize(vwb200_corr* h, int x0, int y0, int x1, int y1,
                              float* dest, ptrdiff_t dest_pitch, int dest_on_device, void* stream);
/* levels prerasterize() would use for a bbox of this size (CorrelationView.cc:301-310) */
int  vwb200_corr_num_levels(const vwb200_corr* h, int bw, int bh);
void vwb200_corr_destroy(vwb200_corr* h);

/* ---------------------------------------------------------------------------------------------
 * Multi-GPU sharding (SURVEY.md section 8e; the reference has no distributed code): the unit of the path is the output
 * tile (tools/correlate.cc:266, Image/ImageIO.h:289-311), tiles are independent, so a raster shards into contiguous
 * output-row bands, one rank per GPU, with no reduction.  When the INPUT rasters are row-sharded the same way, rank r
 * needs from rank r + 1 the rows its last kernel windows and search rows reach into (ky - 1 rows of the left raster,
 * ky - 1 + sy - 1 of the right one): vwb200_shard_exchange_halos moves them with ncclSend / ncclRecv in one NCCL group.
 * NCCL is bound at run time (libnccl.so.2); without it vwb200_shard_create(world > 1) returns VWB200_ENOIMPL.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t rank, world;
  int32_t y0, y1;                 /* output rows [y0, y1) of this rank */
  int32_t left_rows, right_rows;  /* rows of the left / right raster this rank's launch reads */
  int32_t own_left, own_right;    /* rows resident on this rank before the exchange */
  int32_t recv_left, recv_right;  /* halo rows received from rank + 1 */
  int32_t send_left, send_right;  /* rows sent to rank - 1 (its halo) */
} vwb200_band_plan;
typedef struct vwb200_shard vwb200_shard;
/* band arithmetic for out_rows output rows (left_total_rows / right_total_rows <= 0: out_rows + ky - 1 [+ sy - 1]) */
int  vwb200_shard_plan(int rank, int world, int out_rows, int ky, int sy, int left_total_rows, int right_total_rows,
                       vwb200_band_plan* plan);
/* rank 0 calls this and hands the 128 bytes to every rank (MPI_Bcast, a file, torch.distributed, ...) */
int  vwb200_shard_unique_id(void* id128);
/* collective: every rank calls it with the same id on its own (current) device */
int  vwb200_shard_create(const void* id128, int rank, int world, vwb200_shard** out);
/* asynchronous on `stream` (NULL = the legacy default stream) */
int  vwb200_shard_exchange_halos(vwb200_shard* s, const vwb200_band_plan* plan, float* left_band, int lcols, ptrdiff_t lpitch,
                                 float* right_band, int rcols, ptrdiff_t rpitch, void* stream);
void vwb200_shard_destroy(vwb200_shard* s);

/* ---- a20 / K12: interest point detection and description (ipfind --interest-operator iagd, sgrad descriptor) -----------
 * Rasters are single-channel float (pitches in floats), in host or device memory (on_device), on `stream`.  Point lists are
 * host arrays of vwb200_ip_point.  Every call is bit for bit the reference's (tools/ipfind.cc:253-401):
 *  - normalize: normalize(image), or with has_nodata apply_mask(normalize(create_mask(image, nodata))) (min / max of the
 *    pixels != (float)nodata; those pixels become 0).  NaN or +-inf anywhere, or no valid pixel, is VWB200_EARG.
 *  - detect: detect_interest_points(image, IntegralAutoGainDetector(ip_per_tile), ip_per_tile) with default_tile_size
 *    tile_size (detection tiles are max(1024, tile_size) square).  ip_per_tile 0 keeps every point.  At most cap points are
 *    written; *n receives the count, and a count above cap is VWB200_EARG (call again with cap >= *n).
 *  - remove_near_nodata: remove_ip_near_nodata(raw, nodata, list, radius) in place (*n in: count, out: kept).
 *  - describe: describe_interest_points(image, SGradDescriptorGenerator, list): the list is reordered as its per-tile
 *    std::partition does, x / y take the crop round trip's rounding, and desc receives n * 180 floats in the new order.
 *    cos / sin of -orientation are taken on the host with the C library.  A point whose (int)x, (int)y lies outside the
 *    image is VWB200_EARG. */
typedef struct { float x, y; int32_t ix, iy; float scale, interest, orientation; } vwb200_ip_point;
int vwb200_ipfind_normalize(const float* in, int w, int h, ptrdiff_t pitch, int has_nodata, double nodata, float* out, ptrdiff_t out_pitch,
                            int on_device, void* stream);
int vwb200_ipfind_detect(const float* image, int w, int h, ptrdiff_t pitch, int tile_size, int ip_per_tile, vwb200_ip_point* out,
                         long long cap, long long* n, int on_device, void* stream);
int vwb200_ipfind_remove_near_nodata(const float* raw, int w, int h, ptrdiff_t pitch, double nodata, int radius, vwb200_ip_point* pts,
                                     long long* n, int on_device, void* stream);
int vwb200_ipfind_describe(const float* image, int w, int h, ptrdiff_t pitch, int tile_size, vwb200_ip_point* pts, long long n,
                           float* desc, int on_device, void* stream);
/* generate_gaussian_kernel(k, 2, 9): the Harris taps the detector weights by (host, no device needed) */
int vwb200_ipfind_gaussian_taps(double* k9);
/* the last detect / describe on this thread: tiles, raw extrema, points kept after the auto-gain and Harris thresholds,
 * tiles culled to their num_ip, and points described */
typedef struct { long long tiles, extrema, kept, culled_tiles, described; } vwb200_ipfind_stats;
int vwb200_last_ipfind_stats(vwb200_ipfind_stats* out);

/* Scratch memory is stream-ordered and stays cached in the device's default memory pool between calls (returning it at
 * every synchronisation costs ~100 ms per 8K x 8K call).  vwb200_trim() hands the cached memory back to the driver. */
int vwb200_trim(void);

/* total number of CUDA kernels this library has launched in this process (bench.py's gpu_launches) */
long long vwb200_kernel_launches(void);

#ifdef __cplusplus
}
#endif
#endif /* VWB200_H */
