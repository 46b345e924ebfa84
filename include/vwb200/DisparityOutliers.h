// DisparityOutliers.h -- C++ shim: the neighbourhood outlier filters of Stereo/DisparityMap.h with the reference's parameter
// lists, computed on the device through vwb200_outlier_filter (include/vwb200.h), for ImageView<PixelMask<Vector2i>> and
// ImageView<PixelMask<Vector2f>>:
//   b200_rm_outliers_using_thresh   / b200_disparity_cleanup_using_thresh   (DisparityMap.h:400-442)
//   b200_rm_outliers_using_mean     / b200_disparity_cleanup_using_mean     (:567-598)
//   b200_rm_outliers_using_stddev   / b200_disparity_cleanup_using_stddev   (:737-767)
// The reference returns a lazy UnaryPerPixelAccessorView; these return the rasterised ImageView, computed once over the
// whole image.  Results are bit for bit the reference's for finite disparities with |dx|, |dy| < 2^30 (DESIGN.md
// section 3).  Zero half kernels throw ArgumentErr with the reference's message; windows beyond the kernel's shared
// memory throw NoImplErr.
#pragma once
#include "PyramidCorrelationView.h"

namespace vw { namespace stereo {

namespace b200_detail {
template <class PixelT> struct OutlierPixel;
template <> struct OutlierPixel<PixelMask<Vector2i>> { enum { type = VWB200_DISP_I32 }; };
template <> struct OutlierPixel<PixelMask<Vector2f>> { enum { type = VWB200_DISP_F32 }; };

template <class PixelT>
inline ImageView<PixelT> outlier_filter(ImageView<PixelT> const& in, int method, int cleanup, int32 half_h, int32 half_v,
                                        double pixel_threshold, double rejection_threshold, double max_mean_diff) {
  static_assert(sizeof(PixelT) == 12, "disparity pixels must be {dx, dy, valid} triples of 4-byte values");
  ImageView<PixelT> out(in.cols(), in.rows());
  vwb200_outlier_params p;
  p.method = method; p.cleanup = cleanup; p.half_h = half_h; p.half_v = half_v;
  p.pixel_threshold = pixel_threshold; p.rejection_threshold = rejection_threshold; p.max_mean_diff = max_mean_diff;
  check(vwb200_outlier_filter(&p, OutlierPixel<PixelT>::type, in.data(), in.cols(), in.rows(), in.rstride(), out.data(), out.rstride(),
                              /*on_device=*/0, nullptr));
  return out;
}
}  // namespace b200_detail

template <class PixelT>
inline ImageView<PixelT> b200_rm_outliers_using_thresh(ImageView<PixelT> const& disparity_map, int32 half_h_kernel, int32 half_v_kernel,
                                                       double pixel_threshold, double rejection_threshold) {
  return b200_detail::outlier_filter(disparity_map, VWB200_OUTLIERS_THRESH, 0, half_h_kernel, half_v_kernel, pixel_threshold,
                                     rejection_threshold, 0.0);
}
template <class PixelT>
inline ImageView<PixelT> b200_disparity_cleanup_using_thresh(ImageView<PixelT> const& disparity_map, int32 h_half_kernel,
                                                             int32 v_half_kernel, double pixel_threshold, double rejection_threshold) {
  return b200_detail::outlier_filter(disparity_map, VWB200_OUTLIERS_THRESH, 1, h_half_kernel, v_half_kernel, pixel_threshold,
                                     rejection_threshold, 0.0);
}
template <class PixelT>
inline ImageView<PixelT> b200_rm_outliers_using_mean(ImageView<PixelT> const& disparity_map, int32 half_h_kernel, int32 half_v_kernel,
                                                     double max_mean_diff) {
  return b200_detail::outlier_filter(disparity_map, VWB200_OUTLIERS_MEAN, 0, half_h_kernel, half_v_kernel, 0.0, 0.0, max_mean_diff);
}
template <class PixelT>
inline ImageView<PixelT> b200_disparity_cleanup_using_mean(ImageView<PixelT> const& disparity_map, int32 h_half_kernel, int32 v_half_kernel,
                                                           double max_mean_diff) {
  return b200_detail::outlier_filter(disparity_map, VWB200_OUTLIERS_MEAN, 1, h_half_kernel, v_half_kernel, 0.0, 0.0, max_mean_diff);
}
template <class PixelT>
inline ImageView<PixelT> b200_rm_outliers_using_stddev(ImageView<PixelT> const& disparity_map, int32 half_h_kernel, int32 half_v_kernel,
                                                       double pixel_threshold, double rejection_threshold) {
  return b200_detail::outlier_filter(disparity_map, VWB200_OUTLIERS_STDDEV, 0, half_h_kernel, half_v_kernel, pixel_threshold,
                                     rejection_threshold, 0.0);
}
template <class PixelT>
inline ImageView<PixelT> b200_disparity_cleanup_using_stddev(ImageView<PixelT> const& disparity_map, int32 h_half_kernel,
                                                             int32 v_half_kernel, double pixel_threshold, double rejection_threshold) {
  return b200_detail::outlier_filter(disparity_map, VWB200_OUTLIERS_STDDEV, 1, h_half_kernel, v_half_kernel, pixel_threshold,
                                     rejection_threshold, 0.0);
}

}}  // namespace vw::stereo
