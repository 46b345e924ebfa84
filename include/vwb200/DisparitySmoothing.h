// DisparitySmoothing.h -- C++ shim: the disparity smoothing filters of Stereo/Algorithms.{h,cc} with the reference's
// signatures, computed on the device through the C ABI of include/vwb200.h:
//   b200_disparity_median_filter              <-> disparity_median_filter              (Algorithms.h:133-135, .cc:26-67)
//   b200_texture_measure                      <-> texture_measure                      (Algorithms.h:144-209)
//   b200_texture_preserving_disparity_filter  <-> texture_preserving_disparity_filter  (Algorithms.h:213-281), T = float
// As in the reference, `disparity_out = disparity_in` is ImageView's shallow copy: out shares in's buffer, the filter
// runs in place on it, in raster order, and the caller's input holds the result too.  Results are bit for bit the
// reference's (DESIGN.md section 3); kernel sizes above 31 throw NoImplErr, and an oversized per-pixel kernel of the
// texture filter is skipped without the reference's message on stdout.
#pragma once
#include "PyramidCorrelationView.h"

namespace vw { namespace stereo {

inline void b200_disparity_median_filter(ImageView<PixelMask<Vector2f>> const& disparity_in,
                                         ImageView<PixelMask<Vector2f>>& disparity_out, int kernel_size) {
  static_assert(sizeof(PixelMask<Vector2f>) == 12, "PixelMask<Vector2f> must be {dx, dy, valid} floats");
  disparity_out = disparity_in;
  b200_detail::check(vwb200_disparity_median_filter(reinterpret_cast<float*>(disparity_out.data()), disparity_out.cols(),
                                                    disparity_out.rows(), disparity_out.rstride(), kernel_size, /*on_device=*/0, nullptr));
}

template <class ImageT>
inline void b200_texture_measure(ImageT const& input_image, ImageView<float>& output_image, int kernel_size = 9,
                                 double gradient_weight = 0.5, double stddev_weight = 0.5) {
  ImageView<float> img = input_image;                     // rasterise a lazy input once
  output_image.set_size(img.cols(), img.rows());
  b200_detail::check(vwb200_texture_measure(img.data(), img.cols(), img.rows(), img.rstride(), kernel_size, gradient_weight,
                                            stddev_weight, output_image.data(), output_image.rstride(), /*on_device=*/0, nullptr));
}

inline void b200_texture_preserving_disparity_filter(ImageView<PixelMask<Vector2f>> const& disparity_in,
                                                     ImageView<PixelMask<Vector2f>>& disparity_out,
                                                     ImageView<float> const& texture_image, float texture_max = 0.15,
                                                     int max_kernel_size = 11) {
  if (texture_image.cols() < disparity_in.cols() || texture_image.rows() < disparity_in.rows())
    vw_throw(ArgumentErr() << "texture_preserving_disparity_filter: the texture image is smaller than the disparity");
  disparity_out = disparity_in;
  b200_detail::check(vwb200_texture_preserving_disparity_filter(
      reinterpret_cast<float*>(disparity_out.data()), disparity_out.cols(), disparity_out.rows(), disparity_out.rstride(),
      texture_image.data(), texture_image.rstride(), texture_max, max_kernel_size, /*on_device=*/0, nullptr));
}

}}  // namespace vw::stereo
