// DisparityResampling.h -- C++ shim: the resampling, range and transform operations of Stereo/DisparityMap.h with the
// reference's parameter lists, computed on the device through include/vwb200.h, for ImageView<PixelMask<Vector2i>> and
// ImageView<PixelMask<Vector2f>>:
//   b200_disparity_subsample / b200_disparity_upsample     disparity_subsample / disparity_upsample      (:1251-1358)
//   b200_get_disparity_range                               get_disparity_range                           (:48-66)
//   b200_disparity_range_mask                              disparity_range_mask                          (:255-300)
//   b200_transform_disparities(disparity, H)               transform_disparities(disparity, HomographyTransform(H)) (:1016-1057)
//   b200_transform_disparities(do_round, subregion, T, disparity)                                       (:1190-1224)
// The reference returns lazy views; these return the rasterised ImageView (BBox2f for the range), computed once over the
// whole image.  Results are bit for bit the reference's inside the value limits of include/vwb200.h; created pixels carry
// the engine's valid word (1), not ChannelRange::max().  The lazy transform applies vw::math::inverse(H), the call
// HomographyTransform's constructor makes, so under the real VW headers the device applies the reference's matrix.
#pragma once
#include "PyramidCorrelationView.h"

namespace vw { namespace stereo {

namespace b200_detail {
template <class PixelT> struct DispPixel;
template <> struct DispPixel<PixelMask<Vector2i>> { enum { type = VWB200_DISP_I32 }; typedef int32 channel; };
template <> struct DispPixel<PixelMask<Vector2f>> { enum { type = VWB200_DISP_F32 }; typedef float channel; };

template <class PixelT, class Fn>
inline ImageView<PixelT> disp_call(ImageView<PixelT> const& in, int32 ocols, int32 orows, Fn fn) {
  static_assert(sizeof(PixelT) == 12, "disparity pixels must be {dx, dy, valid} triples of 4-byte values");
  ImageView<PixelT> out(ocols, orows);
  check(fn(DispPixel<PixelT>::type, in.data(), in.cols(), in.rows(), in.rstride(), out.data(), out.rstride()));
  return out;
}
template <class MatrixT>
inline void matrix9(MatrixT const& m, double* out) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) out[3 * r + c] = m(r, c);
}
}  // namespace b200_detail

template <class PixelT>
inline ImageView<PixelT> b200_disparity_subsample(ImageView<PixelT> const& view) {
  const int32 c = view.cols() ? 1 + (view.cols() - 1) / 2 : 0, r = view.rows() ? 1 + (view.rows() - 1) / 2 : 0;
  return b200_detail::disp_call(view, c, r, [](int t, const void* in, int w, int h, ptrdiff_t p, void* out, ptrdiff_t op) {
    return vwb200_disparity_subsample(t, in, w, h, p, out, op, /*on_device=*/0, nullptr);
  });
}

template <class PixelT>
inline ImageView<PixelT> b200_disparity_upsample(ImageView<PixelT> const& view) {
  return b200_detail::disp_call(view, view.cols() * 2, view.rows() * 2, [](int t, const void* in, int w, int h, ptrdiff_t p, void* out, ptrdiff_t op) {
    return vwb200_disparity_upsample(t, in, w, h, p, out, op, 0, nullptr);
  });
}

template <class PixelT>
inline BBox2f b200_get_disparity_range(ImageView<PixelT> const& disparity_map) {
  float r[4];
  b200_detail::check(vwb200_get_disparity_range(b200_detail::DispPixel<PixelT>::type, disparity_map.data(), disparity_map.cols(), disparity_map.rows(),
                                   disparity_map.rstride(), r, nullptr, 0, nullptr));
  return BBox2f(Vector2f(r[0], r[1]), Vector2f(r[2], r[3]));
}

template <class PixelT>
inline ImageView<PixelT> b200_disparity_range_mask(ImageView<PixelT> const& disparity_map, PixelT const& min, PixelT const& max) {
  typedef typename b200_detail::DispPixel<PixelT>::channel C;
  const C mn[2] = {min.child()[0], min.child()[1]}, mx[2] = {max.child()[0], max.child()[1]};
  return b200_detail::disp_call(disparity_map, disparity_map.cols(), disparity_map.rows(),
                                [&](int t, const void* in, int w, int h, ptrdiff_t p, void* out, ptrdiff_t op) {
                                  return vwb200_disparity_range_mask(t, in, w, h, p, mn, mx, out, op, 0, nullptr);
                                });
}

// transform_disparities(disparity_map, HomographyTransform(H)): reverse(loc + d) - loc
template <class PixelT>
inline ImageView<PixelT> b200_transform_disparities(ImageView<PixelT> const& disparity_map, Matrix3x3 const& H) {
  double m[9];
  b200_detail::matrix9(math::inverse(H), m);
  return b200_detail::disp_call(disparity_map, disparity_map.cols(), disparity_map.rows(),
                                [&](int t, const void* in, int w, int h, ptrdiff_t p, void* out, ptrdiff_t op) {
                                  return vwb200_transform_disparities(t, VWB200_TRANSFORM_LAZY, m, 0, nullptr, in, w, h, p, out, op, 0, nullptr);
                                });
}

// transform_disparities(do_round, subregion, T, disparity); T: a matrix with rows(), cols() and T(row, col), e.g. Matrix<double>
// or Matrix3x3.  In the reference's order: a subregion of another size than the disparity throws ArgumentErr; then, as the
// reference's HomographyTransform H(T), a T that is not 3 x 3 throws ArgumentErr and a singular T throws MathErr from
// inverse(), although only T itself is applied.
template <class MatrixT, class PixelT>
inline ImageView<PixelT> b200_transform_disparities(bool do_round, BBox2i subregion, MatrixT const& T, ImageView<PixelT> const& disparity) {
  if (subregion.max()[0] - subregion.min()[0] != disparity.cols() || subregion.max()[1] - subregion.min()[1] != disparity.rows())
    vw_throw(ArgumentErr() << "transform_disparities: The sizes of subregion and disparity don't match.\n");
  if (T.rows() != 3 || T.cols() != 3) vw_throw(ArgumentErr() << "Matrix must have dimensions 3x3.");
  Matrix3x3 H;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) H(r, c) = T(r, c);
  math::inverse(H);
  double m[9];
  b200_detail::matrix9(H, m);
  const int32_t box[4] = {subregion.min()[0], subregion.min()[1], subregion.max()[0], subregion.max()[1]};
  return b200_detail::disp_call(disparity, disparity.cols(), disparity.rows(),
                                [&](int t, const void* in, int w, int h, ptrdiff_t p, void* out, ptrdiff_t op) {
                                  return vwb200_transform_disparities(t, VWB200_TRANSFORM_EXPLICIT, m, do_round ? 1 : 0, box, in, w, h, p, out, op,
                                                                      0, nullptr);
                                });
}

}}  // namespace vw::stereo
