// ImageTransform.h -- C++ shim: transform(image, tx[, width, height | bbox][, edge[, interp]]) of Image/Transform.h:485-601 on
// ImageView<PixelGray<float>>, computed on the device through vwb200_transform_image (include/vwb200.h):
//   b200_transform(image, H, ...)                                  transform(image, HomographyTransform(H), ...)
//   b200_transform(image, B200DisparityTransform(disparity), ...)  transform(image, DisparityTransform(disparity), ...)
// with the reference's three output forms (the image's size, width x height from (0, 0), a bbox of the transformed image)
// and its edge (ZeroEdgeExtension, ConstantEdgeExtension) and interpolation (BilinearInterpolation, BicubicInterpolation,
// NearestPixelInterpolation) tags; the defaults are zero edges and bilinear interpolation, as there.  The reference returns a
// lazy TransformView (cropped for the bbox form); these return the rasterised ImageView.  Results are bit for bit the
// reference's where both reversed coordinates are finite with |c| < 2^30, 0.0f elsewhere.  H is inverted with
// vw::math::inverse, the call HomographyTransform's constructor makes, so a singular H throws MathErr as there.
#pragma once
#include "PyramidCorrelationView.h"
#ifdef VWB200_USE_REAL_VW
#include <vw/Image/EdgeExtension.h>
#include <vw/Image/Interpolation.h>
#include <vw/Math/Matrix.h>
#endif

namespace vw { namespace stereo {

// DisparityTransform(disparity) of Stereo/DisparityMap.h:1164-1187 on a rasterised PixelMask<Vector2f> disparity (shared, not
// copied): reverse(p) = p + offset where the offset pixel at p is valid, (-1, p.y) elsewhere
struct B200DisparityTransform {
  ImageView<PixelMask<Vector2f>> disparity;
  explicit B200DisparityTransform(ImageView<PixelMask<Vector2f>> const& d) : disparity(d) {}
};

namespace b200_detail {
template <class EdgeT> struct EdgeCode;
template <> struct EdgeCode<ZeroEdgeExtension> { enum { value = VWB200_EDGE_ZERO }; };
template <> struct EdgeCode<ConstantEdgeExtension> { enum { value = VWB200_EDGE_CONSTANT }; };
template <class InterpT> struct InterpCode;
template <> struct InterpCode<BilinearInterpolation> { enum { value = VWB200_INTERP_BILINEAR }; };
template <> struct InterpCode<BicubicInterpolation> { enum { value = VWB200_INTERP_BICUBIC }; };
template <> struct InterpCode<NearestPixelInterpolation> { enum { value = VWB200_INTERP_NEAREST }; };

struct WarpTx {
  vwb200_warp_params p;
  ImageView<PixelMask<Vector2f>> disparity;
};
inline WarpTx warp_tx(Matrix3x3 const& H) {
  WarpTx t{};
  t.p.kind = VWB200_WARP_HOMOGRAPHY;
  const Matrix3x3 inv = math::inverse(H);                  // m_H_inverse, the matrix reverse() applies
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) t.p.matrix[3 * r + c] = inv(r, c);
  return t;
}
inline WarpTx warp_tx(B200DisparityTransform const& d) {
  static_assert(sizeof(PixelMask<Vector2f>) == 12, "PixelMask<Vector2f> must be {dx, dy, valid} floats");
  WarpTx t{};
  t.p.kind = VWB200_WARP_DISPARITY;
  t.disparity = d.disparity;
  return t;
}
inline ImageView<PixelGray<float>> warp(ImageView<PixelGray<float>> const& image, WarpTx t, BBox2i const& bbox, int edge, int interp) {
  static_assert(sizeof(PixelGray<float>) == 4, "PixelGray<float> must be one float");
  t.p.edge = edge;
  t.p.interp = interp;
  ImageView<PixelGray<float>> out(bbox.width(), bbox.height());
  const ImageView<PixelMask<Vector2f>>& d = t.disparity;
  check(vwb200_transform_image(&t.p, reinterpret_cast<const float*>(image.data()), image.cols(), image.rows(), image.rstride(), d.data(),
                               d.cols(), d.rows(), d.rstride(), bbox.min()[0], bbox.min()[1], reinterpret_cast<float*>(out.data()),
                               out.cols(), out.rows(), out.rstride(), /*on_device=*/0, nullptr));
  return out;
}
}  // namespace b200_detail

// the image's own size (Transform.h:485-514)
template <class TxT, class EdgeT, class InterpT, int E = b200_detail::EdgeCode<EdgeT>::value, int I = b200_detail::InterpCode<InterpT>::value>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx, EdgeT const&, InterpT const&) {
  return b200_detail::warp(image, b200_detail::warp_tx(tx), BBox2i(0, 0, image.cols(), image.rows()), E, I);
}
template <class TxT, class EdgeT, int E = b200_detail::EdgeCode<EdgeT>::value>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx, EdgeT const& edge) {
  return b200_transform(image, tx, edge, BilinearInterpolation());
}
template <class TxT>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx) {
  return b200_transform(image, tx, ZeroEdgeExtension(), BilinearInterpolation());
}

// width x height from (0, 0) (Transform.h:521-558)
template <class TxT, class EdgeT, class InterpT, int E = b200_detail::EdgeCode<EdgeT>::value, int I = b200_detail::InterpCode<InterpT>::value>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx, int32 width, int32 height,
                                                  EdgeT const&, InterpT const&) {
  return b200_detail::warp(image, b200_detail::warp_tx(tx), BBox2i(0, 0, width, height), E, I);
}
template <class TxT, class EdgeT, int E = b200_detail::EdgeCode<EdgeT>::value>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx, int32 width, int32 height,
                                                  EdgeT const& edge) {
  return b200_transform(image, tx, width, height, edge, BilinearInterpolation());
}
template <class TxT>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx, int32 width, int32 height) {
  return b200_transform(image, tx, width, height, ZeroEdgeExtension(), BilinearInterpolation());
}

// a bbox of the transformed image: crop(TransformView, bbox) rasterised (Transform.h:561-601)
template <class TxT, class EdgeT, class InterpT, int E = b200_detail::EdgeCode<EdgeT>::value, int I = b200_detail::InterpCode<InterpT>::value>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx, BBox2i const& bbox, EdgeT const&,
                                                  InterpT const&) {
  return b200_detail::warp(image, b200_detail::warp_tx(tx), bbox, E, I);
}
template <class TxT, class EdgeT, int E = b200_detail::EdgeCode<EdgeT>::value>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx, BBox2i const& bbox, EdgeT const& edge) {
  return b200_transform(image, tx, bbox, edge, BilinearInterpolation());
}
template <class TxT>
inline ImageView<PixelGray<float>> b200_transform(ImageView<PixelGray<float>> const& image, TxT const& tx, BBox2i const& bbox) {
  return b200_transform(image, tx, bbox, ZeroEdgeExtension(), BilinearInterpolation());
}

}}  // namespace vw::stereo
