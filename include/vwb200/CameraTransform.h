// CameraTransform.h -- C++ shim: epipolar rectification of pinhole stereo pairs (Camera/CameraTransform.h:125-183,
// Camera/PinholeModel.cc:679-732, Camera/EpipolarUtils.cc:37-144) with the reference's argument lists, computed through
// include/vwb200.h:
//   b200_camera_transform(image, src, dst[, size | bbox][, edge[, interp]])   camera_transform's six overloads on
//                                ImageView<PixelGray<float>> (every interpolation; zero or constant edges) or
//                                ImageView<PixelMask<float>> (bilinear; zero, constant or ValueEdgeExtension edges); the
//                                reference returns a lazy TransformView, these the rasterised ImageView
//   b200_epipolar(src0, src1, dst0, dst1)                                      epipolar()
//   b200_resize_epipolar_cameras_to_fit(cam1, cam2, epi1, epi2, roi1, roi2, size1, size2)
//   b200_epipolar_transformed_images(left, right, left_epi, right_epi, left_in, right_in, left_roi, right_roi, left_size,
//                                    right_size, left_out, right_out, edge)   epipolar_transformed_images with the
//                                PinholeModels themselves in place of camera files (fitPinholeModel(..., "TsaiLensDistortion",
//                                false) returns NULL and TSAI cameras unchanged, CameraUtilities.cc:596-613)
// and, for JPL CAHV / CAHVOR cameras (Camera/CAHVModel.cc, CAHVORModel.cc:460-547, Camera/CameraTransform.h:185-225,
// Camera/EpipolarUtils.cc:148-222):
//   b200_camera_transform(image, src, dst, ...)  the same six overloads with a camera::CAHVModel or camera::CAHVORModel src
//                                and a camera::CAHVModel dst (no point_to_pixel check: the CAHV family has none)
//   b200_epipolar(src0, src1, dst0, dst1)        epipolar() of two CAHVModels
//   b200_linearize_camera(cahvor, cahvor_image_size, cahv_image_size)   linearize_camera(); also (cahvor, ix, iy, ox, oy)
//   b200_linearize_camera_transform(image, cahvor[, edge[, interp]])    linearize_camera_transform()
//   b200_epipolar_transformed_cahv_images(left, right, left_epi, right_epi, left_in, right_in, left_out, right_out, edge)
//                                the CAHV / CAHVOR branches of epipolar_transformed_cahv_images with the camera models
//                                themselves in place of camera files
// Pinhole cameras must be camera::PinholeModel with a NULL or TSAI lens (NoImplErr otherwise).  A failed point_to_pixel check
// throws camera::PointToPixelErr, cameras at different centers LogicErr, as the reference does.  Results are bit for bit the
// reference's (see include/vwb200.h).
#pragma once
#ifdef VWB200_USE_REAL_VW
#include <vw/Camera/CameraTransform.h>
#include <vw/Camera/EpipolarUtils.h>
#include <vw/Camera/CAHVModel.h>
#include <vw/Camera/CAHVORModel.h>
#endif
#include <type_traits>
#include "ImageTransform.h"
#include "StereoView.h"

namespace vw { namespace camera {

namespace b200_detail {
using stereo::b200_detail::InterpCode;

inline void check(int rc) {
  if (rc == VWB200_EPROJECT) vw_throw(PointToPixelErr() << vwb200_last_error());
  stereo::b200_detail::check(rc);
}

// the PinholeModel of an engine camera (NULL lens: epipolar cameras only come back that way)
inline PinholeModel pinhole_model(vwb200_pinhole const& p) {
  Matrix3x3 R;
  for (int i = 0; i < 9; ++i) R(i / 3, i % 3) = p.rotation[i];
  NullLensDistortion lens;
  return PinholeModel(Vector3(p.center[0], p.center[1], p.center[2]), R, p.fu, p.fv, p.cu, p.cv,
                      Vector3(p.u_direction[0], p.u_direction[1], p.u_direction[2]),
                      Vector3(p.v_direction[0], p.v_direction[1], p.v_direction[2]),
                      Vector3(p.w_direction[0], p.w_direction[1], p.w_direction[2]), &lens, p.pixel_pitch);
}

template <class PixelT> struct PixelCode;
template <> struct PixelCode<PixelGray<float>> { enum { value = VWB200_PIXEL_GRAY_F32 }; };
template <> struct PixelCode<PixelMask<float>> { enum { value = VWB200_PIXEL_MASK_F32 }; };

// an edge extension as the ABI's code and edge value
struct Edge { int code; float value[2]; };
inline Edge edge_of(ZeroEdgeExtension const&) { return Edge{VWB200_EDGE_ZERO, {0.0f, 0.0f}}; }
inline Edge edge_of(ConstantEdgeExtension const&) { return Edge{VWB200_EDGE_CONSTANT, {0.0f, 0.0f}}; }
inline Edge edge_of(ValueEdgeExtension<PixelMask<float>> const& e) {
  return Edge{VWB200_EDGE_VALUE, {e.m_pix.child(), e.m_pix.valid()}};
}

template <class PixelT>
inline ImageView<PixelT> transform(ImageView<PixelT> const& image, PinholeModel const& src, PinholeModel const& dst, BBox2i const& bbox,
                                   Edge const& edge, int interp) {
  const vwb200_pinhole s = stereo::b200_detail::pinhole_of(&src), d = stereo::b200_detail::pinhole_of(&dst);
  ImageView<PixelT> out(bbox.width(), bbox.height());
  check(vwb200_camera_transform(&s, &d, PixelCode<PixelT>::value, interp, edge.code, edge.value, image.data(), image.cols(), image.rows(),
                                image.rstride(), bbox.min()[0], bbox.min()[1], out.data(), out.cols(), out.rows(), out.rstride(),
                                /*on_device=*/0, nullptr));
  return out;
}

// the CAHV-family cameras camera_transform takes as a source
template <class T> struct IsCahvSource : std::false_type {};
template <> struct IsCahvSource<CAHVModel> : std::true_type {};
template <> struct IsCahvSource<CAHVORModel> : std::true_type {};

inline vwb200_cahv cahv_of(CameraModel const& cam) {
  vwb200_cahv c;
  if (!stereo::b200_detail::cahv_of(&cam, &c)) vw_throw(NoImplErr() << "b200: not a CAHV or CAHVOR camera");
  return c;
}
inline CAHVModel cahv_model(vwb200_cahv const& c) {
  return CAHVModel(Vector3(c.C[0], c.C[1], c.C[2]), Vector3(c.A[0], c.A[1], c.A[2]), Vector3(c.H[0], c.H[1], c.H[2]),
                   Vector3(c.V[0], c.V[1], c.V[2]));
}

template <class PixelT, class SrcT>
inline ImageView<PixelT> transform(ImageView<PixelT> const& image, SrcT const& src, CAHVModel const& dst, BBox2i const& bbox, Edge const& edge,
                                   int interp) {
  const vwb200_cahv s = cahv_of(src), d = cahv_of(dst);
  ImageView<PixelT> out(bbox.width(), bbox.height());
  check(vwb200_cahv_camera_transform(&s, &d, PixelCode<PixelT>::value, interp, edge.code, edge.value, image.data(), image.cols(), image.rows(),
                                     image.rstride(), bbox.min()[0], bbox.min()[1], out.data(), out.cols(), out.rows(), out.rstride(),
                                     /*on_device=*/0, nullptr));
  return out;
}
}  // namespace b200_detail

// size (CameraTransform.h:125-131)
template <class PixelT, class EdgeT, class InterpT, int I = b200_detail::InterpCode<InterpT>::value>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, PinholeModel const& src, PinholeModel const& dst, Vector2i size,
                                               EdgeT const& edge, InterpT const&) {
  return b200_detail::transform(image, src, dst, BBox2i(0, 0, size[0], size[1]), b200_detail::edge_of(edge), I);
}
// the image's own size (:135-141)
template <class PixelT, class EdgeT, class InterpT, int I = b200_detail::InterpCode<InterpT>::value>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, PinholeModel const& src, PinholeModel const& dst, EdgeT const& edge,
                                               InterpT const&) {
  return b200_detail::transform(image, src, dst, BBox2i(0, 0, image.cols(), image.rows()), b200_detail::edge_of(edge), I);
}
// bilinear (:145-151)
template <class PixelT, class EdgeT>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, PinholeModel const& src, PinholeModel const& dst, EdgeT const& edge) {
  return b200_camera_transform(image, src, dst, edge, BilinearInterpolation());
}
// zero edges, bilinear (:155-161)
template <class PixelT>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, PinholeModel const& src, PinholeModel const& dst) {
  return b200_camera_transform(image, src, dst, ZeroEdgeExtension(), BilinearInterpolation());
}
// zero edges, bilinear, size (:165-172)
template <class PixelT>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, PinholeModel const& src, PinholeModel const& dst, Vector2i size) {
  return b200_camera_transform(image, src, dst, size, ZeroEdgeExtension(), BilinearInterpolation());
}
// zero edges, bilinear, a bbox of the transformed image (:176-183; the reference's BBox2 crops at integer corners)
template <class PixelT>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, PinholeModel const& src, PinholeModel const& dst,
                                               BBox2i const& bbox) {
  return b200_detail::transform(image, src, dst, bbox, b200_detail::edge_of(ZeroEdgeExtension()), VWB200_INTERP_BILINEAR);
}

inline void b200_epipolar(PinholeModel const& src_camera0, PinholeModel const& src_camera1, PinholeModel& dst_camera0, PinholeModel& dst_camera1) {
  const vwb200_pinhole s0 = stereo::b200_detail::pinhole_of(&src_camera0), s1 = stereo::b200_detail::pinhole_of(&src_camera1);
  vwb200_pinhole d0, d1;
  b200_detail::check(vwb200_pinhole_epipolar(&s0, &s1, &d0, &d1));
  dst_camera0 = b200_detail::pinhole_model(d0);
  dst_camera1 = b200_detail::pinhole_model(d1);
}

inline void b200_resize_epipolar_cameras_to_fit(PinholeModel const& cam1, PinholeModel const& cam2, PinholeModel& epi_cam1, PinholeModel& epi_cam2,
                                                BBox2i const& roi1, BBox2i const& roi2, Vector2i& epi_size1, Vector2i& epi_size2) {
  const vwb200_pinhole c1 = stereo::b200_detail::pinhole_of(&cam1), c2 = stereo::b200_detail::pinhole_of(&cam2);
  vwb200_pinhole e1 = stereo::b200_detail::pinhole_of(&epi_cam1), e2 = stereo::b200_detail::pinhole_of(&epi_cam2);
  const int32_t r1[4] = {roi1.min()[0], roi1.min()[1], roi1.max()[0], roi1.max()[1]};
  const int32_t r2[4] = {roi2.min()[0], roi2.min()[1], roi2.max()[0], roi2.max()[1]};
  int32_t s1[2], s2[2];
  b200_detail::check(vwb200_resize_epipolar_cameras_to_fit(&c1, &c2, &e1, &e2, r1, r2, s1, s2, nullptr));
  epi_cam1.set_point_offset(Vector2<double>(e1.cu, e1.cv));
  epi_cam2.set_point_offset(Vector2<double>(e2.cu, e2.cv));
  epi_size1 = Vector2i(s1[0], s1[1]);
  epi_size2 = Vector2i(s2[0], s2[1]);
}

inline void b200_epipolar_transformed_images(PinholeModel const& left_camera, PinholeModel const& right_camera, PinholeModel const& left_epi_cam,
                                             PinholeModel const& right_epi_cam, ImageView<PixelMask<float>> const& left_image_in,
                                             ImageView<PixelMask<float>> const& right_image_in, BBox2i const& left_image_in_roi,
                                             BBox2i const& right_image_in_roi, Vector2i const& left_image_out_size,
                                             Vector2i const& right_image_out_size, ImageView<PixelMask<float>>& left_image_out,
                                             ImageView<PixelMask<float>>& right_image_out, ValueEdgeExtension<PixelMask<float>> const& edge_ext) {
  if (left_image_in_roi.min()[0] != 0 || left_image_in_roi.min()[1] != 0 || right_image_in_roi.min()[0] != 0 || right_image_in_roi.min()[1] != 0)
    vw_throw(NoImplErr() << "b200_epipolar_transformed_images: a ROI whose origin is not (0, 0) (AdjustedCameraModel) has no device form");
  left_image_out = b200_camera_transform(left_image_in, left_camera, left_epi_cam, left_image_out_size, edge_ext, BilinearInterpolation());
  right_image_out = b200_camera_transform(right_image_in, right_camera, right_epi_cam, right_image_out_size, edge_ext, BilinearInterpolation());
}

// ---- CAHV / CAHVOR sources into a CAHV destination: camera_transform's six overloads --------------------------------------------
template <class PixelT, class SrcT, class EdgeT, class InterpT, int I = b200_detail::InterpCode<InterpT>::value,
          typename std::enable_if<b200_detail::IsCahvSource<SrcT>::value, int>::type = 0>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, SrcT const& src, CAHVModel const& dst, Vector2i size,
                                               EdgeT const& edge, InterpT const&) {
  return b200_detail::transform(image, src, dst, BBox2i(0, 0, size[0], size[1]), b200_detail::edge_of(edge), I);
}
template <class PixelT, class SrcT, class EdgeT, class InterpT, int I = b200_detail::InterpCode<InterpT>::value,
          typename std::enable_if<b200_detail::IsCahvSource<SrcT>::value, int>::type = 0>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, SrcT const& src, CAHVModel const& dst, EdgeT const& edge,
                                               InterpT const&) {
  return b200_detail::transform(image, src, dst, BBox2i(0, 0, image.cols(), image.rows()), b200_detail::edge_of(edge), I);
}
template <class PixelT, class SrcT, class EdgeT, typename std::enable_if<b200_detail::IsCahvSource<SrcT>::value, int>::type = 0>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, SrcT const& src, CAHVModel const& dst, EdgeT const& edge) {
  return b200_camera_transform(image, src, dst, edge, BilinearInterpolation());
}
template <class PixelT, class SrcT, typename std::enable_if<b200_detail::IsCahvSource<SrcT>::value, int>::type = 0>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, SrcT const& src, CAHVModel const& dst) {
  return b200_camera_transform(image, src, dst, ZeroEdgeExtension(), BilinearInterpolation());
}
template <class PixelT, class SrcT, typename std::enable_if<b200_detail::IsCahvSource<SrcT>::value, int>::type = 0>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, SrcT const& src, CAHVModel const& dst, Vector2i size) {
  return b200_camera_transform(image, src, dst, size, ZeroEdgeExtension(), BilinearInterpolation());
}
template <class PixelT, class SrcT, typename std::enable_if<b200_detail::IsCahvSource<SrcT>::value, int>::type = 0>
inline ImageView<PixelT> b200_camera_transform(ImageView<PixelT> const& image, SrcT const& src, CAHVModel const& dst, BBox2i const& bbox) {
  return b200_detail::transform(image, src, dst, bbox, b200_detail::edge_of(ZeroEdgeExtension()), VWB200_INTERP_BILINEAR);
}

// epipolar(CAHVModel, CAHVModel, CAHVModel&, CAHVModel&) (Camera/CAHVModel.cc:297-337)
inline void b200_epipolar(CAHVModel const& src_camera0, CAHVModel const& src_camera1, CAHVModel& dst_camera0, CAHVModel& dst_camera1) {
  const vwb200_cahv s0 = b200_detail::cahv_of(src_camera0), s1 = b200_detail::cahv_of(src_camera1);
  vwb200_cahv d0, d1;
  b200_detail::check(vwb200_cahv_epipolar(&s0, &s1, &d0, &d1));
  dst_camera0 = b200_detail::cahv_model(d0);
  dst_camera1 = b200_detail::cahv_model(d1);
}

// linearize_camera (Camera/CAHVORModel.cc:460-553)
inline CAHVModel b200_linearize_camera(CAHVORModel const& camera_model, Vector2i const& cahvor_image_size, Vector2i const& cahv_image_size) {
  const vwb200_cahv c = b200_detail::cahv_of(camera_model);
  const int32_t in[2] = {cahvor_image_size[0], cahvor_image_size[1]}, out[2] = {cahv_image_size[0], cahv_image_size[1]};
  vwb200_cahv o;
  b200_detail::check(vwb200_linearize_camera(&c, in, out, &o));
  return b200_detail::cahv_model(o);
}
inline CAHVModel b200_linearize_camera(CAHVORModel const& camera_model, int32 ix, int32 iy, int32 ox, int32 oy) {
  return b200_linearize_camera(camera_model, Vector2i(ix, iy), Vector2i(ox, oy));
}

// linearize_camera_transform (Camera/CameraTransform.h:185-225): into the linearized camera of the image's own size
template <class PixelT, class EdgeT, class InterpT, int I = b200_detail::InterpCode<InterpT>::value>
inline ImageView<PixelT> b200_linearize_camera_transform(ImageView<PixelT> const& image, CAHVORModel const& src_camera, EdgeT const& edge,
                                                         InterpT const& interp) {
  const Vector2i size(image.cols(), image.rows());
  return b200_camera_transform(image, src_camera, b200_linearize_camera(src_camera, size, size), edge, interp);
}
template <class PixelT, class EdgeT>
inline ImageView<PixelT> b200_linearize_camera_transform(ImageView<PixelT> const& image, CAHVORModel const& src_camera, EdgeT const& edge) {
  return b200_linearize_camera_transform(image, src_camera, edge, BilinearInterpolation());
}
template <class PixelT>
inline ImageView<PixelT> b200_linearize_camera_transform(ImageView<PixelT> const& image, CAHVORModel const& src_camera) {
  return b200_linearize_camera_transform(image, src_camera, ZeroEdgeExtension(), BilinearInterpolation());
}

// the CAHV and CAHVOR branches of epipolar_transformed_cahv_images (Camera/EpipolarUtils.cc:148-222): each image resampled
// from its camera into its epipolar CAHV camera at its own size, bilinear, with edge_ext
template <class SrcT, typename std::enable_if<b200_detail::IsCahvSource<SrcT>::value, int>::type = 0>
inline void b200_epipolar_transformed_cahv_images(SrcT const& left_camera, SrcT const& right_camera, CAHVModel const& left_epipolar_cahv,
                                                  CAHVModel const& right_epipolar_cahv, ImageView<PixelMask<float>> const& left_image_in,
                                                  ImageView<PixelMask<float>> const& right_image_in, ImageView<PixelMask<float>>& left_image_out,
                                                  ImageView<PixelMask<float>>& right_image_out,
                                                  ValueEdgeExtension<PixelMask<float>> const& edge_ext) {
  left_image_out = b200_camera_transform(left_image_in, left_camera, left_epipolar_cahv, edge_ext, BilinearInterpolation());
  right_image_out = b200_camera_transform(right_image_in, right_camera, right_epipolar_cahv, edge_ext, BilinearInterpolation());
}

}}  // namespace vw::camera
