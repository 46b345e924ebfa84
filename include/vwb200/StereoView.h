// StereoView.h -- C++ shim: dense two-camera triangulation of Stereo/StereoView.h and Stereo/StereoModel.cc with the
// reference's parameter lists, computed on the device through include/vwb200.h:
//   b200_stereo_triangulate(disparity, cam1, cam2)      stereo_triangulate (StereoView.h:125-130) on ImageView<PixelMask<Vector2i>>
//                                                       or ImageView<PixelMask<Vector2f>>: a view whose prerasterize(bbox) is one
//                                                       device call; operator() throws NoImplErr
//   B200StereoModel(cam1, cam2, angle_tol)              StereoModel's two-camera constructor and its image operator()
//                                                       (StereoModel.cc:254-309) on ImageView<PixelMask<Vector2f>>
//   b200_universe_radius(points, origin, near, far)     UniverseRadiusFunc (StereoView.h:139-186) applied in place to an
//                                                       ImageView<Vector3>; returns the rejected and total counts
// The cameras must both be camera::PinholeModel with a NULL or TSAI lens distortion, or each be a camera::CAHVModel or
// camera::CAHVORModel; anything else, a pinhole with a CAHV-family camera included, throws NoImplErr.  Results are bit for bit
// the reference's.
#pragma once
#ifdef VWB200_USE_REAL_VW
#include <vw/Camera/CameraModel.h>
#include <vw/Camera/LensDistortion.h>
#include <vw/Camera/PinholeModel.h>
#include <vw/Camera/CAHVModel.h>
#include <vw/Camera/CAHVORModel.h>
#endif
#include <cfloat>
#include <utility>
#include "DisparityResampling.h"

namespace vw { namespace stereo {

namespace b200_detail {
// the PinholeModel constructor parameters of a camera, read through its public accessors
inline vwb200_pinhole pinhole_of(camera::CameraModel const* cam) {
  camera::PinholeModel const* p = dynamic_cast<camera::PinholeModel const*>(cam);
  if (!p) vw_throw(NoImplErr() << "b200 triangulation: only camera::PinholeModel cameras have a device form");
  vwb200_pinhole o;
  std::memset(&o, 0, sizeof o);
  const Vector3 c = p->camera_center();
  Vector3 u, v, w;
  p->coordinate_frame(u, v, w);
  for (int i = 0; i < 3; ++i) {
    o.center[i] = c[i];
    o.u_direction[i] = u[i]; o.v_direction[i] = v[i]; o.w_direction[i] = w[i];
    for (int j = 0; j < 3; ++j) o.rotation[3 * i + j] = p->get_rotation_matrix()(i, j);
  }
  o.fu = p->focal_length()[0]; o.fv = p->focal_length()[1];
  o.cu = p->point_offset()[0]; o.cv = p->point_offset()[1];
  o.pixel_pitch = p->pixel_pitch();
  const std::string lens = p->lens_distortion()->name();
  if (lens == "TSAI") {
    const auto k = p->lens_distortion()->distortion_parameters();
    o.lens = VWB200_LENS_TSAI;
    o.num_lens_params = int(k.size());
    for (size_t i = 0; i < k.size() && i < 5; ++i) o.lens_params[i] = k[i];
  } else if (lens != "NULL") {
    vw_throw(NoImplErr() << "b200 triangulation: lens distortion " << lens << " has no device form (NULL and TSAI do)");
  }
  return o;
}

// a CAHVModel or CAHVORModel as the ABI's camera; false for any other camera
inline bool cahv_of(camera::CameraModel const* cam, vwb200_cahv* o) {
  std::memset(o, 0, sizeof *o);
  auto put = [](double* d, Vector3 const& v) { for (int i = 0; i < 3; ++i) d[i] = v[i]; };
  if (camera::CAHVORModel const* c = dynamic_cast<camera::CAHVORModel const*>(cam)) {
    o->model = VWB200_CAMERA_CAHVOR;
    put(o->C, c->C); put(o->A, c->A); put(o->H, c->H); put(o->V, c->V); put(o->O, c->O); put(o->R, c->R);
    return true;
  }
  if (camera::CAHVModel const* c = dynamic_cast<camera::CAHVModel const*>(cam)) {
    o->model = VWB200_CAMERA_CAHV;
    put(o->C, c->C); put(o->A, c->A); put(o->H, c->H); put(o->V, c->V);
    return true;
  }
  return false;
}

// one camera of a triangulation: a pinhole, or a CAHV / CAHVOR camera
struct TriCamera {
  bool cahv;
  vwb200_pinhole pin;
  vwb200_cahv c;
};
inline TriCamera tri_camera(camera::CameraModel const* cam) {
  TriCamera t;
  std::memset(&t, 0, sizeof t);
  t.cahv = cahv_of(cam, &t.c);
  if (!t.cahv) t.pin = pinhole_of(cam);
  return t;
}
// both cameras of one call are of one family
inline void same_family(TriCamera const& a, TriCamera const& b) {
  if (a.cahv != b.cahv) vw_throw(NoImplErr() << "b200 triangulation: a pinhole and a CAHV-family camera in one call have no device form");
}
}  // namespace b200_detail

template <class ImageT>
class B200StereoView : public ImageViewBase<B200StereoView<ImageT>> {
  ImageT m_disparity;
  b200_detail::TriCamera m_cam1, m_cam2;
  double m_angle_tol;

public:
  typedef Vector3 pixel_type;
  typedef const Vector3 result_type;
  typedef ProceduralPixelAccessor<B200StereoView<ImageT>> pixel_accessor;

  B200StereoView(ImageT const& disparity, camera::CameraModel const* cam1, camera::CameraModel const* cam2, double angle_tol = 0.0)
    : m_disparity(disparity), m_cam1(b200_detail::tri_camera(cam1)), m_cam2(b200_detail::tri_camera(cam2)), m_angle_tol(angle_tol) {
    b200_detail::same_family(m_cam1, m_cam2);
  }

  int32 cols() const { return m_disparity.cols(); }
  int32 rows() const { return m_disparity.rows(); }
  int32 planes() const { return 1; }
  pixel_accessor origin() const { return pixel_accessor(*this, 0, 0); }

  result_type operator()(int32 /*i*/, int32 /*j*/, int32 /*p*/ = 0) const {
    vw_throw(NoImplErr() << "B200StereoView::operator() is not implemented: rasterize it");
    return Vector3();
  }

  typedef CropView<ImageView<Vector3>> prerasterize_type;
  prerasterize_type prerasterize(BBox2i const& bbox) const {
    typedef typename ImageT::pixel_type dpixel;
    static_assert(sizeof(dpixel) == 12, "disparity pixels must be {dx, dy, valid} triples of 4-byte values");
    ImageView<Vector3> win(bbox.width(), bbox.height());
    if (m_cam1.cahv)
      b200_detail::check(vwb200_cahv_stereo_triangulate(b200_detail::DispPixel<dpixel>::type, m_disparity.data(), m_disparity.cols(),
                                                        m_disparity.rows(), m_disparity.rstride(), bbox.min()[0], bbox.min()[1], win.cols(),
                                                        win.rows(), &m_cam1.c, &m_cam2.c, m_angle_tol, reinterpret_cast<double*>(win.data()),
                                                        win.rstride(), /*on_device=*/0, nullptr));
    else
      b200_detail::check(vwb200_stereo_triangulate(b200_detail::DispPixel<dpixel>::type, m_disparity.data(), m_disparity.cols(), m_disparity.rows(),
                                                   m_disparity.rstride(), bbox.min()[0], bbox.min()[1], win.cols(), win.rows(), &m_cam1.pin, &m_cam2.pin,
                                                   m_angle_tol, reinterpret_cast<double*>(win.data()), win.rstride(), /*on_device=*/0, nullptr));
    return prerasterize_type(win, -bbox.min()[0], -bbox.min()[1], cols(), rows());
  }

  template <class DestT>
  void rasterize(DestT const& dest, BBox2i const& bbox) const { vw::rasterize(prerasterize(bbox), dest, bbox); }
};

template <class ImageT>
inline B200StereoView<ImageT> b200_stereo_triangulate(ImageT const& disparity, camera::CameraModel const* cam1,
                                                      camera::CameraModel const* cam2) {
  return B200StereoView<ImageT>(disparity, cam1, cam2);
}

class B200StereoModel {
  b200_detail::TriCamera m_cam1, m_cam2;
  double m_angle_tol;

public:
  B200StereoModel(camera::CameraModel const* camera_model1, camera::CameraModel const* camera_model2, double angle_tol = 0.0)
    : m_cam1(b200_detail::tri_camera(camera_model1)), m_cam2(b200_detail::tri_camera(camera_model2)), m_angle_tol(angle_tol) {
    b200_detail::same_family(m_cam1, m_cam2);
  }

  // StereoModel::operator()(disparity_map, error); the statistics the reference prints are vwb200_last_triangulation_stats
  ImageView<Vector3> operator()(ImageView<PixelMask<Vector2f>> const& disparity_map, ImageView<double>& error) const {
    ImageView<Vector3> xyz(disparity_map.cols(), disparity_map.rows());
    error.set_size(disparity_map.cols(), disparity_map.rows());
    const float* d = reinterpret_cast<const float*>(disparity_map.data());
    double* p = reinterpret_cast<double*>(xyz.data());
    if (m_cam1.cahv)
      b200_detail::check(vwb200_cahv_stereo_model_points(d, disparity_map.cols(), disparity_map.rows(), disparity_map.rstride(), &m_cam1.c, &m_cam2.c,
                                                         m_angle_tol, p, xyz.rstride(), error.data(), error.rstride(), 0, nullptr));
    else
      b200_detail::check(vwb200_stereo_model_points(d, disparity_map.cols(), disparity_map.rows(), disparity_map.rstride(), &m_cam1.pin, &m_cam2.pin,
                                                    m_angle_tol, p, xyz.rstride(), error.data(), error.rstride(), 0, nullptr));
    return xyz;
  }
};

// UniverseRadiusFunc(origin, near_radius, far_radius) over points, in place; returns {rejected, total}.  The reference's
// asserts (radii >= 0, near <= far) throw ArgumentErr.
inline std::pair<long long, long long> b200_universe_radius(ImageView<Vector3>& points, Vector3 const& universe_origin, double near_radius = 0,
                                               double far_radius = DBL_MAX) {
  long long rejected = 0, total = 0;
  const double o[3] = {universe_origin[0], universe_origin[1], universe_origin[2]};
  double* p = reinterpret_cast<double*>(points.data());
  b200_detail::check(vwb200_universe_radius(p, points.cols(), points.rows(), points.rstride(), o, near_radius, far_radius, p, points.rstride(),
                                            &rejected, &total, 0, nullptr));
  return std::make_pair(rejected, total);
}

}}  // namespace vw::stereo
