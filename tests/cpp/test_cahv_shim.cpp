// test_cahv_shim.cpp -- exercises the CAHV / CAHVOR overloads of include/vwb200/CameraTransform.h and StereoView.h the way Vision
// Workbench code would (linearize_camera, epipolar(CAHV, CAHV), camera_transform from a CAHVOR or CAHV camera,
// linearize_camera_transform, epipolar_transformed_cahv_images, stereo_triangulate and StereoModel through a CAHVOR pair) and
// checks them against the CPU oracle bit for bit.  linearize_camera and epipolar are host arithmetic and are checked first,
// without a device.  Exit codes: 0 ok, 1 mismatch, 3 no CUDA device.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/CameraTransform.h"
extern "C" {
#include "../../oracle/vw_cahv_oracle.h"
}

using namespace vw;

static vwc_cahv oracle_cam(camera::CameraModel const& c) {
  vwb200_cahv a;
  if (!stereo::b200_detail::cahv_of(&c, &a)) std::abort();
  vwc_cahv o;
  static_assert(sizeof(o) == sizeof(a), "the oracle's camera has the ABI's layout");
  std::memcpy(&o, &a, sizeof o);
  return o;
}

static long differ(const void* got, const void* want, size_t bytes) { return std::memcmp(got, want, bytes) != 0; }
static long differ_cam(camera::CameraModel const& got, vwc_cahv const& want) {
  const vwc_cahv g = oracle_cam(got);
  return differ(&g, &want, sizeof g);
}

// the oracle's camera_transform over (0, 0, ow, oh): reverse() of every pixel, then the interpolation
template <class PixelT>
static std::vector<float> oracle_transform(ImageView<PixelT> const& img, vwc_cahv const& src, vwc_cahv const& dst, int ow, int oh, int interp,
                                           int edge, const float* ev) {
  std::vector<double> coords(size_t(ow) * oh * 2);
  vwc_camera_reverse_window(&src, &dst, 0, 0, ow, oh, coords.data());
  const bool masked = sizeof(PixelT) == 8;
  std::vector<float> out(size_t(ow) * oh * (masked ? 2 : 1));
  if (masked)
    vww_sample_masked(edge, ev, reinterpret_cast<const float*>(img.data()), img.cols(), img.rows(), coords.data(), (long long)ow * oh, out.data());
  else
    vww_sample(interp, edge, reinterpret_cast<const float*>(img.data()), img.cols(), img.rows(), coords.data(), (long long)ow * oh, out.data());
  return out;
}

int main() {
  const int W = 97, H = 61;
  // a rover-like CAHVOR pair looking along +x, 0.5 apart along y
  const Vector3 A(0.9995, 0.02, -0.0245), O(0.999, 0.03, -0.0316);
  camera::CAHVORModel cam1(Vector3(0.0, 0.0, 0.0), A, Vector3(1.9, 87.0, 0.05), Vector3(1.5, -1.0, -88.0), O, Vector3(1e-3, -2e-2, 1.8e-1));
  camera::CAHVORModel cam2(Vector3(0.02, 0.5, 0.01), A, Vector3(2.2, 88.0, 0.04), Vector3(1.4, -1.1, -87.5), O, Vector3(2e-3, -1e-2, 1e-1));
  long bad = 0;
  // linearize_camera and epipolar: host arithmetic
  const vwc_cahv o1 = oracle_cam(cam1), o2 = oracle_cam(cam2);
  const int size[2] = {W, H};
  vwc_cahv l1, l2, w1, w2;
  vwc_linearize(&o1, size, size, &l1);
  vwc_linearize(&o2, size, size, &l2);
  camera::CAHVModel lin1 = camera::b200_linearize_camera(cam1, Vector2i(W, H), Vector2i(W, H));
  camera::CAHVModel lin2 = camera::b200_linearize_camera(cam2, W, H, W, H);
  bad += differ_cam(lin1, l1) + differ_cam(lin2, l2);
  vwc_epipolar(&l1, &l2, &w1, &w2);
  camera::CAHVModel epi1, epi2;
  camera::b200_epipolar(lin1, lin2, epi1, epi2);
  bad += differ_cam(epi1, w1) + differ_cam(epi2, w2);
  if (bad) { std::printf("FAIL: linearize_camera or epipolar differs from the oracle\n"); return 1; }

  uint32_t seed = 11u;
  auto rnd = [&seed]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
  ImageView<PixelGray<float>> gray(W, H);
  ImageView<PixelMask<float>> masked(W, H);
  ImageView<PixelMask<Vector2f>> df(W, H);
  ImageView<PixelMask<Vector2i>> di(W, H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      gray(x, y) = PixelGray<float>(255.0f * rnd());
      PixelMask<float> p(255.0f * rnd());
      if (rnd() < 0.2f) p.invalidate();
      masked(x, y) = p;
      PixelMask<Vector2f> d(Vector2f(-5.0f - 20.0f * rnd(), 2.0f * rnd() - 1.0f));
      PixelMask<Vector2i> q{Vector2i(-5 - int(20 * rnd()), int(3 * rnd()) - 1)};
      if (rnd() < 0.1f) { d.invalidate(); q.invalidate(); }
      df(x, y) = d;
      di(x, y) = q;
    }
  try {
    // camera_transform: the size form with bicubic and constant edges, the default form, a bbox form from a CAHV source
    ImageView<PixelGray<float>> a = camera::b200_camera_transform(gray, cam1, lin1, Vector2i(W, H), ConstantEdgeExtension(), BicubicInterpolation());
    std::vector<float> wa = oracle_transform(gray, o1, l1, W, H, VWB200_INTERP_BICUBIC, VWB200_EDGE_CONSTANT, nullptr);
    bad += differ(a.data(), wa.data(), wa.size() * 4);
    ImageView<PixelGray<float>> b = camera::b200_camera_transform(gray, cam2, lin2);
    std::vector<float> wb = oracle_transform(gray, o2, l2, W, H, VWB200_INTERP_BILINEAR, VWB200_EDGE_ZERO, nullptr);
    bad += differ(b.data(), wb.data(), wb.size() * 4);
    ImageView<PixelGray<float>> c = camera::b200_camera_transform(gray, lin1, epi1, Vector2i(W, H), ZeroEdgeExtension(), NearestPixelInterpolation());
    std::vector<float> wc = oracle_transform(gray, l1, w1, W, H, VWB200_INTERP_NEAREST, VWB200_EDGE_ZERO, nullptr);
    bad += differ(c.data(), wc.data(), wc.size() * 4);
    // linearize_camera_transform
    ImageView<PixelGray<float>> d = camera::b200_linearize_camera_transform(gray, cam1, ConstantEdgeExtension());
    std::vector<float> wd = oracle_transform(gray, o1, l1, W, H, VWB200_INTERP_BILINEAR, VWB200_EDGE_CONSTANT, nullptr);
    bad += differ(d.data(), wd.data(), wd.size() * 4);
    // epipolar_transformed_cahv_images from the CAHVOR cameras straight into the epipolar ones
    camera::CAHVModel e1 = epi1, e2 = epi2;
    e1.C = cam1.C;
    e2.C = cam2.C;
    const vwc_cahv we1 = oracle_cam(e1), we2 = oracle_cam(e2);
    ImageView<PixelMask<float>> lo, ro;
    PixelMask<float> edge_pix(1.0f);
    camera::b200_epipolar_transformed_cahv_images(cam1, cam2, e1, e2, masked, masked, lo, ro, ValueEdgeExtension<PixelMask<float>>(edge_pix));
    const float ev[2] = {1.0f, 1.0f};
    std::vector<float> wl = oracle_transform(masked, o1, we1, W, H, VWB200_INTERP_BILINEAR, VWB200_EDGE_VALUE, ev);
    std::vector<float> wr = oracle_transform(masked, o2, we2, W, H, VWB200_INTERP_BILINEAR, VWB200_EDGE_VALUE, ev);
    bad += differ(lo.data(), wl.data(), wl.size() * 4) + differ(ro.data(), wr.data(), wr.size() * 4);
    // triangulation through the CAHVOR pair and through the epipolar CAHV pair
    std::vector<double> want(size_t(W) * H * 3), err_want(size_t(W) * H);
    long long it;
    ImageView<Vector3> pf = stereo::b200_stereo_triangulate(df, &cam1, &cam2);
    vwc_stereo_triangulate(1, df.data(), W, H, 0, 0, W, H, &o1, &o2, 0.0, want.data(), &it);
    bad += differ(pf.data(), want.data(), want.size() * 8);
    ImageView<Vector3> pi = stereo::b200_stereo_triangulate(di, &e1, &e2);
    vwc_stereo_triangulate(0, di.data(), W, H, 0, 0, W, H, &we1, &we2, 0.0, want.data(), &it);
    bad += differ(pi.data(), want.data(), want.size() * 8);
    ImageView<double> err;
    ImageView<Vector3> xyz = stereo::B200StereoModel(&cam1, &e2, 1e-3)(df, err);
    double st[4];
    vwc_stereo_model(reinterpret_cast<const float*>(df.data()), W, H, &o1, &we2, 1e-3, want.data(), err_want.data(), st, &it);
    bad += differ(xyz.data(), want.data(), want.size() * 8) + differ(err.data(), err_want.data(), err_want.size() * 8);
    // the errors: a pinhole with a CAHV camera, cameras at different centers
    Matrix3x3 R;
    R.set_identity();
    camera::PinholeModel pin(Vector3(0, 0, 0), R, 90.0, 90.0, 48.0, 30.0);
    bool threw = false;
    try { stereo::b200_stereo_triangulate(df, &cam1, &pin); }
    catch (NoImplErr const&) { threw = true; }
    if (!threw) { std::printf("FAIL: a pinhole with a CAHVOR camera was accepted\n"); return 1; }
    threw = false;
    try { camera::b200_camera_transform(gray, cam1, epi2); }
    catch (LogicErr const& e) { threw = std::strstr(e.what(), "camera center") != nullptr; }
    if (!threw) { std::printf("FAIL: cameras at different centers were accepted\n"); return 1; }
    std::printf("cahv shim: %ld mismatches\n", bad);
    return bad ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
