// test_epipolar_shim.cpp -- exercises include/vwb200/CameraTransform.h the way Vision Workbench code would, with the reference's
// argument lists (epipolar(cam0, cam1, epi0, epi1), resize_epipolar_cameras_to_fit(...), camera_transform(image, src, dst, ...),
// epipolar_transformed_images(...)), on PixelGray<float> and PixelMask<float> images, and checks it against the CPU oracle bit
// for bit.  epipolar() is host arithmetic and is checked first, without a device.  Exit codes: 0 ok, 1 mismatch, 3 no CUDA
// device.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/CameraTransform.h"
extern "C" {
#include "../../oracle/vw_epipolar_oracle.h"
}

using namespace vw;

static vwt_pinhole oracle_cam(camera::PinholeModel const& c) {
  const vwb200_pinhole p = stereo::b200_detail::pinhole_of(&c);
  vwt_pinhole o;
  static_assert(sizeof(o) == sizeof(p), "the oracle's camera has the ABI's layout");
  std::memcpy(&o, &p, sizeof o);
  return o;
}

static long differ(const void* got, const void* want, size_t bytes) { return std::memcmp(got, want, bytes) != 0; }

// the oracle's camera_transform over (0, 0, ow, oh): reverse() of every pixel, then the interpolation
template <class PixelT>
static std::vector<float> oracle_transform(ImageView<PixelT> const& img, vwt_pinhole const& src, vwt_pinhole const& dst, int ow, int oh, int interp,
                                           int edge, const float* ev) {
  std::vector<double> coords(size_t(ow) * oh * 2);
  long long fail;
  vwt_camera_reverse_window(&src, &dst, 0, 0, ow, oh, coords.data(), &fail);
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
  Matrix3x3 R0, R1;
  R0.set_identity();
  R1.set_identity();
  const double c = 0.995, s = 0.0998749217771909;                   // a small rotation about y
  R1(0, 0) = c; R1(0, 2) = s; R1(2, 0) = -s; R1(2, 2) = c;
  camera::TsaiLensDistortion tsai(std::vector<double>{-0.12, 0.03, 1e-3, -2e-3, 0.01});
  camera::PinholeModel cam1(Vector3(0.0, 0.0, 0.0), R0, 90.0, 91.0, 48.0, 30.0, &tsai);
  camera::PinholeModel cam2(Vector3(1.0, 0.05, 0.02), R1, 88.0, 88.5, 49.0, 31.0, Vector3(1, 0, 0), Vector3(0, 1, 0), Vector3(0, 0, 1), &tsai, 1.0);
  camera::PinholeModel epi1 = cam1, epi2 = cam2;
  long bad = 0;
  // epipolar(): host arithmetic
  camera::b200_epipolar(cam1, cam2, epi1, epi2);
  const vwt_pinhole o1 = oracle_cam(cam1), o2 = oracle_cam(cam2);
  vwt_pinhole w1, w2;
  vwt_epipolar(&o1, &o2, &w1, &w2);
  const vwt_pinhole g1 = oracle_cam(epi1), g2 = oracle_cam(epi2);
  bad += differ(&g1, &w1, sizeof g1) + differ(&g2, &w2, sizeof g2);
  if (bad) { std::printf("FAIL: epipolar differs from the oracle\n"); return 1; }

  uint32_t seed = 7u;
  auto rnd = [&seed]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
  ImageView<PixelGray<float>> gray(W, H);
  ImageView<PixelMask<float>> masked(W, H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      gray(x, y) = PixelGray<float>(255.0f * rnd());
      PixelMask<float> p(255.0f * rnd());
      if (rnd() < 0.2f) p.invalidate();
      masked(x, y) = p;
    }
  try {
    // resize_epipolar_cameras_to_fit
    Vector2i s1, s2;
    const BBox2i roi(0, 0, W, H);
    camera::b200_resize_epipolar_cameras_to_fit(cam1, cam2, epi1, epi2, roi, roi, s1, s2);
    vwt_pinhole r1 = w1, r2 = w2;
    const int ri[4] = {0, 0, W, H};
    int ws1[2], ws2[2], fcam;
    long long fk;
    vwt_resize_epipolar(&o1, &o2, &r1, &r2, ri, ri, ws1, ws2, &fk, &fcam);
    const vwt_pinhole e1 = oracle_cam(epi1), e2 = oracle_cam(epi2);
    bad += differ(&e1, &r1, sizeof e1) + differ(&e2, &r2, sizeof e2) + (s1[0] != ws1[0]) + (s1[1] != ws1[1]) + (s2[0] != ws2[0]) + (s2[1] != ws2[1]);
    // camera_transform: the size form with bicubic and constant edges, the default form, and the masked value-edge form
    ImageView<PixelGray<float>> a = camera::b200_camera_transform(gray, cam1, epi1, s1, ConstantEdgeExtension(), BicubicInterpolation());
    std::vector<float> wa = oracle_transform(gray, o1, e1, s1[0], s1[1], VWB200_INTERP_BICUBIC, VWB200_EDGE_CONSTANT, nullptr);
    bad += differ(a.data(), wa.data(), wa.size() * 4);
    ImageView<PixelGray<float>> b = camera::b200_camera_transform(gray, cam2, epi2);
    std::vector<float> wb = oracle_transform(gray, o2, e2, W, H, VWB200_INTERP_BILINEAR, VWB200_EDGE_ZERO, nullptr);
    bad += differ(b.data(), wb.data(), wb.size() * 4);
    ImageView<PixelMask<float>> lo, ro;
    PixelMask<float> edge_pix;                                     // PixelMask<float>(): {0, 0}, invalid
    camera::b200_epipolar_transformed_images(cam1, cam2, epi1, epi2, masked, masked, roi, roi, s1, s2, lo, ro,
                                             ValueEdgeExtension<PixelMask<float>>(edge_pix));
    const float ev[2] = {0.0f, 0.0f};
    std::vector<float> wl = oracle_transform(masked, o1, e1, s1[0], s1[1], VWB200_INTERP_BILINEAR, VWB200_EDGE_VALUE, ev);
    std::vector<float> wr = oracle_transform(masked, o2, e2, s2[0], s2[1], VWB200_INTERP_BILINEAR, VWB200_EDGE_VALUE, ev);
    bad += differ(lo.data(), wl.data(), wl.size() * 4) + differ(ro.data(), wr.data(), wr.size() * 4);
    // the errors: a ROI offset (AdjustedCameraModel), cameras at different centers, a failed point_to_pixel check
    bool threw = false;
    try { camera::b200_epipolar_transformed_images(cam1, cam2, epi1, epi2, masked, masked, BBox2i(1, 0, 5, 5), roi, s1, s2, lo, ro,
                                                   ValueEdgeExtension<PixelMask<float>>(edge_pix)); }
    catch (NoImplErr const&) { threw = true; }
    if (!threw) { std::printf("FAIL: a ROI offset was accepted\n"); return 1; }
    threw = false;
    try { camera::b200_camera_transform(gray, cam1, epi2); }
    catch (LogicErr const&) { threw = true; }
    if (!threw) { std::printf("FAIL: cameras at different centers were accepted\n"); return 1; }
    camera::TsaiLensDistortion strong(std::vector<double>{-1.0 / 3.0, 0.0, 0.0, 0.0, 0.0});
    camera::PinholeModel s_cam(Vector3(0, 0, 0), R0, 30.0, 30.0, 48.0, 30.0, &strong), n_cam(Vector3(0, 0, 0), R0, 30.0, 30.0, 48.0, 30.0);
    threw = false;
    try { camera::b200_camera_transform(gray, s_cam, n_cam, BBox2i(300, 200, 50, 10)); }
    catch (camera::PointToPixelErr const& e) { threw = std::strstr(e.what(), "Projection into pinhole camera is inaccurate") != nullptr; }
    if (!threw) { std::printf("FAIL: the failed point_to_pixel check was not PointToPixelErr\n"); return 1; }
    std::printf("epipolar shim: %ld mismatches\n", bad);
    return bad ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
