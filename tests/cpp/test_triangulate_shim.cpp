// test_triangulate_shim.cpp -- exercises include/vwb200/StereoView.h the way Vision Workbench code would, with the reference's
// argument lists (PinholeModel constructors, stereo_triangulate(disparity, &cam1, &cam2), StereoModel(&cam1, &cam2, angle_tol),
// UniverseRadiusFunc(origin, near, far)), on PixelMask<Vector2i> and PixelMask<Vector2f> disparities, and checks it against the
// CPU oracle bit for bit.  Exit codes: 0 ok, 1 mismatch, 3 no CUDA device.
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/StereoView.h"
extern "C" {
#include "../../oracle/vw_triangulate_oracle.h"
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

struct NotPinhole : camera::CameraModel { std::string type() const override { return "Other"; } };

int main() {
  const int W = 97, H = 61;
  Matrix3x3 R;
  R.set_identity();
  const double c = 0.8, s = 0.6;                                   // a rotation about y
  R(0, 0) = c; R(0, 2) = s; R(2, 0) = -s; R(2, 2) = c;
  camera::TsaiLensDistortion tsai(std::vector<double>{-0.12, 0.03, 1e-3, -2e-3, 0.01});
  camera::PinholeModel cam1(Vector3(0.5, -0.2, 1.0), R, 500.0, 505.0, 48.0, 30.0);
  camera::PinholeModel cam2(Vector3(0.5 + c, -0.2, 1.0 - s), R, 500.0, 505.0, 48.0, 30.0, Vector3(1, 0, 0), Vector3(0, 1, 0), Vector3(0, 0, 1),
                            &tsai, 1.0);
  uint32_t seed = 99u;
  auto rnd = [&seed]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
  ImageView<PixelMask<Vector2f>> df(W, H);
  ImageView<PixelMask<Vector2i>> di(W, H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      PixelMask<Vector2f> p(Vector2f(-10.0f - 40.0f * rnd(), 2.0f * rnd() - 1.0f));
      PixelMask<Vector2i> q{Vector2i(-10 - int(40 * rnd()), int(3 * rnd()) - 1)};
      if (rnd() < 0.1f) { p.invalidate(); q.invalidate(); }
      df(x, y) = p;
      di(x, y) = q;
    }
  const vwt_pinhole o1 = oracle_cam(cam1), o2 = oracle_cam(cam2);
  long bad = 0;
  try {
    bool threw = false;
    NotPinhole other;
    try { stereo::b200_stereo_triangulate(df, &cam1, &other); }
    catch (NoImplErr const&) { threw = true; }
    if (!threw) { std::printf("FAIL: a camera that is not a PinholeModel was accepted\n"); return 1; }
    // the ImageView<Vector3> result = stereo_triangulate(...) form, and rasterize() over windows
    std::vector<double> want(size_t(W) * H * 3);
    ImageView<Vector3> pf = stereo::b200_stereo_triangulate(df, &cam1, &cam2);
    vwt_stereo_triangulate(1, df.data(), W, H, 0, 0, W, H, &o1, &o2, 0.0, want.data());
    bad += differ(pf.data(), want.data(), want.size() * 8);
    ImageView<Vector3> pi = stereo::b200_stereo_triangulate(di, &cam1, &cam2);
    vwt_stereo_triangulate(0, di.data(), W, H, 0, 0, W, H, &o1, &o2, 0.0, want.data());
    bad += differ(pi.data(), want.data(), want.size() * 8);
    const int wins[3][4] = {{10, 7, 40, 33}, {0, 0, 1, 1}, {W - 25, H - 9, 25, 9}};
    for (auto const& w : wins) {
      std::vector<double> ww(size_t(w[2]) * w[3] * 3);
      ImageView<Vector3> out(w[2], w[3]);
      stereo::b200_stereo_triangulate(df, &cam1, &cam2).rasterize(out, BBox2i(w[0], w[1], w[2], w[3]));
      vwt_stereo_triangulate(1, df.data(), W, H, w[0], w[1], w[2], w[3], &o1, &o2, 0.0, ww.data());
      bad += differ(out.data(), ww.data(), ww.size() * 8);
    }
    // StereoModel's image form
    for (double tol : {0.0, 0.02}) {
      ImageView<double> err;
      ImageView<Vector3> xyz = stereo::B200StereoModel(&cam1, &cam2, tol)(df, err);
      std::vector<double> we(size_t(W) * H);
      double st[4];
      vwt_stereo_model(reinterpret_cast<const float*>(df.data()), W, H, &o1, &o2, tol, want.data(), we.data(), st);
      bad += differ(xyz.data(), want.data(), want.size() * 8) + differ(err.data(), we.data(), we.size() * 8);
      // UniverseRadiusFunc in place
      std::vector<double> wr(want.size());
      long long counts[2];
      const double org[3] = {0.5, -0.2, 1.0};
      vwt_universe_radius(want.data(), W, H, org, 5.0, 60.0, wr.data(), counts);
      std::pair<long long, long long> got = stereo::b200_universe_radius(xyz, Vector3(0.5, -0.2, 1.0), 5.0, 60.0);
      bad += differ(xyz.data(), wr.data(), wr.size() * 8) + (got.first != counts[0]) + (got.second != counts[1]);
    }
    threw = false;
    ImageView<Vector3> pts(2, 2);
    try { stereo::b200_universe_radius(pts, Vector3(), 2.0, 1.0); }
    catch (ArgumentErr const& e) { threw = std::strstr(e.what(), "near radius must be <= far radius") != nullptr; }
    if (!threw) { std::printf("FAIL: near > far was accepted\n"); return 1; }
    std::printf("triangulate shim: %ld mismatches\n", bad);
    return bad ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
