// test_dispmap_shim.cpp -- exercises include/vwb200/DisparityResampling.h the way Vision Workbench code would, with the
// reference's argument lists, on PixelMask<Vector2i> and PixelMask<Vector2f> disparities, and checks every call against the
// CPU oracle bit for bit.  Exit codes: 0 ok, 1 mismatch, 3 no CUDA device.
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/DisparityResampling.h"
extern "C" {
#include "../../oracle/vw_dispmap_oracle.h"
}

using namespace vw;
using namespace vw::stereo;

template <class PixelT>
static long differ(ImageView<PixelT> const& got, std::vector<PixelT> const& want) {
  if (size_t(got.cols()) * got.rows() != want.size()) return 1000000;
  long bad = 0;
  for (int y = 0; y < got.rows(); ++y)
    for (int x = 0; x < got.cols(); ++x) bad += std::memcmp(&got(x, y), &want[size_t(y) * got.cols() + x], sizeof(PixelT)) != 0;
  return bad;
}

template <class PixelT>
static long run_all(ImageView<PixelT> const& disp, int type, PixelT const& mn, PixelT const& mx) {
  const int W = disp.cols(), H = disp.rows();
  long bad = 0;
  std::vector<PixelT> want(size_t(2 * W) * 2 * H);
  want.resize(size_t(1 + (W - 1) / 2) * (1 + (H - 1) / 2));
  vwd_subsample(type, disp.data(), W, H, want.data());
  bad += differ(b200_disparity_subsample(disp), want);
  want.resize(size_t(2 * W) * 2 * H);
  vwd_upsample(type, disp.data(), W, H, want.data());
  bad += differ(b200_disparity_upsample(disp), want);
  float r[4];
  vwd_range(type, disp.data(), W, H, r);
  const BBox2f b = b200_get_disparity_range(disp);
  bad += std::memcmp(r, &b.min()[0], 8) != 0 || std::memcmp(r + 2, &b.max()[0], 8) != 0;
  want.resize(size_t(W) * H);
  vwd_range_mask(type, disp.data(), W, H, &mn.child()[0], &mx.child()[0], want.data());
  bad += differ(b200_disparity_range_mask(disp, mn, mx), want);
  Matrix3x3 Hm;
  Hm.set_identity();
  Hm(0, 0) = 0.98; Hm(0, 1) = 0.03; Hm(0, 2) = 12.5; Hm(1, 0) = -0.02; Hm(1, 1) = 1.01; Hm(1, 2) = -7.25; Hm(2, 0) = 1.5e-5; Hm(2, 1) = -2e-5;
  const Matrix3x3 inv = math::inverse(Hm);
  vwd_transform(type, 0, inv.m, 0, 0, 0, disp.data(), W, H, want.data());
  bad += differ(b200_transform_disparities(disp, Hm), want);
  for (int do_round = 0; do_round < 2; ++do_round) {
    vwd_transform(type, 1, Hm.m, do_round, 7, -3, disp.data(), W, H, want.data());
    bad += differ(b200_transform_disparities(do_round != 0, BBox2i(7, -3, W, H), Hm, disp), want);
  }
  return bad;
}

// a 2 x 3 matrix with the interface of vw::Matrix<double>: the explicit form must refuse it
struct Matrix2x3 {
  size_t rows() const { return 2; } size_t cols() const { return 3; }
  double operator()(size_t r, size_t c) const { return r == c ? 1.0 : 0.0; }
};

int main() {
  const int W = 161, H = 119;
  uint32_t s = 4242u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (s >> 8) * (1.0f / 16777216.0f); };
  ImageView<PixelMask<Vector2f>> df(W, H);
  ImageView<PixelMask<Vector2i>> di(W, H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      float dx = 0.1f * x + 8.0f * (rnd() - 0.5f), dy = -0.05f * y + 5.0f * (rnd() - 0.5f);
      PixelMask<Vector2f> p(Vector2f(dx, dy));
      PixelMask<Vector2i> q{Vector2i(static_cast<int32>(dx), static_cast<int32>(dy))};
      if (rnd() < 0.2f) { p.invalidate(); q.invalidate(); }
      df(x, y) = p;
      di(x, y) = q;
    }
  try {
    bool threw = false;
    try { b200_transform_disparities(false, BBox2i(0, 0, W - 1, H), Matrix3x3(), df); }
    catch (ArgumentErr const& e) { threw = std::strstr(e.what(), "The sizes of subregion and disparity don't match") != nullptr; }
    if (!threw) { std::printf("FAIL: a subregion of the wrong size was accepted\n"); return 1; }
    threw = false;
    try { b200_transform_disparities(false, BBox2i(0, 0, W, H), Matrix2x3(), df); }
    catch (ArgumentErr const& e) { threw = std::strstr(e.what(), "3x3") != nullptr; }
    if (!threw) { std::printf("FAIL: a 2 x 3 matrix was accepted\n"); return 1; }
    threw = false;
    Matrix3x3 singular;
    singular(0, 0) = 1.0; singular(1, 1) = 1.0;            // third row zero
    try { b200_transform_disparities(true, BBox2i(0, 0, W, H), singular, di); }
    catch (MathErr const& e) { threw = std::strstr(e.what(), "singular") != nullptr; }
    if (!threw) { std::printf("FAIL: a singular matrix was accepted\n"); return 1; }
    const long fbad = run_all(df, VWB200_DISP_F32, PixelMask<Vector2f>(Vector2f(-3.0f, -2.0f)), PixelMask<Vector2f>(Vector2f(W - 4.0f, H + 1.5f)));
    const long ibad = run_all(di, VWB200_DISP_I32, PixelMask<Vector2i>(Vector2i(-3, -2)), PixelMask<Vector2i>(Vector2i(W - 4, H + 1)));
    std::printf("dispmap shim: %ld float, %ld int mismatches\n", fbad, ibad);
    return (fbad || ibad) ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
