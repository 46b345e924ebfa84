// test_outliers_shim.cpp -- exercises include/vwb200/DisparityOutliers.h the way Vision Workbench code would, on
// PixelMask<Vector2i> and PixelMask<Vector2f> disparities, and checks all six filters against the CPU oracle bit for bit.
// Exit codes: 0 ok, 1 mismatch, 3 no CUDA device.
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/DisparityOutliers.h"
#include "../../oracle/vw_outlier_oracle.h"

using namespace vw;
using namespace vw::stereo;

template <class PixelT>
static long run_all(ImageView<PixelT> const& disp, int type) {
  const int W = disp.cols(), H = disp.rows();
  std::vector<PixelT> want(size_t(W) * H);
  long bad = 0;
  for (int method = 0; method < 3; ++method)
    for (int cleanup = 0; cleanup < 2; ++cleanup) {
      const double pt = 2.0, rt = method == 2 ? 0.5 : 0.4, mmd = 3.0;
      ImageView<PixelT> got;
      if (method == 0) got = cleanup ? b200_disparity_cleanup_using_thresh(disp, 3, 2, pt, rt) : b200_rm_outliers_using_thresh(disp, 3, 2, pt, rt);
      if (method == 1) got = cleanup ? b200_disparity_cleanup_using_mean(disp, 3, 2, mmd) : b200_rm_outliers_using_mean(disp, 3, 2, mmd);
      if (method == 2) got = cleanup ? b200_disparity_cleanup_using_stddev(disp, 3, 2, pt, rt) : b200_rm_outliers_using_stddev(disp, 3, 2, pt, rt);
      if (vwo_outlier_filter(method, cleanup, type, disp.data(), W, H, 3, 2, pt, rt, mmd, want.data())) return -1;
      long changed = 0;
      for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
          bad += std::memcmp(&got(x, y), &want[size_t(y) * W + x], sizeof(PixelT)) != 0;
          changed += std::memcmp(&got(x, y), &disp(x, y), sizeof(PixelT)) != 0;
        }
      if (!changed) bad += 1000000;                 // every filter rejects something on this raster
    }
  return bad;
}

int main() {
  const int W = 160, H = 120;
  uint32_t s = 4242u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (s >> 8) * (1.0f / 16777216.0f); };
  ImageView<PixelMask<Vector2f>> df(W, H);
  ImageView<PixelMask<Vector2i>> di(W, H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      float dx = 0.1f * x + 0.8f * rnd(), dy = -0.05f * y + 0.5f * rnd();
      if (rnd() < 0.05f) dx += 60.0f * (rnd() - 0.5f);
      PixelMask<Vector2f> p(Vector2f(dx, dy));
      PixelMask<Vector2i> q{Vector2i(static_cast<int32>(dx), static_cast<int32>(dy))};
      if (rnd() < 0.15f) { p.invalidate(); q.invalidate(); }
      df(x, y) = p;
      di(x, y) = q;
    }
  try {
    bool threw = false;
    try { b200_rm_outliers_using_mean(df, 0, 1, 1.0); } catch (ArgumentErr const& e) { threw = std::strstr(e.what(), "RmOutliersUsingMeanFunc") != nullptr; }
    if (!threw) { std::printf("FAIL: zero half kernel accepted\n"); return 1; }
    const long fbad = run_all(df, VWB200_DISP_F32), ibad = run_all(di, VWB200_DISP_I32);
    std::printf("outliers shim: %ld float, %ld int mismatches\n", fbad, ibad);
    return (fbad || ibad) ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
