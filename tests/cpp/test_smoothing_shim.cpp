// test_smoothing_shim.cpp -- exercises include/vwb200/DisparitySmoothing.h the way Vision Workbench code would
// (tools/correlate.cc:234-247: texture_measure of the left image, then texture_preserving_disparity_filter; and
// disparity_median_filter) and checks the results against the CPU oracle, bit for bit (-0.0 == +0.0), together with the
// reference's aliasing: out shares in's buffer.  Exit codes: 0 ok, 1 mismatch, 3 no CUDA device.
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/DisparitySmoothing.h"
#include "../../oracle/vw_smoothing_oracle.h"

using namespace vw;
using namespace vw::stereo;

static long mismatches(const float* a, const float* b, size_t n) {
  long bad = 0;
  for (size_t i = 0; i < n; ++i) bad += !(a[i] == b[i]);
  return bad;
}

int main() {
  const int W = 200, H = 150;
  uint32_t s = 777u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (s >> 8) * (1.0f / 16777216.0f); };
  ImageView<PixelGray<float>> left(W, H);
  ImageView<PixelMask<Vector2f>> disp(W, H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      left(x, y) = (x > 60 && x < 140 && y > 40 && y < 110) ? 100.0f : float(int(rnd() * 255));
      PixelMask<Vector2f> p(Vector2f(0.05f * x + 4.0f * rnd(), -0.02f * y + 2.0f * rnd()));
      if (rnd() < 0.1f) p.invalidate();
      disp(x, y) = p;
    }
  std::vector<float> orig(reinterpret_cast<float*>(disp.data()), reinterpret_cast<float*>(disp.data()) + size_t(W) * H * 3);
  try {
    bool threw = false;
    ImageView<PixelMask<Vector2f>> out;
    try { b200_disparity_median_filter(disp, out, 33); } catch (NoImplErr const&) { threw = true; }
    if (!threw) { std::printf("FAIL: kernel 33 accepted\n"); return 1; }
    threw = false;
    ImageView<float> tex;
    try { b200_texture_measure(left, tex, 0); } catch (ArgumentErr const&) { threw = true; }
    if (!threw) { std::printf("FAIL: kernel 0 accepted\n"); return 1; }

    // texture chain of tools/correlate.cc:234-247
    b200_texture_measure(left, tex, 15);
    std::vector<float> lref(size_t(W) * H), tref(size_t(W) * H);
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) lref[size_t(y) * W + x] = left(x, y);
    if (vwo_texture_measure(lref.data(), W, H, W, 15, 0.5, 0.5, tref.data())) return 1;
    const long tbad = mismatches(tex.data(), tref.data(), tref.size());
    float tmax = 0;
    for (float v : tref) tmax = v > tmax ? v : tmax;
    tmax = 0.85f * tmax;
    std::vector<float> dref(orig);
    if (vwo_texture_preserving_disparity_filter(dref.data(), W, H, W, tref.data(), W, tmax, 13)) return 1;
    ImageView<PixelMask<Vector2f>> filtered;
    b200_texture_preserving_disparity_filter(disp, filtered, tex, tmax, 13);
    const bool shared = filtered.data() == disp.data();
    const long fbad = mismatches(reinterpret_cast<float*>(disp.data()), dref.data(), dref.size());
    long changed = 0;
    for (size_t i = 0; i < dref.size(); ++i) changed += dref[i] != orig[i];

    // median, in place on the same buffer
    if (vwo_disparity_median_filter(dref.data(), W, H, W, 5)) return 1;
    ImageView<PixelMask<Vector2f>> med;
    b200_disparity_median_filter(disp, med, 5);
    const long mbad = mismatches(reinterpret_cast<float*>(med.data()), dref.data(), dref.size());
    std::printf("smoothing shim: %ld texture, %ld texture-filter, %ld median mismatches; %ld floats smoothed; aliasing %s\n", tbad, fbad,
                mbad, changed, shared && med.data() == disp.data() ? "kept" : "LOST");
    return (tbad || fbad || mbad || !changed || !shared || med.data() != disp.data()) ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
