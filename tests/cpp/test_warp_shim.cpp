// test_warp_shim.cpp -- exercises include/vwb200/ImageTransform.h the way Vision Workbench code would: every overload of
// b200_transform (the image's size, width x height, a bbox; default, edge-only and edge + interpolation tags) with a homography
// and with a B200DisparityTransform, each checked against the CPU oracle bit for bit.  Exit codes: 0 ok, 1 mismatch,
// 3 no CUDA device.
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/ImageTransform.h"
extern "C" {
#include "../../oracle/vw_warp_oracle.h"
}

using namespace vw;
using namespace vw::stereo;

struct Tx {
  int kind;
  double m[9];
  const float* disp;
  int dw, dh;
};

static long differ(ImageView<PixelGray<float>> const& got, ImageView<PixelGray<float>> const& image, Tx const& tx, int edge, int interp,
                   int x0, int y0, int ow, int oh) {
  if (got.cols() != ow || got.rows() != oh) return 1000000;
  std::vector<float> want(size_t(ow) * oh);
  vww_transform(tx.kind, interp, edge, tx.m, reinterpret_cast<const float*>(image.data()), image.cols(), image.rows(), tx.disp, tx.dw, tx.dh,
                x0, y0, want.data(), ow, oh);
  long bad = 0;
  for (int y = 0; y < oh; ++y)
    for (int x = 0; x < ow; ++x) bad += std::memcmp(&got(x, y), &want[size_t(y) * ow + x], 4) != 0;
  return bad;
}

// every overload for one transform argument; `tx` describes it to the oracle
template <class TxT>
static long run_all(ImageView<PixelGray<float>> const& im, TxT const& t, Tx const& tx) {
  const int W = im.cols(), H = im.rows();
  const ZeroEdgeExtension zero;
  const ConstantEdgeExtension constant;
  const BBox2i box(-7, 5, W + 11, H - 9);
  long bad = 0;
  bad += differ(b200_transform(im, t), im, tx, 0, 0, 0, 0, W, H);
  bad += differ(b200_transform(im, t, constant), im, tx, 1, 0, 0, 0, W, H);
  bad += differ(b200_transform(im, t, zero, BicubicInterpolation()), im, tx, 0, 1, 0, 0, W, H);
  bad += differ(b200_transform(im, t, constant, NearestPixelInterpolation()), im, tx, 1, 2, 0, 0, W, H);
  bad += differ(b200_transform(im, t, W / 2, H + 3), im, tx, 0, 0, 0, 0, W / 2, H + 3);
  bad += differ(b200_transform(im, t, W + 4, H / 3, constant), im, tx, 1, 0, 0, 0, W + 4, H / 3);
  bad += differ(b200_transform(im, t, W, H, constant, BicubicInterpolation()), im, tx, 1, 1, 0, 0, W, H);
  bad += differ(b200_transform(im, t, box), im, tx, 0, 0, -7, 5, W + 11, H - 9);
  bad += differ(b200_transform(im, t, box, constant), im, tx, 1, 0, -7, 5, W + 11, H - 9);
  bad += differ(b200_transform(im, t, box, zero, NearestPixelInterpolation()), im, tx, 0, 2, -7, 5, W + 11, H - 9);
  bad += differ(b200_transform(im, t, box, constant, BilinearInterpolation()), im, tx, 1, 0, -7, 5, W + 11, H - 9);
  return bad;
}

int main() {
  const int W = 173, H = 91;
  uint32_t s = 777u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (s >> 8) * (1.0f / 16777216.0f); };
  ImageView<PixelGray<float>> im(W, H);
  ImageView<PixelMask<Vector2f>> disp(W - 20, H - 10);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) im(x, y) = PixelGray<float>(100.0f * rnd() - 50.0f);
  for (int y = 0; y < disp.rows(); ++y)
    for (int x = 0; x < disp.cols(); ++x) {
      PixelMask<Vector2f> p(Vector2f(12.0f * rnd() - 6.0f, 4.0f * rnd() - 2.0f));
      if (rnd() < 0.25f) p.invalidate();
      disp(x, y) = p;
    }
  Matrix3x3 Hm;
  Hm.set_identity();
  Hm(0, 0) = 1.02; Hm(0, 1) = 0.04; Hm(0, 2) = -6.5; Hm(1, 0) = -0.03; Hm(1, 1) = 0.97; Hm(1, 2) = 3.25; Hm(2, 0) = 2e-4; Hm(2, 1) = -1e-4;
  Tx th{0, {}, nullptr, 0, 0};
  const Matrix3x3 inv = math::inverse(Hm);
  std::memcpy(th.m, inv.m, sizeof(th.m));
  Tx td{1, {1, 0, 0, 0, 1, 0, 0, 0, 1}, reinterpret_cast<const float*>(disp.data()), disp.cols(), disp.rows()};
  try {
    bool threw = false;
    Matrix3x3 singular;
    singular(0, 0) = 1.0; singular(1, 1) = 1.0;            // third row zero
    try { b200_transform(im, singular); }
    catch (MathErr const& e) { threw = std::strstr(e.what(), "singular") != nullptr; }
    if (!threw) { std::printf("FAIL: a singular homography was accepted\n"); return 1; }
    const long hbad = run_all(im, Hm, th);
    const long dbad = run_all(im, B200DisparityTransform(disp), td);
    std::printf("warp shim: %ld homography, %ld disparity mismatches\n", hbad, dbad);
    return (hbad || dbad) ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
