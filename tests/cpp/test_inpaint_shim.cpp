// test_inpaint_shim.cpp -- exercises include/vwb200/InpaintView.h the way Vision Workbench code would, with the reference's
// argument list, on PixelMask<Vector2i> and PixelMask<Vector2f> disparities, and checks it against the CPU oracle bit for bit:
// the whole image (the ImageView<PixelT> result = fill_holes_grass(...) form) and rasterize() over sub-windows.
// Exit codes: 0 ok, 1 mismatch, 3 no CUDA device.
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/InpaintView.h"
extern "C" {
#include "../../oracle/vw_inpaint_oracle.h"
}

using namespace vw;

template <class PixelT>
static long differ(ImageView<PixelT> const& got, std::vector<PixelT> const& want) {
  if (size_t(got.cols()) * got.rows() != want.size()) return 1000000;
  long bad = 0;
  for (int y = 0; y < got.rows(); ++y)
    for (int x = 0; x < got.cols(); ++x) bad += std::memcmp(&got(x, y), &want[size_t(y) * got.cols() + x], sizeof(PixelT)) != 0;
  return bad;
}

template <class PixelT>
static long run_all(ImageView<PixelT> const& disp, int type) {
  const int W = disp.cols(), H = disp.rows();
  long bad = 0;
  for (int len : {0, 1, 3, 8, 20}) {
    std::vector<PixelT> want(size_t(W) * H);
    vwi_fill_holes_grass(type, disp.data(), W, H, len, 0, 0, W, H, want.data(), nullptr);
    ImageView<PixelT> whole = b200_fill_holes_grass(disp, len);
    bad += differ(whole, want);
    const int wins[3][4] = {{10, 7, 40, 33}, {0, 0, 1, 1}, {W - 25, H - 9, 25, 9}};
    for (auto const& w : wins) {
      want.assign(size_t(w[2]) * w[3], PixelT());
      vwi_fill_holes_grass(type, disp.data(), W, H, len, w[0], w[1], w[2], w[3], want.data(), nullptr);
      ImageView<PixelT> out(w[2], w[3]);
      b200_fill_holes_grass(disp, len).rasterize(out, BBox2i(w[0], w[1], w[2], w[3]));
      bad += differ(out, want);
    }
  }
  return bad;
}

int main() {
  const int W = 131, H = 97;
  uint32_t s = 777u;
  auto rnd = [&s]() { s = s * 1664525u + 1013904223u; return (s >> 8) * (1.0f / 16777216.0f); };
  ImageView<PixelMask<Vector2f>> df(W, H);
  ImageView<PixelMask<Vector2i>> di(W, H);
  for (int y = 0; y < H; ++y)
    for (int x = 0; x < W; ++x) {
      float dx = 0.1f * x + 8.0f * (rnd() - 0.5f), dy = -0.05f * y + 5.0f * (rnd() - 0.5f);
      PixelMask<Vector2f> p(Vector2f(dx, dy));
      PixelMask<Vector2i> q{Vector2i(static_cast<int32>(dx * 10), static_cast<int32>(dy * 10))};
      const int cx = (x / 16) * 16 + 8, cy = (y / 16) * 16 + 8, r2 = (x - cx) * (x - cx) + (y - cy) * (y - cy);
      if (rnd() < 0.03f || r2 <= ((x / 16 + y / 16) % 6)) { p.invalidate(); q.invalidate(); }
      df(x, y) = p;
      di(x, y) = q;
    }
  try {
    bool threw = false;
    try { b200_fill_holes_grass(df, 3)(0, 0); }
    catch (NoImplErr const& e) { threw = std::strstr(e.what(), "FillHolesGrass::operator() is not implemented") != nullptr; }
    if (!threw) { std::printf("FAIL: operator() did not throw NoImplErr\n"); return 1; }
    threw = false;
    try { ImageView<PixelMask<Vector2f>> o = b200_fill_holes_grass(df, -1); (void)o; }
    catch (ArgumentErr const& e) { threw = std::strstr(e.what(), "negative") != nullptr; }
    if (!threw) { std::printf("FAIL: a negative hole_fill_len was accepted\n"); return 1; }
    const long fbad = run_all(df, VWB200_DISP_F32);
    const long ibad = run_all(di, VWB200_DISP_I32);
    std::printf("inpaint shim: %ld float, %ld int mismatches\n", fbad, ibad);
    return (fbad || ibad) ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
