// test_ipfind_shim.cpp -- exercises include/vwb200/InterestPointDetector.h the way ipfind does: normalize (the oracle's),
// detect_interest_points with IntegralAutoGainDetector, remove_ip_near_nodata, then describe_interest_points with
// SGradDescriptorGenerator, every field and descriptor float checked against the CPU oracle as raw bits.
// Exit codes: 0 ok, 1 mismatch, 3 no CUDA device.
#include <cstdio>
#include <cstring>
#include <vector>
#include "vwb200/InterestPointDetector.h"
extern "C" {
#include "../../oracle/vw_ipfind_oracle.h"
}

using namespace vw;
using namespace vw::ip;

static uint32_t s = 777u;
static float rnd() { s = s * 1664525u + 1013904223u; return (s >> 8) * (1.0f / 16777216.0f); }

static bool same(float a, float b) { return std::memcmp(&a, &b, 4) == 0; }

static long compare(InterestPointList const& got, const vwf_point* want, long long n, const float* desc) {
  long bad = long(got.size() != size_t(n)) * 1000;
  long long i = 0;
  for (auto const& ip : got) {
    if (i >= n) break;
    const vwf_point& p = want[i];
    bad += long(!same(ip.x, p.x) || !same(ip.y, p.y) || ip.ix != p.ix || ip.iy != p.iy || !same(ip.scale, p.scale) ||
                !same(ip.interest, p.interest) || !same(ip.orientation, p.orientation));
    if (desc) bad += long(ip.descriptor.size() != 180 || std::memcmp(ip.descriptor.data(), desc + i * 180, 180 * 4) != 0);
    ++i;
  }
  return bad;
}

int main() {
  try {
    const int w = 1300, h = 1100;
    std::vector<float> coarse(size_t(w / 4 + 2) * (h / 4 + 2));
    for (float& v : coarse) v = rnd();
    std::vector<float> raw(size_t(w) * h), img(raw.size());
    for (int r = 0; r < h; ++r)
      for (int c = 0; c < w; ++c) raw[size_t(r) * w + c] = float(int(coarse[size_t(r / 4) * (w / 4 + 2) + c / 4] * 255.0f));
    for (int r = 200; r < 240; ++r)
      for (int c = 300; c < 360; ++c) raw[size_t(r) * w + c] = 0.0f;                       // nodata 0, as ipfind without one
    vwf_normalize(raw.data(), w, h, 0, 0.0, img.data());
    ImageView<float> image(w, h), raw_image(w, h);
    std::memcpy(image.data(), img.data(), img.size() * 4);
    std::memcpy(raw_image.data(), raw.data(), raw.size() * 4);
    long bad = 0;
    for (int ipt : {250, 7}) {
      IntegralAutoGainDetector detector(ipt);
      InterestPointList ip = detect_interest_points(image, detector, ipt);
      vwf_point* want = nullptr;
      long long n = 0, stats[5];
      vwf_detect(img.data(), w, h, 1024, ipt, &want, &n, stats);
      bad += compare(ip, want, n, nullptr);
      remove_ip_near_nodata(raw_image, 0.0, ip, 2);
      n = vwf_remove_near_nodata(raw.data(), w, h, 0.0, 2, want, n);
      bad += compare(ip, want, n, nullptr);
      SGradDescriptorGenerator gen;
      describe_interest_points(image, gen, ip);
      std::vector<float> desc(size_t(n) * 180);
      vwf_describe(img.data(), w, h, 1024, want, n, desc.data());
      bad += compare(ip, want, n, desc.data());
      vwf_free(want);
    }
    bool threw = false;
    try { IntegralAutoGainDetector d(100, 5); detect_interest_points(image, d, 10); }
    catch (NoImplErr const&) { threw = true; }
    if (!threw) { std::printf("FAIL: a 5-scale detector was accepted\n"); return 1; }
    std::printf("ipfind shim: %ld mismatches\n", bad);
    return bad ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
