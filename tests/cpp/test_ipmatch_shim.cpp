// test_ipmatch_shim.cpp -- exercises include/vwb200/InterestPointMatcher.h the way Vision Workbench code would: the Simple
// matcher with L2NormMetric and HammingMetric over std::vector and std::list interest point lists, then remove_duplicates,
// checked against the CPU oracle.  Every point's x is its list index, so a matched pair names its indices.
// Exit codes: 0 ok, 1 mismatch, 3 no CUDA device.
#include <cstdio>
#include <cstring>
#include <list>
#include <vector>
#include "vwb200/InterestPointMatcher.h"
extern "C" {
#include "../../oracle/vw_ipmatch_oracle.h"
}

using namespace vw;
using namespace vw::ip;

static uint32_t s = 4242u;
static float rnd() { s = s * 1664525u + 1013904223u; return (s >> 8) * (1.0f / 16777216.0f); }

static std::vector<InterestPoint> make(int n, int dim, bool bytes) {
  std::vector<InterestPoint> v;
  for (int i = 0; i < n; ++i) {
    InterestPoint ip(float(i), float((i * 7) % 13), 1.0f, 0.0f, 0.0f, rnd() < 0.5f);
    for (int k = 0; k < dim; ++k) ip.descriptor.push_back(bytes ? float(int(rnd() * 256.0f)) : rnd() * 4.0f - 2.0f);
    v.push_back(ip);
  }
  return v;
}

template <class MetricT>
static long run(int metric, int n1, int n2, int dim, double thr) {
  std::vector<InterestPoint> a = make(n1, dim, metric == 1), b = make(n2, dim, metric == 1);
  for (int i = 0; i < n2 / 3 && i < n1; ++i) b[size_t(3 * i)].descriptor = a[size_t(i)].descriptor;     // exact and tied matches
  std::vector<float> d1, d2;
  std::vector<uint8_t> p1, p2;
  b200_detail::pack(a, dim, d1, p1);
  b200_detail::pack(b, dim, d2, p2);
  std::vector<int32_t> want(static_cast<size_t>(n1));
  int bl = 0; long long be = 0;
  vwm_match(metric, d1.data(), p1.data(), n1, d2.data(), p2.data(), n2, dim, thr, want.data(), nullptr, nullptr, &bl, &be);
  std::list<InterestPoint> la(a.begin(), a.end()), lb(b.begin(), b.end());
  std::vector<InterestPoint> m1, m2;
  const B200InterestPointMatcherSimple<MetricT, NullConstraint> matcher(thr);
  matcher(la, lb, m1, m2);
  long bad = 0;
  size_t k = 0;
  for (int i = 0; i < n1; ++i)
    if (want[size_t(i)] != -1) {
      if (k >= m1.size() || int(m1[k].x) != i || int(m2[k].x) != want[size_t(i)]) ++bad;
      ++k;
    }
  bad += long(m1.size() != k) + long(m2.size() != k);
  // remove_duplicates against the oracle
  std::vector<float> xy1, xy2;
  for (size_t j = 0; j < m1.size(); ++j) { xy1.push_back(m1[j].x); xy1.push_back(float(int(m1[j].x) % 5)); xy2.push_back(m2[j].x); xy2.push_back(m2[j].y); }
  for (size_t j = 0; j < m1.size(); ++j) m1[j].y = xy1[2 * j + 1], m1[j].x = float(int(m1[j].x) % 11);
  for (size_t j = 0; j < m1.size(); ++j) xy1[2 * j] = m1[j].x;
  std::vector<int32_t> keep(m1.size() + 1);
  int nk = 0;
  vwm_remove_duplicates(xy1.data(), xy2.data(), int(m1.size()), keep.data(), &nk);
  std::vector<InterestPoint> r1 = m1, r2 = m2;
  b200_remove_duplicates(r1, r2);
  if (int(r1.size()) != nk || int(r2.size()) != nk) return bad + 1000;
  for (int j = 0; j < nk; ++j) bad += long(std::memcmp(&r1[size_t(j)].x, &m1[size_t(keep[size_t(j)])].x, 8) != 0);
  return bad;
}

int main() {
  try {
    std::vector<InterestPoint> a = make(3, 4, false), b = make(3, 5, false), m1, m2;
    bool threw = false;
    try { const B200InterestPointMatcherSimple<L2NormMetric, NullConstraint> matcher; matcher(a, b, m1, m2); }
    catch (ArgumentErr const& e) { threw = std::strstr(e.what(), "unequal length") != nullptr; }
    if (!threw) { std::printf("FAIL: descriptors of unequal length were accepted\n"); return 1; }
    long bad = 0;
    bad += run<L2NormMetric>(0, 300, 451, 128, 0.8);
    bad += run<L2NormMetric>(0, 40, 3000, 15, 0.5);
    bad += run<HammingMetric>(1, 500, 260, 32, 0.8);
    bad += run<HammingMetric>(1, 70, 90, 13, 1.0);
    std::printf("ipmatch shim: %ld mismatches\n", bad);
    return bad ? 1 : 0;
  } catch (LogicErr const& e) {
    std::printf("NODEVICE-or-CUDA: %s\n", e.what());
    return 3;
  }
}
