// InterestPointMatcher.h -- C++ shim: InterestPointMatcherSimple<L2NormMetric | HammingMetric, NullConstraint> and
// remove_duplicates of InterestPoint/Matcher.{h,cc} with the reference's argument lists, the matching computed on the device
// through include/vwb200.h.  B200InterestPointMatcherSimple<Metric, Constraint>(threshold)(ip1, ip2, matched_ip1, matched_ip2,
// progress, quiet) fills the matched lists in the reference's order, bit for bit its choices.  Where the reference's behaviour
// is undefined the shim throws ArgumentErr: descriptors of unequal length, Hamming values outside (-1, 256) or NaN, and (in
// b200_remove_duplicates) NaN coordinates.  A Hamming descriptor longer than 2^21 is NoImplErr.
#pragma once
#include <iterator>
#include "PyramidCorrelationView.h"

namespace vw { namespace ip {

namespace b200_detail {
template <class MetricT> struct MetricCode;
template <> struct MetricCode<L2NormMetric> { enum { value = VWB200_METRIC_L2 }; };
template <> struct MetricCode<HammingMetric> { enum { value = VWB200_METRIC_HAMMING }; };

// n x dim dense descriptors and polarity bytes of a list; ArgumentErr for descriptors of unequal length
template <class ListT>
inline void pack(ListT const& ips, int dim, std::vector<float>& desc, std::vector<uint8_t>& pol) {
  desc.clear(); pol.clear();
  desc.reserve(ips.size() * size_t(dim));
  for (auto const& ip : ips) {
    if (int(ip.descriptor.size()) != dim)
      vw_throw(ArgumentErr() << "InterestPointMatcherSimple: descriptors of unequal length (" << ip.descriptor.size() << " and " << dim << ")");
    for (size_t k = 0; k < ip.descriptor.size(); ++k) desc.push_back(float(ip.descriptor[k]));
    pol.push_back(ip.polarity ? 1 : 0);
  }
}
}  // namespace b200_detail

template <class MetricT, class ConstraintT>
class B200InterestPointMatcherSimple {
  double m_threshold;

public:
  B200InterestPointMatcherSimple(double threshold = 0.5, MetricT = MetricT(), ConstraintT = ConstraintT()) : m_threshold(threshold) {}

  template <class ListT, class MatchListT>
  void operator()(ListT const& ip1, ListT const& ip2, MatchListT& matched_ip1, MatchListT& matched_ip2,
                  const ProgressCallback& progress_callback = ProgressCallback::dummy_instance(), bool quiet = false) const {
    matched_ip1.clear(); matched_ip2.clear();
    if (!ip1.size() || !ip2.size()) {
      if (!quiet) progress_callback.report_finished();
      return;
    }
    if (!quiet) progress_callback.report_progress(0);
    const int dim = int(ip1.begin()->descriptor.size());
    std::vector<float> d1, d2;
    std::vector<uint8_t> p1, p2;
    b200_detail::pack(ip1, dim, d1, p1);
    b200_detail::pack(ip2, dim, d2, p2);
    std::vector<int32_t> index(ip1.size());
    stereo::b200_detail::check(vwb200_ip_match(b200_detail::MetricCode<MetricT>::value, d1.data(), p1.data(), int(ip1.size()), d2.data(),
                                               p2.data(), int(ip2.size()), dim, dim, dim, m_threshold, index.data(), nullptr, nullptr,
                                               /*on_device=*/0, nullptr));
    if (!quiet) progress_callback.report_finished();
    std::vector<typename ListT::const_iterator> at2;
    at2.reserve(ip2.size());
    for (auto it = ip2.begin(); it != ip2.end(); ++it) at2.push_back(it);
    size_t i = 0;
    for (auto it = ip1.begin(); it != ip1.end(); ++it, ++i)
      if (index[i] != -1) {
        matched_ip1.push_back(*it);
        matched_ip2.push_back(*at2[size_t(index[i])]);
      }
  }
};

// remove_duplicates (Matcher.cc:151-195): keeps the last of the pairs that share an ip1 or an ip2 position
inline void b200_remove_duplicates(std::vector<InterestPoint>& ip1, std::vector<InterestPoint>& ip2) {
  if (ip1.size() != ip2.size()) vw_throw(ArgumentErr() << "Input vectors are not the same size.");
  std::vector<float> xy1(2 * ip1.size()), xy2(2 * ip2.size());
  for (size_t i = 0; i < ip1.size(); ++i) {
    xy1[2 * i] = ip1[i].x; xy1[2 * i + 1] = ip1[i].y;
    xy2[2 * i] = ip2[i].x; xy2[2 * i + 1] = ip2[i].y;
  }
  std::vector<int32_t> keep(ip1.size());
  int n = 0;
  stereo::b200_detail::check(vwb200_remove_duplicate_matches(xy1.data(), xy2.data(), int(ip1.size()), keep.data(), &n));
  std::vector<InterestPoint> a, b;
  a.reserve(size_t(n)); b.reserve(size_t(n));
  for (int k = 0; k < n; ++k) { a.push_back(ip1[size_t(keep[k])]); b.push_back(ip2[size_t(keep[k])]); }
  ip1.swap(a);
  ip2.swap(b);
}

}}  // namespace vw::ip
