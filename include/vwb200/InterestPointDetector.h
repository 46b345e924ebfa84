// InterestPointDetector.h -- C++ shim: ipfind's default detection and description path with the reference's argument
// lists, computed on the device through include/vwb200.h, bit for bit the reference's points and descriptors:
//   IntegralAutoGainDetector (InterestPoint/IntegralDetector.h:74-103), detect_interest_points(image, detector, desired_num_ip)
//   (DetectorBase.h:302-328), remove_ip_near_nodata(image, nodata, ip_list, radius) (InterestPointUtils.h:45-82),
//   SGradDescriptorGenerator and describe_interest_points(image, generator, ip_list) (Descriptor.h:202-355, 414-471).
// The tile size is the reference's default_tile_size() floor, 1024 (b200_set_default_tile_size changes it).  Images are any
// single-channel view of float-convertible pixels, rasterised once.  Where the device has no exact form the shim throws
// NoImplErr: a detector with other than 8 scales, and desired_num_ip <= 0 with max_points > 0 (the reference then caps every
// tile at max_points without the area scaling).  NaN / inf pixels and points whose support leaves the 2^30 domain are
// ArgumentErr; without a device every call throws LogicErr ("no CUDA device").
#pragma once
#include <algorithm>
#include <cstring>
#include <list>
#include "PyramidCorrelationView.h"

namespace vw { namespace ip {

typedef std::list<InterestPoint> InterestPointList;

namespace b200_detail {
inline int& default_tile_size() { static int ts = 1024; return ts; }
// a dense float copy of a single-channel view
template <class ViewT>
inline std::vector<float> dense(ImageViewBase<ViewT> const& view, int& w, int& h) {
  ViewT const& v = view.impl();
  w = v.cols(); h = v.rows();
  std::vector<float> out(size_t(w) * size_t(h));
  for (int r = 0; r < h; ++r)
    for (int c = 0; c < w; ++c) out[size_t(r) * w + c] = float(v(c, r));
  return out;
}
inline vwb200_ip_point to_point(InterestPoint const& ip) {
  return vwb200_ip_point{ip.x, ip.y, ip.ix, ip.iy, ip.scale, ip.interest, ip.orientation};
}
}  // namespace b200_detail

inline void b200_set_default_tile_size(int tile_size) { b200_detail::default_tile_size() = tile_size; }

class IntegralAutoGainDetector {
public:
  static const int IP_DEFAULT_SCALES = 8;
  IntegralAutoGainDetector(size_t max_points = 200, size_t scales = IP_DEFAULT_SCALES) : m_max_points(int(max_points)), m_scales(int(scales)) {}
  int max_points() const { return m_max_points; }
  int scales() const { return m_scales; }
private:
  int m_max_points, m_scales;
};

class SGradDescriptorGenerator {
public:
  int support_size() const { return 42; }
  int descriptor_size() const { return 180; }
};

template <class ViewT>
inline InterestPointList detect_interest_points(ImageViewBase<ViewT> const& image, IntegralAutoGainDetector& detector, int desired_num_ip) {
  if (detector.scales() != IntegralAutoGainDetector::IP_DEFAULT_SCALES)
    vw_throw(NoImplErr() << "detect_interest_points: only the default 8 OBALoG scales have a device form");
  if (desired_num_ip <= 0 && detector.max_points() > 0)
    vw_throw(NoImplErr() << "detect_interest_points: desired_num_ip <= 0 with max_points > 0 has no device form");
  int w, h;
  const std::vector<float> img = b200_detail::dense(image, w, h);
  const int ipt = desired_num_ip > 0 ? desired_num_ip : 0;
  const int ts = std::max(1024, b200_detail::default_tile_size());
  long long cap = ipt > 0 ? (long long)((w + ts - 1) / ts) * ((h + ts - 1) / ts) * ipt : std::max(4096LL, (long long)w * h / 64);
  std::vector<vwb200_ip_point> pts;
  long long n = 0;
  for (;;) {
    pts.resize(size_t(std::max(cap, 1LL)));
    const int rc = vwb200_ipfind_detect(img.data(), w, h, w, b200_detail::default_tile_size(), ipt, pts.data(), cap, &n, 0, nullptr);
    if (rc == VWB200_EARG && n > cap) { cap = n; continue; }
    stereo::b200_detail::check(rc);
    break;
  }
  InterestPointList out;
  for (long long i = 0; i < n; ++i) {
    InterestPoint ip(pts[size_t(i)].x, pts[size_t(i)].y, pts[size_t(i)].scale, pts[size_t(i)].interest);
    ip.ix = pts[size_t(i)].ix; ip.iy = pts[size_t(i)].iy;
    out.push_back(ip);
  }
  return out;
}

template <class ImageT>
inline void remove_ip_near_nodata(ImageViewBase<ImageT> const& image, double nodata, InterestPointList& ip_list, int radius) {
  int w, h;
  const std::vector<float> img = b200_detail::dense(image, w, h);
  std::vector<vwb200_ip_point> pts;
  for (auto const& ip : ip_list) {
    pts.push_back(b200_detail::to_point(ip));
  }
  // the call reads ix / iy only: interest carries each point's index through the compaction
  for (size_t i = 0; i < pts.size(); ++i) { const int32_t k = int32_t(i); std::memcpy(&pts[i].interest, &k, sizeof k); }
  long long n = (long long)pts.size();
  stereo::b200_detail::check(vwb200_ipfind_remove_near_nodata(img.data(), w, h, w, nodata, radius, pts.data(), &n, 0, nullptr));
  std::vector<InterestPoint> all(ip_list.begin(), ip_list.end());
  InterestPointList kept;
  for (long long i = 0; i < n; ++i) {
    int32_t k;
    std::memcpy(&k, &pts[size_t(i)].interest, sizeof k);
    kept.push_back(all[size_t(k)]);
  }
  ip_list.swap(kept);
}

template <class ViewT>
inline void describe_interest_points(ImageViewBase<ViewT> const& view, SGradDescriptorGenerator& /*descriptor*/, InterestPointList& list) {
  int w, h;
  const std::vector<float> img = b200_detail::dense(view, w, h);
  std::vector<InterestPoint> all(list.begin(), list.end());
  std::vector<vwb200_ip_point> pts;
  for (size_t i = 0; i < all.size(); ++i) {
    vwb200_ip_point p = b200_detail::to_point(all[i]);
    p.ix = int32_t(i);                           // describe reads x, y, scale and orientation only: ix carries the index
    pts.push_back(p);
  }
  std::vector<float> desc(all.size() * 180);
  stereo::b200_detail::check(vwb200_ipfind_describe(img.data(), w, h, w, b200_detail::default_tile_size(), pts.data(), (long long)pts.size(),
                                                    desc.data(), 0, nullptr));
  list.clear();
  for (size_t i = 0; i < pts.size(); ++i) {
    InterestPoint ip = all[size_t(pts[i].ix)];
    ip.x = pts[i].x; ip.y = pts[i].y;
    ip.descriptor.assign(desc.begin() + std::ptrdiff_t(i * 180), desc.begin() + std::ptrdiff_t((i + 1) * 180));
    list.push_back(ip);
  }
}

}}  // namespace vw::ip
