// cahv.cuh -- CAHVModel and CAHVORModel on the device, shared by K8 (camera_transform) and K10 (triangulation):
// pixel_to_vector (Camera/CAHVModel.cc:173-185; CAHVORModel.cc:297-348, the overload without partial derivatives, with its
// Newton loop on k5*u^5 + k3*u^3 + k1*u = 1) and point_to_pixel (CAHVModel.cc:167-171; CAHVORModel.cc:431-448).  Neither
// has a round-trip check.  The camera is a CahvCam; cahvor == 0 is a CAHV camera.  As in pinhole.cuh every product, sum,
// quotient and square root is an explicitly rounded intrinsic in the reference's order (dot products and norms summed from
// 0.0, normalize dividing each component by norm_2), so nothing is contracted into an FMA.  The vector helpers and
// cahv_pixel_to_vector are also the host's: linearize_camera (cameras.cu) evaluates the CAHVOR rays with them.
#pragma once
#include "pinhole.cuh"

namespace vwb200 {
namespace {

constexpr int kCahvorMaxIter = 20;                     // VW_CAHVOR_MAXITER (CAHVORModel.cc:115)
constexpr double kCahvorConv = 1.0e-6;                 // VW_CAHVOR_CONV (:116)

__host__ __device__ __forceinline__ V3 add3(V3 a, V3 b) { return V3{dadd(a.x, b.x), dadd(a.y, b.y), dadd(a.z, b.z)}; }
__host__ __device__ __forceinline__ V3 scale3(double s, V3 a) { return V3{dmul(s, a.x), dmul(s, a.y), dmul(s, a.z)}; }
__host__ __device__ __forceinline__ V3 normalize3(V3 a) {  // Math/Vector.h:1694: each component / norm_2
  const double n = norm3(a);
  return V3{ddiv(a.x, n), ddiv(a.y, n), ddiv(a.z, n)};
}

// pixel_to_vector(pix): normalize(cross(V - y*A, H - x*A)), negated for a left-handed V x H; for CAHVOR the radial
// distortion removed by Newton's method.  *iters counts the Newton passes (each computes poly and deriv).  MAYBE_CAHVOR ==
// false compiles the CAHV form alone, for a camera the host has checked to be CAHV (camera_transform's destination).
template <bool MAYBE_CAHVOR>
__host__ __device__ __forceinline__ V3 cahv_pixel_to_vector(const CahvCam& c, double x, double y, int* iters) {
  const V3 A = ld3(c.A);
  V3 rr = normalize3(cross3(sub3(ld3(c.V), scale3(y, A)), sub3(ld3(c.H), scale3(x, A))));
  if (c.flip) rr = scale3(-1.0, rr);
  if (!MAYBE_CAHVOR || !c.cahvor) return rr;
  const V3 O = ld3(c.O);
  const double omega = dot3(rr, O);
  const V3 lambda = sub3(rr, scale3(omega, O));
  const double tau = ddiv(dot3(lambda, lambda), dmul(omega, omega));
  const double k1 = dadd(1.0, c.R[0]);
  const double k3 = dmul(c.R[1], tau);
  const double k5 = dmul(dmul(c.R[2], tau), tau);
  double u = dsub(1.0, dadd(dadd(c.R[0], k3), k5));
  for (int i = 0; i < kCahvorMaxIter; ++i) {           // the i >= MAXITER exit comes before the step
    ++*iters;
    const double u2 = dmul(u, u);
    const double poly = dsub(dmul(dadd(dmul(dadd(dmul(k5, u2), k3), u2), k1), u), 1.0);
    const double deriv = dadd(dmul(dadd(dmul(dmul(5.0, k5), u2), dmul(3.0, k3)), u2), k1);
    if (deriv <= 0) break;                             // "distortion is too negative": u is kept
    const double du = ddiv(poly, deriv);
    u = dsub(u, du);
    if (fabs(du) < kCahvorConv) break;
  }
  return normalize3(sub3(rr, scale3(dsub(1.0, u), lambda)));
}

// point_to_pixel(point): (dot(p, H) / dot(p, A), dot(p, V) / dot(p, A)) of p = point - C, for CAHVOR p + mu * lambda
__device__ __forceinline__ void cahv_point_to_pixel(const CahvCam& c, V3 point, double* u, double* v) {
  V3 p = sub3(point, ld3(c.C));
  if (c.cahvor) {
    const V3 O = ld3(c.O);
    const double omega = dot3(p, O);
    const V3 lambda = sub3(p, scale3(omega, O));
    const double tau = ddiv(dot3(lambda, lambda), dmul(omega, omega));
    const double mu = dadd(dadd(c.R[0], dmul(c.R[1], tau)), dmul(dmul(c.R[2], tau), tau));
    p = add3(p, scale3(mu, lambda));
  }
  const double alpha = dot3(p, ld3(c.A));
  *u = ddiv(dot3(p, ld3(c.H)), alpha);
  *v = ddiv(dot3(p, ld3(c.V)), alpha);
}

// CameraTransform(src, dst)::reverse (Camera/CameraTransform.h:52-61): src.point_to_pixel(dst.pixel_to_vector(p) + dst.C), with
// dst a CAHV camera (so no Newton loop runs here) and src CAHV or CAHVOR
__device__ __forceinline__ void cahv_camera_map(const CahvCam& from, const CahvCam& to, double x, double y, double* u, double* v) {
  int iters = 0;
  const V3 r = cahv_pixel_to_vector<false>(from, x, y, &iters);
  cahv_point_to_pixel(to, add3(r, ld3(from.C)), u, v);
}

}  // namespace
}  // namespace vwb200
