// pinhole.cuh -- PinholeModel on the device, shared by K8 (camera_transform) and K10 (triangulation): pixel_to_vector
// (Camera/PinholeModel.cc:422-430) with the Tsai Newton-Raphson undistortion (LensDistortion.cc:258-400,
// Math/NewtonRaphson.cc:58-119), and point_to_pixel (:351-397) with the closed-form Tsai distortion (LensDistortion.cc:345-369)
// and the pixel_to_vector round-trip check.  The camera is a TriCam the host builds once per call.  Every product, sum,
// quotient and square root is an explicitly rounded intrinsic in the reference's order -- dot products and norms are sums from
// 0.0 (Math/Vector.h:1593-1604, 1717-1726) -- so nothing is contracted into an FMA and the doubles are the reference's bit for bit.
// The primitives and vector helpers are also the host's (cameras.cu builds and rectifies cameras with them): there each is the
// plain operator, which build.py's -ffp-contract=off keeps the host compiler from contracting.
#pragma once
#include <cfloat>
#include <cmath>

#include "common.cuh"

namespace vwb200 {
namespace {

struct V3 { double x, y, z; };

#ifdef __CUDA_ARCH__
__host__ __device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__host__ __device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__host__ __device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__host__ __device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__host__ __device__ __forceinline__ double dsqrt(double a) { return __dsqrt_rn(a); }
#else
__host__ __device__ __forceinline__ double dadd(double a, double b) { return a + b; }
__host__ __device__ __forceinline__ double dsub(double a, double b) { return a - b; }
__host__ __device__ __forceinline__ double dmul(double a, double b) { return a * b; }
__host__ __device__ __forceinline__ double ddiv(double a, double b) { return a / b; }
__host__ __device__ __forceinline__ double dsqrt(double a) { return std::sqrt(a); }
#endif

__host__ __device__ __forceinline__ V3 ld3(const double* p) { return V3{p[0], p[1], p[2]}; }
__host__ __device__ __forceinline__ V3 sub3(V3 a, V3 b) { return V3{dsub(a.x, b.x), dsub(a.y, b.y), dsub(a.z, b.z)}; }
// dot_prod: a sum from 0.0 (so -0.0 terms give +0.0)
__host__ __device__ __forceinline__ double dot3(V3 a, V3 b) {
  return dadd(dadd(dadd(0.0, dmul(a.x, b.x)), dmul(a.y, b.y)), dmul(a.z, b.z));
}
__host__ __device__ __forceinline__ double norm3(V3 a) { return dsqrt(dot3(a, a)); }
__host__ __device__ __forceinline__ V3 cross3(V3 a, V3 b) {           // Math/Vector.h:1738-1743
  return V3{dsub(dmul(a.y, b.z), dmul(a.z, b.y)), dsub(dmul(a.z, b.x), dmul(a.x, b.z)), dsub(dmul(a.x, b.y), dmul(a.y, b.x))};
}

// TsaiDistortionNorm (LensDistortion.cc:260-276) at (x, y)
__device__ __forceinline__ void tsai_distort(const double* k, double x, double y, double* xo, double* yo) {
  const double k1 = k[0], k2 = k[1], p1 = k[2], p2 = k[3], k3 = k[4];
  const double r2 = dadd(dmul(x, x), dmul(y, y));
  const double rdist = dadd(dadd(dadd(1.0, dmul(k1, r2)), dmul(dmul(k2, r2), r2)), dmul(dmul(dmul(k3, r2), r2), r2));
  *xo = dadd(dmul(x, rdist), dadd(dmul(dmul(dmul(2.0, p1), x), y), dmul(p2, dadd(r2, dmul(dmul(2.0, x), x)))));
  *yo = dadd(dmul(y, rdist), dadd(dmul(p1, dadd(r2, dmul(dmul(2.0, y), y))), dmul(dmul(dmul(2.0, p2), x), y)));
}

// TsaiDistortionJacobian (LensDistortion.cc:286-324) at (x, y): {dfx/dx, dfx/dy, dfy/dx, dfy/dy}
__device__ __forceinline__ void tsai_jacobian(const double* k, double x, double y, double* J) {
  const double k1 = k[0], k2 = k[1], p1 = k[2], p2 = k[3], k3 = k[4];
  const double r2 = dadd(dmul(x, x), dmul(y, y));
  const double dr2dx = dmul(2.0, x), dr2dy = dmul(2.0, y);
  const double rdist = dadd(dadd(dadd(1.0, dmul(k1, r2)), dmul(dmul(k2, r2), r2)), dmul(dmul(dmul(k3, r2), r2), r2));
  // k1 * d + k2 * d * 2.0 * r2 + k3 * d * 3.0 * r2 * r2
  const double ax = dadd(dadd(dmul(k1, dr2dx), dmul(dmul(dmul(k2, dr2dx), 2.0), r2)), dmul(dmul(dmul(dmul(k3, dr2dx), 3.0), r2), r2));
  const double ay = dadd(dadd(dmul(k1, dr2dy), dmul(dmul(dmul(k2, dr2dy), 2.0), r2)), dmul(dmul(dmul(dmul(k3, dr2dy), 3.0), r2), r2));
  J[0] = dadd(dadd(dadd(rdist, dmul(x, ax)), dmul(dmul(2.0, p1), y)), dmul(p2, dadd(dr2dx, dmul(4.0, x))));
  J[1] = dadd(dadd(dmul(x, ay), dmul(dmul(2.0, p1), x)), dmul(p2, dr2dy));
  J[2] = dadd(dmul(y, ax), dadd(dmul(p1, dr2dx), dmul(dmul(2.0, p2), y)));
  J[3] = dadd(dadd(dadd(rdist, dmul(y, ay)), dmul(p1, dadd(dr2dy, dmul(4.0, y)))), dmul(dmul(2.0, p2), x));
}

// TsaiLensDistortion::undistorted_coordinates (LensDistortion.cc:371-400): NewtonRaphson::solve with guess = the normalised
// distorted point, tol 1e-9, at most 19 iterations; *iters counts the iterations run
__device__ __forceinline__ void tsai_undistort(const TriCam& c, double* px, double* py, int* iters) {
  if (c.fu < 1e-300 || c.fv < 1e-300) { *px = *py = HUGE_VAL; return; }
  const double dx = ddiv(dsub(*px, c.cu), c.fu), dy = ddiv(dsub(*py, c.cv), c.fv);
  double X0 = dx, X1 = dy, B0 = dx, B1 = dy, best = DBL_MAX;
  bool done = false;
  for (int count = 1; count < 20; ++count) {
    ++*iters;
    double f0, f1;
    tsai_distort(c.k, X0, X1, &f0, &f1);
    const double F0 = dsub(f0, dx), F1 = dsub(f1, dy);
    const double nf = dsqrt(dadd(dadd(0.0, dmul(F0, F0)), dmul(F1, F1)));
    if (isnan(nf)) break;
    if (nf < best) { best = nf; B0 = X0; B1 = X1; }
    double J[4];
    tsai_jacobian(c.k, X0, X1, J);
    const double det = dsub(dmul(J[0], J[3]), dmul(J[1], J[2]));
    if (fabs(det) < 1e-6 || isnan(det)) break;
    const double D0 = ddiv(dsub(dmul(J[3], F0), dmul(J[1], F1)), det);
    const double D1 = ddiv(dsub(dmul(J[0], F1), dmul(J[2], F0)), det);
    X0 = dsub(X0, D0); X1 = dsub(X1, D1);
    if (dsqrt(dadd(dadd(0.0, dmul(D0, D0)), dmul(D1, D1))) < 1e-9) { done = true; break; }
  }
  const double U0 = done ? X0 : B0, U1 = done ? X1 : B1;
  *px = dadd(dmul(U0, c.fu), c.cu);
  *py = dadd(dmul(U1, c.fv), c.cv);
}

// PinholeModel::pixel_to_vector (PinholeModel.cc:422-430)
template <bool TSAI>
__device__ __forceinline__ V3 pixel_to_vector(const TriCam& c, double u, double v, int* iters) {
  u = dmul(u, c.pitch); v = dmul(v, c.pitch);
  if (TSAI && c.tsai) tsai_undistort(c, &u, &v, iters);
  const V3 p{u, v, 1.0};
  const V3 r{dot3(V3{c.inv[0], c.inv[1], c.inv[2]}, p), dot3(V3{c.inv[3], c.inv[4], c.inv[5]}, p), dot3(V3{c.inv[6], c.inv[7], c.inv[8]}, p)};
  const double n = norm3(r);
  return V3{ddiv(r.x, n), ddiv(r.y, n), ddiv(r.z, n)};
}

// PinholeModel::point_to_pixel (PinholeModel.cc:351-397): the camera matrix row sums left to right, the de-homogenising divide,
// distorted_coordinates (NULL: the identity; TSAI: LensDistortion.cc:345-369), / pixel_pitch, then the check -- the ray back
// through pixel_to_vector against normalize(point - C), retried with their sum.  *ok = false where the reference throws
// PointToPixelErr (the difference still >= 0.01, or NaN).
__device__ __forceinline__ double row4(const double* m, V3 p) { return dadd(dadd(dadd(dmul(m[0], p.x), dmul(m[1], p.y)), dmul(m[2], p.z)), m[3]); }
template <bool TSAI>
__device__ __forceinline__ void point_to_pixel(const TriCam& c, V3 point, double* pu, double* pv, bool* ok, int* iters) {
  const double den = row4(c.P + 8, point);
  double u = ddiv(row4(c.P, point), den), v = ddiv(row4(c.P + 4, point), den);
  if (TSAI && c.tsai) {
    if (c.fu < 1e-300 || c.fv < 1e-300) {
      u = v = HUGE_VAL;
    } else {
      double x, y;
      tsai_distort(c.k, ddiv(dsub(u, c.cu), c.fu), ddiv(dsub(v, c.cv), c.fv), &x, &y);
      u = dadd(dmul(x, c.fu), c.cu);
      v = dadd(dmul(y, c.fv), c.cv);
    }
  }
  u = ddiv(u, c.pitch); v = ddiv(v, c.pitch);
  const V3 pix = pixel_to_vector<TSAI>(c, u, v, iters);
  const V3 d = sub3(point, V3{c.c[0], c.c[1], c.c[2]});
  const double n = norm3(d);
  const V3 phys{ddiv(d.x, n), ddiv(d.y, n), ddiv(d.z, n)};
  double diff = norm3(sub3(pix, phys));
  if (diff >= 0.01) diff = norm3(V3{dadd(pix.x, phys.x), dadd(pix.y, phys.y), dadd(pix.z, phys.z)});
  *ok = !(diff >= 0.01 || diff != diff);
  *pu = u; *pv = v;
}

// CameraTransform::forward / reverse (Camera/CameraTransform.h:52-74): from's pixel_to_vector plus its center, through to's
// point_to_pixel (the centers are equal; the host checks that)
template <bool TSAI>
__device__ __forceinline__ void camera_map(const TriCam& from, const TriCam& to, double x, double y, double* u, double* v, bool* ok, int* iters) {
  const V3 r = pixel_to_vector<TSAI>(from, x, y, iters);
  point_to_pixel<TSAI>(to, V3{dadd(r.x, from.c[0]), dadd(r.y, from.c[1]), dadd(r.z, from.c[2])}, u, v, ok, iters);
}

}  // namespace
}  // namespace vwb200
