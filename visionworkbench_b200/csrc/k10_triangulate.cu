// k10_triangulate.cu -- K10: dense two-camera triangulation of a disparity through pinhole cameras (Stereo/StereoView.h:74-130,
// Stereo/StereoModel.cc:35-147, 254-309, Camera/PinholeModel.cc:422-434, Camera/LensDistortion.cc:258-400,
// Math/NewtonRaphson.cc:58-119), and UniverseRadiusFunc on a Vector3 image (StereoView.h:139-186).
//
// One thread per pixel, grid-stride over rows.  Each warp stages its 32 {x, y, z} results in shared memory and stores them as
// three contiguous 256-byte runs.  The cameras are kernel parameters (TriCam: the inverse camera transform the host builds
// once per call, the center, the pixel pitch and the lens).  Every product, sum, quotient and square root is an explicitly
// rounded intrinsic in the reference's order -- dot products and norms are sums from 0.0 (Math/Vector.h:1593-1604, 1717-1726)
// -- so nothing is contracted into an FMA and the doubles are the reference's bit for bit.
#include <cfloat>

#include "common.cuh"

namespace vwb200 {
namespace {

constexpr int kThreads = 128;                  // pixels of one row per CTA
constexpr int kWarps = kThreads / 32;

struct V3 { double x, y, z; };

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return V3{dsub(a.x, b.x), dsub(a.y, b.y), dsub(a.z, b.z)}; }
// dot_prod: a sum from 0.0 (so -0.0 terms give +0.0)
__device__ __forceinline__ double dot3(V3 a, V3 b) {
  return dadd(dadd(dadd(0.0, dmul(a.x, b.x)), dmul(a.y, b.y)), dmul(a.z, b.z));
}
__device__ __forceinline__ double norm3(V3 a) { return __dsqrt_rn(dot3(a, a)); }
__device__ __forceinline__ V3 cross3(V3 a, V3 b) {           // Math/Vector.h:1738-1743
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
    const double nf = __dsqrt_rn(dadd(dadd(0.0, dmul(F0, F0)), dmul(F1, F1)));
    if (isnan(nf)) break;
    if (nf < best) { best = nf; B0 = X0; B1 = X1; }
    double J[4];
    tsai_jacobian(c.k, X0, X1, J);
    const double det = dsub(dmul(J[0], J[3]), dmul(J[1], J[2]));
    if (fabs(det) < 1e-6 || isnan(det)) break;
    const double D0 = ddiv(dsub(dmul(J[3], F0), dmul(J[1], F1)), det);
    const double D1 = ddiv(dsub(dmul(J[0], F1), dmul(J[2], F0)), det);
    X0 = dsub(X0, D0); X1 = dsub(X1, D1);
    if (__dsqrt_rn(dadd(dadd(0.0, dmul(D0, D0)), dmul(D1, D1))) < 1e-9) { done = true; break; }
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

// StereoModel::operator()(pix1, pix2, errorVec) for two cameras (StereoModel.cc:35-48, 68-91, 97-147)
template <bool TSAI>
__device__ __forceinline__ V3 triangulate(const TriCam& c0, const TriCam& c1, double tol, double l0, double l1, double r0, double r1,
                                          V3* err, int* iters) {
  *err = V3{0.0, 0.0, 0.0};
  const bool ok0 = !(l0 != l0 || l1 != l1) && !(l0 == -1e8 && l1 == -1e8);     // NaN or invalid_pixel(): the ray is skipped
  const bool ok1 = !(r0 != r0 || r1 != r1) && !(r0 == -1e8 && r1 == -1e8);
  if (!ok0 || !ok1) return V3{0.0, 0.0, 0.0};
  const V3 d0 = pixel_to_vector<TSAI>(c0, l0, l1, iters), d1 = pixel_to_vector<TSAI>(c1, r0, r1, iters);
  if (!(dsub(1.0, dot3(d0, d1)) >= tol)) return V3{0.0, 0.0, 0.0};              // nearly parallel (NaN counts as parallel)
  const V3 C0{c0.c[0], c0.c[1], c0.c[2]}, C1{c1.c[0], c1.c[1], c1.c[2]};
  const V3 v12 = cross3(d0, d1), v1 = cross3(v12, d0), v2 = cross3(v12, d1);
  const double s1 = ddiv(dot3(v2, sub3(C1, C0)), dot3(v2, d0));
  const double s2 = ddiv(dot3(v1, sub3(C0, C1)), dot3(v1, d1));
  const V3 p1{dadd(C0.x, dmul(s1, d0.x)), dadd(C0.y, dmul(s1, d0.y)), dadd(C0.z, dmul(s1, d0.z))};
  const V3 p2{dadd(C1.x, dmul(s2, d1.x)), dadd(C1.y, dmul(s2, d1.y)), dadd(C1.z, dmul(s2, d1.z))};
  *err = sub3(p1, p2);
  V3 r{dmul(0.5, dadd(p1.x, p2.x)), dmul(0.5, dadd(p1.y, p2.y)), dmul(0.5, dadd(p1.z, p2.z))};
  if (dot3(sub3(r, C0), d0) < 0 || dot3(sub3(r, C1), d1) < 0)                    // behind a camera: reflect through C0
    r = V3{dadd(-r.x, dmul(2.0, C0.x)), dadd(-r.y, dmul(2.0, C0.y)), dadd(-r.z, dmul(2.0, C0.z))};
  return r;
}

// the 32 {x, y, z} of a warp's consecutive pixels [0, n) to row + 3 * first, as three contiguous runs
__device__ __forceinline__ void store_xyz(double* s, double* row, int n, V3 p) {
  const int lane = threadIdx.x & 31;
  if (lane < n) { s[3 * lane] = p.x; s[3 * lane + 1] = p.y; s[3 * lane + 2] = p.z; }
  __syncwarp();
  for (int k = 0; k < 3; ++k)
    if (k * 32 + lane < 3 * n) row[k * 32 + lane] = s[k * 32 + lane];
  __syncwarp();
}

template <class T> __device__ __forceinline__ float chan(const T& p, int i);
template <> __device__ __forceinline__ float chan<DispF>(const DispF& p, int i) { return i ? p.dy : p.dx; }
template <class T> __device__ __forceinline__ bool valid(const T& p) { return p.valid != 0; }

template <class T> __device__ __forceinline__ double wide(const T& p, int i);
template <> __device__ __forceinline__ double wide<vwb200_dispi>(const vwb200_dispi& p, int i) { return (double)(i ? p.dy : p.dx); }
template <> __device__ __forceinline__ double wide<DispF>(const DispF& p, int i) { return (double)(i ? p.dy : p.dx); }

// stats[0] error sum, [1] max error (bits), [2] points, [3] divergent, [4] Tsai Newton-Raphson iterations
__device__ void flush_stats(unsigned long long* stats, double sum, double mx, unsigned long long pts, unsigned long long div, unsigned long long it) {
  for (int o = 16; o; o >>= 1) {
    sum = dadd(sum, __shfl_xor_sync(0xffffffffu, sum, o));
    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    pts += __shfl_xor_sync(0xffffffffu, pts, o);
    div += __shfl_xor_sync(0xffffffffu, div, o);
    it += __shfl_xor_sync(0xffffffffu, it, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (sum != 0.0) atomicAdd(reinterpret_cast<double*>(stats), sum);
    if (mx > 0.0) atomicMax(stats + 1, (unsigned long long)__double_as_longlong(mx));   // non-negative doubles order as their bits
    if (pts) atomicAdd(stats + 2, pts);
    if (div) atomicAdd(stats + 3, div);
    if (it) atomicAdd(stats + 4, it);
  }
}

// in points at the window's first pixel; (x0, y0) is where the window lies in the disparity.
// MODEL == false: StereoView (form a) over the window (x0, y0, ow, oh): left pixel (i, j), right (i, j) + (double)disparity.
// MODEL == true:  StereoModel::operator()(ImageView<PixelMask<Vector2f>>, error) (form b; x0 = y0 = 0): right pixel
//                 (double)(x + d) summed in float, error = norm_2(errorVec), and the statistics the reference prints.
template <class T, bool MODEL, bool TSAI>
__global__ void __launch_bounds__(kThreads, 4) k10_triangulate_kernel(const T* __restrict__ in, ptrdiff_t ip, int x0, int y0, int ow, int oh,
                                                                   TriCam c0, TriCam c1, double tol, double* __restrict__ xyz, ptrdiff_t xp,
                                                                   double* __restrict__ err, ptrdiff_t ep, unsigned long long* stats) {
  __shared__ double stage[kWarps][96];
  const int first = blockIdx.x * kThreads + (threadIdx.x & ~31);                // the warp's first column
  const int n = min(32, ow - first);
  const int i = blockIdx.x * kThreads + threadIdx.x;
  double sum = 0.0, mx = 0.0;
  unsigned long long pts = 0, div = 0;
  int iters = 0;
  if (n > 0) {
    for (int j = blockIdx.y; j < oh; j += gridDim.y) {
      V3 p{0.0, 0.0, 0.0}, e{0.0, 0.0, 0.0};
      double error = 0.0;
      if (i < ow) {
        const T d = in[(ptrdiff_t)j * ip + i];
        if (valid(d)) {
          const int x = x0 + i, y = y0 + j;
          if constexpr (MODEL) {
            p = triangulate<TSAI>(c0, c1, tol, (double)x, (double)y, (double)__fadd_rn((float)x, chan(d, 0)),
                                  (double)__fadd_rn((float)y, chan(d, 1)), &e, &iters);
            error = norm3(e);
            if (error >= 0) { mx = fmax(mx, error); sum = dadd(sum, error); ++pts; }
            else { p = V3{0.0, 0.0, 0.0}; ++div; }                                 // rays diverged: NaN error
          } else {
            p = triangulate<TSAI>(c0, c1, tol, (double)x, (double)y, dadd((double)x, wide(d, 0)), dadd((double)y, wide(d, 1)), &e, &iters);
          }
        }
        if constexpr (MODEL) err[(ptrdiff_t)j * ep + i] = error;
      }
      store_xyz(stage[threadIdx.x >> 5], xyz + (ptrdiff_t)j * xp * 3 + 3 * (ptrdiff_t)first, n, p);
    }
  }
  if (MODEL || TSAI) flush_stats(stats, sum, mx, pts, div, (unsigned long long)iters);
}

// UniverseRadiusFunc::operator()(Vector3) (StereoView.h:172-186) over a w x h Vector3 image; in may be out (same pitch).
// stats[0] counts the rejected points.
__global__ void __launch_bounds__(kThreads) k10_universe_radius_kernel(const double* in, ptrdiff_t ip, int w, int h, V3 o, double nr,
                                                                       double fr, double* out, ptrdiff_t op, unsigned long long* stats) {
  __shared__ double stage[kWarps][96];
  double* s = stage[threadIdx.x >> 5];
  const int lane = threadIdx.x & 31;
  const int first = blockIdx.x * kThreads + (threadIdx.x & ~31);
  const int n = min(32, w - first);
  unsigned long long rejected = 0;
  if (n > 0) {
    for (int j = blockIdx.y; j < h; j += gridDim.y) {
      const double* src = in + (ptrdiff_t)j * ip * 3 + 3 * (ptrdiff_t)first;
      for (int k = 0; k < 3; ++k)
        if (k * 32 + lane < 3 * n) s[k * 32 + lane] = src[k * 32 + lane];
      __syncwarp();
      V3 p{0.0, 0.0, 0.0};
      if (lane < n) p = V3{s[3 * lane], s[3 * lane + 1], s[3 * lane + 2]};
      __syncwarp();
      if (p.x != 0 || p.y != 0 || p.z != 0) {                                   // pix != Vector3(): -0.0 is zero
        const double dist = norm3(sub3(p, o));
        if ((nr != 0 && dist < nr) || (fr != 0 && dist > fr)) { ++rejected; p = V3{0.0, 0.0, 0.0}; }
      } else {
        p = V3{0.0, 0.0, 0.0};
      }
      store_xyz(s, out + (ptrdiff_t)j * op * 3 + 3 * (ptrdiff_t)first, n, p);
    }
  }
  for (int o2 = 16; o2; o2 >>= 1) rejected += __shfl_xor_sync(0xffffffffu, rejected, o2);
  if (lane == 0 && rejected) atomicAdd(stats, rejected);
}

// columns in CTAs of kThreads, rows grid-strided over about 16 CTAs per SM
dim3 grid_for(int w, int h) {
  const int gx = (w + kThreads - 1) / kThreads;
  const int gy = std::max(1, std::min({h, 65535, (kNumSMs * 16 + gx - 1) / gx}));
  return dim3(gx, gy);
}

}  // namespace

template <class T>
int stereo_triangulate_launch(const T* in, ptrdiff_t ip, int x0, int y0, int ow, int oh, const TriCam& c0, const TriCam& c1, double tol,
                              double* xyz, ptrdiff_t xp, unsigned long long* stats, cudaStream_t st) {
  const dim3 g = grid_for(ow, oh);
  if (c0.tsai || c1.tsai)
    k10_triangulate_kernel<T, false, true><<<g, kThreads, 0, st>>>(in, ip, x0, y0, ow, oh, c0, c1, tol, xyz, xp, nullptr, 0, stats);
  else
    k10_triangulate_kernel<T, false, false><<<g, kThreads, 0, st>>>(in, ip, x0, y0, ow, oh, c0, c1, tol, xyz, xp, nullptr, 0, stats);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}
template int stereo_triangulate_launch<vwb200_dispi>(const vwb200_dispi*, ptrdiff_t, int, int, int, int, const TriCam&, const TriCam&, double,
                                                     double*, ptrdiff_t, unsigned long long*, cudaStream_t);
template int stereo_triangulate_launch<DispF>(const DispF*, ptrdiff_t, int, int, int, int, const TriCam&, const TriCam&, double, double*,
                                              ptrdiff_t, unsigned long long*, cudaStream_t);

int stereo_model_launch(const DispF* in, int w, int h, ptrdiff_t ip, const TriCam& c0, const TriCam& c1, double tol, double* xyz, ptrdiff_t xp,
                        double* err, ptrdiff_t ep, unsigned long long* stats, cudaStream_t st) {
  const dim3 g = grid_for(w, h);
  if (c0.tsai || c1.tsai)
    k10_triangulate_kernel<DispF, true, true><<<g, kThreads, 0, st>>>(in, ip, 0, 0, w, h, c0, c1, tol, xyz, xp, err, ep, stats);
  else
    k10_triangulate_kernel<DispF, true, false><<<g, kThreads, 0, st>>>(in, ip, 0, 0, w, h, c0, c1, tol, xyz, xp, err, ep, stats);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

int universe_radius_launch(const double* in, int w, int h, ptrdiff_t ip, const double* origin, double near_r, double far_r, double* out,
                           ptrdiff_t op, unsigned long long* rejected, cudaStream_t st) {
  k10_universe_radius_kernel<<<grid_for(w, h), kThreads, 0, st>>>(in, ip, w, h, V3{origin[0], origin[1], origin[2]}, near_r, far_r, out, op,
                                                                 rejected);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

}  // namespace vwb200
