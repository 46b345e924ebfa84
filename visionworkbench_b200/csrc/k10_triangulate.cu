// k10_triangulate.cu -- K10: dense two-camera triangulation of a disparity through pinhole or CAHV / CAHVOR cameras
// (Stereo/StereoView.h:74-130, Stereo/StereoModel.cc:35-147, 254-309, Camera/PinholeModel.cc:422-434,
// Camera/LensDistortion.cc:258-400, Math/NewtonRaphson.cc:58-119), and UniverseRadiusFunc on a Vector3 image (StereoView.h:139-186).
//
// One thread per pixel, grid-stride over rows.  Each warp stages its 32 {x, y, z} results in shared memory and stores them as
// three contiguous 256-byte runs.  The cameras are kernel parameters: a TriCam (the inverse camera transform the host builds
// once per call, the center, the pixel pitch and the lens) with pinhole.cuh's camera math, or a CahvCam with cahv.cuh's, both
// bit for bit the reference's.
#include "cahv.cuh"

namespace vwb200 {
namespace {

constexpr int kThreads = 128;                  // pixels of one row per CTA
constexpr int kWarps = kThreads / 32;

// the rays' part of StereoModel::operator()(pix1, pix2, errorVec) (StereoModel.cc:35-48, 68-91, 97-147): the nearly-parallel
// test, triangulate_pair and the reflection through C0; *err is zero on entry
__device__ __forceinline__ V3 intersect(const V3 C0, const V3 C1, const V3 d0, const V3 d1, double tol, V3* err) {
  if (!(dsub(1.0, dot3(d0, d1)) >= tol)) return V3{0.0, 0.0, 0.0};              // nearly parallel (NaN counts as parallel)
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

// each family's camera_center and pixel_to_vector: a pinhole camera's through pinhole.cuh (ITER: the Tsai Newton-Raphson may run),
// a CAHV / CAHVOR camera's through cahv.cuh (ITER: the CAHVOR Newton loop may run); *iters counts the iterations
__device__ __forceinline__ V3 center(const TriCam& c) { return V3{c.c[0], c.c[1], c.c[2]}; }
__device__ __forceinline__ V3 center(const CahvCam& c) { return ld3(c.C); }
template <bool ITER>
__device__ __forceinline__ V3 ray(const TriCam& c, double u, double v, int* iters) { return pixel_to_vector<ITER>(c, u, v, iters); }
template <bool ITER>
__device__ __forceinline__ V3 ray(const CahvCam& c, double u, double v, int* iters) { return cahv_pixel_to_vector<ITER>(c, u, v, iters); }

// StereoModel::operator()(pix1, pix2, errorVec) for two cameras of one family (StereoModel.cc:121-122 takes any camera's
// pixel_to_vector and camera_center)
template <bool ITER, class Cam>
__device__ __forceinline__ V3 triangulate(const Cam& c0, const Cam& c1, double tol, double l0, double l1, double r0, double r1, V3* err,
                                          int* iters) {
  *err = V3{0.0, 0.0, 0.0};
  const bool ok0 = !(l0 != l0 || l1 != l1) && !(l0 == -1e8 && l1 == -1e8);     // NaN or invalid_pixel(): the ray is skipped
  const bool ok1 = !(r0 != r0 || r1 != r1) && !(r0 == -1e8 && r1 == -1e8);
  if (!ok0 || !ok1) return V3{0.0, 0.0, 0.0};
  const V3 d0 = ray<ITER>(c0, l0, l1, iters), d1 = ray<ITER>(c1, r0, r1, iters);
  return intersect(center(c0), center(c1), d0, d1, tol, err);
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

// stats[0] error sum, [1] max error (bits), [2] points, [3] divergent, [4] Newton iterations
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
// ITER == false compiles the rays without their Newton iterations (kernel_for picks it per call).
template <class Cam, class T, bool MODEL, bool ITER>
__global__ void __launch_bounds__(kThreads, 4) k10_triangulate_kernel(const T* __restrict__ in, ptrdiff_t ip, int x0, int y0, int ow, int oh,
                                                                   Cam c0, Cam c1, double tol, double* __restrict__ xyz, ptrdiff_t xp,
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
            p = triangulate<ITER>(c0, c1, tol, (double)x, (double)y, (double)__fadd_rn((float)x, chan(d, 0)),
                                  (double)__fadd_rn((float)y, chan(d, 1)), &e, &iters);
            error = norm3(e);
            if (error >= 0) { mx = fmax(mx, error); sum = dadd(sum, error); ++pts; }
            else { p = V3{0.0, 0.0, 0.0}; ++div; }                                 // rays diverged: NaN error
          } else {
            p = triangulate<ITER>(c0, c1, tol, (double)x, (double)y, dadd((double)x, wide(d, 0)), dadd((double)y, wide(d, 1)), &e, &iters);
          }
        }
        if constexpr (MODEL) err[(ptrdiff_t)j * ep + i] = error;
      }
      store_xyz(stage[threadIdx.x >> 5], xyz + (ptrdiff_t)j * xp * 3 + 3 * (ptrdiff_t)first, n, p);
    }
  }
  if (MODEL || ITER) flush_stats(stats, sum, mx, pts, div, (unsigned long long)iters);
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

// the kernel for a camera pair: a pinhole pair's iterates when either camera has the Tsai lens, a CAHV pair's always (whether
// a camera is CAHVOR is a runtime flag)
template <class T, bool MODEL>
auto kernel_for(const TriCam& c0, const TriCam& c1) {
  return c0.tsai || c1.tsai ? k10_triangulate_kernel<TriCam, T, MODEL, true> : k10_triangulate_kernel<TriCam, T, MODEL, false>;
}
template <class T, bool MODEL>
auto kernel_for(const CahvCam&, const CahvCam&) { return k10_triangulate_kernel<CahvCam, T, MODEL, true>; }

}  // namespace

template <class Cam, class T>
int stereo_triangulate_launch(const T* in, ptrdiff_t ip, int x0, int y0, int ow, int oh, const Cam& c0, const Cam& c1, double tol,
                              double* xyz, ptrdiff_t xp, unsigned long long* stats, cudaStream_t st) {
  kernel_for<T, false>(c0, c1)<<<grid_for(ow, oh), kThreads, 0, st>>>(in, ip, x0, y0, ow, oh, c0, c1, tol, xyz, xp, nullptr, 0, stats);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}
template int stereo_triangulate_launch<TriCam, vwb200_dispi>(const vwb200_dispi*, ptrdiff_t, int, int, int, int, const TriCam&, const TriCam&,
                                                             double, double*, ptrdiff_t, unsigned long long*, cudaStream_t);
template int stereo_triangulate_launch<TriCam, DispF>(const DispF*, ptrdiff_t, int, int, int, int, const TriCam&, const TriCam&, double, double*,
                                                      ptrdiff_t, unsigned long long*, cudaStream_t);
template int stereo_triangulate_launch<CahvCam, vwb200_dispi>(const vwb200_dispi*, ptrdiff_t, int, int, int, int, const CahvCam&, const CahvCam&,
                                                              double, double*, ptrdiff_t, unsigned long long*, cudaStream_t);
template int stereo_triangulate_launch<CahvCam, DispF>(const DispF*, ptrdiff_t, int, int, int, int, const CahvCam&, const CahvCam&, double,
                                                       double*, ptrdiff_t, unsigned long long*, cudaStream_t);

template <class Cam>
int stereo_model_launch(const DispF* in, int w, int h, ptrdiff_t ip, const Cam& c0, const Cam& c1, double tol, double* xyz, ptrdiff_t xp,
                        double* err, ptrdiff_t ep, unsigned long long* stats, cudaStream_t st) {
  kernel_for<DispF, true>(c0, c1)<<<grid_for(w, h), kThreads, 0, st>>>(in, ip, 0, 0, w, h, c0, c1, tol, xyz, xp, err, ep, stats);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}
template int stereo_model_launch<TriCam>(const DispF*, int, int, ptrdiff_t, const TriCam&, const TriCam&, double, double*, ptrdiff_t, double*,
                                         ptrdiff_t, unsigned long long*, cudaStream_t);
template int stereo_model_launch<CahvCam>(const DispF*, int, int, ptrdiff_t, const CahvCam&, const CahvCam&, double, double*, ptrdiff_t, double*,
                                          ptrdiff_t, unsigned long long*, cudaStream_t);

int universe_radius_launch(const double* in, int w, int h, ptrdiff_t ip, const double* origin, double near_r, double far_r, double* out,
                           ptrdiff_t op, unsigned long long* rejected, cudaStream_t st) {
  k10_universe_radius_kernel<<<grid_for(w, h), kThreads, 0, st>>>(in, ip, w, h, V3{origin[0], origin[1], origin[2]}, near_r, far_r, out, op,
                                                                 rejected);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

}  // namespace vwb200
