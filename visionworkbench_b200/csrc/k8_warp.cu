// k8_warp.cu -- K8: transform(image, tx, edge, interp) of Image/Transform.h:485-601 on single-channel float images
// (PixelGray<float>), rasterised over an output window.  tx is HomographyTransform (Math/Transform.h:369-389, `reverse`
// applies the matrix given here) or DisparityTransform (Stereo/DisparityMap.h:1164-1187); interp is Bilinear, Bicubic or
// NearestPixel (Image/Interpolation.h:75-225); edge is Zero or Constant (Image/EdgeExtension.tcc:47-61, 89-94).
// Transform() has a zero tolerance, so TransformView::rasterize never builds an ApproximateTransform grid: every output pixel
// is a function of its own coordinates.  Each step is an explicitly rounded intrinsic in the reference's order (no
// contraction), so the results are bit for bit those of the reference built with -ffp-contract=off.
// The internal kinds kCamera (float pixels) and kCameraMasked (PixelMask<float>, bilinear) are CameraTransform(src, dst)
// (Camera/CameraTransform.h:52-61) between pinhole cameras, through pinhole.cuh: reverse(p) = src.point_to_pixel(
// dst.pixel_to_vector(p) + C), with point_to_pixel's check.  k8_camera_bbox_kernel is the bbox pass of
// resize_epipolar_cameras_to_fit through the same cameras.  The internal kinds kCahv and kCahvMasked are the same transform
// from a CAHV or CAHVOR src into a CAHV dst, through cahv.cuh (the src model is a runtime branch on its flag; the dst is CAHV
// at compile time, so the CAHVOR Newton loop is not compiled in; the CAHV family has no point_to_pixel check).
#include <type_traits>
#include "cahv.cuh"

namespace vwb200 {
namespace {

constexpr int kMaxGridY = 65535;                       // the row tiles of taller windows are dealt to the blocks grid-stride
constexpr int kTW = 32, kTH = 8;
// the reversed coordinates the contract covers: beyond them the reference converts out of int32 range (undefined)
constexpr double kDomain = 1073741824.0;               // 2^30
constexpr int kCamera = 2;                             // beside VWB200_WARP_HOMOGRAPHY and VWB200_WARP_DISPARITY
constexpr int kCameraMasked = 3;                       // kCamera over PixelMask<float> {value, valid} pixels
constexpr int kCahv = 4;                               // kCamera through CAHV / CAHVOR cameras
constexpr int kCahvMasked = 5;                         // kCameraMasked through CAHV / CAHVOR cameras

// math::impl::_floor and _round for double -> int32 (Math/Functions.h:48-51, 74-81)
__device__ __forceinline__ int vw_floor(double v) {
  if (v < 0) {
    const int iv = __double2int_rz(v);
    return (double)iv == v ? iv : iv - 1;
  }
  return __double2int_rz(v);
}
__device__ __forceinline__ int vw_round(double v) { return v < 0 ? __double2int_rz(__dsub_rn(v, 0.5)) : __double2int_rz(__dadd_rn(v, 0.5)); }

template <int Edge>
__device__ __forceinline__ float pixel(const float* __restrict__ in, int w, int h, ptrdiff_t ip, int i, int j) {
  if (Edge == VWB200_EDGE_ZERO) {
    if (i >= 0 && j >= 0 && i < w && j < h) return __ldg(in + (ptrdiff_t)j * ip + i);
    return 0.0f;
  }
  i = i < 0 ? 0 : (i >= w ? w - 1 : i);
  j = j < 0 ? 0 : (j >= h ? h - 1 : j);
  return __ldg(in + (ptrdiff_t)j * ip + i);
}

// BilinearInterpolationImpl (:76-110) with real_type float
template <int Edge>
__device__ __forceinline__ float bilinear(const float* __restrict__ in, int w, int h, ptrdiff_t ip, double i, double j) {
  const int x = vw_floor(i), y = vw_floor(j);
  if ((double)x == i && (double)y == j) return pixel<Edge>(in, w, h, ip, x, y);
  const float nx = __fsub_rn(__double2float_rn(i), __int2float_rn(x)), ny = __fsub_rn(__double2float_rn(j), __int2float_rn(y));
  const float n1mx = __fsub_rn(1.0f, nx), n1my = __fsub_rn(1.0f, ny);
  float r = __fmul_rn(pixel<Edge>(in, w, h, ip, x, y), n1mx);
  r = __fadd_rn(r, __fmul_rn(pixel<Edge>(in, w, h, ip, x + 1, y), nx));
  r = __fmul_rn(r, n1my);
  float row = __fmul_rn(pixel<Edge>(in, w, h, ip, x, y + 1), n1mx);
  row = __fadd_rn(row, __fmul_rn(pixel<Edge>(in, w, h, ip, x + 1, y + 1), nx));
  return __fadd_rn(r, __fmul_rn(row, ny));
}

// PixelMask<float> {value, valid} pixels (pitches in pixels).  Zero extension is PixelMask<float>() = {0, 0} (Image/PixelMask.h:59-62),
// value extension the edge pixel as given (Image/EdgeExtension.h:66-76)
struct Px2 { float v, valid; };
template <int Edge>
__device__ __forceinline__ Px2 pixel2(const float* __restrict__ in, int w, int h, ptrdiff_t ip, float2 ev, int i, int j) {
  if (Edge != VWB200_EDGE_CONSTANT) {
    if (i >= 0 && j >= 0 && i < w && j < h) {
      const float* q = in + 2 * ((ptrdiff_t)j * ip + i);
      return Px2{__ldg(q), __ldg(q + 1)};
    }
    return Edge == VWB200_EDGE_ZERO ? Px2{0.0f, 0.0f} : Px2{ev.x, ev.y};
  }
  i = i < 0 ? 0 : (i >= w ? w - 1 : i);
  j = j < 0 ? 0 : (j >= h ? h - 1 : j);
  const float* q = in + 2 * ((ptrdiff_t)j * ip + i);
  return Px2{__ldg(q), __ldg(q + 1)};
}
// BilinearInterpolationImpl on PixelMask<float> (Image/PixelMask.h:321-380, 499-626): pixel * scalar and channel_cast give
// valid = (valid != 0) as 1.0f / 0.0f (NaN counts as valid), += ANDs the validity, *= scalar keeps it.  So the integral
// shortcut returns {value, valid != 0}, and the interpolated value is the float one's with valid = all four neighbours' valid != 0.
template <int Edge>
__device__ __forceinline__ Px2 bilinear2(const float* __restrict__ in, int w, int h, ptrdiff_t ip, float2 ev, double i, double j) {
  const int x = vw_floor(i), y = vw_floor(j);
  if ((double)x == i && (double)y == j) {
    const Px2 p = pixel2<Edge>(in, w, h, ip, ev, x, y);
    return Px2{p.v, p.valid != 0.0f ? 1.0f : 0.0f};
  }
  const float nx = __fsub_rn(__double2float_rn(i), __int2float_rn(x)), ny = __fsub_rn(__double2float_rn(j), __int2float_rn(y));
  const float n1mx = __fsub_rn(1.0f, nx), n1my = __fsub_rn(1.0f, ny);
  const Px2 p00 = pixel2<Edge>(in, w, h, ip, ev, x, y), p10 = pixel2<Edge>(in, w, h, ip, ev, x + 1, y);
  const Px2 p01 = pixel2<Edge>(in, w, h, ip, ev, x, y + 1), p11 = pixel2<Edge>(in, w, h, ip, ev, x + 1, y + 1);
  float r = __fmul_rn(p00.v, n1mx);
  r = __fadd_rn(r, __fmul_rn(p10.v, nx));
  r = __fmul_rn(r, n1my);
  float row = __fmul_rn(p01.v, n1mx);
  row = __fadd_rn(row, __fmul_rn(p11.v, nx));
  const bool ok = p00.valid != 0.0f && p10.valid != 0.0f && p01.valid != 0.0f && p11.valid != 0.0f;
  return Px2{__fadd_rn(r, __fmul_rn(row, ny)), ok ? 1.0f : 0.0f};
}

// BicubicInterpolationImpl (:138-186) in double
__device__ __forceinline__ void cubic_weights(double n, double& w0, double& w1, double& w2, double& w3) {
  w0 = __dmul_rn(__dsub_rn(__dmul_rn(__dsub_rn(2.0, n), n), 1.0), n);                      // ((2-n)*n-1)*n
  w1 = __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(3.0, n), 5.0), n), n), 2.0);     // (3*n-5)*n*n+2
  w2 = __dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(4.0, __dmul_rn(3.0, n)), n), 1.0), n);     // ((4-3*n)*n+1)*n
  w3 = __dmul_rn(__dmul_rn(__dsub_rn(n, 1.0), n), n);                                      // (n-1)*n*n
}
template <int Edge>
__device__ __forceinline__ float bicubic(const float* __restrict__ in, int w, int h, ptrdiff_t ip, double i, double j) {
  const int x = vw_floor(i), y = vw_floor(j);
  if ((double)x == i && (double)y == j) return pixel<Edge>(in, w, h, ip, x, y);
  double s0, s1, s2, s3, t0, t1, t2, t3;
  cubic_weights(__dsub_rn(i, (double)x), s0, s1, s2, s3);
  cubic_weights(__dsub_rn(j, (double)y), t0, t1, t2, t3);
  const double t[4] = {t0, t1, t2, t3};
  double result = 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int yy = y - 1 + k;
    double row = __dmul_rn(s0, (double)pixel<Edge>(in, w, h, ip, x - 1, yy));
    row = __dadd_rn(row, __dmul_rn(s1, (double)pixel<Edge>(in, w, h, ip, x, yy)));
    row = __dadd_rn(row, __dmul_rn(s2, (double)pixel<Edge>(in, w, h, ip, x + 1, yy)));
    row = __dadd_rn(row, __dmul_rn(s3, (double)pixel<Edge>(in, w, h, ip, x + 2, yy)));
    result = k ? __dadd_rn(result, __dmul_rn(t[k], row)) : __dmul_rn(t[k], row);
  }
  return __double2float_rn(__dmul_rn(result, 0.25));
}

struct WarpArgs {
  const float* in; int w, h; ptrdiff_t ip;
  const DispF* disp; int dw, dh; ptrdiff_t dp;
  double m[9];
  int x0, y0;
  float* out; int ow, oh; ptrdiff_t op;
  TriCam src, dst;                                     // kCamera only (appended: the other kinds' parameters keep their offsets)
  unsigned long long* fail;                            // kCamera: {any check failed, first failing row-major window index}
  float2 ev;                                           // kCameraMasked, kCahvMasked: the VWB200_EDGE_VALUE pixel {value, valid}
  CahvCam csrc, cdst;                                  // kCahv, kCahvMasked only (appended, as src and dst were)
};

// one thread per output pixel of a 32 x 8 tile; window pixel (ox, oy) is TransformView pixel (x0 + ox, y0 + oy)
template <int Kind, int Interp, int Edge>
__global__ void __launch_bounds__(kTW * kTH) k8_warp_kernel(const WarpArgs a) {
  const int ox = blockIdx.x * kTW + threadIdx.x;
  if (ox >= a.ow) return;
  const double px = (double)(a.x0 + ox);
  for (int oy = blockIdx.y * kTH + threadIdx.y; oy < a.oh; oy += gridDim.y * kTH) {
    const int iy = a.y0 + oy;
    const double py = (double)iy;
    double rx, ry;
    if (Kind == VWB200_WARP_HOMOGRAPHY) {
      // HomographyTransform::reverse (Math/Transform.h:377-381)
      const double w = __dadd_rn(__dadd_rn(__dmul_rn(a.m[6], px), __dmul_rn(a.m[7], py)), a.m[8]);
      rx = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(a.m[0], px), __dmul_rn(a.m[1], py)), a.m[2]), w);
      ry = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(a.m[3], px), __dmul_rn(a.m[4], py)), a.m[5]), w);
    } else if (Kind == kCamera || Kind == kCameraMasked) {
      bool ok;
      int iters = 0;
      camera_map<true>(a.dst, a.src, px, py, &rx, &ry, &ok, &iters);
      if (!ok) {                                       // the reference throws PointToPixelErr: flag it, keep the first pixel
        a.fail[0] = 1;
        atomicMin(a.fail + 1, (unsigned long long)oy * a.ow + ox);
      }
    } else if (Kind == kCahv || Kind == kCahvMasked) {
      cahv_camera_map(a.cdst, a.csrc, px, py, &rx, &ry);
    } else {
      // DisparityTransform::reverse: the offset read with nearest-pixel interpolation and zero extension at the integer p
      const int ix = a.x0 + ox;
      rx = -1.0; ry = py;
      if (ix >= 0 && iy >= 0 && ix < a.dw && iy < a.dh) {
        const float* d = reinterpret_cast<const float*>(a.disp + (ptrdiff_t)iy * a.dp + ix);
        if (__ldg(d + 2) != 0.0f) { rx = __dadd_rn(px, (double)__ldg(d)); ry = __dadd_rn(py, (double)__ldg(d + 1)); }
      }
    }
    if (Kind == kCameraMasked || Kind == kCahvMasked) {
      Px2 v{0.0f, 0.0f};                               // outside the domain: {0, 0}
      if (fabs(rx) < kDomain && fabs(ry) < kDomain) v = bilinear2<Edge>(a.in, a.w, a.h, a.ip, a.ev, rx, ry);
      float* q = a.out + 2 * ((ptrdiff_t)oy * a.op + ox);
      q[0] = v.v;
      q[1] = v.valid;
      continue;
    }
    float v = 0.0f;                                    // outside the domain (and NaN / inf): 0.0f
    if (fabs(rx) < kDomain && fabs(ry) < kDomain) {
      if (Interp == VWB200_INTERP_BILINEAR) v = bilinear<Edge>(a.in, a.w, a.h, a.ip, rx, ry);
      else if (Interp == VWB200_INTERP_BICUBIC) v = bicubic<Edge>(a.in, a.w, a.h, a.ip, rx, ry);
      else v = pixel<Edge>(a.in, a.w, a.h, a.ip, vw_round(rx), vw_round(ry));
    }
    a.out[(ptrdiff_t)oy * a.op + ox] = v;
  }
}

template <int Kind, int Interp, int Edge>
int launch(const WarpArgs& a, cudaStream_t st) {
  const dim3 grid((a.ow + kTW - 1) / kTW, std::min((a.oh + kTH - 1) / kTH, kMaxGridY));
  k8_warp_kernel<Kind, Interp, Edge><<<grid, dim3(kTW, kTH), 0, st>>>(a);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}
template <int Kind, int Interp>
int launch_edge(int edge, const WarpArgs& a, cudaStream_t st) {
  return edge == VWB200_EDGE_ZERO ? launch<Kind, Interp, VWB200_EDGE_ZERO>(a, st) : launch<Kind, Interp, VWB200_EDGE_CONSTANT>(a, st);
}
template <int Kind>
int launch_interp(int interp, int edge, const WarpArgs& a, cudaStream_t st) {
  if (interp == VWB200_INTERP_BILINEAR) return launch_edge<Kind, VWB200_INTERP_BILINEAR>(edge, a, st);
  if (interp == VWB200_INTERP_BICUBIC) return launch_edge<Kind, VWB200_INTERP_BICUBIC>(edge, a, st);
  return launch_edge<Kind, VWB200_INTERP_NEAREST>(edge, a, st);
}

// perimeter point k of compute_transformed_bbox_fast's four loops (top, bottom, left, right edges) through forward(), grown
// into a BBox2f: NaN coordinates compare false and are skipped, the others enter as float(c), so the bounds are the float
// order statistics whatever the order (a bound that rounds to zero may carry the other sign of zero)
__global__ void __launch_bounds__(128) k8_camera_bbox_kernel(const TriCam src, const TriCam dst, int x0, int y0, int x1, int y1,
                                                             unsigned* keys, unsigned long long* fail) {
  const long long cw = (long long)x1 - x0, ch = (long long)y1 - y0;
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= 2 * (cw + ch)) return;
  double px, py;
  if (k < cw) { px = (double)(x0 + k); py = (double)y0; }
  else if (k < 2 * cw) { px = (double)(x0 + (k - cw)); py = (double)(y1 - 1); }
  else if (k < 2 * cw + ch) { px = (double)x0; py = (double)(y0 + (k - 2 * cw)); }
  else { px = (double)(x1 - 1); py = (double)(y0 + (k - 2 * cw - ch)); }
  double u, v;
  bool ok;
  int iters = 0;
  camera_map<true>(src, dst, px, py, &u, &v, &ok, &iters);
  if (!ok) { fail[0] = 1; atomicMin(fail + 1, (unsigned long long)k); return; }
  if (u == u) { atomicMin(keys, fkey(__double2float_rn(u))); atomicMax(keys + 2, fkey(__double2float_rn(u))); }
  if (v == v) { atomicMin(keys + 1, fkey(__double2float_rn(v))); atomicMax(keys + 3, fkey(__double2float_rn(v))); }
}

}  // namespace

template <class Cam>
int camera_warp_launch(int masked, int interp, int edge, const float* edge_value, const Cam& src, const Cam& dst, const float* in, int w, int h,
                       ptrdiff_t ip, int x0, int y0, float* out, int ow, int oh, ptrdiff_t op, unsigned long long* fail, cudaStream_t st) {
  if (ow <= 0 || oh <= 0) return VWB200_OK;
  WarpArgs a{in, w, h, ip, nullptr, 0, 0, 0, {}, x0, y0, out, ow, oh, op, {}, {}, fail, make_float2(edge_value[0], edge_value[1])};
  constexpr bool cahv = std::is_same<Cam, CahvCam>::value;
  if constexpr (cahv) { a.csrc = src; a.cdst = dst; } else { a.src = src; a.dst = dst; }
  constexpr int kind = cahv ? kCahv : kCamera, masked_kind = cahv ? kCahvMasked : kCameraMasked;
  if (!masked) return launch_interp<kind>(interp, edge, a, st);
  if (edge == VWB200_EDGE_ZERO) return launch<masked_kind, VWB200_INTERP_BILINEAR, VWB200_EDGE_ZERO>(a, st);
  if (edge == VWB200_EDGE_CONSTANT) return launch<masked_kind, VWB200_INTERP_BILINEAR, VWB200_EDGE_CONSTANT>(a, st);
  return launch<masked_kind, VWB200_INTERP_BILINEAR, VWB200_EDGE_VALUE>(a, st);
}
template int camera_warp_launch<TriCam>(int, int, int, const float*, const TriCam&, const TriCam&, const float*, int, int, ptrdiff_t, int, int,
                                        float*, int, int, ptrdiff_t, unsigned long long*, cudaStream_t);
template int camera_warp_launch<CahvCam>(int, int, int, const float*, const CahvCam&, const CahvCam&, const float*, int, int, ptrdiff_t, int, int,
                                         float*, int, int, ptrdiff_t, unsigned long long*, cudaStream_t);

int camera_bbox_launch(const TriCam& src, const TriCam& dst, int x0, int y0, int x1, int y1, unsigned* keys4, unsigned long long* fail,
                       cudaStream_t st) {
  const long long n = 2 * ((long long)x1 - x0 + (long long)y1 - y0);
  if (n <= 0) return VWB200_OK;
  k8_camera_bbox_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(src, dst, x0, y0, x1, y1, keys4, fail);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

int warp_launch(const vwb200_warp_params& p, const float* in, int w, int h, ptrdiff_t ip, const DispF* disp, int dw, int dh, ptrdiff_t dp,
                int x0, int y0, float* out, int ow, int oh, ptrdiff_t op, cudaStream_t st) {
  if (ow <= 0 || oh <= 0) return VWB200_OK;
  WarpArgs a{in, w, h, ip, disp, dw, dh, dp, {}, x0, y0, out, ow, oh, op, {}, {}, nullptr, {}, {}, {}};
  for (int i = 0; i < 9; ++i) a.m[i] = p.matrix[i];
  if (p.kind == VWB200_WARP_HOMOGRAPHY) return launch_interp<VWB200_WARP_HOMOGRAPHY>(p.interp, p.edge, a, st);
  return launch_interp<VWB200_WARP_DISPARITY>(p.interp, p.edge, a, st);
}

}  // namespace vwb200
