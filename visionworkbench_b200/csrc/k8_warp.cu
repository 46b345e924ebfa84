// k8_warp.cu -- K8: transform(image, tx, edge, interp) of Image/Transform.h:485-601 on single-channel float images
// (PixelGray<float>), rasterised over an output window.  tx is HomographyTransform (Math/Transform.h:369-389, `reverse`
// applies the matrix given here) or DisparityTransform (Stereo/DisparityMap.h:1164-1187); interp is Bilinear, Bicubic or
// NearestPixel (Image/Interpolation.h:75-225); edge is Zero or Constant (Image/EdgeExtension.tcc:47-61, 89-94).
// Transform() has a zero tolerance, so TransformView::rasterize never builds an ApproximateTransform grid: every output pixel
// is a function of its own coordinates.  Each step is an explicitly rounded intrinsic in the reference's order (no
// contraction), so the results are bit for bit those of the reference built with -ffp-contract=off.
#include "common.cuh"

namespace vwb200 {
namespace {

constexpr int kMaxGridY = 65535;                       // the row tiles of taller windows are dealt to the blocks grid-stride
constexpr int kTW = 32, kTH = 8;
// the reversed coordinates the contract covers: beyond them the reference converts out of int32 range (undefined)
constexpr double kDomain = 1073741824.0;               // 2^30

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
    } else {
      // DisparityTransform::reverse: the offset read with nearest-pixel interpolation and zero extension at the integer p
      const int ix = a.x0 + ox;
      rx = -1.0; ry = py;
      if (ix >= 0 && iy >= 0 && ix < a.dw && iy < a.dh) {
        const float* d = reinterpret_cast<const float*>(a.disp + (ptrdiff_t)iy * a.dp + ix);
        if (__ldg(d + 2) != 0.0f) { rx = __dadd_rn(px, (double)__ldg(d)); ry = __dadd_rn(py, (double)__ldg(d + 1)); }
      }
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

}  // namespace

int warp_launch(const vwb200_warp_params& p, const float* in, int w, int h, ptrdiff_t ip, const DispF* disp, int dw, int dh, ptrdiff_t dp,
                int x0, int y0, float* out, int ow, int oh, ptrdiff_t op, cudaStream_t st) {
  if (ow <= 0 || oh <= 0) return VWB200_OK;
  WarpArgs a{in, w, h, ip, disp, dw, dh, dp, {}, x0, y0, out, ow, oh, op};
  for (int i = 0; i < 9; ++i) a.m[i] = p.matrix[i];
  if (p.kind == VWB200_WARP_HOMOGRAPHY) return launch_interp<VWB200_WARP_HOMOGRAPHY>(p.interp, p.edge, a, st);
  return launch_interp<VWB200_WARP_DISPARITY>(p.interp, p.edge, a, st);
}

}  // namespace vwb200
