// k7_dispmap.cu -- K7: the resampling, range and transform operations of Stereo/DisparityMap.h on integer ({int32 x3},
// vwb200_dispi) or float ({float x3}, DispF) disparity pixels:
//   disparity_subsample (:1251-1322), disparity_upsample (:1324-1358), get_disparity_range (:48-66),
//   disparity_range_mask (:255-300), transform_disparities (lazy :1016-1057, explicit :1190-1224).
// Every double step is an explicitly rounded intrinsic, in the reference's order (no contraction), so the results are bit
// for bit those of the reference built with -ffp-contract=off.  Created pixels get valid = 1; pixels the reference passes
// through are copied unchanged.
#include "common.cuh"
#include <type_traits>

namespace vwb200 {
namespace {

// the channel arithmetic the two pixel types need
template <class T> struct Px;
template <> struct Px<vwb200_dispi> {
  typedef int32_t C;
  typedef long long Acc;                                  // AccumulatorType<int32> (Core/FundamentalTypes.h:111-122)
  static __device__ __forceinline__ bool valid(const vwb200_dispi& p) { return p.valid != 0; }
  static __device__ __forceinline__ vwb200_dispi make(C x, C y, bool v) { return vwb200_dispi{x, y, v ? 1 : 0}; }
  // C++'s truncating conversion; a NaN or out-of-range value gives INT32_MIN, as x86-64's cvttsd2si does (C++ leaves it undefined)
  static __device__ __forceinline__ C from_double(double d) {
    return (d > -2147483649.0 && d < 2147483648.0) ? __double2int_rz(d) : INT32_MIN;
  }
  static __device__ __forceinline__ C mul(int k, C v) { return (C)((uint32_t)k * (uint32_t)v); }   // int32 product, wrapping
  static __device__ __forceinline__ float to_float(C v) { return __int2float_rn(v); }
  static __device__ __forceinline__ uint32_t key(C v) { return (uint32_t)v ^ 0x80000000u; }
  static __device__ __forceinline__ bool isnan_(C) { return false; }
};
template <> struct Px<DispF> {
  typedef float C;
  typedef double Acc;                                     // AccumulatorType<float>
  static __device__ __forceinline__ bool valid(const DispF& p) { return p.valid != 0.0f; }
  static __device__ __forceinline__ DispF make(C x, C y, bool v) { return DispF{x, y, v ? 1.0f : 0.0f}; }
  static __device__ __forceinline__ C from_double(double d) { return __double2float_rn(d); }
  static __device__ __forceinline__ C mul(int k, C v) { return __fmul_rn((float)k, v); }
  static __device__ __forceinline__ float to_float(C v) { return v; }
  // -0.0 and +0.0 compare equal: they share a key, and the raster index breaks the tie
  static __device__ __forceinline__ uint32_t key(C v) { return fkey(v == 0.0f ? 0.0f : v); }
  static __device__ __forceinline__ bool isnan_(C v) { return v != v; }
};

// buffer += k * bff_type(p): the term cast to the accumulator before the multiply
__device__ __forceinline__ void acc_cast(long long& b, int k, int32_t v) { b += (long long)k * (long long)v; }
__device__ __forceinline__ void acc_cast(double& b, int k, float v) { b = __dadd_rn(b, __dmul_rn((double)k, (double)v)); }
// buffer += k * p: the product in the pixel type, then widened
__device__ __forceinline__ void acc_px(long long& b, int k, int32_t v) { b += (long long)Px<vwb200_dispi>::mul(k, v); }
__device__ __forceinline__ void acc_px(double& b, int k, float v) { b = __dadd_rn(b, (double)Px<DispF>::mul(k, v)); }
__device__ __forceinline__ int32_t acc_div(long long b, long long n) { return (int32_t)(b / n); }      // truncating int64 division
__device__ __forceinline__ float acc_div(double b, long long n) { return __double2float_rn(__ddiv_rn(b, (double)n)); }

// ---- disparity_subsample: one thread per output pixel, the 2 TW + 1 x 2 TH + 1 parent tile (clamped) in shared memory -------
constexpr int kMaxGridY = 65535;                       // the rows of taller rasters are dealt to the blocks grid-stride
constexpr int kSubTW = 32, kSubTH = 8;
constexpr int kSubSW = 2 * kSubTW + 1, kSubSH = 2 * kSubTH + 1;

template <class T>
__global__ void __launch_bounds__(kSubTW * kSubTH) k7_subsample_kernel(const T* __restrict__ in, int w, int h, ptrdiff_t ip,
                                                                     T* __restrict__ out, int ow, int oh, ptrdiff_t op) {
  typedef Px<T> P;
  typedef typename P::C Ch;
  __shared__ Ch s[kSubSH][3 * kSubSW];
  const int ox0 = blockIdx.x * kSubTW, gx0 = 2 * ox0 - 1;
  const int tid = threadIdx.y * kSubTW + threadIdx.x;
  for (int oy0 = blockIdx.y * kSubTH; oy0 < oh; oy0 += gridDim.y * kSubTH) {     // tile rows, grid-stride
    const int gy0 = 2 * oy0 - 1;
    __syncthreads();                                                   // the previous tile row is done with s
    // staging: consecutive threads read consecutive words of a row (ConstantEdgeExtension clamps the pixel index)
    for (int r = 0; r < kSubSH; ++r) {
      const int gy = min(max(gy0 + r, 0), h - 1);
      const Ch* row = reinterpret_cast<const Ch*>(in + (ptrdiff_t)gy * ip);
      for (int k = tid; k < 3 * kSubSW; k += kSubTW * kSubTH) {
        const int p = k / 3, c = k - 3 * p;
        const int gx = min(max(gx0 + p, 0), w - 1);
        s[r][k] = row[3 * gx + c];
      }
    }
    __syncthreads();
    const int ox = ox0 + threadIdx.x, oy = oy0 + threadIdx.y;
    if (ox >= ow || oy >= oh) continue;
    const int sx = 2 * threadIdx.x + 1, sy = 2 * threadIdx.y + 1;         // (ci, cj) in the tile
    typename P::Acc bx = 0, by = 0;
    long long count = 0;
    // DisparitySubsampleView::operator() (:1267-1305), term for term
#define K7_TERM(DX, DY, K, ACC)                                                       \
    {                                                                                   \
      const Ch* q = &s[sy + (DY)][3 * (sx + (DX))];                                     \
      if (q[2] != 0) { count += K; ACC(bx, K, q[0]); ACC(by, K, q[1]); }                \
    }
    K7_TERM(0, 0, 10, acc_cast)
    K7_TERM(1, 0, 5, acc_cast)
    K7_TERM(0, 1, 5, acc_cast)
    K7_TERM(-1, 0, 5, acc_px)
    K7_TERM(0, -1, 5, acc_px)
    K7_TERM(1, 1, 2, acc_px)
    K7_TERM(-1, -1, 2, acc_px)
    K7_TERM(-1, 1, 2, acc_px)
    K7_TERM(1, -1, 2, acc_px)
#undef K7_TERM
    T* o = out + (ptrdiff_t)oy * op + ox;
    *o = count > 0 ? P::make(acc_div(bx, count * 2), acc_div(by, count * 2), true) : P::make(0, 0, false);
  }
}

// ---- the per-pixel operations: one block per 128 pixels of a row, read and written as coalesced words through shared memory
constexpr int kMapPx = 128;

template <class T, class Op>
__global__ void __launch_bounds__(kMapPx) k7_pixel_kernel(const T* in, int w, int h, ptrdiff_t ip, T* out, ptrdiff_t op, Op f) {
  typedef typename Px<T>::C Ch;
  __shared__ Ch s[3 * kMapPx];
  const int x0 = blockIdx.x * kMapPx;
  const int n = 3 * min(kMapPx, w - x0);
  for (int y = blockIdx.y; y < h; y += gridDim.y) {                  // rows, grid-stride (gridDim.y <= 65535)
    __syncthreads();                                                   // the previous row is done with s
    const Ch* src = reinterpret_cast<const Ch*>(in + (ptrdiff_t)y * ip + x0);
    for (int k = threadIdx.x; k < n; k += kMapPx) s[k] = src[k];
    __syncthreads();
    if (3 * (int)threadIdx.x < n) {
      T p{s[3 * threadIdx.x], s[3 * threadIdx.x + 1], s[3 * threadIdx.x + 2]};
      p = f(p, x0 + (int)threadIdx.x, y);
      s[3 * threadIdx.x] = p.dx; s[3 * threadIdx.x + 1] = p.dy; s[3 * threadIdx.x + 2] = p.valid;
    }
    __syncthreads();
    Ch* dst = reinterpret_cast<Ch*>(out + (ptrdiff_t)y * op + x0);       // out may be in: every word was read above
    for (int k = threadIdx.x; k < n; k += kMapPx) dst[k] = s[k];
  }
}

// DisparityRangeMaskFunc (:264-284): the y coordinate is compared against m_min[0], as in the reference
template <class T> struct RangeMaskOp {
  typedef typename Px<T>::C Ch;
  double min0, max0m1, max1m1;
  __device__ T operator()(const T& p, int x, int y) const {
    if (!Px<T>::valid(p)) return p;
    const double ax = __dadd_rn((double)x, (double)p.dx), ay = __dadd_rn((double)y, (double)p.dy);
    if (ax < min0 || ax >= max0m1 || ay < min0 || ay >= max1m1) return Px<T>::make(0, 0, false);
    return p;
  }
};

// m(p) of HomographyTransform::forward / reverse (Math/Transform.h:377-387) for the 3 x 3 matrix m
struct Homography {
  double m[9];
  __device__ __forceinline__ void apply(double px, double py, double& qx, double& qy) const {
    const double w = __dadd_rn(__dadd_rn(__dmul_rn(m[6], px), __dmul_rn(m[7], py)), m[8]);
    qx = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], px), __dmul_rn(m[1], py)), m[2]), w);
    qy = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[3], px), __dmul_rn(m[4], py)), m[5]), w);
  }
};

// TransformDisparitiesFunc (:1023-1044) with m = inverse(H): invalid pixels stay invalid and receive the new values
template <class T> struct TransformLazyOp {
  Homography H;
  __device__ T operator()(const T& p, int x, int y) const {
    const double lx = (double)x, ly = (double)y;
    double nx, ny;
    H.apply(__dadd_rn(lx, (double)p.dx), __dadd_rn(ly, (double)p.dy), nx, ny);
    return Px<T>::make(Px<T>::from_double(__dsub_rn(nx, lx)), Px<T>::from_double(__dsub_rn(ny, ly)), Px<T>::valid(p));
  }
};

// transform_disparities(do_round, subregion, T, disparity) (:1190-1224): invalid pixels give {0, 0, invalid}
template <class T> struct TransformExplicitOp {
  Homography H;
  int sx0, sy0, do_round;
  __device__ T operator()(const T& p, int x, int y) const {
    if (!Px<T>::valid(p)) return Px<T>::make(0, 0, false);
    const double bx = __dadd_rn((double)sx0, (double)x), by = __dadd_rn((double)sy0, (double)y);
    double tx, ty;
    H.apply(__dadd_rn(bx, (double)p.dx), __dadd_rn(by, (double)p.dy), tx, ty);
    double dx = __dsub_rn(tx, bx), dy = __dsub_rn(ty, by);
    if (do_round) { dx = round(dx); dy = round(dy); }    // std::round: halves away from zero
    return Px<T>::make(Px<T>::from_double(dx), Px<T>::from_double(dy), true);
  }
};

// ---- disparity_upsample: one thread per input pixel writes its 2 x 2 block; child * 2 in the pixel type ---------------------
template <class T>
__global__ void k7_upsample_kernel(const T* __restrict__ in, int w, int h, ptrdiff_t ip, T* __restrict__ out, ptrdiff_t op) {
  typedef Px<T> P;
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= w) return;
  for (int y = blockIdx.y; y < h; y += gridDim.y) {                  // rows, grid-stride (gridDim.y <= 65535)
    const T p = in[(ptrdiff_t)y * ip + x];
    const T q = P::make(P::mul(2, p.dx), P::mul(2, p.dy), P::valid(p));
    T* o = out + (ptrdiff_t)(2 * y) * op + 2 * x;
    o[0] = q; o[1] = q; o[op] = q; o[op + 1] = q;
  }
}

// ---- get_disparity_range: PixelAccumulator<EWMinMaxAccumulator> in raster order (Image/Statistics.h:193-223, :286-288) -----
// Five 64-bit keys, each reduced by minimum: [0] the raster index of the first valid pixel; [1 + 2c] (value key << 32 | index)
// of channel c's smallest non-NaN value, [2 + 2c] (~value key << 32 | index) of its largest.  Equal values (-0.0 / +0.0)
// share a key, so the earliest pixel wins, as the sequential `<` / `>` updates keep it.
__device__ __forceinline__ unsigned long long warp_min64(unsigned long long v) {
  for (int o = 16; o; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <class T>
__global__ void __launch_bounds__(256) k7_range_kernel(const T* __restrict__ in, int w, int h, ptrdiff_t ip,
                                                      unsigned long long* __restrict__ keys) {
  typedef Px<T> P;
  unsigned long long k[5] = {~0ull, ~0ull, ~0ull, ~0ull, ~0ull};
  for (int y = blockIdx.x; y < h; y += gridDim.x)
    for (int x = threadIdx.x; x < w; x += blockDim.x) {
      const T p = in[(ptrdiff_t)y * ip + x];
      if (!P::valid(p)) continue;
      const unsigned long long idx = (unsigned long long)y * w + x;
      k[0] = min(k[0], idx);
      if (!P::isnan_(p.dx)) {
        const unsigned long long kk = P::key(p.dx);
        k[1] = min(k[1], kk << 32 | idx); k[2] = min(k[2], (unsigned long long)(~(uint32_t)kk) << 32 | idx);
      }
      if (!P::isnan_(p.dy)) {
        const unsigned long long kk = P::key(p.dy);
        k[3] = min(k[3], kk << 32 | idx); k[4] = min(k[4], (unsigned long long)(~(uint32_t)kk) << 32 | idx);
      }
    }
  __shared__ unsigned long long s[5][8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    k[j] = warp_min64(k[j]);
    if (!lane) s[j][wid] = k[j];
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    unsigned long long m = ~0ull;
    for (int j = 0; j < (int)(blockDim.x >> 5); ++j) m = min(m, s[threadIdx.x][j]);
    if (m != ~0ull) atomicMin(keys + threadIdx.x, m);
  }
}

// the final step: BBox2f(min, max), or (0, 0, 0, 0) without a valid pixel.  A NaN channel of the first valid pixel sticks.
template <class T>
__global__ void k7_range_final_kernel(const T* __restrict__ in, int w, ptrdiff_t ip, const unsigned long long* __restrict__ keys,
                                      float* __restrict__ res5) {
  typedef Px<T> P;
  if (threadIdx.x) return;
  const auto at = [&](unsigned long long key) { const long long i = (long long)(key & 0xffffffffull); return in[(i / w) * ip + i % w]; };
  if (keys[0] == ~0ull) { res5[0] = res5[1] = res5[2] = res5[3] = 0.0f; res5[4] = 0.0f; return; }
  const T first = at(keys[0]);
  if (P::isnan_(first.dx)) { res5[0] = res5[2] = P::to_float(first.dx); }
  else { res5[0] = P::to_float(at(keys[1]).dx); res5[2] = P::to_float(at(keys[2]).dx); }
  if (P::isnan_(first.dy)) { res5[1] = res5[3] = P::to_float(first.dy); }
  else { res5[1] = P::to_float(at(keys[3]).dy); res5[3] = P::to_float(at(keys[4]).dy); }
  res5[4] = 1.0f;
}

template <class T, class Op>
int pixel_launch(const T* in, int w, int h, ptrdiff_t ip, T* out, ptrdiff_t op, const Op& f, cudaStream_t st) {
  if (w <= 0 || h <= 0) return VWB200_OK;
  k7_pixel_kernel<T, Op><<<dim3((w + kMapPx - 1) / kMapPx, std::min(h, kMaxGridY)), kMapPx, 0, st>>>(in, w, h, ip, out, op, f);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

}  // namespace

template <class T>
int dispmap_subsample_launch(const T* in, int w, int h, ptrdiff_t ip, T* out, ptrdiff_t op, cudaStream_t st) {
  const int ow = 1 + (w - 1) / 2, oh = 1 + (h - 1) / 2;
  if (w <= 0 || h <= 0) return VWB200_OK;
  const dim3 grid((ow + kSubTW - 1) / kSubTW, std::min((oh + kSubTH - 1) / kSubTH, kMaxGridY));
  k7_subsample_kernel<T><<<grid, dim3(kSubTW, kSubTH), 0, st>>>(in, w, h, ip, out, ow, oh, op);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

template <class T>
int dispmap_upsample_launch(const T* in, int w, int h, ptrdiff_t ip, T* out, ptrdiff_t op, cudaStream_t st) {
  if (w <= 0 || h <= 0) return VWB200_OK;
  k7_upsample_kernel<T><<<dim3((w + 127) / 128, std::min(h, kMaxGridY)), 128, 0, st>>>(in, w, h, ip, out, op);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

template <class T>
int dispmap_range_launch(const T* in, int w, int h, ptrdiff_t ip, unsigned long long* keys5, float* res5, cudaStream_t st) {
  VWB_CUDA(cudaMemsetAsync(keys5, 0xff, 5 * sizeof(unsigned long long), st));
  const int blocks = std::max(1, std::min(h, 8 * kNumSMs));          // rows are dealt to the blocks
  k7_range_kernel<T><<<blocks, 256, 0, st>>>(in, w, h, ip, keys5);
  VWB_LAUNCH_CHECK();
  k7_range_final_kernel<T><<<1, 32, 0, st>>>(in, w, ip, keys5, res5);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

template <class T>
int dispmap_range_mask_launch(const T* in, int w, int h, ptrdiff_t ip, const void* min2, const void* max2, T* out, ptrdiff_t op,
                              cudaStream_t st) {
  typedef typename Px<T>::C Ch;
  const Ch* mn = static_cast<const Ch*>(min2);
  const Ch* mx = static_cast<const Ch*>(max2);
  RangeMaskOp<T> f;
  f.min0 = (double)mn[0];
  if constexpr (std::is_same<Ch, float>::value) { f.max0m1 = (double)(float)(mx[0] - 1.0f); f.max1m1 = (double)(float)(mx[1] - 1.0f); }
  else { f.max0m1 = (double)(Ch)((uint32_t)mx[0] - 1u); f.max1m1 = (double)(Ch)((uint32_t)mx[1] - 1u); }
  return pixel_launch(in, w, h, ip, out, op, f, st);
}

template <class T>
int dispmap_transform_launch(int mode, const double* m9, int do_round, int sx0, int sy0, const T* in, int w, int h, ptrdiff_t ip,
                             T* out, ptrdiff_t op, cudaStream_t st) {
  Homography H;
  for (int i = 0; i < 9; ++i) H.m[i] = m9[i];
  if (mode == VWB200_TRANSFORM_LAZY) return pixel_launch(in, w, h, ip, out, op, TransformLazyOp<T>{H}, st);
  return pixel_launch(in, w, h, ip, out, op, TransformExplicitOp<T>{H, sx0, sy0, do_round}, st);
}

#define K7_INST(T)                                                                                                         \
  template int dispmap_subsample_launch<T>(const T*, int, int, ptrdiff_t, T*, ptrdiff_t, cudaStream_t);                      \
  template int dispmap_upsample_launch<T>(const T*, int, int, ptrdiff_t, T*, ptrdiff_t, cudaStream_t);                       \
  template int dispmap_range_launch<T>(const T*, int, int, ptrdiff_t, unsigned long long*, float*, cudaStream_t);           \
  template int dispmap_range_mask_launch<T>(const T*, int, int, ptrdiff_t, const void*, const void*, T*, ptrdiff_t, cudaStream_t); \
  template int dispmap_transform_launch<T>(int, const double*, int, int, int, const T*, int, int, ptrdiff_t, T*, ptrdiff_t, cudaStream_t);
K7_INST(vwb200_dispi)
K7_INST(DispF)
#undef K7_INST

}  // namespace vwb200
