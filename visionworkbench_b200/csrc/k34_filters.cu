// k34_filters.cu -- the O(pixels) stages of the level loop that run between K1 launches:
//   K3  cross_corr_consistency_check        (Stereo/Correlate.cc:1441-1502)
//   K4  rm_outliers_using_thresh / disparity_cleanup_using_thresh / disparity_mask
//       (Stereo/DisparityMap.h:318-442, :97-253)
//   finalize: + search_region.min(), int -> float pixel cast (Stereo/CorrelationView.cc:880-884)
// All are integer work on {dx,dy,valid} triples; HBM-bound.
#include "common.cuh"

namespace vwb200 {

__device__ __forceinline__ int clampi3(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// ---- K3 -------------------------------------------------------------------------------------------
// (qax, qay) is added to the R->L disparity before the comparison (the SGM branch keeps it un-shifted, :548-549, 586);
// diff (optional): the lr_disp_diff image, PixelMask<float> = {value, valid} pairs; pixel (c + dox, r + doy) receives the
// discrepancy of a pixel that passes (Correlate.cc:1476-1484)
__device__ __forceinline__ void consistency_pixel(vwb200_dispi* p, int c, int r, const vwb200_dispi* r2l, int rw, int rh,
                                                  ptrdiff_t rpitch, float thr, int qax = 0, int qay = 0, float2* diff = nullptr,
                                                  ptrdiff_t dpitch = 0, int dox = 0, int doy = 0) {
  const vwb200_dispi v = *p;
  const int x = c + v.dx, y = r + v.dy;
  if (x < 0 || x >= rw || y < 0 || y >= rh) { p->valid = 0; return; }
  const vwb200_dispi q = r2l[(ptrdiff_t)y * rpitch + x];
  if (!v.valid || !q.valid) { p->valid = 0; return; }
  const double a = fabs((double)(v.dx + q.dx + qax)), b = fabs((double)(v.dy + q.dy + qay));
  const float d = (float)(a > b ? a : b);
  if (!(thr >= d)) p->valid = 0;
  else if (diff) diff[(ptrdiff_t)(r + doy) * dpitch + (c + dox)] = make_float2(d, 1.0f);
}
__global__ void consistency_kernel(vwb200_dispi* l2r, int lw, int lh, ptrdiff_t lpitch, const vwb200_dispi* r2l, int rw,
                                   int rh, ptrdiff_t rpitch, float thr, int qax, int qay, float2* diff, ptrdiff_t dpitch, int dox, int doy) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y * blockDim.y + threadIdx.y;
  if (c >= lw || r >= lh) return;
  consistency_pixel(l2r + (ptrdiff_t)r * lpitch + c, c, r, r2l, rw, rh, rpitch, thr, qax, qay, diff, dpitch, dox, doy);
}
int consistency_launch(vwb200_dispi* l2r, int lw, int lh, ptrdiff_t lpitch, const vwb200_dispi* r2l, int rw, int rh,
                       ptrdiff_t rpitch, float thr, cudaStream_t st, int qax, int qay, float* diff, ptrdiff_t dpitch, int dox, int doy) {
  if (lw <= 0 || lh <= 0) return VWB200_OK;
  dim3 b(32, 8), g((lw + 31) / 32, (lh + 7) / 8);
  consistency_kernel<<<g, b, 0, st>>>(l2r, lw, lh, lpitch, r2l, rw, rh, rpitch, thr, qax, qay, reinterpret_cast<float2*>(diff), dpitch, dox, doy);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// Zone-table form used by the level loop: per zone, optional L/R check against that zone's R->L
// image, then "+= zone.disparity_range().min()" (CorrelationView.cc:691-698).  One launch per level.
__global__ void zone_post_kernel(const Tile* __restrict__ tiles, const Zone* __restrict__ zones, const Zone* __restrict__ rlzones,
                                 const int2* __restrict__ post_add, vwb200_dispi* __restrict__ disp,
                                 const vwb200_dispi* __restrict__ rl, float thr, int tile_w, int tile_h, float2* diff, ptrdiff_t dpitch,
                                 int dox, int doy) {
  const Tile t = tiles[blockIdx.x];
  const Zone z = zones[t.zone];
  const int tw = min(tile_w, z.w - t.tx), th = min(tile_h, z.h - t.ty);
  const int2 add = post_add[t.zone];
  for (int k = threadIdx.x; k < tw * th; k += blockDim.x) {
    const int x = t.tx + k % tw, y = t.ty + k / tw;
    vwb200_dispi* p = disp + z.obase + (ptrdiff_t)y * z.opitch + x;
    if (rl) {
      const Zone q = rlzones[t.zone];
      // lr_disp_diff: ul_corner_offset = zone.image_region().min() + bbox.min() - region_ul (CorrelationView.cc:669-676)
      const int zx0 = (int)(z.obase % z.opitch), zy0 = (int)(z.obase / z.opitch);
      consistency_pixel(p, x, y, rl + q.obase, q.w, q.h, q.opitch, thr, 0, 0, diff, dpitch, dox + zx0, doy + zy0);
    }
    p->dx += add.x;
    p->dy += add.y;
  }
}
int zone_post_launch(const Tile* d_tiles, int ntiles, const Zone* d_zones, const Zone* d_rlzones, const int2* d_post_add,
                     vwb200_dispi* disp, const vwb200_dispi* rl, float thr, int tile_w, int tile_h, cudaStream_t st, float* diff,
                     ptrdiff_t dpitch, int dox, int doy) {
  if (ntiles <= 0) return VWB200_OK;
  zone_post_kernel<<<ntiles, 128, 0, st>>>(d_tiles, d_zones, d_rlzones, d_post_add, disp, rl, thr, tile_w, tile_h,
                                           reinterpret_cast<float2*>(diff), dpitch, dox, doy);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// The pixel types of the outlier filters: PixelMask<Vector2i> and PixelMask<Vector2f>, valid when valid != 0.  absdiff is
// the reference's fabs((*acc)[0] - (*col_acc)[0]): the difference in the pixel type (int, or a rounded float), then a
// double.  key is |dx| + |dy| in the pixel type (RmOutliersUsingMeanFunc's len, DisparityMap.h:504) as an order-preserving
// uint32: the int itself, or the float's fkey (the sum is never negative); kval is the key's value as a double.  The thresh
// filter stages an invalid pixel's dx as `absent` (INT_MIN, or NaN), which `present` tells apart.
template <class T> struct OutlierPx;
template <> struct OutlierPx<vwb200_dispi> {
  typedef int V;
  static __device__ __forceinline__ bool valid(const vwb200_dispi& p) { return p.valid != 0; }
  static __device__ __forceinline__ int absent() { return INT_MIN; }
  static __device__ __forceinline__ bool present(int dx) { return dx != INT_MIN; }
  static __device__ __forceinline__ double absdiff(int a, int b) { return fabs((double)(a - b)); }
  static __device__ __forceinline__ unsigned key(int dx, int dy) { return (unsigned)(abs(dx) + abs(dy)); }
  static __device__ __forceinline__ double kval(unsigned k) { return (double)(int)k; }
};
template <> struct OutlierPx<DispF> {
  typedef float V;
  static __device__ __forceinline__ bool valid(const DispF& p) { return p.valid != 0.0f; }
  static __device__ __forceinline__ float absent() { return __int_as_float(0x7fffffff); }
  static __device__ __forceinline__ bool present(float dx) { return !isnan(dx); }
  static __device__ __forceinline__ double absdiff(float a, float b) { return (double)fabsf(__fsub_rn(a, b)); }
  static __device__ __forceinline__ unsigned key(float dx, float dy) { return fkey(__fadd_rn(fabsf(dx), fabsf(dy))); }
  static __device__ __forceinline__ double kval(unsigned k) { return (double)kfloat(k); }
};

// second pass (1,1,3.0,0.20) over the padded first-pass buffer p1 of size (w+2) x (h+2)  (DisparityMap.h:440)
template <class T>
__global__ void cleanup_pass2_kernel(const T* __restrict__ p1, int w, int h, T* __restrict__ out) {
  typedef OutlierPx<T> Px;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const int pw = w + 2;
  T c = p1[(ptrdiff_t)(y + 1) * pw + (x + 1)];
  if (Px::valid(c)) {
    int matched = 0;
#pragma unroll
    for (int yk = -1; yk <= 1; ++yk)
#pragma unroll
      for (int xk = -1; xk <= 1; ++xk) {
        const T n = p1[(ptrdiff_t)(y + 1 + yk) * pw + (x + 1 + xk)];
        if (Px::valid(n) && Px::absdiff(c.dx, n.dx) <= 3.0 && Px::absdiff(c.dy, n.dy) <= 3.0) ++matched;
      }
    if (((double)matched / 9.0) < 0.20) { c.dx = 0; c.dy = 0; c.valid = 0; }
  }
  out[(ptrdiff_t)y * w + x] = c;
}
template <class T>
static int cleanup_pass2_launch_t(const T* p1, int w, int h, T* out, cudaStream_t st) {
  if (w <= 0 || h <= 0) return VWB200_OK;
  dim3 b(32, 8), g((w + 31) / 32, (h + 7) / 8);
  cleanup_pass2_kernel<T><<<g, b, 0, st>>>(p1, w, h, out);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}
int cleanup_pass2_launch(const vwb200_dispi* p1, int w, int h, vwb200_dispi* out, cudaStream_t st) {
  return cleanup_pass2_launch_t(p1, w, h, out, st);
}
int cleanup_pass2_launch(const DispF* p1, int w, int h, DispF* out, cudaStream_t st) {
  return cleanup_pass2_launch_t(p1, w, h, out, st);
}

// ---- K4 on both pixel types: pass 1 of rm_outliers_using_thresh / _mean / _stddev ----------------------------------------
// (DisparityMap.h:359-386, :484-553, :646-723).  One thread per output pixel over [x0,x0+ow) x [y0,y0+oh) of the
// ConstantEdgeExtension of `in`; the output window may extend past the image (the padded first pass of the cleanup
// composites, Image/PerPixelAccessorViews.h:63-85).  The CTA stages its tile + halo in shared memory as {dx}, {dy}, and for
// mean and stddev a key word: kNoKeyO for an invalid pixel, else |dx| + |dy| as a key (mean) or 0.  Thresh folds validity
// into dx instead (Px::absent), so its hot loop reads two planes.  Every sum runs in the reference's row-major order with
// explicitly rounded operations (no contraction).
static constexpr int RO_TW = 32, RO_TH = 8;
static constexpr unsigned kNoKeyO = 0xFFFFFFFFu;   // above every key of a finite |dx| + |dy|
static constexpr size_t kOutlierSmemMax = 200 * 1024;

template <class T, int M>
__global__ void __launch_bounds__(RO_TW * RO_TH)
outlier_pass1_kernel(const T* __restrict__ in, int w, int h, ptrdiff_t ipitch, int hx, int hy, double pt, double rt, double mdsq,
                     int x0, int y0, int ow, int oh, T* __restrict__ out, ptrdiff_t opitch) {
  typedef OutlierPx<T> Px;
  typedef typename Px::V V;
  extern __shared__ unsigned osm[];
  const int sw = RO_TW + 2 * hx, sh = RO_TH + 2 * hy, sn = sw * sh;
  V* sdx = reinterpret_cast<V*>(osm);
  V* sdy = sdx + sn;
  unsigned* skey = osm + 2 * sn;                          // mean and stddev only
  const int bx = x0 + blockIdx.x * RO_TW, by = y0 + blockIdx.y * RO_TH;
  for (int k = threadIdx.y * RO_TW + threadIdx.x; k < sn; k += RO_TW * RO_TH) {
    const int sx = k % sw, sy = k / sw;
    const T v = in[(ptrdiff_t)clampi3(by - hy + sy, 0, h - 1) * ipitch + clampi3(bx - hx + sx, 0, w - 1)];
    sdx[k] = M == VWB200_OUTLIERS_THRESH && !Px::valid(v) ? Px::absent() : v.dx;
    sdy[k] = v.dy;
    if (M != VWB200_OUTLIERS_THRESH) skey[k] = !Px::valid(v) ? kNoKeyO : M == VWB200_OUTLIERS_MEAN ? Px::key(v.dx, v.dy) : 0u;
  }
  __syncthreads();
  const int ox = blockIdx.x * RO_TW + threadIdx.x, oy = blockIdx.y * RO_TH + threadIdx.y;
  if (ox >= ow || oy >= oh) return;
  // the centre keeps all three values, also when invalid ("return *acc")
  T c = in[(ptrdiff_t)clampi3(y0 + oy, 0, h - 1) * ipitch + clampi3(x0 + ox, 0, w - 1)];
  if (Px::valid(c)) {
    const int base = threadIdx.y * sw + threadIdx.x;      // window corner in the tile
    bool reject;
    if (M == VWB200_OUTLIERS_THRESH) {                    // :362-384
      int matched = 0;
      for (int yk = 0; yk <= 2 * hy; ++yk) {
        const int r = base + yk * sw;
        for (int xk = 0; xk <= 2 * hx; ++xk)
          if (Px::present(sdx[r + xk]) && Px::absdiff(c.dx, sdx[r + xk]) <= pt && Px::absdiff(c.dy, sdy[r + xk]) <= pt) ++matched;
      }
      reject = __ddiv_rn((double)matched, (double)((2 * hx + 1) * (2 * hy + 1))) < rt;
    } else if (M == VWB200_OUTLIERS_MEAN) {               // :497-550
      // cutoff = 2 * (the floor(0.75 n)-th smallest len): a bitwise select over the keys, from the highest bit in which the
      // window's smallest and largest keys differ (MedianOp of k6_smoothing.cu, here within one thread)
      unsigned n = 0, mn = kNoKeyO, mx = 0;
      for (int yk = 0; yk <= 2 * hy; ++yk) {
        const unsigned* kr = skey + base + yk * sw;
        for (int xk = 0; xk <= 2 * hx; ++xk) {
          const unsigned k = kr[xk];
          if (k != kNoKeyO) { ++n; mn = min(mn, k); mx = max(mx, k); }
        }
      }
      unsigned t = (unsigned)(int)__dmul_rn(0.75, (double)n), p = mn;
      const int hb = mn == mx ? -1 : 31 - __clz(mn ^ mx);
      if (hb >= 0) p = mn & ~((2u << hb) - 1u);
      for (int b = hb; b >= 0; --b) {                     // kNoKeyO has every bit set: never counted
        const unsigned lim = 1u << b;
        unsigned cnt = 0;
        for (int yk = 0; yk <= 2 * hy; ++yk) {
          const unsigned* kr = skey + base + yk * sw;
          for (int xk = 0; xk <= 2 * hx; ++xk) cnt += (kr[xk] ^ p) < lim;
        }
        if (t >= cnt) { t -= cnt; p |= lim; }
      }
      const double cutoff = __dmul_rn(2.0, Px::kval(p));
      // `if (val > cutoff) continue;` skips col_acc.next_col(): the rest of that window row reads the same pixel, so the
      // row ends there
      unsigned matched = 0;
      double mX = 0.0, mY = 0.0;
      for (int yk = 0; yk <= 2 * hy; ++yk) {
        const int r = base + yk * sw;
        for (int xk = 0; xk <= 2 * hx; ++xk) {
          const unsigned k = skey[r + xk];
          if (k == kNoKeyO) continue;
          if (Px::kval(k) > cutoff) break;
          mX = __dadd_rn(mX, (double)sdx[r + xk]);
          mY = __dadd_rn(mY, (double)sdy[r + xk]);
          ++matched;
        }
      }
      double esq = __dadd_rn(mdsq, 1.0);
      if (matched > 0) {
        mX = __ddiv_rn(mX, (double)matched);
        mY = __ddiv_rn(mY, (double)matched);
        const double ex = __dsub_rn((double)c.dx, mX), ey = __dsub_rn((double)c.dy, mY);
        esq = __dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey));
      }
      reject = esq > mdsq;
    } else {                                              // :659-720
      unsigned matched = 0;
      double mX = 0.0, mY = 0.0;
      for (int yk = 0; yk <= 2 * hy; ++yk) {
        const int r = base + yk * sw;
        for (int xk = 0; xk <= 2 * hx; ++xk)
          if (skey[r + xk] != kNoKeyO) {
            mX = __dadd_rn(mX, (double)sdx[r + xk]);
            mY = __dadd_rn(mY, (double)sdy[r + xk]);
            ++matched;
          }
      }
      reject = matched == 0;
      if (matched > 0) {
        mX = __ddiv_rn(mX, (double)matched);
        mY = __ddiv_rn(mY, (double)matched);
        double sX = 0.0, sY = 0.0;
        for (int yk = 0; yk <= 2 * hy; ++yk) {
          const int r = base + yk * sw;
          for (int xk = 0; xk <= 2 * hx; ++xk)
            if (skey[r + xk] != kNoKeyO) {
              const double dX = __dsub_rn((double)sdx[r + xk], mX), dY = __dsub_rn((double)sdy[r + xk], mY);
              sX = __dadd_rn(sX, __dmul_rn(dX, dX));
              sY = __dadd_rn(sY, __dmul_rn(dY, dY));
            }
        }
        double sdX = __dsqrt_rn(__ddiv_rn(sX, (double)matched)), sdY = __dsqrt_rn(__ddiv_rn(sY, (double)matched));
        if (sdX < rt) sdX = rt;
        if (sdY < rt) sdY = rt;
        const double eX = fabs(__dsub_rn((double)c.dx, mX)), eY = fabs(__dsub_rn((double)c.dy, mY));
        reject = eX > __dmul_rn(pt, sdX) || eY > __dmul_rn(pt, sdY);
      }
    }
    if (reject) { c.dx = 0; c.dy = 0; c.valid = 0; }
  }
  out[(ptrdiff_t)oy * opitch + ox] = c;
}

template <class T>
int outlier_pass1_launch(int method, const T* in, int w, int h, ptrdiff_t ipitch, int hx, int hy, double pt, double rt,
                         double max_mean_diff, int x0, int y0, int ow, int oh, T* out, ptrdiff_t opitch, cudaStream_t st) {
  if (hx <= 0 || hy <= 0) {                               // DisparityMap.h:343-344, :470-471, :631-632
    set_error(method == VWB200_OUTLIERS_MEAN ? "RmOutliersUsingMeanFunc: half kernel sizes must be non-zero."
                                             : "RmOutliersFunc: half kernel sizes must be non-zero.");
    return VWB200_EARG;
  }
  if (ow <= 0 || oh <= 0) return VWB200_OK;
  const size_t planes = method == VWB200_OUTLIERS_THRESH ? 2 : 3;
  const size_t smem = (size_t)(RO_TW + 2 * hx) * (RO_TH + 2 * hy) * planes * sizeof(unsigned);
  if (smem > kOutlierSmemMax) { set_error("outlier filter half kernel %dx%d too large", hx, hy); return VWB200_ENOIMPL; }
  const dim3 b(RO_TW, RO_TH), g((ow + RO_TW - 1) / RO_TW, (oh + RO_TH - 1) / RO_TH);
  if (g.y > 65535) { set_error("outlier filter: %d rows are above the supported %d", oh, 65535 * RO_TH); return VWB200_ENOIMPL; }
  void (*kern)(const T*, int, int, ptrdiff_t, int, int, double, double, double, int, int, int, int, T*, ptrdiff_t) =
      method == VWB200_OUTLIERS_THRESH ? outlier_pass1_kernel<T, VWB200_OUTLIERS_THRESH>
      : method == VWB200_OUTLIERS_MEAN ? outlier_pass1_kernel<T, VWB200_OUTLIERS_MEAN>
                                       : outlier_pass1_kernel<T, VWB200_OUTLIERS_STDDEV>;
  VWB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));   // per-function state shared by all host threads: device maximum
  kern<<<g, b, smem, st>>>(in, w, h, ipitch, hx, hy, pt, rt, max_mean_diff * max_mean_diff, x0, y0, ow, oh, out, opitch);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}
template int outlier_pass1_launch<vwb200_dispi>(int, const vwb200_dispi*, int, int, ptrdiff_t, int, int, double, double, double, int, int,
                                                int, int, vwb200_dispi*, ptrdiff_t, cudaStream_t);
template int outlier_pass1_launch<DispF>(int, const DispF*, int, int, ptrdiff_t, int, int, double, double, double, int, int, int, int,
                                         DispF*, ptrdiff_t, cudaStream_t);

// ---- disparity_mask (DisparityMap.h:142-162) --------------------------------------------------------------
__global__ void disparity_mask_kernel(const vwb200_dispi* __restrict__ in, int w, int h, ImgB lm, ImgB rm, vwb200_dispi* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
  if (i >= w || j >= h) return;
  vwb200_dispi z; z.dx = 0; z.dy = 0; z.valid = 0;
  vwb200_dispi d = in[(ptrdiff_t)j * w + i];
  bool keep = lm.p[(ptrdiff_t)j * lm.pitch + i] != 0 && d.valid;
  if (keep) {
    const int tx = i + d.dx, ty = j + d.dy;
    keep = !(tx < 0 || tx >= rm.w || ty < 0 || ty >= rm.h) && rm.p[(ptrdiff_t)ty * rm.pitch + tx] != 0;
  }
  out[(ptrdiff_t)j * w + i] = keep ? d : z;
}
int disparity_mask_launch(const vwb200_dispi* in, int w, int h, ImgB lmask, ImgB rmask, vwb200_dispi* out, cudaStream_t st) {
  if (w <= 0 || h <= 0) return VWB200_OK;
  dim3 b(32, 8), g((w + 31) / 32, (h + 7) / 8);
  disparity_mask_kernel<<<g, b, 0, st>>>(in, w, h, lmask, rmask, out);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// ---- finalize: disparity + search.min, pixel_cast<PixelMask<Vector2f>> (CorrelationView.cc:880-884) -------
// Writes the [ox,ox+ow) x [oy,oy+oh) window of the w x h tile result to a 12-byte-pixel destination.
__global__ void finalize_kernel(const vwb200_dispi* __restrict__ in, int w, int ax, int ay, float* __restrict__ out,
                                ptrdiff_t opitch_px, int ox, int oy, int ow, int oh) {
  // one thread per output float: fully coalesced 4-byte stores over the 12-byte pixels
  const int k = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (k >= 3 * ow || y >= oh) return;
  const int x = k / 3, c = k % 3;
  const int* src = reinterpret_cast<const int*>(in + (ptrdiff_t)(oy + y) * w + (ox + x));
  float v;
  if (c == 0) v = (float)(src[0] + ax);
  else if (c == 1) v = (float)(src[1] + ay);
  else v = src[2] ? 1.0f : 0.0f;
  out[(ptrdiff_t)y * opitch_px * 3 + k] = v;
}
int finalize_launch(const vwb200_dispi* in, int w, int h, int ax, int ay, float* out, ptrdiff_t opitch_px,
                    int ox, int oy, int ow, int oh, cudaStream_t st) {
  (void)h;
  if (ow <= 0 || oh <= 0) return VWB200_OK;
  dim3 b(256), g((3 * ow + 255) / 256, oh);
  finalize_kernel<<<g, b, 0, st>>>(in, w, ax, ay, out, opitch_px, ox, oy, ow, oh);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}


// ---- lr_disp_diff: invalidate where the final disparity is invalid (CorrelationView.cc:848-857) -----------------------
__global__ void diff_invalidate_kernel(const vwb200_dispi* __restrict__ disp, int w, int h, float2* __restrict__ diff, ptrdiff_t dpitch,
                                       int dox, int doy) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y * blockDim.y + threadIdx.y;
  if (c >= w || r >= h) return;
  if (!disp[(size_t)r * w + c].valid) diff[(ptrdiff_t)(r + doy) * dpitch + (c + dox)].y = 0.0f;
}
int diff_invalidate_launch(const vwb200_dispi* disp, int w, int h, float* diff, ptrdiff_t dpitch, int dox, int doy, cudaStream_t st) {
  if (w <= 0 || h <= 0) return VWB200_OK;
  diff_invalidate_kernel<<<dim3((w + 31) / 32, (h + 7) / 8), dim3(32, 8), 0, st>>>(disp, w, h, reinterpret_cast<float2*>(diff), dpitch, dox, doy);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// ---- SGM branch: result = subpixel_disparity + search_region.min(), valid where both the sub-pixel view and the filtered
// integer disparity are (CorrelationView.cc:859-871; PixelMask sums keep the child values of invalid pixels) ------------------
__global__ void sgm_finalize_kernel(const float* __restrict__ sub, const vwb200_dispi* __restrict__ disp, int w, float ax, float ay,
                                    float* __restrict__ out, ptrdiff_t opitch_px, int ox, int oy, int ow, int oh) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= ow || y >= oh) return;
  const size_t src = (size_t)(oy + y) * w + (ox + x);
  float* o = out + ((ptrdiff_t)y * opitch_px + x) * 3;
  o[0] = __fadd_rn(sub[3 * src], ax);
  o[1] = __fadd_rn(sub[3 * src + 1], ay);
  o[2] = (sub[3 * src + 2] != 0.0f && disp[src].valid) ? 1.0f : 0.0f;
}
int sgm_finalize_launch(const float* sub, const vwb200_dispi* disp, int w, int ax, int ay, float* out, ptrdiff_t opitch_px, int ox, int oy,
                        int ow, int oh, cudaStream_t st) {
  if (ow <= 0 || oh <= 0) return VWB200_OK;
  sgm_finalize_kernel<<<dim3((ow + 127) / 128, oh), 128, 0, st>>>(sub, disp, w, (float)ax, (float)ay, out, opitch_px, ox, oy, ow, oh);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// ---- disparity_blob_filter (CorrelationView.cc:242-271; BlobIndexThreaded, Image/BlobIndex.h:385-454; ErodeView.h:196-218):
// 8-connected components of the valid pixels by union-find on pixel indices (the smaller index is the root, so the forest is
// the same whatever the thread order); components of at most `area` pixels become result_type() = {0, 0, invalid}.
__device__ __forceinline__ int uf_root(const int* parent, int i) { int p; while ((p = parent[i]) != i) i = p; return i; }
__device__ void uf_union(int* parent, int a, int b) {
  while (true) {
    a = uf_root(parent, a); b = uf_root(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }          // a > b: hang a under b
    const int old = atomicMin(parent + a, b);
    if (old == a) return;
    a = old;                                               // somebody else moved a meanwhile: merge its new parent with b
  }
}
__global__ void blob_init_kernel(const vwb200_dispi* __restrict__ d, int n, int* __restrict__ parent, int* __restrict__ size) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  parent[i] = d[i].valid ? i : -1;
  size[i] = 0;
}
__global__ void blob_union_kernel(const vwb200_dispi* __restrict__ d, int w, int h, int* __restrict__ parent) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const int i = y * w + x;
  if (!d[i].valid) return;
  if (x > 0 && d[i - 1].valid) uf_union(parent, i, i - 1);
  if (y > 0) {
    if (d[i - w].valid) uf_union(parent, i, i - w);
    if (x > 0 && d[i - w - 1].valid) uf_union(parent, i, i - w - 1);
    if (x < w - 1 && d[i - w + 1].valid) uf_union(parent, i, i - w + 1);
  }
}
__global__ void blob_count_kernel(int n, int* __restrict__ parent, int* __restrict__ size) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || parent[i] < 0) return;
  const int r = uf_root(parent, i);
  parent[i] = r;                                           // compress (roots keep pointing at themselves)
  atomicAdd(size + r, 1);
}
__global__ void blob_erode_kernel(vwb200_dispi* __restrict__ d, int n, const int* __restrict__ parent, const int* __restrict__ size, int area) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || parent[i] < 0) return;
  if (size[uf_root(parent, i)] <= area) { vwb200_dispi z; z.dx = 0; z.dy = 0; z.valid = 0; d[i] = z; }
}
int blob_filter_launch(vwb200_dispi* d, int w, int h, int area, int* work /* 2 * w * h ints */, cudaStream_t st) {
  if (area < 1 || w <= 0 || h <= 0) return VWB200_OK;      // CorrelationView.cc:249-250
  const int n = w * h;
  int* parent = work; int* size = work + n;
  blob_init_kernel<<<(n + 255) / 256, 256, 0, st>>>(d, n, parent, size);
  VWB_LAUNCH_CHECK();
  blob_union_kernel<<<dim3((w + 31) / 32, (h + 7) / 8), dim3(32, 8), 0, st>>>(d, w, h, parent);
  VWB_LAUNCH_CHECK();
  blob_count_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, parent, size);
  VWB_LAUNCH_CHECK();
  blob_erode_kernel<<<(n + 255) / 256, 256, 0, st>>>(d, n, parent, size, area);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// ====================================================================================================
// a11: ParabolaSubpixelView (Stereo/ParabolaSubpixelView.cc:31-330)
// ====================================================================================================
// min / max of the truncated integer disparity over the valid pixels of a bbox crop (get_disparity_range,
// Stereo/DisparityMap.h:52-66).  r[0..3] = minx, miny, maxx, maxy ; r[4] = any valid
__global__ void disp_range_kernel(const float* __restrict__ disp, int cols, int bx0, int by0, int bw, int bh, int* __restrict__ r) {
  int mnx = INT_MAX, mny = INT_MAX, mxx = INT_MIN, mxy = INT_MIN, any = 0;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < (long long)bw * bh; k += (long long)gridDim.x * blockDim.x) {
    const float* p = disp + ((ptrdiff_t)(by0 + (int)(k / bw)) * cols + bx0 + (int)(k % bw)) * 3;
    if (p[2] != 0.0f) { const int dx = (int)p[0], dy = (int)p[1]; mnx = min(mnx, dx); mxx = max(mxx, dx); mny = min(mny, dy); mxy = max(mxy, dy); any = 1; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    mnx = min(mnx, __shfl_xor_sync(0xffffffffu, mnx, o)); mny = min(mny, __shfl_xor_sync(0xffffffffu, mny, o));
    mxx = max(mxx, __shfl_xor_sync(0xffffffffu, mxx, o)); mxy = max(mxy, __shfl_xor_sync(0xffffffffu, mxy, o));
    any |= __shfl_xor_sync(0xffffffffu, any, o);
  }
  if ((threadIdx.x & 31) == 0 && any) { atomicMin(r + 0, mnx); atomicMin(r + 1, mny); atomicMax(r + 2, mxx); atomicMax(r + 3, mxy); atomicExch(r + 4, 1); }
}
int disp_range_launch(const float* disp, int cols, int bx0, int by0, int bw, int bh, int* d_r5, cudaStream_t st) {
  const int init[5] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN, 0};
  VWB_CUDA(cudaMemcpyAsync(d_r5, init, sizeof(init), cudaMemcpyHostToDevice, st));
  VWB_CUDA(cudaStreamSynchronize(st));
  disp_range_kernel<<<kNumSMs, 256, 0, st>>>(disp, cols, bx0, by0, bw, bh, d_r5);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// out(x,y) = e(x+m, y+m) - g(x+m, y+m): SubtractedMean over a region of the replicate-extended image
__global__ void meansub_region_kernel(const float* __restrict__ e, const float* __restrict__ g, int ew, int m, int w, int h, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const ptrdiff_t k = (ptrdiff_t)(y + m) * ew + (x + m);
  out[(ptrdiff_t)y * w + x] = __fsub_rn(e[k], g[k]);
}
// LoG over a region: Laplacian stencil over the in-image gaussian read at clamped image coordinates
__global__ void log_region_kernel(const float* __restrict__ g, int gw, int gx0, int gy0, int iw, int ih, int rx0, int ry0, int w, int h, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= w || y >= h) return;
  const int cx = rx0 + x, cy = ry0 + y;
#define GAT(X, Y) g[(ptrdiff_t)(clampi3((Y), 0, ih - 1) - gy0) * gw + (clampi3((X), 0, iw - 1) - gx0)]
  float r = __fadd_rn(0.0f, __fmul_rn(1.0f, GAT(cx, cy - 1)));
  r = __fadd_rn(r, __fmul_rn(1.0f, GAT(cx - 1, cy)));
  r = __fadd_rn(r, __fmul_rn(-4.0f, GAT(cx, cy)));
  r = __fadd_rn(r, __fmul_rn(1.0f, GAT(cx + 1, cy)));
  r = __fadd_rn(r, __fmul_rn(1.0f, GAT(cx, cy + 1)));
#undef GAT
  out[(ptrdiff_t)y * w + x] = r;
}
int meansub_region_launch(const float* e, const float* g, int ew, int m, int w, int h, float* out, cudaStream_t st) {
  dim3 b(32, 8), gr((w + 31) / 32, (h + 7) / 8);
  meansub_region_kernel<<<gr, b, 0, st>>>(e, g, ew, m, w, h, out);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}
int log_region_launch(const float* g, int gw, int gx0, int gy0, int iw, int ih, int rx0, int ry0, int w, int h, float* out, cudaStream_t st) {
  dim3 b(32, 8), gr((w + 31) / 32, (h + 7) / 8);
  log_region_kernel<<<gr, b, 0, st>>>(g, gw, gx0, gy0, iw, ih, rx0, ry0, w, h, out);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// One thread per pixel: the 9 AbsoluteCost window sums around the integer disparity (double accumulation of float
// |a-b|, exactly the values the reference's per-zone fast_box_sum produces when sums are exact), the 6x9 float
// pseudo-inverse fit with the reference's operation order, offset kept if its norm is below 5
// (ParabolaSubpixelView.h:82-88, .cc:230-275).
__constant__ float c_pinv[54];
__global__ void parabola_kernel(const float* __restrict__ disp, int cols, int bx0, int by0, int bw, int bh,
                                const float* __restrict__ L, int lw, const float* __restrict__ R, int rw,
                                int srx0, int sry0, int kx, int ky, float* __restrict__ out) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= bw || y >= bh) return;
  const float* p = disp + ((ptrdiff_t)(by0 + y) * cols + bx0 + x) * 3;
  float* o = out + ((ptrdiff_t)y * bw + x) * 3;
  if (p[2] == 0.0f) { o[0] = 0.0f; o[1] = 0.0f; o[2] = 0.0f; return; }
  const int dx = (int)p[0], dy = (int)p[1];
  float c[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int ex = k % 3 - 1, ey = k / 3 - 1;
    // L raster origin = bbox.min - half kernel: window of pixel (x,y) starts at (x,y); R raster origin adds sr.min
    const float* lp = L + (ptrdiff_t)y * lw + x;
    const float* rp = R + (ptrdiff_t)(y + dy + ey - sry0) * rw + (x + dx + ex - srx0);
    double s = 0.0;
    for (int j = 0; j < ky; ++j)
      for (int i = 0; i < kx; ++i) s += (double)fabsf(__fsub_rn(lp[(ptrdiff_t)j * lw + i], rp[(ptrdiff_t)j * rw + i]));
    c[k] = (float)s;
  }
  o[0] = (float)dx; o[1] = (float)dy; o[2] = 1.0f;
  bool alleq = true;
#pragma unroll
  for (int k = 1; k < 9; ++k) alleq = alleq && (c[k] == c[k - 1]);
  if (alleq) return;
  float xs[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    float acc = 0.0f;
#pragma unroll
    for (int k = 0; k < 9; ++k) acc = __fadd_rn(acc, __fmul_rn(c_pinv[r * 9 + k], c[k]));
    xs[r] = acc;
  }
  const float denom = __fsub_rn(__fmul_rn(__fmul_rn(4.0f, xs[0]), xs[1]), __fmul_rn(xs[2], xs[2]));
  const float ox = __fdiv_rn(__fsub_rn(__fmul_rn(xs[2], xs[4]), __fmul_rn(__fmul_rn(2.0f, xs[1]), xs[3])), denom);
  const float oy = __fdiv_rn(__fsub_rn(__fmul_rn(xs[2], xs[3]), __fmul_rn(__fmul_rn(2.0f, xs[0]), xs[4])), denom);
  double nn = 0.0;
  nn += (double)__fmul_rn(ox, ox);
  nn += (double)__fmul_rn(oy, oy);
  nn = (double)(float)nn;
  if (sqrt(nn) < 5.0) { o[0] = __fadd_rn((float)dx, ox); o[1] = __fadd_rn((float)dy, oy); }
}
int parabola_launch(const float* disp, int cols, int bx0, int by0, int bw, int bh, const float* L, int lw, const float* R, int rw,
                    int srx0, int sry0, int kx, int ky, float* out, cudaStream_t st) {
  static const double pd[54] = {
     1.0/6, -1.0/3,  1.0/6,  1.0/6, -1.0/3,  1.0/6,   1.0/6, -1.0/3,  1.0/6,
     1.0/6,  1.0/6,  1.0/6, -1.0/3, -1.0/3, -1.0/3,   1.0/6,  1.0/6,  1.0/6,
     1.0/4,    0.0, -1.0/4,    0.0,    0.0,    0.0,  -1.0/4,    0.0,  1.0/4,
    -1.0/6,    0.0,  1.0/6, -1.0/6,    0.0,  1.0/6,  -1.0/6,    0.0,  1.0/6,
    -1.0/6, -1.0/6, -1.0/6,    0.0,    0.0,    0.0,   1.0/6,  1.0/6,  1.0/6,
    -1.0/9,  2.0/9, -1.0/9,  2.0/9,   5.0/9, 2.0/9,  -1.0/9,  2.0/9, -1.0/9 };
  float pf[54];
  for (int i = 0; i < 54; ++i) pf[i] = (float)pd[i];
  VWB_CUDA(cudaMemcpyToSymbolAsync(c_pinv, pf, sizeof(pf), 0, cudaMemcpyHostToDevice, st));
  VWB_CUDA(cudaStreamSynchronize(st));
  dim3 b(32, 8), g((bw + 31) / 32, (bh + 7) / 8);
  parabola_kernel<<<g, b, 0, st>>>(disp, cols, bx0, by0, bw, bh, L, lw, R, rw, srx0, sry0, kx, ky, out);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

}  // namespace vwb200
