// k12_ipfind.cu -- K12: ipfind's default path on the device (tools/ipfind.cc:253-401, --interest-operator iagd, sgrad):
// normalize, IntegralAutoGainDetector through detect_interest_points, remove_ip_near_nodata and SGradDescriptorGenerator
// through describe_interest_points.  Every float / double operation the reference performs is an explicitly rounded
// intrinsic in its order (no contraction); the host parts (tile lists, Gaussian taps, partition, crop boxes, cos / sin) are
// compiled with -ffp-contract=off.  Citations are file:line under the reference's src/vw/.
#include <cmath>
#include "common.cuh"

namespace vwb200 {
namespace {

constexpr int kBatchTiles = 64;                       // detection tiles whose scratch is live at once
constexpr size_t kBatchBytes = size_t(4) << 30;
constexpr int kDesc = 180;
constexpr double kDomain = 1073741824.0;              // 2^30, the support coordinates the contract covers
constexpr int kMaxTile = 16384;                       // 6 * 16384^2 < 2^31 candidate positions per tile

// OBALoG tables (InterestPoint/IntegralInterestOperator.cc:28-62), scales 0..7; the weights as SumBox's float
constexpr double kSigma[8] = {1.2, 1.5, 1.875, 2.34375, 2.9296875, 3.662109, 4.577636, 5.722046};
__constant__ int c_bw[8][6] = {{11,7,5,3,3,1}, {13,9,7,5,3,1}, {17,11,9,5,5,3}, {21,13,11,7,7,3},
                               {27,17,13,9,9,5}, {33,21,17,11,11,5}, {41,27,21,13,13,7}, {51,33,27,17,17,7}};
__constant__ int c_bh[8][6] = {{11,5,7,3,1,3}, {13,7,9,1,3,5}, {17,9,11,5,3,5}, {21,11,13,3,7,7},
                               {27,13,17,5,9,9}, {33,17,21,5,11,11}, {41,21,27,7,13,13}, {51,27,33,7,17,17}};
__constant__ int c_step[8] = {1, 1, 1, 2, 2, 3, 4, 5};    // Harris step int(float(SCALE_LOG_SIGMA[s]))
__constant__ float c_wt[8][6];                        // (float)SCALE_BOX_WEIGHT, set from the host table below
__constant__ float c_harris_w[81];                    // (float)(k[ix] * k[iy]), iy-major
const double kBoxWeight[8][6] = {
  {0.0006179999909,0.008283999749,0.008283999749,-0.03556599841,-0.05576400086,-0.05576400086},
  {0.0002659999882,0.004889999982,0.004889999982,-0.0221420005,-0.0488499999,-0.0221420005},
  {0.0002659424644,0.003207367443,0.003207367443,-0.001847865087,-0.022190776,-0.022190776},
  {0.000218920823,0.002005755751,0.002005755751,-0.01499466244,-0.0008247125278,-0.01499466244},
  {0.0001030362087,0.00137811946,0.00137811946,-0.009606413672,0.002226325845,-0.009606413672},
  {7.198028372e-05,0.0008259398524,0.0008259398524,-0.006072390568,-1.177469443e-06,-0.006072390568},
  {3.803569417e-05,0.0005251058097,0.0005251058097,-0.003885340628,0.0002823550512,-0.003885340628},
  {2.892054582e-05,0.0003287680581,0.0003287680581,-0.002447736656,-0.0002717150913,-0.002447736656}};

struct TileT { int x0, y0, w, h, num_ip; };

// ---- normalize (Image/AutoNormalize.h:76-86, ChannelNormalizeFunctor Image/Algorithms.h:106-126) -----------------------
// acc: [0] fkey min, [1] fkey max of the valid pixels, [2] non-finite pixels, [3] valid pixels
__global__ void k12_norm_stats_kernel(ImgF img, int has_nodata, float nd, unsigned* acc) {
  unsigned mn = 0xFFFFFFFFu, mx = 0, bad = 0, valid = 0;
  const long long n = (long long)img.w * img.h;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const float v = img.p[(ptrdiff_t)(k / img.w) * img.pitch + (k % img.w)];
    if (!isfinite(v)) { bad = 1; continue; }
    if (has_nodata && v == nd) continue;
    valid = 1;
    mn = min(mn, fkey(v)); mx = max(mx, fkey(v));
  }
  for (int o = 16; o > 0; o >>= 1) {
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    bad |= __shfl_xor_sync(0xffffffffu, bad, o); valid |= __shfl_xor_sync(0xffffffffu, valid, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (valid) { atomicMin(acc, mn); atomicMax(acc + 1, mx); atomicOr(acc + 3, 1u); }
    if (bad) atomicOr(acc + 2, 1u);
  }
}
// the reference's accumulator keeps the first of equal values, so a min / max of zero may be -0.0 there; (v - min) * ratio + 0
// is +0.0 or the same nonzero value either way, and max - min only decides between ratio 0 and the same ratio
__global__ void k12_norm_apply_kernel(ImgF img, int has_nodata, float nd, float mn, double ratio, float* out, ptrdiff_t op) {
  const long long n = (long long)img.w * img.h;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(k / img.w), x = (int)(k % img.w);
    const float v = img.p[(ptrdiff_t)y * img.pitch + x];
    out[(ptrdiff_t)y * op + x] = (has_nodata && v == nd) ? 0.0f : __double2float_rn(__dadd_rn(__dmul_rn((double)__fsub_rn(v, mn), ratio), 0.0));
  }
}

// ---- integral image (InterestPoint/IntegralImage.h:41-91): I[y][x] = ((v + I[y][x-1]) + I[y-1][x]) - I[y-1][x-1] -----
// One 1024-thread block per tile.  Thread t runs row b0 + t of a band of up to 1024 rows, skewed by t columns: at step d it
// computes column d - t.  Its `left` stays in a register; `up` is what thread t-1 computed the step before (a shuffle, or
// for lane 0 a shared slot written by the warp above), and `up-left` is the `up` it received one step earlier.  The band's
// first row reads the row above it from memory (zeros, or the previous band's last row).
__global__ void __launch_bounds__(1024) k12_integral_kernel(ImgF img, const TileT* tiles, float* scratch, size_t stride) {
  __shared__ float pub[2][32];
  const TileT T = tiles[blockIdx.x];
  float* I = scratch + stride * blockIdx.x;
  const int iw = T.w + 1, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int x = t; x < iw; x += 1024) I[x] = 0.0f;
  for (int y = 1 + t; y <= T.h; y += 1024) I[(size_t)y * iw] = 0.0f;
  __syncthreads();
  for (int b0 = 0; b0 < T.h; b0 += 1024) {
    const int nrows = min(1024, T.h - b0), r = b0 + t;
    const bool active = t < nrows;
    const float* src = img.p + (ptrdiff_t)(T.y0 + r) * img.pitch + T.x0;
    float* dst = I + (size_t)(r + 1) * iw + 1;
    const float* above = I + (size_t)b0 * iw;
    float left = 0.0f, cur = 0.0f, prev_up = 0.0f;
    const int steps = T.w + nrows - 1;
    for (int d = 0; d < steps; ++d) {
      float recv = __shfl_up_sync(0xffffffffu, cur, 1);
      if (lane == 0) recv = (warp > 0 && d > 0) ? pub[(d - 1) & 1][warp - 1] : 0.0f;
      const int x = d - t;
      float ncur = 0.0f;
      if (active && x >= 0 && x < T.w) {
        const float up = t == 0 ? above[x + 1] : recv, upleft = t == 0 ? above[x] : prev_up;
        ncur = __fsub_rn(__fadd_rn(__fadd_rn(__ldg(src + x), left), up), upleft);
        dst[x] = ncur;
        left = ncur;
      }
      prev_up = recv;
      cur = ncur;
      if (lane == 31) pub[d & 1][warp] = cur;
      __syncthreads();
    }
    __syncthreads();
  }
}

// ---- interest images: abs(box_filter(integral, scale s)) (BoxFilter.h:48-114, IntegralInterestOperator.h:95-114) ---------
// interest[tile][s][y][x]; keys[tile][s] = {min, max} float bits (the values are >= +0.0, so the bits order them)
__global__ void k12_interest_kernel(const TileT* tiles, const float* scratch, size_t stride, float* interest, size_t istride,
                                    unsigned* keys) {
  const int tile = blockIdx.z;
  const TileT T = tiles[tile];
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  const bool in = x < T.w && y < T.h;
  const float* I = scratch + stride * tile;
  const int iw = T.w + 1;
  for (int s = 0; s < 8; ++s) {
    float v = 0.0f;
    const int pb = c_bw[s][0] >> 1;
    if (in && x >= pb && x < T.w - pb && y >= pb && y < T.h - pb) {
      float result = 0.0f;
#pragma unroll
      for (int b = 0; b < 6; ++b) {
        const int bw = c_bw[s][b], bh = c_bh[s][b];
        const size_t o = (size_t)(y - (bh >> 1)) * iw + (x - (bw >> 1));
        float box = __fsub_rn(__fsub_rn(I[o], I[o + bw]), I[o + (size_t)bh * iw]);
        box = __fadd_rn(box, I[o + (size_t)bh * iw + bw]);
        result = __fadd_rn(result, __fmul_rn(c_wt[s][b], box));
      }
      v = fabsf(result);
    }
    unsigned mn = in ? __float_as_uint(v) : 0xFFFFFFFFu, mx = in ? __float_as_uint(v) : 0u;
    for (int o = 16; o > 0; o >>= 1) { mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o)); mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o)); }
    if ((threadIdx.x & 31) == 0 && mx >= mn) { atomicMin(keys + 2 * (tile * 8 + s), mn); atomicMax(keys + 2 * (tile * 8 + s) + 1, mx); }
    if (in) interest[istride * tile + (size_t)s * T.w * T.h + (size_t)y * T.w + x] = v;
  }
}

// ---- extrema, auto gain and Harris (IntegralDetector.cc:106-134, 300-343; IntegralInterestOperator.h:123-153) ----------
// flags[tile][m - 1][y][x] = 1 for a point of middle scale m that survives both thresholds
__global__ void k12_extrema_kernel(const TileT* tiles, const float* interest, size_t istride, const unsigned* keys, uint8_t* flags,
                                   size_t fstride) {
  const int tile = blockIdx.z / 6, m = 1 + blockIdx.z % 6;
  const TileT T = tiles[tile];
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= T.w || y >= T.h) return;
  const size_t plane = (size_t)T.w * T.h;
  uint8_t keep = 0;
  if (x >= 1 && y >= 1 && x < T.w - 1 && y < T.h - 1) {
    const float* mid = interest + istride * tile + plane * m;
    const float* lo = mid - plane, *hi = mid + plane;
    const size_t c = (size_t)y * T.w + x;
    const float v = mid[c];
    bool ext = v > lo[c] && v > hi[c];
    for (int dy = -1; dy <= 1 && ext; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        if (!dx && !dy) continue;
        const size_t q = c + (ptrdiff_t)dy * T.w + dx;
        if (!(v > lo[q] && v > mid[q] && v > hi[q])) { ext = false; break; }
      }
    if (ext) {
      keep = 2;                                      // an extremum (counted); 3 once it passes the thresholds
      const float imin = __uint_as_float(keys[2 * (tile * 8 + m)]), imax = __uint_as_float(keys[2 * (tile * 8 + m) + 1]);
      const float thr = __double2float_rn(__dadd_rn((double)imin, __dmul_rn(0.001, (double)__fsub_rn(imax, imin))));
      if (!(v < thr)) {
        const int step = c_step[m], offset = 4 * step;
        float sxx = 0.0f, syy = 0.0f, sxy = 0.0f;
        for (int jy = 0; jy < 9; ++jy) {
          const int yy = y - offset + jy * step;
          for (int jx = 0; jx < 9; ++jx) {
            const int xx = x - offset + jx * step;
            const size_t p = (size_t)yy * T.w + xx;
            const float Lx = __fsub_rn(mid[p - 1], mid[p + 1]), Ly = __fsub_rn(mid[p - T.w], mid[p + T.w]);
            const float w = c_harris_w[jy * 9 + jx];
            sxx = __fadd_rn(sxx, __fmul_rn(__fmul_rn(Lx, Lx), w));
            syy = __fadd_rn(syy, __fmul_rn(__fmul_rn(Ly, Ly), w));
            sxy = __fadd_rn(sxy, __fmul_rn(__fmul_rn(Lx, Ly), w));
          }
        }
        const float trace = __fadd_rn(sxx, syy), det = __fsub_rn(__fmul_rn(sxx, syy), __fmul_rn(sxy, sxy));
        if (__fdiv_rn(__fmul_rn(trace, trace), det) < 12.0f) keep = 3;
      }
    }
  }
  flags[fstride * tile + (size_t)(m - 1) * plane + (size_t)y * T.w + x] = keep;
}

// ---- compaction and cull (IntegralDetector.cc:354-367) -------------------------------------------------------------------
// One block per tile.  The flags are walked in (scale, row, column) order with a block-wide scan, so the candidate list
// is the reference's append order.  When it holds more than num_ip points, the num_ip-th largest interest is found by a
// radix select on its bits, and every point at or above it takes its rank in (descending interest, list position) --
// std::list::sort's stable order -- and lands there if the rank is below num_ip.
struct Cand { float interest; int pos; };            // pos: (m - 1) * w * h + y * w + x
__device__ __forceinline__ int block_excl_scan(int v, int* sh, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int s = v;
  for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += u; }
  if (lane == 31) sh[warp] = s;
  __syncthreads();
  if (warp == 0) {
    int w = lane < (blockDim.x >> 5) ? sh[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
    sh[32 + lane] = w;
  }
  __syncthreads();
  const int base = warp ? sh[32 + warp - 1] : 0;
  *total = sh[32 + (blockDim.x >> 5) - 1];
  __syncthreads();
  return base + s - v;
}

__global__ void __launch_bounds__(1024) k12_cull_kernel(const TileT* tiles, const uint8_t* flags, size_t fstride, const float* interest, size_t istride,
                                                        Cand* cand, size_t cstride, Cand* kept, size_t kstride, long long* counts) {
  __shared__ int sh[64];
  __shared__ unsigned hist[256];
  __shared__ unsigned s_prefix, s_need;
  const int tile = blockIdx.x;
  const TileT T = tiles[tile];
  const size_t plane = (size_t)T.w * T.h, n = 6 * plane;
  const uint8_t* f = flags + fstride * tile;
  Cand* c = cand + cstride * tile;
  const float* in = interest + istride * tile;
  int count = 0, extrema = 0;
  for (size_t base = 0; base < n; base += blockDim.x) {
    const size_t i = base + threadIdx.x;
    const uint8_t fl = i < n ? f[i] : 0;
    int total, etotal;
    const int o = block_excl_scan(fl == 3, sh, &total);
    block_excl_scan(fl >= 2, sh, &etotal);
    if (fl == 3) c[count + o] = Cand{in[plane + i], (int)i};   // interest of scale m = 1 + i / plane
    count += total;
    extrema += etotal;
  }
  __syncthreads();                                    // the last chunk's candidate writes, before any thread reads the list
  const int num_ip = T.num_ip;
  Cand* k = kept + kstride * tile;
  if (num_ip <= 0 || count <= num_ip) {
    for (int i = threadIdx.x; i < count; i += blockDim.x) k[i] = c[i];
    if (threadIdx.x == 0) { counts[3 * tile] = count; counts[3 * tile + 1] = extrema; counts[3 * tile + 2] = count; }
    return;
  }
  // radix select of the num_ip-th largest key (interests are >= +0.0: their bits order them)
  if (threadIdx.x == 0) { s_prefix = 0; s_need = num_ip; }
  __syncthreads();
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const unsigned prefix = s_prefix, mask = shift == 24 ? 0u : (0xFFFFFFFFu << (shift + 8));
    for (int i = threadIdx.x; i < count; i += blockDim.x) {
      const unsigned b = __float_as_uint(c[i].interest);
      if ((b & mask) == prefix) atomicAdd(&hist[(b >> shift) & 255], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned need = s_need;
      int d = 255;
      for (; d > 0; --d) { if (hist[d] >= need) break; need -= hist[d]; }
      s_prefix = prefix | ((unsigned)d << shift);
      s_need = need;
    }
    __syncthreads();
  }
  const unsigned kth = s_prefix;
  for (int i = threadIdx.x; i < count; i += blockDim.x) {
    const unsigned bi = __float_as_uint(c[i].interest);
    if (bi < kth) continue;
    int rank = 0;
    for (int j = 0; j < count && rank < num_ip; ++j) {
      const unsigned bj = __float_as_uint(c[j].interest);
      rank += (bj > bi) || (bj == bi && j < i);
    }
    if (rank < num_ip) k[rank] = c[i];
  }
  if (threadIdx.x == 0) { counts[3 * tile] = num_ip; counts[3 * tile + 1] = extrema; counts[3 * tile + 2] = count; }
}

// ---- remove_ip_near_nodata (InterestPoint/InterestPointUtils.h:45-82): one thread per point ----------------------------
__global__ void k12_nodata_kernel(ImgF raw, double nodata, int radius, const int2* ixy, int n, uint8_t* keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int px = ixy[i].x, py = ixy[i].y;
  uint8_t k = px >= radius && py >= radius && px < raw.w - radius && py < raw.h - radius;
  for (int y = py - radius; y <= py + radius && k; ++y)
    for (int x = px - radius; x <= px + radius; ++x)
      if ((double)raw.p[(ptrdiff_t)y * raw.pitch + x] == nodata) { k = 0; break; }
  keep[i] = k;
}

// ---- SGradDescriptorGenerator (InterestPoint/Descriptor.h:236-255, 414-471; Descriptor.cc:27-29): one warp per point ----
// get_support's AffineTransform reverse (ai, bi, ci, di, offset ox, oy), built on the host from the crop-relative point, and
// the tile's crop (x0, y0, cw, ch)
struct DescPt { double ai, bi, ci, di, ox, oy; int x0, y0, cw, ch; };
constexpr int kDescWarps = 3;                      // 3 x 15.2 KB of static shared memory per block
__constant__ int c_strt[5] = {17, 15, 9, 6, 0}, c_bsz[5] = {2, 4, 8, 10, 14}, c_bhf[5] = {1, 2, 4, 5, 7};
__constant__ float c_inv_bh2[5];                       // 1 / float(box_half^2), set from the host

__device__ __forceinline__ int vw_floor_d(double v) {
  if (v < 0) { const int iv = __double2int_rz(v); return (double)iv == v ? iv : iv - 1; }
  return __double2int_rz(v);
}
__device__ __forceinline__ float crop_px(ImgF img, const DescPt& p, int i, int j) {
  if (i < 0 || j < 0 || i >= p.cw || j >= p.ch) return 0.0f;
  const int x = p.x0 + i, y = p.y0 + j;
  if (x < 0 || y < 0 || x >= img.w || y >= img.h) return 0.0f;
  return __ldg(img.p + (ptrdiff_t)y * img.pitch + x);
}
// BilinearInterpolation (Image/Interpolation.h:76-110), real_type float, zero edge, as K8's
__device__ __forceinline__ float bilinear_crop(ImgF img, const DescPt& p, double i, double j) {
  const int x = vw_floor_d(i), y = vw_floor_d(j);
  if ((double)x == i && (double)y == j) return crop_px(img, p, x, y);
  const float nx = __fsub_rn(__double2float_rn(i), __int2float_rn(x)), ny = __fsub_rn(__double2float_rn(j), __int2float_rn(y));
  const float n1mx = __fsub_rn(1.0f, nx), n1my = __fsub_rn(1.0f, ny);
  float r = __fmul_rn(crop_px(img, p, x, y), n1mx);
  r = __fadd_rn(r, __fmul_rn(crop_px(img, p, x + 1, y), nx));
  r = __fmul_rn(r, n1my);
  float row = __fmul_rn(crop_px(img, p, x, y + 1), n1mx);
  row = __fadd_rn(row, __fmul_rn(crop_px(img, p, x + 1, y + 1), nx));
  return __fadd_rn(r, __fmul_rn(row, ny));
}

__global__ void __launch_bounds__(32 * kDescWarps) k12_describe_kernel(ImgF img, const DescPt* pts, int n, float* desc) {
  __shared__ float s_sup[kDescWarps][42 * 42];
  __shared__ float s_int[kDescWarps][43 * 43];
  __shared__ float s_out[kDescWarps][kDesc];
  const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5, i = blockIdx.x * kDescWarps + wl;
  if (i >= n) return;
  const DescPt p = pts[i];
  float* sup = s_sup[wl];
  float* I = s_int[wl];
  const double ai = p.ai, bi = p.bi, ci = p.ci, di = p.di, ox = p.ox, oy = p.oy;
  for (int k = lane; k < 42 * 42; k += 32) {
    const double px = __dsub_rn((double)(k % 42), ox), py = __dsub_rn((double)(k / 42), oy);
    const double rx = __dadd_rn(__dmul_rn(ai, px), __dmul_rn(bi, py)), ry = __dadd_rn(__dmul_rn(ci, px), __dmul_rn(di, py));
    sup[k] = bilinear_crop(img, p, rx, ry);
  }
  // IntegralImage of the support, 43 x 43: lane l runs row l (then l + 32), skewed by l columns
  for (int k = lane; k < 43; k += 32) { I[k] = 0.0f; I[k * 43] = 0.0f; }
  __syncwarp();
  for (int r0 = 0; r0 < 42; r0 += 32) {
    const int r = r0 + lane, rows = min(32, 42 - r0);
    float left = 0.0f;
    for (int step = 0; step < 42 + rows - 1; ++step) {
      const int x = step - lane;
      if (lane < rows && x >= 0 && x < 42) {
        const float* q = I + (r + 1) * 43 + (x + 1);
        left = __fsub_rn(__fadd_rn(__fadd_rn(sup[r * 42 + x], left), q[-43]), q[-44]);
        I[(r + 1) * 43 + (x + 1)] = left;
      }
      __syncwarp();
    }
  }
  // 5 scales x 9 quads x 4 gradients
  for (int o = lane; o < kDesc; o += 32) {
    const int s = o / 36, qi = (o % 36) / 4, g = o % 4, ii = qi / 3, jj = qi % 3, bh = c_bhf[s];
    const int tx = c_strt[s] + ii * c_bsz[s], ty = c_strt[s] + jj * c_bsz[s];
    float q[4];
    const int x0s[4] = {tx, tx + bh, tx, tx + bh}, y0s[4] = {ty, ty, ty + bh, ty + bh};
#pragma unroll
    for (int k = 0; k < 4; ++k) {                    // IntegralBlock (InterestPoint/IntegralImage.cc:27-53)
      const int x0 = x0s[k], y0 = y0s[k], x1 = x0 + bh, y1 = y0 + bh;
      float v = I[y0 * 43 + x0];
      v = __fadd_rn(v, I[y1 * 43 + x1]);
      v = __fsub_rn(v, I[y1 * 43 + x0]);
      v = __fsub_rn(v, I[y0 * 43 + x1]);
      q[k] = v;
    }
    const float inv_bh2 = c_inv_bh2[s];
    const float gv = g == 0 ? __fsub_rn(q[0], q[2]) : g == 1 ? __fsub_rn(q[1], q[3]) : g == 2 ? __fsub_rn(q[0], q[1]) : __fsub_rn(q[2], q[3]);
    s_out[wl][o] = __fmul_rn(gv, inv_bh2);
  }
  __syncwarp();
  float inv = 0.0f;
  if (lane == 0) {
    float sqr = 0.0f;
    for (int o = 0; o < kDesc; ++o) sqr = __fadd_rn(sqr, __fmul_rn(s_out[wl][o], s_out[wl][o]));
    // the unqualified sqrt is ::sqrt(double) (vw/Math/Functions.h:167 over <cmath>), so 1.0f / sqrt(...) is a double quotient
    inv = __double2float_rn(__ddiv_rn(1.0, __dsqrt_rn((double)sqr)));
    if (!(fabsf(inv) >= 1.17549435e-38f && fabsf(inv) <= 3.40282347e38f)) inv = 0.0f;   // !std::isnormal
  }
  inv = __shfl_sync(0xffffffffu, inv, 0);
  for (int o = lane; o < kDesc; o += 32) desc[(size_t)i * kDesc + o] = __fmul_rn(s_out[wl][o], inv);
}

// ---- host side ---------------------------------------------------------------------------------------------------------
thread_local vwb200_ipfind_stats t_stats = {0, 0, 0, 0, 0};

void gaussian_taps(double* k) {                      // generate_gaussian_kernel(k, 2, 9) (Image/Filter.tcc:37-80), ::erf
  const int center = 4;
  const double z = 1 / (std::sqrt(2.0) * 2.0);
  double sum = 0.0, tap;
  for (int i = 1; i <= center; ++i) {
    tap = ::erf((i + 0.5) * z) - ::erf((i - 0.5) * z);
    sum += tap;
    k[center + i] = k[center - i] = tap;
  }
  sum *= 2.0;
  tap = ::erf(0.5 * z) - ::erf(-0.5 * z);
  sum += tap;
  k[center] = tap;
  const double norm = 1.0 / sum;
  for (int i = 0; i < 9; ++i) k[i] *= norm;
}

int upload_tables(cudaStream_t st) {
  double k[9];
  gaussian_taps(k);
  float hw[81], wt[8][6];
  for (int iy = 0; iy < 9; ++iy)
    for (int ix = 0; ix < 9; ++ix) hw[iy * 9 + ix] = (float)(k[ix] * k[iy]);
  for (int s = 0; s < 8; ++s)
    for (int b = 0; b < 6; ++b) wt[s][b] = (float)kBoxWeight[s][b];
  VWB_CUDA(cudaMemcpyToSymbolAsync(c_harris_w, hw, sizeof hw, 0, cudaMemcpyHostToDevice, st));
  VWB_CUDA(cudaMemcpyToSymbolAsync(c_wt, wt, sizeof wt, 0, cudaMemcpyHostToDevice, st));
  return VWB200_OK;
}
int upload_sgrad_tables(cudaStream_t st) {
  const int bh[5] = {1, 2, 4, 5, 7};
  float inv[5];
  for (int s = 0; s < 5; ++s) inv[s] = 1 / float(bh[s] * bh[s]);
  VWB_CUDA(cudaMemcpyToSymbolAsync(c_inv_bh2, inv, sizeof inv, 0, cudaMemcpyHostToDevice, st));
  return VWB200_OK;
}

bool bad_raster(const char* what, const void* p, int w, int h, ptrdiff_t pitch) {
  if (w < 0 || h < 0 || (w > 0 && h > 0 && (!p || pitch < w))) {
    set_error("%s: bad raster (w %d, h %d, pitch %td)", what, w, h, pitch);
    return true;
  }
  return false;
}

// the tiles of subdivide_bbox (Image/AlgorithmFunctions.cc:27-80) in raster order
std::vector<TileT> make_tiles(int w, int h, int ts, int ip_per_tile) {
  std::vector<TileT> v;
  for (int y0 = 0; y0 < h; y0 += ts)
    for (int x0 = 0; x0 < w; x0 += ts) {
      TileT t{x0, y0, std::min(ts, w - x0), std::min(ts, h - y0), 0};
      if (ip_per_tile > 0) {                           // InterestDetectionQueue::get_next_task (DetectorBase.h:276-290)
        const double fraction = (double)t.w * t.h / ((double)ts * ts);
        int num_ip = (int)std::ceil(fraction * (double)ip_per_tile);
        t.num_ip = std::max(1, std::min(num_ip, ip_per_tile));
      }
      v.push_back(t);
    }
  return v;
}

// the support's AffineTransform (Descriptor.h:262-276) restated on the host for the crop boxes
struct Affine { double ai, bi, ci, di, x, y; };
Affine support_tx(float x, float y, float scale, double c, double s) {
  const float half = ((float)(42 - 1)) / 2.0f, scaling = 1.0f / scale;
  const double a = scaling * c, b = -scaling * s, cc = scaling * s, d = scaling * c;
  Affine t;
  t.x = scaling * (s * y - c * x) + half;
  t.y = -scaling * (s * x + c * y) + half;
  const double det = a * d - b * cc;
  t.ai = d / det; t.bi = -b / det; t.ci = -cc / det; t.di = a / det;
  return t;
}

}  // namespace

extern "C" {

int vwb200_ipfind_gaussian_taps(double* k9) {
  if (!k9) return VWB200_EARG;
  gaussian_taps(k9);
  return VWB200_OK;
}

int vwb200_last_ipfind_stats(vwb200_ipfind_stats* out) { if (!out) return VWB200_EARG; *out = t_stats; return VWB200_OK; }

int vwb200_ipfind_normalize(const float* in, int w, int h, ptrdiff_t pitch, int has_nodata, double nodata, float* out, ptrdiff_t out_pitch,
                            int on_device, void* stream) {
  const char* what = "vwb200_ipfind_normalize";
  if (bad_raster(what, in, w, h, pitch) || bad_raster(what, out, w, h, out_pitch)) return VWB200_EARG;
  if (rasters_overlap(in, w, h, pitch, out, w, h, out_pitch, 4, 4) && !(in == out && pitch == out_pitch)) {
    set_error("%s: out overlaps in (only out == in, with the same pitch, is allowed)", what);
    return VWB200_EARG;
  }
  VWB_TRY(ensure_device());
  if ((long long)w * h == 0) return VWB200_OK;
  AbiCall c;
  VWB_TRY(c.open(stream, on_device));
  const float* din; ptrdiff_t dp;
  VWB_TRY(c.in(in, w, h, pitch, on_device, &din, &dp));
  float* dout; ptrdiff_t dop;
  VWB_TRY(c.out(out, w, h, out_pitch, on_device, &dout, &dop));
  unsigned* acc;
  VWB_TRY(c.ar.alloc(&acc, 4));
  const unsigned init[4] = {0xFFFFFFFFu, 0u, 0u, 0u};
  VWB_CUDA(cudaMemcpyAsync(acc, init, sizeof init, cudaMemcpyHostToDevice, c.st));
  const ImgF img{din, w, h, dp};
  const float nd = (float)nodata;
  k12_norm_stats_kernel<<<2 * kNumSMs, 256, 0, c.st>>>(img, has_nodata, nd, acc);
  VWB_LAUNCH_CHECK();
  unsigned h_acc[4];
  VWB_CUDA(cudaMemcpyAsync(h_acc, acc, sizeof h_acc, cudaMemcpyDeviceToHost, c.st));
  VWB_CUDA(cudaStreamSynchronize(c.st));
  if (h_acc[2]) { set_error("%s: NaN or inf in the image (undefined in the reference)", what); return VWB200_EARG; }
  if (!h_acc[3]) { set_error("%s: MinMaxAccumulator: no valid samples", what); return VWB200_EARG; }
  const float mn = kfloat(h_acc[0]), mx = kfloat(h_acc[1]);
  const double ratio = mx == mn ? 0.0 : (1.0f - 0.0f) / (double)(mx - mn);   // ChannelNormalizeFunctor's, on the host
  k12_norm_apply_kernel<<<4 * kNumSMs, 256, 0, c.st>>>(img, has_nodata, nd, mn, ratio, dout, dop);
  VWB_LAUNCH_CHECK();
  return c.finish();
}

int vwb200_ipfind_detect(const float* image, int w, int h, ptrdiff_t pitch, int tile_size, int ip_per_tile, vwb200_ip_point* out,
                         long long cap, long long* n, int on_device, void* stream) {
  const char* what = "vwb200_ipfind_detect";
  if (bad_raster(what, image, w, h, pitch)) return VWB200_EARG;
  if (!n || cap < 0 || (cap > 0 && !out) || ip_per_tile < 0) { set_error("%s: bad output or ip_per_tile", what); return VWB200_EARG; }
  if (tile_size > kMaxTile) {
    // Cand.pos indexes 6 * tile^2 positions as int32, and the grids' y dimension counts tile / 8 rows
    set_error("%s: tile_size %d is above %d, the largest tile the kernels index", what, tile_size, kMaxTile);
    return VWB200_EARG;
  }
  VWB_TRY(ensure_device());
  t_stats = vwb200_ipfind_stats{0, 0, 0, 0, 0};
  *n = 0;
  if ((long long)w * h == 0) return VWB200_OK;
  const int ts = std::max(1024, tile_size);       // DetectorBase.h:307-310
  const std::vector<TileT> tiles = make_tiles(w, h, ts, ip_per_tile);
  AbiCall c;
  VWB_TRY(c.open(stream, on_device));
  const float* din; ptrdiff_t dp;
  VWB_TRY(c.in(image, w, h, pitch, on_device, &din, &dp));
  VWB_TRY(upload_tables(c.st));
  const int tw_max = std::min(ts, w), th_max = std::min(ts, h);
  // about 54 bytes of scratch per tile pixel: batches of up to 64 tiles within kBatchBytes
  const size_t per_tile = (size_t)(tw_max + 1) * (th_max + 1) * 54;
  const int nb = (int)std::max<size_t>(1, std::min<size_t>({tiles.size(), (size_t)kBatchTiles, kBatchBytes / per_tile}));
  const size_t stride = (size_t)(tw_max + 1) * (th_max + 1), plane = (size_t)tw_max * th_max, istride = 8 * plane;
  const size_t cstride = 6 * (size_t)((tw_max + 1) / 2) * ((th_max + 1) / 2) + 1;
  size_t kstride = 0;
  for (const TileT& t : tiles) kstride = std::max<size_t>(kstride, t.num_ip > 0 ? (size_t)t.num_ip : cstride);
  kstride = std::min(kstride, cstride);
  TileT* dt; float* integ; float* inter; unsigned* keys; uint8_t* flags; Cand* cand; Cand* kept; long long* counts;
  VWB_TRY(c.ar.alloc(&dt, tiles.size()));
  VWB_TRY(c.ar.alloc(&integ, stride * nb));
  VWB_TRY(c.ar.alloc(&inter, istride * nb));
  VWB_TRY(c.ar.alloc(&keys, 16 * (size_t)nb));
  VWB_TRY(c.ar.alloc(&flags, 6 * plane * nb));
  VWB_TRY(c.ar.alloc(&cand, cstride * nb));
  VWB_TRY(c.ar.alloc(&kept, kstride * nb));
  VWB_TRY(c.ar.alloc(&counts, 3 * (size_t)nb));
  VWB_CUDA(cudaMemcpyAsync(dt, tiles.data(), tiles.size() * sizeof(TileT), cudaMemcpyHostToDevice, c.st));
  std::vector<unsigned> kinit(16 * (size_t)nb);
  for (size_t i = 0; i < kinit.size(); i += 2) { kinit[i] = 0xFFFFFFFFu; kinit[i + 1] = 0u; }
  std::vector<long long> hcounts(3 * (size_t)nb);
  std::vector<Cand> hkept;
  const ImgF img{din, w, h, dp};
  long long total = 0;
  for (size_t t0 = 0; t0 < tiles.size(); t0 += nb) {
    const int bt = (int)std::min<size_t>(nb, tiles.size() - t0);
    VWB_CUDA(cudaMemcpyAsync(keys, kinit.data(), kinit.size() * sizeof(unsigned), cudaMemcpyHostToDevice, c.st));
    k12_integral_kernel<<<bt, 1024, 0, c.st>>>(img, dt + t0, integ, stride);
    VWB_LAUNCH_CHECK();
    const dim3 g((tw_max + 31) / 32, (th_max + 7) / 8, bt);
    k12_interest_kernel<<<g, 256, 0, c.st>>>(dt + t0, integ, stride, inter, istride, keys);
    VWB_LAUNCH_CHECK();
    const dim3 g6((tw_max + 31) / 32, (th_max + 7) / 8, bt * 6);
    k12_extrema_kernel<<<g6, 256, 0, c.st>>>(dt + t0, inter, istride, keys, flags, 6 * plane);
    VWB_LAUNCH_CHECK();
    k12_cull_kernel<<<bt, 1024, 0, c.st>>>(dt + t0, flags, 6 * plane, inter, istride, cand, cstride, kept, kstride, counts);
    VWB_LAUNCH_CHECK();
    VWB_CUDA(cudaMemcpyAsync(hcounts.data(), counts, 3 * bt * sizeof(long long), cudaMemcpyDeviceToHost, c.st));
    VWB_CUDA(cudaStreamSynchronize(c.st));
    hkept.resize(kstride * bt);
    for (int b = 0; b < bt; ++b)                     // only each tile's kept prefix
      if (hcounts[3 * b])
        VWB_CUDA(cudaMemcpyAsync(hkept.data() + kstride * b, kept + kstride * b, hcounts[3 * b] * sizeof(Cand), cudaMemcpyDeviceToHost, c.st));
    VWB_CUDA(cudaStreamSynchronize(c.st));
    for (int b = 0; b < bt; ++b) {
      const TileT& T = tiles[t0 + b];
      const long long kc = hcounts[3 * b];
      t_stats.tiles++;
      t_stats.extrema += hcounts[3 * b + 1];
      t_stats.kept += hcounts[3 * b + 2];
      if (hcounts[3 * b + 2] > kc) t_stats.culled_tiles++;
      for (long long q = 0; q < kc; ++q, ++total) {
        if (total >= cap) continue;
        const Cand& cd = hkept[kstride * b + q];
        const int m = 1 + (int)(cd.pos / ((long long)T.w * T.h)), rem = (int)(cd.pos % ((long long)T.w * T.h));
        const int x = rem % T.w, y = rem / T.w;
        // InterestPoint(c+1, r+1, float(SCALE_LOG_SIGMA[m]), interest), then the tile origin (DetectorBase.h:231-236)
        out[total] = vwb200_ip_point{(float)x + (float)T.x0, (float)y + (float)T.y0, x + T.x0, y + T.y0, (float)kSigma[m], cd.interest, 0.0f};
      }
    }
  }
  *n = total;
  VWB_TRY(c.finish());
  if (total > cap) { set_error("%s: %lld points do not fit in cap %lld", what, total, cap); return VWB200_EARG; }
  return VWB200_OK;
}

int vwb200_ipfind_remove_near_nodata(const float* raw, int w, int h, ptrdiff_t pitch, double nodata, int radius, vwb200_ip_point* pts,
                                     long long* n, int on_device, void* stream) {
  const char* what = "vwb200_ipfind_remove_near_nodata";
  if (bad_raster(what, raw, w, h, pitch)) return VWB200_EARG;
  if (!n || *n < 0 || (*n > 0 && !pts) || radius < 0 || *n > INT32_MAX) { set_error("%s: bad point list or radius", what); return VWB200_EARG; }
  VWB_TRY(ensure_device());
  const int np = (int)*n;
  if (np == 0) return VWB200_OK;
  if ((long long)w * h == 0) { *n = 0; return VWB200_OK; }
  AbiCall c;
  VWB_TRY(c.open(stream, on_device));
  const float* din; ptrdiff_t dp;
  VWB_TRY(c.in(raw, w, h, pitch, on_device, &din, &dp));
  std::vector<int2> ixy(np);
  for (int i = 0; i < np; ++i) ixy[i] = make_int2(pts[i].ix, pts[i].iy);
  int2* dxy; uint8_t* dkeep;
  VWB_TRY(c.ar.alloc(&dxy, np));
  VWB_TRY(c.ar.alloc(&dkeep, np));
  VWB_CUDA(cudaMemcpyAsync(dxy, ixy.data(), np * sizeof(int2), cudaMemcpyHostToDevice, c.st));
  k12_nodata_kernel<<<(np + 255) / 256, 256, 0, c.st>>>(ImgF{din, w, h, dp}, nodata, radius, dxy, np, dkeep);
  VWB_LAUNCH_CHECK();
  std::vector<uint8_t> keep(np);
  VWB_CUDA(cudaMemcpyAsync(keep.data(), dkeep, np, cudaMemcpyDeviceToHost, c.st));
  VWB_TRY(c.finish());
  long long o = 0;
  for (int i = 0; i < np; ++i)
    if (keep[i]) pts[o++] = pts[i];
  *n = o;
  return VWB200_OK;
}

int vwb200_ipfind_describe(const float* image, int w, int h, ptrdiff_t pitch, int tile_size, vwb200_ip_point* pts, long long n,
                           float* desc, int on_device, void* stream) {
  const char* what = "vwb200_ipfind_describe";
  if (bad_raster(what, image, w, h, pitch)) return VWB200_EARG;
  if (n < 0 || n > INT32_MAX || (n > 0 && (!pts || !desc))) { set_error("%s: bad point list", what); return VWB200_EARG; }
  for (long long i = 0; i < n; ++i)
    if (!(std::isfinite(pts[i].x) && std::isfinite(pts[i].y) && std::isfinite(pts[i].orientation) && std::isfinite(pts[i].scale) &&
          pts[i].scale > 0)) {
      set_error("%s: point %lld has a non-finite coordinate or orientation or a scale <= 0", what, i);
      return VWB200_EARG;
    }
  // the reference converts the supports' reverse_bbox to int32, and its bilinear reads floor the support coordinates again:
  // beyond 2^30 (K8's domain) that is undefined, so such points (a huge scale or a far coordinate) are refused up front
  for (long long i = 0; i < n; ++i) {
    const Affine t = support_tx(pts[i].x, pts[i].y, pts[i].scale, ::cos((double)-pts[i].orientation), ::sin((double)-pts[i].orientation));
    for (int k = 0; k < 4; ++k) {
      const double px = (k & 1 ? 41 : 0) - t.x, py = (k & 2 ? 41 : 0) - t.y;
      const double rx = t.ai * px + t.bi * py, ry = t.ci * px + t.di * py;
      if (!(std::fabs(rx) < kDomain && std::fabs(ry) < kDomain)) {
        set_error("%s: the support of point %lld reaches beyond 2^30 (a huge scale or coordinate)", what, i);
        return VWB200_EARG;
      }
    }
  }
  VWB_TRY(ensure_device());
  t_stats.described = 0;
  if (n == 0) return VWB200_OK;
  const int ts = std::max(1024, tile_size);       // Descriptor.h:332-336
  const std::vector<TileT> tiles = make_tiles(w, h, ts, 0);
  std::vector<DescPt> dp(n);
  auto in_tile = [](const vwb200_ip_point& p, const TileT& T) {   // IsInBBox: Vector2i(ip.x, ip.y)
    const int x = (int)p.x, y = (int)p.y;
    return x >= T.x0 && y >= T.y0 && x < T.x0 + T.w && y < T.y0 + T.h;
  };
  long long first = 0;
  for (const TileT& T : tiles) {
    // std::partition over a std::list: libstdc++'s bidirectional swapping scan
    long long f = first, l = n;
    for (;;) {
      while (f != l && in_tile(pts[f], T)) ++f;
      if (f == l) break;
      --l;
      while (f != l && !in_tile(pts[l], T)) --l;
      if (f == l) break;
      std::swap(pts[f], pts[l]);
      ++f;
    }
    const long long s0 = first, s1 = f;
    first = f;
    if (s0 == s1) continue;
    // InterestPointDescriptionTask (Descriptor.h:259-301): the union of the supports' reverse_bbox, expanded by 1
    int bx0 = 0, by0 = 0, bx1 = 0, by1 = 0;
    for (long long q = s0; q < s1; ++q) {
      const Affine t = support_tx(pts[q].x, pts[q].y, pts[q].scale, ::cos((double)-pts[q].orientation), ::sin((double)-pts[q].orientation));
      double mnx = 0, mny = 0, mxx = 0, mxy = 0;
      for (int k = 0; k < 4; ++k) {
        const double px = (k & 1 ? 41 : 0) - t.x, py = (k & 2 ? 41 : 0) - t.y;
        const double rx = t.ai * px + t.bi * py, ry = t.ci * px + t.di * py;
        if (!k) { mnx = mxx = rx; mny = mxy = ry; continue; }
        if (rx > mxx) mxx = rx;
        if (rx < mnx) mnx = rx;
        if (ry > mxy) mxy = ry;
        if (ry < mny) mny = ry;
      }
      const int ix0 = (int)std::floor(mnx), iy0 = (int)std::floor(mny), ix1 = (int)std::floor(mxx) + 1, iy1 = (int)std::floor(mxy) + 1;
      if (q == s0) { bx0 = ix0; by0 = iy0; bx1 = ix1; by1 = iy1; continue; }
      bx0 = std::min(bx0, ix0); by0 = std::min(by0, iy0); bx1 = std::max(bx1, ix1); by1 = std::max(by1, iy1);
    }
    bx0 -= 1; by0 -= 1; bx1 += 1; by1 += 1;
    for (long long q = s0; q < s1; ++q) {
      pts[q].x -= bx0;
      pts[q].y -= by0;
      // get_support (Descriptor.h:242-254) on the crop-relative point
      const Affine t = support_tx(pts[q].x, pts[q].y, pts[q].scale, ::cos((double)-pts[q].orientation), ::sin((double)-pts[q].orientation));
      dp[q] = DescPt{t.ai, t.bi, t.ci, t.di, t.x, t.y, bx0, by0, bx1 - bx0, by1 - by0};
      pts[q].x += bx0;
      pts[q].y += by0;
    }
  }
  if (first != n) { set_error("%s: %lld points lie outside the image's tiles", what, n - first); return VWB200_EARG; }
  AbiCall c;
  VWB_TRY(c.open(stream, on_device));
  const float* din; ptrdiff_t dpitch;
  VWB_TRY(c.in(image, w, h, pitch, on_device, &din, &dpitch));
  VWB_TRY(upload_sgrad_tables(c.st));
  DescPt* d_pts; float* d_desc;
  VWB_TRY(c.ar.alloc(&d_pts, n));
  VWB_TRY(c.ar.alloc(&d_desc, (size_t)n * kDesc));
  VWB_CUDA(cudaMemcpyAsync(d_pts, dp.data(), n * sizeof(DescPt), cudaMemcpyHostToDevice, c.st));
  k12_describe_kernel<<<(unsigned)((n + kDescWarps - 1) / kDescWarps), 32 * kDescWarps, 0, c.st>>>(ImgF{din, w, h, dpitch}, d_pts, (int)n, d_desc);
  VWB_LAUNCH_CHECK();
  VWB_CUDA(cudaMemcpyAsync(desc, d_desc, (size_t)n * kDesc * sizeof(float), cudaMemcpyDeviceToHost, c.st));
  VWB_TRY(c.finish());
  t_stats.described = n;
  return VWB200_OK;
}

}  // extern "C"

}  // namespace vwb200
