// k9_inpaint.cu -- K9: fill_holes_grass(img, hole_fill_len) of Image/InpaintView.h:239-311 on integer (PixelMask<Vector2i>)
// and float (PixelMask<Vector2f>) disparities, rasterised over an output window.
//
// The tile is the window grown by len and cropped to the image.  Its holes are the 8-connected components of its invalid
// pixels, labelled by union-find; a hole is filled when it passes the two culls (pixel count <= len*len, bounding box at most
// len wide and tall) and the edge test of InpaintTask (InpaintView.h:76-80), and its bounding box meets the window (a hole
// outside it changes no output pixel).  Each filled hole is then one independent job, run by one worker (a warp for small
// holes, a CTA for large ones) that keeps the hole's bbox.expand(1) crop in shared memory, or in per-CTA global scratch
// beyond the shared-memory limit:
//   1. distance: the city-block distance to the nearest non-hole pixel (what grassfire computes), by min relaxation;
//   2. levels:   level(p) = 1 + the largest level of p's 8-neighbours in the hole that come before p in the processing order
//                (distance, then column, then row); two pixels of one level are never adjacent;
//   3. sweeps:   10 * max_distance^2 Gauss-Seidel sweeps, each as `levels` synchronised steps: a step updates every pixel of
//                its level at once, so each pixel reads its predecessors' new values and its successors' old ones, exactly
//                as the reference's in-place sequential loop does.
// Every product and sum is an explicitly rounded intrinsic in the reference's order: the product in double, the += of the
// float accumulator through double (InpaintView.h:119-137).
#include <climits>

#include "common.cuh"

namespace vwb200 {
namespace {

constexpr int kCtaThreads = 256;
constexpr int kWarpArea = 448;                 // holes whose bbox.expand(1) has at most this many pixels go to a warp
constexpr int kWarpsPerCta = 8;
constexpr int kBytesPerPx = 16;                // two 32-bit children, the distance and the level
constexpr int kSmemLimit = 227 * 1024;         // sm_90a opt-in maximum per CTA

template <class T> struct Px;
template <> struct Px<vwb200_dispi> {
  typedef int32_t C;
  __device__ static bool invalid(const vwb200_dispi& p) { return p.valid == 0; }
  __device__ static double wide(int32_t v) { return (double)v; }
  __device__ static int32_t store(float s) { return __float2int_rz(s); }   // float -> int32 conversion truncates
  __device__ static vwb200_dispi make(int32_t a, int32_t b) { vwb200_dispi p; p.dx = a; p.dy = b; p.valid = 1; return p; }
};
template <> struct Px<DispF> {
  typedef float C;
  __device__ static bool invalid(const DispF& p) { return p.valid == 0.0f; }
  __device__ static double wide(float v) { return (double)v; }
  __device__ static float store(float s) { return s; }
  __device__ static DispF make(float a, float b) { DispF p; p.dx = a; p.dy = b; p.valid = 1.0f; return p; }
};

// ---- labelling ----------------------------------------------------------------------------------------------------------
// parent[i] over the tile's tw x th pixels: -1 for a valid pixel, else a union-find forest whose roots are the smallest index
// of their component.  After k9_claim_kernel a root holds -2 - (its hole's index).
__device__ __forceinline__ int root_of(const int* parent, int i) { int p; while ((p = parent[i]) != i) i = p; return i; }
__device__ void unite(int* parent, int a, int b) {
  while (true) {
    a = root_of(parent, a); b = root_of(parent, b);
    if (a == b) return;
    if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(parent + a, b);
    if (old == a) return;
    a = old;
  }
}

struct HoleTile { int x0, y0, w, h; };             // the tile in image coordinates

template <class T>
__global__ void k9_label_init_kernel(const T* __restrict__ in, ptrdiff_t ip, HoleTile t, int* __restrict__ parent) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= t.w || y >= t.h) return;
  const int i = y * t.w + x;
  parent[i] = Px<T>::invalid(in[(ptrdiff_t)(t.y0 + y) * ip + t.x0 + x]) ? i : -1;
}
__global__ void k9_union_kernel(HoleTile t, int* __restrict__ parent) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= t.w || y >= t.h) return;
  const int w = t.w, i = y * w + x;
  if (parent[i] < 0) return;
  if (x > 0 && parent[i - 1] >= 0) unite(parent, i, i - 1);
  if (y > 0) {
    if (parent[i - w] >= 0) unite(parent, i, i - w);
    if (x > 0 && parent[i - w - 1] >= 0) unite(parent, i, i - w - 1);
    if (x < w - 1 && parent[i - w + 1] >= 0) unite(parent, i, i - w + 1);
  }
}
__global__ void k9_flatten_kernel(int n, int* __restrict__ parent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || parent[i] < 0) return;
  parent[i] = root_of(parent, i);
}
// Hole records: size, then the half-open bbox x0, y0, x1, y1 in tile coordinates.
struct Hole { int size, x0, y0, x1, y1; };
__global__ void k9_claim_kernel(int n, int* __restrict__ parent, Hole* __restrict__ holes, int* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || parent[i] != i) return;
  const int id = atomicAdd(count, 1);
  Hole h; h.size = 0; h.x0 = h.y0 = INT_MAX; h.x1 = h.y1 = INT_MIN;
  holes[id] = h;
  parent[i] = -2 - id;
}
__device__ __forceinline__ int hole_of(const int* parent, int i) {
  const int p = parent[i];
  if (p == -1) return -1;
  return p <= -2 ? -2 - p : -2 - parent[p];
}
__global__ void k9_stats_kernel(HoleTile t, const int* __restrict__ parent, Hole* __restrict__ holes) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= t.w || y >= t.h) return;
  const int id = hole_of(parent, y * t.w + x);
  if (id < 0) return;
  Hole* h = holes + id;
  atomicAdd(&h->size, 1);
  atomicMin(&h->x0, x); atomicMin(&h->y0, y);
  atomicMax(&h->x1, x + 1); atomicMax(&h->y1, y + 1);
}
// the culls, the edge test and the window test; survivors go to the warp list (0) or the CTA list (1) with their crop area
struct Select { int count[2]; int max_area[2]; };
__global__ void k9_select_kernel(const int* __restrict__ nholes, const Hole* __restrict__ holes, HoleTile t, int len, int area_limit,
                                 int wx0, int wy0, int wx1, int wy1, int* __restrict__ lists, int cap, Select* __restrict__ sel) {
  const int n = *nholes;
  for (int id = blockIdx.x * blockDim.x + threadIdx.x; id < n; id += gridDim.x * blockDim.x) {
    const Hole h = holes[id];
    if (area_limit > 0 && h.size > area_limit) continue;                        // BlobIndex.h:445-453
    if (h.x1 - h.x0 > len || h.y1 - h.y0 > len) continue;                       // wipe_big_blobs, :457-477
    if (h.x0 - 1 < 0 || h.y0 - 1 < 0 || h.x1 + 1 >= t.w || h.y1 + 1 >= t.h) continue;   // InpaintView.h:76-80
    if (h.x1 <= wx0 || h.x0 >= wx1 || h.y1 <= wy0 || h.y0 >= wy1) continue;    // changes no pixel of the window
    const int a = (h.x1 - h.x0 + 2) * (h.y1 - h.y0 + 2);
    const int c = a <= kWarpArea ? 0 : 1;
    lists[c * cap + atomicAdd(&sel->count[c], 1)] = id;
    atomicMax(&sel->max_area[c], a);
  }
}

// ---- one hole -----------------------------------------------------------------------------------------------------------
// A worker is a warp (WARP) or the whole CTA; its state for a hole of crop area A is A children pairs, A distances, A levels.
template <bool WARP> struct Group {
  __device__ static int rank() { return WARP ? (threadIdx.x & 31) : threadIdx.x; }
  __device__ static int size() { return WARP ? 32 : blockDim.x; }
  __device__ static void sync() { if (WARP) __syncwarp(); else __syncthreads(); }
  __device__ static bool any(bool p) { return WARP ? __any_sync(0xffffffffu, p) != 0 : __syncthreads_or(p) != 0; }
  __device__ static int max(int v) {
    if (WARP) {
      for (int o = 16; o; o >>= 1) v = ::max(v, __shfl_xor_sync(0xffffffffu, v, o));
      return v;
    }
    __shared__ int red;
    if (threadIdx.x == 0) red = 0;
    __syncthreads();
    atomicMax(&red, v);
    __syncthreads();
    const int r = red;
    __syncthreads();
    return r;
  }
};

struct FillStats { unsigned long long max_sweeps, max_levels, max_steps; };

template <class T, bool WARP>
__device__ void fill_hole(const T* __restrict__ in, ptrdiff_t ip, HoleTile t, const int* __restrict__ parent, const Hole& h, int id,
                          typename Px<T>::C* val, int* dist, int* lev, int wx0, int wy0, int wx1, int wy1, T* __restrict__ out,
                          ptrdiff_t op, FillStats* stats) {
  typedef Group<WARP> G;
  typedef typename Px<T>::C C;
  const int cx0 = h.x0 - 1, cy0 = h.y0 - 1, cw = h.x1 - h.x0 + 2, ch = h.y1 - h.y0 + 2, A = cw * ch;
  const int r = G::rank(), nt = G::size();
  constexpr int kInf = 0x3fffffff;
  for (int k = r; k < A; k += nt) {
    const int x = cx0 + k % cw, y = cy0 + k / cw;
    const T p = in[(ptrdiff_t)(t.y0 + y) * ip + t.x0 + x];
    val[2 * k] = p.dx; val[2 * k + 1] = p.dy;
    dist[k] = hole_of(parent, y * t.w + x) == id ? kInf : 0;
    lev[k] = 1;
  }
  G::sync();
  // 1. distance: the crop's border is never in the hole, so every hole pixel has its four neighbours in the crop
  bool changed;
  do {
    changed = false;
    for (int k = r; k < A; k += nt) {
      const int d = dist[k];
      if (!d) continue;
      const int m = 1 + ::min(::min(dist[k - 1], dist[k + 1]), ::min(dist[k - cw], dist[k + cw]));
      if (m < d) { dist[k] = m; changed = true; }
    }
  } while (G::any(changed));
  int dmax = 0;
  for (int k = r; k < A; k += nt) dmax = ::max(dmax, dist[k]);
  dmax = G::max(dmax);
  // 2. levels: q precedes p when (dist, column, row) of q is smaller
  int lmax;
  do {
    changed = false;
    lmax = 0;
    for (int k = r; k < A; k += nt) {
      const int d = dist[k];
      if (!d) continue;
      const int x = k % cw, y = k / cw;
      int l = 1;
      for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const int q = k + dy * cw + dx, dq = dist[q];
          if (!dq || (dx == 0 && dy == 0)) continue;
          const bool before = dq < d || (dq == d && (x + dx < x || (dx == 0 && y + dy < y)));
          if (before) l = ::max(l, lev[q] + 1);
        }
      if (l > lev[k]) { lev[k] = l; changed = true; }
      lmax = ::max(lmax, lev[k]);
    }
  } while (G::any(changed));
  lmax = G::max(lmax);
  // 3. the sweeps (InpaintView.h:114-137)
  const long long sweeps = 10LL * dmax * dmax;
  const double kC = .176765, kE = .073235;
  for (long long s = 0; s < sweeps; ++s)
    for (int l = 1; l <= lmax; ++l) {
      for (int k = r; k < A; k += nt) {
        if (!dist[k] || lev[k] != l) continue;
        const C* a = val + 2 * (k - cw - 1);
        const C* b = val + 2 * (k - 1);
        const C* c = val + 2 * (k + cw - 1);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          float sum = 0.0f;
          sum = __double2float_rn(__dadd_rn((double)sum, __dmul_rn(kC, Px<T>::wide(a[j]))));
          sum = __double2float_rn(__dadd_rn((double)sum, __dmul_rn(kE, Px<T>::wide(a[2 + j]))));
          sum = __double2float_rn(__dadd_rn((double)sum, __dmul_rn(kC, Px<T>::wide(a[4 + j]))));
          sum = __double2float_rn(__dadd_rn((double)sum, __dmul_rn(kE, Px<T>::wide(b[j]))));
          sum = __double2float_rn(__dadd_rn((double)sum, __dmul_rn(kE, Px<T>::wide(b[4 + j]))));
          sum = __double2float_rn(__dadd_rn((double)sum, __dmul_rn(kC, Px<T>::wide(c[j]))));
          sum = __double2float_rn(__dadd_rn((double)sum, __dmul_rn(kE, Px<T>::wide(c[2 + j]))));
          sum = __double2float_rn(__dadd_rn((double)sum, __dmul_rn(kC, Px<T>::wide(c[4 + j]))));
          val[2 * k + j] = Px<T>::store(sum);
        }
      }
      G::sync();
    }
  // the hole's pixels inside the window, valid
  for (int k = r; k < A; k += nt) {
    if (!dist[k]) continue;
    const int x = t.x0 + cx0 + k % cw, y = t.y0 + cy0 + k / cw;
    if (x < wx0 || x >= wx1 || y < wy0 || y >= wy1) continue;
    out[(ptrdiff_t)(y - wy0) * op + (x - wx0)] = Px<T>::make(val[2 * k], val[2 * k + 1]);
  }
  if (r == 0) {
    atomicMax(&stats->max_sweeps, (unsigned long long)sweeps);
    atomicMax(&stats->max_levels, (unsigned long long)lmax);
    atomicMax(&stats->max_steps, (unsigned long long)sweeps * lmax);
  }
  G::sync();
}

// Persistent workers draw holes from the list's ticket.  SMEM: the state lives in dynamic shared memory (WARP: one slice of
// kWarpArea pixels per warp), else in `scratch`, `area` pixels per CTA.
template <class T, bool WARP, bool SMEM>
__global__ void __launch_bounds__(kCtaThreads) k9_fill_kernel(const T* __restrict__ in, ptrdiff_t ip, HoleTile t, const int* __restrict__ parent,
                                                              const Hole* __restrict__ holes, const int* __restrict__ list, int count,
                                                              int* __restrict__ ticket, int area, unsigned char* __restrict__ scratch,
                                                              int wx0, int wy0, int wx1, int wy1, T* __restrict__ out, ptrdiff_t op,
                                                              FillStats* stats) {
  typedef typename Px<T>::C C;
  extern __shared__ __align__(16) unsigned char smem[];
  const int worker = WARP ? threadIdx.x >> 5 : 0;
  unsigned char* base = SMEM ? smem + (size_t)worker * area * kBytesPerPx : scratch + (size_t)blockIdx.x * area * kBytesPerPx;
  C* val = (C*)base;
  int* dist = (int*)(base + (size_t)area * 8);
  int* lev = (int*)(base + (size_t)area * 12);
  __shared__ int next[kWarpsPerCta];
  while (true) {
    if (WARP) {
      if ((threadIdx.x & 31) == 0) next[worker] = atomicAdd(ticket, 1);
      __syncwarp();
    } else {
      if (threadIdx.x == 0) next[0] = atomicAdd(ticket, 1);
      __syncthreads();
    }
    const int b = next[worker];
    if (WARP) __syncwarp(); else __syncthreads();
    if (b >= count) return;
    const int id = list[b];
    fill_hole<T, WARP>(in, ip, t, parent, holes[id], id, val, dist, lev, wx0, wy0, wx1, wy1, out, op, stats);
  }
}

}  // namespace

template <class T>
int fill_holes_grass_launch(const T* in, int w, int h, ptrdiff_t ip, int len, int x0, int y0, T* out, int ow, int oh, ptrdiff_t op,
                            Arena& ar, cudaStream_t st, vwb200_fill_stats* fs) {
  *fs = vwb200_fill_stats{0, 0, 0, 0, 0};
  // every pixel of the window passes through; the filled holes overwrite theirs
  VWB_CUDA(cudaMemcpy2DAsync(out, (size_t)op * sizeof(T), in + (ptrdiff_t)y0 * ip + x0, (size_t)ip * sizeof(T), (size_t)ow * sizeof(T), oh,
                             cudaMemcpyDeviceToDevice, st));
  const long long lx0 = std::max<long long>((long long)x0 - len, 0), ly0 = std::max<long long>((long long)y0 - len, 0);
  const long long lx1 = std::min<long long>((long long)x0 + ow + len, w), ly1 = std::min<long long>((long long)y0 + oh + len, h);
  const HoleTile t{(int)lx0, (int)ly0, (int)(lx1 - lx0), (int)(ly1 - ly0)};
  if (len == 0) return VWB200_OK;                                            // wipe_big_blobs(0) removes every hole
  if ((long long)t.w * t.h > INT_MAX / 2) {
    set_error("fill_holes_grass: the %d x %d tile (window grown by hole_fill_len) exceeds 2^30 pixels", t.w, t.h);
    return VWB200_ENOIMPL;
  }
  const int n = t.w * t.h;
  const int cap = ((t.w + 1) / 2) * ((t.h + 1) / 2);                          // at most one hole per 2 x 2 cell
  int* parent; Hole* holes; int* lists; int* counters; Select* sel; FillStats* stats;
  VWB_TRY(ar.alloc(&parent, (size_t)n));
  VWB_TRY(ar.alloc(&holes, (size_t)cap));
  VWB_TRY(ar.alloc(&lists, 2 * (size_t)cap));
  VWB_TRY(ar.alloc(&counters, 4));                                           // hole count, two tickets
  VWB_TRY(ar.alloc(&sel, 1));
  VWB_TRY(ar.alloc(&stats, 1));
  VWB_CUDA(cudaMemsetAsync(counters, 0, 4 * sizeof(int), st));
  VWB_CUDA(cudaMemsetAsync(sel, 0, sizeof(Select), st));
  VWB_CUDA(cudaMemsetAsync(stats, 0, sizeof(FillStats), st));
  const dim3 b2(32, 8), g2((t.w + 31) / 32, (t.h + 7) / 8);
  k9_label_init_kernel<T><<<g2, b2, 0, st>>>(in, ip, t, parent);
  VWB_LAUNCH_CHECK();
  k9_union_kernel<<<g2, b2, 0, st>>>(t, parent);
  VWB_LAUNCH_CHECK();
  k9_flatten_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, parent);
  VWB_LAUNCH_CHECK();
  k9_claim_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, parent, holes, counters);
  VWB_LAUNCH_CHECK();
  k9_stats_kernel<<<g2, b2, 0, st>>>(t, parent, holes);
  VWB_LAUNCH_CHECK();
  const int area_limit = len * len;
  const int wx0 = x0 - t.x0, wy0 = y0 - t.y0;
  k9_select_kernel<<<2 * kNumSMs, 256, 0, st>>>(counters, holes, t, len, area_limit, wx0, wy0, wx0 + ow, wy0 + oh, lists, cap, sel);
  VWB_LAUNCH_CHECK();
  // the worker shapes depend on how many holes there are and how large: one small read-back
  int nholes = 0;
  Select hs;
  VWB_CUDA(cudaMemcpyAsync(&nholes, counters, sizeof(int), cudaMemcpyDeviceToHost, st));
  VWB_CUDA(cudaMemcpyAsync(&hs, sel, sizeof(Select), cudaMemcpyDeviceToHost, st));
  VWB_CUDA(cudaStreamSynchronize(st));
  fs->holes = nholes;
  fs->filled = hs.count[0] + hs.count[1];
  if (hs.count[0]) {
    const int area = hs.max_area[0];
    const size_t smem = (size_t)kWarpsPerCta * area * kBytesPerPx;
    VWB_CUDA(cudaFuncSetAttribute(k9_fill_kernel<T, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = std::min((hs.count[0] + kWarpsPerCta - 1) / kWarpsPerCta, 8 * kNumSMs);
    k9_fill_kernel<T, true, true><<<grid, 32 * kWarpsPerCta, smem, st>>>(in, ip, t, parent, holes, lists, hs.count[0], counters + 1, area,
                                                                         nullptr, x0, y0, x0 + ow, y0 + oh, out, op, stats);
    VWB_LAUNCH_CHECK();
  }
  if (hs.count[1]) {
    const int area = hs.max_area[1];
    const size_t bytes = (size_t)area * kBytesPerPx;
    if (bytes <= (size_t)kSmemLimit - 1024) {
      VWB_CUDA(cudaFuncSetAttribute(k9_fill_kernel<T, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
      const int per_sm = std::max(1, std::min(8, (int)((kSmemLimit - 1024) / bytes)));
      const int grid = std::min(hs.count[1], per_sm * kNumSMs);
      k9_fill_kernel<T, false, true><<<grid, kCtaThreads, bytes, st>>>(in, ip, t, parent, holes, lists + cap, hs.count[1], counters + 2,
                                                                       area, nullptr, x0, y0, x0 + ow, y0 + oh, out, op, stats);
    } else {
      const int grid = std::min(hs.count[1], 2 * kNumSMs);
      unsigned char* scratch;
      VWB_TRY(ar.alloc(&scratch, (size_t)grid * bytes));
      k9_fill_kernel<T, false, false><<<grid, kCtaThreads, 0, st>>>(in, ip, t, parent, holes, lists + cap, hs.count[1], counters + 2,
                                                                    area, scratch, x0, y0, x0 + ow, y0 + oh, out, op, stats);
    }
    VWB_LAUNCH_CHECK();
  }
  // the engine has to know the stats once the call has finished; they are small
  FillStats hst;
  VWB_CUDA(cudaMemcpyAsync(&hst, stats, sizeof(FillStats), cudaMemcpyDeviceToHost, st));
  VWB_CUDA(cudaStreamSynchronize(st));
  fs->max_sweeps = (long long)hst.max_sweeps;
  fs->max_levels = (long long)hst.max_levels;
  fs->critical_steps = (long long)hst.max_steps;
  return VWB200_OK;
}

template int fill_holes_grass_launch<vwb200_dispi>(const vwb200_dispi*, int, int, ptrdiff_t, int, int, int, vwb200_dispi*, int, int, ptrdiff_t,
                                                   Arena&, cudaStream_t, vwb200_fill_stats*);
template int fill_holes_grass_launch<DispF>(const DispF*, int, int, ptrdiff_t, int, int, int, DispF*, int, int, ptrdiff_t, Arena&,
                                            cudaStream_t, vwb200_fill_stats*);

}  // namespace vwb200
