// k6_smoothing.cu -- the disparity smoothing filters of Stereo/Algorithms.{h,cc}:
//   disparity_median_filter              (Algorithms.cc:26-67)
//   texture_measure                      (Algorithms.h:144-209)
//   texture_preserving_disparity_filter  (Algorithms.h:213-281)
//
// The two disparity filters run IN PLACE and in raster order, as the reference's shallow `disparity_out = disparity_in`
// makes them do: a pixel's window reads the filtered values of the rows above and of the pixels to its left, and the
// original values below and to the right.  They share one wavefront sweep:
//   * one warp per row; rows are handed out by an atomic ticket in increasing order, so a warp only ever waits on a row
//     whose warp is already running (no co-residency assumption: safe under any occupancy and next to other work);
//   * row r may process column c once row r-1 has completed column min(c + h, W - 1) (h = the half window), and every
//     row follows the rule at every column, processed or not, so that by induction row r-j has completed
//     min(c + j*h, W - 1): no row ever reads a cell another row is still going to write;
//   * after a pixel is written, the writing lane fences and then publishes the row's progress; readers load progress
//     with ld.acquire and read neighbour rows with ld.global.cg (L2), never through L1, whose copies may be stale;
//   * waits back off with __nanosleep and are bounded: past kStallNs the warp sets the error word and leaves, every
//     waiting warp leaves when it sees the word, and the host reports VWB200_ELOGIC.
// No FMA contraction anywhere: every float / double operation is an explicitly rounded intrinsic.
#include "common.cuh"
#include <climits>

namespace vwb200 {
namespace {

constexpr int kSweepWarps = 4;                               // rows in flight per CTA
constexpr unsigned long long kStallNs = 10000000000ull;      // 10 s without progress of the row above = stalled
constexpr unsigned kNoKey = 0xFFFFFFFFu;                     // invalid window entry (above every finite key)

__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed(int* p, int v) {
  asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// sweep state: progress[row] = columns of the row completed; ticket; error word (1 = stalled)
struct Sweep { int* progress; int* ticket; int* error; };

// Waits until row - 1 has completed `need` columns (`seen`: its progress as last read).  false: the sweep is abandoned.
__device__ bool wait_row_above(const Sweep& s, int row, int need, int& seen) {
  if (row == 0 || seen >= need) return true;
  const int lane = threadIdx.x & 31;
  unsigned sleep = 32;
  unsigned long long t0 = 0;
  for (;;) {
    int p = ld_acquire(s.progress + row - 1);          // every lane acquires: its own later loads are ordered after it
    p = __shfl_sync(~0u, p, 0);
    seen = p;
    if (p >= need) break;
    int quit = 0;
    if (lane == 0) {
      const unsigned long long t = global_ns();
      if (*(volatile int*)s.error) quit = 1;
      else if (t0 == 0) t0 = t;
      else if (t - t0 > kStallNs) { atomicExch(s.error, 1); quit = 1; }
    }
    if (__shfl_sync(~0u, quit, 0)) return false;
    __nanosleep(sleep);
    sleep = min(sleep * 2, 1024u);
  }
  __syncwarp();
  return true;
}

// The wavefront: Op::pixel(row, col, lane, scratch) is called by the whole warp for every pixel of a row in order and
// returns (in every lane) whether lane 0 wrote the pixel.
template <class Op>
__global__ void __launch_bounds__(kSweepWarps * 32) smooth_sweep_kernel(Op op, Sweep s, int W, int H, int h) {
  extern __shared__ float smooth_scratch[];
  const int lane = threadIdx.x & 31;
  float* scratch = smooth_scratch + (threadIdx.x >> 5) * op.scratch_floats();
  op.prepare(lane);
  for (;;) {
    int row = 0;
    if (lane == 0) row = atomicAdd(s.ticket, 1);
    row = __shfl_sync(~0u, row, 0);
    if (row >= H) return;
    int seen = 0;
    for (int c = 0; c < W; ++c) {
      if (!wait_row_above(s, row, min(c + h, W - 1) + 1, seen)) return;
      const bool wrote = op.pixel(row, c, lane, scratch);
      if (lane == 0) {
        if (wrote) __threadfence();                     // the pixel is visible before the progress that covers it
        st_relaxed(s.progress + row, c + 1);
      }
    }
  }
}

// ---- disparity_median_filter (Algorithms.cc:26-67) -----------------------------------------------------------------
// The window's valid values become keys spread over the lanes (NPL per lane, row-major window slots lane, lane + 32, ...);
// a bitwise select over the keys, from the highest bit in which the window's smallest and largest keys differ, finds the
// n/2-th smallest (and, for even n, the next lower one) of x and y together.  math::destructive_median's sort order and
// this one agree up to the order of equal values, so the selected values are the sorted vector's.
template <int NPL>
struct MedianOp {
  float* d; long long pitch; int W, H, half, kw;
  int off[NPL];                                          // float offset of each slot from the window's corner

  __host__ __device__ int scratch_floats() const { return 0; }
  __device__ void prepare(int lane) {
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      const int i = j * 32 + lane, dr = i / kw, dc = i - dr * kw;
      off[j] = i < kw * kw ? (int)((dr * pitch + dc) * 3) : -1;
    }
  }
  __device__ bool pixel(int row, int col, int lane, float*) {
    if (row < half || row >= H - half || col < half || col >= W - half) return false;
    float* p = d + (row * pitch + col) * 3;
    __syncwarp();                                        // lane 0's write of the pixel to the left is visible to all lanes
    if (__ldcg(p + 2) == 0.0f) return false;
    const float* base = d + ((row - half) * pitch + (col - half)) * 3;
    unsigned kx[NPL], ky[NPL];
    unsigned nloc = 0, mnx = kNoKey, mny = kNoKey, mxx = 0, mxy = 0;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
      kx[j] = ky[j] = kNoKey;
      if (off[j] >= 0) {
        const float* q = base + off[j];
        const float x = __ldcg(q), y = __ldcg(q + 1), v = __ldcg(q + 2);
        if (v != 0.0f) {
          kx[j] = fkey(x); ky[j] = fkey(y); ++nloc;
          mnx = min(mnx, kx[j]); mxx = max(mxx, kx[j]);
          mny = min(mny, ky[j]); mxy = max(mxy, ky[j]);
        }
      }
    }
    const unsigned n = __reduce_add_sync(~0u, nloc);     // >= 1: the pixel itself is valid
    mnx = __reduce_min_sync(~0u, mnx); mxx = __reduce_max_sync(~0u, mxx);
    mny = __reduce_min_sync(~0u, mny); mxy = __reduce_max_sync(~0u, mxy);
    // rank n/2 (0-based) of x and y
    unsigned px = mnx, py = mny, tx = n / 2, ty = n / 2;
    const int hbx = mnx == mxx ? -1 : 31 - __clz(mnx ^ mxx), hby = mny == mxy ? -1 : 31 - __clz(mny ^ mxy);
    if (hbx >= 0) px = mnx & ~((2u << hbx) - 1u);
    if (hby >= 0) py = mny & ~((2u << hby) - 1u);
    for (int b = max(hbx, hby); b >= 0; --b) {
      const unsigned lim = 1u << b;
      unsigned cx = 0, cy = 0;
#pragma unroll
      for (int j = 0; j < NPL; ++j) { cx += (kx[j] ^ px) < lim; cy += (ky[j] ^ py) < lim; }
      if (b <= hbx) { const unsigned c = __reduce_add_sync(~0u, cx); if (tx >= c) { tx -= c; px |= lim; } }
      if (b <= hby) { const unsigned c = __reduce_add_sync(~0u, cy); if (ty >= c) { ty -= c; py |= lim; } }
    }
    float rx = kfloat(px), ry = kfloat(py);
    if (n % 2 == 0) {                                    // (vec[n/2 - 1] + vec[n/2]) / 2.0 in double
      unsigned lx = 0, ly = 0, bx = 0, by = 0;           // keys below the median: how many, and the largest
#pragma unroll
      for (int j = 0; j < NPL; ++j) {
        if (kx[j] < px) { ++lx; bx = max(bx, kx[j]); }
        if (ky[j] < py) { ++ly; by = max(by, ky[j]); }
      }
      lx = __reduce_add_sync(~0u, lx); ly = __reduce_add_sync(~0u, ly);
      bx = __reduce_max_sync(~0u, bx); by = __reduce_max_sync(~0u, by);
      const float ax = lx <= n / 2 - 1 ? rx : kfloat(bx), ay = ly <= n / 2 - 1 ? ry : kfloat(by);
      rx = __double2float_rn(__dmul_rn(__dadd_rn((double)ax, (double)rx), 0.5));
      ry = __double2float_rn(__dmul_rn(__dadd_rn((double)ay, (double)ry), 0.5));
    }
    if (lane == 0) { p[0] = rx; p[1] = ry; p[2] = 1.0f; }
    return true;
  }
};

// ---- texture_preserving_disparity_filter<float> (Algorithms.h:213-281) ----------------------------------------------
// The lanes stage the pixel's clamped window in shared memory; lane 0 sums it in the reference's row-major order (the
// double sums are order-sensitive).
struct TextureFilterOp {
  float* d; long long pitch; const float* tex; long long tpitch; int W, H, max_k;
  float texture_max, scale;

  __host__ __device__ int scratch_floats() const { return 2 * max_k * max_k + 32; }
  __device__ void prepare(int) {}
  __device__ bool pixel(int row, int col, int lane, float* scratch) {
    float* p = d + (row * pitch + col) * 3;
    __syncwarp();
    if (__ldcg(p + 2) == 0.0f) return false;             // :240
    const float t = __ldg(tex + row * tpitch + col);
    if (t < 0.0f) return false;
    float adj = __fsub_rn(texture_max, t);               // :243-245
    if (adj < 0.0f) adj = 0.0f;
    const float f = floorf(__fmul_rn(adj, scale));       // :246; int(NaN / out of range) is INT_MIN on x86-64
    int k = (f >= -2147483648.0f && f < 2147483648.0f) ? (int)f : INT_MIN;
    if (k % 2 == 0) k += 1;                              // :247-248
    if (k < 3 || k > max_k) return false;                // :249-257 (the reference prints when k > max_k)
    const int half = (k - 1) / 2, n = k * k;
    float* xs = scratch;
    float* ys = scratch + max_k * max_k;
    unsigned* valid = reinterpret_cast<unsigned*>(scratch + 2 * max_k * max_k);
    for (int j = 0; j * 32 < n; ++j) {
      const int i = j * 32 + lane;
      bool v = false;
      if (i < n) {
        const int dr = i / k, dc = i - dr * k;
        const int r = min(max(row - half + dr, 0), H - 1), c = min(max(col - half + dc, 0), W - 1);
        const float* q = d + (r * pitch + c) * 3;
        v = __ldcg(q + 2) != 0.0f;
        xs[i] = __ldcg(q); ys[i] = __ldcg(q + 1);
      }
      const unsigned m = __ballot_sync(~0u, v);
      if (lane == 0) valid[j] = m;
    }
    __syncwarp();
    if (lane == 0) {                                     // :263-277
      double sx = 0.0, sy = 0.0, count = 0.0;
      for (int i = 0; i < n; ++i)
        if (valid[i >> 5] >> (i & 31) & 1u) {
          sx = __dadd_rn(sx, (double)xs[i]); sy = __dadd_rn(sy, (double)ys[i]); count = __dadd_rn(count, 1.0);
        }
      if (count >= 1.0) {
        p[0] = __double2float_rn(__ddiv_rn(sx, count));
        p[1] = __double2float_rn(__ddiv_rn(sy, count));
        p[2] = 1.0f;
      }
    }
    return true;
  }
};

template <class Op>
int sweep_launch(const Op& op, int W, int H, int h, int* work, int* err_host, cudaStream_t st) {
  const Sweep s{work + 2, work, work + 1};
  VWB_CUDA(cudaMemsetAsync(work, 0, (size_t)(H + 2) * sizeof(int), st));
  const size_t smem = (size_t)kSweepWarps * op.scratch_floats() * sizeof(float);
  auto kern = smooth_sweep_kernel<Op>;
  if (smem > 48 * 1024) VWB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  VWB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kSweepWarps * 32, smem));
  const int blocks = std::max(1, std::min((H + kSweepWarps - 1) / kSweepWarps, std::max(per_sm, 1) * kNumSMs));
  kern<<<blocks, kSweepWarps * 32, smem, st>>>(op, s, W, H, h);
  VWB_LAUNCH_CHECK();
  VWB_CUDA(cudaMemcpyAsync(err_host, work + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
  return VWB200_OK;
}

template <int NPL>
int median_launch_n(float* d, int W, int H, ptrdiff_t pitch, int half, int* work, int* err, cudaStream_t st) {
  MedianOp<NPL> op;
  op.d = d; op.pitch = pitch; op.W = W; op.H = H; op.half = half; op.kw = 2 * half + 1;
  return sweep_launch(op, W, H, half, work, err, st);
}

// ---- texture_measure (Algorithms.h:144-209) of a plain float image --------------------------------------------------
// One thread per output pixel; the CTA's tile of input values and of |dx| + |dy| (a float add, as in the reference)
// is computed once, halo included, at clamped positions.  Per pixel, the direct window sums in the reference's order
// (sliding sums would reorder the double additions).
constexpr int kTmX = 32, kTmY = 8;

__device__ __forceinline__ float deriv3(float lo, float mid, float hi) {
  // correlate_1d_at_point with the reversed kernel {-0.5, 0, 0.5}, accumulated in float from 0 (Convolution.h:53-65)
  return __fadd_rn(__fadd_rn(__fadd_rn(0.0f, __fmul_rn(-0.5f, lo)), __fmul_rn(0.0f, mid)), __fmul_rn(0.5f, hi));
}

__global__ void __launch_bounds__(kTmX * kTmY) texture_measure_kernel(ImgF img, int half, double gw, double sw, float* out,
                                                                       ptrdiff_t opitch) {
  extern __shared__ float tm_tile[];
  const int tw = kTmX + 2 * half, th = kTmY + 2 * half;
  float* tv = tm_tile;
  float* tg = tm_tile + tw * th;
  const int x0 = blockIdx.x * kTmX - half, y0 = blockIdx.y * kTmY - half;
  const int W = img.w, H = img.h;
  for (int i = threadIdx.y * kTmX + threadIdx.x; i < tw * th; i += kTmX * kTmY) {
    const int ty = i / tw, tx = i - ty * tw;
    const int cx = min(max(x0 + tx, 0), W - 1), cy = min(max(y0 + ty, 0), H - 1);
    const float* r = img.p + cy * img.pitch;
    const float v = __ldg(r + cx);
    const float dx = deriv3(__ldg(r + max(cx - 1, 0)), v, __ldg(r + min(cx + 1, W - 1)));
    const float dy = deriv3(__ldg(img.p + max(cy - 1, 0) * img.pitch + cx), v, __ldg(img.p + min(cy + 1, H - 1) * img.pitch + cx));
    tv[i] = v;
    tg[i] = __fadd_rn(fabsf(dx), fabsf(dy));
  }
  __syncthreads();
  const int col = blockIdx.x * kTmX + threadIdx.x, row = blockIdx.y * kTmY + threadIdx.y;
  if (col >= W || row >= H) return;
  const int kw = 2 * half + 1;
  double mean = 0.0, count = 0.0;                                    // :176-187
  for (int r = 0; r < kw; ++r) {
    const float* t = tv + (threadIdx.y + r) * tw + threadIdx.x;
    for (int c = 0; c < kw; ++c) { mean = __dadd_rn(mean, (double)t[c]); count = __dadd_rn(count, 1.0); }
  }
  mean = __ddiv_rn(mean, count);
  double grad = 0.0, sd = 0.0;                                       // :189-198
  for (int r = 0; r < kw; ++r) {
    const float* t = tv + (threadIdx.y + r) * tw + threadIdx.x;
    const float* g = tg + (threadIdx.y + r) * tw + threadIdx.x;
    for (int c = 0; c < kw; ++c) {
      grad = __dadd_rn(grad, (double)g[c]);
      const double e = __dsub_rn((double)t[c], mean);
      sd = __dadd_rn(sd, __dmul_rn(e, e));                           // pow(e, 2)
    }
  }
  grad = __ddiv_rn(grad, __dmul_rn(2.0, count));                     // :200-204
  sd = __dsqrt_rn(__ddiv_rn(sd, count));
  out[row * opitch + col] = __double2float_rn(__dadd_rn(__dmul_rn(grad, gw), __dmul_rn(sd, sw)));
}

}  // namespace

int median_sweep_launch(float* d, int W, int H, ptrdiff_t pitch, int kernel_size, int* work, int* err_host, cudaStream_t st) {
  const int half = (kernel_size - 1) / 2, kw = 2 * half + 1, npl = (kw * kw + 31) / 32;
  if (npl <= 1) return median_launch_n<1>(d, W, H, pitch, half, work, err_host, st);
  if (npl <= 2) return median_launch_n<2>(d, W, H, pitch, half, work, err_host, st);
  if (npl <= 4) return median_launch_n<4>(d, W, H, pitch, half, work, err_host, st);
  if (npl <= 8) return median_launch_n<8>(d, W, H, pitch, half, work, err_host, st);
  if (npl <= 16) return median_launch_n<16>(d, W, H, pitch, half, work, err_host, st);
  if (npl <= 31) return median_launch_n<31>(d, W, H, pitch, half, work, err_host, st);
  set_error("disparity_median_filter: kernel_size %d is above the supported %d", kernel_size, kSmoothMaxKernel);
  return VWB200_ENOIMPL;
}

int texture_filter_sweep_launch(float* d, int W, int H, ptrdiff_t pitch, const float* tex, ptrdiff_t tpitch, float texture_max,
                                int max_kernel_size, int* work, int* err_host, cudaStream_t st) {
  TextureFilterOp op;
  op.d = d; op.pitch = pitch; op.tex = tex; op.tpitch = tpitch; op.W = W; op.H = H; op.max_k = max_kernel_size;
  op.texture_max = texture_max;
  op.scale = (float)max_kernel_size / texture_max;                  // :222, float division
  return sweep_launch(op, W, H, (max_kernel_size - 1) / 2, work, err_host, st);
}

int texture_measure_launch(ImgF img, int kernel_size, double gw, double sw, float* out, ptrdiff_t opitch, cudaStream_t st) {
  const int half = (kernel_size - 1) / 2;
  const size_t smem = (size_t)2 * (kTmX + 2 * half) * (kTmY + 2 * half) * sizeof(float);
  if (smem > 48 * 1024) VWB_CUDA(cudaFuncSetAttribute(texture_measure_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((img.w + kTmX - 1) / kTmX, (img.h + kTmY - 1) / kTmY);
  texture_measure_kernel<<<grid, dim3(kTmX, kTmY), smem, st>>>(img, half, gw, sw, out, opitch);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

}  // namespace vwb200
