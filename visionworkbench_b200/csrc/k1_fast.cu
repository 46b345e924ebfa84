// k1_fast.cu -- exact-integer fast path of the fused cost-volume + arg-best kernel (AbsoluteCost).
//
// When both rasters are integer valued with (max-min)*8 < 2^16 (8..13-bit imagery), every quantity
// of best_of_search_convolution (Stereo/Correlation.cc:33-137) is an exact integer: the float
// per-pixel cost |a-b|, the double box sums and therefore the comparison results.  The kernel below
// evaluates the same cost volume in int32 and applies the same selection rule (strict '<', dy-major /
// dx-minor order => first disparity wins ties; all-equal => invalid), so it is bit-identical to the
// reference while doing ~10 issue slots per (pixel, disparity) instead of ~70 bytes of DRAM traffic.
//
// Decomposition (persistent CTAs of 12 warps at <= 168 registers, one CTA per SM = 3 warps per sub-partition; work
// item = 236-column x th-row band, th chosen by fast_geom within the shared-memory budget -- 84 rows at 128 x 128 / 21 x 21):
//   * values are pre-packed (pack kernels) as u16 (v-vmin)*8, one contiguous row per strip, so that a
//     lane fetches its 8 left / 16 right columns with conflict-free 16-byte LDS.128 loads
//   * the left tile (th+ky-1 rows) and a ring of right rows are staged in shared memory with TMA bulk
//     copies (cp.async.bulk + mbarrier); the dy range runs in periods of sd (<= 3) dy rows with one barrier each,
//     and the next period's sd right rows are prefetched while the CTA computes
//   * a period's work units are its (dy, octet) pairs; warp w takes units w, w+12, ... and slides each over every
//     row of the band, so the ky rows that seed its vertical sums are summed once per (dy, octet) and band
//   * lane l owns padded columns 8l..8l+7 and 8 consecutive dx: V[8][8] vertical sliding sums live in
//     registers (VABSDIFF accumulate: +new row, -old row)
//   * the kx-wide horizontal sums are formed without shared memory: in-lane prefix sums + 9 warp
//     shuffles per 8 outputs (blocked-prefix scheme), 3-input IADD3
//   * arg-best: costs are pre-scaled by 8 so key = cost*8 + b; min over the 8 dx is 7 VIADDMNMX;
//     a shared-memory plane holds the best high word (cost*8 | 7) per band pixel, the threshold of the hot loop;
//     the (rare) candidates with a cost <= it lower it with a 32-bit atomicMin and send the exact 64-bit key
//     (cost << 32 | raster index) to a per-CTA plane in global memory with a 64-bit atomicMin reduction -- neither
//     is waited for -- so the lowest cost and, among equal costs, the first disparity in raster order wins
//     whichever warp reaches it first
//   * pixels whose arg-best is disparity (0,0) are re-checked by a small kernel for the
//     "every disparity gave the same cost => invalid" rule (Correlation.cc:121-133)
#include "k1_fast_common.cuh"

namespace vwb200 {

// ---- min / max / integer-valuedness reduction -------------------------------------------------------
// order-preserving float -> int key so that integer atomics can be used; taken from the sign bit, so -0.0 and +0.0 both
// map to 0 (a key from `v >= 0` would send -0.0 to INT_MIN, below every negative pixel).  image_stats_fini inverts it.
static __device__ __forceinline__ int stats_key(float v) {
  const int b = __float_as_int(v);
  return b >= 0 ? b : (int)(0x80000000u - (unsigned)b);
}
__global__ void image_stats_kernel(ImgF img, float* __restrict__ result) {
  float mn = INFINITY, mx = -INFINITY; int allint = 1;
  const long long n = (long long)img.w * img.h;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const float v = img.p[(ptrdiff_t)(k / img.w) * img.pitch + (k % img.w)];
    mn = fminf(mn, v); mx = fmaxf(mx, v);
    if (!isfinite(v) || v != rintf(v)) allint = 0;          // NaN/inf -> not integer
  }
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    allint &= __shfl_xor_sync(0xffffffffu, allint, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMin(reinterpret_cast<int*>(result) + 0, stats_key(mn));
    atomicMax(reinterpret_cast<int*>(result) + 1, stats_key(mx));
    if (!allint) atomicExch(reinterpret_cast<int*>(result) + 2, 0);
  }
}
__global__ void image_stats_init(float* result) {
  reinterpret_cast<int*>(result)[0] = INT_MAX; reinterpret_cast<int*>(result)[1] = INT_MIN; reinterpret_cast<int*>(result)[2] = 1;
}
__global__ void image_stats_fini(float* result) {
  int* r = reinterpret_cast<int*>(result);
  for (int i = 0; i < 2; ++i) {
    const int o = r[i];
    result[i] = o >= 0 ? __int_as_float(o) : __int_as_float((int)(0x80000000u - (unsigned)o));
  }
  result[2] = r[2] ? 1.0f : 0.0f;
}
int image_stats_launch(ImgF img, float* d_result3, cudaStream_t st) {
  image_stats_init<<<1, 1, 0, st>>>(d_result3);
  VWB_LAUNCH_CHECK();
  image_stats_kernel<<<2 * kNumSMs, 256, 0, st>>>(img, d_result3);
  VWB_LAUNCH_CHECK();
  image_stats_fini<<<1, 1, 0, st>>>(d_result3);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

// ---- band geometry ------------------------------------------------------------------------------------------------
static constexpr int FK_WARPS = 12;                  // per CTA: 3 per SM sub-partition, at most 168 registers per thread
static constexpr int FK_THREADS = FK_WARPS * 32;
static constexpr int FK_SD_MAX = 3;                  // dy rows per synchronisation period (ring depth)
static constexpr int FK_TH_MAX = 96;                 // tallest band considered
static constexpr size_t FK_SMEM = 227 * 1024;
static constexpr uint32_t FK_INIT_HI = 0x7fffffffu;  // high word of an empty key: above every (cost*8 | 7)

// best plane [th][256] (u32) | left tile [th+ky-1][256] (u16) | right ring [ring_slots][rw] (u16) | 2 mbarriers
static size_t fast_smem_bytes(const FastGeom& g) {
  return (size_t)g.th * F_COLS * 4 + (size_t)g.ltile_rows * F_COLS * 2 + (size_t)g.ring_slots * g.rw * 2 + 64;
}

// A period of sd dy rows is ngroups * sd work units (one (dy, octet) pass each), dealt statically to the 12 warps:
// take the depth whose units fill the warps best (48 units = 4 per warp at 16 octets), the deeper one on a tie (fewer
// barriers).  The ring holds the period's ltile_rows + sd - 1 right rows while the next period's sd rows arrive.
static FastGeom fast_make_geom(int W, int H, int sx, int sy, int kx, int ky, int th) {
  FastGeom g = make_geom(W, H, sx, sy, kx, ky, th);
  const int ngroups = (sx + F_B - 1) / F_B;
  double best = -1.0;
  for (int sd = 1; sd <= FK_SD_MAX && sd <= g.dy_per; ++sd) {
    const int units = ngroups * sd;
    const double eff = (double)units / (double)(((units + FK_WARPS - 1) / FK_WARPS) * FK_WARPS);
    if (eff >= best - 1e-9) { best = eff; g.sd = sd; }
  }
  g.ring_slots = g.ltile_rows + 2 * g.sd - 1;
  return g;
}

// Band height: a taller band spreads the seeding of each (dy, octet) -- ky rows of vertical sums plus a first row
// without the sliding update, about 0.15*ky row steps -- over more rows, but makes fewer, longer work items.  Take
// the height between F_TH and what the shared memory holds with the least estimated time: waves of work items x
// row steps per item (make_geom picks the dy chunking J for each height).
static FastGeom fast_geom(int W, int H, int sx, int sy, int kx, int ky) {
  FastGeom best = fast_make_geom(W, H, sx, sy, kx, ky, F_TH);
  double tbest = -1.0;
  for (int th = F_TH; th <= FK_TH_MAX; ++th) {
    const FastGeom g = fast_make_geom(W, H, sx, sy, kx, ky, th);
    if (fast_smem_bytes(g) > FK_SMEM) break;
    const long long waves = ((long long)g.NS * g.NB * g.J + kNumSMs - 1) / kNumSMs;
    const double t = (double)waves * g.dy_per * ((th < H ? th : H) + 0.15 * ky) * (1.0 + 0.004 * (g.J - 1));
    if (tbest < 0.0 || t < tbest) { tbest = t; best = g; }
  }
  return best;
}

int k1_fast_supported(int cost, int kx, int ky, int sx, int sy, float vmin, float vmax, bool integer_valued) {
  if (cost != VWB200_ABSOLUTE_DIFFERENCE && cost != VWB200_SQUARED_DIFFERENCE) return VWB200_ENOIMPL;
  if (!integer_valued) return VWB200_ENOIMPL;
  if (cost == VWB200_SQUARED_DIFFERENCE) {        // window sums of (a-b)^2 must fit uint32
    const double r = (double)vmax - (double)vmin;
    // |a-b| <= 4095 keeps the reference's FLOAT (a-b)*(a-b) exact (< 2^24); beyond that it rounds and only the
    // general kernel (which issues the same float multiply) reproduces it
    if (!(r <= 4095.0) || !(r * r * kx * ky < 4294967295.0)) return VWB200_ENOIMPL;
  } else if (!(vmax - vmin <= 8191.0f)) return VWB200_ENOIMPL;
  if ( !(fabsf(vmin) < 1.0e6f) || !(fabsf(vmax) < 1.0e6f)) return VWB200_ENOIMPL;
  if (kx < 3 || kx > 31 || ky < 1 || ky > 41) return VWB200_ENOIMPL;
  if (sx < F_B || sx > 512 || sy < 1) return VWB200_ENOIMPL;
  if ((long long)sx * sy > 65536) return VWB200_ENOIMPL;
  if ((long long)sx * sy < 64) return VWB200_ENOIMPL;      // tiny searches: the generic kernel is as good
  if (fast_smem_bytes(fast_make_geom(256, F_TH, sx, sy, kx, ky, F_TH)) > FK_SMEM) return VWB200_ENOIMPL;
  return VWB200_OK;
}

size_t k1_fast_workspace_bytes(int W, int H, int sx, int sy, int kx, int ky) {
  FastGeom g = fast_geom(W, H, sx, sy, kx, ky);
  size_t l = (size_t)g.NS * g.lrows * F_COLS * 2;
  size_t r = (size_t)g.NS * g.rrows * g.rw * 2;
  size_t part = g.J > 1 ? (size_t)g.J * W * H * 6 + 64 : 0;      // per-dy-chunk partial (cost u32, index u16)
  size_t keys = (size_t)kNumSMs * g.th * F_COLS * 8 + 64;           // one 64-bit key plane per persistent CTA
  return l + r + part + keys + 512;
}

// ---- pack kernels: float raster -> u16 (v - vmin) * 4 in the lane-transposed strip layout ------------
__global__ void pack_left_kernel(ImgF img, float vmin, FastGeom g, uint16_t* __restrict__ out) {
  const int row = blockIdx.x, strip = blockIdx.y;
  const int s0 = strip * g.out_cols;
  uint16_t* o = out + ((size_t)strip * g.lrows + row) * F_COLS;
  for (int c = threadIdx.x; c < F_COLS; c += blockDim.x) {      // c = strip-relative padded column (coalesced reads)
    const int gx = s0 + c;
    uint16_t v = 0;      // logical raster = (W+kx-1) x (H+ky-1) at (lox,loy); constant edge extension of the image beyond it
    if (row < g.H + g.ky - 1 && gx < g.W + g.kx - 1) {
      const int iy = min(max(g.loy + row, 0), img.h - 1), ix = min(max(g.lox + gx, 0), img.w - 1);
      v = (uint16_t)((int)(img.p[(ptrdiff_t)iy * img.pitch + ix] - vmin) * g.scale);
    }
    o[c] = v;
  }
}
__global__ void pack_right_kernel(ImgF img, float vmin, FastGeom g, uint16_t* __restrict__ out) {
  const int row = blockIdx.x, strip = blockIdx.y;
  const int s0 = strip * g.out_cols;
  uint16_t* o = out + ((size_t)strip * g.rrows + row) * g.rw;
  for (int c = threadIdx.x; c < g.rw; c += blockDim.x) {
    const int gx = s0 + c;
    uint16_t v = 0;
    if (row < g.H + g.ky - 1 + g.sy - 1 && gx < g.W + g.kx - 1 + g.sx - 1) {
      const int iy = min(max(g.roy + row, 0), img.h - 1), ix = min(max(g.rox + gx, 0), img.w - 1);
      v = (uint16_t)((int)(img.p[(ptrdiff_t)iy * img.pitch + ix] - vmin) * g.scale);
    }
    o[c] = v;
  }
}

// ---- one pass: 8 consecutive dx (octet g) x 8 columns per lane, sliding down the warp's rows ----------------
// The AbsoluteCost row step is bound by the integer ALU pipe (VABSDIFF, IADD3, VIADDMNMX), so it splits the halves on
// the FMA pipe: hi = IMAD.HI(v, 2^16), lo = IMAD(hi, -2^16, v).  Written as `v >> 16` / `v & 0xffff`, ptxas emits SHF /
// LOP3 on the ALU pipe, which the SquaredCost step keeps: its (a-b)^2 already loads the FMA pipe more than the ALU pipe.
template <bool FMA>
__device__ __forceinline__ void unpack2(const uint32_t v, int& lo, int& hi) {
  if (FMA) {
    uint32_t h, l;
    asm("mul.hi.u32 %0, %1, 65536;" : "=r"(h) : "r"(v));
    asm("mad.lo.u32 %0, %1, -65536, %2;" : "=r"(l) : "r"(h), "r"(v));
    lo = (int)l; hi = (int)h;
  } else {
    lo = v & 0xffff; hi = v >> 16;
  }
}
template <bool FMA>
__device__ __forceinline__ void unpack8(const uint4 v, int (&o)[8]) {
  unpack2<FMA>(v.x, o[0], o[1]); unpack2<FMA>(v.y, o[2], o[3]); unpack2<FMA>(v.z, o[4], o[5]); unpack2<FMA>(v.w, o[6], o[7]);
}
template <bool FMA>
__device__ __forceinline__ void load_row(const uint16_t* lrow, const uint16_t* rrow, int (&Lv)[8], int (&Rv)[16]) {
  unpack8<FMA>(*reinterpret_cast<const uint4*>(lrow), Lv);
  int t[8];
  unpack8<FMA>(*reinterpret_cast<const uint4*>(rrow), t);
#pragma unroll
  for (int i = 0; i < 8; ++i) Rv[i] = t[i];
  unpack8<FMA>(*reinterpret_cast<const uint4*>(rrow + 8), t);
#pragma unroll
  for (int i = 0; i < 8; ++i) Rv[8 + i] = t[i];
}

// A candidate: keep the lower cost and, for equal costs, the lower raster index (= the first disparity).  The exact
// 64-bit key (hi << 32 | raster index) goes to the CTA's plane in global memory, where a 64-bit atomicMin is one
// native reduction; the shared plane keeps only the high word, the threshold the hot loop compares with (a native
// 32-bit shared atomicMin).  Neither result is waited for.  A stale threshold only lets more candidates through.
__device__ __forceinline__ void offer_key(uint32_t* best, unsigned long long* key, uint32_t hi, uint32_t idx) {
  atomicMin(best, hi);
  atomicMin(key, ((unsigned long long)hi << 32) | idx);
}

template <int KX, bool FULL>
__device__ __forceinline__ void fast_pass(const uint16_t* __restrict__ ltile, const uint16_t* __restrict__ rring,
                                          uint32_t* __restrict__ best, unsigned long long* __restrict__ keys,
                                          int lane, int g, int ky, int ring_slots, int rw, int ring_base, int idx_base, int nrows, int nb) {
  int V[8][F_B];
  // Row pointers: the left rows advance by 256, the right rows by rw and wrap around the ring, so a row step computes no
  // slot * rw.  The seed wraps rnew before each load, so rnew may sit at rend after it, to be wrapped at the first cut.
  const uint16_t* lnew = ltile + 8 * lane;                      // left row y + ky - 1  (16-byte aligned)
  const uint16_t* lold = lnew;                                  // left row y - 1
  const uint16_t* const rring_lane = rring + 8 * (lane + g);
  const uint16_t* const rend = rring_lane + ring_slots * rw;
  const int rspan = ring_slots * rw;
  const uint16_t* rnew = rring_lane + ring_base * rw;           // right row dy + y + ky - 1
  const uint16_t* rold = rnew;                                  // right row dy + y - 1
  // ---- seed: first ky rows ----
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < F_B; ++b) V[a][b] = 0;
  for (int t = 0; t < ky; ++t) {
    if (rnew == rend) rnew -= rspan;
    int Lv[8], Rv[16];
    load_row<true>(lnew, rnew, Lv, Rv);
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
      for (int b = 0; b < F_B; ++b) V[a][b] = __sad(Lv[a], Rv[a + b], V[a][b]);
    lnew += F_COLS;
    rnew += rw;
  }
  // ---- slide the vertical sums down to row y: + row y + ky - 1, - row y - 1 ----
  auto slide = [&]() {
    {
      int Lv[8], Rv[16];
      load_row<true>(lnew, rnew, Lv, Rv);
#pragma unroll
      for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < F_B; ++b) V[a][b] = __sad(Lv[a], Rv[a + b], V[a][b]);
    }
    {
      int Lo[8], Ro[16];
      load_row<true>(lold, rold, Lo, Ro);
#pragma unroll
      for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < F_B; ++b) V[a][b] -= __sad(Lo[a], Ro[a + b], 0);
    }
    lnew += F_COLS; lold += F_COLS;
    rnew += rw; rold += rw;
  };
  // The pass reads nrows + ky - 1 <= ring_slots consecutive ring rows, so each right pointer wraps at most once: rnew
  // before the slide to row ynew, rold (ky rows behind) before the slide to row yold.  Rows between those cuts run in
  // one inner loop whose pointers advance without a test.
  const int ynew = ring_slots - ring_base - ky + 1, yold = ynew + ky;
  uint32_t* brow = best + lane;
  // row y = 0 has no sliding update; the inner loop leaves after the arg-best of its last row, so the update of every
  // following row needs no test of y
  for (int y = 0;;) {
    const int yend = min(nrows, y < ynew ? ynew : y < yold ? yold : nrows);
    for (;;) {
      // ---- horizontal window sums + min over the 8 dx (keys = cost*8 + b) ----
      int m[8];
      if (FULL) {
        // dx b and b + 4 together: two independent prefix / shuffle / add chains (the keys make the min order-free)
#pragma unroll
        for (int b = 0; b < F_B / 2; ++b) {
          int p0[8], p1[8], o0[8], o1[8];
          p0[0] = V[0][b]; p1[0] = V[0][b + 4];
#pragma unroll
          for (int a = 1; a < 8; ++a) { p0[a] = p0[a - 1] + V[a][b]; p1[a] = p1[a - 1] + V[a][b + 4]; }
          window_sums2<KX>(p0, p1, o0, o1);
#pragma unroll
          for (int r = 0; r < 8; ++r) m[r] = min(o1[r] + b + 4, (b == 0) ? o0[r] : min(o0[r] + b, m[r]));
        }
      } else {
#pragma unroll
        for (int b = 0; b < F_B; ++b) {
          if (b >= nb) break;               // last octet of a search width that is not a multiple of 8 (warp uniform)
          int p[8], o[8];
          p[0] = V[0][b];
#pragma unroll
          for (int a = 1; a < 8; ++a) p[a] = p[a - 1] + V[a][b];
          window_sums<KX>(p, o);
#pragma unroll
          for (int r = 0; r < 8; ++r) m[r] = (b == 0) ? o[r] : min(o[r] + b, m[r]);
        }
      }
      // ---- running best: high words hold cost*8 | 7, so m <= s <=> cost <= best cost.  Equal costs are candidates
      //      too: another warp may hold the same cost at a later disparity ----
      bool cand = false;
#pragma unroll
      for (int r = 0; r < 8; ++r) cand |= ((uint32_t)m[r] <= brow[r * 32]);
      if (cand) {                // rare once the search has seen the neighbourhood of the true match
        // The thresholds are read again (volatile), so the common path keeps one predicate rather than eight.  A threshold
        // lowered meanwhile by another warp only holds back an offer that could not win.
        const volatile uint32_t* vrow = brow;
        unsigned long long* krow = keys + y * F_COLS + lane;
#pragma unroll
        for (int r = 0; r < 8; ++r)
          if ((uint32_t)m[r] <= vrow[r * 32]) offer_key(brow + r * 32, krow + r * 32, (uint32_t)m[r] | 7u, (uint32_t)(idx_base + (m[r] & 7)));
      }
      brow += F_COLS;
      if (++y == yend) break;
      slide();
    }
    if (y == nrows) break;
    if (y == ynew) rnew -= rspan;
    if (y == yold) rold -= rspan;
    slide();
  }
}

// ---- SquaredCost variant of the integer pass ----------------------------------------------------------------
// (a-b)^2 of integer imagery is an exact integer in the reference's float arithmetic as long as |a-b| < 4096, and
// the double window sums are exact; here they are uint32 (the host checks kx*ky*range^2 < 2^32).  Costs do not
// leave room for the key trick, so the arg-min over the octet is tracked with compare/select.
template <int KX>
__device__ __forceinline__ void fast_pass_sq(const uint16_t* __restrict__ ltile, const uint16_t* __restrict__ rring,
                                             uint32_t* __restrict__ best, unsigned long long* __restrict__ keys,
                                             int lane, int g, int ky, int ring_slots, int rw, int ring_base, int idx_base, int nrows, int nb) {
  int V[8][F_B];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < F_B; ++b) V[a][b] = 0;
  const uint16_t* lp = ltile + 8 * lane;
  const uint16_t* rp = rring + 8 * (lane + g);
  int slot_new = ring_base;
  for (int t = 0; t < ky; ++t) {
    int Lv[8], Rv[16];
    load_row<false>(lp + t * F_COLS, rp + slot_new * rw, Lv, Rv);
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
      for (int b = 0; b < F_B; ++b) { const int d = Lv[a] - Rv[a + b]; V[a][b] += d * d; }
    if (++slot_new == ring_slots) slot_new = 0;
  }
  int slot_old = ring_base;
  for (int y = 0; y < nrows; ++y) {
    if (y > 0) {
      {
        int Lv[8], Rv[16];
        load_row<false>(lp + (y + ky - 1) * F_COLS, rp + slot_new * rw, Lv, Rv);
#pragma unroll
        for (int a = 0; a < 8; ++a)
#pragma unroll
          for (int b = 0; b < F_B; ++b) { const int d = Lv[a] - Rv[a + b]; V[a][b] += d * d; }
      }
      {
        int Lo[8], Ro[16];
        load_row<false>(lp + (y - 1) * F_COLS, rp + slot_old * rw, Lo, Ro);
#pragma unroll
        for (int a = 0; a < 8; ++a)
#pragma unroll
          for (int b = 0; b < F_B; ++b) { const int d = Lo[a] - Ro[a + b]; V[a][b] -= d * d; }
      }
      if (++slot_new == ring_slots) slot_new = 0;
      if (++slot_old == ring_slots) slot_old = 0;
    }
    uint32_t m[8];
    int mb[8];
#pragma unroll
    for (int b = 0; b < F_B; ++b) {
      if (b >= nb) break;
      int p[8], o[8];
      p[0] = V[0][b];
#pragma unroll
      for (int a = 1; a < 8; ++a) p[a] = p[a - 1] + V[a][b];     // wraps mod 2^32 like the uint32 sums they stand for
      window_sums<KX>(p, o);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const uint32_t c = (uint32_t)o[r];
        if (b == 0) { m[r] = c; mb[r] = 0; }
        else if (c < m[r]) { m[r] = c; mb[r] = b; }
      }
    }
    uint32_t* brow = best + y * F_COLS + lane;                 // high words: the uint32 cost
    unsigned long long* krow = keys + y * F_COLS + lane;
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if (m[r] <= brow[r * 32]) offer_key(brow + r * 32, krow + r * 32, m[r], (uint32_t)(idx_base + mb[r]));
  }
}

template <int KX, bool SQ = false>
__global__ void __launch_bounds__(FK_THREADS, 1)
k1_fast_abs_kernel(const uint16_t* __restrict__ L16, const uint16_t* __restrict__ R16, FastGeom G,
                   vwb200_dispi* __restrict__ out, ptrdiff_t opitch, uint32_t* __restrict__ part_cost, uint16_t* __restrict__ part_idx,
                   unsigned long long* __restrict__ gkeys) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint32_t* best = reinterpret_cast<uint32_t*>(smem);                                  // [th][8][32]: best high word
  unsigned long long* keys = gkeys + (size_t)blockIdx.x * G.th * F_COLS;               // [th][8][32]: (high word << 32) | raster index
  uint16_t* ltile = reinterpret_cast<uint16_t*>(smem + (size_t)G.th * F_COLS * 4);
  uint16_t* rring = ltile + (size_t)G.ltile_rows * F_COLS;
  uint64_t* bars = reinterpret_cast<uint64_t*>(rring + (size_t)G.ring_slots * G.rw);
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int ngroups = (G.sx + F_B - 1) / F_B, SD = G.sd;
  // above every integer key / above every uint32 cost; low word above every raster index
  const unsigned long long kinit = ((unsigned long long)(SQ ? 0xffffffffu : FK_INIT_HI) << 32) | 0xffffffffu;
  if (tid == 0) { mbar_init(&bars[0], 1); mbar_init(&bars[1], 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  uint32_t ph0 = 0, ph1 = 0;
  const uint32_t lbytes = (uint32_t)G.ltile_rows * F_COLS * 2, rrow_bytes = (uint32_t)G.rw * 2;
  for (int item = blockIdx.x; item < G.NS * G.NB * G.J; item += gridDim.x) {
    const int chunk = item % G.J, rest = item / G.J;
    const int strip = rest % G.NS, band = rest / G.NS;
    const int y0 = band * G.th, nrows = min(G.th, G.H - y0);
    const int dy0 = chunk * G.dy_per, ndy = min(G.sy, dy0 + G.dy_per) - dy0;
    const uint16_t* lsrc = L16 + ((size_t)strip * G.lrows + y0) * F_COLS;
    const uint16_t* rsrc = R16 + ((size_t)strip * G.rrows + y0 + dy0) * G.rw;
    if (tid == 0) {
      // first period: right rows 0 .. ltile_rows + min(sd, ndy) - 2 -> slots 0.. (never past the chunk's last row)
      const uint32_t rbytes0 = (uint32_t)(G.ltile_rows + min(SD, ndy) - 1) * rrow_bytes;
      fence_proxy_async();
      mbar_expect_tx(&bars[0], lbytes + rbytes0);
      tma_load_1d(ltile, lsrc, lbytes, &bars[0]);
      tma_load_1d(rring, rsrc, rbytes0, &bars[0]);
    }
    for (int k = tid; k < nrows * F_COLS; k += FK_THREADS) { best[k] = (uint32_t)(kinit >> 32); keys[k] = kinit; }
    __syncthreads();
    mbar_wait(&bars[0], ph0); ph0 ^= 1;
    for (int dyp = 0; dyp < ndy; dyp += SD) {      // periods of sd dy rows, relative to the chunk's first row dy0
      const int dcur = min(SD, ndy - dyp);               // dy rows of this period
      const int nnext = min(SD, ndy - dyp - dcur);       // dy rows of the next one: their last right rows are fetched now
      if (tid == 0 && nnext > 0) {                       // into the slots the previous period freed
        fence_proxy_async();
        mbar_expect_tx(&bars[1], (uint32_t)nnext * rrow_bytes);
        for (int j = 0; j < nnext; ++j) {
          const int rr = dyp + SD - 1 + G.ltile_rows + j;
          tma_load_1d(rring + (size_t)(rr % G.ring_slots) * G.rw, rsrc + (size_t)rr * G.rw, rrow_bytes, &bars[1]);
        }
      }
      // units u = dl * ngroups + g of the period, dealt statically: warp w runs u = w, w + 12, ...  Warps on different dy
      // of the period offer to the same key plane; the 64-bit atomicMin makes the result independent of their timing.
      for (int u = w; u < dcur * ngroups; u += FK_WARPS) {
        const int dy = dyp + u / ngroups, g = u % ngroups;
        const int ring_base = dy % G.ring_slots;
        const int idx_base = (dy0 + dy) * G.sx + F_B * g;
        if (SQ) fast_pass_sq<KX>(ltile, rring, best, keys, lane, g, G.ky, G.ring_slots, G.rw, ring_base, idx_base, nrows, min(F_B, G.sx - F_B * g));
        else if (G.sx - F_B * g >= F_B)
          fast_pass<KX, true>(ltile, rring, best, keys, lane, g, G.ky, G.ring_slots, G.rw, ring_base, idx_base, nrows, F_B);
        else
          fast_pass<KX, false>(ltile, rring, best, keys, lane, g, G.ky, G.ring_slots, G.rw, ring_base, idx_base, nrows, G.sx - F_B * g);
      }
      if (nnext > 0) { mbar_wait(&bars[1], ph1); ph1 ^= 1; }
      __syncthreads();
    }
    // ---- write {dx, dy, valid} (or this dy chunk's partial result) ----
    const int s0 = strip * G.out_cols;
    for (int pix = tid; pix < nrows * G.out_cols; pix += FK_THREADS) {
      const int x = pix % G.out_cols, y = pix / G.out_cols;
      const int gx = s0 + x, gy = y0 + y;
      if (gx >= G.W) continue;
      // the reductions were performed in L2 after the barrier that ended the dy loop: read past L1
      const unsigned long long key = __ldcg(keys + y * F_COLS + (x & 7) * 32 + (x >> 3));
      const int bidx = (int)(uint32_t)key;
      if (G.J > 1) {             // partial result of this dy chunk; k1_fast_merge_kernel finishes the pixel
        const size_t pk = ((size_t)chunk * G.H + gy) * G.W + gx;
        part_cost[pk] = (uint32_t)(key >> 32); part_idx[pk] = (uint16_t)bidx;
        continue;
      }
      vwb200_dispi o;
      o.dx = bidx % G.sx + G.addx; o.dy = bidx / G.sx + G.addy; o.valid = 1;
      out[(ptrdiff_t)gy * opitch + gx] = o;
    }
    __syncthreads();
  }
}

// merge of the dy chunks (ascending chunk = ascending raster order: an equal cost keeps the earlier chunk)
__global__ void k1_fast_merge_kernel(FastGeom G, const uint32_t* __restrict__ part_cost, const uint16_t* __restrict__ part_idx,
                                     vwb200_dispi* __restrict__ out, ptrdiff_t opitch) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= G.W || y >= G.H) return;
  const size_t plane = (size_t)G.W * G.H, k = (size_t)y * G.W + x;
  uint32_t best = part_cost[k];
  int bidx = part_idx[k];
  for (int c = 1; c < G.J; ++c) {
    const uint32_t cc = part_cost[c * plane + k];
    if (cc < best) { best = cc; bidx = part_idx[c * plane + k]; }
  }
  vwb200_dispi o;
  o.dx = bidx % G.sx + G.addx; o.dy = bidx / G.sx + G.addy; o.valid = 1;
  out[(ptrdiff_t)y * opitch + x] = o;
}

// ---- "every disparity gave the same cost" fix-up for pixels whose arg-best is (0,0) --------------------------
__global__ void k1_fast_allequal_fixup(ImgF L, ImgF R, FastGeom g, vwb200_dispi* __restrict__ out, ptrdiff_t opitch) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= g.W || y >= g.H) return;
  vwb200_dispi* o = out + (ptrdiff_t)y * opitch + x;
  if (o->dx != g.addx || o->dy != g.addy) return;
  // arg-best (0,0): valid iff some disparity has a different (necessarily larger) cost.  Integer-valued inputs:
  // exact integer arithmetic.  Reads follow the pack kernels (constant edge extension around the logical rasters).
  auto lv = [&](int xx, int yy) { return (int)L.p[(ptrdiff_t)min(max(g.loy + yy, 0), L.h - 1) * L.pitch + min(max(g.lox + xx, 0), L.w - 1)]; };
  auto rv = [&](int xx, int yy) { return (int)R.p[(ptrdiff_t)min(max(g.roy + yy, 0), R.h - 1) * R.pitch + min(max(g.rox + xx, 0), R.w - 1)]; };
  long long c0 = 0;
  for (int j = 0; j < g.ky; ++j)
    for (int i = 0; i < g.kx; ++i) { const long long d = lv(x + i, y + j) - rv(x + i, y + j); c0 += g.scale == 1 ? d * d : (d < 0 ? -d : d); }
  for (int dy = 0; dy < g.sy; ++dy)
    for (int dx = 0; dx < g.sx; ++dx) {
      if (dx == 0 && dy == 0) continue;
      long long c = 0;
      for (int j = 0; j < g.ky; ++j)
        for (int i = 0; i < g.kx; ++i) { const long long d = lv(x + i, y + j) - rv(x + i + dx, y + j + dy); c += g.scale == 1 ? d * d : (d < 0 ? -d : d); }
      if (c != c0) return;      // not all equal -> stays valid
    }
  o->valid = 0;
}

int k1_fast_launch(int cost, ImgF left, ImgF right, int W, int H, int sx, int sy, int kx, int ky, float vmin, float vmax,
                   vwb200_dispi* out, ptrdiff_t opitch, void* workspace, size_t workspace_bytes, cudaStream_t st,
                   const KEvents* ev, const FastOrigin* org) {
  (void)workspace_bytes;
  const bool sq = cost == VWB200_SQUARED_DIFFERENCE;
  FastGeom g = fast_geom(W, H, sx, sy, kx, ky);
  g.scale = sq ? 1 : F_B;
  if (org) { g.lox = org->lox; g.loy = org->loy; g.rox = org->rox; g.roy = org->roy; g.addx = org->addx; g.addy = org->addy; }
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  uint16_t* L16 = reinterpret_cast<uint16_t*>(ws);
  uint16_t* R16 = L16 + (size_t)g.NS * g.lrows * F_COLS;
  uint32_t* part_cost = reinterpret_cast<uint32_t*>((reinterpret_cast<uintptr_t>(R16 + (size_t)g.NS * g.rrows * g.rw) + 63) & ~(uintptr_t)63);
  uint16_t* part_idx = reinterpret_cast<uint16_t*>(part_cost + (size_t)g.J * W * H);
  const uintptr_t kbase = g.J > 1 ? reinterpret_cast<uintptr_t>(part_idx + (size_t)g.J * W * H) : reinterpret_cast<uintptr_t>(part_cost);
  unsigned long long* gkeys = reinterpret_cast<unsigned long long*>((kbase + 63) & ~(uintptr_t)63);
  {
    dim3 gl(g.lrows, g.NS), gr(g.rrows, g.NS);
    pack_left_kernel<<<gl, 256, 0, st>>>(left, vmin, g, L16);
    VWB_LAUNCH_CHECK();
    pack_right_kernel<<<gr, 256, 0, st>>>(right, vmin, g, R16);
    VWB_LAUNCH_CHECK();
  }
  int dev = 0, nsm = kNumSMs;
  VWB_CUDA(cudaGetDevice(&dev));
  VWB_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
  const int items = g.NS * g.NB * g.J;
  const int grid = std::min(items, std::min(nsm, kNumSMs));      // the workspace holds kNumSMs key planes
  const size_t smem = fast_smem_bytes(g);
  void (*kern)(const uint16_t*, const uint16_t*, FastGeom, vwb200_dispi*, ptrdiff_t, uint32_t*, uint16_t*, unsigned long long*) = nullptr;
  switch (kx) {
#define KCASE(K) case K: kern = sq ? k1_fast_abs_kernel<K, true> : k1_fast_abs_kernel<K, false>; break;
    KCASE(3) KCASE(5) KCASE(7) KCASE(9) KCASE(11) KCASE(13) KCASE(15) KCASE(17) KCASE(19) KCASE(21) KCASE(23) KCASE(25)
    KCASE(27) KCASE(29) KCASE(31)
#undef KCASE
    default: set_error("k1_fast: unsupported kernel width %d", kx); return VWB200_ENOIMPL;
  }
  VWB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FK_SMEM));   // per-function state shared by all host threads: device maximum
  if (ev && ev->e0) cudaEventRecord(ev->e0, st);
  kern<<<grid, FK_THREADS, smem, st>>>(L16, R16, g, out, opitch, part_cost, part_idx, gkeys);
  VWB_LAUNCH_CHECK();
  if (ev && ev->e1) cudaEventRecord(ev->e1, st);
  if (g.J > 1) {
    dim3 mb(32, 8), mg((W + 31) / 32, (H + 7) / 8);
    k1_fast_merge_kernel<<<mg, mb, 0, st>>>(g, part_cost, part_idx, out, opitch);
    VWB_LAUNCH_CHECK();
  }
  dim3 b(32, 8), gg((W + 31) / 32, (H + 7) / 8);
  k1_fast_allequal_fixup<<<gg, b, 0, st>>>(left, right, g, out, opitch);
  VWB_LAUNCH_CHECK();
  return VWB200_OK;
}

}  // namespace vwb200
