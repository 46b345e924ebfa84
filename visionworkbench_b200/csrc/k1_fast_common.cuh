// k1_fast_common.cuh -- pieces shared by the exact-integer fast kernels (k1_fast.cu: AbsoluteCost / SquaredCost,
// k1_screen.cu: NCC and SquaredCost screening): tile geometry, mbarrier + TMA bulk-copy PTX wrappers, shuffle-based window sums.
#pragma once
#include "common.cuh"

namespace vwb200 {

static constexpr int F_TH = 32;        // output rows per band of k1_screen (k1_fast: FastGeom::th)
static constexpr int F_COLS = 256;     // padded columns per strip (32 lanes x 8)
static constexpr int F_WARPS = 8;       // per CTA (2 per SM sub-partition)
static constexpr int F_THREADS = F_WARPS * 32;
static constexpr int F_B = 8;          // consecutive dx per thread (one "octet"); keys are cost*8 + b

// ---- geometry -----------------------------------------------------------------------------------------
struct FastGeom {
  int W, H, sx, sy, kx, ky;
  int out_cols;      // output columns per strip = 256 - (kx-1)
  int NS, NB;        // strips, bands
  int lrows, rrows;  // padded row counts of the packed arrays
  int ltile_rows;    // th + ky - 1
  int ring_slots;    // th + ky; ltile_rows + 2*sd - 1 with periods of sd dy rows
  int rw;            // u16 per packed right row = 256 + sx (multiple of 8)
  int scale;                // values are packed as (v - vmin) * scale: 8 for AbsoluteCost (keys = cost*8+b), 1 for SquaredCost
  int J, dy_per;            // the dy range is split into J chunks of dy_per rows (more, smaller work items for small rasters)
  int lox, loy, rox, roy;   // origin of the (logical) left / right rasters inside the images passed to the pack kernels
  int addx, addy;           // constant added to the output disparities
  int sd;                   // dy rows per synchronisation period (ring depth)
  int th;                   // output rows per band (F_TH for k1_screen; k1_fast sizes it from its shared-memory budget)
};
static inline FastGeom make_geom(int W, int H, int sx, int sy, int kx, int ky, int th = F_TH) {
  FastGeom g;
  g.W = W; g.H = H; g.sx = sx; g.sy = sy; g.kx = kx; g.ky = ky; g.th = th;
  g.out_cols = F_COLS - (kx - 1);
  g.NS = (W + g.out_cols - 1) / g.out_cols;
  g.NB = (H + th - 1) / th;
  g.ltile_rows = th + ky - 1;
  g.ring_slots = th + ky;
  g.lrows = g.NB * th + ky - 1;
  g.rrows = g.NB * th + ky - 1 + sy;
  g.rw = ((F_COLS + sx + 7) / 8) * 8 + 8;
  g.lox = g.loy = g.rox = g.roy = 0; g.addx = g.addy = 0; g.scale = F_B; g.sd = 1;
  // The work items (strip x band x dy-chunk) are dealt round-robin to kNumSMs persistent CTAs, so the last partial wave idles
  // part of the chip: 1120 items = 8.48 waves run as 9 (efficiency 0.943 -- the 8-GPU share of the 8192^2 raster).  Split
  // the dy range into J chunks (merged by k1_fast_merge) so that items * J fills its last wave: pick the J with the best
  // wave efficiency, charging each extra chunk a fixed 0.004 for its partial planes and the merge pass.  Small
  // rasters additionally want >= ~6 waves for balance.
  g.J = 1;
  const int items = g.NS * g.NB;
  const int jmax = sy / 8 < 1 ? 1 : (sy / 8 > 8 ? 8 : sy / 8);
  if (items < 64 * kNumSMs) {
    double best = -1.0;
    for (int J = 1; J <= jmax; ++J) {
      const double w = (double)items * J / kNumSMs;
      const long long full = (long long)((items * (long long)J + kNumSMs - 1) / kNumSMs);
      double eff = w / (double)full * (1.0 - 0.004 * (J - 1));
      if (w < 6.0) eff *= 0.5 + w / 12.0;          // few waves: uneven items (edge strips / bands) are not averaged out
      if (eff > best + 1e-9) { best = eff; g.J = J; }
    }
  }
  g.dy_per = (sy + g.J - 1) / g.J;
  g.J = (sy + g.dy_per - 1) / g.dy_per;
  return g;
}
// ---- PTX helpers: mbarrier + TMA bulk copy -----------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra WAIT_%=;\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- horizontal kx-window sums of 8 per-lane columns via in-lane prefix + warp shuffles -----------------------
// p[a] = inclusive prefix of the lane's 8 column sums.  out[r] = sum of the KX columns starting at
// column 8*lane + r.  Static structure for a given KX (all loops unrolled).
template <int KX>
__device__ __forceinline__ void window_sums(const int (&p)[8], int (&out)[8]) {
  const int T = p[7];
  constexpr int MAXL = (KX - 1) / 8;            // most full following lanes any window needs
  // W[k] = T_l + T_{l+1} + ... + T_{l+k}
  int W[MAXL + 1];
  W[0] = T;
#pragma unroll
  for (int k = 1; k <= MAXL; ++k) W[k] = W[k - 1] + __shfl_down_sync(0xffffffffu, T, k);
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int own = 8 - r;                      // columns available in the own lane from r
    if (KX <= own) {
      out[r] = r ? p[r + KX - 1] - p[r - 1] : p[KX - 1];
    } else {
      const int rem = KX - own;                 // columns still needed from the following lanes
      const int full = rem / 8, part = rem % 8;
      if (part) {
        const int q = __shfl_down_sync(0xffffffffu, p[part - 1], full + 1);
        out[r] = r ? (W[full] + q) - p[r - 1] : W[full] + q;      // one IADD3
      } else {
        out[r] = r ? W[full] - p[r - 1] : W[full];
      }
    }
  }
}

// window_sums of two independent prefix rows (two dx of an octet), the same outputs: every shuffle of both is issued
// before the adds that consume them, so each batch of shuffles has two chains to overlap instead of one.
template <int KX>
__device__ __forceinline__ void window_sums2(const int (&p0)[8], const int (&p1)[8], int (&o0)[8], int (&o1)[8]) {
  constexpr int MAXL = (KX - 1) / 8;
  int t0[MAXL + 1], t1[MAXL + 1], q0[8], q1[8];
#pragma unroll
  for (int k = 1; k <= MAXL; ++k) {
    t0[k] = __shfl_down_sync(0xffffffffu, p0[7], k);
    t1[k] = __shfl_down_sync(0xffffffffu, p1[7], k);
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int rem = KX - (8 - r), full = rem / 8, part = rem % 8;
    if (rem > 0 && part) {
      q0[r] = __shfl_down_sync(0xffffffffu, p0[part - 1], full + 1);
      q1[r] = __shfl_down_sync(0xffffffffu, p1[part - 1], full + 1);
    }
  }
  int W0[MAXL + 1], W1[MAXL + 1];
  W0[0] = p0[7]; W1[0] = p1[7];
#pragma unroll
  for (int k = 1; k <= MAXL; ++k) { W0[k] = W0[k - 1] + t0[k]; W1[k] = W1[k - 1] + t1[k]; }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const int rem = KX - (8 - r), full = rem / 8, part = rem % 8;
    if (rem <= 0) {
      o0[r] = r ? p0[r + KX - 1] - p0[r - 1] : p0[KX - 1];
      o1[r] = r ? p1[r + KX - 1] - p1[r - 1] : p1[KX - 1];
    } else if (part) {
      o0[r] = r ? (W0[full] + q0[r]) - p0[r - 1] : W0[full] + q0[r];
      o1[r] = r ? (W1[full] + q1[r]) - p1[r - 1] : W1[full] + q1[r];
    } else {
      o0[r] = r ? W0[full] - p0[r - 1] : W0[full];
      o1[r] = r ? W1[full] - p1[r - 1] : W1[full];
    }
  }
}


}  // namespace vwb200
