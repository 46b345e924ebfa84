// row_step_bench.cu -- cycles per warp row step of K1 fast's AbsoluteCost row step (fast_pass<21, true> of
// csrc/k1_fast.cu), run on synthetic shared-memory rows at the kernel's occupancy: one CTA of 12 warps per SM, the
// headline's 84-row band, 21 x 21 kernel and 128-wide search, each warp sliding 4 (dy, octet) units over the band, and
// each period of 3 dy starting 3 ring rows further on, so that the passes cross the end of the ring as in the kernel.
// Variants of the row step, to see which part sets its pace:
//   full       the row step as the kernel runs it (horizontal window sums + arg-best + threshold test, then the slide)
//   slide      the vertical slide alone (loads, u16 unpack, VABSDIFF accumulate / subtract, pointer advance)
//   horizontal the horizontal stage and threshold test alone, on vertical sums that the compiler must treat as new
//              every row (an empty asm statement, no instruction)
// The body is a copy of the kernel's row step and shares window_sums2 with it (csrc/k1_fast_common.cuh); keep the two
// in step when either changes.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/row_step_bench tools/row_step_bench.cu
// Usage: tools/row_step_bench [reps]   (default 20 sweeps of the band per warp)
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../visionworkbench_b200/csrc/k1_fast_common.cuh"

using namespace vwb200;

enum Variant { FULL = 0, SLIDE = 1, HORIZONTAL = 2 };
static const char* kVariantName[] = {"full", "slide", "horizontal"};

static constexpr int KX = 21, KY = 21, SX = 128, SD = 3, TH = 84, WARPS = 12;
static constexpr int NGROUPS = SX / F_B;
static constexpr int LTILE_ROWS = TH + KY - 1;
static constexpr int RING_SLOTS = LTILE_ROWS + 2 * SD - 1;
static constexpr int RW = ((F_COLS + SX + 7) / 8) * 8 + 8;
static constexpr size_t SMEM = (size_t)TH * F_COLS * 4 + (size_t)LTILE_ROWS * F_COLS * 2 + (size_t)RING_SLOTS * RW * 2;

__device__ __forceinline__ void unpack2(const uint32_t v, int& lo, int& hi) {
  uint32_t h, l;
  asm("mul.hi.u32 %0, %1, 65536;" : "=r"(h) : "r"(v));
  asm("mad.lo.u32 %0, %1, -65536, %2;" : "=r"(l) : "r"(h), "r"(v));
  lo = (int)l; hi = (int)h;
}
__device__ __forceinline__ void unpack8(const uint4 v, int (&o)[8]) {
  unpack2(v.x, o[0], o[1]); unpack2(v.y, o[2], o[3]); unpack2(v.z, o[4], o[5]); unpack2(v.w, o[6], o[7]);
}
__device__ __forceinline__ void load_row(const uint16_t* lrow, const uint16_t* rrow, int (&Lv)[8], int (&Rv)[16]) {
  unpack8(*reinterpret_cast<const uint4*>(lrow), Lv);
  int t[8];
  unpack8(*reinterpret_cast<const uint4*>(rrow), t);
#pragma unroll
  for (int i = 0; i < 8; ++i) Rv[i] = t[i];
  unpack8(*reinterpret_cast<const uint4*>(rrow + 8), t);
#pragma unroll
  for (int i = 0; i < 8; ++i) Rv[8 + i] = t[i];
}

// The band geometry arrives at run time, as in the kernel, so the compiler cannot unroll or specialise the row loop.
struct Geom { int ky, nrows, ring_slots, rw; };

// One (dy, octet) pass; returns the clock64 cycles of its row loop (the seeding excluded).  Offers are counted, not
// made: the threshold plane is 0, below every key, so the rare path never runs.
template <int VAR>
__device__ __forceinline__ long long pass(const uint16_t* ltile, const uint16_t* rring, const uint32_t* best, int lane,
                                          int g, int ring_base, Geom G, int& sink) {
  int V[8][F_B];
  const uint16_t* lnew = ltile + 8 * lane;
  const uint16_t* lold = lnew;
  const uint16_t* const rring_lane = rring + 8 * (lane + g);
  const uint16_t* const rend = rring_lane + G.ring_slots * G.rw;
  const int rspan = G.ring_slots * G.rw;
  const uint16_t* rnew = rring_lane + ring_base * G.rw;
  const uint16_t* rold = rnew;
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < F_B; ++b) V[a][b] = 0;
  for (int t = 0; t < G.ky; ++t) {
    if (rnew == rend) rnew -= rspan;
    int Lv[8], Rv[16];
    load_row(lnew, rnew, Lv, Rv);
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
      for (int b = 0; b < F_B; ++b) V[a][b] = __sad(Lv[a], Rv[a + b], V[a][b]);
    lnew += F_COLS;
    rnew += G.rw;
  }
  auto slide = [&]() {
    if (VAR == HORIZONTAL) {
#pragma unroll
      for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < F_B; ++b) asm volatile("" : "+r"(V[a][b]));
      return;
    }
    {
      int Lv[8], Rv[16];
      load_row(lnew, rnew, Lv, Rv);
#pragma unroll
      for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < F_B; ++b) V[a][b] = __sad(Lv[a], Rv[a + b], V[a][b]);
    }
    {
      int Lo[8], Ro[16];
      load_row(lold, rold, Lo, Ro);
#pragma unroll
      for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < F_B; ++b) V[a][b] -= __sad(Lo[a], Ro[a + b], 0);
    }
    lnew += F_COLS; lold += F_COLS;
    rnew += G.rw; rold += G.rw;
  };
  const int ynew = G.ring_slots - ring_base - G.ky + 1, yold = ynew + G.ky;
  const uint32_t* brow = best + lane;
  int offers = 0;
  const long long t0 = clock64();
  for (int y = 0;;) {
    const int yend = min(G.nrows, y < ynew ? ynew : y < yold ? yold : G.nrows);
    for (;;) {
      if (VAR != SLIDE) {
        int m[8];
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
        bool cand = false;
#pragma unroll
        for (int r = 0; r < 8; ++r) cand |= ((uint32_t)m[r] <= brow[r * 32]);
        if (cand) ++offers;
      }
      brow += F_COLS;
      if (++y == yend) break;
      slide();
    }
    if (y == G.nrows) break;
    if (y == ynew) rnew -= rspan;
    if (y == yold) rold -= rspan;
    slide();
  }
  const long long t1 = clock64();
  int s = offers;
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < F_B; ++b) s += V[a][b];
  sink += s;
  return t1 - t0;
}

template <int VAR>
__global__ void __launch_bounds__(WARPS * 32, 1) row_step_kernel(const uint16_t* __restrict__ gl, const uint16_t* __restrict__ gr,
                                                                 Geom G, int reps, long long* __restrict__ cycles, int* __restrict__ sink) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint32_t* best = reinterpret_cast<uint32_t*>(smem);
  uint16_t* ltile = reinterpret_cast<uint16_t*>(smem + (size_t)TH * F_COLS * 4);
  uint16_t* rring = ltile + (size_t)LTILE_ROWS * F_COLS;
  for (int k = threadIdx.x; k < TH * F_COLS; k += blockDim.x) best[k] = 0;
  for (int k = threadIdx.x; k < LTILE_ROWS * F_COLS; k += blockDim.x) ltile[k] = gl[k];
  for (int k = threadIdx.x; k < RING_SLOTS * RW; k += blockDim.x) rring[k] = gr[k];
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  long long cyc = 0;
  int s = 0;
  for (int rep = 0; rep < reps; ++rep)
    for (int u = w; u < SD * NGROUPS; u += WARPS) cyc += pass<VAR>(ltile, rring, best, lane, u % NGROUPS, (rep * SD + u / NGROUPS) % G.ring_slots, G, s);
  if (lane == 0) cycles[blockIdx.x * WARPS + w] = cyc;
  sink[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int VAR>
static void run(const uint16_t* dl, const uint16_t* dr, int nsm, int reps) {
  auto kern = row_step_kernel<VAR>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM);
  long long* dc; int* ds;
  cudaMalloc(&dc, (size_t)nsm * WARPS * 8);
  cudaMalloc(&ds, (size_t)nsm * WARPS * 32 * 4);
  const Geom G = {KY, TH, RING_SLOTS, RW};
  kern<<<nsm, WARPS * 32, SMEM>>>(dl, dr, G, 1, dc, ds);                 // warm-up
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  kern<<<nsm, WARPS * 32, SMEM>>>(dl, dr, G, reps, dc, ds);
  cudaEventRecord(e1);
  cudaError_t err = cudaEventSynchronize(e1);
  if (err != cudaSuccess) { fprintf(stderr, "%s: %s\n", kVariantName[VAR], cudaGetErrorString(err)); exit(1); }
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  std::vector<long long> h((size_t)nsm * WARPS);
  cudaMemcpy(h.data(), dc, h.size() * 8, cudaMemcpyDeviceToHost);
  double avg = 0; for (long long c : h) avg += (double)c; avg /= (double)h.size();
  // a warp runs SD*NGROUPS/WARPS passes of TH-1 row steps (plus the first row) per rep; 3 warps share a sub-partition
  const double steps = (double)reps * (SD * NGROUPS / WARPS) * TH;
  printf("%-11s %8.1f cycles per warp row step per sub-partition  (%.1f per warp, %.2f ms)\n", kVariantName[VAR],
         avg / steps / (WARPS / 4), avg / steps, ms);
  cudaFree(dc); cudaFree(ds);
}

int main(int argc, char** argv) {
  const int reps = argc > 1 ? atoi(argv[1]) : 20;
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  printf("%s  SMs=%d  kx=%d ky=%d sx=%d  %d warps per SM  %d-row band  reps=%d\n", p.name, p.multiProcessorCount, KX, KY, SX,
         WARPS, TH, reps);
  // 12-bit values packed as the kernel packs them, (v - vmin) * 8
  std::vector<uint16_t> hl((size_t)LTILE_ROWS * F_COLS), hr((size_t)RING_SLOTS * RW);
  uint32_t st = 12345u;
  auto rnd = [&]() { st = st * 1664525u + 1013904223u; return (uint16_t)(((st >> 16) % 4096u) * 8u); };
  for (auto& v : hl) v = rnd();
  for (auto& v : hr) v = rnd();
  uint16_t *dl, *dr;
  cudaMalloc(&dl, hl.size() * 2); cudaMalloc(&dr, hr.size() * 2);
  cudaMemcpy(dl, hl.data(), hl.size() * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(dr, hr.data(), hr.size() * 2, cudaMemcpyHostToDevice);
  run<FULL>(dl, dr, p.multiProcessorCount, reps);
  run<SLIDE>(dl, dr, p.multiProcessorCount, reps);
  run<HORIZONTAL>(dl, dr, p.multiProcessorCount, reps);
  return 0;
}
