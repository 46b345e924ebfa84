// k11_ipmatch.cu -- K11: exact brute-force interest point matching (InterestPoint/Matcher.h:415-509,
// Matcher.cc:33-100): for every query descriptor the lowest-index nearest candidate of the same polarity and the
// second-nearest distance, by L2NormMetric or HammingMetric, then the reference's ratio test.
//
// The match kernel is shaped like an SGEMM: a CTA owns kBM queries x a range of candidates, both descriptor lists go through
// shared memory in chunks of kKC elements, and each thread keeps a kTM x kTN micro-tile of running distances in registers
// across the chunks, so every pair accumulates k = 0..D-1 in order for any D.  L2 rounds each step as the reference's x86-64
// code does -- sub, mul, add, no FMA (the intrinsics below keep nvcc's default --fmad=true from contracting them).  Chunks are
// zero-padded past D: (0 - 0)^2 = +0 and popc(0 ^ 0) = 0 leave every sum, inf and NaN included, unchanged.
#include "common.cuh"
#include <cfloat>
#include <math_constants.h>
#include <climits>
#include <type_traits>

namespace vwb200 {
namespace {

constexpr int kBM = 64, kBN = 64, kKC = 16, kTM = 4, kTN = 4, kThreads = 256;
constexpr int kPad = 4;                       // row padding of the staged chunks: 2-way instead of 16-way store conflicts

__device__ __forceinline__ void top2_insert(IpTop2& t, float d, int j) {
  // candidates arrive in ascending j: strict < keeps the lowest j among equal minima, a distance equal to best becomes second,
  // and an inf or NaN distance is never taken (the reference's double first_pick / second_pick start at 1e100)
  if (d < t.best) { t.second = t.best; t.best = d; t.j = j; }
  else if (d < t.second) t.second = d;
}

// two summaries of disjoint candidate sets: the smaller (best, j) wins and the second is the smaller of the winner's second
// and the loser's best -- the lowest j among equal minima and the second-smallest distance of the union, whatever the order
__device__ __forceinline__ IpTop2 ip_merge(IpTop2 a, IpTop2 c) {
  const bool cw = c.best < a.best || (c.best == a.best && c.j < a.j);
  const IpTop2 w = cw ? c : a, l = cw ? a : c;
  return IpTop2{w.best, w.j, fminf(w.second, l.best)};
}

template <bool HAM>
__global__ void __launch_bounds__(kThreads) k11_match_kernel(const typename std::conditional<HAM, uint32_t, float>::type* __restrict__ A,
                                                             ptrdiff_t lda, const uint8_t* __restrict__ pa, int n1,
                                                             const typename std::conditional<HAM, uint32_t, float>::type* __restrict__ B,
                                                             ptrdiff_t ldb, const uint8_t* __restrict__ pb, int n2, int K, int per_split,
                                                             IpTop2* __restrict__ part) {
  typedef typename std::conditional<HAM, uint32_t, float>::type E;
  __shared__ __align__(16) E As[kKC][kBM + kPad];
  __shared__ __align__(16) E Bs[kKC][kBN + kPad];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int q0 = blockIdx.x * kBM;
  const int jbeg = blockIdx.y * per_split, jend = min(n2, jbeg + per_split);

  IpTop2 top[kTM];
  bool qpol[kTM];
#pragma unroll
  for (int i = 0; i < kTM; ++i) {
    top[i] = IpTop2{CUDART_INF_F, INT_MAX, CUDART_INF_F};
    const int q = q0 + ty * kTM + i;
    qpol[i] = q < n1 && pa[q] != 0;
  }

  for (int c0 = jbeg; c0 < jend; c0 += kBN) {
    E acc[kTM][kTN];
#pragma unroll
    for (int i = 0; i < kTM; ++i)
#pragma unroll
      for (int j = 0; j < kTN; ++j) acc[i][j] = E(0);

    for (int k0 = 0; k0 < K; k0 += kKC) {
#pragma unroll
      for (int e = threadIdx.x; e < kBM * kKC; e += kThreads) {
        const int r = e / kKC, k = e % kKC, kk = k0 + k;
        const int q = q0 + r, c = c0 + r;
        As[k][r] = (q < n1 && kk < K) ? A[(ptrdiff_t)q * lda + kk] : E(0);
        Bs[k][r] = (c < jend && kk < K) ? B[(ptrdiff_t)c * ldb + kk] : E(0);
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kKC; ++k) {
        E a[kTM], b[kTN];
#pragma unroll
        for (int i = 0; i < kTM; ++i) a[i] = As[k][ty * kTM + i];
#pragma unroll
        for (int j = 0; j < kTN; ++j) b[j] = Bs[k][tx * kTN + j];
#pragma unroll
        for (int i = 0; i < kTM; ++i)
#pragma unroll
          for (int j = 0; j < kTN; ++j) {
            if constexpr (HAM) {
              acc[i][j] += __popc(a[i] ^ b[j]);
            } else {
              const float d = __fsub_rn(a[i], b[j]);
              acc[i][j] = __fadd_rn(acc[i][j], __fmul_rn(d, d));
            }
          }
      }
      __syncthreads();
    }

#pragma unroll
    for (int j = 0; j < kTN; ++j) {
      const int c = c0 + tx * kTN + j;
      if (c >= jend) break;
      const bool cp = pb[c] != 0;
#pragma unroll
      for (int i = 0; i < kTM; ++i)
        if (qpol[i] == cp) top2_insert(top[i], (float)acc[i][j], c);   // Hamming: an integer <= 8 D <= 2^24, exact in float
    }
  }

  // the 16 threads of one query row are one half-warp: merge their summaries (order-free, see ip_merge)
#pragma unroll
  for (int i = 0; i < kTM; ++i) {
#pragma unroll
    for (int off = 8; off; off >>= 1) {
      IpTop2 o;
      o.best = __shfl_xor_sync(0xffffffffu, top[i].best, off);
      o.j = __shfl_xor_sync(0xffffffffu, top[i].j, off);
      o.second = __shfl_xor_sync(0xffffffffu, top[i].second, off);
      top[i] = ip_merge(top[i], o);
    }
    const int q = q0 + ty * kTM + i;
    if (tx == 0 && q < n1) part[(ptrdiff_t)blockIdx.y * n1 + q] = top[i];
  }
}

// the partial summaries of one query in split order, then the reference's ratio test in double
__global__ void k11_finalize_kernel(const IpTop2* __restrict__ part, int n1, int nsplit, double threshold, int* __restrict__ index,
                                    double* __restrict__ first, double* __restrict__ second, unsigned long long* __restrict__ matches) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n1) return;
  IpTop2 t{CUDART_INF_F, INT_MAX, CUDART_INF_F};
  for (int s = 0; s < nsplit; ++s) t = ip_merge(t, part[(ptrdiff_t)s * n1 + q]);
  const double f = t.best < CUDART_INF_F ? (double)t.best : 1e100;
  const double sd = t.second < CUDART_INF_F ? (double)t.second : 1e100;
  int m = t.best < CUDART_INF_F ? t.j : -1;
  if (f > threshold * sd) m = -1;
  index[q] = m;
  if (first) first[q] = f;
  if (second) second[q] = sd;
  if (m >= 0) atomicAdd(matches, 1ull);
}

// HammingMetric's static_cast<uint8> (truncation toward zero), four bytes per little-endian word, zero-padded to W words.
// A value outside (-1, 256) or NaN -- undefined behaviour in the reference -- lowers *bad to its row-major element index.
__global__ void k11_pack_kernel(const float* __restrict__ in, ptrdiff_t pitch, int n, int D, int W, uint32_t* __restrict__ out,
                                unsigned long long* __restrict__ bad) {
  const long long total = (long long)n * W;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(e / W), w = (int)(e % W);
    uint32_t word = 0;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int k = 4 * w + b;
      if (k >= D) break;
      const float v = in[(ptrdiff_t)r * pitch + k];
      if (!(v > -1.0f && v < 256.0f)) atomicMin(bad, (unsigned long long)r * D + k);
      else word |= (uint32_t)(int)v << (8 * b);
    }
    out[e] = word;
  }
}

template <bool HAM>
int match_grid(int n1, int n2, int* nsplit, int* per_split) {
  int occ = 0;
  VWB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k11_match_kernel<HAM>, kThreads, 0));
  const long long qtiles = (n1 + kBM - 1) / kBM, ctiles = (n2 + kBN - 1) / kBN;
  // few queries cannot fill the SMs: split the candidates over about four waves of CTAs; the partial summaries merge in
  // split order, and the merge is order-free, so the split never changes a result
  const long long want = (4ll * std::max(occ, 1) * kNumSMs + qtiles - 1) / qtiles;
  const long long s = std::max(1ll, std::min(ctiles, want));
  *per_split = (int)(((ctiles + s - 1) / s) * kBN);
  *nsplit = (int)((n2 + *per_split - 1) / *per_split);
  return VWB200_OK;
}

}  // namespace

int ip_match_launch(int metric, const float* d1, ptrdiff_t p1, const uint8_t* pol1, int n1, const float* d2, ptrdiff_t p2,
                    const uint8_t* pol2, int n2, int dim, double threshold, int* index, double* first, double* second, Arena& ar,
                    cudaStream_t st, IpMatchInfo* info) {
  const bool ham = metric == VWB200_METRIC_HAMMING;
  int nsplit = 0, per_split = 0;
  if (n2 > 0) {
    if (ham) VWB_TRY(match_grid<true>(n1, n2, &nsplit, &per_split));
    else VWB_TRY(match_grid<false>(n1, n2, &nsplit, &per_split));
  }
  info->splits = nsplit;
  IpTop2* part = nullptr;
  unsigned long long* counters;                                      // [0] matches, [1] / [2] first bad element of desc1 / desc2
  VWB_TRY(ar.alloc(&counters, 3));
  VWB_CUDA(cudaMemsetAsync(counters, 0, 8, st));
  VWB_CUDA(cudaMemsetAsync(counters + 1, 0xff, 16, st));
  if (nsplit > 0) {
    VWB_TRY(ar.alloc(&part, (size_t)nsplit * n1));
    const dim3 grid((n1 + kBM - 1) / kBM, nsplit);
    if (ham) {
      const int W = (dim + 3) / 4;
      uint32_t *w1, *w2;
      VWB_TRY(ar.alloc(&w1, (size_t)n1 * W));
      VWB_TRY(ar.alloc(&w2, (size_t)n2 * W));
      if (W > 0) {
        const long long t1 = (long long)n1 * W, t2 = (long long)n2 * W;
        k11_pack_kernel<<<(int)std::min<long long>((t1 + 255) / 256, 8 * kNumSMs), 256, 0, st>>>(d1, p1, n1, dim, W, w1, counters + 1);
        VWB_LAUNCH_CHECK();
        k11_pack_kernel<<<(int)std::min<long long>((t2 + 255) / 256, 8 * kNumSMs), 256, 0, st>>>(d2, p2, n2, dim, W, w2, counters + 2);
        VWB_LAUNCH_CHECK();
        VWB_CUDA(cudaMemcpyAsync(info->bad, counters + 1, 16, cudaMemcpyDeviceToHost, st));
        VWB_CUDA(cudaStreamSynchronize(st));
        if (info->bad[0] != ~0ull || info->bad[1] != ~0ull) return VWB200_EARG;     // the caller names the element
      }
      k11_match_kernel<true><<<grid, kThreads, 0, st>>>(w1, W, pol1, n1, w2, W, pol2, n2, W, per_split, part);
    } else {
      k11_match_kernel<false><<<grid, kThreads, 0, st>>>(d1, p1, pol1, n1, d2, p2, pol2, n2, dim, per_split, part);
    }
    VWB_LAUNCH_CHECK();
  }
  k11_finalize_kernel<<<(n1 + 255) / 256, 256, 0, st>>>(part, n1, nsplit, threshold, index, first, second, counters);
  VWB_LAUNCH_CHECK();
  VWB_CUDA(cudaMemcpyAsync(&info->matches, counters, 8, cudaMemcpyDeviceToHost, st));
  return VWB200_OK;
}

}  // namespace vwb200
