// microbench.cu -- per-SM issue throughput of the instructions the fused cost-volume kernel is built
// from, measured on an H100 (sm_90a).  Output feeds DESIGN.md's ALU/MIO roofline for K1.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench microbench.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define ITERS 4096
#define NCHAIN 8

template <int OP>
__global__ void __launch_bounds__(1024) bench(float* out, int seed, long long* cycles) {
  __shared__ float sm[4096];
  for (int i = threadIdx.x; i < 4096; i += blockDim.x) sm[i] = (float)(i + seed);
  __syncthreads();
  float f[NCHAIN]; int v[NCHAIN]; double d[NCHAIN];
#pragma unroll
  for (int k = 0; k < NCHAIN; ++k) { f[k] = (float)(threadIdx.x + k + seed); v[k] = threadIdx.x * 3 + k + seed; d[k] = f[k]; }
  float fa = (float)seed * 0.5f + 1.0f; int ia = seed | 1;
  const unsigned short* s16 = reinterpret_cast<const unsigned short*>(sm);
  long long t0 = clock64();
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll
    for (int k = 0; k < NCHAIN; ++k) {
      if (OP == 0) f[k] = __fadd_rn(f[k], fa);
      if (OP == 1) f[k] = __fmaf_rn(f[k], fa, fa);
      if (OP == 2) v[k] = v[k] + ia - it;                // IADD3
      if (OP == 3) v[k] = __sad(v[k], ia, v[k]);
      if (OP == 4) v[k] = min(v[k] + 0, ia ^ it);        // IMNMX (plus whatever the xor costs once)
      if (OP == 5) f[k] = fminf(f[k], fa);
      if (OP == 6) v[k] = (v[k] & ia) ^ it;               // LOP3
      if (OP == 7) v[k] = v[k] * ia + it;                 // IMAD
      if (OP == 8) v[k] = __shfl_down_sync(0xffffffffu, v[k], 3);
      if (OP == 9) f[k] = sm[(v[k] + threadIdx.x) & 4095] + f[k];        // LDS.32 + FADD (address dependent)
      if (OP == 10) v[k] = s16[(v[k] + threadIdx.x) & 8191] + v[k];      // LDS.U16 + IADD
      if (OP == 11) d[k] = __dadd_rn(d[k], (double)fa);
      if (OP == 12) f[k] = __fadd_rn(f[k], fabsf(fa - f[k]));           // sub + add|.|  (2 FADD, abs modifier free?)
      if (OP == 13) { int t = __vabsdiffs2(v[k], ia); v[k] += t; }
      if (OP == 14) v[k] = abs(v[k] - ia) + it;                           // IABS path
      if (OP == 15) { asm volatile("{.reg .pred p; setp.lt.s32 p, %1, %0; @p mov.s32 %0, %1;}" : "+r"(v[k]) : "r"(ia ^ it)); }
      if (OP == 16) { if (k & 1) f[k] = __fadd_rn(f[k], fa); else v[k] = __sad(v[k], ia, v[k]); }   // ALU and FMA pipes side by side
      if (OP == 17) v[k] = min(v[k] + ia, it);                                                       // VIADDMNMX
    }
  }
  long long t1 = clock64();
  float acc = 0; int iacc = 0; double dacc = 0;
#pragma unroll
  for (int k = 0; k < NCHAIN; ++k) { acc += f[k]; iacc += v[k]; dacc += d[k]; }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc + (float)iacc + (float)dacc;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int OP>
void run(const char* name, int threads, int blocks_per_sm, int nsm) {
  float* out; long long* cyc;
  int blocks = nsm * blocks_per_sm;
  cudaMalloc(&out, (size_t)blocks * threads * 4);
  cudaMalloc(&cyc, blocks * 8);
  bench<OP><<<blocks, threads>>>(out, 1, cyc);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  bench<OP><<<blocks, threads>>>(out, 2, cyc);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  long long h[4096]; cudaMemcpy(h, cyc, blocks * 8, cudaMemcpyDeviceToHost);
  double avg = 0; for (int i = 0; i < blocks; ++i) avg += h[i]; avg /= blocks;
  double warp_instr_per_sm = (double)ITERS * NCHAIN * (threads / 32) * blocks_per_sm;
  printf("%-22s threads/SM=%4d  cycles=%9.0f  warp-instr/clk/SM=%6.3f  lanes/clk/SM=%7.2f  (%.3f ms)\n", name,
         threads * blocks_per_sm, avg, warp_instr_per_sm / avg, 32 * warp_instr_per_sm / avg, ms);
  cudaFree(out); cudaFree(cyc);
}

// Usage: microbench [threads per SM ...]   (default: 128 256 1024; K1 fast runs 256 = 8 warps per SM)
int main(int argc, char** argv) {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  printf("%s  SMs=%d  clock=%d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
  int nsm = p.multiProcessorCount;
  int cfgs[16] = {128, 256, 1024}, ncfg = 3;
  if (argc > 1) { ncfg = 0; for (int i = 1; i < argc && ncfg < 16; ++i) cfgs[ncfg++] = atoi(argv[i]); }
  for (int cfg = 0; cfg < ncfg; ++cfg) {
    int threads = cfgs[cfg], bps = 1;
    printf("---- %d threads per SM ----\n", threads);
    run<0>("FADD", threads, bps, nsm);
    run<1>("FFMA", threads, bps, nsm);
    run<2>("IADD3", threads, bps, nsm);
    run<3>("SAD(|a-b|+c)", threads, bps, nsm);
    run<4>("IMNMX(+xor)", threads, bps, nsm);
    run<5>("FMNMX", threads, bps, nsm);
    run<6>("LOP3", threads, bps, nsm);
    run<7>("IMAD", threads, bps, nsm);
    run<8>("SHFL", threads, bps, nsm);
    run<9>("LDS.32+FADD", threads, bps, nsm);
    run<10>("LDS.U16+IADD", threads, bps, nsm);
    run<11>("DADD", threads, bps, nsm);
    run<12>("FSUB+FADD|.|", threads, bps, nsm);
    run<13>("VABSDIFF2+IADD", threads, bps, nsm);
    run<14>("IABS(a-b)+c", threads, bps, nsm);
    run<15>("SETP+predMOV", threads, bps, nsm);
    run<16>("SAD|FADD 1:1", threads, bps, nsm);
    run<17>("VIADDMNMX", threads, bps, nsm);
  }
  return 0;
}
