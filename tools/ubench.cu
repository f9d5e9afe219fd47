// ubench.cu -- issue-rate microbenchmarks for the instructions the SSV kernel is built from, and for the shared-memory
// atomics of the k-mer histogram (kmers.cu), and for the AND + POPC pair of the merge Gram kernel (merge.cu).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench tools/ubench.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#define CHECK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

template <int MODE>
__global__ void k(unsigned *out, int iters, unsigned seed) {
  __shared__ uint4 sm[2048];
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) sm[i] = make_uint4(i, i + 1, i + 2, i + 3);
  __syncthreads();
  unsigned a0 = seed + threadIdx.x, a1 = a0 * 3, a2 = a0 * 5, a3 = a0 * 7, a4 = a0 * 11, a5 = a0 * 13, a6 = a0 * 17, a7 = a0 * 19;
  unsigned d = seed | 0x00010001u, x = 0;
  const int lane = threadIdx.x & 31;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      if (MODE == 0) {        // VIADDMNMX.S16x2, 8 independent chains
        a0 = __viaddmax_s16x2(a0, d, 0u); a1 = __viaddmax_s16x2(a1, d, 0u); a2 = __viaddmax_s16x2(a2, d, 0u); a3 = __viaddmax_s16x2(a3, d, 0u);
        a4 = __viaddmax_s16x2(a4, d, 0u); a5 = __viaddmax_s16x2(a5, d, 0u); a6 = __viaddmax_s16x2(a6, d, 0u); a7 = __viaddmax_s16x2(a7, d, 0u);
      } else if (MODE == 1) { // VIMNMX3.S16x2
        a0 = __vimax3_s16x2(a0, a1, d); a1 = __vimax3_s16x2(a1, a2, d); a2 = __vimax3_s16x2(a2, a3, d); a3 = __vimax3_s16x2(a3, a4, d);
        a4 = __vimax3_s16x2(a4, a5, d); a5 = __vimax3_s16x2(a5, a6, d); a6 = __vimax3_s16x2(a6, a7, d); a7 = __vimax3_s16x2(a7, a0, d);
      } else if (MODE == 2) { // HFMA2.RELU
        __half2 one = __float2half2_rn(1.0f), dd = *(__half2 *)&d;
#define HR(v) { __half2 h = *(__half2 *)&v; h = __hfma2_relu(h, one, dd); v = *(unsigned *)&h; }
        HR(a0) HR(a1) HR(a2) HR(a3) HR(a4) HR(a5) HR(a6) HR(a7)
      } else if (MODE == 3) { // mixed: 4 HFMA2.RELU + 2 VIMNMX3 per "row" (x2)
        __half2 one = __float2half2_rn(1.0f), dd = *(__half2 *)&d;
        HR(a0) HR(a1) HR(a2) HR(a3)
        x = __vimax3_u16x2(x, a0, a1); x = __vimax3_u16x2(x, a2, a3);
        HR(a4) HR(a5) HR(a6) HR(a7)
        x = __vimax3_u16x2(x, a4, a5); x = __vimax3_u16x2(x, a6, a7);
      } else if (MODE == 4) { // mixed DPX: 4 VIADDMNMX + 2 VIMNMX3 (x2)
        a0 = __viaddmax_s16x2(a0, d, 0u); a1 = __viaddmax_s16x2(a1, d, 0u); a2 = __viaddmax_s16x2(a2, d, 0u); a3 = __viaddmax_s16x2(a3, d, 0u);
        x = __vimax3_s16x2(x, a0, a1); x = __vimax3_s16x2(x, a2, a3);
        a4 = __viaddmax_s16x2(a4, d, 0u); a5 = __viaddmax_s16x2(a5, d, 0u); a6 = __viaddmax_s16x2(a6, d, 0u); a7 = __viaddmax_s16x2(a7, d, 0u);
        x = __vimax3_s16x2(x, a4, a5); x = __vimax3_s16x2(x, a6, a7);
      } else if (MODE == 5) { // LDS.128, conflict-free, address depends on previous data slightly
        uint4 v = sm[((a0 & 63) * 32 + lane) & 2047]; a0 += v.x; a1 += v.y; a2 += v.z; a3 += v.w;
        v = sm[((a1 & 63) * 32 + lane) & 2047]; a4 += v.x; a5 += v.y; a6 += v.z; a7 += v.w;
      } else if (MODE == 6) { // SHFL
        a0 = __shfl_sync(0xffffffffu, a0, (lane + 31) & 31); a1 = __shfl_sync(0xffffffffu, a1, (lane + 31) & 31);
        a2 = __shfl_sync(0xffffffffu, a2, (lane + 31) & 31); a3 = __shfl_sync(0xffffffffu, a3, (lane + 31) & 31);
      } else if (MODE == 7) { // full SSV-like row: LDS.128 + 4 VIADDMNMX + 2 VIMNMX3 + SHFL + PRMT (DPX)
        uint4 v = sm[((x & 31) * 32 + lane) & 2047];
        unsigned sh = __shfl_sync(0xffffffffu, a3, (lane + 31) & 31);
        a3 = __viaddmax_s16x2(a2, v.w, 0u); a2 = __viaddmax_s16x2(a1, v.z, 0u); a1 = __viaddmax_s16x2(a0, v.y, 0u);
        a0 = __viaddmax_s16x2(__byte_perm(sh, 0, lane ? 0x3210 : 0x1054), v.x, 0u);
        x = __vimax3_s16x2(x, a0, a1); x = __vimax3_s16x2(x, a2, a3);
      } else if (MODE == 8) { // same with HFMA2.RELU
        __half2 one = __float2half2_rn(1.0f);
        uint4 v = sm[((x & 31) * 32 + lane) & 2047];
        unsigned sh = __shfl_sync(0xffffffffu, a3, (lane + 31) & 31);
#define HR2(dst, src, dv) { __half2 h = *(__half2 *)&src; __half2 e = *(__half2 *)&dv; h = __hfma2_relu(h, one, e); dst = *(unsigned *)&h; }
        HR2(a3, a2, v.w) HR2(a2, a1, v.z) HR2(a1, a0, v.y)
        unsigned p0 = __byte_perm(sh, 0, lane ? 0x3210 : 0x1054);
        HR2(a0, p0, v.x)
        x = __vimax3_u16x2(x, a0, a1); x = __vimax3_u16x2(x, a2, a3);
      } else if (MODE == 9) { // PRMT with the sign-replicating selector the SSV int8 unpack uses
#define PR(v) asm volatile("prmt.b32 %0, %0, %1, 0x9180;" : "+r"(v) : "r"(d));
        PR(a0) PR(a1) PR(a2) PR(a3) PR(a4) PR(a5) PR(a6) PR(a7)
      } else if (MODE >= 10 && MODE <= 13) { // shared-memory add into a per-warp 256-word histogram (+1 IMAD each):
        // 10 red.add, random bins; 11 red.add, one bin for the whole warp (homopolymer); 12 red.add, two bins
        // (dinucleotide repeat); 13 atom.add (result used), random bins
        const unsigned hist = (unsigned)__cvta_generic_to_shared(sm) + (threadIdx.x >> 5) * 1024u;
#define HB(v) { v = v * 1664525u + 1013904223u; \
                const unsigned bin = MODE == 11 ? (v & 0u) : MODE == 12 ? (lane & 1u) * 37u + (v & 0u) : v >> 24; \
                if (MODE == 13) { unsigned o; asm volatile("atom.shared.add.u32 %0, [%1], 1;" : "=r"(o) : "r"(hist + bin * 4u) : "memory"); x += o; } \
                else asm volatile("red.shared.add.u32 [%0], 1;" :: "r"(hist + bin * 4u) : "memory"); }
        HB(a0) HB(a1) HB(a2) HB(a3)
      } else if (MODE == 14) { // POPC of (a & d), accumulated: the inner step of merge_gram_kernel, 8 independent chains
#define PC(v) v += __popc(v & d);
        PC(a0) PC(a1) PC(a2) PC(a3) PC(a4) PC(a5) PC(a6) PC(a7)
      }
    }
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a0 ^ a1 ^ a2 ^ a3 ^ a4 ^ a5 ^ a6 ^ a7 ^ x;
}

template <int MODE>
int run(const char *name, double ops_per_iter, int threads) {
  unsigned *out; int nsm;
  cudaDeviceProp pr; CHECK(cudaGetDeviceProperties(&pr, 0)); nsm = pr.multiProcessorCount;
  CHECK(cudaMalloc(&out, sizeof(unsigned) * nsm * threads));
  int iters = 20000;
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k<MODE><<<nsm, threads>>>(out, 100, 1); CHECK(cudaDeviceSynchronize());
  cudaEventRecord(a); k<MODE><<<nsm, threads>>>(out, iters, 1); cudaEventRecord(b); CHECK(cudaDeviceSynchronize());
  float ms; cudaEventElapsedTime(&ms, a, b);
  int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  double warp_instr = (double)iters * 8 * ops_per_iter * (threads / 32);   // per SM
  printf("%-34s threads=%4d  %.3f ms  %.2f warp-instr/ns/SM  (%.2f per clk @%.0f MHz nominal)\n", name, threads, ms,
         warp_instr / (ms * 1e6), warp_instr / (ms * 1e6) / (clk / 1e6), clk / 1e3);
  cudaFree(out);
  return 0;
}

int main() {
  for (int threads : {256, 512, 1024}) {
    run<0>("VIADDMNMX.S16x2", 8, threads);
    run<1>("VIMNMX3.S16x2", 8, threads);
    run<2>("HFMA2.RELU", 8, threads);
    run<3>("4xHFMA2.RELU+2xVIMNMX3 (x2)", 12, threads);
    run<4>("4xVIADDMNMX+2xVIMNMX3 (x2)", 12, threads);
    run<5>("LDS.128 (x2, +8 IADD)", 2, threads);
    run<6>("SHFL (x4)", 4, threads);
    run<7>("SSV row DPX (1 row = 256 cells)", 1, threads);
    run<8>("SSV row HFMA2 (1 row = 256 cells)", 1, threads);
    run<9>("PRMT (sign-extend)", 8, threads);
    run<10>("red.shared.add random bins (x4)", 4, threads);
    run<11>("red.shared.add one bin/warp (x4)", 4, threads);
    run<12>("red.shared.add two bins/warp (x4)", 4, threads);
    run<13>("atom.shared.add random bins (x4)", 4, threads);
    run<14>("POPC(a & b) + IADD (x8; POPC counted)", 8, threads);
  }
  return 0;
}
