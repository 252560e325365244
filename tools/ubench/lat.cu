// Dependent-issue latencies seen by ONE warp on sm_90a (cycles per operation in a dependent chain):
// the numbers that bound the sequential assignment loop of k_schedule_pass (DESIGN.md §5.3/§7).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench/lat tools/ubench/lat.cu && tools/ubench/lat
#include <cstdio>
#include <cuda_runtime.h>

#define N 4096
#define FULL 0xffffffffu

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long k) {
  unsigned hi = (unsigned)(k >> 32);
  unsigned mhi = __reduce_min_sync(FULL, hi);
  unsigned lo = (hi == mhi) ? (unsigned)k : 0xFFFFFFFFu;
  unsigned mlo = __reduce_min_sync(FULL, lo);
  return ((unsigned long long)mhi << 32) | mlo;
}

__global__ void k_lat(long long* out, unsigned seed) {
  __shared__ unsigned chase[1024];
  __shared__ unsigned long long wide[64];
  const unsigned l = threadIdx.x;
  for (unsigned i = l; i < 1024; i += 32) chase[i] = (i * 37u + 11u) & 1023u;
  for (unsigned i = l; i < 64; i += 32) wide[i] = (unsigned long long)(i * 2654435761u) << 13 | i;
  __syncwarp();
  long long t0, t1;
  unsigned x = seed + l;
  unsigned long long y = ((unsigned long long)seed << 32) | l;

  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = x * 3u + 1u;  // IMAD chain
  t1 = clock64();
  if (l == 0) out[0] = t1 - t0;

  unsigned p = seed & 1023u;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) p = chase[p];  // LDS -> address -> LDS
  t1 = clock64();
  if (l == 0) out[1] = t1 - t0;
  x += p;

  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = __reduce_min_sync(FULL, x + l) + 1u;  // redux chain
  t1 = clock64();
  if (l == 0) out[2] = t1 - t0;

  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) y = warp_min_u64(y + l) + 1ull;  // the 64-bit arg-min of the assignment loop (K64, chain_run)
  t1 = clock64();
  if (l == 0) out[3] = t1 - t0;

  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = __shfl_sync(FULL, x, (x + 1u) & 31u) + 1u;  // shfl chain
  t1 = clock64();
  if (l == 0) out[4] = t1 - t0;

  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x += __ballot_sync(FULL, (x >> (l & 7u)) & 1u);  // vote chain
  t1 = clock64();
  if (l == 0) out[5] = t1 - t0;

  t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < N; ++i) {  // one taken branch + one dependent add per trip
    x += 1u;
    if (x == 0xdeadbeefu) break;
  }
  t1 = clock64();
  if (l == 0) out[6] = t1 - t0;

  // the common case of the assignment loop in miniature: 2 LDS, SWAR test, 64-bit min, compare, subtract
  const unsigned long long G = 0x8000400020000000ull;
  unsigned long long xg = (y | G) + ((unsigned long long)l << 20);
  unsigned acc = 0;
  t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < N; ++i) {
    const unsigned long long preq = wide[i & 63] & ~G & 0x0000000fffffffffull;
    const unsigned long long fk = wide[(i + 7) & 63] | G;
    const bool fit = (((xg - preq) & G) == G);
    const unsigned long long kmin = warp_min_u64(fit ? xg : ~0ull);
    if (kmin < fk) {
      if (fit && xg == kmin) xg -= preq;
      acc += (unsigned)kmin;
    } else {
      acc ^= (unsigned)fk;
      xg += 1ull << 40;
    }
  }
  t1 = clock64();
  if (l == 0) out[7] = t1 - t0;
  if (x == 12345u && y == 678ull && acc == 9u && xg == 1ull) out[8] = 1;  // keep everything live
}

int main() {
  long long *d, h[9] = {0};
  cudaMalloc(&d, sizeof(h));
  cudaMemset(d, 0, sizeof(h));
  for (int rep = 0; rep < 2; ++rep) k_lat<<<1, 32>>>(d, 12345u + rep);
  if (cudaDeviceSynchronize() != cudaSuccess) {
    printf("kernel failed: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
  const char* name[8] = {"IMAD (dependent)", "LDS pointer chase", "redux.min.u32 chain", "64-bit warp min (2x redux)", "shfl.idx chain",
                         "vote.ballot chain", "loop trip (add+cmp+taken branch)", "assignment-loop miniature (per trip)"};
  for (int i = 0; i < 8; ++i) printf("%-40s %7.1f cycles\n", name[i], (double)h[i] / N);
  return 0;
}
