// Miniatures of the node-assignment chain (DESIGN.md §5.3) on ONE warp: cycles per placement for
//   A  64-bit guard key, two redux.sync, one placement after the other (the previous place() loop, K64)
//   B  32-bit compact compare key, one redux.sync, one placement after the other (the previous place() loop, K32)
//   C  B with the second placement of each pair decided ahead: both of its compare values (the lane
//      won the first one / it did not) are ready before the first minimum arrives (chain_swar<K32>, place_pair)
//   D  B with every placement decided one record ahead, one placement per loop trip
// with the rare paths out of line behind unlikely branches, records prefetched two ahead.  The rare
// path takes and returns the loop state by value: passing its address would keep the state in local
// memory and put a memory round trip on the chain.  C, the fastest of B, C and D, is the kernel's form.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench/chain tools/ubench/chain.cu && tools/ubench/chain
#include <cstdio>
#include <cuda_runtime.h>
#define FULL 0xffffffffu
#define NREC 2048
__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long k) {
  unsigned hi = (unsigned)(k >> 32);
  unsigned mhi = __reduce_min_sync(FULL, hi);
  unsigned lo = (hi == mhi) ? (unsigned)k : 0xFFFFFFFFu;
  unsigned mlo = __reduce_min_sync(FULL, lo);
  return ((unsigned long long)mhi << 32) | mlo;
}
__device__ __forceinline__ unsigned warp_min_u32(unsigned v) {
  unsigned m;
  asm volatile("redux.sync.min.u32 %0, %1, 0xffffffff;" : "=r"(m) : "r"(v));
  return m;
}
struct Rare {
  unsigned have;
  unsigned long long Y;
};
__device__ __noinline__ Rare rare(unsigned have, unsigned long long Y, unsigned s) { return Rare{have | 1u << s, Y + (1ull << 40)}; }
template <int MODE>
__global__ void k_chain(long long* out, uint4* grec, unsigned seed, int reps) {
  __shared__ uint4 rec[NREC + 2];
  __shared__ unsigned won[NREC];  // the winner of every placement (records stay as they are: .w is the compact request)
  const unsigned l = threadIdx.x;
  for (unsigned i = l; i < NREC + 2; i += 32) rec[i] = grec[i < NREC ? i : NREC - 1];
  __syncwarp();
  // three 11-bit fields at bits 18, 30 and 42 with their guard bits above them, the lane in the low bits;
  // every lane starts with at least 1024 in each field, so all NREC records of a repetition fit
  unsigned long long G = ((1ull << 29) | (1ull << 41) | (1ull << 53)) << 1;
  asm volatile("mov.b64 %0, %0;" : "+l"(G));
  auto row_of = [&](unsigned r) {
    const unsigned h = (seed + l * 977u + r) * 2654435761u;
    const unsigned long long f = (1024ull + (h & 1023u)) | (1024ull + ((h >> 10) & 1023u)) << 12 | (1024ull + ((h >> 20) & 1023u)) << 24;
    return (f << 18 | l | (G >> 1)) << 1;
  };
  unsigned long long Y = row_of(0);
  unsigned ck = ((seed + l * 977u) & 0x3ffffffu) << 6 | l << 1;
  unsigned mystat = 0xffffffffu, fullstat = 0xffffffffu, have = 0xffffffffu, acc = 0;
  auto do_rare = [&](unsigned s) {
    const Rare r = rare(have, Y, s);
    have = r.have;
    Y = r.Y;
  };
  auto preq_of = [](const uint4 rc) { return ((unsigned long long)rc.y << 32) | rc.x; };
  auto fits = [&](unsigned long long d, unsigned stat, const uint4 rc) { return ((d & G) == G) && ((stat >> (rc.z & 0xFFu)) & 1u); };
  long long t0 = clock64();
  for (int r = 0; r < reps; ++r) {
    const unsigned total = NREC;
    unsigned t = 0;
    if (MODE <= 1) {
      auto step = [&](const uint4 rc, unsigned tt) -> bool {
        const unsigned long long preq = preq_of(rc);
        const unsigned s = rc.z & 0xFFu;
        const unsigned long long d = Y - preq;
        const bool fit = fits(d, mystat, rc);
        if (MODE == 0) {
          const unsigned long long m = warp_min_u64(fit ? Y : ~0ull);
          if (__builtin_expect(m == ~0ull, 0)) return true;
          if (Y == m) {
            Y = d & ~1ull;
            mystat = fullstat;
          }
          if (l == 0) won[tt] = (unsigned)(m >> 1) & 0x1ffffu;
          if (__builtin_expect((unsigned)m & 1u, 0)) do_rare(s);
        } else {
          const unsigned m = warp_min_u32(fit ? ck : 0xFFFFFFFFu);
          if (__builtin_expect(m == 0xFFFFFFFFu, 0)) return true;
          if (ck == m) {
            Y = d;
            ck -= rc.w;
            mystat = fullstat;
            won[tt] = l;
          }
          if (__builtin_expect(m & 1u, 0)) do_rare(s);
        }
        return false;
      };
      uint4 ra = rec[0], rb = rec[1];
      for (; t + 1 < total; t += 2) {
        if (step(ra, t)) break;
        ra = rec[t + 2];
        if (step(rb, t + 1)) break;
        rb = rec[t + 3];
      }
    } else if (MODE == 2) {
      uint4 ra = rec[0], rb = rec[1];
      for (; t + 1 < total; t += 2) {
        const unsigned long long da = Y - preq_of(ra), db = Y - preq_of(rb), dab = da - preq_of(rb);
        const unsigned sa = (ck & 1u) ? fullstat : mystat, cka = (ck - ra.w) & ~1u;
        const bool fa = fits(da, mystat, ra), fb = fits(db, mystat, rb), fab = fa && fits(dab, sa, rb);
        const unsigned ma = warp_min_u32(fa ? ck : 0xFFFFFFFFu);
        const bool wa = ck == ma;
        const unsigned mb = warp_min_u32(wa ? (fab ? cka : 0xFFFFFFFFu) : (fb ? ck : 0xFFFFFFFFu));
        if (__builtin_expect(ma == 0xFFFFFFFFu, 0)) break;
        if (wa) {
          Y = da;
          ck = cka;
          mystat = sa;
          won[t] = l;
        }
        if (__builtin_expect(ma & 1u, 0)) do_rare(ra.z & 0xFFu);
        ra = rec[t + 2];
        if (__builtin_expect(mb == 0xFFFFFFFFu, 0)) {
          ++t;
          break;
        }
        if (ck == mb) {
          Y -= preq_of(rb);
          mystat = (ck & 1u) ? fullstat : mystat;
          ck = (ck - rb.w) & ~1u;
          won[t + 1] = l;
        }
        if (__builtin_expect(mb & 1u, 0)) do_rare(rb.z & 0xFFu);
        rb = rec[t + 3];
      }
    } else {
      uint4 r0 = rec[0], r1 = rec[1], r2 = rec[2];
      unsigned m = warp_min_u32(fits(Y - preq_of(r0), mystat, r0) ? ck : 0xFFFFFFFFu);
      for (;;) {
        const unsigned long long Y1 = Y - preq_of(r0);
        const unsigned ck1 = (ck - r0.w) & ~1u, s1 = (ck & 1u) ? fullstat : mystat;
        const unsigned v0 = fits(Y - preq_of(r1), mystat, r1) ? ck : 0xFFFFFFFFu;
        const unsigned v1 = fits(Y1 - preq_of(r1), s1, r1) ? ck1 : 0xFFFFFFFFu;
        const bool win = ck == m;
        const unsigned mn = warp_min_u32(win ? v1 : v0);
        if (__builtin_expect(m == 0xFFFFFFFFu, 0)) break;
        if (win) {
          Y = Y1;
          ck = ck1;
          mystat = s1;
          won[t] = l;
        }
        if (__builtin_expect(m & 1u, 0)) do_rare(r0.z & 0xFFu);
        if (++t == total) break;
        r0 = r1;
        r1 = r2;
        r2 = rec[t + 2];
        m = mn;
      }
    }
    acc += t;
    // top the rows up again so that the next repetition fits too
    Y = row_of(r + 1);
    ck = ((seed + l * 977u + r) & 0x3ffffffu) << 6 | l << 1;
  }
  long long t1 = clock64();
  if (l == 0) {
    out[0] = t1 - t0;
    out[1] = acc;
  }
  __syncwarp();
  if (l == 0) {  // the winners of the last repetition: B, C and D decide the same placements
    unsigned long long sum = 0;
    for (unsigned i = 0; i < NREC; ++i) sum = sum * 31u + won[i];
    out[2] = (long long)sum;
  }
  if (Y == 1 && ck == 7 && have == 3) out[3] = 1;
}
int main() {
  long long *d, h[4];
  uint4 *rec, hr[NREC];
  for (int i = 0; i < NREC; ++i) {
    // small requests in each field so that most lanes fit; window in z; compact request in w
    unsigned long long pq = ((unsigned long long)(1 + i % 3) << 18 | (unsigned long long)(i % 5) << 30 | (unsigned long long)(i % 2) << 42) << 1;
    hr[i] = make_uint4((unsigned)pq, (unsigned)(pq >> 32), (unsigned)(i % 5), (1u + i % 3) << 6);
  }
  cudaMalloc(&d, sizeof(h));
  cudaMalloc(&rec, sizeof(hr));
  cudaMemcpy(rec, hr, sizeof(hr), cudaMemcpyHostToDevice);
  const int reps = 8;
  const char* name[4] = {"A 64-bit key, 2x redux", "B 32-bit key, 1x redux", "C B, 2nd of each pair ahead", "D B, every placement one ahead"};
  for (int mode = 0; mode < 4; ++mode) {
    for (int w = 0; w < 2; ++w) {
      if (mode == 0) k_chain<0><<<1, 32>>>(d, rec, 12345u, reps);
      else if (mode == 1) k_chain<1><<<1, 32>>>(d, rec, 12345u, reps);
      else if (mode == 2) k_chain<2><<<1, 32>>>(d, rec, 12345u, reps);
      else k_chain<3><<<1, 32>>>(d, rec, 12345u, reps);
      cudaMemcpy(rec, hr, sizeof(hr), cudaMemcpyHostToDevice);
    }
    if (cudaDeviceSynchronize() != cudaSuccess) {
      printf("kernel failed: %s\n", cudaGetErrorString(cudaGetLastError()));
      return 1;
    }
    cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
    printf("%-32s %.1f cycles per placement (%lld placements, winners %016llx)\n", name[mode], (double)h[0] / (double)h[1], h[1],
           (unsigned long long)h[2]);
  }
  return 0;
}
