// Micro-benchmark: register-only radix-16 butterfly networks, to measure the integer-pipe ceiling
// of the lazy Harvey butterfly on an H100 (no memory traffic).  Build: nvcc -arch=sm_90a -O3.
#include <cstdio>
#include <cuda_runtime.h>
#include "../helib_b200/csrc/hb_device_v1.cuh"

__device__ __forceinline__ void ct_exact(u64& x, u64& y, u64 w, u64 ws, u64 q, u64 q2) {
  u64 xr = x >= q2 ? x - q2 : x;
  u64 t = y * w - __umul64hi(y, ws) * q;
  x = xr + t; y = xr - t + q2;
}
template <int MODE>
__global__ void __launch_bounds__(256) kb(u64* out, u64 q, u64 nq, u64 qb, u64 seed, int rounds) {
  u64 a[16];
  Hb1TwReg tw;
  hb1_unroll<16>([&](auto i) { a[i] = (seed + threadIdx.x * 977 + i * 131 + blockIdx.x) % q; });
  tw.load([&](int k, int g) {
    const int i = (1 << k) - 1 + g;
    u64 w = (seed * (i + 3) + 12345) % q;
    return make_ulonglong2(w, (u64)(((unsigned __int128)w << 64) / q));
  });
  for (int r = 0; r < rounds; r++) {
    Hb1Mod M; M.nq = nq; M.qb = qb; M.qb2 = qb + qb; M.qt = (unsigned)((q - 1) >> 52); M.qsh = 20;   // q = 237*2^52 + 1
    if (MODE == 0) hb1_r16_fwd<false>(a, tw, M);
    else if (MODE == 1) hb1_r16_inv<false>(a, tw, M);
    else if (MODE == 3) hb1_r16_fwd<true>(a, tw, M);
    else {
      hb1_unroll<4>([&](auto k) { constexpr int d = 8 >> k;
        hb1_unroll<(1 << k)>([&](auto g) { const ulonglong2 w = tw.template get<k, g>();
          hb1_unroll<d>([&](auto o) { ct_exact(a[g * 2 * d + o], a[g * 2 * d + o + d], w.x, w.y, q, q + q); }); }); });
    }
    hb1_unroll<16>([&](auto i) { a[i] = hb1_csub_hi(hb1_csub_hi(a[i], qb), qb); });   // keep bounded between rounds
  }
  u64 s = 0;
  hb1_unroll<16>([&](auto i) { s ^= a[i]; });
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// 128-bit MAC throughput
__global__ void __launch_bounds__(256) kmac(u64* out, u64 seed, int rounds) {
  u64 hi[8], lo[8], y[8];
#pragma unroll
  for (int i = 0; i < 8; i++) { hi[i] = 0; lo[i] = i; y[i] = seed * (threadIdx.x + i + 1); }
  u64 c = seed | 1;
  for (int r = 0; r < rounds; r++) {
#pragma unroll
    for (int i = 0; i < 8; i++) hb1_mac128(hi[i], lo[i], y[i], c);
    c += 2;
  }
  u64 s = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) s ^= hi[i] ^ lo[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main() {
  u64 q = 1067353111686807553ULL;
  int nsm = 0; cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);
  u64* out; cudaMalloc(&out, (size_t)nsm * 16 * 256 * 8);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int rounds = 2000;
  for (int mode = 0; mode < 4; mode++)
    for (int bps : {2, 8}) {
      int blocks = nsm * bps;
      for (int rep = 0; rep < 2; rep++) {
        cudaEventRecord(e0);
        if (mode == 0) kb<0><<<blocks, 256>>>(out, q, 0 - q, 4 * q, 7, rounds);
        if (mode == 1) kb<1><<<blocks, 256>>>(out, q, 0 - q, 4 * q, 7, rounds);
        if (mode == 2) kb<2><<<blocks, 256>>>(out, q, 0 - q, 4 * q, 7, rounds);
        if (mode == 3) kb<3><<<blocks, 256>>>(out, q, 0 - q, 4 * q, 7, rounds);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
      }
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      double bf = (double)blocks * 256 * rounds * 32;
      printf("mode %d (%s) blocks/SM %d: %.3f ms  %.3e butterflies/s\n", mode, mode == 0 ? "ct approx" : mode == 1 ? "gs approx" : mode == 2 ? "ct exact" : "ct approx, q=t*2^s+1 shift form", bps, ms, bf / (ms * 1e-3));
    }
  for (int bps : {2, 8}) {
    int blocks = nsm * bps;
    for (int rep = 0; rep < 2; rep++) { cudaEventRecord(e0); kmac<<<blocks, 256>>>(out, 12345, 20000); cudaEventRecord(e1); cudaEventSynchronize(e1); }
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("mac128 blocks/SM %d: %.3f ms %.3e mac/s\n", bps, ms, (double)blocks * 256 * 20000 * 8 / (ms * 1e-3));
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
