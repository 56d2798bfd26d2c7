// Micro-benchmark: the memory access pattern of the blk-phase transform kernels (k1_fwd_blk, k1_inv_blk) with the
// arithmetic taken out, to find out whether their natural-order side (256 pieces of 128 B, 2 KB apart, per unit) is what
// holds them at ~1.8 TB/s, and what exchanging tiles across a thread-block cluster would give.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_blk_pattern ubench_blk_pattern.cu
//
// Shape: N = 2^16 (n1 = 8, G = 16 groups of 16 blocks per row), 19 rows x 64 items, src and dst of 608 MiB each.
// Every variant is a persistent grid with the dynamic shared memory of k1_fwd_blk (2 CTAs per SM) that walks units
// (row, block range, item), item fastest, in balanced contiguous chunks, and stages each unit's input with cp.async one
// unit ahead as the kernels do (in B the owners load and store their natural rows directly).
//   A  as shipped: a unit is (row, group of 16 blocks, item); its natural side is 256 x 128 B at 2 KB stride.
//      fwd3: block-side read, natural-side read of old values and write (the mod-down epilogue, 3 rows per row)
//      fwd2: block-side read, natural-side write (2 rows)
//      inv : natural-side read, block-side write
//   D  the cluster work split of B (cluster of C CTAs walks (row, C adjacent groups, item); rank k owns group k) but
//      without the exchange: each CTA still moves its own 128 B pieces.  Separates co-scheduling from run length.
//   B  cluster exchange: the same split, the tiles cross the cluster through distributed shared memory so that rank k
//      reads / writes natural rows [k*256/C, (k+1)*256/C) of all 16*C columns: runs of 128*C bytes.
//   S  streaming: the same bytes read and written contiguously.
// A also runs at one CTA per SM (the shared memory of k1_fwd_blk_tensor) to separate occupancy from the pattern.
// Output: best-of-5 time and algorithmic GB/s per variant.  Measured results and what they rule out: DESIGN.md §8.
#include <cstdio>
#include <cstdlib>
#include <cooperative_groups.h>
#include <cuda_runtime.h>
namespace cg = cooperative_groups;
typedef unsigned long long u64;

#define LOGN 16
#define N1 256                       // 2^(LOGN-8)
#define G 16                         // block groups per row
#define ROWS 19
#define ITEMS 64
#define RS 17
#define BS 273
#define STAGE (16 * BS + 8)
#define SMEM ((2 * STAGE + 16 * 256) * 8 + 256 * 16)   // k1_fwd_blk's S[2] | O | TW1

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ unsigned brev4(unsigned x) { return __brev(x) >> 28; }
__device__ __forceinline__ unsigned brev8(unsigned x) { return __brev(x) >> 24; }
__device__ __forceinline__ void cp8(u64* s, const u64* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(s)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int K> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(K) : "memory"); }
__device__ __forceinline__ void cl_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cl_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

enum { FWD3, FWD2, INV };
struct Unit { int row, ug, it; };

// MODE FWD3/FWD2/INV; C = cluster size (1: as shipped); X = exchange through distributed shared memory
template <int MODE, int C, bool X>
__global__ void __launch_bounds__(256, 2) kpat(const u64* __restrict__ src, u64* __restrict__ dst) {
  extern __shared__ u64 sm[];
  u64* S = sm;
  u64* O = S + 2 * STAGE;           // old values (A, D) / receive tile (B): [256/C rows][16*C columns]
  const int tid = threadIdx.x;
  const int blk1 = tid >> 4, lo = tid & 15, hi = tid >> 4, blk2 = tid & 15;
  const unsigned hrev = brev4(hi);
  const int rank = blockIdx.x % C, ncl = gridDim.x / C, cl = blockIdx.x / C;
  const long U = (long)ROWS * (G / C) * ITEMS;
  const long ubeg = U * cl / ncl, uend = U * (cl + 1) / ncl;
  auto unit = [&](long u) {
    Unit x; x.row = (int)(u / ((G / C) * ITEMS)); int rem = (int)(u % ((G / C) * ITEMS));
    x.ug = (rem / ITEMS) * C + rank; x.it = rem % ITEMS; return x;
  };
  auto row_of = [&](auto* b, const Unit& x) { return b + ((size_t)x.it * ROWS + x.row) * ((size_t)1 << LOGN); };
  const int own = MODE == INV ? blk2 * BS + RS * hi : blk1 * BS + lo;
  // stage the unit's input: block side (forward) or natural side (inverse, A/D only)
  auto stage = [&](u64* Sb, const Unit& x) {
    if (MODE != INV) {
      const u64* s = row_of(src, x) + ((size_t)brev8((x.ug << 4) + blk1) << 8) + lo;
      for (int r = 0; r < 16; r++) cp8(Sb + own + RS * r, s + 16 * r);
    } else if (!X) {
      const u64* s = row_of(src, x) + (x.ug << 4) + blk2;
      for (int l = 0; l < 16; l++) cp8(Sb + own + l, s + ((size_t)((brev4(l) << 4) | hrev) << 8));
    }
  };
  constexpr int RR = 256 / C, RC = 16 * C;      // receive tile rows / columns
  cg::cluster_group cluster = cg::this_cluster();
  if (ubeg < uend) stage(S, unit(ubeg));
  cp_commit();
  int buf = 0;
  if (X) cl_arrive();                            // phase 0: "receive tiles free"
  for (long u = ubeg; u < uend; u++, buf ^= 1) {
    const Unit cur = unit(u);
    u64* Sb = S + buf * STAGE;
    if (MODE == INV && X) {
      // owner: read natural rows [rank*RR, +RR) x RC columns as runs, scatter each block's 16 columns to the rank owning it
      cl_wait();                                 // every CTA's Sb is free
      const u64* s = row_of(src, cur) + (size_t)(cur.ug - rank) * 16;
      u64 v[16];
      for (int i = 0; i < 16; i++) { const int e = i * 256 + tid, r = e / RC, c = e % RC; v[i] = s[(size_t)(rank * RR + r) * N1 + c]; }
      for (int i = 0; i < 16; i++) {
        const int e = i * 256 + tid, r = e / RC, c = e % RC, p = rank * RR + r;   // natural row p, block column c
        const int tgt = c >> 4, b2 = c & 15, h = brev4(p & 15), l = brev4(p >> 4);
        u64* rs = cluster.map_shared_rank(Sb, tgt);
        rs[b2 * BS + RS * h + l] = v[i];
      }
      cl_arrive(); cl_wait();                    // tiles complete
    }
    if (MODE != INV && !X && MODE == FWD3) {
      const u64* old = row_of(dst, cur) + (cur.ug << 4) + blk2;
      for (int l = 0; l < 16; l++) cp8(O + l * 256 + tid, old + ((size_t)((brev4(l) << 4) | hrev) << 8));
    }
    cp_commit();
    if (u + 1 < uend) stage(S + (buf ^ 1) * STAGE, unit(u + 1));
    cp_commit();
    cp_wait<1>();
    __syncthreads();
    u64 a[16];
    if (MODE != INV) {
      for (int l = 0; l < 16; l++) a[l] = Sb[blk2 * BS + RS * hi + l] ^ 0x5a5a;
      if (!X) {
        u64* d = row_of(dst, cur) + (cur.ug << 4) + blk2;
        for (int l = 0; l < 16; l++) {
          const size_t o = (size_t)((brev4(l) << 4) | hrev) << 8;
          d[o] = MODE == FWD3 ? O[l * 256 + tid] - a[l] : a[l];
        }
      } else {
        cl_wait();                               // receive tiles drained by their owners
        for (int l = 0; l < 16; l++) {
          const int p = (brev4(l) << 4) | hrev;
          u64* rt = cluster.map_shared_rank(O, p / RR);
          rt[(p % RR) * RC + rank * 16 + blk2] = a[l];
        }
        cl_arrive(); cl_wait();
        u64* d = row_of(dst, cur) + (size_t)(cur.ug - rank) * 16;
        u64 old[16];
        if (MODE == FWD3) for (int i = 0; i < 16; i++) { const int e = i * 256 + tid; old[i] = d[(size_t)(rank * RR + e / RC) * N1 + e % RC]; }
        for (int i = 0; i < 16; i++) {
          const int e = i * 256 + tid;
          d[(size_t)(rank * RR + e / RC) * N1 + e % RC] = MODE == FWD3 ? old[i] - O[e] : O[e];
        }
        cl_arrive();
      }
    } else {
      for (int r = 0; r < 16; r++) a[r] = Sb[blk1 * BS + RS * r + lo] ^ 0x5a5a;
      u64* d = row_of(dst, cur) + ((size_t)brev8((cur.ug << 4) + blk1) << 8) + lo;
      for (int r = 0; r < 16; r++) d[16 * r] = a[r];
      if (X) cl_arrive();
    }
    __syncthreads();
  }
  cp_wait<0>();
  if (X) cl_wait();                              // no CTA leaves while a peer may still write into its shared memory
}

// streaming: NR rows read and 1 written per row, contiguous
template <int NR>
__global__ void __launch_bounds__(256) kstream(const u64* __restrict__ src, u64* __restrict__ dst, size_t n) {
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n / 2; i += (size_t)gridDim.x * 256) {
    ulonglong2 a = ((const ulonglong2*)src)[i];
    if (NR == 2) { const ulonglong2 b = ((const ulonglong2*)dst)[i]; a.x -= b.x; a.y -= b.y; }
    ((ulonglong2*)dst)[i] = a;
  }
}

static cudaEvent_t e0, e1;
template <class F> static double time_ms(F&& f) {
  f(); CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int rep = 0; rep < 5; rep++) {
    CK(cudaEventRecord(e0)); f(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms;
  }
  return best;
}

template <int MODE, int C, bool X>
static void run(const char* name, const u64* src, u64* dst, double bytes, int nsm, int smem = SMEM) {
  auto k = kpat<MODE, C, X>;
  CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (C > 8) CK(cudaFuncSetAttribute(k, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = C; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem; cfg.attrs = at; cfg.numAttrs = 1;
  int grid = (smem > SMEM ? 1 : 2) * nsm;
  if (C > 1) {
    int ncl = 0;
    cfg.gridDim = dim3(C * 64);
    cudaError_t e = cudaOccupancyMaxActiveClusters(&ncl, k, &cfg);
    if (e != cudaSuccess || ncl == 0) { printf("%-34s C=%2d  does not schedule (%s)\n", name, C, cudaGetErrorString(e)); cudaGetLastError(); return; }
    grid = ncl * C;
  }
  cfg.gridDim = dim3(grid);
  const double ms = time_ms([&] { CK(cudaLaunchKernelEx(&cfg, k, src, dst)); });
  printf("%-34s C=%2d grid %3d: %7.3f ms  %7.1f GB/s\n", name, C, grid, ms, bytes / (ms * 1e-3) / 1e9);
}

int main() {
  int nsm = 0; CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0));
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  printf("device: %s, %d SMs\n", prop.name, nsm);
  const size_t n = (size_t)ITEMS * ROWS << LOGN;     // u64 per buffer
  const double row_bytes = (double)n * 8;
  u64 *src, *dst;
  CK(cudaMalloc(&src, n * 8)); CK(cudaMalloc(&dst, n * 8));
  CK(cudaMemset(src, 1, n * 8)); CK(cudaMemset(dst, 2, n * 8));
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  printf("working set: %d items x %d rows x %d KiB = %.0f MiB per buffer\n", ITEMS, ROWS, (8 << LOGN) >> 10, row_bytes / (1 << 20));
  const double b3 = 3 * row_bytes, b2 = 2 * row_bytes;
  run<FWD3, 1, false>("A fwd3 (read blk, rmw natural)", src, dst, b3, nsm);
  run<FWD2, 1, false>("A fwd2 (read blk, write natural)", src, dst, b2, nsm);
  run<INV, 1, false>("A inv  (read natural, write blk)", src, dst, b2, nsm);
  run<FWD3, 1, false>("A fwd3, 1 CTA per SM (205 KB smem)", src, dst, b3, nsm, 205 * 1024);
  run<FWD2, 1, false>("A fwd2, 1 CTA per SM (205 KB smem)", src, dst, b2, nsm, 205 * 1024);
  run<FWD3, 2, false>("D fwd3 cluster split, no exchange", src, dst, b3, nsm);
  run<FWD3, 4, false>("D fwd3 cluster split, no exchange", src, dst, b3, nsm);
  run<FWD3, 8, false>("D fwd3 cluster split, no exchange", src, dst, b3, nsm);
  run<FWD2, 8, false>("D fwd2 cluster split, no exchange", src, dst, b2, nsm);
  run<INV, 8, false>("D inv  cluster split, no exchange", src, dst, b2, nsm);
  run<FWD3, 2, true>("B fwd3 exchange", src, dst, b3, nsm);
  run<FWD3, 4, true>("B fwd3 exchange", src, dst, b3, nsm);
  run<FWD3, 8, true>("B fwd3 exchange", src, dst, b3, nsm);
  run<FWD3, 16, true>("B fwd3 exchange", src, dst, b3, nsm);
  run<FWD2, 2, true>("B fwd2 exchange", src, dst, b2, nsm);
  run<FWD2, 4, true>("B fwd2 exchange", src, dst, b2, nsm);
  run<FWD2, 8, true>("B fwd2 exchange", src, dst, b2, nsm);
  run<FWD2, 16, true>("B fwd2 exchange", src, dst, b2, nsm);
  run<INV, 2, true>("B inv  exchange", src, dst, b2, nsm);
  run<INV, 4, true>("B inv  exchange", src, dst, b2, nsm);
  run<INV, 8, true>("B inv  exchange", src, dst, b2, nsm);
  run<INV, 16, true>("B inv  exchange", src, dst, b2, nsm);
  {
    const double ms2 = time_ms([&] { kstream<1><<<4 * nsm, 256>>>(src, dst, n); });
    printf("%-34s              %7.3f ms  %7.1f GB/s\n", "S stream copy (2 rows)", ms2, b2 / (ms2 * 1e-3) / 1e9);
    const double ms3 = time_ms([&] { kstream<2><<<4 * nsm, 256>>>(src, dst, n); });
    printf("%-34s              %7.3f ms  %7.1f GB/s\n", "S stream rmw (3 rows)", ms3, b3 / (ms3 * 1e-3) / 1e9);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
