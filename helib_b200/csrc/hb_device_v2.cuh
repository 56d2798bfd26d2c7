// hb_device_v2.cuh -- TMA-staged, warp-specialised "blk" phases of the length-N transform (N = N1 x 256, n1 >= 4).
//
// Same arithmetic and the same work decomposition as k1_fwd_blk / k1_inv_blk (hb_device_v1.cuh): unit = (row, group of
// 16 blocks, batch item), persistent CTAs over balanced contiguous unit chunks.  What changed is how tiles move:
//
//   * ONE thread of a dedicated I/O warp moves whole 32 KB tiles with the tensor-memory accelerator
//     (cp.async.bulk.tensor, mbarrier complete_tx): no per-thread address arithmetic, no LDGSTS, no STG in the eight
//     compute warps.  Two views of every [nprimes][N] matrix are described by tensor maps (built once per buffer):
//        BLK  {256 i, G u, 16 slot, prime}  box {256,1,16,1}  -> the 16 blocks b = slot*G + brev(ug) of a unit, dense [16][256]
//        NAT  {N1 c, 256 k, prime}          box {16,256,1}    -> 256 natural-order rows of 16 adjacent outputs (128-byte
//                                                                segments), SWIZZLE_128B in shared memory
//   * a warp owns two blocks (logical j = 2w, 2w+1) in BOTH passes, so the 16x16 exchange between the two radix-16 passes
//     stays inside the warp: in place in the tile, XOR-swizzled (element (r,lo) of block j at 16r + (lo ^ r ^ (j&1)))
//     -- conflict-free for both access patterns, __syncwarp only.  There is no CTA-wide barrier in the steady state;
//     warps drift apart and cover each other's latencies.
//   * the second-pass lane order (hi&1, hi>>1, j&1) makes a half-warp touch eight distinct 16-byte chunks of the
//     hardware-swizzled NAT tile: stores of results / loads of the old destination values are conflict-free.
//   * mod-down epilogue: the old destination tile is TMA-loaded INTO the output buffer; every thread reads and rewrites
//     its own 16 positions, the same buffer is stored back.
//
//   * a CTA holds TWO independent teams (8 compute warps + 1 I/O warp each, 18 warps = 576 threads, 1 CTA / SM): same
//     16 resident compute warps per SM as two 9-warp CTAs, but 112 registers per thread instead of 96 (register
//     allocation rounds a 288-thread CTA up to 320).
//
// Measured on an H100 SXM (80 GB HBM3, 400 W limit), two runs each in one session: both kernels together are slower than
// k1_fwd_blk / k1_inv_blk (2 504-2 507 against 2 543-2 548 mult/s on the multiply benchmark), so they run only with HB_BLK_V2=1.
//
// smem per team (1024-byte aligned): IN[2][4096] | OUT[4096] | TW1[16][16] | 7 mbarriers  (101 KB; 203 KB per CTA)
#pragma once
#include "hb_device_v1.cuh"

#ifdef HB_SIM
// CPU stand-in of a tiled tensor map (tests/cusim): same addressing, same 128-byte swizzle
struct HbTmap {
  u64* base; int rank; int swz128;
  u64 dim[4]; u64 stride[4];     // elements
  unsigned box[4];
};
#else
#include <cuda.h>
typedef CUtensorMap HbTmap;
#endif

#define HB2_TILE 4096            // u64 per tile (32 KB)
#define HB2_TILE_BYTES 32768u
#define HB2_THREADS 576          // 2 teams x 8 compute warps, then one I/O warp per team
#define HB2_TEAM_U64 (101 * 128) // u64 per team region (101 KB: a multiple of 1024 bytes keeps every tile 1024-byte aligned)
#define HB2_SMEM_BYTES (2 * HB2_TEAM_U64 * 8 + 1024)

// ---- mbarrier / TMA wrappers ---------------------------------------------------------------
#ifdef HB_SIM
// u64 word: [31:0] completed phases, [47:32] pending arrivals, [63:48] arrival count
__device__ __forceinline__ void hb2_mbar_init(u64* bar, unsigned count) { *bar = ((u64)count << 48) | ((u64)count << 32); }
__device__ __forceinline__ void hb2_mbar_arrive(u64* bar) {
  u64 v = *bar; unsigned cnt = (unsigned)(v >> 48), pend = (unsigned)((v >> 32) & 0xffff), ph = (unsigned)v;
  if (--pend == 0) { pend = cnt; ph++; }
  *bar = ((u64)cnt << 48) | ((u64)pend << 32) | ph;
}
__device__ __forceinline__ void hb2_mbar_expect(u64* bar, unsigned) { hb2_mbar_arrive(bar); }   // copies are synchronous in the simulator
__device__ __forceinline__ void hb2_mbar_wait(u64* bar, unsigned parity) { while ((((unsigned)*bar) & 1u) == parity) cusim::yield(); }
__device__ __forceinline__ void hb2_fence_async() {}
__device__ __forceinline__ void hb2_fence_init() {}
__device__ __forceinline__ void hb2_store_commit() {}
__device__ __forceinline__ void hb2_store_wait_read() {}
__device__ __forceinline__ void hb2_store_wait_all() {}
__device__ inline void hb2_sim_copy(u64* smem, const HbTmap* m, const int* c, bool load) {
  size_t n = 1; for (int d = 0; d < m->rank; d++) n *= m->box[d];
  for (size_t lin = 0; lin < n; lin++) {
    size_t rem = lin, g = 0;
    for (int d = 0; d < m->rank; d++) { size_t x = rem % m->box[d]; rem /= m->box[d]; g += ((size_t)c[d] + x) * m->stride[d]; }
    size_t off = lin * 8;
    if (m->swz128) off ^= ((off >> 7) & 7) << 4;
    if (load) smem[off / 8] = m->base[g]; else m->base[g] = smem[off / 8];
  }
}
__device__ __forceinline__ void hb2_tma_load4(u64* dst, const HbTmap* m, u64*, int c0, int c1, int c2, int c3) { int c[4] = {c0, c1, c2, c3}; hb2_sim_copy(dst, m, c, true); }
__device__ __forceinline__ void hb2_tma_load3(u64* dst, const HbTmap* m, u64*, int c0, int c1, int c2) { int c[4] = {c0, c1, c2, 0}; hb2_sim_copy(dst, m, c, true); }
__device__ __forceinline__ void hb2_tma_store4(const HbTmap* m, int c0, int c1, int c2, int c3, u64* src) { int c[4] = {c0, c1, c2, c3}; hb2_sim_copy(src, m, c, false); }
__device__ __forceinline__ void hb2_tma_store3(const HbTmap* m, int c0, int c1, int c2, u64* src) { int c[4] = {c0, c1, c2, 0}; hb2_sim_copy(src, m, c, false); }
__device__ __forceinline__ void hb2_bulk_store(u64* gdst, const u64* src, unsigned bytes) { memcpy(gdst, src, bytes); }
#else
__device__ __forceinline__ unsigned hb2_saddr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void hb2_mbar_init(u64* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(hb2_saddr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void hb2_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void hb2_mbar_arrive(u64* bar) {
  asm volatile("{ .reg .b64 st; mbarrier.arrive.shared::cta.b64 st, [%0]; }" ::"r"(hb2_saddr(bar)) : "memory");
}
__device__ __forceinline__ void hb2_mbar_expect(u64* bar, unsigned bytes) {
  asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1; }" ::"r"(hb2_saddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void hb2_mbar_wait(u64* bar, unsigned parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "W_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra D_%=;\n\t"
      "bra W_%=;\n\t"
      "D_%=:\n\t}"
      ::"r"(hb2_saddr(bar)), "r"(parity) : "memory");
}
// generic-proxy writes to shared memory become visible to the async proxy (TMA stores read them)
__device__ __forceinline__ void hb2_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void hb2_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void hb2_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void hb2_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void hb2_tma_load4(u64* dst, const HbTmap* m, u64* bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(hb2_saddr(dst)), "l"(m), "r"(hb2_saddr(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void hb2_tma_load3(u64* dst, const HbTmap* m, u64* bar, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(hb2_saddr(dst)), "l"(m), "r"(hb2_saddr(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void hb2_tma_store4(const HbTmap* m, int c0, int c1, int c2, int c3, u64* src) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(m), "r"(hb2_saddr(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void hb2_tma_store3(const HbTmap* m, int c0, int c1, int c2, u64* src) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(m), "r"(hb2_saddr(src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// contiguous shared -> global copy (no tensor map): bytes and both addresses multiples of 16
__device__ __forceinline__ void hb2_bulk_store(u64* gdst, const u64* src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(hb2_saddr(src)), "r"(bytes) : "memory");
}
#endif

__device__ __forceinline__ u64* hb2_align1024(u64* p) {
#ifdef HB_SIM
  return (u64*)(((uintptr_t)p + 1023) & ~(uintptr_t)1023);
#else
  const unsigned a = hb2_saddr(p), pad = (1024u - (a & 1023u)) & 1023u;
  return (u64*)((char*)p + pad);
#endif
}

// forward epilogues as in Hb1BlkJob (0 plain, 1 dst = (dst - x)*scal, 3 dst = x and dst2 = (dst2 - x)*scal where scal != 0);
// inverse: epi 2 = lazy outputs (the consumer is a register kernel), 0 = canonical.
struct Hb2BlkJob {
  int logN, epi, lazy;
  HbRows rows;
  u64 scal[HB_MAXROWS], scal_s[HB_MAXROWS];
  int nitems;
  const HbTmap* src[HB_MAXB];    // forward: BLK view of the source;      inverse: NAT view
  const HbTmap* dst[HB_MAXB];    // forward: NAT view of the destination; inverse: BLK view
  const HbTmap* dst2[HB_MAXB];   // forward epilogue 3: NAT view of the matrix updated in place
  u64* dstp[HB_MAXB];            // inverse: the destination matrices themselves (each warp stores its own two blocks)
};

// barrier slots
#define HB2_FULL0 0
#define HB2_EMPTY0 2
#define HB2_OUTFULL 4
#define HB2_OUTFREE 5
#define HB2_OLDFULL 6

// ------------------------------------------------------------------------------------------
// Forward "blk" phase: last 8 Cooley-Tukey stages inside 256-blocks + un-bit-reversal.
template <bool SP>
__global__ void __launch_bounds__(HB2_THREADS, 1) k2_fwd_blk(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb2BlkJob J) {
  HB_SMEM_DECL
  const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
  const int team = wid >= 16 ? wid - 16 : wid >> 3, warp = wid >= 16 ? 8 : wid & 7;   // warp 8 = the team's I/O warp
  u64* IN = hb2_align1024(HB_SMEM) + (size_t)team * HB2_TEAM_U64;
  u64* OUT = IN + 2 * HB2_TILE;
  ulonglong2* TW1 = (ulonglong2*)(OUT + HB2_TILE);
  u64* BAR = (u64*)(TW1 + 256);
  const int n1 = J.logN - 8;
  const int G = 1 << (n1 - 4);
  const long U = (long)J.rows.n * G * J.nitems;
  const long vcta = 2L * blockIdx.x + team, vgrid = 2L * gridDim.x;          // every team is a persistent worker of its own
  const long ubeg = U * vcta / vgrid, uend = U * (vcta + 1) / vgrid;
  const int nu = (int)(uend - ubeg);
  const bool epi1 = J.epi == 1, epi3 = J.epi == 3, lazy = J.lazy != 0;
  if (warp == 8 && lane == 0) {
    hb2_mbar_init(BAR + HB2_FULL0, 1); hb2_mbar_init(BAR + HB2_FULL0 + 1, 1);
    hb2_mbar_init(BAR + HB2_EMPTY0, 8); hb2_mbar_init(BAR + HB2_EMPTY0 + 1, 8);
    hb2_mbar_init(BAR + HB2_OUTFULL, 8); hb2_mbar_init(BAR + HB2_OUTFREE, 1); hb2_mbar_init(BAR + HB2_OLDFULL, 1);
    hb2_fence_init();
  }
  __syncthreads();
  if (nu <= 0) return;

  if (warp == 8) {
    // ---------------- I/O warp: one thread drives the TMA
    if (lane != 0) return;
    Hb1Unit cur = hb1_unit(ubeg, G, J.nitems), ahead = cur;
    auto load_in = [&](const Hb1Unit& x, int slot) {
      hb2_mbar_expect(BAR + HB2_FULL0 + slot, HB2_TILE_BYTES);
      hb2_tma_load4(IN + slot * HB2_TILE, J.src[x.it], BAR + HB2_FULL0 + slot, 0, (int)hb_brev((unsigned)x.ug, n1 - 4), 0, J.rows.prime[x.rowi]);
    };
    load_in(ahead, 0);
    if (nu > 1) { ahead = hb1_unit_next(ahead, G, J.nitems); load_in(ahead, 1); }
    unsigned pf = 0;   // parity of the next OUTFULL phase
    for (int k = 0; k < nu; k++) {
      const int prime = J.rows.prime[cur.rowi];
      const bool e = epi1 || (epi3 && J.scal[cur.rowi] != 0);
      if (e) {   // old destination tile into OUT (free: the previous store has been read out)
        hb2_mbar_expect(BAR + HB2_OLDFULL, HB2_TILE_BYTES);
        hb2_tma_load3(OUT, (epi3 ? J.dst2 : J.dst)[cur.it], BAR + HB2_OLDFULL, cur.ug << 4, 0, prime);
      }
      hb2_mbar_wait(BAR + HB2_EMPTY0 + (k & 1), (unsigned)(k >> 1) & 1u);   // pass 1 of unit k has left its slot
      if (k + 2 < nu) { ahead = hb1_unit_next(ahead, G, J.nitems); load_in(ahead, k & 1); }
      hb2_mbar_wait(BAR + HB2_OUTFULL, pf); pf ^= 1u;
      if (epi3 && e) {
        hb2_tma_store3(J.dst2[cur.it], cur.ug << 4, 0, prime, OUT);
        hb2_store_commit(); hb2_store_wait_read();
        hb2_mbar_arrive(BAR + HB2_OUTFREE);
        hb2_mbar_wait(BAR + HB2_OUTFULL, pf); pf ^= 1u;
      }
      hb2_tma_store3(J.dst[cur.it], cur.ug << 4, 0, prime, OUT);
      hb2_store_commit(); hb2_store_wait_read();
      hb2_mbar_arrive(BAR + HB2_OUTFREE);
      cur = hb1_unit_next(cur, G, J.nitems);
    }
    hb2_store_wait_all();
    return;
  }

  // ---------------- compute warps
  const int lo = lane & 15, jj1 = lane >> 4;
  const int j1 = 2 * warp + jj1, slot1 = (int)hb1_brev4((unsigned)j1);
  const int hi = (((lane & 15) >> 1) << 1) | (lane >> 4), jj2 = lane & 1;
  const int j2 = 2 * warp + jj2, slot2 = (int)hb1_brev4((unsigned)j2);
  const unsigned hrev = hb1_brev4((unsigned)hi);
  const int p1 = slot1 * 256, x1 = lo ^ jj1;                 // pass 1: element r at p1 + 16r + lo, written back at p1 + 16r + (x1 ^ r)
  const int p2 = slot2 * 256 + 16 * hi, x2 = hi ^ jj2;       // pass 2: element l at p2 + (x2 ^ l)
  const int po = (int)hrev * 16 + (((warp ^ (int)(hrev & 7u)) << 1) | jj2);   // NAT tile: row brev8(16hi + l) = brev4(l)*16 + hrev, column j2
  Hb1TwPtr tw1;
  tw1.p[0] = TW1 + j1 * 16; tw1.p[1] = tw1.p[0] + 1; tw1.p[2] = tw1.p[0] + 3; tw1.p[3] = tw1.p[0] + 7;
  Hb1Unit cur = hb1_unit(ubeg, G, J.nitems);
  int key = -1;
  u64 q = 0, sc = 0, sc_s = 0;
  Hb1Mod M; M.nq = 0; M.qb = 0; M.qb2 = 0; M.qt = 0; M.qsh = 0;
  Hb1TwReg tw2;
  unsigned pfree = 1, pold = 0;
  for (int k = 0; k < nu; k++) {
    if (cur.rowi * G + cur.ug != key) {   // new (row, block group): modulus and twiddles
      key = cur.rowi * G + cur.ug;
      const HbPrimeDev P = primes[J.rows.prime[cur.rowi]];
      q = P.q; M.nq = P.nq; M.qb = P.qb; M.qb2 = P.qb + P.qb; M.qt = P.qt; M.qsh = P.qsh;
      sc = J.scal[cur.rowi]; sc_s = J.scal_s[cur.rowi];
      const unsigned ugr = hb_brev((unsigned)cur.ug, n1 - 4);
      const unsigned b1 = (unsigned)slot1 * (unsigned)G + ugr, b2 = (unsigned)slot2 * (unsigned)G + ugr;
      __syncwarp();   // the previous unit's pass-1 reads of TW1 are complete
      if (lo < 15) {
        const int e = lo, kk = e >= 7 ? 3 : (e >= 3 ? 2 : (e >= 1 ? 1 : 0));
        const int g = e - ((1 << kk) - 1);
        TW1[j1 * 16 + e] = P.fw[((size_t)1 << (n1 + kk)) + ((size_t)b1 << kk) + g];
      }
      tw2.load([&](int kk, int g) { return P.fw[((size_t)1 << (n1 + 4 + kk)) + ((size_t)b2 << (4 + kk)) + ((size_t)hi << kk) + g]; });
      __syncwarp();
    }
    const bool e = epi1 || (epi3 && sc != 0);
    u64* T = IN + (k & 1) * HB2_TILE;
    hb2_mbar_wait(BAR + HB2_FULL0 + (k & 1), (unsigned)(k >> 1) & 1u);
    u64 a[16];
    hb1_unroll<16>([&](auto r) { a[r] = T[p1 + 16 * r + lo]; });
    hb1_r16_fwd<SP>(a, tw1, M);
    __syncwarp();   // every lane holds its inputs: the block may be overwritten
    hb1_unroll<16>([&](auto r) { T[p1 + 16 * r + (x1 ^ r)] = a[r]; });
    __syncwarp();
    hb1_unroll<16>([&](auto l) { a[l] = T[p2 + (x2 ^ l)]; });
    hb2_fence_async();   // the in-place exchange wrote the slot through the generic proxy; the refill is an async-proxy write
    __syncwarp();
    if (lane == 0) hb2_mbar_arrive(BAR + HB2_EMPTY0 + (k & 1));   // the slot can be refilled
    hb1_r16_fwd<SP>(a, tw2, M);
    hb2_mbar_wait(BAR + HB2_OUTFREE, pfree); pfree ^= 1u;
    if (e) {
      hb2_mbar_wait(BAR + HB2_OLDFULL, pold); pold ^= 1u;
      hb1_unroll<16>([&](auto l) {
        u64* o = OUT + po + 256 * (int)hb1_brev4((unsigned)l);
        u64 v = hb1_shoup4<SP>(*o - a[l] + (M.qb2 + M.qb), sc, sc_s, M);   // (old - x) * scal, x in [0, 8q + 2^32), old < 4q
        if (!lazy) v = hb1_canon4(v, q);
        *o = v;
      });
      if (epi3) {   // two stores from one buffer: the updated matrix first, then x itself
        hb2_fence_async();
        __syncwarp();
        if (lane == 0) hb2_mbar_arrive(BAR + HB2_OUTFULL);
        hb2_mbar_wait(BAR + HB2_OUTFREE, pfree); pfree ^= 1u;
      }
    }
    if (!epi1) {
      hb1_unroll<16>([&](auto l) { OUT[po + 256 * (int)hb1_brev4((unsigned)l)] = lazy ? a[l] : hb1_canon_fwd(a[l], q, M.qb); });
    }
    hb2_fence_async();
    __syncwarp();
    if (lane == 0) hb2_mbar_arrive(BAR + HB2_OUTFULL);
    cur = hb1_unit_next(cur, G, J.nitems);
  }
}

// ------------------------------------------------------------------------------------------
// Inverse "blk" phase: bit-reversal + first 8 Gentleman-Sande stages.
template <bool SP>
__global__ void __launch_bounds__(HB2_THREADS, 1) k2_inv_blk(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb2BlkJob J) {
  HB_SMEM_DECL
  const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
  const int team = wid >= 16 ? wid - 16 : wid >> 3, warp = wid >= 16 ? 8 : wid & 7;
  u64* IN = hb2_align1024(HB_SMEM) + (size_t)team * HB2_TEAM_U64;
  u64* OUT = IN + 2 * HB2_TILE;
  ulonglong2* TW1 = (ulonglong2*)(OUT + HB2_TILE);
  u64* BAR = (u64*)(TW1 + 256);
  const int n1 = J.logN - 8;
  const int G = 1 << (n1 - 4);
  const long U = (long)J.rows.n * G * J.nitems;
  const long vcta = 2L * blockIdx.x + team, vgrid = 2L * gridDim.x;
  const long ubeg = U * vcta / vgrid, uend = U * (vcta + 1) / vgrid;
  const int nu = (int)(uend - ubeg);
  if (warp == 8 && lane == 0) {
    hb2_mbar_init(BAR + HB2_FULL0, 1); hb2_mbar_init(BAR + HB2_FULL0 + 1, 1);
    hb2_mbar_init(BAR + HB2_EMPTY0, 8); hb2_mbar_init(BAR + HB2_EMPTY0 + 1, 8);
    hb2_fence_init();
  }
  __syncthreads();
  if (nu <= 0) return;

  if (warp == 8) {
    if (lane != 0) return;
    Hb1Unit ahead = hb1_unit(ubeg, G, J.nitems);
    auto load_in = [&](const Hb1Unit& x, int slot) {
      hb2_mbar_expect(BAR + HB2_FULL0 + slot, HB2_TILE_BYTES);
      hb2_tma_load3(IN + slot * HB2_TILE, J.src[x.it], BAR + HB2_FULL0 + slot, x.ug << 4, 0, J.rows.prime[x.rowi]);
    };
    load_in(ahead, 0);
    if (nu > 1) { ahead = hb1_unit_next(ahead, G, J.nitems); load_in(ahead, 1); }
    for (int k = 0; k + 2 < nu; k++) {   // loads only: every compute warp stores its own two blocks
      hb2_mbar_wait(BAR + HB2_EMPTY0 + (k & 1), (unsigned)(k >> 1) & 1u);
      ahead = hb1_unit_next(ahead, G, J.nitems); load_in(ahead, k & 1);
    }
    return;
  }

  const int lo = lane & 15, jj1 = lane >> 4;
  const int j1 = 2 * warp + jj1, slot1 = (int)hb1_brev4((unsigned)j1);
  const int hi = (((lane & 15) >> 1) << 1) | (lane >> 4), jj2 = lane & 1;
  const int j2 = 2 * warp + jj2, slot2 = (int)hb1_brev4((unsigned)j2);
  const unsigned hrev = hb1_brev4((unsigned)hi);
  const int p1 = slot1 * 256, x1 = lo ^ jj1;
  const int p2 = slot2 * 256 + 16 * hi, x2 = hi ^ jj2;
  const int po = (int)hrev * 16 + (((warp ^ (int)(hrev & 7u)) << 1) | jj2);
  Hb1TwPtr tw1;
  tw1.p[0] = TW1 + j1 * 16; tw1.p[1] = tw1.p[0] + 1; tw1.p[2] = tw1.p[0] + 3; tw1.p[3] = tw1.p[0] + 7;
  Hb1Unit cur = hb1_unit(ubeg, G, J.nitems);
  int key = -1;
  u64 q = 0;
  Hb1Mod M; M.nq = 0; M.qb = 0; M.qb2 = 0; M.qt = 0; M.qsh = 0;
  Hb1TwReg tw2;
  for (int k = 0; k < nu; k++) {
    if (cur.rowi * G + cur.ug != key) {
      key = cur.rowi * G + cur.ug;
      const HbPrimeDev P = primes[J.rows.prime[cur.rowi]];
      q = P.q; M.nq = P.nq; M.qb = P.qb; M.qb2 = P.qb + P.qb; M.qt = P.qt; M.qsh = P.qsh;
      const unsigned ugr = hb_brev((unsigned)cur.ug, n1 - 4);
      const unsigned b1 = (unsigned)slot1 * (unsigned)G + ugr, b2 = (unsigned)slot2 * (unsigned)G + ugr;
      __syncwarp();
      if (lo < 15) {
        const int e = lo, kk = e >= 7 ? 3 : (e >= 3 ? 2 : (e >= 1 ? 1 : 0));
        const int g = e - ((1 << kk) - 1);
        TW1[j1 * 16 + e] = P.iw[((size_t)1 << (n1 + kk)) + ((size_t)b1 << kk) + g];
      }
      tw2.load([&](int kk, int g) { return P.iw[((size_t)1 << (n1 + 4 + kk)) + ((size_t)b2 << (4 + kk)) + ((size_t)hi << kk) + g]; });
      __syncwarp();
    }
    const u64* T = IN + (k & 1) * HB2_TILE;
    hb2_mbar_wait(BAR + HB2_FULL0 + (k & 1), (unsigned)(k >> 1) & 1u);
    u64 a[16];
    hb1_unroll<16>([&](auto l) { a[l] = T[po + 256 * (int)hb1_brev4((unsigned)l)]; });
    __syncwarp();
    if (lane == 0) hb2_mbar_arrive(BAR + HB2_EMPTY0 + (k & 1));
    hb1_r16_inv<SP>(a, tw2, M);
    // the exchange happens in the output tile (block-contiguous, so each warp's two blocks are private to it): only this
    // warp's own previous store has to be done reading them
    if (lane == 0) hb2_store_wait_read();
    __syncwarp();
    hb1_unroll<16>([&](auto l) { OUT[p2 + (x2 ^ l)] = a[l]; });
    __syncwarp();
    hb1_unroll<16>([&](auto r) { a[r] = OUT[p1 + 16 * r + (x1 ^ r)]; });
    hb1_r16_inv<SP>(a, tw1, M);
    __syncwarp();   // all swizzled reads done before the dense results land
    hb1_unroll<16>([&](auto r) { OUT[p1 + 16 * r + lo] = J.epi == 2 ? a[r] : hb1_canon_inv(a[r], q); });
    hb2_fence_async();
    __syncwarp();
    if (lane == 0) {   // block b = slot*G + brev(ug) of the row, 2 KB contiguous each
      const unsigned ugr = hb_brev((unsigned)cur.ug, n1 - 4);
      u64* d = J.dstp[cur.it] + ((size_t)J.rows.prime[cur.rowi] << J.logN);
      const int s0 = (int)hb1_brev4((unsigned)(2 * warp)), s1 = (int)hb1_brev4((unsigned)(2 * warp + 1));
      hb2_bulk_store(d + (((size_t)s0 * G + ugr) << 8), OUT + s0 * 256, 2048);
      hb2_bulk_store(d + (((size_t)s1 * G + ugr) << 8), OUT + s1 * 256, 2048);
      hb2_store_commit();
    }
    cur = hb1_unit_next(cur, G, J.nitems);
  }
  if (lane == 0) hb2_store_wait_all();
}
