// hb_device_v1.cuh -- register-blocked transform kernels (the fast path for N >= 2^12).
//
// A 256-point sub-transform (either phase of the N = N1 x 256 split) is done as radix-16 x
// radix-16: each thread holds 16 residues in registers, runs 4 butterfly stages (Harvey lazy
// butterflies, Shoup twiddles, values kept in [0,6q) forward / [0,3q) inverse), exchanges through
// a padded shared-memory tile (row stride 17, block stride 273: conflict-free for 64-bit
// accesses), and runs the other 4 stages.  Values crossing a kernel boundary are canonical.
//
//   k1_fwd_blk / k1_inv_blk : "blk" phases, 16 blocks (= 16 adjacent natural-order outputs,
//                             128-byte segments) per CTA, twiddles kept in registers across the
//                             batch-item loop.                       needs log_blk = 8, n1 >= 4
//   k1_fwd_cols/k1_inv_cols : "cols" phases, 16 columns per CTA.     needs n1 = 8 (N = 2^16)
//   k1_conv                 : fused iNTT-cols -> exact CRT -> NTT-cols with 64-thread groups
//                             working on different rows concurrently.  needs n1 = 8
#pragma once
#include <utility>
#include "hb_device.cuh"

#define HB1_RS 17     // row stride inside a 256-element transform tile
#define HB1_BS 273    // tile stride (16*17 + 1)

__device__ __forceinline__ void hb_group_sync(int group, int nthreads) {
#ifdef HB_SIM
  cusim::bar_sync(1 + group, nthreads);
#else
  asm volatile("bar.sync %0, %1;" ::"r"(1 + group), "r"(nthreads) : "memory");
#endif
}

// (hi,lo) += a*b with an explicit carry chain
__device__ __forceinline__ void hb1_mac128(u64& hi, u64& lo, u64 a, u64 b) {
#ifdef HB_SIM
  hb_mac128(hi, lo, a, b);
#else
  asm("{\n\t.reg .u64 pl, ph;\n\t"
      "mul.lo.u64 pl, %2, %3;\n\t"
      "mul.hi.u64 ph, %2, %3;\n\t"
      "add.cc.u64 %0, %0, pl;\n\t"
      "addc.u64 %1, %1, ph;\n\t}"
      : "+l"(lo), "+l"(hi)
      : "l"(a), "l"(b));
#endif
}

// ---- lazy arithmetic of the register kernels (requires q < 2^60) ---------------------------
// The butterflies issue on the ALU pipe (IADD3 / ISETP / SEL / SHF) next to the FMA-heavy pipe that runs IMAD, so every
// helper below is written for the fewest ALU instructions.
//
// Value ranges (B = 4q, kept as the opaque table value qb):
//   Shoup product t = y*w - Qe*q with Qe in [Q-3, Q]  =>  t in [0, 4q) for ANY 64-bit y;
//   forward (CT): x, y in [0, 8q + 2^32)  ->  same;   inverse (GS): x, y in [0, 4q + e), e < 2^48  ->  same
//   (the conditional subtraction compares high words only, which leaves a slack below 2^32 per use).
// Everything stays below 13q + 2^49 < 2^64.

// 32x32 -> 64 product that ptxas keeps as one IMAD.WIDE (and folds a following 64-bit add/sub into its addend)
__device__ __forceinline__ u64 hb1_mulwide(unsigned a, unsigned b) {
#ifdef HB_SIM
  return (u64)a * b;
#else
  u64 r; asm("mul.wide.u32 %0, %1, %2;" : "=l"(r) : "r"(a), "r"(b)); return r;
#endif
}
// Approximate high word of a 64x64 product: hi*hi plus the HIGH halves of the two cross products (one IMAD.WIDE and
// two IMAD.HI); the dropped low parts make the result floor(a*b/2^64) - {0,1,2}.
__device__ __forceinline__ u64 hb1_mulhi_approx(u64 a, u64 b) {
  const unsigned alo = (unsigned)a, ahi = (unsigned)(a >> 32), blo = (unsigned)b, bhi = (unsigned)(b >> 32);
  return hb1_mulwide(ahi, bhi) + (u64)__umulhi(alo, bhi) + (u64)__umulhi(ahi, blo);
}
// Modulus view of the butterfly network.  Generic: nq = 2^64 - q (the subtraction of hi*q is folded into
// the multiply-add chain).  Special (HElib's q = qt*2^s + 1, s >= 32): hi*q mod 2^64 = hi + ((lo32(hi)*qt) << s),
// one 32-bit IMAD and a shift instead of a 64-bit multiply.
struct Hb1Mod {
  u64 nq, qb, qb2;     // 2^64 - q, B = 4q, 2B
  unsigned qt, qsh;
};
#define HB1_MOD(M, P) Hb1Mod M; M.nq = (P).nq; M.qb = (P).qb; M.qb2 = (P).qb + (P).qb; M.qt = (P).qt; M.qsh = (P).qsh
// y*w mod q up to a multiple of q: result in [0,4q) for ANY 64-bit y (Shoup quotient off by <= 3).
template <bool SP>
__device__ __forceinline__ u64 hb1_shoup4(u64 y, u64 w, u64 ws, const Hb1Mod& M) {
  const u64 hi = hb1_mulhi_approx(y, ws);
  if (SP) {
    const unsigned tl = (unsigned)hi * M.qt;
    const unsigned ylo = (unsigned)y, yhi = (unsigned)(y >> 32), wlo = (unsigned)w, whi = (unsigned)(w >> 32);
    const u64 R = hb1_mulwide(ylo, wlo) - hi;                                        // IMAD.WIDE with negated addend
    const unsigned rhi = (unsigned)(R >> 32) + yhi * wlo + ylo * whi - (tl << M.qsh);   // the rest only touches the high word
    return ((u64)rhi << 32) | (unsigned)R;
  }
  return y * w + hi * M.nq;
}
// x in [0,2m) -> [0,m) by one conditional subtraction decided on the sign of x-m (both < 2^63): exact
__device__ __forceinline__ u64 hb1_csub(u64 x, u64 m) {
  const u64 d = x - m;
  return (i64)d < 0 ? x : d;
}
// Lazy conditional subtraction: x -= m when the HIGH word of x exceeds that of m (then x > m).  Otherwise x < m + 2^32.
// One ISETP and a predicated subtract.
__device__ __forceinline__ u64 hb1_csub_hi(u64 x, u64 m) {
#ifdef HB_SIM
  if ((unsigned)(x >> 32) > (unsigned)(m >> 32)) x -= m;
  return x;
#else
  unsigned xl = (unsigned)x, xh = (unsigned)(x >> 32);
  asm("{ .reg .pred p; setp.gt.u32 p, %1, %3; @p sub.cc.u32 %0, %0, %2; @p subc.u32 %1, %1, %3; }"
      : "+r"(xl), "+r"(xh) : "r"((unsigned)m), "r"((unsigned)(m >> 32)));
  return ((u64)xh << 32) | xl;
#endif
}
// Cooley-Tukey butterfly, x,y in [0, 8q + 2^32) -> same
template <bool SP>
__device__ __forceinline__ void hb1_ct(u64& x, u64& y, u64 w, u64 ws, const Hb1Mod& M) {
  const u64 xr = hb1_csub_hi(x, M.qb);          // < 4q + 2^32
  const u64 t = hb1_shoup4<SP>(y, w, ws, M);    // < 4q
  x = xr + t;
  y = xr - t + M.qb;
}
// Gentleman-Sande butterfly, x,y in [0, 4q + e) -> [0, 4q + max(2e, 2^32)), [0, 4q)
template <bool SP>
__device__ __forceinline__ void hb1_gs(u64& x, u64& y, u64 w, u64 ws, const Hb1Mod& M) {
  const u64 s = x + y;
  const u64 d = x - y + M.qb2;                  // > 0 despite the slack of y
  x = hb1_csub_hi(s, M.qb);
  y = hb1_shoup4<SP>(d, w, ws, M);
}
__device__ __forceinline__ u64 hb1_canon4(u64 x, u64 q) {  // exact [0,4q) -> [0,q)
  x = hb1_csub(x, q + q);
  return hb1_csub(x, q);
}
__device__ __forceinline__ u64 hb1_canon_fwd(u64 x, u64 q, u64 qb) {  // forward network output [0, 8q + 2^32) -> [0,q)
  x = hb1_csub_hi(x, qb);                        // < 4q + 2^32 < 2^63: the exact form is valid from here on
  x = hb1_csub(x, q + q);                        // < 2q + 2^32
  x = hb1_csub(x, q);                            // < q + 2^32 < 2q
  return hb1_csub(x, q);
}
__device__ __forceinline__ u64 hb1_canon_inv(u64 x, u64 q) {  // inverse network output [0, 4q + 2^48) -> [0,q)
  x = hb1_csub(x, q + q);                        // < 2q + 2^48   (4q + 2^48 < 2^63)
  x = hb1_csub(x, q);                            // < q + 2^48 < 2q
  return hb1_csub(x, q);
}

// ---- compile-time unrolling ----------------------------------------------------------------
// hb1_unroll<N>(f) calls f(HbC<0>{}), ..., f(HbC<N-1>{}): the index is a constant of the C++ program itself, so every
// access to a per-thread array (the 16 residues, the twiddle pairs, the MAC accumulators) has a constant subscript and
// the array lives in registers.  #pragma unroll only asks the loop unroller, whose decisions depend on the target: on
// sm_90a it left the nested network loops partly rolled and put a[16] and the twiddles in local memory (a 368-byte stack
// frame in every transform kernel), which the sm_100a code generation did not.  Every 16-wide loop around the
// network uses this instead of #pragma unroll.
template <int I> struct HbC {
  static constexpr int value = I;
  __device__ constexpr operator int() const { return I; }
};
template <class F, int... I>
__device__ __forceinline__ void hb1_unroll_seq(F&& f, std::integer_sequence<int, I...>) { (f(HbC<I>{}), ...); }
template <int N, class F>
__device__ __forceinline__ void hb1_unroll(F&& f) { hb1_unroll_seq(f, std::make_integer_sequence<int, N>{}); }

// 4 forward stages on 16 registers; twiddle of stage k (distance 8>>k), group g is tw[(1<<k)-1+g]
struct Hb1TwReg {
  ulonglong2 t[15];
  template <int K, int G> __device__ __forceinline__ ulonglong2 get() const { return t[(1 << K) - 1 + G]; }
  // t[(1<<k)-1+g] = f(k, g) for every stage k and group g
  template <class F> __device__ __forceinline__ void load(F&& f) {
    hb1_unroll<4>([&](auto k) { hb1_unroll<(1 << k)>([&](auto g) { t[(1 << k) - 1 + g] = f((int)k, (int)g); }); });
  }
};
// twiddles read through a pointer per stage (uniform/broadcast loads or shared memory)
struct Hb1TwPtr {
  const ulonglong2* p[4];
  template <int K, int G> __device__ __forceinline__ ulonglong2 get() const { return p[K][G]; }
};
template <bool SP, class TW>
__device__ __forceinline__ void hb1_r16_fwd(u64 (&a)[16], const TW& tw, const Hb1Mod& M) {
  hb1_unroll<4>([&](auto k) {
    constexpr int d = 8 >> k;
    hb1_unroll<(1 << k)>([&](auto g) {
      const ulonglong2 w = tw.template get<k, g>();
      hb1_unroll<d>([&](auto o) { hb1_ct<SP>(a[g * 2 * d + o], a[g * 2 * d + o + d], w.x, w.y, M); });
    });
  });
}
template <bool SP, class TW>
__device__ __forceinline__ void hb1_r16_inv(u64 (&a)[16], const TW& tw, const Hb1Mod& M) {
  hb1_unroll<4>([&](auto kr) {
    constexpr int k = 3 - kr, d = 8 >> k;
    hb1_unroll<(1 << k)>([&](auto g) {
      const ulonglong2 w = tw.template get<k, g>();
      hb1_unroll<d>([&](auto o) { hb1_gs<SP>(a[g * 2 * d + o], a[g * 2 * d + o + d], w.x, w.y, M); });
    });
  });
}
__device__ __forceinline__ unsigned hb1_brev4(unsigned x) {
  return ((x & 1u) << 3) | ((x & 2u) << 1) | ((x & 4u) >> 1) | ((x & 8u) >> 3);
}

// forward epilogues:  0 store x;  1 dst = (dst - x) * scal[row]  (scaleDownToSet, src/DoubleCRT.cpp:1512-1515);
//   3 (fused breakIntoDigits, src/DoubleCRT.cpp:540-556): dst = x and, on rows with scal != 0 (the rows of the later digits),
//     dst2 = (dst2 - x) * scal[row] in the same pass -- the mixed-radix update without a separate pointwise launch.
// lazy != 0: stored values are only reduced to [0,4q) (epilogue products) / [0, 8q + 2^32) (plain x): every consumer inside the
//   fused ciphertext paths (tensor product, evk inner product, inverse blk phase) takes such values.
struct Hb1BlkJob {
  int logN, epi, lazy;
  HbRows rows;
  u64 scal[HB_MAXROWS], scal_s[HB_MAXROWS];
  int nitems;
  const u64* src[HB_MAXB];
  u64* dst[HB_MAXB];
  u64* dst2[HB_MAXB];
};

// 8-byte asynchronous global->shared copy (LDGSTS) and its group fences
__device__ __forceinline__ void hb1_cp8(u64* dst_smem, const u64* src) {
#ifdef HB_SIM
  *dst_smem = *src;
#else
  unsigned sa = (unsigned)__cvta_generic_to_shared(dst_smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(sa), "l"(src) : "memory");
#endif
}
__device__ __forceinline__ void hb1_cp_commit() {
#ifndef HB_SIM
  asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
template <int N> __device__ __forceinline__ void hb1_cp_wait() {
#ifndef HB_SIM
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
#endif
}

// 128-byte shared->global bulk copy (TMA, bulk_group completion): the issuing thread does not wait for the global write,
// so a warp that stores a scattered tile this way goes back to the network instead of stalling on its store queue.
// Both addresses are multiples of 16 bytes.  The writes to the shared source must be fenced into the async proxy first.
__device__ __forceinline__ void hb1_bulk_store128(u64* gdst, const u64* ssrc) {
#ifdef HB_SIM
  for (int i = 0; i < 16; i++) gdst[i] = ssrc[i];
#else
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], 128;"
               ::"l"(gdst), "r"((unsigned)__cvta_generic_to_shared(ssrc)) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void hb1_fence_async() {
#ifndef HB_SIM
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
#endif
}
// the bulk copies of this thread have read their shared source (wait_read) / completed their global writes (wait_all)
__device__ __forceinline__ void hb1_bulk_wait_read() {
#ifndef HB_SIM
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
#endif
}
__device__ __forceinline__ void hb1_bulk_wait_all() {
#ifndef HB_SIM
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
#endif
}

#define HB1_STAGE (16 * HB1_BS + 8)   // u64 per staging/exchange buffer

// Work decomposition of the "blk" kernels: unit = (row, group of 16 blocks, batch item), numbered
// row-major with the item fastest.  A persistent grid of CTAs takes contiguous, balanced chunks of
// units, so consecutive units of a CTA mostly share (row, block group) and re-use its twiddles.
struct Hb1Unit { int rowi, ug, it; };
__device__ __forceinline__ Hb1Unit hb1_unit_next(Hb1Unit x, int G, int nitems) {   // successor without divisions
  if (++x.it == nitems) { x.it = 0; if (++x.ug == G) { x.ug = 0; ++x.rowi; } }
  return x;
}
__device__ __forceinline__ Hb1Unit hb1_unit(long u, int G, int nitems) {
  Hb1Unit x;
  const unsigned per_row = (unsigned)(G * nitems), uu = (unsigned)u;   // unit counts are far below 2^31
  x.rowi = (int)(uu / per_row);
  const int rem = (int)(uu - (unsigned)x.rowi * per_row);
  x.ug = rem / nitems;
  x.it = rem - x.ug * nitems;
  return x;
}
// The CTA's chunk [ubeg, uend) of the rows.n * G * nitems units; false when it is empty.
__device__ __forceinline__ bool hb1_units(const Hb1BlkJob& J, int G, long& ubeg, long& uend) {
  const long U = (long)J.rows.n * G * J.nitems;
  ubeg = U * blockIdx.x / gridDim.x; uend = U * (blockIdx.x + 1) / gridDim.x;
  return ubeg < uend;
}
// Thread tid of a blk kernel works as (blk1, lo) = (tid >> 4, tid & 15) in the pass on r and as (hi, blk2) = (tid >> 4, tid & 15)
// in the pass on lo.  Its twiddles of the pass on r are block blk1's 15 entries of TW1, entry (1<<k)-1+g at TW1[blk1 * 16 + (1<<k)-1+g].
__device__ __forceinline__ Hb1TwPtr hb1_tw1(const ulonglong2* TW1, int tid) {
  Hb1TwPtr tw1;
  tw1.p[0] = TW1 + (tid >> 4) * 16; tw1.p[1] = tw1.p[0] + 1; tw1.p[2] = tw1.p[0] + 3; tw1.p[3] = tw1.p[0] + 7;
  return tw1;
}
// A new (row, block group ug): the modulus view M of the row's prime P and, from its twiddle table tw (P.fw forward, P.iw
// inverse), the twiddles of the pass on r of the group's 16 blocks into TW1 (lane lo < 15 of block blk1 writes entry lo) and
// the thread's twiddles of the pass on lo (block blk2, row hi) into tw2.  Ends with the barrier that makes TW1 visible (the
// previous unit's trailing barrier ordered its last use).  Returns b1, the bit-reversed index of block blk1.
__device__ __forceinline__ unsigned hb1_blk_reload(const HbPrimeDev& P, const ulonglong2* tw, int n1, int ug, int tid, Hb1Mod& M,
                                                   ulonglong2* TW1, Hb1TwReg& tw2) {
  const int blk1 = tid >> 4, lo = tid & 15, hi = tid >> 4, blk2 = tid & 15;
  M.nq = P.nq; M.qb = P.qb; M.qb2 = P.qb + P.qb; M.qt = P.qt; M.qsh = P.qsh;
  const unsigned b1 = hb_brev((ug << 4) + blk1, n1), b2 = hb_brev((ug << 4) + blk2, n1);
  if (lo < 15) {  // entry e = (1<<k)-1+g of block blk1
    int e = lo, k = e >= 7 ? 3 : (e >= 3 ? 2 : (e >= 1 ? 1 : 0));
    int g = e - ((1 << k) - 1);
    TW1[blk1 * 16 + e] = tw[((size_t)1 << (n1 + k)) + ((size_t)b1 << k) + g];
  }
  tw2.load([&](int k, int g) { return tw[((size_t)1 << (n1 + 4 + k)) + ((size_t)b2 << (4 + k)) + ((size_t)hi << k) + g]; });
  __syncthreads();
  return b1;
}

// Forward "blk" phase, 16 blocks per unit, persistent CTAs (grid.x CTAs, 256 threads).
// Software pipelined: each thread prefetches its own 16 inputs of the NEXT unit (and, for the
// mod-down epilogue, the 16 old destination values of the CURRENT unit) into shared memory with
// cp.async while it computes; the staging tile doubles as the exchange tile.  The output rows go out as 128-byte bulk
// copies from shared memory (the epilogue's row from O, the plain row from the exchange tile just read): 8-byte stores
// scattered over 256 natural-order pieces held every warp at its store queue, so the network and the stores did not overlap.
// smem: S[2][HB1_STAGE] | O[16][256] | TW1[256]
template <bool SP>
__global__ void __launch_bounds__(256, 2) k1_fwd_blk(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1BlkJob J) {
  HB_SMEM_DECL
  u64* S = HB_SMEM;
  u64* O = S + 2 * HB1_STAGE;
  ulonglong2* TW1 = (ulonglong2*)(O + 16 * 256);
  const int tid = threadIdx.x;
  const int n1 = J.logN - 8;
  const int G = 1 << (n1 - 4);
  long ubeg, uend;
  if (!hb1_units(J, G, ubeg, uend)) return;
  const int blk1 = tid >> 4, lo = tid & 15;
  const int hi = tid >> 4, blk2 = tid & 15;
  const unsigned hrev = hb1_brev4(hi);
  const bool epi1 = J.epi == 1, epi3 = J.epi == 3, lazy = J.lazy != 0;
  const int own = blk1 * HB1_BS + lo;   // + HB1_RS * r
  const Hb1TwPtr tw1 = hb1_tw1(TW1, tid);

  auto src_ptr = [&](const Hb1Unit& x) {
    const unsigned b = hb_brev((x.ug << 4) + blk1, n1);
    return J.src[x.it] + ((size_t)J.rows.prime[x.rowi] << J.logN) + ((size_t)b << 8) + lo;
  };
  Hb1Unit cur = hb1_unit(ubeg, G, J.nitems);
  {
    const u64* src = src_ptr(cur);
    hb1_unroll<16>([&](auto r) { hb1_cp8(S + own + HB1_RS * r, src + 16 * r); });
  }
  hb1_cp_commit();
  int key = -1, buf = 0;
  u64 q = 0, sc = 0, sc_s = 0;
  Hb1Mod M; M.nq = 0; M.qb = 0; M.qb2 = 0; M.qt = 0; M.qsh = 0;
  Hb1TwReg tw2;
  for (long u = ubeg; u < uend; u++, buf ^= 1) {
    if (cur.rowi * G + cur.ug != key) {   // new (row, block group): reload modulus and twiddles
      key = cur.rowi * G + cur.ug;
      const HbPrimeDev P = primes[J.rows.prime[cur.rowi]];
      q = P.q;
      sc = J.scal[cur.rowi]; sc_s = J.scal_s[cur.rowi];
      hb1_blk_reload(P, P.fw, n1, cur.ug, tid, M, TW1, tw2);
    }
    u64* Sb = S + buf * HB1_STAGE;
    const size_t doff = ((size_t)J.rows.prime[cur.rowi] << J.logN) + (cur.ug << 4) + blk2;
    u64* dst = J.dst[cur.it] + doff;
    const bool epi = epi1 || (epi3 && sc != 0);           // uniform per unit
    u64* old = epi3 ? J.dst2[cur.it] + doff : dst;        // where the value to be updated lives
    if (epi) {
      hb1_unroll<16>([&](auto l) { hb1_cp8(O + l * 256 + tid, old + ((size_t)((hb1_brev4(l) << 4) | hrev) << n1)); });
    }
    hb1_cp_commit();
    Hb1Unit nxt = cur;
    if (u + 1 < uend) {
      nxt = hb1_unit_next(cur, G, J.nitems);
      const u64* src = src_ptr(nxt);
      u64* Sn = S + (buf ^ 1) * HB1_STAGE;
      hb1_unroll<16>([&](auto r) { hb1_cp8(Sn + own + HB1_RS * r, src + 16 * r); });
    }
    hb1_cp_commit();
    hb1_cp_wait<2>();   // this unit's inputs have landed (issued one iteration ago)
    u64 a[16];
    hb1_unroll<16>([&](auto r) { a[r] = Sb[own + HB1_RS * r]; });
    hb1_r16_fwd<SP>(a, tw1, M);
    hb1_unroll<16>([&](auto r) { Sb[own + HB1_RS * r] = a[r]; });
    __syncthreads();
    hb1_unroll<16>([&](auto l) { a[l] = Sb[blk2 * HB1_BS + HB1_RS * hi + l]; });
    hb1_r16_fwd<SP>(a, tw2, M);
    hb1_cp_wait<1>();   // old destination values (epilogue) have landed
    // Output rows leave through 128-byte bulk stores from shared memory, value (l, hi) of the unit at T[l * 256 + tid], so
    // T[l * 256 + 16 * h ..] is the natural-order piece brev8(16 * h + l) * N1 + [16 blocks]: the epilogue's row from O
    // (each value over its own old value), the plain row from Sb once the exchange reads of every thread are done.
    hb1_unroll<16>([&](auto l) {
      if (epi) {
        u64 v = hb1_shoup4<SP>(O[l * 256 + tid] - a[l] + (M.qb2 + M.qb), sc, sc_s, M);   // (old - x) * P^-1, x in [0, 8q + 2^32), old < 4q
        if (!lazy) v = hb1_canon4(v, q);
        O[l * 256 + tid] = v;
      }
      if (!epi1 && !lazy) a[l] = hb1_canon_fwd(a[l], q, M.qb);
    });
    __syncthreads();   // exchange reads of Sb / TW1 done before they are overwritten
    if (!epi1) hb1_unroll<16>([&](auto l) { Sb[l * 256 + tid] = a[l]; });
    hb1_fence_async();
    __syncthreads();
    {   // thread (l, h) = (tid >> 4, tid & 15) sends piece (l, h) of each output row
      const int l = tid >> 4, h = tid & 15;
      const size_t o = (size_t)((hb1_brev4(l) << 4) | hb1_brev4(h)) << n1;
      if (epi) hb1_bulk_store128(old - blk2 + o, O + l * 256 + 16 * h);
      if (!epi1) hb1_bulk_store128(dst - blk2 + o, Sb + l * 256 + 16 * h);
      hb1_bulk_wait_read();
    }
    __syncthreads();   // O and Sb are read out before the next unit's copies land in them
    cur = nxt;
  }
  hb1_cp_wait<0>();
  hb1_bulk_wait_all();
}

// The rescale of NP operand parts fused with their product in one forward blk pass: the body of k1_fwd_blk_tensor (NP = 4)
// and k1_fwd_blk_square (NP = 2).  nitems counts products; src[NP*it + k] is the coefficient-side tile of part k left by
// the conversion, dst[NP*it + k] that part's rows.  A unit (row, group of 16 blocks, item) runs the forward blk phase of the
// NP parts in turn with the twiddles loaded once and applies the subscale epilogue of k1_fwd_blk (v = (old - x) * P^-1, lazy
// in [0,4q)).  The pass-2 positions of a thread do not depend on the part, so the product is thread-local: the earlier
// parts' rescaled values wait in per-thread slots V of shared memory (held in registers they take the kernel past 255
// registers and into local memory), and the last parts combine them.  Part k's old values are read before the unit stores
// anything over them.  Part k stages in S[k & 1] and prefetches part k+1 (part 0 of the next unit after the last part)
// while it computes.  The part loop stays rolled: four unrolled copies of the network (180 KB of code) ran from the
// instruction cache's misses at a third of the speed.
//   NP = 4, a multiplication (scaleDownToSet of a0, a1, b0, b1, then Ctxt::tensorProduct, src/Ctxt.cpp:1563-1608): stores,
//     canonical, a0 <- a0*b0, a1 <- a0*b1 + a1*b0, b0 <- a1*b1 and b1 <- b1' (lazy, as the separate rescale leaves it).
//     a0', a1' and then a1'*b0' mod q wait in V[3]; o0 goes out with part 2 into a0 (read by part 0), o1, o2 and b1' with
//     part 3 into a1, b0 and b1 (read by parts 1, 2, 3).
//   NP = 2, a squaring (bringToSet(naturalPrimeSet()) of a0, a1, then Ctxt::tensorProduct(*this, *this),
//     src/Ctxt.cpp:1704-1708, 1563-1608): stores, canonical, a0 <- a0'^2, a1 <- 2*a0'*a1' and dst2[it] <- a1'^2
//     (2*a0'*a1' is the 128-bit sum a0'*a1' + a0'*a1', below 2^125, reduced once, as a0'*b1' + a1'*b0' is).  a0' waits in
//     V[1]; all three outputs go out with part 1, after its own old values have landed.
// smem: S[2][HB1_STAGE] | O[16][256] | TW1[256] | V[NP - 1][16][256]
template <bool SP, int NP>
__device__ __forceinline__ void hb1_fwd_blk_parts(const HbPrimeDev* __restrict__ primes, const Hb1BlkJob& J) {
  HB_SMEM_DECL
  u64* S = HB_SMEM;
  u64* O = S + 2 * HB1_STAGE;
  ulonglong2* TW1 = (ulonglong2*)(O + 16 * 256);
  u64* V = (u64*)(TW1 + 256);
  const int tid = threadIdx.x;
  const int n1 = J.logN - 8;
  const int G = 1 << (n1 - 4);
  long ubeg, uend;
  if (!hb1_units(J, G, ubeg, uend)) return;
  const int blk1 = tid >> 4, lo = tid & 15;
  const int hi = tid >> 4, blk2 = tid & 15;
  const unsigned hrev = hb1_brev4(hi);
  const int own = blk1 * HB1_BS + lo;   // + HB1_RS * r
  u64* const Vt = V + tid;              // slot j of position l: Vt[j * 4096 + l * 256]
  const Hb1TwPtr tw1 = hb1_tw1(TW1, tid);

  auto prefetch = [&](u64* Sn, const Hb1Unit& x, int k) {
    const unsigned b = hb_brev((x.ug << 4) + blk1, n1);
    const u64* src = J.src[NP * x.it + k] + ((size_t)J.rows.prime[x.rowi] << J.logN) + ((size_t)b << 8) + lo;
    hb1_unroll<16>([&](auto r) { hb1_cp8(Sn + own + HB1_RS * r, src + 16 * r); });
  };
  Hb1Unit cur = hb1_unit(ubeg, G, J.nitems);
  prefetch(S, cur, 0);
  hb1_cp_commit();
  int key = -1;
  u64 q = 0, sc = 0, sc_s = 0, c64 = 0, c64_s = 0, one_s = 0;
  Hb1Mod M; M.nq = 0; M.qb = 0; M.qb2 = 0; M.qt = 0; M.qsh = 0;
  Hb1TwReg tw2;
  for (long u = ubeg; u < uend; u++) {
    if (cur.rowi * G + cur.ug != key) {   // new (row, block group): reload modulus and twiddles
      key = cur.rowi * G + cur.ug;
      const HbPrimeDev P = primes[J.rows.prime[cur.rowi]];
      q = P.q; c64 = P.c64; c64_s = P.c64_s; one_s = P.one_s;
      sc = J.scal[cur.rowi]; sc_s = J.scal_s[cur.rowi];
      hb1_blk_reload(P, P.fw, n1, cur.ug, tid, M, TW1, tw2);
    }
    const size_t doff = ((size_t)J.rows.prime[cur.rowi] << J.logN) + (cur.ug << 4) + blk2;
    u64* const* dst = J.dst + NP * cur.it;
    u64* const o2 = J.dst2[cur.it];   // NP = 2 only
    const bool more = u + 1 < uend;
    const Hb1Unit nxt = more ? hb1_unit_next(cur, G, J.nitems) : cur;
#pragma unroll 1
    for (int k = 0; k < NP; k++) {
      u64* Sb = S + (NP == 2 ? k : k & 1) * HB1_STAGE;   // S[k & 1]: two parts need no mask (and ptxas keeps one)
      const u64* old = dst[k] + doff;
      hb1_unroll<16>([&](auto l) { hb1_cp8(O + l * 256 + tid, old + ((size_t)((hb1_brev4(l) << 4) | hrev) << n1)); });
      hb1_cp_commit();
      if (k < NP - 1) prefetch(S + ((k + 1) & 1) * HB1_STAGE, cur, k + 1);
      else if (more) prefetch(S, nxt, 0);
      hb1_cp_commit();
      hb1_cp_wait<2>();   // this part's inputs have landed (issued one part ago)
      u64 a[16];
      hb1_unroll<16>([&](auto r) { a[r] = Sb[own + HB1_RS * r]; });
      hb1_r16_fwd<SP>(a, tw1, M);
      hb1_unroll<16>([&](auto r) { Sb[own + HB1_RS * r] = a[r]; });
      __syncthreads();
      hb1_unroll<16>([&](auto l) { a[l] = Sb[blk2 * HB1_BS + HB1_RS * hi + l]; });
      hb1_r16_fwd<SP>(a, tw2, M);
      hb1_cp_wait<1>();   // old values of this part have landed
      hb1_unroll<16>([&](auto l) {   // (old - x) * P^-1 in [0,4q), x in [0, 8q + 2^32), old < 4q
        a[l] = hb1_shoup4<SP>(O[l * 256 + tid] - a[l] + (M.qb2 + M.qb), sc, sc_s, M);
      });
      if constexpr (NP == 4) {
        if (k < 2) {   // a0', a1'
          hb1_unroll<16>([&](auto l) { Vt[k * 4096 + l * 256] = a[l]; });
        } else if (k == 2) {   // b0': o0 = a0'*b0' out, a1'*b0' kept
          hb1_unroll<16>([&](auto l) {
            const size_t o = doff + ((size_t)((hb1_brev4(l) << 4) | hrev) << n1);
            const u64 x0 = Vt[l * 256], x1 = Vt[4096 + l * 256], v = a[l];
            dst[0][o] = hb_reduce128(__umul64hi(x0, v), x0 * v, q, c64, c64_s, one_s);
            Vt[2 * 4096 + l * 256] = hb_reduce128(__umul64hi(x1, v), x1 * v, q, c64, c64_s, one_s);
          });
        } else {   // b1': o1 = a0'*b1' + a1'*b0', o2 = a1'*b1'
          hb1_unroll<16>([&](auto l) {
            const size_t o = doff + ((size_t)((hb1_brev4(l) << 4) | hrev) << n1);
            const u64 x0 = Vt[l * 256], x1 = Vt[4096 + l * 256], v = a[l];
            u64 h = 0, w = Vt[2 * 4096 + l * 256];
            hb1_mac128(h, w, x0, v);
            dst[1][o] = hb_reduce128(h, w, q, c64, c64_s, one_s);
            dst[2][o] = hb_reduce128(__umul64hi(x1, v), x1 * v, q, c64, c64_s, one_s);
            dst[3][o] = v;
          });
        }
      } else {
        if (k == 0) {   // a0'
          hb1_unroll<16>([&](auto l) { Vt[l * 256] = a[l]; });
        } else {        // a1': a0'^2, 2*a0'*a1', a1'^2 out
          hb1_unroll<16>([&](auto l) {
            const size_t o = doff + ((size_t)((hb1_brev4(l) << 4) | hrev) << n1);
            const u64 x0 = Vt[l * 256], v = a[l];
            u64 h = 0, w = 0;
            hb1_mac128(h, w, x0, v);
            hb1_mac128(h, w, x0, v);
            dst[0][o] = hb_reduce128(__umul64hi(x0, x0), x0 * x0, q, c64, c64_s, one_s);
            dst[1][o] = hb_reduce128(h, w, q, c64, c64_s, one_s);
            o2[o] = hb_reduce128(__umul64hi(v, v), v * v, q, c64, c64_s, one_s);
          });
        }
      }
      __syncthreads();   // exchange reads of Sb / TW1 done before they are overwritten
    }
    cur = nxt;
  }
  hb1_cp_wait<0>();
}
template <bool SP>
__global__ void __launch_bounds__(256, 1) k1_fwd_blk_tensor(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1BlkJob J) {
  hb1_fwd_blk_parts<SP, 4>(primes, J);
}
template <bool SP>
__global__ void __launch_bounds__(256, 1) k1_fwd_blk_square(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1BlkJob J) {
  hb1_fwd_blk_parts<SP, 2>(primes, J);
}

// Inverse "blk" phase (bit-reversal + first 8 GS stages), same decomposition and pipelining.
// smem: S[2][HB1_STAGE] | TW1[256]
template <bool SP>
__global__ void __launch_bounds__(256, 2) k1_inv_blk(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1BlkJob J) {
  HB_SMEM_DECL
  u64* S = HB_SMEM;
  ulonglong2* TW1 = (ulonglong2*)(S + 2 * HB1_STAGE);
  const int tid = threadIdx.x;
  const int n1 = J.logN - 8;
  const int G = 1 << (n1 - 4);
  long ubeg, uend;
  if (!hb1_units(J, G, ubeg, uend)) return;
  const int blk1 = tid >> 4, lo = tid & 15;   // second pass (on r)
  const int hi = tid >> 4, blk2 = tid & 15;   // first pass (on lo)
  const unsigned hrev = hb1_brev4(hi);
  const Hb1TwPtr tw1 = hb1_tw1(TW1, tid);
  const int own = blk2 * HB1_BS + HB1_RS * hi;   // + l
  auto src_ptr = [&](const Hb1Unit& x) {
    return J.src[x.it] + ((size_t)J.rows.prime[x.rowi] << J.logN) + (x.ug << 4) + blk2;
  };
  Hb1Unit cur = hb1_unit(ubeg, G, J.nitems);
  {
    const u64* src = src_ptr(cur);
    hb1_unroll<16>([&](auto l) { hb1_cp8(S + own + l, src + ((size_t)((hb1_brev4(l) << 4) | hrev) << n1)); });
  }
  hb1_cp_commit();
  int key = -1, buf = 0;
  u64 q = 0;
  Hb1Mod M; M.nq = 0; M.qb = 0; M.qb2 = 0; M.qt = 0; M.qsh = 0;
  unsigned b1 = 0;
  Hb1TwReg tw2;
  for (long u = ubeg; u < uend; u++, buf ^= 1) {
    if (cur.rowi * G + cur.ug != key) {
      key = cur.rowi * G + cur.ug;
      const HbPrimeDev P = primes[J.rows.prime[cur.rowi]];
      q = P.q;
      b1 = hb1_blk_reload(P, P.iw, n1, cur.ug, tid, M, TW1, tw2);
    }
    u64* Sb = S + buf * HB1_STAGE;
    Hb1Unit nxt = cur;
    if (u + 1 < uend) {
      nxt = hb1_unit_next(cur, G, J.nitems);
      const u64* src = src_ptr(nxt);
      u64* Sn = S + (buf ^ 1) * HB1_STAGE;
      hb1_unroll<16>([&](auto l) { hb1_cp8(Sn + own + l, src + ((size_t)((hb1_brev4(l) << 4) | hrev) << n1)); });
    }
    hb1_cp_commit();
    hb1_cp_wait<1>();
    u64 a[16];
    hb1_unroll<16>([&](auto l) { a[l] = Sb[own + l]; });
    hb1_r16_inv<SP>(a, tw2, M);
    hb1_unroll<16>([&](auto l) { Sb[own + l] = a[l]; });
    __syncthreads();
    hb1_unroll<16>([&](auto r) { a[r] = Sb[blk1 * HB1_BS + HB1_RS * r + lo]; });
    hb1_r16_inv<SP>(a, tw1, M);
    u64* dst = J.dst[cur.it] + ((size_t)J.rows.prime[cur.rowi] << J.logN) + ((size_t)b1 << 8) + lo;
    hb1_unroll<16>([&](auto r) { dst[16 * r] = J.epi == 2 ? a[r] : hb1_canon_inv(a[r], q); });   // epi 2: the consumer is a register kernel (lazy values are fine)
    __syncthreads();
    cur = nxt;
  }
  hb1_cp_wait<0>();
}

struct Hb1ColsJob {
  int logN;
  HbRows rows;
  int nitems;
  const u64* src[HB_MAXB];
  u64* dst[HB_MAXB];
  // inverse phase of the prime-sharded conversion (hb_conv_make_y[_bcast]): the final factor is scal[row] (= N^-1 * (Q_D/q_j)^-1,
  // Shoup companion in scal_s) instead of N^-1, and every result is also stored into the same place of up to 8 peer GPUs' buffers
  // (CUDA-IPC mappings, the stores travel over NVLink): the y rows cross the fabric once, straight from the producing kernel
  int has_scal, npeers;
  u64 scal[HB_MAXROWS], scal_s[HB_MAXROWS];
  u64* peer[8][HB_MAXB];
};

// "cols" phases for n1 = 8 (N = 2^16): tile [256][16 columns].  grid = (16, nrows, item-groups).
template <bool SP>
__global__ void __launch_bounds__(256, 2) k1_fwd_cols(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1ColsJob J) {
  HB_SMEM_DECL
  u64* T = HB_SMEM;
  const int tid = threadIdx.x;
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  HB1_MOD(M, P);
  const size_t rowoff = (size_t)pi << J.logN;
  const unsigned c0 = blockIdx.x << 4;
  const int c = tid & 15, x = tid >> 4;  // x = lo in pass 1 (on r), hi in pass 2 (on lo)
  Hb1TwPtr tw1;
  tw1.p[0] = P.fw + 1; tw1.p[1] = P.fw + 2; tw1.p[2] = P.fw + 4; tw1.p[3] = P.fw + 8;
  Hb1TwReg tw2;
  tw2.load([&](int k, int g) { return P.fw[(16 << k) + (x << k) + g]; });
  for (int it = blockIdx.z; it < J.nitems; it += gridDim.z) {
    const u64* src = J.src[it] + rowoff + c0 + c;
    u64* dst = J.dst[it] + rowoff + c0 + c;
    u64 a[16];
    hb1_unroll<16>([&](auto r) { a[r] = src[(size_t)(16 * r + x) << 8]; });
    hb1_r16_fwd<SP>(a, tw1, M);
    hb1_unroll<16>([&](auto r) { T[c * HB1_BS + HB1_RS * r + x] = a[r]; });
    __syncthreads();
    hb1_unroll<16>([&](auto l) { a[l] = T[c * HB1_BS + HB1_RS * x + l]; });
    hb1_r16_fwd<SP>(a, tw2, M);
    hb1_unroll<16>([&](auto l) { dst[(size_t)(16 * x + l) << 8] = a[l]; });   // lazy, [0, 8q + 2^32): the consumer is always k1_fwd_blk
    __syncthreads();
  }
}
template <bool SP>
__global__ void __launch_bounds__(256, 2) k1_inv_cols(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1ColsJob J) {
  HB_SMEM_DECL
  u64* T = HB_SMEM;
  const int tid = threadIdx.x;
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const u64 q = P.q; HB1_MOD(M, P);
  const size_t rowoff = (size_t)pi << J.logN;
  const unsigned c0 = blockIdx.x << 4;
  const int c = tid & 15, x = tid >> 4;  // x = hi in pass 1 (on lo), lo in pass 2 (on r)
  Hb1TwPtr tw1;
  tw1.p[0] = P.iw + 1; tw1.p[1] = P.iw + 2; tw1.p[2] = P.iw + 4; tw1.p[3] = P.iw + 8;
  Hb1TwReg tw2;
  tw2.load([&](int k, int g) { return P.iw[(16 << k) + (x << k) + g]; });
  for (int it = blockIdx.z; it < J.nitems; it += gridDim.z) {
    const u64* src = J.src[it] + rowoff + c0 + c;
    u64* dst = J.dst[it] + rowoff + c0 + c;
    u64 a[16];
    hb1_unroll<16>([&](auto l) { a[l] = src[(size_t)(16 * x + l) << 8]; });
    hb1_r16_inv<SP>(a, tw2, M);
    hb1_unroll<16>([&](auto l) { T[c * HB1_BS + HB1_RS * x + l] = a[l]; });
    __syncthreads();
    hb1_unroll<16>([&](auto r) { a[r] = T[c * HB1_BS + HB1_RS * r + x]; });
    hb1_r16_inv<SP>(a, tw1, M);
    const u64 fm = J.has_scal ? J.scal[blockIdx.y] : P.ninv, fs = J.has_scal ? J.scal_s[blockIdx.y] : P.ninv_s;
    hb1_unroll<16>([&](auto r) {
      const u64 v = hb_mul_shoup(a[r], fm, fs, q);
      const size_t o = (size_t)(16 * r + x) << 8;
      dst[o] = v;
      for (int p = 0; p < J.npeers; p++) J.peer[p][it][rowoff + c0 + c + o] = v;
    });
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// Fused exact base conversion, n1 = 8, 4 columns per CTA, NG groups of 64 threads.
// Row tile layout: Y[c*HB1C_BS + 17*(i1>>4) + (i1&15)], c in [0,4), i1 in [0,256).
#define HB1C_BS 276           // column stride in k1_conv (2*276 mod 32 = 8: 4 cols x 4 rows conflict-free)
#define HB1_TS (4 * HB1C_BS)  // u64 per row tile (1104)
#define HB1_VS 260            // column stride of the quotient tile (260 mod 16 = 4)

struct Hb1ConvJob {
  const HbConvDev* cv;
  int logN, ngroups;
  int nitems;
  const u64* src[HB_MAXB];
  u64* dst[HB_MAXB];
  u64* stats;
  int src_is_y;   // 1: sources are y_j coefficient rows already (prime-sharded path)
  double* frac[HB_MAXB];   // optional x/Q per coefficient for the embedding norm
};

template <bool SP>
__global__ void __launch_bounds__(640, 1) k1_conv(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1ConvJob J) {
  HB_SMEM_DECL
  const HbConvDev* cv = J.cv;
  const int n = cv->n, nt = cv->nt, NG = J.ngroups;
  u64* Y = HB_SMEM;                               // [n][HB1_TS]
  i64* Vb = (i64*)(Y + (size_t)n * HB1_TS);       // [4][HB1_VS]  index c*HB1_VS + i1 (padded: the 4 columns of a half-warp hit different banks)
  u64* W = (u64*)(Vb + 4 * HB1_VS);               // [NG][HB1_TS]
  const int tid = threadIdx.x;
  const int grp = tid >> 6, gt = tid & 63;
  const int c = gt & 3, x = gt >> 2;              // x in [0,16)
  const unsigned c0 = blockIdx.x << 2;
  const u64* src = J.src[blockIdx.y];
  u64* dst = J.dst[blockIdx.y];

  // ---- sources: inverse cols phase, * (Q/q_j)^-1 * N^-1, canonical y_j into Y[j]
  for (int j = grp; j < n; j += NG) {
    const int pi = cv->src_prime[j];
    const HbPrimeDev P = primes[pi];
    const u64 q = P.q; HB1_MOD(M, P);
    const u64* s = src + ((size_t)pi << J.logN) + c0 + c;
    u64* Yj = Y + (size_t)j * HB1_TS + c * HB1C_BS;
    u64 a[16];
    hb1_unroll<16>([&](auto l) { a[l] = s[(size_t)(16 * x + l) << 8]; });
    if (J.src_is_y) {   // uniform per launch: no transform, just stage the tile
      hb1_unroll<16>([&](auto l) { Yj[HB1_RS * x + l] = a[l]; });
      continue;
    }
    {
      Hb1TwPtr tw;
      tw.p[0] = P.iw + 16 + x; tw.p[1] = P.iw + 32 + 2 * x; tw.p[2] = P.iw + 64 + 4 * x; tw.p[3] = P.iw + 128 + 8 * x;
      hb1_r16_inv<SP>(a, tw, M);
    }
    hb1_unroll<16>([&](auto l) { Yj[HB1_RS * x + l] = a[l]; });
    hb_group_sync(grp, 64);
    hb1_unroll<16>([&](auto r) { a[r] = Yj[HB1_RS * r + x]; });
    {
      Hb1TwPtr tw;
      tw.p[0] = P.iw + 1; tw.p[1] = P.iw + 2; tw.p[2] = P.iw + 4; tw.p[3] = P.iw + 8;
      hb1_r16_inv<SP>(a, tw, M);
    }
    const u64 t = cv->tn[j], ts = cv->tn_s[j];
    hb1_unroll<16>([&](auto r) { Yj[HB1_RS * r + x] = hb_mul_shoup(a[r], t, ts, q); });
  }
  __syncthreads();
  // ---- v (multiple of Q to subtract, incl. the BGV correction) per coefficient
  for (int e = tid; e < 1024; e += blockDim.x) {
    const int cc = e >> 8, i1 = e & 255;
    double* fr = J.frac[blockIdx.y];
    double f;
    Vb[cc * HB1_VS + i1] = hb_conv_v(cv, Y + cc * HB1C_BS + HB1_RS * (i1 >> 4) + (i1 & 15), HB1_TS, J.stats, fr ? &f : nullptr);
    if (fr) fr[((size_t)i1 << 8) + c0 + cc] = f;
  }
  __syncthreads();
  // ---- targets: x mod q_t in registers, forward cols phase, store
  u64* Wg = W + (size_t)grp * HB1_TS + c * HB1C_BS;
  for (int t = grp; t < nt; t += NG) {
    const int pi = cv->tgt_prime[t];
    const HbPrimeDev P = primes[pi];
    HB1_MOD(M, P);
    const u64* ct = cv->c + (size_t)t * n;
    u64 a[16];
    {
      const u64 negq = cv->negQ[t], posq = cv->Qmod[t];
      hb1_unroll<2>([&](auto h) {   // two halves of 8 coefficients: 32 accumulator registers live
        u64 ahi[8], alo[8];
        hb1_unroll<8>([&](auto r) {
          const i64 v = Vb[c * HB1_VS + 16 * (8 * h + r) + x];
          const u64 m = v >= 0 ? (u64)v : (u64)(-v);
          const u64 f = v >= 0 ? negq : posq;
          if ((m >> 32) == 0) {   // |v| <= n/2 + p/2: one word unless the plaintext modulus is huge -- 32x64 product, two wide multiplies
            const u64 p0 = hb1_mulwide((unsigned)m, (unsigned)f);
            const u64 p1 = hb1_mulwide((unsigned)m, (unsigned)(f >> 32)) + (p0 >> 32);
            alo[r] = (p1 << 32) | (unsigned)p0; ahi[r] = p1 >> 32;
          } else { alo[r] = m * f; ahi[r] = __umul64hi(m, f); }
        });
        for (int j = 0; j < n; j++) {
          const u64 cj = ct[j];
          const u64* Yj = Y + (size_t)j * HB1_TS + c * HB1C_BS + x + HB1_RS * 8 * h;
          hb1_unroll<8>([&](auto r) { hb1_mac128(ahi[r], alo[r], Yj[HB1_RS * r], cj); });
        }
        hb1_unroll<8>([&](auto r) { a[8 * h + r] = hb_reduce128_lazy(ahi[r], alo[r], P); });   // [0,4q): fine for the CT network
      });
    }
    {
      Hb1TwPtr tw;
      tw.p[0] = P.fw + 1; tw.p[1] = P.fw + 2; tw.p[2] = P.fw + 4; tw.p[3] = P.fw + 8;
      hb1_r16_fwd<SP>(a, tw, M);
    }
    hb_group_sync(grp, 64);   // previous target's pass-2 reads of Wg are complete
    hb1_unroll<16>([&](auto r) { Wg[HB1_RS * r + x] = a[r]; });
    hb_group_sync(grp, 64);
    hb1_unroll<16>([&](auto l) { a[l] = Wg[HB1_RS * x + l]; });
    {
      Hb1TwPtr tw;
      tw.p[0] = P.fw + 16 + x; tw.p[1] = P.fw + 32 + 2 * x; tw.p[2] = P.fw + 64 + 4 * x; tw.p[3] = P.fw + 128 + 8 * x;
      hb1_r16_fwd<SP>(a, tw, M);
    }
    u64* d = dst + ((size_t)pi << J.logN) + c0 + c;
    hb1_unroll<16>([&](auto l) { d[(size_t)(16 * x + l) << 8] = a[l]; });   // lazy: k1_fwd_blk finishes the transform
  }
}

// ------------------------------------------------------------------------------------------
// Conversion from ONE source prime (the CKKS rescale / any single-prime mod-down without a plaintext
// correction): x = balanced(y), y the coefficient modulo q_s, so there is no MAC loop and no fixed-point
// quotient -- x mod q_t = (y mod q_t) - [y > (q_s-1)/2] * (q_s mod q_t).  CQ quads of 4 columns per CTA keep
// more groups busy during the (single-row) source phase.
// smem: Y[CQ][HB1_TS] | W[NG][HB1_TS]
struct Hb1Conv1Job {
  int logN, ngroups, cq, nitems;
  int src_prime, nt;
  int tgt_prime[HB_MAXROWS];
  u64 qs_mod[HB_MAXROWS];      // q_s mod q_t
  unsigned char nored[HB_MAXROWS];   // q_s <= 7 q_t: y (< q_s) needs no reduction modulo q_t before the lazy forward network
  u64 ninv, ninv_s;            // N^-1 mod q_s (+Shoup): the (Q/q_j)^-1 factor is 1 for a single prime
  const u64* src[HB_MAXB];
  u64* dst[HB_MAXB];
};
template <bool SP>
__global__ void __launch_bounds__(640, 1) k1_conv1(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1Conv1Job J) {
  HB_SMEM_DECL
  const int NG = J.ngroups, CQ = J.cq, nt = J.nt;
  u64* Y = HB_SMEM;                               // [CQ][HB1_TS]
  u64* W = Y + (size_t)CQ * HB1_TS;               // [NG][HB1_TS]
  const int tid = threadIdx.x;
  const int grp = tid >> 6, gt = tid & 63;
  const int c = gt & 3, x = gt >> 2;
  const unsigned c0 = blockIdx.x * 4u * (unsigned)CQ;
  const u64* src = J.src[blockIdx.y];
  u64* dst = J.dst[blockIdx.y];
  const HbPrimeDev PS = primes[J.src_prime];
  // ---- source: inverse cols phase of the quads, canonical coefficients into Y
  for (int qd = grp; qd < CQ; qd += NG) {
    HB1_MOD(M, PS);
    const u64* s = src + ((size_t)J.src_prime << J.logN) + c0 + 4 * qd + c;
    u64* Yq = Y + (size_t)qd * HB1_TS + c * HB1C_BS;
    u64 a[16];
    hb1_unroll<16>([&](auto l) { a[l] = s[(size_t)(16 * x + l) << 8]; });
    {
      Hb1TwPtr tw;
      tw.p[0] = PS.iw + 16 + x; tw.p[1] = PS.iw + 32 + 2 * x; tw.p[2] = PS.iw + 64 + 4 * x; tw.p[3] = PS.iw + 128 + 8 * x;
      hb1_r16_inv<SP>(a, tw, M);
    }
    hb1_unroll<16>([&](auto l) { Yq[HB1_RS * x + l] = a[l]; });
    hb_group_sync(grp, 64);
    hb1_unroll<16>([&](auto r) { a[r] = Yq[HB1_RS * r + x]; });
    {
      Hb1TwPtr tw;
      tw.p[0] = PS.iw + 1; tw.p[1] = PS.iw + 2; tw.p[2] = PS.iw + 4; tw.p[3] = PS.iw + 8;
      hb1_r16_inv<SP>(a, tw, M);
    }
    hb1_unroll<16>([&](auto r) { Yq[HB1_RS * r + x] = hb_mul_shoup(a[r], J.ninv, J.ninv_s, PS.q); });
  }
  __syncthreads();
  // ---- targets
  const u64 qs_half = (PS.q - 1) >> 1;
  u64* Wg = W + (size_t)grp * HB1_TS + c * HB1C_BS;
  for (int w = grp; w < nt * CQ; w += NG) {
    const int t = w / CQ, qd = w - t * CQ;
    const int pi = J.tgt_prime[t];
    const HbPrimeDev P = primes[pi];
    HB1_MOD(M, P);
    const u64 adj = P.q - J.qs_mod[t];          // -(q_s mod q_t) mod q_t, in (0, q_t]
    const u64* Yq = Y + (size_t)qd * HB1_TS + c * HB1C_BS + x;
    const bool nored = J.nored[t] != 0;         // uniform per target: same-size primes (every ctxt / special prime of a chain)
    u64 a[16];
    hb1_unroll<16>([&](auto r) {
      const u64 y = Yq[HB1_RS * r];
      u64 v = nored ? y : y - __umul64hi(y, P.one_s) * P.q;   // y < 7 q_t as it is, or y mod q_t in [0, 2 q_t)
      if (y > qs_half) v += adj;                  // balanced representative: subtract q_s   -> below 8 q_t: fine for the CT network
      a[r] = v;
    });
    {
      Hb1TwPtr tw;
      tw.p[0] = P.fw + 1; tw.p[1] = P.fw + 2; tw.p[2] = P.fw + 4; tw.p[3] = P.fw + 8;
      hb1_r16_fwd<SP>(a, tw, M);
    }
    hb_group_sync(grp, 64);   // the previous item's pass-2 reads of Wg are complete
    hb1_unroll<16>([&](auto r) { Wg[HB1_RS * r + x] = a[r]; });
    hb_group_sync(grp, 64);
    hb1_unroll<16>([&](auto l) { a[l] = Wg[HB1_RS * x + l]; });
    {
      Hb1TwPtr tw;
      tw.p[0] = P.fw + 16 + x; tw.p[1] = P.fw + 32 + 2 * x; tw.p[2] = P.fw + 64 + 4 * x; tw.p[3] = P.fw + 128 + 8 * x;
      hb1_r16_fwd<SP>(a, tw, M);
    }
    u64* d = dst + ((size_t)pi << J.logN) + c0 + 4 * qd + c;
    hb1_unroll<16>([&](auto l) { d[(size_t)(16 * x + l) << 8] = a[l]; });   // lazy: k1_fwd_blk finishes the transform
  }
}

// ------------------------------------------------------------------------------------------
// Ctxt::keySwitchDigits (src/Ctxt.cpp:191-230), streaming form for power-of-two m: every thread owns two adjacent
// coefficients of one row (128-bit loads and stores), keeps the 2*ND evaluation-key words of that position in registers
// and loops over the batch items, so the key rows are fetched once per launch instead of once per item.
// modes 0 and 1 of HbKsJob (mode 2, the hoisted automorphism, gathers and stays with k_ks_inner).
// grid = (N / 512, nrows, item groups)
__device__ __forceinline__ ulonglong2 hb1_ld2(const u64* p) { return *reinterpret_cast<const ulonglong2*>(p); }
__device__ __forceinline__ void hb1_st2(u64* p, u64 x, u64 y) { ulonglong2 v; v.x = x; v.y = y; *reinterpret_cast<ulonglong2*>(p) = v; }
template <int ND>
__global__ void __launch_bounds__(256) k1_ks_inner(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbKsJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t o = (size_t)pi * (size_t)J.N + 2 * ((size_t)blockIdx.x * 256 + threadIdx.x);
  ulonglong2 ea[ND], eb[ND];
#pragma unroll
  for (int i = 0; i < ND; i++) { ea[i] = hb1_ld2(J.evk_a[i] + o); eb[i] = hb1_ld2(J.evk_b[i] + o); }
  const int own = J.own_dig[blockIdx.y];
  const u64 sc = J.scal[blockIdx.y];
  const bool rd = J.mode == 0 || sc != 0;
  for (int it = blockIdx.z; it < J.nitems; it += gridDim.z) {
    ulonglong2 d[ND];
#pragma unroll
    for (int i = 0; i < ND; i++) d[i] = hb1_ld2((i == own ? J.own[it] : J.dig[it][i]) + o);
    u64 h0x = 0, l0x = 0, h0y = 0, l0y = 0, h1x = 0, l1x = 0, h1y = 0, l1y = 0;
    if (rd) {
      const ulonglong2 p0 = hb1_ld2(J.out0[it] + o), p1 = hb1_ld2(J.out1[it] + o);
      if (J.mode == 0) { l0x = p0.x; l0y = p0.y; l1x = p1.x; l1y = p1.y; }
      else { hb1_mac128(h0x, l0x, p0.x, sc); hb1_mac128(h0y, l0y, p0.y, sc); hb1_mac128(h1x, l1x, p1.x, sc); hb1_mac128(h1y, l1y, p1.y, sc); }
    }
#pragma unroll
    for (int i = 0; i < ND; i++) {
      hb1_mac128(h0x, l0x, d[i].x, eb[i].x); hb1_mac128(h0y, l0y, d[i].y, eb[i].y);
      hb1_mac128(h1x, l1x, d[i].x, ea[i].x); hb1_mac128(h1y, l1y, d[i].y, ea[i].y);
    }
    hb1_st2(J.out0[it] + o, hb_reduce128(h0x, l0x, P), hb_reduce128(h0y, l0y, P));
    hb1_st2(J.out1[it] + o, hb_reduce128(h1x, l1x, P), hb_reduce128(h1y, l1y, P));
  }
}

// ------------------------------------------------------------------------------------------
// Ctxt::tensorProduct (src/Ctxt.cpp:1563-1608), streaming form for power-of-two m: two adjacent coefficients per thread,
// 128-bit loads and stores (the generic k_pointwise moves 8 bytes per access).  Inputs may be lazy up to 2^63.5: a0*b1 +
// a1*b0 is summed in 128 bits before its one reduction, and two products of 64-bit values could pass 2^128 (the callers
// pass values below 8q + 2^32 < 2^63); outputs canonical.  In place is allowed (every thread reads its four inputs before
// it writes).     grid = (N / 512, nrows, nitems)
struct Hb1TensorJob {
  u64 N;
  HbRows rows;
  int nitems;
  const u64* a0[HB_MAXB]; const u64* a1[HB_MAXB]; const u64* b0[HB_MAXB]; const u64* b1[HB_MAXB];
  u64* o0[HB_MAXB]; u64* o1[HB_MAXB]; u64* o2[HB_MAXB];
};
__global__ void __launch_bounds__(256) k1_tensor(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1TensorJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const int it = blockIdx.z;
  const size_t o = (size_t)pi * (size_t)J.N + 2 * ((size_t)blockIdx.x * 256 + threadIdx.x);
  const ulonglong2 a0 = hb1_ld2(J.a0[it] + o), a1 = hb1_ld2(J.a1[it] + o), b0 = hb1_ld2(J.b0[it] + o), b1 = hb1_ld2(J.b1[it] + o);
  u64 hx = 0, lx = 0, hy = 0, ly = 0;
  hb1_mac128(hx, lx, a0.x, b1.x); hb1_mac128(hx, lx, a1.x, b0.x);
  hb1_mac128(hy, ly, a0.y, b1.y); hb1_mac128(hy, ly, a1.y, b0.y);
  hb1_st2(J.o0[it] + o, hb_mulmod(a0.x, b0.x, P), hb_mulmod(a0.y, b0.y, P));
  hb1_st2(J.o1[it] + o, hb_reduce128(hx, lx, P), hb_reduce128(hy, ly, P));
  hb1_st2(J.o2[it] + o, hb_mulmod(a1.x, b1.x, P), hb_mulmod(a1.y, b1.y, P));
}

// ------------------------------------------------------------------------------------------
// innerProduct (src/Ctxt.cpp:2878-2893) before its one reLinearize: the tensor products of the pairs of every item, summed,
//   o0 (+)= sum_j a0_j*b0_j,   o1 (+)= sum_j (a0_j*b1_j + a1_j*b0_j),   o2 (+)= sum_j a1_j*b1_j   (mod q)
// in k1_tensor's streaming form (two adjacent coefficients per thread, 128-bit loads and stores), with the six 128-bit sums in
// registers and each output written once.  Inputs may be lazy below 8q + 2^32 (the lazy scale-down); every word is reduced to
// [0, q) on load, so each product is at most (q-1)^2 < 2^120 (q < 2^60) and 255 products plus one 64-bit value fit 128 bits:
// o1 takes two products per pair, so every HB_TSUM_GROUP = 127 pairs the sums are reduced and carried on canonical.  The old
// outputs (accumulate) may be any 64-bit values; the outputs are canonical.  a and b may alias (sums of squares); the
// outputs alias no input.  Pair j of item t of the launch reads slot t*npairs + j.     grid = (N / 512, nrows, nitems)
#define HB_TSUM_GROUP 127       // pairs per 128-bit accumulation
#define HB_TSUM_SLOTS 128       // pair slots (pairs x items) per launch
struct Hb1TensorSumJob {
  u64 N;
  HbRows rows;
  int npairs, nitems, accumulate;
  const u64* a0[HB_TSUM_SLOTS]; const u64* a1[HB_TSUM_SLOTS]; const u64* b0[HB_TSUM_SLOTS]; const u64* b1[HB_TSUM_SLOTS];
  u64* o0[HB_MAXB]; u64* o1[HB_MAXB]; u64* o2[HB_MAXB];
};
__device__ __forceinline__ u64 hb1_canon(u64 x, const HbPrimeDev& P) {   // any x < 2^64 -> [0, q)
  u64 r = x - __umul64hi(x, P.one_s) * P.q;   // [0, 2q)
  return r >= P.q ? r - P.q : r;
}
__global__ void __launch_bounds__(256) k1_tensor_sum(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1TensorSumJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const int it = blockIdx.z;
  const size_t o = (size_t)pi * (size_t)J.N + 2 * ((size_t)blockIdx.x * 256 + threadIdx.x);
  u64 h0x = 0, l0x = 0, h0y = 0, l0y = 0, h1x = 0, l1x = 0, h1y = 0, l1y = 0, h2x = 0, l2x = 0, h2y = 0, l2y = 0;
  if (J.accumulate) {
    const ulonglong2 p0 = hb1_ld2(J.o0[it] + o), p1 = hb1_ld2(J.o1[it] + o), p2 = hb1_ld2(J.o2[it] + o);
    l0x = p0.x; l0y = p0.y; l1x = p1.x; l1y = p1.y; l2x = p2.x; l2y = p2.y;
  }
  const int s0 = it * J.npairs;
  for (int j0 = 0; j0 < J.npairs; j0 += HB_TSUM_GROUP) {
    if (j0 > 0) {   // carry the group's sums on canonical
      l0x = hb_reduce128(h0x, l0x, P); l0y = hb_reduce128(h0y, l0y, P); l1x = hb_reduce128(h1x, l1x, P);
      l1y = hb_reduce128(h1y, l1y, P); l2x = hb_reduce128(h2x, l2x, P); l2y = hb_reduce128(h2y, l2y, P);
      h0x = h0y = h1x = h1y = h2x = h2y = 0;
    }
    const int j1 = J.npairs - j0 < HB_TSUM_GROUP ? J.npairs : j0 + HB_TSUM_GROUP;
    for (int j = j0; j < j1; j++) {
      const int s = s0 + j;
      const ulonglong2 A0 = hb1_ld2(J.a0[s] + o), A1 = hb1_ld2(J.a1[s] + o), B0 = hb1_ld2(J.b0[s] + o), B1 = hb1_ld2(J.b1[s] + o);
      const u64 a0x = hb1_canon(A0.x, P), a0y = hb1_canon(A0.y, P), a1x = hb1_canon(A1.x, P), a1y = hb1_canon(A1.y, P);
      const u64 b0x = hb1_canon(B0.x, P), b0y = hb1_canon(B0.y, P), b1x = hb1_canon(B1.x, P), b1y = hb1_canon(B1.y, P);
      hb1_mac128(h0x, l0x, a0x, b0x); hb1_mac128(h0y, l0y, a0y, b0y);
      hb1_mac128(h1x, l1x, a0x, b1x); hb1_mac128(h1x, l1x, a1x, b0x);
      hb1_mac128(h1y, l1y, a0y, b1y); hb1_mac128(h1y, l1y, a1y, b0y);
      hb1_mac128(h2x, l2x, a1x, b1x); hb1_mac128(h2y, l2y, a1y, b1y);
    }
  }
  hb1_st2(J.o0[it] + o, hb_reduce128(h0x, l0x, P), hb_reduce128(h0y, l0y, P));
  hb1_st2(J.o1[it] + o, hb_reduce128(h1x, l1x, P), hb_reduce128(h1y, l1y, P));
  hb1_st2(J.o2[it] + o, hb_reduce128(h2x, l2x, P), hb_reduce128(h2y, l2y, P));
}

// ------------------------------------------------------------------------------------------
// Scaled sums of two-part ciphertexts (polyEval's simplePolyEval leaves, src/polyEval.cpp:223-255, as one linear pass):
//   out_k[t][j] (+)= sum_i scal[j][i][r] * in_k[t][i]  (+ cst[j][r] on part 0)   (mod q_r, k = 0, 1)
// on every row r of a set U.  The scalars and constants are canonical residues mod q_r, shared by the items; a zero scalar
// means the input row is not read (an input over a smaller prime set contributes nothing there).  The job's tables live in
// context-owned device memory: scal[(j*nin + i)*nU + r], cst[j*nU + r] (or null), the inputs of item t at in0/in1[t*nin + i]
// and its outputs at out0/out1[t*nout + j].  One thread per coefficient: it reduces the words of every input that some
// output reads on this row to [0, q) (any 64-bit word is accepted) and keeps them in shared memory (ni inputs x 2 parts x
// blockDim words), then forms every output from them, so each input row is read once and each output row written once.
// Each product is below 2^120, so the 128-bit sums carry on canonical every HB_TSUM_GROUP inputs; old outputs (accumulate)
// may be any 64-bit values and the outputs are canonical.  Inputs [i0, i0 + ni) of the job take part in this launch.
// grid = (ceil(N / blockDim), rows of the launch, items of the launch)
#define HB_SSUM_SMEM (96 * 1024)                   // dynamic shared memory of k1_scaled_sums at most
#define HB_SSUM_MAXIN (HB_SSUM_SMEM / (16 * 32 + 1))  // inputs one launch stages (32 threads): later groups accumulate
struct Hb1ScaledSumsJob {
  u64 N;
  HbRows rows;        // prime indices of the launch's rows
  int r0;             // position of rows.prime[0] in U
  int nU, nin, nout, i0, ni, item0, accumulate, with_cst;
  const u64* scal; const u64* cst;
  const u64* const* in0; const u64* const* in1;
  u64* const* out0; u64* const* out1;
};
__global__ void __launch_bounds__(256) k1_scaled_sums(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT Hb1ScaledSumsJob J) {
  HB_SMEM_DECL
  u64* X = HB_SMEM;                                     // [ni][2][blockDim]
  unsigned char* used = (unsigned char*)(X + (size_t)J.ni * 2 * blockDim.x);   // [ni]
  const int pi = J.rows.prime[blockIdx.y];
  const int r = J.r0 + blockIdx.y;
  const HbPrimeDev P = primes[pi];
  const int it = J.item0 + blockIdx.z;
  const int T = blockDim.x, tid = threadIdx.x;
  for (int i = tid; i < J.ni; i += T) {   // does any output read input i on this row?
    unsigned char u = 0;
    for (int j = 0; j < J.nout && !u; j++) u = __ldg(J.scal + ((size_t)j * J.nin + J.i0 + i) * J.nU + r) != 0;
    used[i] = u;
  }
  __syncthreads();
  const size_t c = (size_t)blockIdx.x * T + tid;
  if (c >= J.N) return;
  const size_t o = (size_t)pi * J.N + c;
  for (int i = 0; i < J.ni; i++) {
    u64 a = 0, b = 0;
    if (used[i]) {
      const size_t s = (size_t)it * J.nin + J.i0 + i;
      a = hb1_canon(J.in0[s][o], P); b = hb1_canon(J.in1[s][o], P);
    }
    X[(size_t)(2 * i) * T + tid] = a; X[(size_t)(2 * i + 1) * T + tid] = b;
  }
  for (int j = 0; j < J.nout; j++) {
    u64 h0 = 0, l0 = 0, h1 = 0, l1 = 0;
    u64* const d0 = J.out0[(size_t)it * J.nout + j] + o;
    u64* const d1 = J.out1[(size_t)it * J.nout + j] + o;
    if (J.accumulate) { l0 = *d0; l1 = *d1; }
    if (J.with_cst) { const u64 k = __ldg(J.cst + (size_t)j * J.nU + r); l0 += k; h0 += l0 < k; }
    const u64* sc = J.scal + ((size_t)j * J.nin + J.i0) * J.nU + r;
    for (int g0 = 0; g0 < J.ni; g0 += HB_TSUM_GROUP) {
      if (g0 > 0) { l0 = hb_reduce128(h0, l0, P); l1 = hb_reduce128(h1, l1, P); h0 = h1 = 0; }   // carry on canonical
      const int g1 = J.ni - g0 < HB_TSUM_GROUP ? J.ni : g0 + HB_TSUM_GROUP;
      for (int i = g0; i < g1; i++) {
        const u64 s = __ldg(sc + (size_t)i * J.nU);
        if (s == 0) continue;
        hb1_mac128(h0, l0, s, X[(size_t)(2 * i) * T + tid]);
        hb1_mac128(h1, l1, s, X[(size_t)(2 * i + 1) * T + tid]);
      }
    }
    *d0 = hb_reduce128(h0, l0, P);
    *d1 = hb_reduce128(h1, l1, P);
  }
}

