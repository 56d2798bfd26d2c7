// hb_device.cuh -- sm_90a device code of the H100 DoubleCRT engine.
//
// Data model (DESIGN.md section 3): a DoubleCRT is a dense matrix u64[nprimes][N] in HBM; the
// row of chain prime i lives at base + i*N and holds canonical residues in [0,q_i) in HElib's
// natural evaluation order row[j] = f(psi^(2j+1)) (reference: src/CModulus.cpp:392-426).
//
// The length-N negacyclic transform is split N = N1 x BLK (BLK = 2^log_blk, 256 for N >= 2^11):
//   forward :  "cols" phase  (first n1 = logN-log_blk Cooley-Tukey stages, stride-BLK columns)
//              "blk"  phase  (last log_blk stages inside contiguous BLK-blocks + un-bit-reversal)
//   inverse :  "blk" phase (bit-reversal + first log_blk Gentleman-Sande stages), "cols" phase.
// The coefficient side of both directions is the "cols" layout, so the exact base conversion
// (iNTT-cols -> CRT -> NTT-cols) is fused in one kernel (k_conv) that never leaves shared memory.
#pragma once

#ifdef HB_SIM
#include "cusim.h"
#define HB_SMEM_DECL
#define HB_SMEM ((u64*)cusim::smem_)
#define HB_NOINLINE __attribute__((noinline))
#define HB_GRID_CONSTANT
#else
#define HB_GRID_CONSTANT __grid_constant__   // job descriptors are read straight from the constant bank (no local copy)
#define HB_NOINLINE __noinline__
#include <cuda_runtime.h>
#define HB_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define HB_SMEM_DECL extern __shared__ unsigned long long hb_smem_[];
#define HB_SMEM hb_smem_
#endif

#include <stdint.h>

typedef unsigned long long u64;
typedef long long i64;

#define HB_MAXROWS 64   // rows per launch (larger sets are chunked by the host)
#ifndef HB_MAXB
#define HB_MAXB 64      // batch items per launch (job descriptors above 4 KB rely on the 32 KB kernel-parameter space of CUDA 12.1+)
#endif
#define HB_MAXDIG 8     // digits per key-switching matrix
#define HB_THREADS 256

// ------------------------------------------------------------------------------------------
// per-prime device table
struct HbPrimeDev {
  u64 q;
  u64 ninv, ninv_s;        // N^-1 mod q (+ Shoup companion floor(w*2^64/q))
  u64 c64, c64_s;          // 2^64 mod q (+ Shoup)
  u64 one_s;               // floor(2^64 / q)
  u64 nq, qb;              // 2^64 - q and 4q (the lazy bound B of the register kernels), kept as opaque table values so ptxas does not re-derive them from q
  unsigned qt, qsh;        // HElib primes are q = qt*2^s + 1 with s >= 32 (PrimeGenerator picks k maximal,
                           // src/PrimeGenerator.h:54-124): qsh = s-32, qt = (q-1)>>s.  qt = 0 if s < 32 or qt >= 2^32.
  const ulonglong2* fw;    // fw[k] = (psi^brev(k), shoup), k = 1..N-1   (Cooley-Tukey, merged twist)
  const ulonglong2* iw;    // iw[k] = (psi^-brev(k), shoup)              (Gentleman-Sande)
};

// ------------------------------------------------------------------------------------------
// modular arithmetic.  All moduli < 2^62.

__device__ __forceinline__ u64 hb_addmod(u64 a, u64 b, u64 q) { u64 s = a + b; return s >= q ? s - q : s; }
__device__ __forceinline__ u64 hb_submod(u64 a, u64 b, u64 q) { return a >= b ? a - b : a + q - b; }

// a*w mod q with ws = floor(w*2^64/q); a may be ANY 64-bit value, w < q.  Result in [0,2q).
__device__ __forceinline__ u64 hb_mul_shoup_lazy(u64 a, u64 w, u64 ws, u64 q) {
  u64 hi = __umul64hi(a, ws);
  return a * w - hi * q;
}
__device__ __forceinline__ u64 hb_mul_shoup(u64 a, u64 w, u64 ws, u64 q) {
  u64 r = hb_mul_shoup_lazy(a, w, ws, q);
  return r >= q ? r - q : r;
}
// (hi,lo) += a*b
__device__ __forceinline__ void hb_mac128(u64& hi, u64& lo, u64 a, u64 b) {
  u64 pl = a * b, ph = __umul64hi(a, b);
  lo += pl;
  hi += ph + (lo < pl ? 1ULL : 0ULL);
}
// (hi*2^64 + lo) mod q, canonical.  Any hi, lo.
__device__ __forceinline__ u64 hb_reduce128(u64 hi, u64 lo, u64 q, u64 c64, u64 c64_s, u64 one_s) {
  u64 r1 = hb_mul_shoup_lazy(hi, c64, c64_s, q);          // hi*2^64 mod q, in [0,2q)
  u64 r2 = lo - __umul64hi(lo, one_s) * q;                // lo mod q, in [0,2q)
  u64 r = r1 + r2;                                        // < 4q < 2^64
  u64 q2 = q + q;
  if (r >= q2) r -= q2;
  if (r >= q) r -= q;
  return r;
}
// same, but only reduced to [0,4q) (input of a lazy butterfly network)
__device__ __forceinline__ u64 hb_reduce128_lazy(u64 hi, u64 lo, const HbPrimeDev& P) {
  return hb_mul_shoup_lazy(hi, P.c64, P.c64_s, P.q) + (lo - __umul64hi(lo, P.one_s) * P.q);
}
__device__ __forceinline__ u64 hb_reduce128(u64 hi, u64 lo, const HbPrimeDev& P) {
  return hb_reduce128(hi, lo, P.q, P.c64, P.c64_s, P.one_s);
}
__device__ __forceinline__ u64 hb_mulmod(u64 a, u64 b, const HbPrimeDev& P) {
  return hb_reduce128(__umul64hi(a, b), a * b, P);
}
__device__ __forceinline__ unsigned hb_brev(unsigned x, int bits) {
  unsigned r = 0;
  for (int i = 0; i < bits; i++) { r = (r << 1) | (x & 1u); x >>= 1; }
  return r;
}

// ------------------------------------------------------------------------------------------
// shared-memory tile transforms (v0: radix-2 stages, CTA-wide barriers, canonical values)

// "cols" tile: T[i1*w + c], i1 in [0,2^n1), c in [0,w) (w = 2^logw).  First n1 CT stages.
__device__ __forceinline__ void hb_tile_fwd_cols(u64* T, int n1, int logw, const ulonglong2* fw, u64 q) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int half = (1 << n1) >> 1;
  const int cnt = half << logw;
  for (int s = 0; s < n1; s++) {
    const int logt = n1 - 1 - s;  // t = N1 >> (s+1)
    const int m = 1 << s;
    for (int e = tid; e < cnt; e += nthr) {
      int c = e & ((1 << logw) - 1);
      int bf = e >> logw;
      int i = bf >> logt, o = bf & ((1 << logt) - 1);
      int j = (i << (logt + 1)) + o;
      ulonglong2 tw = fw[m + i];
      u64* pa = T + ((size_t)j << logw) + c;
      u64* pb = T + ((size_t)(j + (1 << logt)) << logw) + c;
      u64 U = *pa, V = hb_mul_shoup(*pb, tw.x, tw.y, q);
      *pa = hb_addmod(U, V, q);
      *pb = hb_submod(U, V, q);
    }
    __syncthreads();
  }
}
// inverse: last n1 GS stages (t = 1 .. N1/2 in units of rows); caller applies N^-1.
__device__ __forceinline__ void hb_tile_inv_cols(u64* T, int n1, int logw, const ulonglong2* iw, u64 q) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int half = (1 << n1) >> 1;
  const int cnt = half << logw;
  for (int s = n1 - 1; s >= 0; s--) {
    const int logt = n1 - 1 - s;
    const int h = 1 << s;
    for (int e = tid; e < cnt; e += nthr) {
      int c = e & ((1 << logw) - 1);
      int bf = e >> logw;
      int i = bf >> logt, o = bf & ((1 << logt) - 1);
      int j = (i << (logt + 1)) + o;
      ulonglong2 tw = iw[h + i];
      u64* pa = T + ((size_t)j << logw) + c;
      u64* pb = T + ((size_t)(j + (1 << logt)) << logw) + c;
      u64 U = *pa, V = *pb;
      *pa = hb_addmod(U, V, q);
      *pb = hb_mul_shoup(hb_submod(U, V, q), tw.x, tw.y, q);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// job descriptors (passed by value as kernel parameters; < 4 KB each)

struct HbRows {
  int n;
  int prime[HB_MAXROWS];
};

struct HbBlkJob {
  int logN, log_blk, logwb;          // wb = 2^logwb blocks per CTA
  int epi;                           // forward only: 0 = store, 1 = dst = (dst - res) * scal[row]
  HbRows rows;
  u64 scal[HB_MAXROWS], scal_s[HB_MAXROWS];
  int nitems;
  const u64* src[HB_MAXB];
  u64* dst[HB_MAXB];
};

struct HbColsJob {
  int logN, log_blk, logw;           // w = 2^logw columns per CTA
  HbRows rows;
  int nitems;
  const u64* src[HB_MAXB];
  u64* dst[HB_MAXB];
};

// Exact base conversion tables for (source set D -> target set T [, plaintext modulus p]).
struct HbConvDev {
  int n, nt, L, has_p;
  const int* src_prime;   // [n]
  const u64* tn;          // [n]  (Q/q_j)^-1 * N^-1 mod q_j      (N^-1 of the inverse transform folded in)
  const u64* tn_s;        // [n]  Shoup companion
  const u64* fmul;        // [n]  floor(2^(63+b_j)/q_j), b_j = bitlen(q_j)
  const int* fshift;      // [n]  b_j - 1
  const int* tgt_prime;   // [nt]
  const u64* c;           // [nt][n]  (Q/q_j) mod q_t
  const u64* negQ;        // [nt]  (-Q) mod q_t
  const u64* Qmod;        // [nt]  Q mod q_t
  u64 p, p_c64, p_c64_s, p_one_s;  // plaintext modulus (has_p) as a pseudo-prime for hb_reduce128
  u64 Qinv_p, Qinv_p_s;   // Q^-1 mod p (+Shoup wrt p)
  u64 negQ_p;             // (-Q) mod p
  const u64* cp;          // [n]  (Q/q_j) mod p
  const u64* Q;           // [L]   limbs of Q
  const u64* Qhalf;       // [L]   limbs of (Q-1)/2
  const u64* Qj;          // [n][L] limbs of Q/q_j
};

struct HbConvJob {
  const HbConvDev* cv;
  int logN, log_blk, logw;
  int nitems;
  const u64* src[HB_MAXB];   // "blk"-phase output of the inverse transform (rows src_prime)
  u64* dst[HB_MAXB];         // "cols"-phase output of the forward transform (rows tgt_prime)
  u64* stats;                // [0] += number of exact-fallback evaluations
  int src_is_y;              // 1: src rows already hold y_j = coeff * (Q/q_j)^-1 mod q_j in coefficient order
  double* frac[HB_MAXB];     // optional: x/Q per coefficient (natural coefficient order) for the embedding norm
};

struct HbCrtJob {            // DoubleCRT::toPoly: exact balanced integer per coefficient
  const HbConvDev* cv;
  int N, Lout, positive;
  const u64* src;            // coefficient-form rows (after full inverse transform incl. N^-1 ... see k_crt)
  u64* out;                  // [N][Lout] two's complement limbs
  u64 factor, factor_s;      // k_crt_modp: result multiplier mod p (+Shoup wrt p)
  u64* stats;                // k_crt_modp: [0] += number of exact-fallback evaluations
};

enum {
  HB_PW_ADD = 0, HB_PW_SUB, HB_PW_MUL, HB_PW_NEG, HB_PW_SCALE, HB_PW_SUBSCALE, HB_PW_ZERO, HB_PW_COPY,
  HB_PW_TENSOR, HB_PW_AUTOMORPH, HB_PW_MULADD
};

struct HbPwJob {
  int op, logN;
  u64 N;                    // row length = row stride (phi(m); not a power of two for general m)
  HbRows rows;
  u64 scal[HB_MAXROWS], scal_s[HB_MAXROWS];
  int nitems;
  u64* dst[HB_MAXB];
  u64* dst1[HB_MAXB];
  u64* dst2[HB_MAXB];
  const u64* a[HB_MAXB];
  const u64* b[HB_MAXB];
  const u64* c[HB_MAXB];
  const u64* d[HB_MAXB];
  u64 k, m;                 // automorphism
};

struct HbKsJob {            // Ctxt::keySwitchDigits inner product
  int logN, ndig;
  u64 N;
  HbRows rows;
  int nitems;
  const u64* dig[HB_MAXB][HB_MAXDIG];
  const u64* evk_a[HB_MAXDIG];
  const u64* evk_b[HB_MAXDIG];
  u64* out0[HB_MAXB];
  u64* out1[HB_MAXB];
  int mode;                 // 0: out += sum;  1: out = scal[row]*out + sum (scal 0 => out = sum, old value not read):
  u64 scal[HB_MAXROWS];     //    folds the addPrimesAndScale of the (1, s) parts (src/Ctxt.cpp:764-768) into the inner product
  // mode 2: hoisted automorphism (BasicAutomorphPrecon::automorph, src/matmul.cpp:112-184): the digits and the
  // constant part are read through sigma_k (new[j] = old[idx(rep(j)*k mod m)], src/DoubleCRT.cpp:1160-1202):
  //   out0 = scal*sigma_k(c0) + sum_i sigma_k(D_i)*b_i ,  out1 = sum_i sigma_k(D_i)*a_i       (power-of-two m)
  u64 ak, am;
  const u64* c0[HB_MAXB];
  // fused breakIntoDigits: the rows of digit i's own primes live in own[item] (the part being switched, updated in place
  // by the mixed-radix steps) instead of dig[item][i];  own_dig[row] = that digit, or -1
  const u64* own[HB_MAXB];
  signed char own_dig[HB_MAXROWS];
};

// ------------------------------------------------------------------------------------------
// kernels

// Forward "blk" phase (last log_blk CT stages inside BLK-blocks) + natural-order store.
// Replaces the tail of Cmodulus::FFT_aux incl. BitReverseCopy (src/CModulus.cpp:408-426).
// grid = (N1 >> logwb, nrows, nitems)
__global__ void __launch_bounds__(HB_THREADS) k_fwd_blk(const HbPrimeDev* __restrict__ primes, HbBlkJob J) {
  HB_SMEM_DECL
  u64* T = HB_SMEM;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int n1 = J.logN - J.log_blk, lb = J.log_blk;
  const int BLK = 1 << lb, RS = BLK + 1, wb = 1 << J.logwb;
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const u64 q = P.q;
  const size_t rowoff = (size_t)pi << J.logN;
  const u64* src = J.src[blockIdx.z] + rowoff;
  u64* dst = J.dst[blockIdx.z] + rowoff;
  const unsigned u0 = blockIdx.x << J.logwb;

  for (int e = tid; e < (wb << lb); e += nthr) {
    int ub = e >> lb, c = e & (BLK - 1);
    unsigned b = hb_brev(u0 + ub, n1);
    T[ub * RS + c] = src[((size_t)b << lb) + c];
  }
  __syncthreads();
  for (int s = 0; s < lb; s++) {
    const int logt = lb - 1 - s;
    for (int e = tid; e < (wb << (lb - 1)); e += nthr) {
      int ub = e >> (lb - 1), bf = e & ((BLK >> 1) - 1);
      int i = bf >> logt, o = bf & ((1 << logt) - 1);
      int j = (i << (logt + 1)) + o;
      unsigned b = hb_brev(u0 + ub, n1);
      ulonglong2 tw = P.fw[((size_t)1 << (n1 + s)) + ((size_t)b << s) + i];
      u64* pa = T + ub * RS + j;
      u64* pb = pa + (1 << logt);
      u64 U = *pa, V = hb_mul_shoup(*pb, tw.x, tw.y, q);
      *pa = hb_addmod(U, V, q);
      *pb = hb_submod(U, V, q);
    }
    __syncthreads();
  }
  const u64 sc = J.scal[blockIdx.y], sc_s = J.scal_s[blockIdx.y];
  for (int e = tid; e < (wb << lb); e += nthr) {
    int v = e >> J.logwb, ub = e & (wb - 1);
    unsigned c = hb_brev(v, lb);
    u64 val = T[ub * RS + c];
    size_t o = ((size_t)v << n1) + u0 + ub;
    if (J.epi == 1) val = hb_mul_shoup(hb_submod(dst[o], val, q), sc, sc_s, q);
    dst[o] = val;
  }
}

// Inverse "blk" phase: bit-reversal load + first log_blk GS stages.
// Replaces BitReverseCopy + head of NTL::FFTRev1 in Cmodulus::iFFT (src/CModulus.cpp:510-535).
__global__ void __launch_bounds__(HB_THREADS) k_inv_blk(const HbPrimeDev* __restrict__ primes, HbBlkJob J) {
  HB_SMEM_DECL
  u64* T = HB_SMEM;
  const int tid = threadIdx.x, nthr = blockDim.x;
  const int n1 = J.logN - J.log_blk, lb = J.log_blk;
  const int BLK = 1 << lb, RS = BLK + 1, wb = 1 << J.logwb;
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const u64 q = P.q;
  const size_t rowoff = (size_t)pi << J.logN;
  const u64* src = J.src[blockIdx.z] + rowoff;
  u64* dst = J.dst[blockIdx.z] + rowoff;
  const unsigned u0 = blockIdx.x << J.logwb;

  for (int e = tid; e < (wb << lb); e += nthr) {
    int v = e >> J.logwb, ub = e & (wb - 1);
    unsigned c = hb_brev(v, lb);
    T[ub * RS + c] = src[((size_t)v << n1) + u0 + ub];
  }
  __syncthreads();
  for (int s = lb - 1; s >= 0; s--) {
    const int logt = lb - 1 - s;
    for (int e = tid; e < (wb << (lb - 1)); e += nthr) {
      int ub = e >> (lb - 1), bf = e & ((BLK >> 1) - 1);
      int i = bf >> logt, o = bf & ((1 << logt) - 1);
      int j = (i << (logt + 1)) + o;
      unsigned b = hb_brev(u0 + ub, n1);
      ulonglong2 tw = P.iw[((size_t)1 << (n1 + s)) + ((size_t)b << s) + i];
      u64* pa = T + ub * RS + j;
      u64* pb = pa + (1 << logt);
      u64 U = *pa, V = *pb;
      *pa = hb_addmod(U, V, q);
      *pb = hb_mul_shoup(hb_submod(U, V, q), tw.x, tw.y, q);
    }
    __syncthreads();
  }
  for (int e = tid; e < (wb << lb); e += nthr) {
    int ub = e >> lb, c = e & (BLK - 1);
    unsigned b = hb_brev(u0 + ub, n1);
    dst[((size_t)b << lb) + c] = T[ub * RS + c];
  }
}

__device__ __forceinline__ void hb_cols_load(u64* T, const u64* src, int n1, int lb, int logw, unsigned c0) {
  const int cnt = 1 << (n1 + logw);
  for (int e = threadIdx.x; e < cnt; e += blockDim.x) {
    int i1 = e >> logw, c = e & ((1 << logw) - 1);
    T[e] = src[((size_t)i1 << lb) + c0 + c];
  }
}
__device__ __forceinline__ void hb_cols_store(const u64* T, u64* dst, int n1, int lb, int logw, unsigned c0) {
  const int cnt = 1 << (n1 + logw);
  for (int e = threadIdx.x; e < cnt; e += blockDim.x) {
    int i1 = e >> logw, c = e & ((1 << logw) - 1);
    dst[((size_t)i1 << lb) + c0 + c] = T[e];
  }
}

// Forward "cols" phase alone (coefficients -> intermediate).  grid = (BLK >> logw, nrows, nitems)
// Head of Cmodulus::FFT_aux: the psi^i twist (src/CModulus.cpp:392-397) is merged into the twiddles.
__global__ void __launch_bounds__(HB_THREADS) k_fwd_cols(const HbPrimeDev* __restrict__ primes, HbColsJob J) {
  HB_SMEM_DECL
  u64* T = HB_SMEM;
  const int n1 = J.logN - J.log_blk;
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t rowoff = (size_t)pi << J.logN;
  const unsigned c0 = blockIdx.x << J.logw;
  hb_cols_load(T, J.src[blockIdx.z] + rowoff, n1, J.log_blk, J.logw, c0);
  __syncthreads();
  hb_tile_fwd_cols(T, n1, J.logw, P.fw, P.q);
  hb_cols_store(T, J.dst[blockIdx.z] + rowoff, n1, J.log_blk, J.logw, c0);
}

// Inverse "cols" phase alone (intermediate -> coefficients in [0,q), incl. N^-1 and psi^-i,
// src/CModulus.cpp:533-546).
__global__ void __launch_bounds__(HB_THREADS) k_inv_cols(const HbPrimeDev* __restrict__ primes, HbColsJob J) {
  HB_SMEM_DECL
  u64* T = HB_SMEM;
  const int n1 = J.logN - J.log_blk;
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t rowoff = (size_t)pi << J.logN;
  const unsigned c0 = blockIdx.x << J.logw;
  hb_cols_load(T, J.src[blockIdx.z] + rowoff, n1, J.log_blk, J.logw, c0);
  __syncthreads();
  hb_tile_inv_cols(T, n1, J.logw, P.iw, P.q);
  const int cnt = 1 << (n1 + J.logw);
  for (int e = threadIdx.x; e < cnt; e += blockDim.x) T[e] = hb_mul_shoup(T[e], P.ninv, P.ninv_s, P.q);
  __syncthreads();
  hb_cols_store(T, J.dst[blockIdx.z] + rowoff, n1, J.log_blk, J.logw, c0);
}

// ---- exact CRT pieces -------------------------------------------------------------------

#define HB_MAXL 66

// Exact balanced reconstruction of one coefficient (the multi-precision part of DoubleCRT::toPoly,
// src/DoubleCRT.cpp:1076-1100).  y[j*ystride] = r_j * (Q/q_j)^-1 mod q_j.  Returns v with
// x = sum_j y_j*(Q/q_j) - v*Q in [-(Q-1)/2,(Q-1)/2]; *sign = sign(x); optionally writes x.
__device__ HB_NOINLINE int hb_crt_exact(const HbConvDev* cv, const u64* y, int ystride, int* sign, u64* xout, int Lout, int positive) {
  const int n = cv->n, L = cv->L;  // L limbs hold Q; X needs L+1
  u64 X[HB_MAXL + 1];
  for (int l = 0; l <= L; l++) X[l] = 0;
  for (int j = 0; j < n; j++) {
    const u64 yj = y[(size_t)j * ystride];
    const u64* Qj = cv->Qj + (size_t)j * L;
    u64 carry = 0;
    for (int l = 0; l < L; l++) {
      u64 lo = yj * Qj[l], hi = __umul64hi(yj, Qj[l]);
      u64 s = X[l] + lo; u64 c1 = s < lo;
      u64 s2 = s + carry; u64 c2 = s2 < carry;
      X[l] = s2; carry = hi + c1 + c2;
    }
    X[L] += carry;
  }
  // X >= 0.  Subtract Q while X > (positive ? Q-1 : Qhalf).
  int v = 0;
  for (;;) {
    // compare X (L+1 limbs, signed) with bound (L limbs, non-negative)
    bool neg = (X[L] >> 63) != 0;
    int cmp = 0;  // sign of X - bound
    if (neg) cmp = -1;
    else if (X[L] != 0) cmp = 1;
    else {
      for (int l = L - 1; l >= 0; l--) {
        u64 bl = positive ? cv->Q[l] : cv->Qhalf[l];
        if (X[l] != bl) { cmp = X[l] < bl ? -1 : 1; break; }
      }
      if (positive && cmp == 0) cmp = 1;  // X == Q  -> subtract
    }
    if (cmp <= 0) break;
    u64 borrow = 0;
    for (int l = 0; l < L; l++) {
      u64 a = X[l], b = cv->Q[l];
      u64 d = a - b; u64 b1 = a < b;
      u64 d2 = d - borrow; u64 b2 = d < borrow;
      X[l] = d2; borrow = b1 + b2;
    }
    X[L] -= borrow;
    v++;
  }
  bool neg = (X[L] >> 63) != 0;
  bool zero = true;
  for (int l = 0; l <= L; l++) if (X[l]) zero = false;
  *sign = neg ? -1 : (zero ? 0 : 1);
  if (xout) {
    u64 ext = neg ? ~0ULL : 0ULL;
    for (int l = 0; l < Lout; l++) xout[l] = l <= L ? X[l] : ext;
  }
  return v;
}

// v = round(sum_j y_j/q_j) via 0.64 fixed point; exact fallback when within the error margin of
// the rounding boundary.  With has_p: also the BGV correction of DoubleCRT::scaleDownToSet
// (src/DoubleCRT.cpp:1485-1511) folded into the returned multiple of Q.
__device__ __forceinline__ i64 hb_conv_v(const HbConvDev* cv, const u64* y, int ystride, u64* stats, double* frac = nullptr, bool bgv = true) {
  const int n = cv->n;
  u64 shi = 0, slo = 0;
  for (int j = 0; j < n; j++) {
    const u64 yj = y[(size_t)j * ystride];
    u64 m = cv->fmul[j];
    int sh = cv->fshift[j];
    u64 lo = yj * m, hi = __umul64hi(yj, m);
    u64 f = sh == 0 ? lo : ((lo >> sh) | (hi << (64 - sh)));  // y*M < 2^(63+b) => f < 2^64
    slo += f;
    shi += (slo < f) ? 1ULL : 0ULL;
  }
  u64 F = slo + 0x8000000000000000ULL;
  i64 v = (i64)(shi + (F < slo ? 1ULL : 0ULL));
  const u64 margin = 4ULL * (u64)n;
  int sign = 2;  // unknown
  if (F >= 0 - margin) {  // could round up once the truncation error is added back: decide exactly
    const i64 ve = hb_crt_exact(cv, y, ystride, &sign, nullptr, 0, 0);
    if (ve != v) F = 0;   // rounded up: x/Q is -1/2 (within the margin), not the +1/2 the truncated F reads
    v = ve;
    if (stats) atomicAdd(stats, 1ULL);
  }
  if (bgv && cv->has_p) {
    const u64 p = cv->p;
    u64 hi = 0, lo = 0;
    for (int j = 0; j < n; j++) hb_mac128(hi, lo, y[(size_t)j * ystride], cv->cp[j]);
    hb_mac128(hi, lo, (u64)v, cv->negQ_p);
    u64 u = hb_reduce128(hi, lo, p, cv->p_c64, cv->p_c64_s, cv->p_one_s);
    if (u != 0) {
      u = hb_mul_shoup(u, cv->Qinv_p, cv->Qinv_p_s, p);
      const u64 half = p >> 1;
      bool minus = u > half;
      if (!minus && (p & 1ULL) == 0 && u == half) {  // tie: needs sign(delta)
        if (sign == 2) {
          if (F >= 0x8000000000000000ULL) sign = 1;             // x > 0 (x != 0 because u != 0)
          else if (F < 0x8000000000000000ULL - margin) sign = -1;
          else { hb_crt_exact(cv, y, ystride, &sign, nullptr, 0, 0); if (stats) atomicAdd(stats, 1ULL); }
        }
        minus = sign < 0;
      }
      const i64 v2 = minus ? (i64)u - (i64)p : (i64)u;
      v += v2;
      if (frac) *frac = (double)(i64)(F ^ 0x8000000000000000ULL) * 5.421010862427522e-20 - (double)v2;  // delta'/P
      return v;
    }
  }
  // x / Q in (-1/2, 1/2): the 0.64 fixed-point fraction re-centred (FP64 noise metadata, src/norms.cpp:443-485)
  if (frac) *frac = (double)(i64)(F ^ 0x8000000000000000ULL) * 5.421010862427522e-20;
  return v;
}

// Fused exact base conversion: inverse "cols" phase of the n source rows, exact CRT (balanced),
// optional BGV correction, reduction modulo each target prime, forward "cols" phase.
// Replaces toPoly + FFT inside DoubleCRT::addPrimes (src/DoubleCRT.cpp:565-599) and
// DoubleCRT::scaleDownToSet (src/DoubleCRT.cpp:1464-1516).
// grid = (BLK >> logw, nitems);  smem = (n + 2) * TILE u64, TILE = 2^(n1+logw)
__global__ void __launch_bounds__(HB_THREADS) k_conv(const HbPrimeDev* __restrict__ primes, HbConvJob J) {
  HB_SMEM_DECL
  const HbConvDev* cv = J.cv;
  const int n = cv->n, nt = cv->nt;
  const int n1 = J.logN - J.log_blk, lb = J.log_blk, logw = J.logw;
  const int TILE = 1 << (n1 + logw);
  u64* Y = HB_SMEM;                  // [n][TILE]
  i64* Vb = (i64*)(Y + (size_t)n * TILE);
  u64* W = (u64*)(Vb + TILE);
  const int tid = threadIdx.x, nthr = blockDim.x;
  const unsigned c0 = blockIdx.x << logw;
  const u64* src = J.src[blockIdx.y];
  u64* dst = J.dst[blockIdx.y];

  for (int j = 0; j < n; j++) {
    const int pi = cv->src_prime[j];
    const HbPrimeDev P = primes[pi];
    u64* T = Y + (size_t)j * TILE;
    hb_cols_load(T, src + ((size_t)pi << J.logN), n1, lb, logw, c0);
    __syncthreads();
    if (J.src_is_y) continue;   // prime-sharded path: y_j rows were produced (and all-gathered) beforehand
    hb_tile_inv_cols(T, n1, logw, P.iw, P.q);
    const u64 t = cv->tn[j], ts = cv->tn_s[j];
    for (int e = tid; e < TILE; e += nthr) T[e] = hb_mul_shoup(T[e], t, ts, P.q);
  }
  __syncthreads();
  double* fr = J.frac[blockIdx.y];
  for (int e = tid; e < TILE; e += nthr) {
    double f;
    Vb[e] = hb_conv_v(cv, Y + e, TILE, J.stats, fr ? &f : nullptr);
    if (fr) fr[((size_t)(e >> logw) << lb) + c0 + (e & ((1 << logw) - 1))] = f;
  }
  __syncthreads();
  for (int t = 0; t < nt; t++) {
    const int pi = cv->tgt_prime[t];
    const HbPrimeDev P = primes[pi];
    const u64* ct = cv->c + (size_t)t * n;
    const u64 nq = cv->negQ[t], pq = cv->Qmod[t];
    for (int e = tid; e < TILE; e += nthr) {
      u64 hi = 0, lo = 0;
      for (int j = 0; j < n; j++) hb_mac128(hi, lo, Y[(size_t)j * TILE + e], ct[j]);
      i64 v = Vb[e];
      if (v >= 0) hb_mac128(hi, lo, (u64)v, nq);
      else hb_mac128(hi, lo, (u64)(-v), pq);
      W[e] = hb_reduce128(hi, lo, P);
    }
    __syncthreads();
    hb_tile_fwd_cols(W, n1, logw, P.fw, P.q);
    hb_cols_store(W, dst + ((size_t)pi << J.logN), n1, lb, logw, c0);
    __syncthreads();
  }
}

// DoubleCRT::toPoly's CRT stage for all coefficients (src/DoubleCRT.cpp:1062-1102).
// src rows hold coefficients already multiplied by N^-1 (k_inv_cols); y_j = r_j * t_j here.
struct HbCrtTabs { const u64* t; const u64* t_s; };  // (Q/q_j)^-1 mod q_j (+Shoup), no N^-1
__global__ void __launch_bounds__(HB_THREADS) k_crt(const HbPrimeDev* __restrict__ primes, HbCrtJob J, HbCrtTabs tabs) {
  const HbConvDev* cv = J.cv;
  const int n = cv->n;
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (size_t)J.N) return;
  u64 y[HB_MAXROWS];
  for (int j = 0; j < n; j++) {
    int pi = cv->src_prime[j];
    u64 q = primes[pi].q;
    y[j] = hb_mul_shoup(J.src[(size_t)pi * J.N + k], tabs.t[j], tabs.t_s[j], q);
  }
  int sign;
  hb_crt_exact(cv, y, 1, &sign, J.out + k * J.Lout, J.Lout, J.positive);
}

// Tail of SecKey::Decrypt (src/keys.cpp:1381-1399): the balanced integer x = toPoly(ptxt) is never materialised;
// out[k] = factor * (x mod p) mod p in [0,p), from x = sum_j y_j*(Q/q_j) - v*Q with the exact v.
__global__ void __launch_bounds__(HB_THREADS) k_crt_modp(const HbPrimeDev* __restrict__ primes, HbCrtJob J, HbCrtTabs tabs) {
  const HbConvDev* cv = J.cv;
  const int n = cv->n;
  size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (size_t)J.N) return;
  u64 y[HB_MAXROWS];
  for (int j = 0; j < n; j++) {
    int pi = cv->src_prime[j];
    y[j] = hb_mul_shoup(J.src[(size_t)pi * J.N + k], tabs.t[j], tabs.t_s[j], primes[pi].q);
  }
  const i64 v = hb_conv_v(cv, y, 1, J.stats, nullptr, false);
  u64 hi = 0, lo = 0;
  for (int j = 0; j < n; j++) hb_mac128(hi, lo, y[j], cv->cp[j]);
  hb_mac128(hi, lo, (u64)v, cv->negQ_p);
  const u64 u = hb_reduce128(hi, lo, cv->p, cv->p_c64, cv->p_c64_s, cv->p_one_s);
  J.out[k] = hb_mul_shoup(u, J.factor, J.factor_s, cv->p);
}

// DoubleCRT(const zzX&/ZZX&, context, s) -> FFT(poly, s) (src/DoubleCRT.cpp:68-105): the per-prime reduction of the
// coefficients (src/CModulus.cpp:453-457, timer FFT_remainder) done on the device from ONE copy of the polynomial.
struct HbFromJob {
  u64 N; int L, nitems;
  HbRows rows;
  const u64* src[HB_MAXB];   // [N] signed 64-bit coefficients (L == 0) or [N][L] two's-complement limbs
  u64* dst[HB_MAXB];
};
__global__ void __launch_bounds__(HB_THREADS) k_from_coeffs(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbFromJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const u64 q = P.q;
  const size_t N = (size_t)J.N;
  const int it = blockIdx.z, L = J.L;
  u64 top = 0;                       // 2^(64 L) mod q: what a negative two's-complement value is short of
  if (L > 0) { top = 1; for (int l = 0; l < L; l++) top = hb_reduce128(top, 0, P); }
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < N; k += (size_t)gridDim.x * blockDim.x) {
    u64 r;
    if (L == 0) {
      const i64 c = (i64)J.src[it][k];
      const u64 a = c < 0 ? 0 - (u64)c : (u64)c;
      r = a - __umul64hi(a, P.one_s) * q;
      if (r >= q) r -= q;
      if (c < 0 && r) r = q - r;
    } else {
      const u64* x = J.src[it] + k * (size_t)L;
      r = 0;
      for (int l = L - 1; l >= 0; l--) r = hb_reduce128(r, x[l], P);
      if (x[L - 1] >> 63) r = hb_submod(r, top, q);
    }
    J.dst[it][(size_t)pi * N + k] = r;
  }
}

// Row-wise pointwise operations: DoubleCRT::Op<Add/Sub/Mul>, Negate, operator/=, Op(ZZ)
// (src/DoubleCRT.cpp:216-384,1122-1139), addPrimesAndScale's scaling (src/DoubleCRT.cpp:620-636),
// Ctxt::tensorProduct (src/Ctxt.cpp:1563-1608), DoubleCRT::automorph (src/DoubleCRT.cpp:1160-1202).
// grid = (N / (HB_THREADS*4) or 1, nrows, nitems)
__global__ void __launch_bounds__(HB_THREADS) k_pointwise(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbPwJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const u64 q = P.q;
  const size_t N = (size_t)J.N;
  const size_t off = (size_t)pi * N;
  const int it = blockIdx.z;
  const u64 sc = J.scal[blockIdx.y], sc_s = J.scal_s[blockIdx.y];
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < N; k += (size_t)gridDim.x * blockDim.x) {
    const size_t o = off + k;
    switch (J.op) {
      case HB_PW_ADD: J.dst[it][o] = hb_addmod(J.dst[it][o], J.a[it][o], q); break;
      case HB_PW_SUB: J.dst[it][o] = hb_submod(J.dst[it][o], J.a[it][o], q); break;
      case HB_PW_MUL: J.dst[it][o] = hb_mulmod(J.dst[it][o], J.a[it][o], P); break;
      case HB_PW_NEG: { u64 x = J.a[it][o]; J.dst[it][o] = x ? q - x : 0; } break;
      case HB_PW_SCALE: J.dst[it][o] = hb_mul_shoup(J.dst[it][o], sc, sc_s, q); break;
      case HB_PW_SUBSCALE: J.dst[it][o] = hb_mul_shoup(hb_submod(J.dst[it][o], J.a[it][o], q), sc, sc_s, q); break;
      case HB_PW_ZERO: J.dst[it][o] = 0; break;
      case HB_PW_COPY: J.dst[it][o] = J.a[it][o]; break;
      case HB_PW_TENSOR: {
        u64 a0 = J.a[it][o], a1 = J.b[it][o], b0 = J.c[it][o], b1 = J.d[it][o];
        J.dst[it][o] = hb_mulmod(a0, b0, P);
        u64 hi = 0, lo = 0;
        hb_mac128(hi, lo, a0, b1);
        hb_mac128(hi, lo, a1, b0);
        J.dst1[it][o] = hb_reduce128(hi, lo, P);
        J.dst2[it][o] = hb_mulmod(a1, b1, P);
      } break;
      case HB_PW_MULADD: {   // dst += a*b (one read-modify-write pass instead of a product temp + an add)
        u64 hi = 0, lo = J.dst[it][o];
        hb_mac128(hi, lo, J.a[it][o], J.b[it][o]);
        J.dst[it][o] = hb_reduce128(hi, lo, P);
      } break;
      case HB_PW_AUTOMORPH: {
        // new[j] = old[idx(rep(j)*k mod m)], rep(j) = 2j+1, idx(r) = (r-1)/2  (power-of-two m)
        u64 r = ((2 * (u64)k + 1) * J.k) & (J.m - 1);
        J.dst[it][o] = J.a[it][off + (r >> 1)];
      } break;
    }
  }
}

// Ctxt::keySwitchDigits (src/Ctxt.cpp:191-230): out0 += sum_i D_i*b_i ; out1 += sum_i D_i*a_i,
// all digits of all batch items in one launch, one 128-bit accumulation + one reduction per output.
__global__ void __launch_bounds__(HB_THREADS) k_ks_inner(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbKsJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t N = (size_t)J.N;
  const size_t off = (size_t)pi * N;
  const int it = blockIdx.z;
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < N; k += (size_t)gridDim.x * blockDim.x) {
    const size_t o = off + k;
    size_t g = o;   // where the digit (and c0) element is read from
    u64 h0 = 0, l0 = 0, h1 = 0, l1 = 0;
    if (J.mode == 0) { l0 = J.out0[it][o]; l1 = J.out1[it][o]; }
    else if (J.mode == 1) {
      const u64 sc = J.scal[blockIdx.y];
      if (sc) { hb_mac128(h0, l0, J.out0[it][o], sc); hb_mac128(h1, l1, J.out1[it][o], sc); }
    } else {
      g = off + ((((2 * (u64)k + 1) * J.ak) & (J.am - 1)) >> 1);
      const u64 sc = J.scal[blockIdx.y];
      if (sc) hb_mac128(h0, l0, J.c0[it][g], sc);
    }
    for (int i = 0; i < J.ndig; i++) {
      u64 d = J.dig[it][i][g];
      hb_mac128(h0, l0, d, J.evk_b[i][o]);
      hb_mac128(h1, l1, d, J.evk_a[i][o]);
    }
    J.out0[it][o] = hb_reduce128(h0, l0, P);
    J.out1[it][o] = hb_reduce128(h1, l1, P);
  }
}

// Hoisted linear map (the loop body of MatMul1DExec::mul's native FULL branch, src/matmul.cpp:1226-1252): for every amount t
// of the launch, the hoisted key switch of k_ks_inner mode 2 times the constant cst[t], summed over the amounts:
//   acc0 (+)= sum_t cst_t * ( scal*sigma_kt(c0) + [k_t != 1] sum_i sigma_kt(D_i)*b_{t,i} )
//   acc1 (+)= sum_t cst_t * ( [k_t == 1] scal*c1 + [k_t != 1] sum_i sigma_kt(D_i)*a_{t,i} )
// Each inner product is summed in 128 bits and reduced once; its products with the constants are summed in 128 bits across
// the amounts and reduced once, when the accumulators are written.  All terms are below 2^120 (q < 2^60), so 255 fit:
// at most HB_LINMAP_MAXAMT amounts plus the accumulator's old value.
#define HB_LINMAP_MAXAMT 64
struct HbLinJob {
  u64 N, m;
  const int* rep; const int* irep;   // general m: sigma_k(x)[j] = x[irep[rep[j]*k mod m]];  null: power-of-two m
  int ndig, nitems, namt, accumulate;
  HbRows rows;
  u64 scal[HB_MAXROWS];              // P mod q on the rows of S, 0 on the special rows (addPrimesAndScale)
  u64 k[HB_LINMAP_MAXAMT];
  const u64* cst[HB_LINMAP_MAXAMT];
  const u64* evk_a[HB_LINMAP_MAXAMT][HB_MAXDIG];
  const u64* evk_b[HB_LINMAP_MAXAMT][HB_MAXDIG];
  const u64* dig[HB_MAXB][HB_MAXDIG];
  const u64* c0[HB_MAXB];
  const u64* c1[HB_MAXB];
  u64* acc0[HB_MAXB];
  u64* acc1[HB_MAXB];
};
// grid = (coefficient blocks, rows, item groups of NI): the NI items of a group share every key and constant word a thread
// loads, and keep their accumulators in registers (NI is a template parameter, so the per-item arrays are fully unrolled).
template <int NI>
__global__ void __launch_bounds__(HB_THREADS) k_ks_linmap(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbLinJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t N = (size_t)J.N;
  const size_t off = (size_t)pi * N;
  const u64 sc = J.scal[blockIdx.y];
  const int it0 = blockIdx.z * NI;
  const int cnt = J.nitems - it0 < NI ? J.nitems - it0 : NI;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += (size_t)gridDim.x * blockDim.x) {
    const size_t o = off + j;
    u64 h0[NI], l0[NI], h1[NI], l1[NI];
#pragma unroll
    for (int u = 0; u < NI; u++) {
      h0[u] = 0; l0[u] = 0; h1[u] = 0; l1[u] = 0;
      if (J.accumulate && u < cnt) { l0[u] = J.acc0[it0 + u][o]; l1[u] = J.acc1[it0 + u][o]; }
    }
    const u64 rj = J.rep ? (u64)J.rep[j] : 2 * (u64)j + 1;   // m <= 2^20: rj*k < 2^41
    for (int t = 0; t < J.namt; t++) {
      const u64 k = J.k[t];
      const u64 cw = J.cst[t][o];
      if (k == 1) {   // no automorphism, no key switch: cst * P * (c0, c1)
        const u64 scw = hb_mulmod(sc, cw, P);
#pragma unroll
        for (int u = 0; u < NI; u++)
          if (u < cnt) { hb_mac128(h0[u], l0[u], J.c0[it0 + u][o], scw); hb_mac128(h1[u], l1[u], J.c1[it0 + u][o], scw); }
        continue;
      }
      const size_t g = off + (J.rep ? (size_t)J.irep[(rj * k) % J.m] : (size_t)(((rj * k) & (J.m - 1)) >> 1));
      u64 p0h[NI], p0l[NI], p1h[NI], p1l[NI];
#pragma unroll
      for (int u = 0; u < NI; u++) {
        p0h[u] = 0; p0l[u] = 0; p1h[u] = 0; p1l[u] = 0;
        if (sc && u < cnt) hb_mac128(p0h[u], p0l[u], J.c0[it0 + u][g], sc);
      }
      for (int i = 0; i < J.ndig; i++) {
        const u64 b = J.evk_b[t][i][o], a = J.evk_a[t][i][o];
#pragma unroll
        for (int u = 0; u < NI; u++)
          if (u < cnt) { const u64 d = J.dig[it0 + u][i][g]; hb_mac128(p0h[u], p0l[u], d, b); hb_mac128(p1h[u], p1l[u], d, a); }
      }
#pragma unroll
      for (int u = 0; u < NI; u++) {
        hb_mac128(h0[u], l0[u], hb_reduce128(p0h[u], p0l[u], P), cw);
        hb_mac128(h1[u], l1[u], hb_reduce128(p1h[u], p1l[u], P), cw);
      }
    }
#pragma unroll
    for (int u = 0; u < NI; u++)
      if (u < cnt) { J.acc0[it0 + u][o] = hb_reduce128(h0[u], l0[u], P); J.acc1[it0 + u][o] = hb_reduce128(h1[u], l1[u], P); }
  }
}

// BSGS giant steps (MatMul1DExec::mul's non-iterative BSGS branches, src/matmul.cpp:1022-1057, 1097-1142), first pass: for
// every giant step t and item u of the launch, both parts of
//   out[t][u] (+)= sigma_kt( scal_t * sum_b cst[t][b] * baby[u][b] )
// sigma_k is applied on the write side: the thread of position j loads baby word j of every item once, uses it for all the
// giant steps of the launch, and writes each sum to the position that sigma_k moves j to, pi_{k^-1}(j) (the inverse of
// DoubleCRT::automorph's gather; kinv = k^-1 mod m).  Sums of up to HB_BSGS_MAXBABY products below 2^120 fit 128 bits and
// are reduced once.
#define HB_BSGS_MACW 8          // giant steps x items per launch (NT x NI): their 128-bit sums stay in registers
#define HB_BSGS_CST 1024        // constant rows per launch (giant steps x baby steps)
#define HB_BSGS_BABY 512        // baby rows per launch and part (items x baby steps)
#define HB_BSGS_MAXBABY 240     // baby steps per launch
struct HbBsgsMacJob {
  u64 N, m;
  const int* rep; const int* irep;   // general m; null: power-of-two m
  int nb, nt, ni, accumulate;
  HbRows rows;
  u64 kinv[HB_BSGS_MACW];
  u64 scal[HB_BSGS_MACW];
  const u64* cst[HB_BSGS_CST];       // [t*nb + b]; null: a zero diagonal
  const u64* baby0[HB_BSGS_BABY];    // [u*nb + b]
  const u64* baby1[HB_BSGS_BABY];
  u64* out0[HB_BSGS_MACW];           // [t*NI + u]
  u64* out1[HB_BSGS_MACW];
};
template <int NI>
__global__ void __launch_bounds__(HB_THREADS) k_bsgs_mac(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbBsgsMacJob J) {
  constexpr int NT = HB_BSGS_MACW / NI;
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t N = (size_t)J.N;
  const size_t off = (size_t)pi * N;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += (size_t)gridDim.x * blockDim.x) {
    const size_t o = off + j;
    u64 h0[NT][NI], l0[NT][NI], h1[NT][NI], l1[NT][NI];
#pragma unroll
    for (int t = 0; t < NT; t++)
#pragma unroll
      for (int u = 0; u < NI; u++) { h0[t][u] = 0; l0[t][u] = 0; h1[t][u] = 0; l1[t][u] = 0; }
    for (int b = 0; b < J.nb; b++) {
      u64 x0[NI], x1[NI];
#pragma unroll
      for (int u = 0; u < NI; u++) {
        x0[u] = 0; x1[u] = 0;
        if (u < J.ni) { x0[u] = J.baby0[u * J.nb + b][o]; x1[u] = J.baby1[u * J.nb + b][o]; }
      }
#pragma unroll
      for (int t = 0; t < NT; t++) {
        const u64* c = t < J.nt ? J.cst[t * J.nb + b] : nullptr;
        if (!c) continue;
        const u64 w = c[o];
#pragma unroll
        for (int u = 0; u < NI; u++) { hb_mac128(h0[t][u], l0[t][u], x0[u], w); hb_mac128(h1[t][u], l1[t][u], x1[u], w); }
      }
    }
    const u64 rj = J.rep ? (u64)J.rep[j] : 2 * (u64)j + 1;   // m <= 2^20: rj*kinv < 2^40
#pragma unroll
    for (int t = 0; t < NT; t++) {
      if (t < J.nt) {
        const u64 kk = J.kinv[t];
        const size_t g = off + (J.rep ? (size_t)J.irep[(rj * kk) % J.m] : (size_t)(((rj * kk) & (J.m - 1)) >> 1));
        const u64 s = hb_reduce128(0, J.scal[t], P);
#pragma unroll
        for (int u = 0; u < NI; u++) {
          if (u < J.ni) {
            u64* d0 = J.out0[t * NI + u];
            u64* d1 = J.out1[t * NI + u];
            u64 v0 = hb_mulmod(hb_reduce128(h0[t][u], l0[t][u], P), s, P);
            u64 v1 = hb_mulmod(hb_reduce128(h1[t][u], l1[t][u], P), s, P);
            if (J.accumulate) { v0 = hb_addmod(v0, d0[g], P.q); v1 = hb_addmod(v1, d1[g], P.q); }
            d0[g] = v0; d1[g] = v1;
          }
        }
      }
    }
  }
}

// BSGS giant steps, last pass: the key switch of every rotated term (Ctxt::keySwitchPart after breakIntoDigits, with the
// addPrimesAndScale of c0 folded in) and the unrotated terms, summed into the accumulators in one pass per group of terms:
//   acc0 (+)= sum_t [rotated] ( P*x0_t + sum_i D_{t,i}*b_{t,i} )  +  [unrotated] scx*x0_t
//   acc1 (+)= sum_t [rotated] (          sum_i D_{t,i}*a_{t,i} )  +  [unrotated] scx*x1_t
// Every product is below 2^120 and is summed in 128 bits without reduction: the host keeps nt*(ndig+1) + 1 <= 255.
// Term t of item it reads slot t*nitems + it.  grid = (coefficient blocks, rows, item groups of NI), as k_ks_linmap.
#define HB_BSGS_GROUP 32        // giant steps x items per group: the scratch of rotated sums, mod-downs and digits
struct HbGiantJob {
  u64 N;
  int ndig, nitems, nt, accumulate;
  HbRows rows;
  u64 scp[HB_MAXROWS];               // P mod q on the rows of S, 0 on the special rows (addPrimesAndScale)
  u64 scx[HB_MAXROWS];               // the factor of an unrotated term: scp (baby steps over S) or 1 (over S | special)
  unsigned char plain[HB_BSGS_GROUP];
  const u64* evk_a[HB_BSGS_GROUP][HB_MAXDIG];
  const u64* evk_b[HB_BSGS_GROUP][HB_MAXDIG];
  const u64* x0[HB_BSGS_GROUP];
  const u64* x1[HB_BSGS_GROUP];
  const u64* dig[HB_BSGS_GROUP][HB_MAXDIG];
  u64* acc0[HB_BSGS_GROUP];
  u64* acc1[HB_BSGS_GROUP];
};
template <int NI>
__global__ void __launch_bounds__(HB_THREADS) k_ks_giant(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbGiantJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t N = (size_t)J.N;
  const size_t off = (size_t)pi * N;
  const u64 sp = J.scp[blockIdx.y], sx = J.scx[blockIdx.y];
  const int it0 = blockIdx.z * NI;
  const int cnt = J.nitems - it0 < NI ? J.nitems - it0 : NI;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += (size_t)gridDim.x * blockDim.x) {
    const size_t o = off + j;
    u64 h0[NI], l0[NI], h1[NI], l1[NI];
#pragma unroll
    for (int u = 0; u < NI; u++) {
      h0[u] = 0; l0[u] = 0; h1[u] = 0; l1[u] = 0;
      if (J.accumulate && u < cnt) { l0[u] = J.acc0[it0 + u][o]; l1[u] = J.acc1[it0 + u][o]; }
    }
    for (int t = 0; t < J.nt; t++) {
      const int s0 = t * J.nitems + it0;
      if (J.plain[t]) {
        if (sx) {
#pragma unroll
          for (int u = 0; u < NI; u++)
            if (u < cnt) { hb_mac128(h0[u], l0[u], J.x0[s0 + u][o], sx); hb_mac128(h1[u], l1[u], J.x1[s0 + u][o], sx); }
        }
        continue;
      }
      if (sp) {
#pragma unroll
        for (int u = 0; u < NI; u++)
          if (u < cnt) hb_mac128(h0[u], l0[u], J.x0[s0 + u][o], sp);
      }
      for (int i = 0; i < J.ndig; i++) {
        const u64 b = J.evk_b[t][i][o], a = J.evk_a[t][i][o];
#pragma unroll
        for (int u = 0; u < NI; u++)
          if (u < cnt) { const u64 d = J.dig[s0 + u][i][o]; hb_mac128(h0[u], l0[u], d, b); hb_mac128(h1[u], l1[u], d, a); }
      }
    }
#pragma unroll
    for (int u = 0; u < NI; u++)
      if (u < cnt) { J.acc0[it0 + u][o] = hb_reduce128(h0[u], l0[u], P); J.acc1[it0 + u][o] = hb_reduce128(h1[u], l1[u], P); }
  }
}

// Block linear map (BlockMatMul1DExec::mul's non-iterative branches, src/matmul.cpp:1782-1974), first pass: the hoisted
// rotations BasicAutomorphPrecon::automorph(k_t) of a chunk of inner amounts, written for the items of a launch, i.e.
// k_ks_linmap's inner loop without the constant:
//   k_t != 1: out0 = scal*sigma_kt(c0) + sum_i sigma_kt(D_i)*b_{t,i},  out1 = sum_i sigma_kt(D_i)*a_{t,i}
//   k_t == 1: out0 = scal*c0, out1 = scal*c1                      (addPrimesAndScale of the S ciphertext)
// Each inner product (at most HB_MAXDIG + 1 products below 2^120) is summed in 128 bits and reduced once.  Amount t of
// item it writes slot t*nitems + it.  grid = (coefficient blocks, rows, item groups of NI), as k_ks_linmap.
#define HB_HOIST_MAXAMT 64      // inner amounts per launch
#define HB_HOIST_SLOTS 128      // rotations x items in a chunk: the rotation scratch of hb_block_linear_map
struct HbHoistJob {
  u64 N, m;
  const int* rep; const int* irep;   // general m; null: power-of-two m
  int ndig, nitems, namt;
  HbRows rows;
  u64 scal[HB_MAXROWS];              // P mod q on the rows of S, 0 on the special rows
  u64 k[HB_HOIST_MAXAMT];
  const u64* evk_a[HB_HOIST_MAXAMT][HB_MAXDIG];
  const u64* evk_b[HB_HOIST_MAXAMT][HB_MAXDIG];
  const u64* dig[HB_MAXB][HB_MAXDIG];
  const u64* c0[HB_MAXB];
  const u64* c1[HB_MAXB];
  u64* out0[HB_HOIST_SLOTS];
  u64* out1[HB_HOIST_SLOTS];
};
template <int NI>
__global__ void __launch_bounds__(HB_THREADS) k_ks_hoist(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbHoistJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t N = (size_t)J.N;
  const size_t off = (size_t)pi * N;
  const u64 sc = J.scal[blockIdx.y];
  const int it0 = blockIdx.z * NI;
  const int cnt = J.nitems - it0 < NI ? J.nitems - it0 : NI;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += (size_t)gridDim.x * blockDim.x) {
    const size_t o = off + j;
    const u64 rj = J.rep ? (u64)J.rep[j] : 2 * (u64)j + 1;   // m <= 2^20: rj*k < 2^41
    for (int t = 0; t < J.namt; t++) {
      const u64 k = J.k[t];
      const int s0 = t * J.nitems + it0;
      if (k == 1) {
#pragma unroll
        for (int u = 0; u < NI; u++)
          if (u < cnt) {
            J.out0[s0 + u][o] = hb_mulmod(J.c0[it0 + u][o], sc, P);
            J.out1[s0 + u][o] = hb_mulmod(J.c1[it0 + u][o], sc, P);
          }
        continue;
      }
      const size_t g = off + (J.rep ? (size_t)J.irep[(rj * k) % J.m] : (size_t)(((rj * k) & (J.m - 1)) >> 1));
      u64 p0h[NI], p0l[NI], p1h[NI], p1l[NI];
#pragma unroll
      for (int u = 0; u < NI; u++) {
        p0h[u] = 0; p0l[u] = 0; p1h[u] = 0; p1l[u] = 0;
        if (sc && u < cnt) hb_mac128(p0h[u], p0l[u], J.c0[it0 + u][g], sc);
      }
      for (int i = 0; i < J.ndig; i++) {
        const u64 b = J.evk_b[t][i][o], a = J.evk_a[t][i][o];
#pragma unroll
        for (int u = 0; u < NI; u++)
          if (u < cnt) { const u64 d = J.dig[it0 + u][i][g]; hb_mac128(p0h[u], p0l[u], d, b); hb_mac128(p1h[u], p1l[u], d, a); }
      }
#pragma unroll
      for (int u = 0; u < NI; u++)
        if (u < cnt) { J.out0[s0 + u][o] = hb_reduce128(p0h[u], p0l[u], P); J.out1[s0 + u][o] = hb_reduce128(p1h[u], p1l[u], P); }
    }
  }
}

// Full linear map leaves (MatMulFullExec::rec_mul's last dimension, src/matmul.cpp:2141-2148, each leaf a hoisted
// MatMul1DExec::mul, :1226-1283): k_ks_linmap's hoisted key switch with the roles changed.  All leaves share the amounts
// and the matrices; leaf l of item it has its own digits, (c0, c1) over S and constants cst[l][t].  For every item:
//   acc (+)= sum_l sum_t cst[l][t] * r_{l,t},  r_{l,t} = the hoisted rotation by k_t of leaf l (k_t == 1: scal*(c0, c1))
//   BAD:  y_l (+)= sum_t cst1[l][t] * r_{l,t}   per leaf (HElib rotates and mods down every leaf's acc1 on its own)
// The thread of position j holds LI leaves of one item: it loads each key word once for all of them.  Each inner product is
// summed in 128 bits and reduced once; the products with the constants (below 2^120) go into one 128-bit sum per item
// across leaves and amounts, reduced and carried before it holds 255 terms (its old value counts as one).  A y_l sum has
// at most HB_LEAF_MAXAMT + 1 terms.  NULL constants are zero diagonals, skipped as MulAdd skips them.
// Slot s = l*nitems + it holds leaf l of item it.  grid = (coefficient blocks, rows, items).  LI is 1, 2 or 4: at two CTAs
// per SM (at most 128 registers) every instance keeps its state in registers, with no stack frame and no spill.
#define HB_LEAF_PAIRS 32        // (item, leaf) pairs per launch: the leaf scratch of hb_full_linear_map_leaves
#define HB_LEAF_MAXAMT 32       // amounts per launch
struct HbLeafJob {
  u64 N, m;
  const int* rep; const int* irep;   // general m; null: power-of-two m
  int ndig, nitems, nleaves, namt, accumulate, accumulate1;
  HbRows rows;
  u64 scal[HB_MAXROWS];              // P mod q on the rows of S, 0 on the special rows (addPrimesAndScale)
  u64 k[HB_LEAF_MAXAMT];
  const u64* evk_a[HB_LEAF_MAXAMT][HB_MAXDIG];
  const u64* evk_b[HB_LEAF_MAXAMT][HB_MAXDIG];
  const u64* cst[HB_LEAF_PAIRS * HB_LEAF_MAXAMT];    // [l*namt + t]; null: a zero diagonal
  const u64* cst1[HB_LEAF_PAIRS * HB_LEAF_MAXAMT];   // the bad dimension's second set, same layout
  const u64* dig[HB_LEAF_PAIRS][HB_MAXDIG];          // slot s
  const u64* c0[HB_LEAF_PAIRS];
  const u64* c1[HB_LEAF_PAIRS];
  u64* y0[HB_LEAF_PAIRS];                            // BAD: the per-leaf sums, slot s
  u64* y1[HB_LEAF_PAIRS];
  u64* acc0[HB_LEAF_PAIRS];                          // [it]
  u64* acc1[HB_LEAF_PAIRS];
};
template <int LI, bool BAD>
__global__ void __launch_bounds__(HB_THREADS, 2) k_ks_leafmap(const HbPrimeDev* __restrict__ primes, const HB_GRID_CONSTANT HbLeafJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const HbPrimeDev P = primes[pi];
  const size_t N = (size_t)J.N;
  const size_t off = (size_t)pi * N;
  const u64 sc = J.scal[blockIdx.y];
  const int it = blockIdx.z, ni = J.nitems, na = J.namt;
  for (size_t j = (size_t)blockIdx.x * blockDim.x + threadIdx.x; j < N; j += (size_t)gridDim.x * blockDim.x) {
    const size_t o = off + j;
    u64 h0 = 0, l0 = 0, h1 = 0, l1 = 0;
    if (J.accumulate) { l0 = J.acc0[it][o]; l1 = J.acc1[it][o]; }
    int terms = 1;   // terms in (h, l): the old value
    const u64 rj = J.rep ? (u64)J.rep[j] : 2 * (u64)j + 1;   // m <= 2^20: rj*k < 2^41
    for (int lg = 0; lg < J.nleaves; lg += LI) {
      const int cnt = J.nleaves - lg < LI ? J.nleaves - lg : LI;
      u64 yh0[LI], yl0[LI], yh1[LI], yl1[LI];
#pragma unroll
      for (int u = 0; u < LI; u++) {
        yh0[u] = 0; yl0[u] = 0; yh1[u] = 0; yl1[u] = 0;
        if (BAD && J.accumulate1 && u < cnt) { const int s = (lg + u) * ni + it; yl0[u] = J.y0[s][o]; yl1[u] = J.y1[s][o]; }
      }
      for (int t = 0; t < na; t++) {
        bool any = false;
#pragma unroll
        for (int u = 0; u < LI; u++)
          if (u < cnt) any = any || J.cst[(lg + u) * na + t] || (BAD && J.cst1[(lg + u) * na + t]);
        if (!any) continue;
        if (terms > 254 - LI) { l0 = hb_reduce128(h0, l0, P); l1 = hb_reduce128(h1, l1, P); h0 = 0; h1 = 0; terms = 1; }
        terms += LI;
        const u64 k = J.k[t];
        u64 r0[LI], r1[LI];
        if (k == 1) {   // no automorphism, no key switch: P*(c0, c1)
#pragma unroll
          for (int u = 0; u < LI; u++) {
            r0[u] = 0; r1[u] = 0;
            if (sc && u < cnt) {
              const int s = (lg + u) * ni + it;
              r0[u] = hb_mulmod(J.c0[s][o], sc, P); r1[u] = hb_mulmod(J.c1[s][o], sc, P);
            }
          }
        } else {
          const size_t g = off + (J.rep ? (size_t)J.irep[(rj * k) % J.m] : (size_t)(((rj * k) & (J.m - 1)) >> 1));
          u64 p0h[LI], p0l[LI], p1h[LI], p1l[LI];
#pragma unroll
          for (int u = 0; u < LI; u++) {
            p0h[u] = 0; p0l[u] = 0; p1h[u] = 0; p1l[u] = 0;
            if (sc && u < cnt) hb_mac128(p0h[u], p0l[u], J.c0[(lg + u) * ni + it][g], sc);
          }
          for (int i = 0; i < J.ndig; i++) {
            const u64 b = J.evk_b[t][i][o], a = J.evk_a[t][i][o];
#pragma unroll
            for (int u = 0; u < LI; u++)
              if (u < cnt) { const u64 d = J.dig[(lg + u) * ni + it][i][g]; hb_mac128(p0h[u], p0l[u], d, b); hb_mac128(p1h[u], p1l[u], d, a); }
          }
#pragma unroll
          for (int u = 0; u < LI; u++) { r0[u] = hb_reduce128(p0h[u], p0l[u], P); r1[u] = hb_reduce128(p1h[u], p1l[u], P); }
        }
#pragma unroll
        for (int u = 0; u < LI; u++) {
          if (u >= cnt) continue;
          const u64* c = J.cst[(lg + u) * na + t];
          if (c) { const u64 w = c[o]; hb_mac128(h0, l0, r0[u], w); hb_mac128(h1, l1, r1[u], w); }
          if (BAD) {
            const u64* c1 = J.cst1[(lg + u) * na + t];
            if (c1) { const u64 w = c1[o]; hb_mac128(yh0[u], yl0[u], r0[u], w); hb_mac128(yh1[u], yl1[u], r1[u], w); }
          }
        }
      }
      if (BAD) {
#pragma unroll
        for (int u = 0; u < LI; u++)
          if (u < cnt) { const int s = (lg + u) * ni + it; J.y0[s][o] = hb_reduce128(yh0[u], yl0[u], P); J.y1[s][o] = hb_reduce128(yh1[u], yl1[u], P); }
      }
    }
    J.acc0[it][o] = hb_reduce128(h0, l0, P);
    J.acc1[it][o] = hb_reduce128(h1, l1, P);
  }
}


// ------------------------------------------------------------------------------------------
// Canonical-embedding norm (noise metadata): max_j |f(zeta^(2j+1))|, zeta = e^(i*pi/N), in FP64.
// Replaces embeddingLargestCoeff (src/norms.cpp:204-261,443-485) for power-of-two m.
// frac[k] -> z[k] = frac[k] * e^(i*pi*k/N); length-N complex DIF FFT, radix-16 per pass; max |z|.
#ifdef HB_SIM
#include <cmath>
struct double2 { double x, y; };
static inline void sincospi(double a, double* s, double* c) { *s = sin(a * 3.14159265358979323846); *c = cos(a * 3.14159265358979323846); }
#endif
struct HbNormJob { int logN; int npoly; const double* frac; double2* z; unsigned long long* maxbits; };
__global__ void __launch_bounds__(HB_THREADS) k_norm_twist(HbNormJob J) {
  const size_t N = (size_t)1 << J.logN;
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < N; k += (size_t)gridDim.x * blockDim.x) {
    double s, c;
    sincospi((double)k / (double)N, &s, &c);
    const double f = J.frac[(size_t)blockIdx.y * N + k];
    double2 o; o.x = f * c; o.y = f * s;
    J.z[(size_t)blockIdx.y * N + k] = o;
  }
}
// one radix-2 DIF stage at distance d = 2^logd (in place); the last stage also reduces max |z|^2
__global__ void __launch_bounds__(HB_THREADS) k_norm_stage(HbNormJob J, int logd, int last) {
  const size_t N = (size_t)1 << J.logN, half = N >> 1, d = (size_t)1 << logd;
  double2* z = J.z + (size_t)blockIdx.y * N;
  double m = 0.0;
  for (size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x; b < half; b += (size_t)gridDim.x * blockDim.x) {
    const size_t o = b & (d - 1), p = ((b >> logd) << (logd + 1)) + o;
    const double2 u = z[p], v = z[p + d];
    double s, c;
    sincospi(-(double)o / (double)d, &s, &c);   // W_{2d}^o
    double2 a, t, w;
    a.x = u.x + v.x; a.y = u.y + v.y;
    t.x = u.x - v.x; t.y = u.y - v.y;
    w.x = t.x * c - t.y * s; w.y = t.x * s + t.y * c;
    z[p] = a; z[p + d] = w;
    if (last) { const double ma = a.x * a.x + a.y * a.y, mw = w.x * w.x + w.y * w.y; m = ma > m ? ma : m; m = mw > m ? mw : m; }
  }
  if (last) {
#ifdef HB_SIM
    unsigned long long bits; memcpy(&bits, &m, 8);
    if (bits > J.maxbits[blockIdx.y]) J.maxbits[blockIdx.y] = bits;
#else
    atomicMax(J.maxbits + blockIdx.y, (unsigned long long)__double_as_longlong(m));  // non-negative doubles order like integers
#endif
  }
}


// Scale rows by per-row constants and write the result to the local destination AND to the same rows of
// up to 8 peer GPUs' buffers (peer device memory mapped through CUDA IPC, stores travel over NVLink).
// This is the tail of the prime-sharded conversion's "make y" step fused with its all-gather: the y rows
// cross the fabric exactly once, straight into place (no pack / collective / unpack passes).
#define HB_MAXPEERS 8
struct HbBcastJob {
  u64 N;
  HbRows rows;
  u64 scal[HB_MAXROWS], scal_s[HB_MAXROWS];
  int nitems, npeers;
  u64* loc[HB_MAXB];                   // in/out, local
  u64* peer[HB_MAXPEERS][HB_MAXB];     // out, remote
};
__global__ void __launch_bounds__(HB_THREADS) k_scale_bcast(const HbPrimeDev* __restrict__ primes, const HbBcastJob J) {
  const int pi = J.rows.prime[blockIdx.y];
  const u64 q = primes[pi].q;
  const size_t N = (size_t)J.N, off = (size_t)pi * N;
  const int it = blockIdx.z;
  const u64 sc = J.scal[blockIdx.y], sc_s = J.scal_s[blockIdx.y];
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < N; k += (size_t)gridDim.x * blockDim.x) {
    const u64 v = hb_mul_shoup(J.loc[it][off + k], sc, sc_s, q);
    J.loc[it][off + k] = v;
    for (int p = 0; p < J.npeers; p++) J.peer[p][it][off + k] = v;
  }
}
