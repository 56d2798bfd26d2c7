// hb_engine.cu -- host side of the H100 DoubleCRT engine and its C ABI (include/helib_b200.h).
//
// Host C++ owns the chain metadata (primes, psi, digit partition), builds the per-prime twiddle
// tables and the exact-CRT conversion tables, and issues stream-ordered launches of the kernels
// in hb_device.cuh.  There is no CPU compute path: without a CUDA device hb_ctx_create fails.
#include "hb_device.cuh"
#include "hb_device_v1.cuh"
#include "hb_device_v2.cuh"
#include "hb_device_gen.cuh"
#include "hb_device_prg.cuh"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/helib_b200.h"

typedef unsigned __int128 u128;

// k1_fwd_blk_tensor (nparts 4) and k1_fwd_blk_square (nparts 2): S[2][HB1_STAGE] | O[16][256] | TW1[256] | V[nparts - 1][16][256]
static size_t blk_parts_smem(int nparts) {
  return (2 * HB1_STAGE + 16 * 256 + (nparts - 1) * 16 * 256) * sizeof(u64) + 256 * sizeof(ulonglong2);
}

// ------------------------------------------------------------------------------------------
// errors
static thread_local char g_err[512] = "";
static thread_local int g_chunk = HB_MAXB;   // batch items per launch for the current call (hb_ctx::chunk)
static int hb_fail(int code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
  return code;
}
#define HB_CUDA(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return hb_fail(HB_ERR_CUDA, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)
#define HB_TRY(x) do { int r_ = (x); if (r_ != HB_OK) return r_; } while (0)

// ------------------------------------------------------------------------------------------
// host modular arithmetic
static inline u64 h_mulmod(u64 a, u64 b, u64 q) { return (u64)((u128)a * b % q); }
static inline u64 h_powmod(u64 a, u64 e, u64 q) {
  u64 r = 1 % q; a %= q;
  while (e) { if (e & 1) r = h_mulmod(r, a, q); a = h_mulmod(a, a, q); e >>= 1; }
  return r;
}
static inline u64 h_shoup(u64 w, u64 q) { return (u64)(((u128)w << 64) / q); }
static bool h_invmod(u64 a, u64 m, u64* out) {  // extended Euclid, m need not be prime
  __int128 t0 = 0, t1 = 1, r0 = m, r1 = a % m;
  while (r1 != 0) { __int128 qq = r0 / r1, t2 = t0 - qq * t1, r2 = r0 - qq * r1; t0 = t1; t1 = t2; r0 = r1; r1 = r2; }
  if (r0 != 1) return false;
  *out = (u64)(((t0 % (__int128)m) + (__int128)m) % (__int128)m);
  return true;
}
static int h_bitlen(u64 x) { int b = 0; while (x) { b++; x >>= 1; } return b; }

// ------------------------------------------------------------------------------------------
struct ConvEntry {
  HbConvDev h;          // host copy of the descriptor (device pointers inside)
  HbConvDev* d;         // device descriptor
  void* blob;           // device blob
  const u64* d_t; const u64* d_t_s;  // (Q/q_j)^-1 without N^-1 (for k_crt)
};

struct hb_ctx {
  int device;
  u64 m; size_t N; int logN, log_blk, nprimes;
  std::vector<u64> q, psi;
  std::vector<HbPrimeDev> h_primes;
  HbPrimeDev* d_primes;
  ulonglong2* d_tw;
  cudaStream_t stream; cudaStream_t own_stream; bool stream_external = false;
  std::vector<int> digit_of; int ndigits; std::vector<int> special;
  u64* tmpA; u64* tmpB;
  double* d_frac; void* d_z; unsigned long long* d_max;   // embedding-norm scratch (allocated on first use)
  u64* d_stats;
  HbBcastJob* d_bcast = nullptr;   // job descriptor of k_scale_bcast (too large for kernel parameters)
  std::map<std::string, ConvEntry> convs;
  std::vector<hb_poly*> pool;
  size_t bytes; u64 launches;
  cudaEvent_t ev0, ev1;
  size_t max_smem;
  bool force_v0;     // HB_FORCE_V0=1: generic radix-2 kernels only (A/B testing)
  bool conv1;        // dedicated single-source conversion kernel k1_conv1 (HB_CONV1=0 falls back to the general k1_conv)
  int chunk;         // batch items per launch (<= HB_MAXB; HB_CHUNK overrides): keeps the phase scratch L2-sized
  int resident_ctas; // CTAs the v1 transform kernels keep resident (2 per SM)
  // TMA-staged blk kernels (hb_device_v2.cuh): tensor maps of every matrix they touch, built on first use
  bool blk_v2;       // HB_BLK_V2=1 selects the TMA-staged kernels k2_fwd_blk / k2_inv_blk instead of k1_fwd_blk / k1_inv_blk
  struct TmapKey { const void* base; int logN; bool operator<(const TmapKey& o) const { return base != o.base ? base < o.base : logN < o.logN; } };
  std::map<TmapKey, HbTmap*> tmaps;      // -> device pair {BLK view, NAT view}
  std::vector<HbTmap*> tmap_slabs; size_t tmap_used = 0;
  // general (non power-of-two) m: Bluestein state
  struct Gen {
    bool on = false;
    u64 m = 0, phim = 0, L = 0, d = 0; int logL = 0, log_blk_L = 0;
    u64 L2 = 0; int logL2 = 0, log_blk_L2 = 0;        // short cyclic plan of the division by Phi_m: L2 = 2^ceil(log2 max(phi(m), 2d-1)) <= L
    int* d_rep = nullptr; int* d_irep = nullptr;
    HbGenPrime* d_gp = nullptr;
    HbPrimeDev* d_primes_cyc = nullptr; HbPrimeDev* d_primes_cyc2 = nullptr;
    void* tab = nullptr;
    double2* d_W = nullptr;                             // e^(2 pi I j/m), j < m (embedding norms; built on first use)
    u64 *w0 = nullptr, *w1 = nullptr, *wt = nullptr;   // [HB_MAXB][nprimes][L]
    u64 *cA = nullptr, *cB = nullptr;                   // [HB_MAXB][nprimes][phim]
  } gen;
  struct Pw {   // powerful basis (src/powerful.cpp): built on first use or by hb_ctx_set_powerful
    bool ready = false, triv = true;
    std::vector<long> mvec, pvec, bvec, long_prod;     // m_d = p_d^e_d, p_d, p_d^(e_d-1), products of the trailing dimensions
    std::vector<int> cube_to_poly, short_to_long;      // host copies (the mirror's powerfulToZZX needs them)
    int* d_cube_to_poly = nullptr; int* d_short_to_long = nullptr;
    u64* cube = nullptr;                               // [nprimes][m]
    u64* rows = nullptr;                               // [nprimes][phim] powerful-basis rows
  } pw;
  // optional per-launch profiling (bench.py): CUDA events around every kernel launch
  bool profiling;
  struct ProfRec { const char* name; cudaEvent_t a, b; u64 bytes; };
  std::vector<ProfRec> prof_pending;
  struct ProfAgg { std::string name; u64 launches; double ms; u64 bytes; };
  std::vector<ProfAgg> prof;
  // seeded row expansion (hb_poly_randomize): row starts, per-buffer offsets and the CTA ticket of k_prg_count
  u64* prg_start = nullptr; unsigned* prg_off = nullptr; unsigned long long* prg_ticket = nullptr;
  size_t prg_start_cap = 0, prg_off_cap = 0;
  int prg_window = 0;   // HB_PRG_WINDOW=w: count w buffers per row in parallel instead of the statistical bound (tests the slow path)
  std::vector<hb_poly*> ks_a;   // a_i regenerated from a seeded evk_a for the key switch in flight (allocated on first use)
  std::vector<hb_poly*> bsgs;   // hb_bsgs_linear_map: rotated sums and their digits, HB_BSGS_GROUP*(2+ndig) polys (first use)
  std::vector<hb_poly*> block;  // hb_block_linear_map: rotations, rotated sums, digits and set-1 sums (first use)
  std::vector<hb_poly*> ip;     // hb_inner_product: the s^2 part of each item of a chunk (first use)
  std::vector<hb_poly*> leaf;   // hb_full_linear_map_leaves: cleaned leaves, their digits, per-leaf sums, final matrix (first use)
  u64* ssum = nullptr; size_t ssum_cap = 0;   // hb_ctxt_scaled_sums: its scalar, constant and pointer tables (grown on demand)
};
// The row schedule of a seeded set (hb_poly_create_seeded): the ChaCha20 key, the rows, and in one device allocation the
// first buffer of every schedule row (start[T+1]) and the exclusive row offset of every counted buffer (off[T*wmax]).
// Schedule row p*n + r is row idx[r] of poly p.  Shared by the set's handles, freed with the last one.
struct HbSeedSched {
  HbPrgKey key;
  std::vector<int32_t> idx;
  std::vector<HbPrgRow> rows;   // per schedule row: candidate format and counted window (row pointers unset)
  int wmax = 1;
  void* blk = nullptr; size_t bytes = 0;
  u64* start = nullptr; unsigned* off = nullptr;
  int refs = 0;
};
// A seeded poly (sched != nullptr) has no rows: d is null.  Only the key-switching entry points (as evk_a) and hb_poly_expand
// accept one; everything else rejects it before launching anything.
struct hb_poly { hb_ctx* ctx; u64* d; bool owned = true; bool ipc = false; HbSeedSched* sched = nullptr; int sched_poly = 0; };

static int ctx_alloc(hb_ctx* c, void** p, size_t bytes) {
  cudaError_t e = cudaMalloc(p, bytes);
  if (e != cudaSuccess) return hb_fail(HB_ERR_OOM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
  c->bytes += bytes;
  return HB_OK;
}
static int ctx_scratch(hb_ctx* c) {
  if (c->tmpA) return HB_OK;
  size_t sz = (size_t)HB_MAXB * c->nprimes * c->N * sizeof(u64);
  HB_TRY(ctx_alloc(c, (void**)&c->tmpA, sz));
  HB_TRY(ctx_alloc(c, (void**)&c->tmpB, sz));
  return HB_OK;
}
static void pre_launch(hb_ctx* c) {
#ifndef HB_SIM
  if (c->profiling) {
    hb_ctx::ProfRec r; r.name = nullptr; r.bytes = 0;
    cudaEventCreate(&r.a); cudaEventCreate(&r.b);
    cudaEventRecord(r.a, c->stream);
    c->prof_pending.push_back(r);
  }
#endif
}
// bytes = algorithmic HBM bytes of this launch (rows read once + rows written once)
static int post_launch(hb_ctx* c, const char* what, u64 bytes = 0) {
  c->launches++;
  static const bool trace = getenv("HB_TRACE") != nullptr;
  if (trace) fprintf(stderr, "[hb] launch %s alg_bytes=%llu\n", what, (unsigned long long)bytes);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hb_fail(HB_ERR_CUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
#ifndef HB_SIM
  if (c->profiling && !c->prof_pending.empty()) {
    hb_ctx::ProfRec& r = c->prof_pending.back();
    r.name = what; r.bytes = bytes;
    cudaEventRecord(r.b, c->stream);
  }
#else
  if (c->profiling) {   // the simulator has no events: launch names and counts only, so tests can see which kernels ran
    bool found = false;
    for (auto& a : c->prof) if (a.name == what) { a.launches++; a.bytes += bytes; found = true; break; }
    if (!found) c->prof.push_back({what, 1, 0.0, bytes});
  }
#endif
  return HB_OK;
}

// ------------------------------------------------------------------------------------------
extern "C" int hb_version(void) { return 100; }
extern "C" const char* hb_last_error(void) { return g_err; }
extern "C" int hb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

static u64 find_psi(u64 q, u64 two_n) {
  u64 g = 2;
  while (h_powmod(g, (q - 1) / 2, q) != q - 1) g++;
  return h_powmod(g, (q - 1) / two_n, q);
}

static int gen_init(hb_ctx* c, const uint64_t* psi);
static int ctx_build(hb_ctx* c, hb_ctx** out, int device, uint64_t m, int nprimes, const uint64_t* q, const uint64_t* psi, bool pow2);
extern "C" int hb_ctx_create(hb_ctx** out, int device, uint64_t m, int nprimes, const uint64_t* q, const uint64_t* psi) {
  if (!out || !q || nprimes <= 0) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_create: null argument or nprimes <= 0");
  if (m < 3 || m > (1ULL << 20)) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_create: m=%llu out of range [3, 2^20]", (unsigned long long)m);
  const bool pow2 = (m & (m - 1)) == 0;
  int ndev = hb_device_count();
  if (ndev <= 0) return hb_fail(HB_ERR_NO_DEVICE, "hb_ctx_create: no CUDA device (the engine has no CPU path)");
  if (device < 0 || device >= ndev) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_create: device %d out of range [0,%d)", device, ndev);
  HB_CUDA(cudaSetDevice(device));
  hb_ctx* c = new hb_ctx();   // value-initialised: every pointer null, so hb_ctx_destroy can unwind a partial construction
  const int rc = ctx_build(c, out, device, m, nprimes, q, psi, pow2);
  if (rc != HB_OK) hb_ctx_destroy(c);
  return rc;
}
static int ctx_build(hb_ctx* c, hb_ctx** out, int device, uint64_t m, int nprimes, const uint64_t* q, const uint64_t* psi, bool pow2) {
  c->device = device; c->m = m; c->N = pow2 ? m / 2 : 0; c->nprimes = nprimes;
  c->logN = 0; while (((size_t)1 << c->logN) < c->N) c->logN++;
  c->log_blk = c->logN >= 11 ? 8 : 0;
  c->tmpA = c->tmpB = nullptr; c->d_frac = nullptr; c->d_z = nullptr; c->d_max = nullptr; c->bytes = 0; c->launches = 0; c->ndigits = 0;
  c->d_primes = nullptr; c->d_tw = nullptr; c->d_stats = nullptr; c->profiling = false;
  c->digit_of.assign(nprimes, -1);
  c->max_smem = 200 * 1024;
  { const char* e = getenv("HB_FORCE_V0"); c->force_v0 = e && e[0] == '1'; }
  { const char* e = getenv("HB_CONV1"); c->conv1 = !(e && e[0] == '0'); }
  { const char* e = getenv("HB_BLK_V2"); c->blk_v2 = e && e[0] == '1'; }
  { const char* e = getenv("HB_CHUNK"); int v = e ? atoi(e) : HB_MAXB; c->chunk = v >= 1 && v <= HB_MAXB ? v : HB_MAXB; }
  { const char* e = getenv("HB_PRG_WINDOW"); int v = e ? atoi(e) : 0; c->prg_window = v >= 1 ? v : 0; }
  c->resident_ctas = 264;   // 2 per SM on a 132-SM H100 if the device query fails
#ifdef HB_SIM
  c->resident_ctas = 7;   // few, odd: every simulated CTA walks several units and crosses (row, block-group) boundaries
#endif
#ifndef HB_SIM
  { cudaDeviceProp prop; if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->resident_ctas = 2 * prop.multiProcessorCount; }
#endif
  const size_t N = c->N;
  for (int i = 0; i < nprimes; i++) {
    u64 qi = q[i];
    // HElib primes are < 2^HELIB_SP_NBITS = 2^60 (src/macro.h:16-23); the lazy butterflies need 13q + 2^49 < 2^64
    if (qi < 3 || qi >= (1ULL << 60) || (qi - 1) % m != 0) { return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_create: q[%d]=%llu is not < 2^60 with m | q-1", i, (unsigned long long)qi); }
    u64 ps = 0;
    if (pow2) {
      ps = psi ? psi[i] : find_psi(qi, m);
      if (h_powmod(ps, N, qi) != qi - 1) { return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_create: psi[%d] is not a primitive %llu-th root of unity mod q", i, (unsigned long long)m); }
    }
    c->q.push_back(qi); c->psi.push_back(ps);
  }
  HB_CUDA(cudaStreamCreate(&c->stream));
  c->own_stream = c->stream;
#ifndef HB_SIM
  HB_CUDA(cudaEventCreate(&c->ev0)); HB_CUDA(cudaEventCreate(&c->ev1));
#endif
  if (!pow2) {   // general m: Bluestein rows (src/bluestein.cpp); no negacyclic tables
    c->h_primes.resize(nprimes);
    for (int i = 0; i < nprimes; i++) {
      u64 qi = c->q[i];
      HbPrimeDev& P = c->h_primes[i];
      memset(&P, 0, sizeof(P));
      P.q = qi; P.c64 = (u64)(((u128)1 << 64) % qi); P.c64_s = h_shoup(P.c64, qi); P.one_s = (u64)(((u128)1 << 64) / qi);
      P.nq = 0 - qi; P.qb = 4 * qi;
      { int sh = 0; u64 t = qi - 1; while ((t & 1) == 0) { t >>= 1; sh++; }
        if (sh >= 32 && t < (1ULL << 32)) { P.qt = (unsigned)t; P.qsh = (unsigned)(sh - 32); } }
    }
    HB_TRY(ctx_alloc(c, (void**)&c->d_primes, sizeof(HbPrimeDev) * nprimes));
    HB_CUDA(cudaMemcpy(c->d_primes, c->h_primes.data(), sizeof(HbPrimeDev) * nprimes, cudaMemcpyHostToDevice));
    HB_TRY(ctx_alloc(c, (void**)&c->d_stats, 4 * sizeof(u64)));
    HB_CUDA(cudaMemset(c->d_stats, 0, 4 * sizeof(u64)));
#ifndef HB_SIM
    HB_CUDA(cudaFuncSetAttribute(k_fwd_blk, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    HB_CUDA(cudaFuncSetAttribute(k_inv_blk, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    HB_CUDA(cudaFuncSetAttribute(k1_fwd_blk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_fwd_blk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
    HB_CUDA(cudaFuncSetAttribute(k1_inv_blk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_inv_blk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
    HB_CUDA(cudaFuncSetAttribute(k2_fwd_blk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HB2_SMEM_BYTES));
    HB_CUDA(cudaFuncSetAttribute(k2_fwd_blk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HB2_SMEM_BYTES));
    HB_CUDA(cudaFuncSetAttribute(k2_inv_blk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HB2_SMEM_BYTES));
    HB_CUDA(cudaFuncSetAttribute(k2_inv_blk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HB2_SMEM_BYTES));
#endif
    HB_TRY(gen_init(c, psi));
    *out = c;
    return HB_OK;
  }
  // twiddle tables: fw[k] = psi^brev(k), iw[k] = psi^-brev(k)
  std::vector<ulonglong2> tw((size_t)nprimes * 2 * N);
  std::vector<u64> pw(N);
  std::vector<unsigned> brev(N);
  for (size_t k = 0; k < N; k++) { unsigned r = 0; for (int b = 0; b < c->logN; b++) if (k >> b & 1) r |= 1u << (c->logN - 1 - b); brev[k] = r; }
  HB_TRY(ctx_alloc(c, (void**)&c->d_tw, tw.size() * sizeof(ulonglong2)));
  c->h_primes.resize(nprimes);
  for (int i = 0; i < nprimes; i++) {
    u64 qi = c->q[i];
    for (int dir = 0; dir < 2; dir++) {
      u64 base = dir == 0 ? c->psi[i] : h_powmod(c->psi[i], qi - 2, qi);
      u64 w = 1;
      for (size_t e = 0; e < N; e++) { pw[e] = w; w = h_mulmod(w, base, qi); }
      ulonglong2* t = &tw[((size_t)i * 2 + dir) * N];
      for (size_t k = 0; k < N; k++) { u64 v = pw[brev[k]]; t[k] = make_ulonglong2(v, h_shoup(v, qi)); }
    }
    HbPrimeDev& P = c->h_primes[i];
    P.q = qi;
    P.ninv = h_powmod((u64)N % qi, qi - 2, qi); P.ninv_s = h_shoup(P.ninv, qi);
    P.c64 = (u64)(((u128)1 << 64) % qi); P.c64_s = h_shoup(P.c64, qi);
    P.one_s = (u64)(((u128)1 << 64) / qi);
    P.nq = 0 - qi; P.qb = 4 * qi;
    { int sh = 0; u64 t = qi - 1; while ((t & 1) == 0) { t >>= 1; sh++; }
      if (sh >= 32 && t < (1ULL << 32)) { P.qt = (unsigned)t; P.qsh = (unsigned)(sh - 32); } else { P.qt = 0; P.qsh = 0; } }
    P.fw = c->d_tw + ((size_t)i * 2 + 0) * N;
    P.iw = c->d_tw + ((size_t)i * 2 + 1) * N;
  }
  HB_CUDA(cudaMemcpy(c->d_tw, tw.data(), tw.size() * sizeof(ulonglong2), cudaMemcpyHostToDevice));
  HB_TRY(ctx_alloc(c, (void**)&c->d_primes, sizeof(HbPrimeDev) * nprimes));
  HB_CUDA(cudaMemcpy(c->d_primes, c->h_primes.data(), sizeof(HbPrimeDev) * nprimes, cudaMemcpyHostToDevice));
  HB_TRY(ctx_alloc(c, (void**)&c->d_stats, 4 * sizeof(u64)));
  HB_CUDA(cudaMemset(c->d_stats, 0, 4 * sizeof(u64)));
#ifndef HB_SIM
  HB_CUDA(cudaFuncSetAttribute(k_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c->max_smem + 1024));
  HB_CUDA(cudaFuncSetAttribute(k_fwd_blk, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k_inv_blk, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k2_fwd_blk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HB2_SMEM_BYTES));
  HB_CUDA(cudaFuncSetAttribute(k2_fwd_blk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HB2_SMEM_BYTES));
  HB_CUDA(cudaFuncSetAttribute(k2_inv_blk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HB2_SMEM_BYTES));
  HB_CUDA(cudaFuncSetAttribute(k2_inv_blk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HB2_SMEM_BYTES));
  HB_CUDA(cudaFuncSetAttribute(k1_conv1<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_conv1<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_conv<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_scaled_sums, cudaFuncAttributeMaxDynamicSharedMemorySize, HB_SSUM_SMEM));
  HB_CUDA(cudaFuncSetAttribute(k1_conv<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_fwd_blk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_fwd_blk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_inv_blk<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_inv_blk<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 80 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k1_fwd_blk_tensor<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)blk_parts_smem(4)));
  HB_CUDA(cudaFuncSetAttribute(k1_fwd_blk_tensor<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)blk_parts_smem(4)));
  HB_CUDA(cudaFuncSetAttribute(k1_fwd_blk_square<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)blk_parts_smem(2)));
  HB_CUDA(cudaFuncSetAttribute(k1_fwd_blk_square<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)blk_parts_smem(2)));
#endif
  *out = c;
  return HB_OK;
}

extern "C" void hb_ctx_destroy(hb_ctx* c) {
  if (!c) return;
  if (c->stream) cudaStreamSynchronize(c->stream);
  for (auto& kv : c->convs) { cudaFree(kv.second.blob); cudaFree(kv.second.d); }
  for (hb_poly* p : c->pool) { cudaFree(p->d); delete p; }
  cudaFree(c->pw.d_cube_to_poly); cudaFree(c->pw.d_short_to_long); cudaFree(c->pw.cube); cudaFree(c->pw.rows);
  cudaFree(c->d_frac); cudaFree(c->d_z); cudaFree(c->d_max); cudaFree(c->d_bcast);
  cudaFree(c->gen.d_rep); cudaFree(c->gen.d_irep); cudaFree(c->gen.d_gp); cudaFree(c->gen.d_primes_cyc); cudaFree(c->gen.d_primes_cyc2); cudaFree(c->gen.tab);
  cudaFree(c->gen.d_W);
  cudaFree(c->gen.w0); cudaFree(c->gen.w1); cudaFree(c->gen.wt); cudaFree(c->gen.cA); cudaFree(c->gen.cB);
  cudaFree(c->tmpA); cudaFree(c->tmpB); cudaFree(c->d_tw); cudaFree(c->d_primes); cudaFree(c->d_stats);
  cudaFree(c->prg_start); cudaFree(c->prg_off); cudaFree(c->prg_ticket);
  for (hb_poly* p : c->ks_a) { cudaFree(p->d); delete p; }
  for (hb_poly* p : c->bsgs) { cudaFree(p->d); delete p; }
  for (hb_poly* p : c->block) { cudaFree(p->d); delete p; }
  for (hb_poly* p : c->leaf) { cudaFree(p->d); delete p; }
  cudaFree(c->ssum);
  for (hb_poly* p : c->ip) { cudaFree(p->d); delete p; }
  for (HbTmap* sl : c->tmap_slabs) cudaFree(sl);
  if (c->own_stream) cudaStreamDestroy(c->own_stream);
  delete c;
}

extern "C" int hb_ctx_set_chain(hb_ctx* c, const int32_t* digit_of, int ndigits, const int32_t* special, int nspecial) {
  if (!c || !digit_of || ndigits < 0 || ndigits > HB_MAXDIG || nspecial < 0 || (nspecial && !special))
    return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_chain: bad argument (ndigits must be <= %d)", HB_MAXDIG);
  for (int i = 0; i < c->nprimes; i++) if (digit_of[i] < -1 || digit_of[i] >= ndigits) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_chain: digit_of[%d] out of range", i);
  for (int i = 0; i < nspecial; i++) if (special[i] < 0 || special[i] >= c->nprimes || digit_of[special[i]] != -1) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_chain: bad special prime index");
  c->digit_of.assign(digit_of, digit_of + c->nprimes); c->ndigits = ndigits;
  c->special.assign(special, special + nspecial);
  std::sort(c->special.begin(), c->special.end());
  return HB_OK;
}
extern "C" int hb_ctx_get_psi(hb_ctx* c, uint64_t* out) {
  if (!c || !out) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_get_psi: null");
  for (int i = 0; i < c->nprimes; i++) out[i] = c->psi[i];
  return HB_OK;
}
extern "C" int hb_ctx_sync(hb_ctx* c) {
  if (!c) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_sync: null");
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}
extern "C" int hb_ctx_stats(hb_ctx* c, uint64_t* out3) {
  if (!c || !out3) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_stats: null");
  HB_CUDA(cudaStreamSynchronize(c->stream));
  u64 s[4];
  HB_CUDA(cudaMemcpy(s, c->d_stats, sizeof(s), cudaMemcpyDeviceToHost));
  out3[0] = s[0]; out3[1] = c->launches; out3[2] = c->bytes;
  return HB_OK;
}
extern "C" int hb_ctx_reset_stats(hb_ctx* c) {
  if (!c) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_reset_stats: null");
  HB_CUDA(cudaMemsetAsync(c->d_stats, 0, 4 * sizeof(u64), c->stream));
  c->launches = 0;
  return HB_OK;
}
extern "C" int hb_ctx_mark_begin(hb_ctx* c) {
  if (!c) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_mark_begin: null");
#ifndef HB_SIM
  HB_CUDA(cudaEventRecord(c->ev0, c->stream));
#endif
  return HB_OK;
}
extern "C" int hb_ctx_mark_end(hb_ctx* c, float* ms) {
  if (!c || !ms) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_mark_end: null");
#ifndef HB_SIM
  HB_CUDA(cudaEventRecord(c->ev1, c->stream));
  HB_CUDA(cudaEventSynchronize(c->ev1));
  HB_CUDA(cudaEventElapsedTime(ms, c->ev0, c->ev1));
#else
  *ms = 0.f;
#endif
  return HB_OK;
}

// ------------------------------------------------------------------------------------------
// polys
extern "C" int hb_poly_create(hb_ctx* c, hb_poly** out) {
  if (!c || !out) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_create: null");
  hb_poly* p = new hb_poly();
  p->ctx = c; p->d = nullptr;
  size_t sz = (size_t)c->nprimes * c->N * sizeof(u64);
  int r = ctx_alloc(c, (void**)&p->d, sz);
  if (r != HB_OK) { delete p; return r; }
  cudaError_t e = cudaMemsetAsync(p->d, 0, sz, c->stream);
  if (e != cudaSuccess) { cudaFree(p->d); c->bytes -= sz; delete p; return hb_fail(HB_ERR_CUDA, "hb_poly_create: memset failed: %s", cudaGetErrorString(e)); }
  *out = p;
  return HB_OK;
}
extern "C" void hb_poly_destroy(hb_poly* p) {
  if (!p) return;
  cudaStreamSynchronize(p->ctx->stream);
  if (HbSeedSched* S = p->sched) {
    if (--S->refs == 0) { if (S->blk) { cudaFree(S->blk); p->ctx->bytes -= S->bytes; } delete S; }
    delete p;
    return;
  }
  if (p->owned) { p->ctx->bytes -= (size_t)p->ctx->nprimes * p->ctx->N * sizeof(u64); cudaFree(p->d); }
#ifndef HB_SIM
  if (p->ipc) cudaIpcCloseMemHandle(p->d);
#endif
  delete p;
}
static int check_idx(hb_ctx* c, const int32_t* idx, int n, const char* who, bool allow_empty = false) {
  if (n < 0 || (n > 0 && !idx) || (n == 0 && !allow_empty)) return hb_fail(HB_ERR_BAD_ARG, "%s: empty or null index list", who);
  for (int i = 0; i < n; i++) {
    if (idx[i] < 0 || idx[i] >= c->nprimes) return hb_fail(HB_ERR_BAD_ARG, "%s: prime index %d out of range", who, idx[i]);
    for (int j = 0; j < i; j++) if (idx[j] == idx[i]) return hb_fail(HB_ERR_BAD_ARG, "%s: duplicate prime index %d", who, idx[i]);
  }
  return HB_OK;
}
// allow_seeded: the evk_a lists of the key-switching entry points, which regenerate seeded entries before any kernel reads them
static int check_polys(hb_poly* const* p, int n, hb_ctx** c, const char* who, bool allow_seeded = false) {
  if (!p || n <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: no polynomials", who);
  for (int i = 0; i < n; i++) {
    if (!p[i]) return hb_fail(HB_ERR_BAD_ARG, "%s: null polynomial handle", who);
    if (p[i]->sched && !allow_seeded) return hb_fail(HB_ERR_BAD_ARG, "%s: a seeded polynomial has no rows (only evk_a and hb_poly_expand take one)", who);
    if (*c == nullptr) { *c = p[i]->ctx; g_chunk = (*c)->chunk; }
    if (p[i]->ctx != *c) return hb_fail(HB_ERR_INDEX_SET, "%s: incompatible objects (different contexts)", who);  // src/DoubleCRT.cpp:222-223
  }
  return HB_OK;
}
// single-poly calls that read or write p->d
static int check_dense(hb_poly* p, const char* who) {
  if (p->sched) return hb_fail(HB_ERR_BAD_ARG, "%s: a seeded polynomial has no rows (only evk_a and hb_poly_expand take one)", who);
  return HB_OK;
}
// rows <-> dense host matrix; runs of consecutive prime indices (the usual case: a prime set is an interval,
// src/Ctxt.cpp:177-186) travel as ONE copy -- the per-call cost of cudaMemcpyAsync otherwise dominates the host side
static int copy_rows(hb_ctx* c, u64* dev, u64* host, const int32_t* idx, int n, bool h2d) {
  for (int j = 0; j < n;) {
    int k = j + 1;
    while (k < n && idx[k] == idx[k - 1] + 1) k++;
    const size_t off = (size_t)idx[j] * c->N, bytes = (size_t)(k - j) * c->N * sizeof(u64);
    if (h2d) HB_CUDA(cudaMemcpyAsync(dev + off, host + off, bytes, cudaMemcpyHostToDevice, c->stream));
    else HB_CUDA(cudaMemcpyAsync(host + off, dev + off, bytes, cudaMemcpyDeviceToHost, c->stream));
    j = k;
  }
  return HB_OK;
}
extern "C" int hb_poly_upload(hb_poly* p, const int32_t* idx, int n, const uint64_t* host) {
  if (!p || !host) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_upload: null");
  HB_TRY(check_dense(p, "hb_poly_upload"));
  hb_ctx* c = p->ctx;
  HB_TRY(check_idx(c, idx, n, "hb_poly_upload"));
  return copy_rows(c, p->d, (u64*)host, idx, n, true);
}
extern "C" int hb_poly_download(hb_poly* p, const int32_t* idx, int n, uint64_t* host) {
  if (!p || !host) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_download: null");
  HB_TRY(check_dense(p, "hb_poly_download"));
  hb_ctx* c = p->ctx;
  HB_TRY(check_idx(c, idx, n, "hb_poly_download"));
  HB_TRY(copy_rows(c, p->d, (u64*)host, idx, n, false));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}
extern "C" int hb_poly_download_async(hb_poly* p, const int32_t* idx, int n, uint64_t* host) {
  if (!p || !host) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_download_async: null");
  HB_TRY(check_dense(p, "hb_poly_download_async"));
  hb_ctx* c = p->ctx;
  HB_TRY(check_idx(c, idx, n, "hb_poly_download_async"));
  HB_TRY(copy_rows(c, p->d, (u64*)host, idx, n, false));
  return HB_OK;
}
static int prof_collect(hb_ctx* c) {
#ifndef HB_SIM
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (auto& r : c->prof_pending) {
    float ms = 0.f;
    if (r.name) {
      cudaEventElapsedTime(&ms, r.a, r.b);
      bool found = false;
      for (auto& a : c->prof) if (a.name == r.name) { a.launches++; a.ms += ms; a.bytes += r.bytes; found = true; break; }
      if (!found) c->prof.push_back({r.name, 1, (double)ms, r.bytes});
    }
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  c->prof_pending.clear();
#endif
  return HB_OK;
}
extern "C" int hb_ctx_profile(hb_ctx* c, int enable) {
  if (!c) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_profile: null");
  HB_TRY(prof_collect(c));
  if (enable && !c->profiling) c->prof.clear();
  c->profiling = enable != 0;
  return HB_OK;
}
extern "C" int hb_ctx_profile_get(hb_ctx* c, int i, char* name, int namelen, uint64_t* launches, double* ms, uint64_t* bytes) {
  if (!c || !name || namelen <= 0) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_profile_get: null");
  HB_TRY(prof_collect(c));
  if (i < 0 || i >= (int)c->prof.size()) return HB_ERR_BAD_ARG;
  snprintf(name, namelen, "%s", c->prof[i].name.c_str());
  if (launches) *launches = c->prof[i].launches;
  if (ms) *ms = c->prof[i].ms;
  if (bytes) *bytes = c->prof[i].bytes;
  return HB_OK;
}
// ---- wire format (SURVEY 8f-3): DoubleCRT::writeTo / read (src/DoubleCRT.cpp:1530-1561) =
// IndexSet::writeTo (int64 card, int64 indices; src/IndexSet.cpp:288-297) followed, per row in index order, by
// write_ntl_vec_long (int32 length, int32 intSize = 8, then little-endian int64 values; src/binio.cpp:103-122).
extern "C" int hb_poly_serialized_size(hb_poly* p, int n, uint64_t* bytes) {
  if (!p || !bytes || n < 0) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_serialized_size: bad argument");
  HB_TRY(check_dense(p, "hb_poly_serialized_size"));
  *bytes = 8 + 8ULL * n + (uint64_t)n * (8 + 8ULL * p->ctx->N);
  return HB_OK;
}
extern "C" int hb_poly_serialize(hb_poly* p, const int32_t* idx, int n, void* buf, uint64_t buflen) {
  if (!p || !buf) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_serialize: null");
  HB_TRY(check_dense(p, "hb_poly_serialize"));
  hb_ctx* c = p->ctx;
  HB_TRY(check_idx(c, idx, n, "hb_poly_serialize", true));
  uint64_t need; hb_poly_serialized_size(p, n, &need);
  if (buflen < need) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_serialize: buffer of %llu bytes, need %llu", (unsigned long long)buflen, (unsigned long long)need);
  std::vector<int32_t> sorted(idx, idx + n); std::sort(sorted.begin(), sorted.end());   // IndexSet iterates in ascending order
  unsigned char* o = (unsigned char*)buf;
  int64_t card = n; memcpy(o, &card, 8); o += 8;
  for (int i = 0; i < n; i++) { int64_t v = sorted[i]; memcpy(o, &v, 8); o += 8; }
  for (int i = 0; i < n; i++) {
    int32_t len = (int32_t)c->N, isz = 8; memcpy(o, &len, 4); memcpy(o + 4, &isz, 4); o += 8;
    HB_CUDA(cudaMemcpyAsync(o, p->d + (size_t)sorted[i] * c->N, c->N * 8, cudaMemcpyDeviceToHost, c->stream));
    o += c->N * 8;
  }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}
// idx_out receives the index set (capacity nprimes), *n_out its size; rows are uploaded into p.
extern "C" int hb_poly_deserialize(hb_poly* p, const void* buf, uint64_t buflen, int32_t* idx_out, int* n_out) {
  if (!p || !buf || !idx_out || !n_out) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_deserialize: null");
  HB_TRY(check_dense(p, "hb_poly_deserialize"));
  hb_ctx* c = p->ctx;
  const unsigned char* o = (const unsigned char*)buf; const unsigned char* end = o + buflen;
  if (buflen < 8) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_deserialize: truncated");
  int64_t card; memcpy(&card, o, 8); o += 8;
  if (card < 0 || card > c->nprimes || o + 8 * card > end) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_deserialize: bad index-set size %lld", (long long)card);
  for (int64_t i = 0; i < card; i++) {
    int64_t v; memcpy(&v, o, 8); o += 8;
    if (v < 0 || v >= c->nprimes) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_deserialize: prime index %lld out of range", (long long)v);
    // IndexSet::writeTo emits the members in ascending order and the rows follow in that order (src/IndexSet.cpp, src/DoubleCRT.cpp:1530-1561):
    // anything else is not a DoubleCRT record
    if (i > 0 && (int32_t)v <= idx_out[i - 1]) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_deserialize: prime indices must be strictly ascending");
    idx_out[i] = (int32_t)v;
  }
  for (int64_t i = 0; i < card; i++) {
    if (o + 8 > end) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_deserialize: truncated row header");
    int32_t len, isz; memcpy(&len, o, 4); memcpy(&isz, o + 4, 4); o += 8;
    if (len != (int32_t)c->N) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_deserialize: row length %d, expected phi(m)=%zu", len, c->N);
    if (isz != 8 && isz != 4) return hb_fail(HB_ERR_BAD_ARG, "intSize must be 32 or 64 bit for binary IO");   // src/binio.cpp:107-109
    if (o + (size_t)len * isz > end) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_deserialize: truncated row");
    const u64 q = c->q[idx_out[i]];
    std::vector<u64> row(c->N);
    for (size_t k = 0; k < c->N; k++) {
      int64_t v;
      if (isz == 8) memcpy(&v, o + 8 * k, 8); else { int32_t w; memcpy(&w, o + 4 * k, 4); v = w; }
      if (v < 0 || (u64)v >= q) return hb_fail(HB_ERR_INDEX_SET, "DoubleCRT object has inconsistent data");   // DoubleCRT::verify, src/DoubleCRT.cpp:121-132
      row[k] = (u64)v;
    }
    o += (size_t)len * isz;
    HB_CUDA(cudaMemcpyAsync(p->d + (size_t)idx_out[i] * c->N, row.data(), c->N * 8, cudaMemcpyHostToDevice, c->stream));   // ordered with the context's stream
    HB_CUDA(cudaStreamSynchronize(c->stream));   // `row` is reused
  }
  *n_out = (int)card;
  return HB_OK;
}

// ---- seeded expansion: SetSeed(seed); for p in polys: p.randomize() over rows idx (src/DoubleCRT.cpp:1258-1378) =====
static int prg_grow(hb_ctx* c, void** p, size_t* cap, size_t bytes) {
  if (*cap >= bytes) return HB_OK;
  if (*p) { HB_CUDA(cudaFree(*p)); c->bytes -= *cap; *p = nullptr; *cap = 0; }   // cudaFree waits for the kernels using it
  HB_TRY(ctx_alloc(c, p, bytes));
  *cap = bytes;
  return HB_OK;
}
// candidate format and counting window of schedule row p*n + r (prime idx[r]); row pointers unset
static void prg_rows(hb_ctx* c, int npolys, const int32_t* idx, int n, std::vector<HbPrgRow>& rows, int* wmax) {
  rows.assign((size_t)npolys * n, HbPrgRow{});
  *wmax = 1;
  for (int r = 0; r < n; r++) {
    const u64 q = c->q[idx[r]];
    const int k = h_bitlen(q - 1), nb = (k + 7) / 8;
    const int w = c->prg_window ? c->prg_window : hb_prg_window(q, k, nb, c->N);
    *wmax = std::max(*wmax, w);
    for (int p = 0; p < npolys; p++) {
      HbPrgRow& R = rows[(size_t)p * n + r];
      R.q = q; R.mask = k >= 64 ? ~0ULL : (1ULL << k) - 1; R.nb = nb; R.window = w; R.row = nullptr;
    }
  }
}
// Step (a), the schedule: the chain of k_prg_count launches over rows[0..T).  start[0] = 0 (a fresh SetSeed); each launch
// reads its row's first buffer from device memory, writes the next row's and its buffers' row offsets at off + t*wstride.
static int prg_count_chain(hb_ctx* c, const HbPrgKey& key, const HbPrgRow* rows, int T, u64* start, unsigned* off, int wstride) {
  if (!c->prg_ticket) {
    HB_TRY(ctx_alloc(c, (void**)&c->prg_ticket, sizeof(unsigned long long)));
    HB_CUDA(cudaMemsetAsync(c->prg_ticket, 0, sizeof(unsigned long long), c->stream));
  }
  HB_CUDA(cudaMemsetAsync(start, 0, sizeof(u64), c->stream));
  HbPrgCountJob C;
  C.key = key; C.N = c->N; C.start = start; C.ticket = c->prg_ticket;
  for (int t = 0; t < T; t++) {
    C.r = rows[t]; C.t = t; C.off = off + (size_t)t * wstride;
    pre_launch(c);
    HB_LAUNCH(k_prg_count, dim3((unsigned)((C.r.window + HB_PRG_WARPS - 1) / HB_PRG_WARPS)), dim3(HB_PRG_THREADS), HB_PRG_SMEM_BYTES, c->stream, C);
    HB_TRY(post_launch(c, "k_prg_count", (u64)C.r.window * sizeof(unsigned) * 2));
  }
  return HB_OK;
}
// Step (b), the values: rows[i] (row pointer set) from schedule row sr[i], up to HB_PRG_MAXT rows per k_prg_fill launch
static int prg_fill(hb_ctx* c, const HbPrgKey& key, const u64* start, const unsigned* off, int wstride, const HbPrgRow* rows, const unsigned* sr, int T) {
  HbPrgFillJob F;
  F.key = key; F.N = c->N; F.start = start; F.off = off; F.wstride = wstride;
  for (int t0 = 0; t0 < T; t0 += HB_PRG_MAXT) {
    const int nt = std::min(HB_PRG_MAXT, T - t0);
    int wl = 1;
    for (int i = 0; i < nt; i++) { F.r[i] = rows[t0 + i]; F.sr[i] = sr[t0 + i]; wl = std::max(wl, F.r[i].window); }
    pre_launch(c);
    HB_LAUNCH(k_prg_fill, dim3((unsigned)((wl + HB_PRG_WARPS - 1) / HB_PRG_WARPS), (unsigned)nt), dim3(HB_PRG_THREADS), HB_PRG_SMEM_BYTES, c->stream, F);
    HB_TRY(post_launch(c, "k_prg_fill", (u64)nt * c->N * 8));
  }
  return HB_OK;
}
static int prg_args(hb_ctx* c, const int32_t* idx, int n, const uint8_t* seed, int seedlen, const char* who) {
  if (seedlen < 0 || (seedlen > 0 && !seed)) return hb_fail(HB_ERR_BAD_ARG, "%s: null seed with length %d", who, seedlen);
  HB_TRY(check_idx(c, idx, n, who, true));
  for (int i = 1; i < n; i++) if (idx[i] <= idx[i - 1]) return hb_fail(HB_ERR_BAD_ARG, "%s: prime indices must be strictly ascending", who);
  return HB_OK;
}
extern "C" int hb_poly_randomize(hb_poly* const* polys, int npolys, const int32_t* idx, int n, const uint8_t* seed, int seedlen) {
  static const char* who = "hb_poly_randomize";
  if (!polys || npolys <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: no polynomials", who);
  hb_ctx* c = nullptr;
  HB_TRY(check_polys(polys, npolys, &c, who));
  HB_TRY(prg_args(c, idx, n, seed, seedlen, who));
  if (n == 0) return HB_OK;
  const HbPrgKey key = hb_prg_derive_key(seed, seedlen);
  const int T = npolys * n;
  std::vector<HbPrgRow> rows;
  int wmax;
  prg_rows(c, npolys, idx, n, rows, &wmax);
  std::vector<unsigned> sr((size_t)T);
  for (int p = 0; p < npolys; p++)
    for (int r = 0; r < n; r++) { rows[(size_t)p * n + r].row = polys[p]->d + (size_t)idx[r] * c->N; sr[(size_t)p * n + r] = (unsigned)(p * n + r); }
  // the schedule lives in context scratch for this call only; every row is filled
  HB_TRY(prg_grow(c, (void**)&c->prg_start, &c->prg_start_cap, (size_t)(T + 1) * sizeof(u64)));
  HB_TRY(prg_grow(c, (void**)&c->prg_off, &c->prg_off_cap, (size_t)T * wmax * sizeof(unsigned)));
  HB_TRY(prg_count_chain(c, key, rows.data(), T, c->prg_start, c->prg_off, wmax));
  return prg_fill(c, key, c->prg_start, c->prg_off, wmax, rows.data(), sr.data(), T);
}

// The schedule's device storage for stride wmax: start[T+1], then off[T*wmax]
static int sched_alloc(hb_ctx* c, HbSeedSched* S) {
  const size_t T = S->rows.size();
  if (S->blk) { HB_CUDA(cudaFree(S->blk)); c->bytes -= S->bytes; S->blk = nullptr; }
  S->bytes = (T + 1) * sizeof(u64) + T * (size_t)S->wmax * sizeof(unsigned);
  HB_TRY(ctx_alloc(c, &S->blk, S->bytes));
  S->start = (u64*)S->blk;
  S->off = (unsigned*)(S->start + T + 1);
  return HB_OK;
}
static int sched_build(hb_ctx* c, HbSeedSched* S) {
  const int T = (int)S->rows.size();
  if (T == 0) return HB_OK;
  HB_TRY(sched_alloc(c, S));
  HB_TRY(prg_count_chain(c, S->key, S->rows.data(), T, S->start, S->off, S->wmax));
  // k_prg_count finishes a row that needs more buffers than its window on its slow path and records no offsets for the extra
  // buffers.  Each row's need is start[t+1] - start[t]: rows that outgrew their window are counted again with exactly that
  // window (the starts do not change), so every buffer of every row has its offset.
  std::vector<u64> st((size_t)T + 1);
  HB_CUDA(cudaMemcpyAsync(st.data(), S->start, st.size() * sizeof(u64), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  bool short_rows = false;
  for (int t = 0; t < T; t++) {
    const int need = (int)(st[(size_t)t + 1] - st[(size_t)t]);
    if (need > S->rows[(size_t)t].window) { S->rows[(size_t)t].window = need; S->wmax = std::max(S->wmax, need); short_rows = true; }
  }
  if (!short_rows) return HB_OK;
  HB_TRY(sched_alloc(c, S));
  return prg_count_chain(c, S->key, S->rows.data(), T, S->start, S->off, S->wmax);
}
extern "C" int hb_poly_create_seeded(hb_ctx* c, int npolys, const int32_t* idx, int n, const uint8_t* seed, int seedlen, hb_poly** out) {
  static const char* who = "hb_poly_create_seeded";
  if (!c || !out) return hb_fail(HB_ERR_BAD_ARG, "%s: null", who);
  if (npolys <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: no polynomials", who);
  HB_TRY(prg_args(c, idx, n, seed, seedlen, who));
  HbSeedSched* S = new HbSeedSched();
  S->key = hb_prg_derive_key(seed, seedlen);
  S->idx.assign(idx, idx + n);
  prg_rows(c, npolys, idx, n, S->rows, &S->wmax);
  const int rc = sched_build(c, S);
  if (rc != HB_OK) {
    cudaStreamSynchronize(c->stream);
    if (S->blk) { cudaFree(S->blk); c->bytes -= S->bytes; }
    delete S;
    return rc;
  }
  for (int p = 0; p < npolys; p++) {
    hb_poly* h = new hb_poly();
    h->ctx = c; h->d = nullptr; h->owned = false; h->sched = S; h->sched_poly = p;
    out[p] = h;
  }
  S->refs = npolys;
  return HB_OK;
}
// rows idx of seeded[p] into the rows of dst[p]: every row is checked against its set before anything is launched, then one
// k_prg_fill launch per schedule (one in practice: the a_i of a matrix share a seed)
static int prg_expand(hb_ctx* c, hb_poly* const* seeded, u64* const* dst, int np, const int32_t* idx, int n, const char* who) {
  std::vector<unsigned> srow((size_t)np * n);
  for (int p = 0; p < np; p++) {
    const HbSeedSched* S = seeded[p]->sched;
    const int ns = (int)S->idx.size();
    for (int r = 0; r < n; r++) {
      const auto it = std::lower_bound(S->idx.begin(), S->idx.end(), idx[r]);
      if (it == S->idx.end() || *it != idx[r]) return hb_fail(HB_ERR_INDEX_SET, "%s: row %d is not in the seeded set", who, idx[r]);
      srow[(size_t)p * n + r] = (unsigned)(seeded[p]->sched_poly * ns + (int)(it - S->idx.begin()));
    }
  }
  std::vector<char> done((size_t)np, 0);
  for (int p0 = 0; p0 < np; p0++) {
    if (done[(size_t)p0]) continue;
    const HbSeedSched* S = seeded[p0]->sched;
    std::vector<HbPrgRow> rows; std::vector<unsigned> sr;
    for (int p = p0; p < np; p++) {
      if (seeded[p]->sched != S) continue;
      done[(size_t)p] = 1;
      for (int r = 0; r < n; r++) {
        const unsigned s = srow[(size_t)p * n + r];
        HbPrgRow R = S->rows[s];
        R.row = dst[p] + (size_t)idx[r] * c->N;
        rows.push_back(R); sr.push_back(s);
      }
    }
    HB_TRY(prg_fill(c, S->key, S->start, S->off, S->wmax, rows.data(), sr.data(), (int)rows.size()));
  }
  return HB_OK;
}
extern "C" int hb_poly_expand(hb_poly* const* seeded, hb_poly* const* dst, int npolys, const int32_t* idx, int n) {
  static const char* who = "hb_poly_expand";
  if (!seeded || npolys <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: no polynomials", who);
  hb_ctx* c = nullptr;
  HB_TRY(check_polys(seeded, npolys, &c, who, true));
  for (int p = 0; p < npolys; p++) if (!seeded[p]->sched) return hb_fail(HB_ERR_BAD_ARG, "%s: seeded[%d] is not a seeded polynomial", who, p);
  HB_TRY(check_polys(dst, npolys, &c, who));
  HB_TRY(check_idx(c, idx, n, who, true));
  if (n == 0) return HB_OK;
  std::vector<u64*> d((size_t)npolys);
  for (int p = 0; p < npolys; p++) d[(size_t)p] = dst[p]->d;
  return prg_expand(c, seeded, d.data(), npolys, idx, n, who);
}
// The seeded entries of evk_a[0..nd): rows idx of each are regenerated into the context's key scratch (nd full-height polys,
// apart from the digit pool; allocated on first use, so a later call neither allocates nor synchronises and stays capturable
// in a CUDA graph).  `use` receives evk_a with those entries replaced.  The entry points call this once per call, before
// their item chunks.  hb_hoisted_linear_map calls it once per group of amounts, with at most HB_LINMAP_SEEDED entries
// (whole matrices), so the scratch holds at most max(HB_MAXDIG, HB_LINMAP_SEEDED) polys whatever the number of amounts.
#define HB_LINMAP_SEEDED (2 * HB_MAXDIG)
static int ks_expand_a(hb_ctx* c, hb_poly* const* evk_a, int nd, const int32_t* idx, int n, std::vector<hb_poly*>& use) {
  use.assign(evk_a, evk_a + nd);
  std::vector<hb_poly*> src; std::vector<u64*> dst;
  for (int i = 0; i < nd; i++) {
    if (!evk_a[i]->sched) continue;
    while ((int)c->ks_a.size() <= i) { hb_poly* p; HB_TRY(hb_poly_create(c, &p)); c->ks_a.push_back(p); }
    use[(size_t)i] = c->ks_a[(size_t)i];
    src.push_back(evk_a[i]); dst.push_back(c->ks_a[(size_t)i]->d);
  }
  if (src.empty()) return HB_OK;
  return prg_expand(c, src.data(), dst.data(), (int)src.size(), idx, n, "key switch (evk_a)");
}

static int pool_get(hb_ctx* c, int n, std::vector<hb_poly*>& out) {
  while ((int)c->pool.size() < n) { hb_poly* p; HB_TRY(hb_poly_create(c, &p)); c->pool.push_back(p); }
  out.assign(c->pool.begin(), c->pool.begin() + n);
  return HB_OK;
}

// ------------------------------------------------------------------------------------------
// launch helpers
static void fill_rows(HbRows& r, const int32_t* idx, int n) { r.n = n; for (int i = 0; i < n; i++) r.prime[i] = idx[i]; }
static int logwb_of(hb_ctx* c) { int n1 = c->logN - c->log_blk; return std::min(n1, 10 - c->log_blk); }
static int logw_cols(hb_ctx* c) { int n1 = c->logN - c->log_blk; int lw = 10 - n1; if (lw < 0) lw = 0; return std::min(lw, c->log_blk); }

static bool all_special(hb_ctx* c) { for (auto& P : c->h_primes) if (P.qt == 0) return false; return !getenv("HB_NO_SPECIAL"); }
static bool v1_blk_ok(hb_ctx* c) { return !c->force_v0 && c->log_blk == 8 && c->logN - 8 >= 4; }
static bool v1_cols_ok(hb_ctx* c) { return !c->force_v0 && c->log_blk == 8 && c->logN - 8 == 8; }
// number of item groups (gridDim.z): each CTA loops over ceil(nitems/z) items re-using its twiddles;
// pick z so the grid fills whole waves of resident CTAs with the fewest CTAs
static int pick_item_groups(hb_ctx* c, long ctas_per_item_group, int nitems) {
  int best = 1; double best_eff = -1;
  for (int z = 1; z <= nitems; z++) {
    long ctas = ctas_per_item_group * z;
    long waves = (ctas + c->resident_ctas - 1) / c->resident_ctas;
    int per = (nitems + z - 1) / z;
    double eff = (double)ctas / (double)(waves * c->resident_ctas) * ((double)nitems / (double)(per * z));
    if (eff > best_eff + 0.02) { best_eff = eff; best = z; }
  }
  return best;
}
static int launch_blk_v1(hb_ctx* c, int dir, const u64* const* src, u64* const* dst, int nitems, const int32_t* idx, int n,
                         int epi, const u64* scal, int lazy = 0, u64* const* dst2 = nullptr) {
  const int n1 = c->logN - 8;
  const size_t smem = (2 * HB1_STAGE + (dir > 0 ? 16 * 256 : 0)) * sizeof(u64) + 256 * sizeof(ulonglong2);
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    int nr = std::min(HB_MAXROWS, n - r0);
    Hb1BlkJob J; memset(&J, 0, sizeof(J));
    J.logN = c->logN; J.epi = epi; J.lazy = lazy;
    if (dir < 0) J.epi = v1_cols_ok(c) ? 2 : 0;   // inverse: the next phase is a register kernel (cols or fused conversion) -> lazy values may stay
    fill_rows(J.rows, idx + r0, nr);
    for (int i = 0; i < nr; i++) if (scal) { J.scal[i] = scal[r0 + i]; J.scal_s[i] = h_shoup(scal[r0 + i], c->q[idx[r0 + i]]); }
    J.nitems = nitems;
    for (int i = 0; i < nitems; i++) { J.src[i] = src[i]; J.dst[i] = dst[i]; if (dst2) J.dst2[i] = dst2[i]; }
    long units = (long)nr * nitems << (n1 - 4);
    dim3 grid((unsigned)std::min<long>(units, c->resident_ctas));   // persistent CTAs, balanced contiguous chunks
    pre_launch(c);
    const bool sp = all_special(c);
    if (dir > 0) { if (sp) HB_LAUNCH(k1_fwd_blk<true>, grid, dim3(256), smem, c->stream, c->d_primes, J); else HB_LAUNCH(k1_fwd_blk<false>, grid, dim3(256), smem, c->stream, c->d_primes, J); HB_TRY(post_launch(c, epi == 1 ? "k1_fwd_blk_subscale" : (epi == 3 ? "k1_fwd_blk_digits" : "k1_fwd_blk"), (u64)(epi == 1 ? 3 : 2) * nr * nitems * c->N * 8)); }
    else { if (sp) HB_LAUNCH(k1_inv_blk<true>, grid, dim3(256), smem, c->stream, c->d_primes, J); else HB_LAUNCH(k1_inv_blk<false>, grid, dim3(256), smem, c->stream, c->d_primes, J); HB_TRY(post_launch(c, "k1_inv_blk", (u64)2 * nr * nitems * c->N * 8)); }
  }
  return HB_OK;
}
// The rescale of nitems items' parts fused with their product (src / dst: nparts per item): k1_fwd_blk_tensor for nparts 4
// (a0 a1 b0 b1 of an operand pair), k1_fwd_blk_square for nparts 2 (a0 a1 of a ciphertext, its a1^2 into o2[item])
static int launch_blk_parts_v1(hb_ctx* c, int nparts, const u64* const* src, u64* const* dst, u64* const* o2, int nitems,
                               const int32_t* idx, int n, const u64* scal) {
  const int n1 = c->logN - 8;
  const bool sq = nparts == 2;
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    int nr = std::min(HB_MAXROWS, n - r0);
    Hb1BlkJob J; memset(&J, 0, sizeof(J));
    J.logN = c->logN; J.epi = 1; J.lazy = 1;
    fill_rows(J.rows, idx + r0, nr);
    for (int i = 0; i < nr; i++) { J.scal[i] = scal[r0 + i]; J.scal_s[i] = h_shoup(scal[r0 + i], c->q[idx[r0 + i]]); }
    J.nitems = nitems;
    for (int i = 0; i < nparts * nitems; i++) { J.src[i] = src[i]; J.dst[i] = dst[i]; }
    if (sq) for (int i = 0; i < nitems; i++) J.dst2[i] = o2[i];
    long units = (long)nr * nitems << (n1 - 4);
    dim3 grid((unsigned)std::min<long>(units, std::max(1, c->resident_ctas / 2)));   // persistent CTAs, one per SM
    const size_t smem = blk_parts_smem(nparts);
    pre_launch(c);
    const bool sp = all_special(c);
    if (sq) { if (sp) HB_LAUNCH(k1_fwd_blk_square<true>, grid, dim3(256), smem, c->stream, c->d_primes, J); else HB_LAUNCH(k1_fwd_blk_square<false>, grid, dim3(256), smem, c->stream, c->d_primes, J); }
    else { if (sp) HB_LAUNCH(k1_fwd_blk_tensor<true>, grid, dim3(256), smem, c->stream, c->d_primes, J); else HB_LAUNCH(k1_fwd_blk_tensor<false>, grid, dim3(256), smem, c->stream, c->d_primes, J); }
    // tensor: 4 tiles + 4 old rows read, 4 rows written; square: 2 tiles + 2 old rows read, 3 rows written
    HB_TRY(post_launch(c, sq ? "k1_fwd_blk_square" : "k1_fwd_blk_tensor", (u64)(sq ? 7 : 12) * nr * nitems * c->N * 8));
  }
  return HB_OK;
}

// ---- tensor maps for the TMA-staged blk kernels ------------------------------------------------
// Two tiled views per [nprimes][N] matrix (hb_device_v2.cuh): BLK {256, G, 16, nprimes} box {256,1,16,1} and
// NAT {N1, 256, nprimes} box {16,256,1} with SWIZZLE_128B.  Encoded on the host once per (buffer, logN), kept in device memory.
#define HB_TMAP_SLAB 512   // matrices per slab
#ifndef HB_SIM
typedef CUresult (*hb_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                       const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                       CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static hb_encode_tiled_fn hb_encode_tiled() {
  static hb_encode_tiled_fn fn = [] {
    void* p = nullptr; cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) p = nullptr;
    return (hb_encode_tiled_fn)p;
  }();
  return fn;
}
#endif
static bool v2_blk_ok(hb_ctx* c) {
  if (!c->blk_v2 || c->force_v0 || c->log_blk != 8 || c->logN - 8 < 4) return false;
#ifndef HB_SIM
  if (!hb_encode_tiled()) return false;
#endif
  return true;
}
static int get_tmaps(hb_ctx* c, const u64* base, const HbTmap** out) {
  hb_ctx::TmapKey key{base, c->logN};
  auto it = c->tmaps.find(key);
  if (it != c->tmaps.end()) { *out = it->second; return HB_OK; }
  if (c->tmap_slabs.empty() || c->tmap_used == HB_TMAP_SLAB) {
    HbTmap* sl = nullptr;
    HB_TRY(ctx_alloc(c, (void**)&sl, sizeof(HbTmap) * 2 * HB_TMAP_SLAB));
    c->tmap_slabs.push_back(sl); c->tmap_used = 0;
  }
  HbTmap* d = c->tmap_slabs.back() + 2 * c->tmap_used++;
  const int n1 = c->logN - 8;
  const u64 N = (u64)1 << c->logN, N1 = (u64)1 << n1, G = (u64)1 << (n1 - 4);
  HbTmap h[2];
#ifdef HB_SIM
  memset(h, 0, sizeof(h));
  h[0].base = (u64*)base; h[0].rank = 4; h[0].swz128 = 0;
  h[0].dim[0] = 256; h[0].dim[1] = G; h[0].dim[2] = 16; h[0].dim[3] = c->nprimes;
  h[0].stride[0] = 1; h[0].stride[1] = 256; h[0].stride[2] = 256 * G; h[0].stride[3] = N;
  h[0].box[0] = 256; h[0].box[1] = 1; h[0].box[2] = 16; h[0].box[3] = 1;
  h[1].base = (u64*)base; h[1].rank = 3; h[1].swz128 = 1;
  h[1].dim[0] = N1; h[1].dim[1] = 256; h[1].dim[2] = c->nprimes;
  h[1].stride[0] = 1; h[1].stride[1] = N1; h[1].stride[2] = N;
  h[1].box[0] = 16; h[1].box[1] = 256; h[1].box[2] = 1;
#else
  const cuuint32_t ones[4] = {1, 1, 1, 1};
  {
    const cuuint64_t dim[4] = {256, G, 16, (cuuint64_t)c->nprimes};
    const cuuint64_t str[3] = {256 * 8, 256 * 8 * G, N * 8};
    const cuuint32_t box[4] = {256, 1, 16, 1};
    CUresult r = hb_encode_tiled()(&h[0], CU_TENSOR_MAP_DATA_TYPE_UINT64, 4, (void*)base, dim, str, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return hb_fail(HB_ERR_CUDA, "cuTensorMapEncodeTiled(BLK view) failed: %d", (int)r);
  }
  {
    const cuuint64_t dim[3] = {N1, 256, (cuuint64_t)c->nprimes};
    const cuuint64_t str[2] = {N1 * 8, N * 8};
    const cuuint32_t box[3] = {16, 256, 1};
    CUresult r = hb_encode_tiled()(&h[1], CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, (void*)base, dim, str, box, ones, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return hb_fail(HB_ERR_CUDA, "cuTensorMapEncodeTiled(NAT view) failed: %d", (int)r);
  }
#endif
  HB_CUDA(cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice));   // once per buffer
  c->tmaps[key] = d;
  *out = d;
  return HB_OK;
}
static int launch_blk_v2(hb_ctx* c, int dir, const u64* const* src, u64* const* dst, int nitems, const int32_t* idx, int n,
                         int epi, const u64* scal, int lazy, u64* const* dst2) {
  const int n1 = c->logN - 8;
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    int nr = std::min(HB_MAXROWS, n - r0);
    Hb2BlkJob J; memset(&J, 0, sizeof(J));
    J.logN = c->logN; J.epi = epi; J.lazy = lazy;
    if (dir < 0) J.epi = v1_cols_ok(c) ? 2 : 0;   // inverse: the next phase is a register kernel (cols or fused conversion) -> lazy values may stay
    fill_rows(J.rows, idx + r0, nr);
    for (int i = 0; i < nr; i++) if (scal) { J.scal[i] = scal[r0 + i]; J.scal_s[i] = h_shoup(scal[r0 + i], c->q[idx[r0 + i]]); }
    J.nitems = nitems;
    for (int i = 0; i < nitems; i++) {
      const HbTmap *ms, *md, *m2;
      HB_TRY(get_tmaps(c, src[i], &ms)); HB_TRY(get_tmaps(c, dst[i], &md));
      J.src[i] = ms + (dir > 0 ? 0 : 1); J.dst[i] = md + (dir > 0 ? 1 : 0);
      if (dst2) { HB_TRY(get_tmaps(c, dst2[i], &m2)); J.dst2[i] = m2 + 1; }
      J.dstp[i] = dst[i];
    }
    long units = (long)nr * nitems << (n1 - 4);
    dim3 grid((unsigned)std::min<long>((units + 1) / 2, std::max(1, c->resident_ctas / 2)));   // one persistent CTA (two teams) per SM
    pre_launch(c);
    const bool sp = all_special(c);
    if (dir > 0) { if (sp) HB_LAUNCH(k2_fwd_blk<true>, grid, dim3(HB2_THREADS), HB2_SMEM_BYTES, c->stream, c->d_primes, J); else HB_LAUNCH(k2_fwd_blk<false>, grid, dim3(HB2_THREADS), HB2_SMEM_BYTES, c->stream, c->d_primes, J); HB_TRY(post_launch(c, epi == 1 ? "k2_fwd_blk_subscale" : (epi == 3 ? "k2_fwd_blk_digits" : "k2_fwd_blk"), (u64)(epi == 1 ? 3 : 2) * nr * nitems * c->N * 8)); }
    else { if (sp) HB_LAUNCH(k2_inv_blk<true>, grid, dim3(HB2_THREADS), HB2_SMEM_BYTES, c->stream, c->d_primes, J); else HB_LAUNCH(k2_inv_blk<false>, grid, dim3(HB2_THREADS), HB2_SMEM_BYTES, c->stream, c->d_primes, J); HB_TRY(post_launch(c, "k2_inv_blk", (u64)2 * nr * nitems * c->N * 8)); }
  }
  return HB_OK;
}
// scal (inverse only, optional): per-row factor that replaces N^-1 (the caller folds N^-1 in); peers / npeers: extra destinations
static int launch_cols_v1(hb_ctx* c, int dir, const u64* const* src, u64* const* dst, int nitems, const int32_t* idx, int n,
                          const u64* scal = nullptr, u64* const* const* peers = nullptr, int npeers = 0) {
  const size_t smem = (16 * HB1_BS + 8) * sizeof(u64);
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    int nr = std::min(HB_MAXROWS, n - r0);
    Hb1ColsJob J; memset(&J, 0, sizeof(J));
    J.logN = c->logN;
    fill_rows(J.rows, idx + r0, nr);
    J.nitems = nitems;
    for (int i = 0; i < nitems; i++) { J.src[i] = src[i]; J.dst[i] = dst[i]; }
    if (scal) { J.has_scal = 1; for (int i = 0; i < nr; i++) { J.scal[i] = scal[r0 + i]; J.scal_s[i] = h_shoup(scal[r0 + i], c->q[idx[r0 + i]]); } }
    J.npeers = npeers;
    for (int p = 0; p < npeers; p++) for (int i = 0; i < nitems; i++) J.peer[p][i] = peers[p][i];
    dim3 grid(16, nr, pick_item_groups(c, 16L * nr, nitems));
    pre_launch(c);
    const bool sp = all_special(c);
    if (dir > 0) { if (sp) HB_LAUNCH(k1_fwd_cols<true>, grid, dim3(256), smem, c->stream, c->d_primes, J); else HB_LAUNCH(k1_fwd_cols<false>, grid, dim3(256), smem, c->stream, c->d_primes, J); HB_TRY(post_launch(c, "k1_fwd_cols", (u64)2 * nr * nitems * c->N * 8)); }
    else { if (sp) HB_LAUNCH(k1_inv_cols<true>, grid, dim3(256), smem, c->stream, c->d_primes, J); else HB_LAUNCH(k1_inv_cols<false>, grid, dim3(256), smem, c->stream, c->d_primes, J); HB_TRY(post_launch(c, npeers ? "k1_inv_cols_bcast" : "k1_inv_cols", (u64)(2 + npeers) * nr * nitems * c->N * 8)); }
  }
  return HB_OK;
}

// direction: +1 forward blk (src -> dst, optional epilogue), -1 inverse blk
static int launch_blk(hb_ctx* c, int dir, const u64* const* src, u64* const* dst, int nitems, const int32_t* idx, int n,
                      int epi, const u64* scal, int lazy = 0, u64* const* dst2 = nullptr) {
  // on an H100 SXM (80 GB HBM3, 400 W limit) the cp.async kernels are ahead of the TMA-staged ones in both directions: 5.30 against
  // 6.06 ms per forward mod-down launch, 1.67 against 2.01 ms inverse, 1 600 against 1 515 mult/s (bench.py, alternated in one run),
  // so the k2 kernels run only when HB_BLK_V2=1 selects them
  if (v2_blk_ok(c)) return launch_blk_v2(c, dir, src, dst, nitems, idx, n, epi, scal, lazy, dst2);
  if (v1_blk_ok(c)) return launch_blk_v1(c, dir, src, dst, nitems, idx, n, epi, scal, lazy, dst2);
  if (lazy || dst2 || epi == 3) return hb_fail(HB_ERR_UNSUPPORTED, "lazy / dual-epilogue blk phase needs the register kernels");
  const int lwb = logwb_of(c);
  const int n1 = c->logN - c->log_blk;
  const size_t smem = ((size_t)1 << lwb) * (((size_t)1 << c->log_blk) + 1) * sizeof(u64);
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    int nr = std::min(HB_MAXROWS, n - r0);
    HbBlkJob J; memset(&J, 0, sizeof(J));
    J.logN = c->logN; J.log_blk = c->log_blk; J.logwb = lwb; J.epi = epi;
    fill_rows(J.rows, idx + r0, nr);
    for (int i = 0; i < nr; i++) if (scal) { J.scal[i] = scal[r0 + i]; J.scal_s[i] = h_shoup(scal[r0 + i], c->q[idx[r0 + i]]); }
    J.nitems = nitems;
    for (int i = 0; i < nitems; i++) { J.src[i] = src[i]; J.dst[i] = dst[i]; }
    dim3 grid(1u << (n1 - lwb), nr, nitems);
    pre_launch(c);
    if (dir > 0) { HB_LAUNCH(k_fwd_blk, grid, dim3(HB_THREADS), smem, c->stream, c->d_primes, J); HB_TRY(post_launch(c, epi ? "k_fwd_blk_subscale" : "k_fwd_blk", (u64)(epi ? 3 : 2) * nr * nitems * c->N * 8)); }
    else { HB_LAUNCH(k_inv_blk, grid, dim3(HB_THREADS), smem, c->stream, c->d_primes, J); HB_TRY(post_launch(c, "k_inv_blk", (u64)2 * nr * nitems * c->N * 8)); }
  }
  return HB_OK;
}
static int launch_cols(hb_ctx* c, int dir, const u64* const* src, u64* const* dst, int nitems, const int32_t* idx, int n) {
  if (v1_cols_ok(c)) return launch_cols_v1(c, dir, src, dst, nitems, idx, n);
  const int lw = logw_cols(c);
  const int n1 = c->logN - c->log_blk;
  const size_t smem = ((size_t)1 << (n1 + lw)) * sizeof(u64);
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    int nr = std::min(HB_MAXROWS, n - r0);
    HbColsJob J; memset(&J, 0, sizeof(J));
    J.logN = c->logN; J.log_blk = c->log_blk; J.logw = lw;
    fill_rows(J.rows, idx + r0, nr);
    J.nitems = nitems;
    for (int i = 0; i < nitems; i++) { J.src[i] = src[i]; J.dst[i] = dst[i]; }
    dim3 grid(1u << (c->log_blk - lw), nr, nitems);
    pre_launch(c);
    if (dir > 0) { HB_LAUNCH(k_fwd_cols, grid, dim3(HB_THREADS), smem, c->stream, c->d_primes, J); HB_TRY(post_launch(c, "k_fwd_cols", (u64)2 * nr * nitems * c->N * 8)); }
    else { HB_LAUNCH(k_inv_cols, grid, dim3(HB_THREADS), smem, c->stream, c->d_primes, J); HB_TRY(post_launch(c, "k_inv_cols", (u64)2 * nr * nitems * c->N * 8)); }
  }
  return HB_OK;
}

struct PwArgs {
  int op;
  u64* const* dst; u64* const* dst1; u64* const* dst2;
  const u64* const* a; const u64* const* b; const u64* const* cc; const u64* const* d;
  const u64* scal; u64 k, m;
};
static int launch_pw(hb_ctx* c, const PwArgs& A, int nitems, const int32_t* idx, int n) {
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    int nr = std::min(HB_MAXROWS, n - r0);
    HbPwJob J; memset(&J, 0, sizeof(J));
    J.op = A.op; J.logN = c->logN; J.N = c->N; J.k = A.k; J.m = A.m;
    fill_rows(J.rows, idx + r0, nr);
    for (int i = 0; i < nr; i++) if (A.scal) { J.scal[i] = A.scal[r0 + i]; J.scal_s[i] = h_shoup(A.scal[r0 + i], c->q[idx[r0 + i]]); }
    J.nitems = nitems;
    for (int i = 0; i < nitems; i++) {
      J.dst[i] = A.dst[i];
      if (A.dst1) J.dst1[i] = A.dst1[i];
      if (A.dst2) J.dst2[i] = A.dst2[i];
      if (A.a) J.a[i] = A.a[i];
      if (A.b) J.b[i] = A.b[i];
      if (A.cc) J.c[i] = A.cc[i];
      if (A.d) J.d[i] = A.d[i];
    }
    unsigned gx = (unsigned)std::max<size_t>(1, c->N / (HB_THREADS * 4));
    dim3 grid(gx, nr, nitems);
    static const int rw[] = {3, 3, 3, 2, 2, 3, 1, 2, 7, 2, 4};  // rows moved per element, by op
    static const char* nm[] = {"k_pw_add", "k_pw_sub", "k_pw_mul", "k_pw_neg", "k_pw_scale", "k_pw_subscale", "k_pw_zero", "k_pw_copy", "k_pw_tensor", "k_pw_automorph", "k_pw_muladd"};
    pre_launch(c);
    HB_LAUNCH(k_pointwise, grid, dim3(HB_THREADS), 0, c->stream, c->d_primes, J);
    HB_TRY(post_launch(c, nm[A.op], (u64)rw[A.op] * nr * nitems * c->N * 8));
  }
  return HB_OK;
}

// run f(item0, count) over chunks of at most `chunk` (<= HB_MAXB) items
template <class F> static int for_items(int nitems, F f) {
  for (int i0 = 0; i0 < nitems; i0 += g_chunk) HB_TRY(f(i0, std::min(g_chunk, nitems - i0)));
  return HB_OK;
}
static void ptrs_of(hb_poly* const* p, int i0, int n, u64** out) { for (int i = 0; i < n; i++) out[i] = p[i0 + i]->d; }
static void tmp_ptrs(hb_ctx* c, u64* base, int n, u64** out) { for (int i = 0; i < n; i++) out[i] = base + (size_t)i * c->nprimes * c->N; }

// ------------------------------------------------------------------------------------------
// conversion tables
static std::string conv_key(const int32_t* src, int n, const int32_t* tgt, int nt, u64 p) {
  std::string k;
  for (int i = 0; i < n; i++) k += std::to_string(src[i]) + ",";
  k += "|";
  for (int i = 0; i < nt; i++) k += std::to_string(tgt[i]) + ",";
  k += "|" + std::to_string(p);
  return k;
}
static void limbs_mul_small(std::vector<u64>& a, u64 s) {
  u128 carry = 0;
  for (size_t i = 0; i < a.size(); i++) { carry += (u128)a[i] * s; a[i] = (u64)carry; carry >>= 64; }
}
static int get_conv(hb_ctx* c, const int32_t* src, int n, const int32_t* tgt, int nt, u64 p, ConvEntry** out) {
  std::string key = conv_key(src, n, tgt, nt, p);
  auto it = c->convs.find(key);
  if (it != c->convs.end()) { *out = &it->second; return HB_OK; }
  if (n > HB_MAXROWS || n > HB_MAXL) return hb_fail(HB_ERR_UNSUPPORTED, "base conversion from %d source primes (max %d)", n, HB_MAXROWS);
  const int L = n;
  std::vector<u64> qs(n);
  for (int j = 0; j < n; j++) qs[j] = c->q[src[j]];
  auto prod_mod_excl = [&](int excl, u64 M) { u64 r = 1 % M; for (int k = 0; k < n; k++) if (k != excl) r = h_mulmod(r, qs[k] % M, M); return r; };
  std::vector<int> h_src(src, src + n), h_tgt(std::max(nt, 1), 0), fshift(n);
  for (int i = 0; i < nt; i++) h_tgt[i] = tgt[i];
  std::vector<u64> t(n), t_s(n), tn(n), tn_s(n), fmul(n), cmat(std::max<size_t>((size_t)nt * n, 1)), negQ(std::max(nt, 1)), Qmod(std::max(nt, 1)), cp(n);
  std::vector<u64> Q(L, 0), Qhalf(L), Qj((size_t)n * L, 0);
  for (int j = 0; j < n; j++) {
    u64 qj = qs[j];
    u64 r = prod_mod_excl(j, qj);
    t[j] = h_powmod(r, qj - 2, qj); t_s[j] = h_shoup(t[j], qj);
    tn[j] = h_mulmod(t[j], c->h_primes[src[j]].ninv, qj); tn_s[j] = h_shoup(tn[j], qj);
    int b = h_bitlen(qj);
    fmul[j] = (u64)(((u128)1 << (63 + b)) / qj);
    fshift[j] = b - 1;
    std::vector<u64> lj(L, 0); lj[0] = 1;
    for (int k = 0; k < n; k++) if (k != j) limbs_mul_small(lj, qs[k]);
    memcpy(&Qj[(size_t)j * L], lj.data(), sizeof(u64) * L);
  }
  Q[0] = 1; for (int k = 0; k < n; k++) limbs_mul_small(Q, qs[k]);
  { // Qhalf = (Q-1)/2  (Q odd)
    std::vector<u64> h = Q; h[0] -= 1;
    for (int l = 0; l < L; l++) Qhalf[l] = (h[l] >> 1) | (l + 1 < L ? h[l + 1] << 63 : 0);
  }
  for (int tt = 0; tt < nt; tt++) {
    u64 qt = c->q[tgt[tt]];
    for (int j = 0; j < n; j++) cmat[(size_t)tt * n + j] = prod_mod_excl(j, qt);
    u64 Qm = prod_mod_excl(-1, qt);
    Qmod[tt] = Qm; negQ[tt] = Qm ? qt - Qm : 0;
  }
  ConvEntry E; memset(&E, 0, sizeof(E));
  HbConvDev& H = E.h;
  H.n = n; H.nt = nt; H.L = L; H.has_p = p > 1 ? 1 : 0;
  if (p > 1) {
    if (p >= (1ULL << 62)) return hb_fail(HB_ERR_UNSUPPORTED, "ptxt_space >= 2^62");
    u64 Qp = prod_mod_excl(-1, p), Qinv;
    if (!h_invmod(Qp, p, &Qinv)) return hb_fail(HB_ERR_BAD_ARG, "ptxt_space %llu is not coprime to the dropped primes", (unsigned long long)p);
    H.p = p; H.p_c64 = (u64)(((u128)1 << 64) % p); H.p_c64_s = h_shoup(H.p_c64, p); H.p_one_s = (u64)(((u128)1 << 64) / p);
    H.Qinv_p = Qinv; H.Qinv_p_s = h_shoup(Qinv, p);
    H.negQ_p = Qp ? p - Qp : 0;
    for (int j = 0; j < n; j++) cp[j] = prod_mod_excl(j, p);
  }
  // pack into one blob
  std::vector<unsigned char> blob;
  auto put = [&](const void* src_, size_t bytes) { size_t off = (blob.size() + 15) & ~(size_t)15; blob.resize(off + bytes); memcpy(&blob[off], src_, bytes); return off; };
  size_t o_src = put(h_src.data(), sizeof(int) * n), o_tgt = put(h_tgt.data(), sizeof(int) * std::max(nt, 1));
  size_t o_fs = put(fshift.data(), sizeof(int) * n);
  size_t o_t = put(t.data(), 8 * n), o_ts = put(t_s.data(), 8 * n), o_tn = put(tn.data(), 8 * n), o_tns = put(tn_s.data(), 8 * n);
  size_t o_fm = put(fmul.data(), 8 * n), o_c = put(cmat.data(), 8 * std::max<size_t>(cmat.size(), 1));
  size_t o_nq = put(negQ.data(), 8 * std::max(nt, 1)), o_qm = put(Qmod.data(), 8 * std::max(nt, 1)), o_cp = put(cp.data(), 8 * n);
  size_t o_Q = put(Q.data(), 8 * L), o_Qh = put(Qhalf.data(), 8 * L), o_Qj = put(Qj.data(), 8 * (size_t)n * L);
  HB_TRY(ctx_alloc(c, &E.blob, blob.size()));
  HB_CUDA(cudaMemcpy(E.blob, blob.data(), blob.size(), cudaMemcpyHostToDevice));
  unsigned char* B = (unsigned char*)E.blob;
  H.src_prime = (const int*)(B + o_src); H.tgt_prime = (const int*)(B + o_tgt); H.fshift = (const int*)(B + o_fs);
  E.d_t = (const u64*)(B + o_t); E.d_t_s = (const u64*)(B + o_ts);
  H.tn = (const u64*)(B + o_tn); H.tn_s = (const u64*)(B + o_tns); H.fmul = (const u64*)(B + o_fm);
  H.c = (const u64*)(B + o_c); H.negQ = (const u64*)(B + o_nq); H.Qmod = (const u64*)(B + o_qm); H.cp = (const u64*)(B + o_cp);
  H.Q = (const u64*)(B + o_Q); H.Qhalf = (const u64*)(B + o_Qh); H.Qj = (const u64*)(B + o_Qj);
  HB_TRY(ctx_alloc(c, (void**)&E.d, sizeof(HbConvDev)));
  HB_CUDA(cudaMemcpy(E.d, &H, sizeof(HbConvDev), cudaMemcpyHostToDevice));
  auto ins = c->convs.emplace(key, E);
  *out = &ins.first->second;
  return HB_OK;
}

// inverse-blk (polys -> tmpA), fused conversion (tmpA -> tmpB), for one chunk of items.
// src_is_y: polys already hold the y_j coefficient rows (prime-sharded path): no inverse phase at all.
static int norm_scratch(hb_ctx* c) {
  if (c->d_frac) return HB_OK;
  HB_TRY(ctx_alloc(c, (void**)&c->d_frac, (size_t)HB_MAXB * c->N * sizeof(double)));
  HB_TRY(ctx_alloc(c, (void**)&c->d_z, (size_t)HB_MAXB * c->N * 2 * sizeof(double)));
  HB_TRY(ctx_alloc(c, (void**)&c->d_max, HB_MAXB * sizeof(unsigned long long)));
  return HB_OK;
}
// max_j |f(zeta^(2j+1))| of the nit fraction polynomials in c->d_frac -> out[0..nit)   (synchronises)
static int norm_chunk(hb_ctx* c, int nit, double* out) {
  HbNormJob J; J.logN = c->logN; J.npoly = nit; J.frac = c->d_frac; J.z = (double2*)c->d_z; J.maxbits = c->d_max;
  HB_CUDA(cudaMemsetAsync(c->d_max, 0, nit * sizeof(unsigned long long), c->stream));
  unsigned gx = (unsigned)std::max<size_t>(1, c->N / (HB_THREADS * 4));
  pre_launch(c);
  HB_LAUNCH(k_norm_twist, dim3(gx, nit), dim3(HB_THREADS), 0, c->stream, J);
  HB_TRY(post_launch(c, "k_norm_twist", (u64)nit * c->N * 24));
  for (int logd = c->logN - 1; logd >= 0; logd--) {
    pre_launch(c);
    HB_LAUNCH(k_norm_stage, dim3(gx, nit), dim3(HB_THREADS), 0, c->stream, J, logd, logd == 0 ? 1 : 0);
    HB_TRY(post_launch(c, "k_norm_stage", (u64)nit * c->N * 32));
  }
  unsigned long long bits[HB_MAXB];
  HB_CUDA(cudaMemcpyAsync(bits, c->d_max, nit * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < nit; i++) { double m2; memcpy(&m2, &bits[i], 8); out[i] = std::sqrt(m2); }
  return HB_OK;
}
static int conv_chunk(hb_ctx* c, u64* const* polys, int nit, const int32_t* src, int n, const int32_t* tgt, int nt, u64 p, int src_is_y = 0, bool want_frac = false) {
  HB_TRY(ctx_scratch(c));
  if (want_frac) HB_TRY(norm_scratch(c));
  ConvEntry* E; HB_TRY(get_conv(c, src, n, tgt, nt, p, &E));
  u64* tA[HB_MAXB]; u64* tB[HB_MAXB];
  tmp_ptrs(c, c->tmpA, nit, tA); tmp_ptrs(c, c->tmpB, nit, tB);
  if (src_is_y) { for (int i = 0; i < nit; i++) tA[i] = polys[i]; }
  else HB_TRY(launch_blk(c, -1, (const u64* const*)polys, tA, nit, src, n, 0, nullptr));
  if (v1_cols_ok(c) && c->conv1 && n == 1 && p <= 1 && !src_is_y && !want_frac && nt <= HB_MAXROWS) {
    // single source prime, no plaintext correction: dedicated kernel without the MAC loop / quotient phase
    Hb1Conv1Job J1; memset(&J1, 0, sizeof(J1));
    // column quads per CTA: the single source row keeps only cq of the ng groups busy during the source phase, so more quads per
    // CTA amortise it (cq + 19 cq target slots over ng groups); 64/cq CTAs per item must still fill whole waves
    static const int cq_env = [] { const char* e = getenv("HB_CONV1_CQ"); int v = e ? atoi(e) : 0; return (v == 1 || v == 2 || v == 4) ? v : 0; }();
    const int cq = cq_env ? cq_env : 4, ng = 10;   // H100 SXM (400 W): 2 and 4 quads give the same k1_conv1 time (2.79 ms per step)
    J1.logN = c->logN; J1.ngroups = ng; J1.cq = cq; J1.nitems = nit; J1.src_prime = src[0]; J1.nt = nt;
    const u64 qs = c->q[src[0]];
    for (int t = 0; t < nt; t++) { J1.tgt_prime[t] = tgt[t]; J1.qs_mod[t] = qs % c->q[tgt[t]]; J1.nored[t] = (u128)qs <= (u128)7 * c->q[tgt[t]] ? 1 : 0; }
    u64 ninv; if (!h_invmod(c->N % qs, qs, &ninv)) return hb_fail(HB_ERR_BAD_ARG, "N not invertible");
    J1.ninv = ninv; J1.ninv_s = h_shoup(ninv, qs);
    for (int i = 0; i < nit; i++) { J1.src[i] = tA[i]; J1.dst[i] = tB[i]; }
    const size_t smem1 = (size_t)(cq + ng) * HB1_TS * sizeof(u64);
    pre_launch(c);
    if (all_special(c)) HB_LAUNCH(k1_conv1<true>, dim3(64 / cq, nit), dim3(64 * ng), smem1, c->stream, c->d_primes, J1);
    else HB_LAUNCH(k1_conv1<false>, dim3(64 / cq, nit), dim3(64 * ng), smem1, c->stream, c->d_primes, J1);
    return post_launch(c, "k1_conv1", (u64)(n + nt) * nit * c->N * 8);
  }
  if (v1_cols_ok(c)) {
    // number of 64-thread row groups: balance of the n source rows / nt target rows, resident warps,
    // and (for small source sets) co-residency of two CTAs so that one CTA's thin source phase
    // overlaps the other's target phase
    int ng = 0; double best = -1; size_t smem1 = 0;
    for (int g = 10; g >= 4; g--) {
      size_t sm = ((size_t)(n + g) * HB1_TS + 4 * HB1_VS) * sizeof(u64);
      if (sm > 224 * 1024) continue;
      int by_smem = (int)((227 * 1024) / (sm + 1024)), by_regs = 65536 / (96 * 64 * g);
      int ctas = std::max(1, std::min(std::min(by_smem, by_regs), 2));
      double work = n + 1.4 * nt, slots = (double)((n + g - 1) / g) + 1.4 * ((nt + g - 1) / g);
      double balance = work / (slots * g);
      double warps = std::min(20.0, 2.0 * g * ctas);
      double score = balance * (0.5 + 0.5 * warps / 20.0) * (ctas >= 2 ? 1.15 : 1.0);
      if (score > best) { best = score; ng = g; smem1 = sm; }
    }
    if (ng > 0) {
      Hb1ConvJob J1; memset(&J1, 0, sizeof(J1));
      J1.cv = E->d; J1.logN = c->logN; J1.ngroups = ng; J1.nitems = nit; J1.stats = c->d_stats; J1.src_is_y = src_is_y;
      if (want_frac) for (int i = 0; i < nit; i++) J1.frac[i] = c->d_frac + (size_t)i * c->N;
      for (int i = 0; i < nit; i++) { J1.src[i] = tA[i]; J1.dst[i] = tB[i]; }
      pre_launch(c);
      if (all_special(c)) HB_LAUNCH(k1_conv<true>, dim3(64, nit), dim3(64 * ng), smem1, c->stream, c->d_primes, J1);
      else HB_LAUNCH(k1_conv<false>, dim3(64, nit), dim3(64 * ng), smem1, c->stream, c->d_primes, J1);
      return post_launch(c, "k1_conv", (u64)(n + nt) * nit * c->N * 8);
    }
  }
  const int n1 = c->logN - c->log_blk;
  int lw = logw_cols(c);
  while (lw > 0 && ((size_t)(n + 2) << (n1 + lw)) * sizeof(u64) > c->max_smem) lw--;
  size_t smem = ((size_t)(n + 2) << (n1 + lw)) * sizeof(u64);
  if (smem > c->max_smem) return hb_fail(HB_ERR_UNSUPPORTED, "base conversion tile needs %zu bytes of shared memory", smem);
  HbConvJob J; memset(&J, 0, sizeof(J));
  J.cv = E->d; J.logN = c->logN; J.log_blk = c->log_blk; J.logw = lw; J.nitems = nit; J.stats = c->d_stats; J.src_is_y = src_is_y;
  if (want_frac) for (int i = 0; i < nit; i++) J.frac[i] = c->d_frac + (size_t)i * c->N;
  for (int i = 0; i < nit; i++) { J.src[i] = tA[i]; J.dst[i] = tB[i]; }
  dim3 grid(1u << (c->log_blk - lw), nit);
  pre_launch(c);
  HB_LAUNCH(k_conv, grid, dim3(HB_THREADS), smem, c->stream, c->d_primes, J);
  return post_launch(c, "k_conv", (u64)(n + nt) * nit * c->N * 8);
}

// ------------------------------------------------------------------------------------------
// general m (Bluestein rows)
struct PlanScope {   // run the power-of-two transform launchers on a cyclic plan: 0 = length L (chirp convolutions), 1 = length L2 (division by Phi_m)
  hb_ctx* c; int logN, log_blk; HbPrimeDev* dp; size_t N;
  PlanScope(hb_ctx* c_, int plan) : c(c_), logN(c_->logN), log_blk(c_->log_blk), dp(c_->d_primes), N(c_->N) {
    if (plan == 0) { c->logN = c->gen.logL; c->log_blk = c->gen.log_blk_L; c->d_primes = c->gen.d_primes_cyc; c->N = c->gen.L; }
    else { c->logN = c->gen.logL2; c->log_blk = c->gen.log_blk_L2; c->d_primes = c->gen.d_primes_cyc2; c->N = c->gen.L2; }
  }
  ~PlanScope() { c->logN = logN; c->log_blk = log_blk; c->d_primes = dp; c->N = N; }
};
static long h_phi(long m) { long r = m, n = m; for (long p = 2; p * p <= n; p++) if (n % p == 0) { while (n % p == 0) n /= p; r -= r / p; } if (n > 1) r -= r / n; return r; }
static long h_gcd(long a, long b) { while (b) { long t = a % b; a = b; b = t; } return a; }
static bool h_isprime_small(long n) { if (n < 2) return false; for (long p = 2; p * p <= n; p++) if (n % p == 0) return false; return true; }
// FindPrimitiveRoot (src/NumbTh.cpp:435-493): deterministic
static u64 h_find_primitive_root(u64 q, u64 e) {
  u64 root = 1, n = e;
  for (u64 p = 2; p <= n; p++) {
    if (n % p) continue;
    u64 pp = 1; while (n % p == 0) { n /= p; pp *= p; }
    u64 g = 2;
    for (;; g++) if (h_isprime_small((long)g) && h_powmod(g, (q - 1) / p, q) != 1) break;
    root = h_mulmod(root, h_powmod(g, (q - 1) / pp, q), q);
  }
  return root;
}
// multiply / exactly divide an integer polynomial by (X^k - 1)
static void poly_mul_binom(std::vector<long>& a, long k) { std::vector<long> r(a.size() + k, 0); for (size_t i = 0; i < a.size(); i++) { r[i + k] += a[i]; r[i] -= a[i]; } a.swap(r); }
static void poly_div_binom(std::vector<long>& a, long k) {   // a / (X^k - 1), exact
  std::vector<long> qv(a.size() - k, 0);
  for (long i = (long)a.size() - 1; i >= k; i--) { long cq = a[i]; qv[i - k] = cq; a[i] -= cq; a[i - k] += cq; }
  a.swap(qv);
}
static int h_mobius(long n) { int mu = 1; for (long p = 2; p * p <= n; p++) if (n % p == 0) { n /= p; if (n % p == 0) return 0; mu = -mu; } if (n > 1) mu = -mu; return mu; }
// Phi_m = prod_{d|m} (X^(m/d) - 1)^mu(d)
static std::vector<long> h_cyclotomic(long m) {
  std::vector<long> a(1, 1);
  for (long d = 1; d <= m; d++) if (m % d == 0 && h_mobius(d) == 1) poly_mul_binom(a, m / d);
  for (long d = 1; d <= m; d++) if (m % d == 0 && h_mobius(d) == -1) poly_div_binom(a, m / d);
  return a;
}

static int gen_cyc_ntt(hb_ctx* c, int dir, u64* const* w, u64* const* tmp, int nit, const int32_t* idx, int n, int plan = 0) {
  PlanScope ps(c, plan);
  if (dir > 0) { HB_TRY(launch_cols(c, +1, (const u64* const*)w, tmp, nit, idx, n)); return launch_blk(c, +1, (const u64* const*)tmp, w, nit, idx, n, 0, nullptr); }
  HB_TRY(launch_blk(c, -1, (const u64* const*)w, tmp, nit, idx, n, 0, nullptr));
  return launch_cols(c, -1, (const u64* const*)tmp, w, nit, idx, n);
}
static int gen_k(hb_ctx* c, int op, int which, const u64* const* src, u64* const* dst, int nit, const int32_t* idx, int n) {
  hb_ctx::Gen& g = c->gen;
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    int nr = std::min(HB_MAXROWS, n - r0);
    HbGenJob J; memset(&J, 0, sizeof(J));
    J.m = g.m; J.phim = g.phim; J.L = g.L; J.L2 = g.L2; J.d = g.d; J.rep = g.d_rep; J.irep = g.d_irep; J.which = which;
    fill_rows(J.rows, idx + r0, nr);
    J.nitems = nit;
    for (int i = 0; i < nit; i++) {
      J.src[i] = src ? src[i] : nullptr; J.dst[i] = dst ? dst[i] : nullptr;
      J.w0[i] = g.w0 + (size_t)i * c->nprimes * g.L; J.w1[i] = g.w1 + (size_t)i * c->nprimes * g.L;
    }
    unsigned gx = (unsigned)std::max<size_t>(1, g.L / (HB_THREADS * 4));
    pre_launch(c);
    HB_LAUNCH(k_gen, dim3(gx, nr, nit), dim3(HB_THREADS), 0, c->stream, c->d_primes, g.d_gp, J, op);
    HB_TRY(post_launch(c, "k_gen", (u64)2 * nr * nit * g.L * 8));
  }
  return HB_OK;
}
static void gen_wptrs(hb_ctx* c, u64* base, int nit, u64** out) { for (int i = 0; i < nit; i++) out[i] = base + (size_t)i * c->nprimes * c->gen.L; }
// coefficient rows (src) -> evaluation rows (dst); Cmodulus::FFT general branch
static int gen_fwd(hb_ctx* c, const u64* const* src, u64* const* dst, int nit, const int32_t* idx, int n) {
  u64 *W0[HB_MAXB], *WT[HB_MAXB]; gen_wptrs(c, c->gen.w0, nit, W0); gen_wptrs(c, c->gen.wt, nit, WT);
  HB_TRY(gen_k(c, HB_GEN_PRE_FWD, 0, src, nullptr, nit, idx, n));
  HB_TRY(gen_cyc_ntt(c, +1, W0, WT, nit, idx, n));
  HB_TRY(gen_k(c, HB_GEN_MULVEC, 0, nullptr, nullptr, nit, idx, n));
  HB_TRY(gen_cyc_ntt(c, -1, W0, WT, nit, idx, n));
  return gen_k(c, HB_GEN_POST_FWD, 0, nullptr, dst, nit, idx, n);
}
// evaluation rows (src) -> coefficient rows in [0,q) (dst); Cmodulus::iFFT general branch
static int gen_inv(hb_ctx* c, const u64* const* src, u64* const* dst, int nit, const int32_t* idx, int n) {
  u64 *W0[HB_MAXB], *W1[HB_MAXB], *WT[HB_MAXB]; gen_wptrs(c, c->gen.w0, nit, W0); gen_wptrs(c, c->gen.w1, nit, W1); gen_wptrs(c, c->gen.wt, nit, WT);
  HB_TRY(gen_k(c, HB_GEN_PRE_INV, 0, src, nullptr, nit, idx, n));
  HB_TRY(gen_cyc_ntt(c, +1, W0, WT, nit, idx, n));
  HB_TRY(gen_k(c, HB_GEN_MULVEC, 1, nullptr, nullptr, nit, idx, n));
  HB_TRY(gen_cyc_ntt(c, -1, W0, WT, nit, idx, n));
  HB_TRY(gen_k(c, HB_GEN_POST_INV, 0, nullptr, dst, nit, idx, n));
  if (c->gen.d > 0) {   // remainder modulo Phi_m(X)
    // both products run on the short plan (rows of stride L2 inside the same work buffers): the quotient is a product of two
    // length-d polynomials, and q*Phi_m is taken modulo X^L2 - 1 -- POST_INV has already folded the known wrapped part into dst
    HB_TRY(gen_cyc_ntt(c, +1, W1, WT, nit, idx, n, 1));
    HB_TRY(gen_k(c, HB_GEN_MULVEC, 2, nullptr, nullptr, nit, idx, n));
    HB_TRY(gen_cyc_ntt(c, -1, W1, WT, nit, idx, n, 1));
    HB_TRY(gen_k(c, HB_GEN_QREV, 0, nullptr, nullptr, nit, idx, n));
    HB_TRY(gen_cyc_ntt(c, +1, W0, WT, nit, idx, n, 1));
    HB_TRY(gen_k(c, HB_GEN_MULVEC, 3, nullptr, nullptr, nit, idx, n));
    HB_TRY(gen_cyc_ntt(c, -1, W0, WT, nit, idx, n, 1));
  } else {
    HB_CUDA(cudaMemsetAsync(c->gen.w0, 0, (size_t)nit * c->nprimes * c->gen.L * sizeof(u64), c->stream));
  }
  return gen_k(c, HB_GEN_FIN, 0, nullptr, dst, nit, idx, n);
}
// exact conversion on coefficient rows: rows src of polys -> x mod q_t as evaluation rows tgt in cB
static int gen_conv(hb_ctx* c, u64* const* polys, int nit, const int32_t* src, int n, const int32_t* tgt, int nt, u64 p, bool want_frac = false) {
  if (want_frac) HB_TRY(norm_scratch(c));
  ConvEntry* E; HB_TRY(get_conv(c, src, n, tgt, nt, p, &E));
  u64 *A[HB_MAXB], *B[HB_MAXB];
  for (int i = 0; i < nit; i++) { A[i] = c->gen.cA + (size_t)i * c->nprimes * c->N; B[i] = c->gen.cB + (size_t)i * c->nprimes * c->N; }
  HB_TRY(gen_inv(c, (const u64* const*)polys, A, nit, src, n));
  HbPlainConvJob J; memset(&J, 0, sizeof(J));
  J.cv = E->d; J.t = E->d_t; J.t_s = E->d_t_s; J.N = c->N; J.nitems = nit; J.stats = c->d_stats;
  for (int i = 0; i < nit; i++) { J.src[i] = A[i]; J.dst[i] = B[i]; if (want_frac) J.frac[i] = c->d_frac + (size_t)i * c->N; }
  pre_launch(c);
  HB_LAUNCH(k_conv_plain, dim3((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS), nit), dim3(HB_THREADS), 0, c->stream, c->d_primes, J);
  HB_TRY(post_launch(c, "k_conv_plain", (u64)(n + nt) * nit * c->N * 8));
  return gen_fwd(c, (const u64* const*)B, B, nit, tgt, nt);
}

// general m: max over Z_m^* of |f(W^i)| for the nit fraction polynomials in c->d_frac -> out[0..nit)   (synchronises)
static int gen_norm_chunk(hb_ctx* c, int nit, double* out) {
  hb_ctx::Gen& g = c->gen;
  if (!g.d_W) {
    std::vector<double2> W(g.m);
    for (u64 j = 0; j < g.m; j++) { const long double a = 2.0L * 3.14159265358979323846264338327950288L * (long double)j / (long double)g.m; W[j].x = (double)cosl(a); W[j].y = (double)sinl(a); }
    HB_TRY(ctx_alloc(c, (void**)&g.d_W, sizeof(double2) * g.m));
    HB_CUDA(cudaMemcpy(g.d_W, W.data(), sizeof(double2) * g.m, cudaMemcpyHostToDevice));
  }
  HB_CUDA(cudaMemsetAsync(c->d_max, 0, nit * sizeof(unsigned long long), c->stream));
  HbGenNormJob J; J.m = g.m; J.phim = g.phim; J.frac = c->d_frac; J.W = g.d_W; J.rep = g.d_rep; J.maxbits = c->d_max;
  pre_launch(c);
  HB_LAUNCH(k_gen_norm, dim3((unsigned)((g.phim + HB_THREADS - 1) / HB_THREADS), nit), dim3(HB_THREADS), 1024 * sizeof(double), c->stream, J);
  HB_TRY(post_launch(c, "k_gen_norm", (u64)nit * g.phim * 8));
  unsigned long long bits[HB_MAXB];
  HB_CUDA(cudaMemcpyAsync(bits, c->d_max, nit * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < nit; i++) { double m2; memcpy(&m2, &bits[i], 8); out[i] = std::sqrt(m2); }
  return HB_OK;
}

static int gen_init(hb_ctx* c, const uint64_t* psi) {
  hb_ctx::Gen& g = c->gen;
  const long m = (long)c->m;
  g.on = true; g.m = m; g.phim = h_phi(m); g.d = g.m - g.phim;
  g.logL = 0; while ((1L << g.logL) < 2 * m - 1) g.logL++;
  g.L = 1ULL << g.logL; g.log_blk_L = g.logL >= 11 ? 8 : 0;
  g.logL2 = 0; while ((1UL << g.logL2) < std::max<u64>(g.phim, 2 * g.d - 1)) g.logL2++;
  g.L2 = 1ULL << g.logL2; g.log_blk_L2 = g.logL2 >= 11 ? 8 : 0;
  c->N = g.phim; c->logN = -1; c->log_blk = 0;
  const u64 e = m % 2 == 0 ? 2 * m : m;
  const int np = c->nprimes; const size_t L = g.L, L2 = g.L2;
  std::vector<int> rep, irep(m, -1);
  for (long i = 1; i < m; i++) if (h_gcd(i, m) == 1) { irep[i] = (int)rep.size(); rep.push_back((int)i); }
  HB_TRY(ctx_alloc(c, (void**)&g.d_rep, sizeof(int) * rep.size()));
  HB_TRY(ctx_alloc(c, (void**)&g.d_irep, sizeof(int) * m));
  HB_CUDA(cudaMemcpy(g.d_rep, rep.data(), sizeof(int) * rep.size(), cudaMemcpyHostToDevice));
  HB_CUDA(cudaMemcpy(g.d_irep, irep.data(), sizeof(int) * m, cudaMemcpyHostToDevice));
  // integer polynomials Phi_m and rev((X^m-1)/Phi_m) mod X^d
  std::vector<long> phi = h_cyclotomic(m);
  std::vector<long> psiq(1, 1);   // (X^m - 1)/Phi_m = prod_{d|m, d>1} (X^(m/d)-1)^(-mu(d))
  for (long dd = 2; dd <= m; dd++) if (m % dd == 0 && h_mobius(dd) == -1) poly_mul_binom(psiq, m / dd);
  for (long dd = 2; dd <= m; dd++) if (m % dd == 0 && h_mobius(dd) == 1) poly_div_binom(psiq, m / dd);
  if ((long)phi.size() != (long)g.phim + 1 || (long)psiq.size() != (long)g.d + 1) return hb_fail(HB_ERR_BAD_ARG, "internal: cyclotomic polynomial degree mismatch");
  // device tables: per prime  pw[m] ipw[m] (ulonglong2)  | 4 vectors of L  | cyclic twiddles 2 x L (ulonglong2)
  const size_t per = (size_t)2 * m * 16 + 4 * L * 8 + 2 * L * 16;
  std::vector<unsigned char> tab(per * np);
  HB_TRY(ctx_alloc(c, &g.tab, tab.size()));
  std::vector<HbGenPrime> gp(np);
  std::vector<HbPrimeDev> pc(np), pc2(np);
  std::vector<unsigned> brev(L);
  for (size_t k = 0; k < L; k++) { unsigned r = 0; for (int b = 0; b < g.logL; b++) if (k >> b & 1) r |= 1u << (g.logL - 1 - b); brev[k] = r; }
  for (int i = 0; i < np; i++) {
    const u64 q = c->q[i];
    if ((q - 1) % e != 0 || (q - 1) % L != 0) return hb_fail(HB_ERR_UNSUPPORTED, "prime %d: q-1 is not divisible by %llu and the Bluestein length %llu", i, (unsigned long long)e, (unsigned long long)L);
    const u64 root = psi ? psi[i] : h_find_primitive_root(q, e);
    if (h_powmod(root, e, q) != 1) return hb_fail(HB_ERR_BAD_ARG, "psi[%d] is not a %llu-th root of unity", i, (unsigned long long)e);
    c->psi[i] = root;
    const u64 rinv = h_powmod(root, q - 2, q);
    unsigned char* base = tab.data() + per * i;
    ulonglong2* pw = (ulonglong2*)base; ulonglong2* ipw = pw + m;
    u64* vec = (u64*)(ipw + m);   // RbHat, iRbHat, invHat, phiHat (raw here, transformed on the device below)
    ulonglong2* fwc = (ulonglong2*)(vec + 4 * L); ulonglong2* iwc = fwc + L;
    memset(vec, 0, 4 * L * 8);
    for (long k = 0; k < m; k++) {
      const u64 ex = (u64)(((u128)k * k) % e);
      const u64 a = h_powmod(root, ex, q), b = h_powmod(rinv, ex, q);
      pw[k] = make_ulonglong2(a, h_shoup(a, q)); ipw[k] = make_ulonglong2(b, h_shoup(b, q));
      // chirp kernels b[m-1 +- k] (src/bluestein.cpp:118-128)
      vec[0 * L + (m - 1 + k)] = b; vec[0 * L + (m - 1 - k)] = b;
      vec[1 * L + (m - 1 + k)] = a; vec[1 * L + (m - 1 - k)] = a;
    }
    for (size_t k = 0; k < g.d; k++) { long v = psiq[g.d - k] % (long)q; vec[2 * L + k] = (u64)(v < 0 ? v + (long)q : v); }   // rev(Psi) mod X^d
    for (size_t k = 0; k <= g.phim; k++) {   // Phi_m modulo X^L2 - 1 (phi(m) = L2 folds the leading 1 onto the constant term)
      long v = phi[k] % (long)q; u64& slot = vec[3 * L + k % L2];
      slot = (slot + (u64)(v < 0 ? v + (long)q : v)) % q;
    }
    // cyclic twiddles: fw[2^s + i] = omega^((L / 2^(s+1)) * brev_s(i))
    u64 gnr = 2; while (h_powmod(gnr, (q - 1) / 2, q) != q - 1) gnr++;
    const u64 om = h_powmod(gnr, (q - 1) / L, q), iom = h_powmod(om, q - 2, q);
    std::vector<u64> opw(L), iopw(L);
    { u64 w = 1, iw = 1; for (size_t k = 0; k < L; k++) { opw[k] = w; iopw[k] = iw; w = h_mulmod(w, om, q); iw = h_mulmod(iw, iom, q); } }
    fwc[0] = iwc[0] = make_ulonglong2(1, h_shoup(1, q));
    for (int s2 = 0; s2 < g.logL; s2++)
      for (size_t ii = 0; ii < (1ULL << s2); ii++) {
        const size_t br = s2 ? (brev[ii] >> (g.logL - s2)) : 0;
        const size_t ex = (L >> (s2 + 1)) * br;
        fwc[(1ULL << s2) + ii] = make_ulonglong2(opw[ex], h_shoup(opw[ex], q));
        iwc[(1ULL << s2) + ii] = make_ulonglong2(iopw[ex], h_shoup(iopw[ex], q));
      }
    unsigned char* dbase = (unsigned char*)g.tab + per * i;
    gp[i].pw = (const ulonglong2*)dbase; gp[i].ipw = gp[i].pw + m;
    const u64* dvec = (const u64*)(gp[i].ipw + m);
    gp[i].RbHat = dvec; gp[i].iRbHat = dvec + L; gp[i].invHat = dvec + 2 * L; gp[i].phiHat = dvec + 3 * L;
    gp[i].minv = h_powmod((u64)m % q, q - 2, q); gp[i].minv_s = h_shoup(gp[i].minv, q);
    pc[i] = c->h_primes[i];
    pc[i].fw = (const ulonglong2*)(dvec + 4 * L); pc[i].iw = pc[i].fw + L;
    pc[i].ninv = h_powmod((u64)L % q, q - 2, q); pc[i].ninv_s = h_shoup(pc[i].ninv, q);
    pc2[i] = pc[i];   // the twiddles of a shorter cyclic length are a prefix of the same table: fw[2^s + i] does not depend on L
    pc2[i].ninv = h_powmod((u64)L2 % q, q - 2, q); pc2[i].ninv_s = h_shoup(pc2[i].ninv, q);
  }
  HB_CUDA(cudaMemcpy(g.tab, tab.data(), tab.size(), cudaMemcpyHostToDevice));
  HB_TRY(ctx_alloc(c, (void**)&g.d_gp, sizeof(HbGenPrime) * np));
  HB_CUDA(cudaMemcpy(g.d_gp, gp.data(), sizeof(HbGenPrime) * np, cudaMemcpyHostToDevice));
  HB_TRY(ctx_alloc(c, (void**)&g.d_primes_cyc, sizeof(HbPrimeDev) * np));
  HB_CUDA(cudaMemcpy(g.d_primes_cyc, pc.data(), sizeof(HbPrimeDev) * np, cudaMemcpyHostToDevice));
  HB_TRY(ctx_alloc(c, (void**)&g.d_primes_cyc2, sizeof(HbPrimeDev) * np));
  HB_CUDA(cudaMemcpy(g.d_primes_cyc2, pc2.data(), sizeof(HbPrimeDev) * np, cudaMemcpyHostToDevice));
  const size_t wsz = (size_t)HB_MAXB * np * L * sizeof(u64), csz = (size_t)HB_MAXB * np * c->N * sizeof(u64);
  HB_TRY(ctx_alloc(c, (void**)&g.w0, wsz)); HB_TRY(ctx_alloc(c, (void**)&g.w1, wsz)); HB_TRY(ctx_alloc(c, (void**)&g.wt, wsz));
  HB_TRY(ctx_alloc(c, (void**)&g.cA, csz)); HB_TRY(ctx_alloc(c, (void**)&g.cB, csz));
  // transform the four fixed vectors of every prime in place (layout per prime is not [np][L], so one prime at a time)
  for (int i = 0; i < np; i++) {
    for (int v = 0; v < 4; v++) {
      u64* dv = (u64*)((unsigned char*)g.tab + per * i + (size_t)2 * m * 16) + (size_t)v * L;
      // stage through w0 row i so that the launchers' row addressing (prime index * plan length) applies
      const size_t Lv = v < 2 ? L : L2;   // the chirp kernels on the long plan, the two division vectors on the short one
      HB_CUDA(cudaMemcpyAsync(g.w0 + (size_t)i * Lv, dv, Lv * 8, cudaMemcpyDeviceToDevice, c->stream));
      u64* W0[1] = {g.w0}; u64* WT[1] = {g.wt}; int32_t one[1] = {i};
      HB_TRY(gen_cyc_ntt(c, +1, W0, WT, 1, one, 1, v < 2 ? 0 : 1));
      HB_CUDA(cudaMemcpyAsync(dv, g.w0 + (size_t)i * Lv, Lv * 8, cudaMemcpyDeviceToDevice, c->stream));
    }
  }
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}

// ------------------------------------------------------------------------------------------
// C ABI: transforms and pointwise
extern "C" int hb_ntt_fwd(hb_poly* const* polys, int nitems, const int32_t* idx, int n) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_ntt_fwd")); HB_TRY(check_idx(c, idx, n, "hb_ntt_fwd"));
  if (c->gen.on) return for_items(nitems, [&](int i0, int nit) { u64* P[HB_MAXB]; ptrs_of(polys, i0, nit, P); return gen_fwd(c, (const u64* const*)P, P, nit, idx, n); });
  HB_TRY(ctx_scratch(c));
  return for_items(nitems, [&](int i0, int nit) {
    u64* P[HB_MAXB]; u64* tA[HB_MAXB]; ptrs_of(polys, i0, nit, P); tmp_ptrs(c, c->tmpA, nit, tA);
    HB_TRY(launch_cols(c, +1, (const u64* const*)P, tA, nit, idx, n));
    return launch_blk(c, +1, (const u64* const*)tA, P, nit, idx, n, 0, nullptr);
  });
}
extern "C" int hb_ntt_inv(hb_poly* const* polys, int nitems, const int32_t* idx, int n) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_ntt_inv")); HB_TRY(check_idx(c, idx, n, "hb_ntt_inv"));
  if (c->gen.on) return for_items(nitems, [&](int i0, int nit) { u64* P[HB_MAXB]; ptrs_of(polys, i0, nit, P); return gen_inv(c, (const u64* const*)P, P, nit, idx, n); });
  HB_TRY(ctx_scratch(c));
  return for_items(nitems, [&](int i0, int nit) {
    u64* P[HB_MAXB]; u64* tA[HB_MAXB]; ptrs_of(polys, i0, nit, P); tmp_ptrs(c, c->tmpA, nit, tA);
    HB_TRY(launch_blk(c, -1, (const u64* const*)P, tA, nit, idx, n, 0, nullptr));
    return launch_cols(c, -1, (const u64* const*)tA, P, nit, idx, n);
  });
}

static int pw_simple(int op, hb_poly* const* dst, hb_poly* const* src, int nitems, const int32_t* idx, int n, const u64* scal, hb_ctx* c) {
  return for_items(nitems, [&](int i0, int nit) {
    u64* D[HB_MAXB]; u64* S[HB_MAXB]; ptrs_of(dst, i0, nit, D); if (src) ptrs_of(src, i0, nit, S);
    PwArgs A; memset(&A, 0, sizeof(A));
    A.op = op; A.dst = D; A.a = src ? (const u64* const*)S : nullptr; A.scal = scal;
    return launch_pw(c, A, nit, idx, n);
  });
}
extern "C" int hb_pointwise(int op, hb_poly* const* dst, hb_poly* const* src, int nitems, const int32_t* idx, int n) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(dst, nitems, &c, "hb_pointwise")); HB_TRY(check_polys(src, nitems, &c, "hb_pointwise"));
  HB_TRY(check_idx(c, idx, n, "hb_pointwise"));
  int dop;
  switch (op) {
    case HB_OP_ADD: dop = HB_PW_ADD; break; case HB_OP_SUB: dop = HB_PW_SUB; break; case HB_OP_MUL: dop = HB_PW_MUL; break;
    case HB_OP_NEG: dop = HB_PW_NEG; break; case HB_OP_COPY: dop = HB_PW_COPY; break;
    default: return hb_fail(HB_ERR_BAD_ARG, "hb_pointwise: unknown op %d", op);
  }
  return pw_simple(dop, dst, src, nitems, idx, n, nullptr, c);
}
extern "C" int hb_scale_rows(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const uint64_t* scalars) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_scale_rows")); HB_TRY(check_idx(c, idx, n, "hb_scale_rows"));
  if (!scalars) return hb_fail(HB_ERR_BAD_ARG, "hb_scale_rows: null scalars");
  for (int i = 0; i < n; i++) if (scalars[i] >= c->q[idx[i]]) return hb_fail(HB_ERR_BAD_ARG, "hb_scale_rows: scalar %d not reduced", i);
  return pw_simple(HB_PW_SCALE, polys, nullptr, nitems, idx, n, (const u64*)scalars, c);
}
static u64 prod_mod(hb_ctx* c, const int32_t* fidx, int nf, u64 q) {
  u64 r = 1 % q; for (int k = 0; k < nf; k++) r = h_mulmod(r, c->q[fidx[k]] % q, q); return r;
}
static int scalars_by_primes(hb_ctx* c, const int32_t* idx, int n, const int32_t* fidx, int nf, int inverse, std::vector<u64>& out) {
  out.resize(n);
  for (int i = 0; i < n; i++) {
    u64 q = c->q[idx[i]]; u64 f = prod_mod(c, fidx, nf, q);
    if (inverse) { if (f == 0) return hb_fail(HB_ERR_BAD_ARG, "division by a multiple of prime %d", idx[i]); f = h_powmod(f, q - 2, q); }
    out[i] = f;
  }
  return HB_OK;
}
extern "C" int hb_scale_by_primes(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const int32_t* fidx, int nf, int inverse) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_scale_by_primes")); HB_TRY(check_idx(c, idx, n, "hb_scale_by_primes"));
  HB_TRY(check_idx(c, fidx, nf, "hb_scale_by_primes(factor)", true));
  std::vector<u64> sc; HB_TRY(scalars_by_primes(c, idx, n, fidx, nf, inverse, sc));
  return pw_simple(HB_PW_SCALE, polys, nullptr, nitems, idx, n, sc.data(), c);
}
extern "C" int hb_zero_rows(hb_poly* const* polys, int nitems, const int32_t* idx, int n) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_zero_rows")); HB_TRY(check_idx(c, idx, n, "hb_zero_rows"));
  return pw_simple(HB_PW_ZERO, polys, nullptr, nitems, idx, n, nullptr, c);
}
static int check_disjoint(const int32_t* a, int na, const int32_t* b, int nb, const char* who) {
  for (int i = 0; i < na; i++) for (int j = 0; j < nb; j++) if (a[i] == b[j]) return hb_fail(HB_ERR_INDEX_SET, "%s: can only be called on a disjoint set (prime %d)", who, a[i]);
  return HB_OK;
}
extern "C" int hb_add_primes_and_scale(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* add, int nadd) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_add_primes_and_scale"));
  HB_TRY(check_idx(c, cur, ncur, "hb_add_primes_and_scale", true)); HB_TRY(check_idx(c, add, nadd, "hb_add_primes_and_scale", true));
  if (nadd == 0) return HB_OK;  // src/DoubleCRT.cpp:605-606
  HB_TRY(check_disjoint(cur, ncur, add, nadd, "addPrimesAndScale"));
  if (ncur > 0) HB_TRY(hb_scale_by_primes(polys, nitems, cur, ncur, add, nadd, 0));
  return hb_zero_rows(polys, nitems, add, nadd);
}
// log_norms (optional, [nitems]): ln of the canonical-embedding norm of the balanced polynomial (toPoly of rows cur)
static int add_primes_impl(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* add, int nadd, double* log_norms) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_add_primes"));
  HB_TRY(check_idx(c, cur, ncur, "hb_add_primes", true)); HB_TRY(check_idx(c, add, nadd, "hb_add_primes", true));
  if (nadd == 0) return HB_OK;  // src/DoubleCRT.cpp:569-572
  HB_TRY(check_disjoint(cur, ncur, add, nadd, "addPrimes"));
  if (ncur == 0) {   // the zero polynomial (src/DoubleCRT.cpp:577-583, 931-935); its norm is 0
    if (log_norms) for (int i = 0; i < nitems; i++) log_norms[i] = -INFINITY;
    return hb_zero_rows(polys, nitems, add, nadd);
  }
  if (c->gen.on) {
    double logQg = 0; for (int j = 0; j < ncur; j++) logQg += std::log((double)c->q[cur[j]]);
    return for_items(nitems, [&](int i0, int nit) {
      u64* P[HB_MAXB]; u64* B[HB_MAXB]; ptrs_of(polys, i0, nit, P);
      for (int i = 0; i < nit; i++) B[i] = c->gen.cB + (size_t)i * c->nprimes * c->N;
      HB_TRY(gen_conv(c, P, nit, cur, ncur, add, nadd, 1, log_norms != nullptr));
      PwArgs A; memset(&A, 0, sizeof(A)); A.op = HB_PW_COPY; A.dst = P; A.a = (const u64* const*)B;
      HB_TRY(launch_pw(c, A, nit, add, nadd));
      if (log_norms) {   // basic_embeddingLargestCoeff (src/norms.cpp:129-157) of x/Q, then + ln Q
        double mm[HB_MAXB]; HB_TRY(gen_norm_chunk(c, nit, mm));
        for (int i = 0; i < nit; i++) log_norms[i0 + i] = (mm[i] > 0 ? std::log(mm[i]) : -INFINITY) + logQg;
      }
      return HB_OK;
    });
  }
  HB_TRY(ctx_scratch(c));
  double logQ = 0; for (int j = 0; j < ncur; j++) logQ += std::log((double)c->q[cur[j]]);
  return for_items(nitems, [&](int i0, int nit) {
    u64* P[HB_MAXB]; u64* tB[HB_MAXB]; ptrs_of(polys, i0, nit, P); tmp_ptrs(c, c->tmpB, nit, tB);
    HB_TRY(conv_chunk(c, P, nit, cur, ncur, add, nadd, 1, 0, log_norms != nullptr));
    HB_TRY(launch_blk(c, +1, (const u64* const*)tB, P, nit, add, nadd, 0, nullptr));
    if (log_norms) {
      double m[HB_MAXB]; HB_TRY(norm_chunk(c, nit, m));
      for (int i = 0; i < nit; i++) log_norms[i0 + i] = (m[i] > 0 ? std::log(m[i]) : -INFINITY) + logQ;
    }
    return HB_OK;
  });
}
extern "C" int hb_add_primes(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* add, int nadd) {
  return add_primes_impl(polys, nitems, cur, ncur, add, nadd, nullptr);
}
extern "C" int hb_add_primes_norm(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* add, int nadd, double* log_norms) {
  if (!log_norms) return hb_fail(HB_ERR_BAD_ARG, "hb_add_primes_norm: null output");
  return add_primes_impl(polys, nitems, cur, ncur, add, nadd, log_norms);
}
// norms (optional, [nitems]): canonical-embedding norm of delta/P (the "fdelta" of Ctxt::modDownToSet, src/Ctxt.cpp:476-505)
// lazy: results only reduced to [0,4q) (register kernels only; for consumers inside the fused ciphertext paths)
// the checks and prime sets of scaleDownToSet: diff = cur \ keep (dropped), kept = cur & keep, sc = prod(diff)^-1 on the kept rows;
// nothing to do when diff comes back empty
static int scale_down_sets(hb_ctx* c, const int32_t* cur, int ncur, const int32_t* keep, int nkeep, uint64_t ptxt_space,
                           std::vector<int32_t>& diff, std::vector<int32_t>& kept, std::vector<u64>& sc) {
  HB_TRY(check_idx(c, cur, ncur, "hb_scale_down")); HB_TRY(check_idx(c, keep, nkeep, "hb_scale_down(keep)", true));
  if (ptxt_space < 1) return hb_fail(HB_ERR_BAD_ARG, "ptxtSpace must be at least 1");  // src/DoubleCRT.cpp:1472
  for (int i = 0; i < ncur; i++) {
    bool k = std::find(keep, keep + nkeep, cur[i]) != keep + nkeep;
    (k ? kept : diff).push_back(cur[i]);
  }
  if (diff.empty()) return HB_OK;  // src/DoubleCRT.cpp:1468-1470
  if (kept.empty()) return hb_fail(HB_ERR_INDEX_SET, "scaleDownToSet: s and the index set must have some intersection");  // :1474-1476
  return scalars_by_primes(c, kept.data(), (int)kept.size(), diff.data(), (int)diff.size(), 1, sc);
}
static int scale_down_impl(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* keep, int nkeep, uint64_t ptxt_space, double* norms, int lazy = 0) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_scale_down"));
  std::vector<int32_t> diff, kept; std::vector<u64> sc;
  HB_TRY(scale_down_sets(c, cur, ncur, keep, nkeep, ptxt_space, diff, kept, sc));
  if (diff.empty()) return HB_OK;
  if (c->gen.on) {
    return for_items(nitems, [&](int i0, int nit) {
      u64* P[HB_MAXB]; u64* B[HB_MAXB]; ptrs_of(polys, i0, nit, P);
      for (int i = 0; i < nit; i++) B[i] = c->gen.cB + (size_t)i * c->nprimes * c->N;
      HB_TRY(gen_conv(c, P, nit, diff.data(), (int)diff.size(), kept.data(), (int)kept.size(), ptxt_space, norms != nullptr));
      PwArgs A; memset(&A, 0, sizeof(A)); A.op = HB_PW_SUBSCALE; A.dst = P; A.a = (const u64* const*)B; A.scal = sc.data();
      HB_TRY(launch_pw(c, A, nit, kept.data(), (int)kept.size()));
      if (norms) HB_TRY(gen_norm_chunk(c, nit, norms + i0));
      return HB_OK;
    });
  }
  HB_TRY(ctx_scratch(c));
  return for_items(nitems, [&](int i0, int nit) {
    u64* P[HB_MAXB]; u64* tB[HB_MAXB]; ptrs_of(polys, i0, nit, P); tmp_ptrs(c, c->tmpB, nit, tB);
    HB_TRY(conv_chunk(c, P, nit, diff.data(), (int)diff.size(), kept.data(), (int)kept.size(), ptxt_space, 0, norms != nullptr));
    HB_TRY(launch_blk(c, +1, (const u64* const*)tB, P, nit, kept.data(), (int)kept.size(), 1, sc.data(), lazy && v1_blk_ok(c) ? 1 : 0));
    if (norms) HB_TRY(norm_chunk(c, nit, norms + i0));
    return HB_OK;
  });
}
extern "C" int hb_scale_down(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* keep, int nkeep, uint64_t ptxt_space) {
  return scale_down_impl(polys, nitems, cur, ncur, keep, nkeep, ptxt_space, nullptr);
}
extern "C" int hb_scale_down_norm(hb_poly* const* polys, int nitems, const int32_t* cur, int ncur, const int32_t* keep, int nkeep, uint64_t ptxt_space, double* norms) {
  if (!norms) return hb_fail(HB_ERR_BAD_ARG, "hb_scale_down_norm: null output");
  return scale_down_impl(polys, nitems, cur, ncur, keep, nkeep, ptxt_space, norms);
}
extern "C" int hb_to_poly(hb_poly* p, const int32_t* idx, int n, int positive, uint64_t* out, int Lout) {
  if (!p || !out) return hb_fail(HB_ERR_BAD_ARG, "hb_to_poly: null");
  HB_TRY(check_dense(p, "hb_to_poly"));
  hb_ctx* c = p->ctx;
  HB_TRY(check_idx(c, idx, n, "hb_to_poly", true));
  if (n == 0) { memset(out, 0, sizeof(u64) * c->N * Lout); return HB_OK; }  // src/DoubleCRT.cpp:931-935
  if (Lout < n) return hb_fail(HB_ERR_BAD_ARG, "hb_to_poly: Lout=%d limbs cannot hold a %d-prime product", Lout, n);
  ConvEntry* E; HB_TRY(get_conv(c, idx, n, nullptr, 0, 1, &E));
  u64* P[1] = {p->d};
  const u64* coef;
  if (c->gen.on) { u64* A[1] = {c->gen.cA}; HB_TRY(gen_inv(c, (const u64* const*)P, A, 1, idx, n)); coef = c->gen.cA; }
  else {
    HB_TRY(ctx_scratch(c));
    u64* tA[1] = {c->tmpA}; u64* tB[1] = {c->tmpB};
    HB_TRY(launch_blk(c, -1, (const u64* const*)P, tA, 1, idx, n, 0, nullptr));
    HB_TRY(launch_cols(c, -1, (const u64* const*)tA, tB, 1, idx, n));
    coef = c->tmpB;
  }
  u64* d_out; size_t bytes = c->N * (size_t)Lout * sizeof(u64);
  HB_CUDA(cudaMalloc((void**)&d_out, bytes));
  HbCrtJob J; J.cv = E->d; J.N = (int)c->N; J.Lout = Lout; J.positive = positive; J.src = coef; J.out = d_out;
  HbCrtTabs T; T.t = E->d_t; T.t_s = E->d_t_s;
  dim3 grid((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS));
  pre_launch(c);
  HB_LAUNCH(k_crt, grid, dim3(HB_THREADS), 0, c->stream, c->d_primes, J, T);
  int r = post_launch(c, "k_crt", (u64)(n + Lout) * c->N * 8);
  if (r == HB_OK) { cudaError_t e = cudaMemcpyAsync(out, d_out, bytes, cudaMemcpyDeviceToHost, c->stream); if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream); if (e != cudaSuccess) r = hb_fail(HB_ERR_CUDA, "hb_to_poly: copy failed: %s", cudaGetErrorString(e)); }
  cudaFree(d_out);
  return r;
}

extern "C" int hb_to_poly_mod_p(hb_poly* p, const int32_t* idx, int n, uint64_t ptxt_space, uint64_t factor, int64_t* out) {
  if (!p || !out) return hb_fail(HB_ERR_BAD_ARG, "hb_to_poly_mod_p: null");
  HB_TRY(check_dense(p, "hb_to_poly_mod_p"));
  hb_ctx* c = p->ctx;
  HB_TRY(check_idx(c, idx, n, "hb_to_poly_mod_p", true));
  if (ptxt_space < 2) return hb_fail(HB_ERR_BAD_ARG, "hb_to_poly_mod_p: ptxt_space must be >= 2");
  if (factor >= ptxt_space) return hb_fail(HB_ERR_BAD_ARG, "hb_to_poly_mod_p: factor not reduced mod ptxt_space");
  if (n == 0) { memset(out, 0, sizeof(int64_t) * c->N); return HB_OK; }
  ConvEntry* E; HB_TRY(get_conv(c, idx, n, nullptr, 0, ptxt_space, &E));
  u64* P[1] = {p->d};
  const u64* coef;
  if (c->gen.on) { u64* A[1] = {c->gen.cA}; HB_TRY(gen_inv(c, (const u64* const*)P, A, 1, idx, n)); coef = c->gen.cA; }
  else {
    HB_TRY(ctx_scratch(c));
    u64* tA[1] = {c->tmpA}; u64* tB[1] = {c->tmpB};
    HB_TRY(launch_blk(c, -1, (const u64* const*)P, tA, 1, idx, n, 0, nullptr));
    HB_TRY(launch_cols(c, -1, (const u64* const*)tA, tB, 1, idx, n));
    coef = c->tmpB;
  }
  u64* d_out; size_t bytes = c->N * sizeof(u64);
  HB_CUDA(cudaMalloc((void**)&d_out, bytes));
  HbCrtJob J; memset(&J, 0, sizeof(J));
  J.cv = E->d; J.N = (int)c->N; J.src = coef; J.out = d_out; J.factor = factor; J.factor_s = h_shoup(factor, ptxt_space); J.stats = c->d_stats;
  HbCrtTabs T; T.t = E->d_t; T.t_s = E->d_t_s;
  dim3 grid((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS));
  pre_launch(c);
  HB_LAUNCH(k_crt_modp, grid, dim3(HB_THREADS), 0, c->stream, c->d_primes, J, T);
  int r = post_launch(c, "k_crt_modp", (u64)(n + 1) * c->N * 8);
  if (r == HB_OK) { cudaError_t e = cudaMemcpyAsync(out, d_out, bytes, cudaMemcpyDeviceToHost, c->stream); if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream); if (e != cudaSuccess) r = hb_fail(HB_ERR_CUDA, "hb_to_poly_mod_p: copy failed: %s", cudaGetErrorString(e)); }
  cudaFree(d_out);
  return r;
}

// coefficient polynomial(s) -> evaluation rows: one H2D copy of the polynomial, per-prime reduction and NTT on the device
static int from_coeffs_impl(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const void* host, int L, const char* who) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, who)); HB_TRY(check_idx(c, idx, n, who, true));
  if (!host) return hb_fail(HB_ERR_BAD_ARG, "%s: null coefficients", who);
  if (n == 0) return HB_OK;
  const size_t per = c->N * (size_t)(L > 0 ? L : 1) * sizeof(u64);
  u64* d_src;
  HB_CUDA(cudaMalloc((void**)&d_src, per * nitems));
  cudaError_t e = cudaMemcpyAsync(d_src, host, per * nitems, cudaMemcpyHostToDevice, c->stream);
  if (e != cudaSuccess) { cudaFree(d_src); return hb_fail(HB_ERR_CUDA, "%s: copy failed: %s", who, cudaGetErrorString(e)); }
  int r = for_items(nitems, [&](int i0, int nit) {
    for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
      int nr = std::min(HB_MAXROWS, n - r0);
      HbFromJob J; memset(&J, 0, sizeof(J));
      J.N = c->N; J.L = L; J.nitems = nit;
      fill_rows(J.rows, idx + r0, nr);
      for (int i = 0; i < nit; i++) { J.src[i] = (const u64*)((const char*)d_src + per * (i0 + i)); J.dst[i] = polys[i0 + i]->d; }
      dim3 grid((unsigned)std::max<size_t>(1, std::min<size_t>(c->N / (HB_THREADS * 4), 64)), nr, nit);
      pre_launch(c);
      HB_LAUNCH(k_from_coeffs, grid, dim3(HB_THREADS), 0, c->stream, c->d_primes, J);
      HB_TRY(post_launch(c, "k_from_coeffs", (u64)nit * c->N * 8 * ((L > 0 ? L : 1) + nr)));
    }
    return HB_OK;
  });
  if (r == HB_OK) r = hb_ntt_fwd(polys, nitems, idx, n);
  cudaStreamSynchronize(c->stream);
  cudaFree(d_src);
  return r;
}
extern "C" int hb_poly_from_i64(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const int64_t* coeffs) {
  return from_coeffs_impl(polys, nitems, idx, n, coeffs, 0, "hb_poly_from_i64");
}
extern "C" int hb_poly_from_limbs(hb_poly* const* polys, int nitems, const int32_t* idx, int n, const uint64_t* limbs, int L) {
  if (L < 1 || L > 1024) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_from_limbs: L=%d", L);
  return from_coeffs_impl(polys, nitems, idx, n, limbs, L, "hb_poly_from_limbs");
}
extern "C" int hb_muladd(hb_poly* const* dst, hb_poly* const* a, hb_poly* const* b, int nitems, const int32_t* idx, int n) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(dst, nitems, &c, "hb_muladd")); HB_TRY(check_polys(a, nitems, &c, "hb_muladd")); HB_TRY(check_polys(b, nitems, &c, "hb_muladd"));
  HB_TRY(check_idx(c, idx, n, "hb_muladd"));
  return for_items(nitems, [&](int i0, int nit) {
    u64* D[HB_MAXB]; u64* A_[HB_MAXB]; u64* B_[HB_MAXB]; ptrs_of(dst, i0, nit, D); ptrs_of(a, i0, nit, A_); ptrs_of(b, i0, nit, B_);
    PwArgs A; memset(&A, 0, sizeof(A));
    A.op = HB_PW_MULADD; A.dst = D; A.a = (const u64* const*)A_; A.b = (const u64* const*)B_;
    return launch_pw(c, A, nit, idx, n);
  });
}

// ------------------------------------------------------------------------------------------
// powerful basis + rawModSwitch (SURVEY 8f-4)
static int pw_init(hb_ctx* c, const int64_t* mvec, int k) {
  hb_ctx::Pw& W = c->pw;
  std::vector<long> mv;
  if (mvec && k > 0) mv.assign(mvec, mvec + k);
  else { long n = (long)c->m; for (long p = 2; p <= n; p++) if (n % p == 0) { long pp = 1; while (n % p == 0) { n /= p; pp *= p; } mv.push_back(pp); } }
  long prod = 1; for (long f : mv) prod *= f;
  if (prod != (long)c->m) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_powerful: factors do not multiply to m");
  W.mvec = mv; W.pvec.clear(); W.bvec.clear();
  for (long f : mv) {
    long p = 2; while (f % p) p++;
    long t = f; while (t % p == 0) t /= p;
    if (f < 2 || t != 1) return hb_fail(HB_ERR_UNSUPPORTED, "hb_ctx_set_powerful: factor %ld is not a prime power", f);
    W.pvec.push_back(p); W.bvec.push_back(f / p);
  }
  const int K = (int)mv.size();
  W.triv = K == 1;                                            // PowerfulDCRT::triv (src/powerful.cpp:250-254)
  W.ready = true;
  if (W.triv) return HB_OK;
  if (!c->gen.on) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_powerful: a power-of-two m has a single factor");
  const long m = (long)c->m, phim = (long)c->N;
  std::vector<long> phiv(K), inv(K), sp(K + 1, 1);
  W.long_prod.assign(K + 1, 1);
  for (int d = K - 1; d >= 0; d--) { phiv[d] = mv[d] / W.pvec[d] * (W.pvec[d] - 1); W.long_prod[d] = W.long_prod[d + 1] * mv[d]; sp[d] = sp[d + 1] * phiv[d]; }
  if (sp[0] != phim) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_powerful: phi mismatch");
  for (int d = 0; d < K; d++) { u64 x; if (!h_invmod((u64)((m / mv[d]) % mv[d]), (u64)mv[d], &x)) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_powerful: factors are not coprime"); inv[d] = (long)x; }
  W.cube_to_poly.assign(m, 0); W.short_to_long.assign(phim, 0);
  for (long i = 0; i < m; i++) {                              // computePowerToCubeMap (src/powerful.cpp:62-84)
    long j = 0;
    for (int d = 0; d < K; d++) j += ((i % mv[d]) * inv[d] % mv[d]) * W.long_prod[d + 1];
    W.cube_to_poly[j] = (int)i;
  }
  for (long i = 0; i < phim; i++) {                           // computeShortToLongMap (src/powerful.cpp:92-112)
    long j = 0;
    for (int d = 0; d < K; d++) j += ((i / sp[d + 1]) % phiv[d]) * W.long_prod[d + 1];
    W.short_to_long[i] = (int)j;
  }
  HB_TRY(ctx_alloc(c, (void**)&W.d_cube_to_poly, sizeof(int) * m));
  HB_TRY(ctx_alloc(c, (void**)&W.d_short_to_long, sizeof(int) * phim));
  HB_CUDA(cudaMemcpy(W.d_cube_to_poly, W.cube_to_poly.data(), sizeof(int) * m, cudaMemcpyHostToDevice));
  HB_CUDA(cudaMemcpy(W.d_short_to_long, W.short_to_long.data(), sizeof(int) * phim, cudaMemcpyHostToDevice));
  HB_TRY(ctx_alloc(c, (void**)&W.cube, sizeof(u64) * c->nprimes * m));
  HB_TRY(ctx_alloc(c, (void**)&W.rows, sizeof(u64) * c->nprimes * phim));
  return HB_OK;
}
extern "C" int hb_ctx_set_powerful(hb_ctx* c, const int64_t* mvec, int k) {
  if (!c) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_powerful: null");
  if (c->pw.ready) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_powerful: already set");
  return pw_init(c, mvec, k);
}
extern "C" int hb_ctx_powerful_info(hb_ctx* c, int32_t* nfactors, int64_t* mvec, int32_t* to_poly) {
  if (!c) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_powerful_info: null");
  if (!c->pw.ready) HB_TRY(pw_init(c, nullptr, 0));
  if (nfactors) *nfactors = (int32_t)c->pw.mvec.size();
  if (mvec) for (size_t i = 0; i < c->pw.mvec.size(); i++) mvec[i] = c->pw.mvec[i];
  if (to_poly) for (size_t i = 0; i < c->N; i++) to_poly[i] = c->pw.triv ? (int32_t)i : c->pw.cube_to_poly[c->pw.short_to_long[i]];
  return HB_OK;
}
// rows idx of p (evaluation form) -> coefficient-like rows in the powerful basis; *out = device rows [nprimes][N]
static int to_powerful_rows(hb_ctx* c, hb_poly* p, const int32_t* idx, int n, const u64** out) {
  if (!c->pw.ready) HB_TRY(pw_init(c, nullptr, 0));
  u64* P[1] = {p->d};
  const u64* coef;
  if (c->gen.on) { u64* A[1] = {c->gen.cA}; HB_TRY(gen_inv(c, (const u64* const*)P, A, 1, idx, n)); coef = c->gen.cA; }
  else {
    HB_TRY(ctx_scratch(c));
    u64* tA[1] = {c->tmpA}; u64* tB[1] = {c->tmpB};
    HB_TRY(launch_blk(c, -1, (const u64* const*)P, tA, 1, idx, n, 0, nullptr));
    HB_TRY(launch_cols(c, -1, (const u64* const*)tA, tB, 1, idx, n));
    coef = c->tmpB;
  }
  if (c->pw.triv) { *out = coef; return HB_OK; }
  hb_ctx::Pw& W = c->pw;
  for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
    const int nr = std::min(HB_MAXROWS, n - r0);
    HbPwJob2 J; memset(&J, 0, sizeof(J));
    J.m = c->m; J.phim = c->N; fill_rows(J.rows, idx + r0, nr);
    J.cube_to_poly = W.d_cube_to_poly; J.short_to_long = W.d_short_to_long; J.src = coef; J.cube = W.cube; J.dst = W.rows;
    dim3 grid((unsigned)std::min<size_t>((c->m + HB_THREADS - 1) / HB_THREADS, 256), nr);
    pre_launch(c);
    HB_LAUNCH(k_pw_scatter, grid, dim3(HB_THREADS), 0, c->stream, J);
    HB_TRY(post_launch(c, "k_pw_scatter", (u64)nr * (c->N + c->m) * 8));
    for (size_t d = 0; d < W.mvec.size(); d++) {
      J.stride = (u64)W.long_prod[d + 1]; J.md = (u64)W.mvec[d]; J.p = (u64)W.pvec[d]; J.b = (u64)W.bvec[d];
      pre_launch(c);
      HB_LAUNCH(k_pw_reduce, grid, dim3(HB_THREADS), 0, c->stream, c->d_primes, J);
      HB_TRY(post_launch(c, "k_pw_reduce", (u64)nr * c->m * 16));
    }
    pre_launch(c);
    HB_LAUNCH(k_pw_gather, grid, dim3(HB_THREADS), 0, c->stream, J);
    HB_TRY(post_launch(c, "k_pw_gather", (u64)nr * c->N * 16));
  }
  *out = W.rows;
  return HB_OK;
}
extern "C" int hb_dcrt_to_powerful(hb_poly* p, const int32_t* idx, int n, uint64_t* out, int Lout) {
  if (!p || !out) return hb_fail(HB_ERR_BAD_ARG, "hb_dcrt_to_powerful: null");
  HB_TRY(check_dense(p, "hb_dcrt_to_powerful"));
  hb_ctx* c = p->ctx;
  HB_TRY(check_idx(c, idx, n, "hb_dcrt_to_powerful"));
  if (Lout < n) return hb_fail(HB_ERR_BAD_ARG, "hb_dcrt_to_powerful: Lout=%d limbs cannot hold a %d-prime product", Lout, n);
  ConvEntry* E; HB_TRY(get_conv(c, idx, n, nullptr, 0, 1, &E));
  const u64* rows; HB_TRY(to_powerful_rows(c, p, idx, n, &rows));
  u64* d_out; size_t bytes = c->N * (size_t)Lout * sizeof(u64);
  HB_CUDA(cudaMalloc((void**)&d_out, bytes));
  HbCrtJob J; memset(&J, 0, sizeof(J));
  J.cv = E->d; J.N = (int)c->N; J.Lout = Lout; J.positive = 0; J.src = rows; J.out = d_out;
  HbCrtTabs T; T.t = E->d_t; T.t_s = E->d_t_s;
  pre_launch(c);
  HB_LAUNCH(k_crt, dim3((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS)), dim3(HB_THREADS), 0, c->stream, c->d_primes, J, T);
  int r = post_launch(c, "k_crt", (u64)(n + Lout) * c->N * 8);
  if (r == HB_OK) { cudaError_t e = cudaMemcpyAsync(out, d_out, bytes, cudaMemcpyDeviceToHost, c->stream); if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream); if (e != cudaSuccess) r = hb_fail(HB_ERR_CUDA, "hb_dcrt_to_powerful: copy failed: %s", cudaGetErrorString(e)); }
  cudaFree(d_out);
  return r;
}
extern "C" int hb_raw_mod_switch(hb_poly* p, const int32_t* idx, int n, uint64_t q, uint64_t p2r, int64_t* out) {
  if (!p || !out) return hb_fail(HB_ERR_BAD_ARG, "hb_raw_mod_switch: null");
  HB_TRY(check_dense(p, "hb_raw_mod_switch"));
  hb_ctx* c = p->ctx;
  HB_TRY(check_idx(c, idx, n, "hb_raw_mod_switch"));
  if (q <= 1) return hb_fail(HB_ERR_BAD_ARG, "q must be greater than 1");                                  // src/Ctxt.cpp:2953
  if (p2r <= 1) return hb_fail(HB_ERR_BAD_ARG, "Plaintext space must be greater than 1 for mod switching");   // :2954-2955
  if (h_gcd((long)q, (long)p2r) != 1) return hb_fail(HB_ERR_BAD_ARG, "New modulus and current plaintext space must be co-prime");   // :2956-2958
  if (q >= (1ULL << 54)) return hb_fail(HB_ERR_UNSUPPORTED, "hb_raw_mod_switch: q >= 2^54");
  for (int j = 0; j < n; j++) if (h_gcd((long)(c->q[idx[j]] % q), (long)q) != 1) return hb_fail(HB_ERR_BAD_ARG, "GCD(Q, q) != 1 in Ctxt::rawModSwitch");   // :2970-2971
  ConvEntry* E; HB_TRY(get_conv(c, idx, n, nullptr, 0, p2r, &E));
  const u64* rows; HB_TRY(to_powerful_rows(c, p, idx, n, &rows));
  i64* d_out; size_t bytes = c->N * sizeof(i64);
  HB_CUDA(cudaMalloc((void**)&d_out, bytes));
  HbRawMsJob J; memset(&J, 0, sizeof(J));
  J.cv = E->d; J.t = E->d_t; J.t_s = E->d_t_s; J.N = c->N; J.q = q; J.src = rows; J.out = d_out; J.stats = c->d_stats;
  pre_launch(c);
  HB_LAUNCH(k_raw_mod_switch, dim3((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS)), dim3(HB_THREADS), 0, c->stream, c->d_primes, J);
  int r = post_launch(c, "k_raw_mod_switch", (u64)(n + 1) * c->N * 8);
  if (r == HB_OK) { cudaError_t e = cudaMemcpyAsync(out, d_out, bytes, cudaMemcpyDeviceToHost, c->stream); if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream); if (e != cudaSuccess) r = hb_fail(HB_ERR_CUDA, "hb_raw_mod_switch: copy failed: %s", cudaGetErrorString(e)); }
  cudaFree(d_out);
  return r;
}

// ------------------------------------------------------------------------------------------
// prime-sharded base conversion (SURVEY 8e): split of hb_add_primes / hb_scale_down at the point
// where residues must cross shards.  make_y is local to the owner of each source row; after an
// all-gather of the y rows every rank converts to the target rows it owns.
extern "C" int hb_conv_make_y(hb_poly* const* polys, int nitems, const int32_t* D, int nD, const int32_t* owned, int nOwned, hb_poly* const* ypolys) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_conv_make_y")); HB_TRY(check_polys(ypolys, nitems, &c, "hb_conv_make_y"));
  HB_TRY(check_idx(c, D, nD, "hb_conv_make_y")); HB_TRY(check_idx(c, owned, nOwned, "hb_conv_make_y(owned)", true));
  if (c->gen.on) return hb_fail(HB_ERR_UNSUPPORTED, "prime-sharded conversion is only built for power-of-two m");
  if (nOwned == 0) return HB_OK;
  std::vector<u64> sc(nOwned);
  for (int k = 0; k < nOwned; k++) {
    if (std::find(D, D + nD, owned[k]) == D + nD) return hb_fail(HB_ERR_INDEX_SET, "hb_conv_make_y: owned prime %d is not in the source set", owned[k]);
    u64 q = c->q[owned[k]], r = 1 % q;
    for (int j = 0; j < nD; j++) if (D[j] != owned[k]) r = h_mulmod(r, c->q[D[j]] % q, q);
    sc[k] = h_powmod(r, q - 2, q);   // (Q_D / q_j)^-1 mod q_j   (src/DoubleCRT.cpp:1033-1041)
  }
  HB_TRY(ctx_scratch(c));
  if (v1_cols_ok(c)) {   // the scaling rides on the N^-1 multiplication of the inverse cols phase
    std::vector<u64> f(nOwned);
    for (int k = 0; k < nOwned; k++) f[k] = h_mulmod(sc[k], c->h_primes[owned[k]].ninv, c->q[owned[k]]);
    return for_items(nitems, [&](int i0, int nit) {
      u64* P[HB_MAXB]; u64* Y[HB_MAXB]; u64* tA[HB_MAXB]; ptrs_of(polys, i0, nit, P); ptrs_of(ypolys, i0, nit, Y); tmp_ptrs(c, c->tmpA, nit, tA);
      HB_TRY(launch_blk(c, -1, (const u64* const*)P, tA, nit, owned, nOwned, 0, nullptr));
      return launch_cols_v1(c, -1, (const u64* const*)tA, Y, nit, owned, nOwned, f.data());
    });
  }
  HB_TRY(for_items(nitems, [&](int i0, int nit) {
    u64* P[HB_MAXB]; u64* Y[HB_MAXB]; u64* tA[HB_MAXB]; ptrs_of(polys, i0, nit, P); ptrs_of(ypolys, i0, nit, Y); tmp_ptrs(c, c->tmpA, nit, tA);
    HB_TRY(launch_blk(c, -1, (const u64* const*)P, tA, nit, owned, nOwned, 0, nullptr));
    return launch_cols(c, -1, (const u64* const*)tA, Y, nit, owned, nOwned);
  }));
  return pw_simple(HB_PW_SCALE, ypolys, nullptr, nitems, owned, nOwned, sc.data(), c);
}
// hb_conv_make_y whose last step also stores the y rows into the peers' y buffers (CUDA IPC mappings)
extern "C" int hb_conv_make_y_bcast(hb_poly* const* polys, int nitems, const int32_t* D, int nD, const int32_t* owned, int nOwned,
                                    hb_poly* const* ypolys, hb_poly* const* peer_ypolys, int npeers) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(polys, nitems, &c, "hb_conv_make_y_bcast")); HB_TRY(check_polys(ypolys, nitems, &c, "hb_conv_make_y_bcast"));
  HB_TRY(check_idx(c, D, nD, "hb_conv_make_y_bcast")); HB_TRY(check_idx(c, owned, nOwned, "hb_conv_make_y_bcast(owned)", true));
  if (c->gen.on) return hb_fail(HB_ERR_UNSUPPORTED, "prime-sharded conversion is only built for power-of-two m");
  if (npeers < 0 || npeers > HB_MAXPEERS || (npeers && !peer_ypolys)) return hb_fail(HB_ERR_BAD_ARG, "hb_conv_make_y_bcast: npeers out of range");
  for (int i = 0; i < npeers * nitems; i++) {   // every peer slot is stored through: a null one is refused here, not dereferenced later
    if (!peer_ypolys[i]) return hb_fail(HB_ERR_BAD_ARG, "hb_conv_make_y_bcast: null peer polynomial handle");
    HB_TRY(check_dense(peer_ypolys[i], "hb_conv_make_y_bcast(peers)"));
  }
  if (nOwned == 0) return HB_OK;
  if (nOwned > HB_MAXROWS) return hb_fail(HB_ERR_UNSUPPORTED, "hb_conv_make_y_bcast: more than %d owned rows", HB_MAXROWS);
  std::vector<u64> sc(nOwned);
  for (int k = 0; k < nOwned; k++) {
    if (std::find(D, D + nD, owned[k]) == D + nD) return hb_fail(HB_ERR_INDEX_SET, "hb_conv_make_y_bcast: owned prime %d is not in the source set", owned[k]);
    u64 q = c->q[owned[k]], r = 1 % q;
    for (int j = 0; j < nD; j++) if (D[j] != owned[k]) r = h_mulmod(r, c->q[D[j]] % q, q);
    sc[k] = h_powmod(r, q - 2, q);
  }
  HB_TRY(ctx_scratch(c));
  if (v1_cols_ok(c) && npeers <= 8) {   // one kernel: inverse cols phase, scaling, local + peer stores
    std::vector<u64> f(nOwned);
    for (int k = 0; k < nOwned; k++) f[k] = h_mulmod(sc[k], c->h_primes[owned[k]].ninv, c->q[owned[k]]);
    return for_items(nitems, [&](int i0, int nit) {
      u64* P[HB_MAXB]; u64* Y[HB_MAXB]; u64* tA[HB_MAXB]; ptrs_of(polys, i0, nit, P); ptrs_of(ypolys, i0, nit, Y); tmp_ptrs(c, c->tmpA, nit, tA);
      u64* PE[8][HB_MAXB]; u64* const* PEp[8];
      for (int p = 0; p < npeers; p++) { for (int i = 0; i < nit; i++) PE[p][i] = peer_ypolys[(size_t)p * nitems + i0 + i]->d; PEp[p] = PE[p]; }
      HB_TRY(launch_blk(c, -1, (const u64* const*)P, tA, nit, owned, nOwned, 0, nullptr));
      return launch_cols_v1(c, -1, (const u64* const*)tA, Y, nit, owned, nOwned, f.data(), PEp, npeers);
    });
  }
  return for_items(nitems, [&](int i0, int nit) {
    u64* P[HB_MAXB]; u64* Y[HB_MAXB]; u64* tA[HB_MAXB]; ptrs_of(polys, i0, nit, P); ptrs_of(ypolys, i0, nit, Y); tmp_ptrs(c, c->tmpA, nit, tA);
    HB_TRY(launch_blk(c, -1, (const u64* const*)P, tA, nit, owned, nOwned, 0, nullptr));
    HB_TRY(launch_cols(c, -1, (const u64* const*)tA, Y, nit, owned, nOwned));
    HbBcastJob J; memset(&J, 0, sizeof(J));
    J.N = c->N; J.nitems = nit; J.npeers = npeers;
    fill_rows(J.rows, owned, nOwned);
    for (int k = 0; k < nOwned; k++) { J.scal[k] = sc[k]; J.scal_s[k] = h_shoup(sc[k], c->q[owned[k]]); }
    for (int i = 0; i < nit; i++) { J.loc[i] = Y[i]; for (int p = 0; p < npeers; p++) J.peer[p][i] = peer_ypolys[(size_t)p * nitems + i0 + i]->d; }
    unsigned gx = (unsigned)std::max<size_t>(1, c->N / (HB_THREADS * 4));
    pre_launch(c);
    HB_LAUNCH(k_scale_bcast, dim3(gx, nOwned, nit), dim3(HB_THREADS), 0, c->stream, c->d_primes, J);   // by value: graph-capturable
    return post_launch(c, "k_scale_bcast", (u64)(2 + npeers) * nOwned * nit * c->N * 8);
  });
}
// CUDA IPC: export a polynomial's device buffer / map a peer's buffer (one process per GPU)
extern "C" int hb_poly_ipc_export(hb_poly* p, void* handle64) {
  if (!p || !handle64) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_ipc_export: null");
  HB_TRY(check_dense(p, "hb_poly_ipc_export"));
#ifdef HB_SIM
  return hb_fail(HB_ERR_UNSUPPORTED, "CUDA IPC is not available in the simulator");
#else
  cudaIpcMemHandle_t h;
  HB_CUDA(cudaIpcGetMemHandle(&h, p->d));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &h, 64);
  return HB_OK;
#endif
}
extern "C" int hb_poly_ipc_open(hb_ctx* c, const void* handle64, hb_poly** out) {
  if (!c || !handle64 || !out) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_ipc_open: null");
#ifdef HB_SIM
  return hb_fail(HB_ERR_UNSUPPORTED, "CUDA IPC is not available in the simulator");
#else
  cudaIpcMemHandle_t h; memcpy(&h, handle64, 64);
  void* ptr = nullptr;
  HB_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
  hb_poly* p = new hb_poly(); p->ctx = c; p->d = (u64*)ptr; p->owned = false; p->ipc = true;
  *out = p;
  return HB_OK;
#endif
}
// mode 0: dst rows tgt = x mod q_t (addPrimes);  mode 1: dst rows tgt = (dst - x)/Q_D (scaleDownToSet)
extern "C" int hb_conv_from_y(hb_poly* const* ypolys, int nitems, const int32_t* D, int nD, const int32_t* tgt, int nT,
                              uint64_t ptxt_space, hb_poly* const* dst, int mode) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(ypolys, nitems, &c, "hb_conv_from_y")); HB_TRY(check_polys(dst, nitems, &c, "hb_conv_from_y"));
  HB_TRY(check_idx(c, D, nD, "hb_conv_from_y")); HB_TRY(check_idx(c, tgt, nT, "hb_conv_from_y(targets)", true));
  if (c->gen.on) return hb_fail(HB_ERR_UNSUPPORTED, "prime-sharded conversion is only built for power-of-two m");
  if (nT == 0) return HB_OK;
  HB_TRY(check_disjoint(D, nD, tgt, nT, "hb_conv_from_y"));
  if (ptxt_space < 1 || mode < 0 || mode > 1) return hb_fail(HB_ERR_BAD_ARG, "hb_conv_from_y: bad ptxt_space or mode");
  std::vector<u64> sc;
  if (mode == 1) HB_TRY(scalars_by_primes(c, tgt, nT, D, nD, 1, sc));
  HB_TRY(ctx_scratch(c));
  return for_items(nitems, [&](int i0, int nit) {
    u64* Y[HB_MAXB]; u64* Dp[HB_MAXB]; u64* tB[HB_MAXB]; ptrs_of(ypolys, i0, nit, Y); ptrs_of(dst, i0, nit, Dp); tmp_ptrs(c, c->tmpB, nit, tB);
    HB_TRY(conv_chunk(c, Y, nit, D, nD, tgt, nT, ptxt_space, 1));
    return launch_blk(c, +1, (const u64* const*)tB, Dp, nit, tgt, nT, mode, mode == 1 ? sc.data() : nullptr);
  });
}
// Alias caller-owned device memory ([nprimes][N] u64) as a polynomial (not freed by hb_poly_destroy).
extern "C" int hb_poly_wrap(hb_ctx* c, void* device_ptr, hb_poly** out) {
  if (!c || !device_ptr || !out) return hb_fail(HB_ERR_BAD_ARG, "hb_poly_wrap: null");
  hb_poly* p = new hb_poly(); p->ctx = c; p->d = (u64*)device_ptr; p->owned = false;
  *out = p;
  return HB_OK;
}
// Run the context's launches on a caller-provided CUDA stream (e.g. torch's current stream, so that
// NCCL collectives issued through torch.distributed are ordered with the kernels).  0 = default stream.
extern "C" int hb_ctx_set_stream(hb_ctx* c, void* cuda_stream) {
  if (!c) return hb_fail(HB_ERR_BAD_ARG, "hb_ctx_set_stream: null");
  HB_CUDA(cudaStreamSynchronize(c->stream));
  c->stream = (cudaStream_t)cuda_stream;
  c->stream_external = true;
  return HB_OK;
}

// ------------------------------------------------------------------------------------------
// digits and key switching

// The prime sets of a key switch over S, which must be a subset of the ctxt primes (src/DoubleCRT.cpp:497-498): the rows
// Sp = S | special (sorted); scp[r] = P mod q_r on the rows of S and 0 on the special rows, addPrimesAndScale(special)
// (src/Ctxt.cpp:764-768) folded into the inner product; nd = the number of digits of S (src/DoubleCRT.cpp:485-493).
struct KsSets { std::vector<int32_t> Sp; std::vector<u64> scp; int nd; };
static int ks_sets(hb_ctx* c, const int32_t* S, int nS, const char* who, KsSets& out) {
  for (int i = 0; i < nS; i++) if (c->digit_of[S[i]] < 0) return hb_fail(HB_ERR_INDEX_SET, "%s: the index set must be a subset of the ctxt primes (prime %d)", who, S[i]);
  std::vector<char> rem(c->nprimes, 0); int left = nS, nd = 0;
  for (int i = 0; i < nS; i++) rem[S[i]] = 1;
  for (; left > 0; nd++) {
    if (nd == c->ndigits) break;   // bounded: after the check above every prime of S has a digit below c->ndigits
    for (int i = 0; i < c->nprimes; i++) if (rem[i] && c->digit_of[i] == nd) { rem[i] = 0; left--; }
  }
  out.nd = nd;
  out.Sp.assign(S, S + nS); out.Sp.insert(out.Sp.end(), c->special.begin(), c->special.end()); std::sort(out.Sp.begin(), out.Sp.end());
  out.scp.assign(out.Sp.size(), 0);
  for (size_t r = 0; r < out.Sp.size(); r++)
    if (c->digit_of[out.Sp[r]] >= 0) out.scp[r] = prod_mod(c, c->special.data(), (int)c->special.size(), c->q[out.Sp[r]]);
  return HB_OK;
}
// breakIntoDigits' partition of S (src/DoubleCRT.cpp:500-513): dset[i] = the primes of S in digit i, notin[i] = the other rows
// of Sp, full[i] = every prime of digit i
static void ks_digits(hb_ctx* c, const int32_t* S, int nS, const KsSets& K, std::vector<std::vector<int32_t>>& dset,
                      std::vector<std::vector<int32_t>>& notin, std::vector<std::vector<int32_t>>& full) {
  dset.assign(K.nd, {}); notin.assign(K.nd, {}); full.assign(K.nd, {});
  for (int i = 0; i < K.nd; i++) {
    for (int j = 0; j < nS; j++) if (c->digit_of[S[j]] == i) dset[i].push_back(S[j]);
    for (int a : K.Sp) if (std::find(dset[i].begin(), dset[i].end(), a) == dset[i].end()) notin[i].push_back(a);
    for (int k = 0; k < c->nprimes; k++) if (c->digit_of[k] == i) full[i].push_back(k);
  }
}
// the amounts of the key-switching entry points; hb_automorph keeps DoubleCRT::automorph's message
static int check_amounts(hb_ctx* c, const uint64_t* k, int n) {
  for (int t = 0; t < n; t++) if (k[t] == 0 || k[t] >= c->m || h_gcd((long)k[t], (long)c->m) != 1) return hb_fail(HB_ERR_INDEX_SET, "automorph: k not in Zm*");
  return HB_OK;
}
// The matrices of n amounts: matrix t is a/b + t*ndig_evk, of which a key switch over nd digits reads the first nd columns.
// An amount k[t] == 1 needs no matrix; k == nullptr: every matrix is needed.
struct KsKeys { int n; const uint64_t* k; hb_poly* const* a; hb_poly* const* b; const char* name; };
template <class F>
static int ks_each_key(const KsKeys* sets, int nsets, int ndig_evk, F f) {
  for (int s = 0; s < nsets; s++)
    for (int t = 0; t < sets[s].n; t++)
      if (!sets[s].k || sets[s].k[t] != 1) HB_TRY(f(sets[s], (size_t)t * ndig_evk));
  return HB_OK;
}
// Every needed matrix is present, has a column for each of the nd digits and is made of this context's polys (a dense evk_b,
// an evk_a that may be seeded), and a seeded evk_a covers every row of Sp, which ks_expand_a regenerates.  Checked before
// anything is launched.  seeded (optional): some needed evk_a is seeded.
static int ks_check_keys(hb_ctx* c, const KsKeys* sets, int nsets, int nd, int ndig_evk, const std::vector<int32_t>& Sp,
                         const char* who, bool* seeded = nullptr) {
  bool any = false, sd = false;
  HB_TRY(ks_each_key(sets, nsets, ndig_evk, [&](const KsKeys& K, size_t) {
    if (!K.a || !K.b) return hb_fail(HB_ERR_BAD_ARG, "%s: no key-switching matrices (%s)", who, K.name);
    any = true;
    return HB_OK;
  }));
  if (any && (nd > ndig_evk || nd > HB_MAXDIG)) return hb_fail(HB_ERR_BAD_ARG, "%s: key-switching matrices have %d columns, need %d", who, ndig_evk, nd);
  const std::string wa = std::string(who) + "(evk_a)", wb = std::string(who) + "(evk_b)";
  HB_TRY(ks_each_key(sets, nsets, ndig_evk, [&](const KsKeys& K, size_t o) {
    hb_ctx* cx = c;
    HB_TRY(check_polys(K.a + o, nd, &cx, wa.c_str(), true)); HB_TRY(check_polys(K.b + o, nd, &cx, wb.c_str()));
    for (int i = 0; i < nd; i++) {
      const HbSeedSched* Q = K.a[o + i]->sched;
      if (!Q) continue;
      sd = true;
      for (int32_t r : Sp) if (!std::binary_search(Q->idx.begin(), Q->idx.end(), r)) return hb_fail(HB_ERR_INDEX_SET, "%s: row %d is not in the seeded set", who, r);
    }
    return HB_OK;
  }));
  if (seeded) *seeded = sd;
  return HB_OK;
}
// The accumulators are written while the operands `in` and the matrices of the sets are still being read: they must be
// distinct and alias none of them.
static int check_acc(std::set<const hb_poly*> in, const KsKeys* sets, int nsets, int nd, int ndig_evk,
                     hb_poly* const* acc0, hb_poly* const* acc1, int nitems, const char* who) {
  ks_each_key(sets, nsets, ndig_evk, [&](const KsKeys& K, size_t o) { in.insert(K.a + o, K.a + o + nd); in.insert(K.b + o, K.b + o + nd); return HB_OK; });
  std::set<const hb_poly*> out(acc0, acc0 + nitems);
  out.insert(acc1, acc1 + nitems);
  if ((int)out.size() != 2 * nitems) return hb_fail(HB_ERR_BAD_ARG, "%s: the accumulators must be distinct polynomials", who);
  for (const hb_poly* p : out) if (in.count(p)) return hb_fail(HB_ERR_BAD_ARG, "%s: an accumulator aliases an input", who);
  return HB_OK;
}

static int break_into_digits_impl(hb_poly* const* src, int nitems, const int32_t* cur, int ncur, hb_poly* const* digits, int maxdig, int* ndig_out, double* log_norms);
extern "C" int hb_break_into_digits(hb_poly* const* src, int nitems, const int32_t* cur, int ncur, hb_poly* const* digits, int maxdig, int* ndig_out) {
  return break_into_digits_impl(src, nitems, cur, ncur, digits, maxdig, ndig_out, nullptr);
}
// log_norms[item*maxdig + i] = ln ||E_i||_canon; the reference returns their sum (src/DoubleCRT.cpp:542-545)
extern "C" int hb_break_into_digits_norm(hb_poly* const* src, int nitems, const int32_t* cur, int ncur, hb_poly* const* digits, int maxdig, int* ndig_out, double* log_norms) {
  if (!log_norms) return hb_fail(HB_ERR_BAD_ARG, "hb_break_into_digits_norm: null output");
  return break_into_digits_impl(src, nitems, cur, ncur, digits, maxdig, ndig_out, log_norms);
}
static int break_into_digits_impl(hb_poly* const* src, int nitems, const int32_t* cur, int ncur, hb_poly* const* digits, int maxdig, int* ndig_out, double* log_norms) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(src, nitems, &c, "hb_break_into_digits")); HB_TRY(check_idx(c, cur, ncur, "hb_break_into_digits"));
  if (!digits || !ndig_out) return hb_fail(HB_ERR_BAD_ARG, "hb_break_into_digits: null");
  KsSets K; HB_TRY(ks_sets(c, cur, ncur, "breakIntoDigits", K));
  const int nd = K.nd;
  if (nd > maxdig) return hb_fail(HB_ERR_BAD_ARG, "breakIntoDigits: n cannot be larger than the size of context.digits");
  hb_ctx* c2 = c; HB_TRY(check_polys(digits, nitems * maxdig, &c2, "hb_break_into_digits(digits)"));
  std::vector<std::vector<int32_t>> dset, notin, full; ks_digits(c, cur, ncur, K, dset, notin, full);
  std::vector<hb_poly*> col(nitems), col2(nitems);
  for (int i = 0; i < nd; i++) {  // digits[i] = *this restricted to digit i  (src/DoubleCRT.cpp:509-513)
    for (int it = 0; it < nitems; it++) col[it] = digits[it * maxdig + i];
    HB_TRY(pw_simple(HB_PW_COPY, col.data(), src, nitems, dset[i].data(), (int)dset[i].size(), nullptr, c));
  }
  for (int i = 0; i < nd; i++) {
    for (int it = 0; it < nitems; it++) col[it] = digits[it * maxdig + i];
    std::vector<double> ln(nitems);
    HB_TRY(add_primes_impl(col.data(), nitems, dset[i].data(), (int)dset[i].size(), notin[i].data(), (int)notin[i].size(), log_norms ? ln.data() : nullptr));
    if (log_norms) for (int it = 0; it < nitems; it++) log_norms[it * maxdig + i] = ln[it];
    for (int j = i + 1; j < nd; j++) {  // digits[j] -= digits[i]; digits[j] /= pi  (src/DoubleCRT.cpp:551-556)
      for (int it = 0; it < nitems; it++) col2[it] = digits[it * maxdig + j];
      std::vector<u64> sc; HB_TRY(scalars_by_primes(c, dset[j].data(), (int)dset[j].size(), full[i].data(), (int)full[i].size(), 1, sc));
      HB_TRY(pw_simple(HB_PW_SUBSCALE, col2.data(), col.data(), nitems, dset[j].data(), (int)dset[j].size(), sc.data(), c));
    }
  }
  *ndig_out = nd;
  return HB_OK;
}

static int keyswitch_digits_impl(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* idx, int n,
                                 hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* out0, hb_poly* const* out1, const u64* scal,
                                 u64 autok, hb_poly* const* c0, hb_poly* const* own = nullptr, const int* own_dig = nullptr);
extern "C" int hb_keyswitch_digits(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* idx, int n,
                                   hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* out0, hb_poly* const* out1) {
  return keyswitch_digits_impl(digits, maxdig, ndig, nitems, idx, n, evk_a, evk_b, out0, out1, nullptr, 0, nullptr, nullptr, nullptr);
}
extern "C" int hb_keyswitch_digits_fused(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* idx, int n,
                                         hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* out0, hb_poly* const* out1,
                                         const uint64_t* scal, hb_poly* const* own, const int32_t* own_dig) {
  if (!scal) return hb_fail(HB_ERR_BAD_ARG, "hb_keyswitch_digits_fused: scal is required");
  if ((own == nullptr) != (own_dig == nullptr)) return hb_fail(HB_ERR_BAD_ARG, "hb_keyswitch_digits_fused: own and own_dig go together");
  std::vector<int> od;
  if (own_dig) { od.assign(own_dig, own_dig + n); for (int r = 0; r < n; r++) if (od[r] >= ndig || od[r] < -1) return hb_fail(HB_ERR_BAD_ARG, "hb_keyswitch_digits_fused: own_dig[%d] out of range", r); }
  if (own) { hb_ctx* c = nullptr; HB_TRY(check_polys(own, nitems, &c, "hb_keyswitch_digits_fused(own)")); }
  return keyswitch_digits_impl(digits, maxdig, ndig, nitems, idx, n, evk_a, evk_b, out0, out1, (const u64*)scal, 0, nullptr, own, own_dig ? od.data() : nullptr);
}
extern "C" int hb_sub_div_by_primes(hb_poly* const* dst, hb_poly* const* src, int nitems, const int32_t* idx, int n, const int32_t* fidx, int nf) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(dst, nitems, &c, "hb_sub_div_by_primes")); HB_TRY(check_polys(src, nitems, &c, "hb_sub_div_by_primes"));
  HB_TRY(check_idx(c, idx, n, "hb_sub_div_by_primes")); HB_TRY(check_idx(c, fidx, nf, "hb_sub_div_by_primes(factor)"));
  std::vector<u64> sc; HB_TRY(scalars_by_primes(c, idx, n, fidx, nf, 1, sc));
  return pw_simple(HB_PW_SUBSCALE, dst, src, nitems, idx, n, sc.data(), c);
}
// Hoisted automorphism + key switch (next row 8f-1): BasicAutomorphPrecon::automorph (src/matmul.cpp:112-184).
extern "C" int hb_automorph_keyswitch_digits(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* S, int nS,
                                             hb_poly* const* c0, uint64_t k, hb_poly* const* evk_a, hb_poly* const* evk_b,
                                             hb_poly* const* out0, hb_poly* const* out1) {
  static const char* who = "hb_automorph_keyswitch_digits";
  hb_ctx* c = nullptr; HB_TRY(check_polys(c0, nitems, &c, who));
  HB_TRY(check_idx(c, S, nS, who));
  KsSets K; HB_TRY(ks_sets(c, S, nS, who, K));
  HB_TRY(check_amounts(c, &k, 1));
  if (ndig <= 0 || ndig > maxdig) return hb_fail(HB_ERR_BAD_ARG, "%s: ndig=%d out of range", who, ndig);
  HB_TRY(check_polys(out0, nitems, &c, "hb_automorph_keyswitch_digits(out0)")); HB_TRY(check_polys(out1, nitems, &c, "hb_automorph_keyswitch_digits(out1)"));
  HB_TRY(check_polys(digits, nitems * maxdig, &c, "hb_automorph_keyswitch_digits(digits)"));
  // the caller's ndig digits are key-switched whatever k is, so the matrix is always read
  const KsKeys key = {1, nullptr, evk_a, evk_b, "evk"};
  HB_TRY(ks_check_keys(c, &key, 1, ndig, ndig, K.Sp, who));
  for (int i = 0; i < nitems; i++) if (c0[i] == out0[i] || c0[i] == out1[i]) return hb_fail(HB_ERR_BAD_ARG, "%s: outputs must not alias c0", who);
  for (int i = 0; i < nitems * maxdig; i++) for (int j = 0; j < nitems; j++) if (digits[i] == out0[j] || digits[i] == out1[j]) return hb_fail(HB_ERR_BAD_ARG, "%s: outputs must not alias the digits", who);
  // ---- every argument is checked: nothing was launched before this point
  const std::vector<int32_t>& Sp = K.Sp;
  if (c->gen.on) {
    // general m: sigma_k is a gather over Z_m^* (src/DoubleCRT.cpp:1160-1202), applied to the digits and to c0 in scratch
    // polynomials (the digits themselves stay reusable for the next amount), then the same inner product
    std::vector<hb_poly*> tmp; HB_TRY(pool_get(c, nitems * ndig, tmp));
    std::vector<hb_poly*> col(nitems), dcol(nitems);
    for (int i = 0; i < ndig; i++) {
      for (int it = 0; it < nitems; it++) { col[it] = tmp[(size_t)it * ndig + i]; dcol[it] = digits[(size_t)it * maxdig + i]; }
      HB_TRY(hb_automorph(col.data(), dcol.data(), nitems, Sp.data(), (int)Sp.size(), k));
    }
    HB_TRY(hb_automorph(out0, c0, nitems, S, nS, k));
    HB_TRY(hb_zero_rows(out1, nitems, Sp.data(), (int)Sp.size()));
    return keyswitch_digits_impl(tmp.data(), ndig, ndig, nitems, Sp.data(), (int)Sp.size(), evk_a, evk_b, out0, out1, K.scp.data(), 0, nullptr, nullptr, nullptr);
  }
  return keyswitch_digits_impl(digits, maxdig, ndig, nitems, Sp.data(), (int)Sp.size(), evk_a, evk_b, out0, out1, K.scp.data(), k, c0, nullptr, nullptr);
}
// scal (optional, [n]): out = scal[r]*out + sum (0 => out = sum): addPrimesAndScale folded in.
// autok != 0: digits and c0 are read through the automorphism sigma_autok (hoisting), out0/out1 are pure outputs.
// own / own_dig (fused breakIntoDigits): rows idx[r] with own_dig[r] = i >= 0 read digit i from own[item] instead of digits[item][i].
static int keyswitch_digits_impl(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* idx, int n,
                                 hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* out0, hb_poly* const* out1, const u64* scal,
                                 u64 autok, hb_poly* const* c0, hb_poly* const* own, const int* own_dig) {
  hb_ctx* c = nullptr;
  HB_TRY(check_polys(out0, nitems, &c, "hb_keyswitch_digits")); HB_TRY(check_polys(out1, nitems, &c, "hb_keyswitch_digits"));
  if (ndig <= 0 || ndig > HB_MAXDIG || ndig > maxdig) return hb_fail(HB_ERR_BAD_ARG, "hb_keyswitch_digits: ndig=%d out of range", ndig);
  HB_TRY(check_polys(evk_a, ndig, &c, "hb_keyswitch_digits(evk_a)", true)); HB_TRY(check_polys(evk_b, ndig, &c, "hb_keyswitch_digits(evk_b)"));
  HB_TRY(check_polys(digits, nitems * maxdig, &c, "hb_keyswitch_digits(digits)"));
  HB_TRY(check_idx(c, idx, n, "hb_keyswitch_digits"));
  // a seeded evk_a is regenerated here, before the item chunks; the fused relinearisation hands in entries it already regenerated
  std::vector<hb_poly*> ka; HB_TRY(ks_expand_a(c, evk_a, ndig, idx, n, ka)); evk_a = ka.data();
  return for_items(nitems, [&](int i0, int nit) {
    for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
      int nr = std::min(HB_MAXROWS, n - r0);
      HbKsJob J; memset(&J, 0, sizeof(J));
      J.logN = c->logN; J.N = c->N; J.ndig = ndig; J.nitems = nit;
      fill_rows(J.rows, idx + r0, nr);
      if (scal) { J.mode = 1; for (int i = 0; i < nr; i++) J.scal[i] = scal[r0 + i]; }
      if (autok) { J.mode = 2; J.ak = autok; J.am = c->m; for (int it = 0; it < nit; it++) J.c0[it] = c0[i0 + it]->d; }
      for (int i = 0; i < ndig; i++) { J.evk_a[i] = evk_a[i]->d; J.evk_b[i] = evk_b[i]->d; }
      for (int it = 0; it < nit; it++) {
        J.out0[it] = out0[i0 + it]->d; J.out1[it] = out1[i0 + it]->d;
        for (int i = 0; i < ndig; i++) J.dig[it][i] = digits[(i0 + it) * maxdig + i]->d;
      }
      for (int i = 0; i < nr; i++) J.own_dig[i] = own_dig ? (signed char)own_dig[r0 + i] : (signed char)-1;
      if (own) for (int it = 0; it < nit; it++) J.own[it] = own[i0 + it]->d;
      const bool stream_form = !c->gen.on && !autok && ndig <= 4 && c->N % 512 == 0 && !getenv("HB_KS_V0");
      if (own && !stream_form) return hb_fail(HB_ERR_UNSUPPORTED, "hb_keyswitch_digits: aliased digit rows need the streaming kernel");
      if (stream_form) {
        // item groups: enough CTAs for a few waves, as few re-fetches of the key rows as possible
        const long per = (long)(c->N / 512) * nr;
        int z = 1; while (z < nit && per * z < 8L * c->resident_ctas) z *= 2;
        dim3 g((unsigned)(c->N / 512), nr, std::min(z, nit));
        pre_launch(c);
        switch (ndig) {
          case 1: HB_LAUNCH(k1_ks_inner<1>, g, dim3(256), 0, c->stream, c->d_primes, J); break;
          case 2: HB_LAUNCH(k1_ks_inner<2>, g, dim3(256), 0, c->stream, c->d_primes, J); break;
          case 3: HB_LAUNCH(k1_ks_inner<3>, g, dim3(256), 0, c->stream, c->d_primes, J); break;
          default: HB_LAUNCH(k1_ks_inner<4>, g, dim3(256), 0, c->stream, c->d_primes, J); break;
        }
        HB_TRY(post_launch(c, "k1_ks_inner", ((u64)(ndig + 4) * nit + 2 * ndig) * nr * c->N * 8));
        continue;
      }
      unsigned gx = (unsigned)std::max<size_t>(1, c->N / (HB_THREADS * 4));
      pre_launch(c);
      HB_LAUNCH(k_ks_inner, dim3(gx, nr, nit), dim3(HB_THREADS), 0, c->stream, c->d_primes, J);
      // reads ndig digit rows + out0,out1 per item, 2*ndig evk rows once; writes out0,out1
      HB_TRY(post_launch(c, "k_ks_inner", ((u64)(ndig + 4) * nit + 2 * ndig) * nr * c->N * 8));
    }
    return HB_OK;
  });
}

// Hoisted linear map (SURVEY 8f-1): the loop body of MatMul1DExec::mul's native FULL branch (src/matmul.cpp:1226-1252),
// sum_j consts[j] * BasicAutomorphPrecon::automorph(k[j]), in one k_ks_linmap launch per group of up to HB_LINMAP_MAXAMT
// amounts (and per item chunk and row chunk).  No permuted digit copies and no intermediate rows: sigma_k is applied while
// the digits and c0 are loaded, for general m too.
extern "C" int hb_hoisted_linear_map(hb_poly* const* digits, int maxdig, int ndig, int nitems, const int32_t* S, int nS,
                                     hb_poly* const* c0, hb_poly* const* c1, int namt, const uint64_t* k, hb_poly* const* consts,
                                     hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* acc0, hb_poly* const* acc1,
                                     int accumulate) {
  static const char* who = "hb_hoisted_linear_map";
  hb_ctx* c = nullptr;
  HB_TRY(check_polys(c0, nitems, &c, who));
  HB_TRY(check_idx(c, S, nS, who));
  if (namt <= 0 || !k || !consts) return hb_fail(HB_ERR_BAD_ARG, "%s: no amounts", who);
  if (ndig <= 0 || ndig > maxdig || ndig > HB_MAXDIG) return hb_fail(HB_ERR_BAD_ARG, "%s: ndig=%d out of range", who, ndig);
  HB_TRY(check_amounts(c, k, namt));
  KsSets K; HB_TRY(ks_sets(c, S, nS, who, K));
  if (!c1 && std::find(k, k + namt, (uint64_t)1) != k + namt) return hb_fail(HB_ERR_BAD_ARG, "%s: c1 is required when some k == 1", who);
  if (c1) HB_TRY(check_polys(c1, nitems, &c, "hb_hoisted_linear_map(c1)"));
  HB_TRY(check_polys(digits, nitems * maxdig, &c, "hb_hoisted_linear_map(digits)"));
  HB_TRY(check_polys(consts, namt, &c, "hb_hoisted_linear_map(consts)"));
  HB_TRY(check_polys(acc0, nitems, &c, "hb_hoisted_linear_map(acc0)")); HB_TRY(check_polys(acc1, nitems, &c, "hb_hoisted_linear_map(acc1)"));
  const KsKeys keys = {namt, k, evk_a, evk_b, "evk"};
  bool seeded; HB_TRY(ks_check_keys(c, &keys, 1, ndig, ndig, K.Sp, who, &seeded));
  std::set<const hb_poly*> in(c0, c0 + nitems);
  in.insert(digits, digits + (size_t)nitems * maxdig); in.insert(consts, consts + namt);
  if (c1) in.insert(c1, c1 + nitems);
  HB_TRY(check_acc(in, &keys, 1, ndig, ndig, acc0, acc1, nitems, who));
  // ---- every argument is checked: nothing was launched before this point
  const std::vector<int32_t>& Sp = K.Sp;
  const int nSp = (int)Sp.size();
  // amounts per launch; with seeded keys also per regeneration, whose scratch stays at HB_LINMAP_SEEDED polys
  const int achunk = seeded ? std::max(1, HB_LINMAP_SEEDED / ndig) : HB_LINMAP_MAXAMT;
  std::vector<hb_poly*> list, ka;
  std::vector<int> slot;
  for (int t0 = 0; t0 < namt; t0 += achunk) {
    const int na = std::min(achunk, namt - t0);
    list.clear(); slot.assign((size_t)na, -1);
    for (int a = 0; a < na; a++)
      if (k[t0 + a] != 1) { slot[(size_t)a] = (int)list.size(); list.insert(list.end(), evk_a + (size_t)(t0 + a) * ndig, evk_a + (size_t)(t0 + a + 1) * ndig); }
    if (!list.empty()) HB_TRY(ks_expand_a(c, list.data(), (int)list.size(), Sp.data(), nSp, ka));
    u64 item_rows = 0, shared_rows = 0;   // rows read per item and shared by the items, per row of the launch
    for (int a = 0; a < na; a++) { item_rows += k[t0 + a] == 1 ? 2 : ndig + 1; shared_rows += k[t0 + a] == 1 ? 1 : 2 * ndig + 1; }
    const bool acc = accumulate || t0 > 0;
    HB_TRY(for_items(nitems, [&](int i0, int nit) {
      for (int r0 = 0; r0 < nSp; r0 += HB_MAXROWS) {
        const int nr = std::min(HB_MAXROWS, nSp - r0);
        HbLinJob J; memset(&J, 0, sizeof(J));
        J.N = c->N; J.m = c->m;
        if (c->gen.on) { J.rep = c->gen.d_rep; J.irep = c->gen.d_irep; }
        J.ndig = ndig; J.nitems = nit; J.namt = na; J.accumulate = acc ? 1 : 0;
        fill_rows(J.rows, Sp.data() + r0, nr);
        for (int i = 0; i < nr; i++) J.scal[i] = K.scp[(size_t)(r0 + i)];
        for (int a = 0; a < na; a++) {
          const int t = t0 + a;
          J.k[a] = k[t]; J.cst[a] = consts[t]->d;
          if (slot[(size_t)a] >= 0)
            for (int i = 0; i < ndig; i++) { J.evk_a[a][i] = ka[(size_t)slot[(size_t)a] + i]->d; J.evk_b[a][i] = evk_b[(size_t)t * ndig + i]->d; }
        }
        for (int it = 0; it < nit; it++) {
          J.c0[it] = c0[i0 + it]->d; J.c1[it] = c1 ? c1[i0 + it]->d : nullptr;
          J.acc0[it] = acc0[i0 + it]->d; J.acc1[it] = acc1[i0 + it]->d;
          for (int i = 0; i < ndig; i++) J.dig[it][i] = digits[(size_t)(i0 + it) * maxdig + i]->d;
        }
        const int ni = nit >= 4 ? 4 : nit >= 2 ? 2 : 1;
        const dim3 g((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS), (unsigned)nr, (unsigned)((nit + ni - 1) / ni));
        pre_launch(c);
        switch (ni) {
          case 1: HB_LAUNCH(k_ks_linmap<1>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
          case 2: HB_LAUNCH(k_ks_linmap<2>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
          default: HB_LAUNCH(k_ks_linmap<4>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
        }
        // per item: its digit and c0 (or c0 and c1) rows per amount, two accumulators written (and read when accumulating);
        // per launch: the key rows and the constant of every amount, once
        HB_TRY(post_launch(c, "k_ks_linmap", ((item_rows + (acc ? 4 : 2)) * nit + shared_rows) * nr * c->N * 8));
      }
      return HB_OK;
    }));
  }
  return HB_OK;
}

// BSGS linear map (SURVEY 8f-1): the giant-step phase of MatMul1DExec::mul's non-iterative BSGS branches (src/matmul.cpp:
// 1022-1057 native, 1097-1142 bad dimension).  Work goes in groups of at most HB_BSGS_GROUP (giant step, item) pairs, so the
// scratch is HB_BSGS_GROUP*(2+ndig) polys whatever the number of giant steps.  Per group: k_bsgs_mac forms the rotated
// inner sums, the extended form's mod-down and breakIntoDigits run once over all of the group's rotated sums, and
// k_ks_giant key-switches and sums them into the accumulators.
static int bsgs_impl(hb_poly* const* baby0, hb_poly* const* baby1, int nbaby, int nitems, const int32_t* S, int nS, int extended,
                     uint64_t ptxt_space, int ngiant, const uint64_t* kgiant, hb_poly* const* consts, const uint64_t* scal,
                     hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk, hb_poly* const* acc0, hb_poly* const* acc1,
                     int accumulate, double* norms);
extern "C" int hb_bsgs_linear_map(hb_poly* const* baby0, hb_poly* const* baby1, int nbaby, int nitems,
                                  const int32_t* S, int nS, int extended, uint64_t ptxt_space,
                                  int ngiant, const uint64_t* kgiant, hb_poly* const* consts, const uint64_t* scal,
                                  hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk,
                                  hb_poly* const* acc0, hb_poly* const* acc1, int accumulate) {
  return bsgs_impl(baby0, baby1, nbaby, nitems, S, nS, extended, ptxt_space, ngiant, kgiant, consts, scal, evk_a, evk_b, ndig_evk,
                   acc0, acc1, accumulate, nullptr);
}
// norms[(item*ngiant + t)*(HB_MAXDIG + 2) + i]: ln ||E_i|| of the digits of rotated giant step t (i < ndig), then ||delta/P||
// of its two parts' mod-down (extended form) -- what keySwitchPart and modDownToSet add to the noise bound
extern "C" int hb_bsgs_linear_map_norm(hb_poly* const* baby0, hb_poly* const* baby1, int nbaby, int nitems,
                                       const int32_t* S, int nS, int extended, uint64_t ptxt_space,
                                       int ngiant, const uint64_t* kgiant, hb_poly* const* consts, const uint64_t* scal,
                                       hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk,
                                       hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms) {
  if (!norms) return hb_fail(HB_ERR_BAD_ARG, "hb_bsgs_linear_map_norm: null output");
  return bsgs_impl(baby0, baby1, nbaby, nitems, S, nS, extended, ptxt_space, ngiant, kgiant, consts, scal, evk_a, evk_b, ndig_evk,
                   acc0, acc1, accumulate, norms);
}
// Terms per k_ks_giant launch: the 128-bit budget, and with seeded keys the key scratch (HB_LINMAP_SEEDED polys)
static int bsgs_tmax(int nd, bool seeded) {
  return std::max(1, std::min(254 / (nd + 1), seeded ? HB_LINMAP_SEEDED / std::max(1, nd) : HB_BSGS_GROUP));
}
// BSGS step 1 over one group of nit items (of at most ic): slot a*nit + it of X0/X1 (+)= sigma_{k_a}( scal[a] * sum_b cst(a, b) * baby(it, b) ) over the rows
// R, for a < ng, it < nit, b < nbaby.  cst(a, b) is the constant (null: a zero diagonal) and baby(it, b) the two parts of a
// baby step; kinv[a] = k_a^-1 mod m; accumulate adds to the sums already in the slots.  One k_bsgs_mac pass per NI items,
// NT terms, nbl baby steps and HB_MAXROWS rows.
template <class CstF, class BabyF>
static int bsgs_mac(hb_ctx* c, const std::vector<int32_t>& R, hb_poly* const* X0, hb_poly* const* X1, int ic, int nit, int ng, int nbaby,
                    const u64* kinv, const uint64_t* scal, bool accumulate, CstF cst, BabyF baby) {
  const int nR = (int)R.size();
  const int NI = ic >= 4 ? 4 : ic >= 2 ? 2 : 1, NT = HB_BSGS_MACW / NI;
  const int nbl = std::min(HB_BSGS_MAXBABY, std::min(HB_BSGS_CST / NT, HB_BSGS_BABY / NI));   // baby steps per k_bsgs_mac launch
  for (int u0 = 0; u0 < nit; u0 += NI) {
    const int ni = std::min(NI, nit - u0);
    for (int a0 = 0; a0 < ng; a0 += NT) {
      const int nt = std::min(NT, ng - a0);
      for (int b0 = 0; b0 < nbaby; b0 += nbl) {
        const int nb = std::min(nbl, nbaby - b0);
        const bool add = accumulate || b0 > 0;
        for (int r0 = 0; r0 < nR; r0 += HB_MAXROWS) {
          const int nr = std::min(HB_MAXROWS, nR - r0);
          HbBsgsMacJob J; memset(&J, 0, sizeof(J));
          J.N = c->N; J.m = c->m;
          if (c->gen.on) { J.rep = c->gen.d_rep; J.irep = c->gen.d_irep; }
          J.nb = nb; J.nt = nt; J.ni = ni; J.accumulate = add;
          fill_rows(J.rows, R.data() + r0, nr);
          u64 ncst = 0;
          for (int a = 0; a < nt; a++) {
            J.kinv[a] = kinv[a0 + a]; J.scal[a] = scal ? scal[a0 + a] : 1;
            for (int b = 0; b < nb; b++) {
              hb_poly* cp = cst(a0 + a, b0 + b);
              J.cst[a * nb + b] = cp ? cp->d : nullptr;
              ncst += cp != nullptr;
            }
            for (int u = 0; u < ni; u++) {
              const int s = (a0 + a) * nit + u0 + u;
              J.out0[a * NI + u] = X0[s]->d; J.out1[a * NI + u] = X1[s]->d;
            }
          }
          for (int u = 0; u < ni; u++)
            for (int b = 0; b < nb; b++) {
              const std::pair<hb_poly*, hb_poly*> x = baby(u0 + u, b0 + b);
              J.baby0[u * nb + b] = x.first->d; J.baby1[u * nb + b] = x.second->d;
            }
          const dim3 g((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS), (unsigned)nr, 1);
          pre_launch(c);
          switch (NI) {
            case 1: HB_LAUNCH(k_bsgs_mac<1>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
            case 2: HB_LAUNCH(k_bsgs_mac<2>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
            default: HB_LAUNCH(k_bsgs_mac<4>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
          }
          // the baby rows of the items and the constant rows of the giant steps once; two sums written per pair
          // (and read when a later baby chunk adds to them)
          HB_TRY(post_launch(c, "k_bsgs_mac", ((u64)2 * ni * nb + ncst + (u64)(add ? 4 : 2) * ni * nt) * nr * c->N * 8));
        }
      }
    }
  }
  return HB_OK;
}
// BSGS steps 2-3 over one group of ng terms of nit items, slot a*nit + it of X0/X1 holding term a's rotated sum (digits in
// DG[slot*nd ..]): for kt[a] != 1 the mod-down to S (extended form) and breakIntoDigits, batched over the group, then the key
// switch with matrix a (evk_a/evk_b + a*ndig_evk) and the unrotated terms, summed into acc0/acc1[it], tmax terms and at most
// HB_BSGS_GROUP slots per k_ks_giant launch.  acc_on: the accumulators hold a sum (becomes true).  norms (optional): term a
// of item it at norms + (it*nstride + a)*(HB_MAXDIG + 2), as hb_bsgs_linear_map_norm lays them out.
static int bsgs_finish(hb_ctx* c, hb_poly* const* X0, hb_poly* const* X1, hb_poly* const* DG, int nit, int ng, const uint64_t* kt,
                       hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk, int nd, const int32_t* S, int nS,
                       const std::vector<int32_t>& Sp, int extended, uint64_t ptxt_space, const std::vector<u64>& scp,
                       const std::vector<u64>& scx, int tmax, bool seeded, hb_poly* const* acc0, hb_poly* const* acc1, bool& acc_on,
                       double* norms, size_t nstride) {
  const int nSp = (int)Sp.size();
  tmax = std::max(1, std::min(tmax, HB_BSGS_GROUP / nit));
  std::vector<hb_poly*> rot0, rot01, rdig, list, ka;
  // 2. the rotated sums' mod-down (extended form) and digits, batched over the group
  for (int a = 0; a < ng; a++) {
    if (kt[a] == 1) continue;
    for (int it = 0; it < nit; it++) {
      const int s = a * nit + it;
      rot0.push_back(X1[s]); rot01.push_back(X0[s]); rot01.push_back(X1[s]);
      for (int i = 0; i < nd; i++) rdig.push_back(DG[(size_t)s * nd + i]);
    }
  }
  if (!rot0.empty()) {
    std::vector<double> sdn(norms && extended ? rot01.size() : 0), ldn(norms ? rdig.size() : 0);
    if (extended) HB_TRY(scale_down_impl(rot01.data(), (int)rot01.size(), Sp.data(), nSp, S, nS, ptxt_space, norms ? sdn.data() : nullptr));
    int ndo = 0;
    HB_TRY(break_into_digits_impl(rot0.data(), (int)rot0.size(), S, nS, rdig.data(), nd, &ndo, norms ? ldn.data() : nullptr));
    for (int a = 0, r = 0; norms && a < ng; a++) {
      if (kt[a] == 1) continue;
      for (int it = 0; it < nit; it++, r++) {
        double* o = norms + ((size_t)it * nstride + a) * (HB_MAXDIG + 2);
        for (int i = 0; i < nd; i++) o[i] = ldn[(size_t)r * nd + i];
        if (extended) { o[HB_MAXDIG] = sdn[(size_t)2 * r]; o[HB_MAXDIG + 1] = sdn[(size_t)2 * r + 1]; }
      }
    }
  }
  // 3. key switch and sum, tmax terms per launch
  for (int a0 = 0; a0 < ng;) {
    int nt = 0, nrot = 0;
    while (a0 + nt < ng && nt < tmax) { nrot += kt[a0 + nt] != 1; nt++; if (seeded && (nrot + 1) * nd > HB_LINMAP_SEEDED) break; }
    list.clear();
    for (int a = 0; a < nt; a++) {
      const int t = a0 + a;
      if (kt[t] != 1) list.insert(list.end(), evk_a + (size_t)t * ndig_evk, evk_a + (size_t)t * ndig_evk + nd);
    }
    if (!list.empty()) HB_TRY(ks_expand_a(c, list.data(), (int)list.size(), Sp.data(), nSp, ka));
    u64 item_rows = 0, key_rows = 0;   // rows read per item and shared by the items, per row of the launch
    for (int r0 = 0; r0 < nSp; r0 += HB_MAXROWS) {
      const int nr = std::min(HB_MAXROWS, nSp - r0);
      HbGiantJob J; memset(&J, 0, sizeof(J));
      J.N = c->N; J.ndig = nd; J.nitems = nit; J.nt = nt; J.accumulate = acc_on ? 1 : 0;
      fill_rows(J.rows, Sp.data() + r0, nr);
      for (int i = 0; i < nr; i++) { J.scp[i] = scp[(size_t)(r0 + i)]; J.scx[i] = scx[(size_t)(r0 + i)]; }
      item_rows = 0; key_rows = 0;
      for (int a = 0, slot = 0; a < nt; a++) {
        const int t = a0 + a;
        J.plain[a] = kt[t] == 1;
        if (!J.plain[a]) {
          for (int i = 0; i < nd; i++) { J.evk_a[a][i] = ka[(size_t)slot * nd + i]->d; J.evk_b[a][i] = evk_b[(size_t)t * ndig_evk + i]->d; }
          slot++;
        }
        item_rows += J.plain[a] ? 2 : nd + 1; key_rows += J.plain[a] ? 0 : 2 * nd;
        for (int it = 0; it < nit; it++) {
          const int s = (a0 + a) * nit + it, sl = a * nit + it;
          J.x0[sl] = X0[s]->d; J.x1[sl] = X1[s]->d;
          for (int i = 0; i < nd && !J.plain[a]; i++) J.dig[sl][i] = DG[(size_t)s * nd + i]->d;
        }
      }
      for (int it = 0; it < nit; it++) { J.acc0[it] = acc0[it]->d; J.acc1[it] = acc1[it]->d; }
      const int ni = nit >= 4 ? 4 : nit >= 2 ? 2 : 1;
      const dim3 g((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS), (unsigned)nr, (unsigned)((nit + ni - 1) / ni));
      pre_launch(c);
      switch (ni) {
        case 1: HB_LAUNCH(k_ks_giant<1>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
        case 2: HB_LAUNCH(k_ks_giant<2>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
        default: HB_LAUNCH(k_ks_giant<4>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
      }
      HB_TRY(post_launch(c, "k_ks_giant", ((item_rows + (acc_on ? 4 : 2)) * nit + key_rows) * nr * c->N * 8));
    }
    acc_on = true;
    a0 += nt;
  }
  return HB_OK;
}
static int bsgs_impl(hb_poly* const* baby0, hb_poly* const* baby1, int nbaby, int nitems, const int32_t* S, int nS, int extended,
                     uint64_t ptxt_space, int ngiant, const uint64_t* kgiant, hb_poly* const* consts, const uint64_t* scal,
                     hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk, hb_poly* const* acc0, hb_poly* const* acc1,
                     int accumulate, double* norms) {
  static const char* who = "hb_bsgs_linear_map";
  hb_ctx* c = nullptr;
  if (nbaby <= 0 || nitems <= 0 || ngiant <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: nbaby, nitems and ngiant must be positive", who);
  if (extended != 0 && extended != 1) return hb_fail(HB_ERR_BAD_ARG, "%s: extended must be 0 or 1", who);
  if (!kgiant || !consts) return hb_fail(HB_ERR_BAD_ARG, "%s: no giant steps", who);
  HB_TRY(check_polys(baby0, nitems * nbaby, &c, "hb_bsgs_linear_map(baby0)"));
  HB_TRY(check_polys(baby1, nitems * nbaby, &c, "hb_bsgs_linear_map(baby1)"));
  HB_TRY(check_idx(c, S, nS, who));
  if (ptxt_space < 1) return hb_fail(HB_ERR_BAD_ARG, "%s: ptxt_space must be at least 1", who);
  if (c->special.empty()) return hb_fail(HB_ERR_BAD_ARG, "%s: context has no special primes", who);
  KsSets K; HB_TRY(ks_sets(c, S, nS, who, K));
  HB_TRY(check_amounts(c, kgiant, ngiant));
  // reLinearize applies relin_CKKS_adjust after the mod-down (src/Ctxt.cpp:733-736), which a factor folded into the sum
  // would precede; it is 1 for BGV, whose bad dimensions are the extended form's callers
  for (int t = 0; extended && scal && t < ngiant; t++) if (scal[t] != 1) return hb_fail(HB_ERR_BAD_ARG, "%s: scal must be 1 in the extended form", who);
  for (int i = 0; i < ngiant * nbaby; i++) if (consts[i]) HB_TRY(check_polys(consts + i, 1, &c, "hb_bsgs_linear_map(consts)"));
  HB_TRY(check_polys(acc0, nitems, &c, "hb_bsgs_linear_map(acc0)")); HB_TRY(check_polys(acc1, nitems, &c, "hb_bsgs_linear_map(acc1)"));
  const KsKeys keys = {ngiant, kgiant, evk_a, evk_b, "evk"};
  const int nd = K.nd;
  bool seeded; HB_TRY(ks_check_keys(c, &keys, 1, nd, ndig_evk, K.Sp, who, &seeded));
  std::set<const hb_poly*> in(baby0, baby0 + (size_t)nitems * nbaby);
  in.insert(baby1, baby1 + (size_t)nitems * nbaby);
  for (int i = 0; i < ngiant * nbaby; i++) if (consts[i]) in.insert(consts[i]);
  HB_TRY(check_acc(in, &keys, 1, nd, ndig_evk, acc0, acc1, nitems, who));
  // ---- every argument is checked: nothing was launched before this point
  const std::vector<int32_t>& Sp = K.Sp;
  const std::vector<u64>& scp = K.scp;
  const std::vector<u64> scx = extended ? std::vector<u64>(Sp.size(), 1) : scp;
  std::vector<u64> kinv((size_t)ngiant);
  for (int t = 0; t < ngiant; t++) h_invmod(kgiant[t], c->m, &kinv[(size_t)t]);
  const std::vector<int32_t> R = extended ? Sp : std::vector<int32_t>(S, S + nS);   // the rows of the baby steps
  // scratch: slot s of a group holds the rotated sum (x0, x1) of one (giant step, item) and its nd digits
  const int G = std::min(HB_BSGS_GROUP, nitems * ngiant);   // a group never holds more pairs than the call has
  while ((int)c->bsgs.size() < G * (2 + nd)) { hb_poly* p; HB_TRY(hb_poly_create(c, &p)); c->bsgs.push_back(p); }
  hb_poly* const* X0 = c->bsgs.data();
  hb_poly* const* X1 = X0 + G;
  hb_poly* const* DG = X0 + 2 * G;
  const int ic = std::min(nitems, G);                 // items per group
  const int gg = std::max(1, G / ic);                 // giant steps per group
  const int tmax = bsgs_tmax(nd, seeded);
  bool acc_on = accumulate != 0;
  for (int i0 = 0; i0 < nitems; i0 += ic) {
    const int nit = std::min(ic, nitems - i0);
    acc_on = accumulate != 0;
    for (int t0 = 0; t0 < ngiant; t0 += gg) {
      const int ng = std::min(gg, ngiant - t0);
      // 1. the rotated inner sums of the group: slot a*nit + it
      HB_TRY(bsgs_mac(c, R, X0, X1, ic, nit, ng, nbaby, kinv.data() + t0, scal ? scal + t0 : nullptr, false,
                      [&](int a, int b) { return consts[(size_t)(t0 + a) * nbaby + b]; },
                      [&](int u, int b) { const size_t e = (size_t)(i0 + u) * nbaby + b; return std::make_pair(baby0[e], baby1[e]); }));
      // 2-3. their mod-down (extended form), digits and key switch, summed into the accumulators
      HB_TRY(bsgs_finish(c, X0, X1, DG, nit, ng, kgiant + t0, evk_a + (size_t)t0 * ndig_evk, evk_b + (size_t)t0 * ndig_evk, ndig_evk, nd,
                         S, nS, Sp, extended, ptxt_space, scp, scx, tmax, seeded, acc0 + i0, acc1 + i0, acc_on,
                         norms ? norms + ((size_t)i0 * ngiant + t0) * (HB_MAXDIG + 2) : nullptr, (size_t)ngiant));
    }
  }
  return HB_OK;
}

// Block linear map (SURVEY 8f-1): BlockMatMul1DExec::mul's non-iterative branches with one interval (src/matmul.cpp:1782-1868
// native, 1869-1974 bad dimension).  Output o < n1*(bad ? 2 : 1) is set o / n1's sum for outer amount k1[o % n1].  Per item
// chunk and per group of outputs: k_ks_hoist writes the hoisted rotations of a chunk of at most HB_HOIST_SLOTS / items
// inner amounts, k_bsgs_mac folds them into the group's rotated sums (the rotations play the baby steps, the outer amounts
// the giant steps), and bsgs_finish mod-downs, key-switches and sums them -- the set-0 sums into the accumulators, the set-1
// sums into a scratch sum that is finally rotated by kfinal and added.  When all inner amounts fit one chunk, the rotations
// are formed once per item chunk; otherwise once per chunk and group.
#define HB_BLOCK_GROUP 64       // outputs x items per group
extern "C" int hb_automorph(hb_poly* const* dst, hb_poly* const* src, int nitems, const int32_t* idx, int n, uint64_t k);
static int block_impl(hb_poly* const* digits, int maxdig, int nitems, const int32_t* S, int nS, hb_poly* const* c0, hb_poly* const* c1,
                      uint64_t ptxt_space, int n0, const uint64_t* k0, hb_poly* const* evk0_a, hb_poly* const* evk0_b,
                      int n1, const uint64_t* k1, hb_poly* const* evk1_a, hb_poly* const* evk1_b,
                      hb_poly* const* consts, hb_poly* const* consts1, uint64_t kfinal, hb_poly* const* evkf_a, hb_poly* const* evkf_b,
                      int ndig_evk, hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms);
extern "C" int hb_block_linear_map(hb_poly* const* digits, int maxdig, int nitems, const int32_t* S, int nS,
                                   hb_poly* const* c0, hb_poly* const* c1, uint64_t ptxt_space,
                                   int n0, const uint64_t* k0, hb_poly* const* evk0_a, hb_poly* const* evk0_b,
                                   int n1, const uint64_t* k1, hb_poly* const* evk1_a, hb_poly* const* evk1_b,
                                   hb_poly* const* consts, hb_poly* const* consts1, uint64_t kfinal,
                                   hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                                   hb_poly* const* acc0, hb_poly* const* acc1, int accumulate) {
  return block_impl(digits, maxdig, nitems, S, nS, c0, c1, ptxt_space, n0, k0, evk0_a, evk0_b, n1, k1, evk1_a, evk1_b, consts, consts1,
                    kfinal, evkf_a, evkf_b, ndig_evk, acc0, acc1, accumulate, nullptr);
}
extern "C" int hb_block_linear_map_norm(hb_poly* const* digits, int maxdig, int nitems, const int32_t* S, int nS,
                                        hb_poly* const* c0, hb_poly* const* c1, uint64_t ptxt_space,
                                        int n0, const uint64_t* k0, hb_poly* const* evk0_a, hb_poly* const* evk0_b,
                                        int n1, const uint64_t* k1, hb_poly* const* evk1_a, hb_poly* const* evk1_b,
                                        hb_poly* const* consts, hb_poly* const* consts1, uint64_t kfinal,
                                        hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                                        hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms) {
  if (!norms) return hb_fail(HB_ERR_BAD_ARG, "hb_block_linear_map_norm: null output");
  return block_impl(digits, maxdig, nitems, S, nS, c0, c1, ptxt_space, n0, k0, evk0_a, evk0_b, n1, k1, evk1_a, evk1_b, consts, consts1,
                    kfinal, evkf_a, evkf_b, ndig_evk, acc0, acc1, accumulate, norms);
}
static int block_impl(hb_poly* const* digits, int maxdig, int nitems, const int32_t* S, int nS, hb_poly* const* c0, hb_poly* const* c1,
                      uint64_t ptxt_space, int n0, const uint64_t* k0, hb_poly* const* evk0_a, hb_poly* const* evk0_b,
                      int n1, const uint64_t* k1, hb_poly* const* evk1_a, hb_poly* const* evk1_b,
                      hb_poly* const* consts, hb_poly* const* consts1, uint64_t kfinal, hb_poly* const* evkf_a, hb_poly* const* evkf_b,
                      int ndig_evk, hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms) {
  static const char* who = "hb_block_linear_map";
  hb_ctx* c = nullptr;
  const bool bad = consts1 != nullptr;
  if (n0 <= 0 || n1 <= 0 || nitems <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: n0, n1 and nitems must be positive", who);
  if (!k0 || !k1 || !consts) return hb_fail(HB_ERR_BAD_ARG, "%s: no amounts", who);
  HB_TRY(check_polys(c0, nitems, &c, "hb_block_linear_map(c0)"));
  HB_TRY(check_polys(c1, nitems, &c, "hb_block_linear_map(c1)"));
  HB_TRY(check_idx(c, S, nS, who));
  if (ptxt_space < 1) return hb_fail(HB_ERR_BAD_ARG, "%s: ptxt_space must be at least 1", who);
  if (c->special.empty()) return hb_fail(HB_ERR_BAD_ARG, "%s: context has no special primes", who);
  KsSets K; HB_TRY(ks_sets(c, S, nS, who, K));
  HB_TRY(check_amounts(c, k0, n0)); HB_TRY(check_amounts(c, k1, n1));
  if (bad) HB_TRY(check_amounts(c, &kfinal, 1));
  for (int i = 0; i < n0 * n1; i++) if (consts[i]) HB_TRY(check_polys(consts + i, 1, &c, "hb_block_linear_map(consts)"));
  for (int i = 0; bad && i < n0 * n1; i++) if (consts1[i]) HB_TRY(check_polys(consts1 + i, 1, &c, "hb_block_linear_map(consts1)"));
  HB_TRY(check_polys(acc0, nitems, &c, "hb_block_linear_map(acc0)")); HB_TRY(check_polys(acc1, nitems, &c, "hb_block_linear_map(acc1)"));
  const int nd = K.nd;
  if (nd > maxdig) return hb_fail(HB_ERR_BAD_ARG, "%s: S has %d digits, maxdig is %d", who, nd, maxdig);
  HB_TRY(check_polys(digits, nitems * maxdig, &c, "hb_block_linear_map(digits)"));
  const KsKeys sets[3] = {{n0, k0, evk0_a, evk0_b, "evk0"}, {n1, k1, evk1_a, evk1_b, "evk1"}, {bad ? 1 : 0, &kfinal, evkf_a, evkf_b, "evkf"}};
  bool seeded; HB_TRY(ks_check_keys(c, sets, 3, nd, ndig_evk, K.Sp, who, &seeded));
  std::set<const hb_poly*> in(c0, c0 + nitems);
  in.insert(c1, c1 + nitems); in.insert(digits, digits + (size_t)nitems * maxdig);
  for (int i = 0; i < n0 * n1; i++) { if (consts[i]) in.insert(consts[i]); if (bad && consts1[i]) in.insert(consts1[i]); }
  HB_TRY(check_acc(in, sets, 3, nd, ndig_evk, acc0, acc1, nitems, who));
  // ---- every argument is checked: nothing was launched before this point
  const std::vector<int32_t>& Sp = K.Sp;
  const int nSp = (int)Sp.size();
  const std::vector<u64>& scp = K.scp;
  const std::vector<u64> scx(Sp.size(), 1);   // the rotated sums are over S | special: extended form
  const int nout = bad ? 2 * n1 : n1;
  const int T = nout + (bad ? 1 : 0);                  // norm entries per item
  std::vector<u64> kinv((size_t)nout);
  std::vector<uint64_t> kout((size_t)nout);
  for (int o = 0; o < nout; o++) { kout[(size_t)o] = k1[o % n1]; h_invmod(kout[(size_t)o], c->m, &kinv[(size_t)o]); }
  // scratch: H*ic rotations (both parts), G rotated sums with their digits, and the set-1 sum of every item of a chunk
  const int G = std::min(HB_BLOCK_GROUP, nitems * nout);
  const int ic = std::min(std::min(nitems, G), HB_BSGS_GROUP);   // items per chunk (k_ks_giant takes at most HB_BSGS_GROUP)
  const int gg = std::max(1, G / ic);                              // outputs per group
  const int H = std::min(n0, HB_HOIST_SLOTS / ic);                 // inner amounts per chunk
  const int nslot = H * ic;
  const size_t need = (size_t)2 * nslot + (size_t)G * (2 + nd) + (bad ? 2 * ic : 0);
  while (c->block.size() < need) { hb_poly* p; HB_TRY(hb_poly_create(c, &p)); c->block.push_back(p); }
  hb_poly* const* ROT0 = c->block.data();
  hb_poly* const* ROT1 = ROT0 + nslot;
  hb_poly* const* X0 = ROT1 + nslot;
  hb_poly* const* X1 = X0 + G;
  hb_poly* const* DG = X1 + G;
  hb_poly* const* Y0 = DG + (size_t)G * nd;             // the set-1 sums
  hb_poly* const* Y1 = Y0 + ic;
  const int tmax = bsgs_tmax(nd, seeded);
  const int achunk = seeded ? std::max(1, HB_LINMAP_SEEDED / nd) : HB_HOIST_MAXAMT;   // inner amounts per k_ks_hoist launch
  std::vector<hb_poly*> list, ka;
  std::vector<int> slot;
  // the rotations of inner amounts h0 .. h0+hc of items i0 .. i0+nit: amount b of item it into slot b*nit + it
  auto hoist = [&](int i0, int nit, int h0, int hc) -> int {
    for (int a0 = 0; a0 < hc; a0 += achunk) {
      const int na = std::min(achunk, hc - a0);
      list.clear(); slot.assign((size_t)na, -1);
      for (int a = 0; a < na; a++) {
        const int t = h0 + a0 + a;
        if (k0[t] != 1) { slot[(size_t)a] = (int)list.size(); list.insert(list.end(), evk0_a + (size_t)t * ndig_evk, evk0_a + (size_t)t * ndig_evk + nd); }
      }
      if (!list.empty()) HB_TRY(ks_expand_a(c, list.data(), (int)list.size(), Sp.data(), nSp, ka));
      u64 item_rows = 0, key_rows = 0;   // rows read and written per item, and read once, per row of the launch
      for (int a = 0; a < na; a++) { item_rows += k0[h0 + a0 + a] == 1 ? 4 : nd + 3; key_rows += k0[h0 + a0 + a] == 1 ? 0 : 2 * nd; }
      for (int r0 = 0; r0 < nSp; r0 += HB_MAXROWS) {
        const int nr = std::min(HB_MAXROWS, nSp - r0);
        HbHoistJob J; memset(&J, 0, sizeof(J));
        J.N = c->N; J.m = c->m;
        if (c->gen.on) { J.rep = c->gen.d_rep; J.irep = c->gen.d_irep; }
        J.ndig = nd; J.nitems = nit; J.namt = na;
        fill_rows(J.rows, Sp.data() + r0, nr);
        for (int i = 0; i < nr; i++) J.scal[i] = scp[(size_t)(r0 + i)];
        for (int a = 0; a < na; a++) {
          const int t = h0 + a0 + a;
          J.k[a] = k0[t];
          if (slot[(size_t)a] >= 0)
            for (int i = 0; i < nd; i++) { J.evk_a[a][i] = ka[(size_t)slot[(size_t)a] + i]->d; J.evk_b[a][i] = evk0_b[(size_t)t * ndig_evk + i]->d; }
          for (int it = 0; it < nit; it++) { J.out0[a * nit + it] = ROT0[(a0 + a) * nit + it]->d; J.out1[a * nit + it] = ROT1[(a0 + a) * nit + it]->d; }
        }
        for (int it = 0; it < nit; it++) {
          J.c0[it] = c0[i0 + it]->d; J.c1[it] = c1[i0 + it]->d;
          for (int i = 0; i < nd; i++) J.dig[it][i] = digits[(size_t)(i0 + it) * maxdig + i]->d;
        }
        const int ni = nit >= 4 ? 4 : nit >= 2 ? 2 : 1;
        const dim3 g((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS), (unsigned)nr, (unsigned)((nit + ni - 1) / ni));
        pre_launch(c);
        switch (ni) {
          case 1: HB_LAUNCH(k_ks_hoist<1>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
          case 2: HB_LAUNCH(k_ks_hoist<2>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
          default: HB_LAUNCH(k_ks_hoist<4>, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J); break;
        }
        HB_TRY(post_launch(c, "k_ks_hoist", (item_rows * nit + key_rows) * nr * c->N * 8));
      }
    }
    return HB_OK;
  };
  const bool once = n0 <= H;
  for (int i0 = 0; i0 < nitems; i0 += ic) {
    const int nit = std::min(ic, nitems - i0);
    bool acc_on = accumulate != 0, y_on = false;
    if (once) HB_TRY(hoist(i0, nit, 0, n0));
    for (int o0 = 0; o0 < nout; o0 += gg) {
      const int ng = std::min(gg, nout - o0);
      // 1. the group's rotated sums sigma_k1( sum_i consts[i*n1 + j] * r_i ): slot a*nit + it
      for (int h0 = 0; h0 < n0; h0 += H) {
        const int hc = std::min(H, n0 - h0);
        if (!once) HB_TRY(hoist(i0, nit, h0, hc));
        HB_TRY(bsgs_mac(c, Sp, X0, X1, ic, nit, ng, hc, kinv.data() + o0, nullptr, h0 > 0,
                        [&](int a, int b) { const int o = o0 + a; return (o < n1 ? consts : consts1)[(size_t)(h0 + b) * n1 + o % n1]; },
                        [&](int u, int b) { return std::make_pair(ROT0[b * nit + u], ROT1[b * nit + u]); }));
      }
      // 2-3. set 0 into the accumulators, set 1 into its sum
      const int split = std::max(0, std::min(ng, n1 - o0));
      double* nb = norms ? norms + ((size_t)i0 * T + o0) * (HB_MAXDIG + 2) : nullptr;
      if (split > 0)
        HB_TRY(bsgs_finish(c, X0, X1, DG, nit, split, kout.data() + o0, evk1_a + (size_t)o0 * ndig_evk, evk1_b + (size_t)o0 * ndig_evk, ndig_evk,
                           nd, S, nS, Sp, 1, ptxt_space, scp, scx, tmax, seeded, acc0 + i0, acc1 + i0, acc_on, nb, (size_t)T));
      if (ng > split) {
        const int j0 = o0 + split - n1;
        HB_TRY(bsgs_finish(c, X0 + (size_t)split * nit, X1 + (size_t)split * nit, DG + (size_t)split * nit * nd, nit, ng - split, k1 + j0,
                           evk1_a + (size_t)j0 * ndig_evk, evk1_b + (size_t)j0 * ndig_evk, ndig_evk, nd, S, nS, Sp, 1, ptxt_space, scp, scx,
                           tmax, seeded, Y0, Y1, y_on, nb ? nb + (size_t)split * (HB_MAXDIG + 2) : nullptr, (size_t)T));
      }
    }
    if (!bad) continue;
    // the bad dimension's last term: the set-1 sum rotated by kfinal (smartAutomorph), added to the accumulators
    double* nf = norms ? norms + ((size_t)i0 * T + nout) * (HB_MAXDIG + 2) : nullptr;
    if (kfinal == 1) {
      HB_TRY(bsgs_finish(c, Y0, Y1, DG, nit, 1, &kfinal, evkf_a, evkf_b, ndig_evk, nd, S, nS, Sp, 1, ptxt_space, scp, scx, tmax, seeded,
                         acc0 + i0, acc1 + i0, acc_on, nf, (size_t)T));
      continue;
    }
    // sigma_kfinal as a gather copy into the group slots: one read and one write of the set-1 sums, once per item chunk.
    // Folding it into a k_bsgs_mac pass would need a constant row of ones to multiply by, which reads as much; the
    // checks of hb_automorph cannot fail here (its operands are this call's scratch, kfinal was checked above).
    HB_TRY(hb_automorph(X0, Y0, nit, Sp.data(), nSp, kfinal));
    HB_TRY(hb_automorph(X1, Y1, nit, Sp.data(), nSp, kfinal));
    HB_TRY(bsgs_finish(c, X0, X1, DG, nit, 1, &kfinal, evkf_a, evkf_b, ndig_evk, nd, S, nS, Sp, 1, ptxt_space, scp, scx, tmax, seeded,
                       acc0 + i0, acc1 + i0, acc_on, nf, (size_t)T));
  }
  return HB_OK;
}

// k_ks_leafmap with li leaves per thread (1, 2 or 4)
template <int LI, bool BAD>
static void leaf_launch1(hb_ctx* c, const dim3& g, const HbLeafJob& J) {
  constexpr auto kern = k_ks_leafmap<LI, BAD>;   // one token for HB_LAUNCH
  HB_LAUNCH(kern, g, dim3(HB_THREADS), 0, c->stream, c->d_primes, J);
}
template <bool BAD>
static void leaf_launch(hb_ctx* c, int li, const dim3& g, const HbLeafJob& J) {
  switch (li) {
    case 1: leaf_launch1<1, BAD>(c, g, J); break;
    case 2: leaf_launch1<2, BAD>(c, g, J); break;
    default: leaf_launch1<4, BAD>(c, g, J); break;
  }
}
// Full linear map leaves (SURVEY 8f-1): the last dimension of MatMulFullExec::rec_mul (src/matmul.cpp:2141-2148), every leaf
// a hoisted MatMul1DExec::mul.  Per chunk of (item, leaf) pairs (slot l*nit + it): the cleanUp of the rotated leaves (a copy
// into scratch and one batched mod-down), the digits of every leaf (one batched breakIntoDigits), then one k_ks_leafmap
// pass per group of amounts and row chunk, all leaves of an item summed into its accumulators; in a bad dimension the
// per-leaf sums are rotated by kfinal, modded down, decomposed and key-switched into the accumulators by bsgs_finish.
static int full_leaves_impl(hb_poly* const* x0, hb_poly* const* x1, int nleaves, int nitems, const int32_t* ext,
                            const int32_t* S, int nS, uint64_t ptxt_space, int namt, const uint64_t* k,
                            hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* consts, hb_poly* const* consts1,
                            uint64_t kfinal, hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                            hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms) {
  static const char* who = "hb_full_linear_map_leaves";
  hb_ctx* c = nullptr;
  const bool bad = consts1 != nullptr;
  if (nleaves <= 0 || nitems <= 0 || namt <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: nleaves, nitems and namt must be positive", who);
  if (!k || !consts) return hb_fail(HB_ERR_BAD_ARG, "%s: no amounts", who);
  HB_TRY(check_polys(x0, nitems * nleaves, &c, "hb_full_linear_map_leaves(x0)"));
  HB_TRY(check_polys(x1, nitems * nleaves, &c, "hb_full_linear_map_leaves(x1)"));
  for (int l = 0; ext && l < nleaves; l++) if (ext[l] != 0 && ext[l] != 1) return hb_fail(HB_ERR_BAD_ARG, "%s: ext[%d] must be 0 or 1", who, l);
  HB_TRY(check_idx(c, S, nS, who));
  if (ptxt_space < 1) return hb_fail(HB_ERR_BAD_ARG, "%s: ptxt_space must be at least 1", who);
  if (c->special.empty()) return hb_fail(HB_ERR_BAD_ARG, "%s: context has no special primes", who);
  KsSets K; HB_TRY(ks_sets(c, S, nS, who, K));
  const int nd = K.nd;
  if (nd > HB_MAXDIG) return hb_fail(HB_ERR_BAD_ARG, "%s: S has %d digits, at most %d are supported", who, nd, HB_MAXDIG);
  HB_TRY(check_amounts(c, k, namt));
  if (bad) HB_TRY(check_amounts(c, &kfinal, 1));
  for (int i = 0; i < nleaves * namt; i++) if (consts[i]) HB_TRY(check_polys(consts + i, 1, &c, "hb_full_linear_map_leaves(consts)"));
  for (int i = 0; bad && i < nleaves * namt; i++) if (consts1[i]) HB_TRY(check_polys(consts1 + i, 1, &c, "hb_full_linear_map_leaves(consts1)"));
  HB_TRY(check_polys(acc0, nitems, &c, "hb_full_linear_map_leaves(acc0)")); HB_TRY(check_polys(acc1, nitems, &c, "hb_full_linear_map_leaves(acc1)"));
  const KsKeys sets[2] = {{namt, k, evk_a, evk_b, "evk"}, {bad ? 1 : 0, &kfinal, evkf_a, evkf_b, "evkf"}};
  bool seeded, seeded_f;
  HB_TRY(ks_check_keys(c, sets, 1, nd, ndig_evk, K.Sp, who, &seeded));
  HB_TRY(ks_check_keys(c, sets + 1, 1, nd, ndig_evk, K.Sp, who, &seeded_f));
  std::set<const hb_poly*> in(x0, x0 + (size_t)nitems * nleaves);
  in.insert(x1, x1 + (size_t)nitems * nleaves);
  for (int i = 0; i < nleaves * namt; i++) { if (consts[i]) in.insert(consts[i]); if (bad && consts1[i]) in.insert(consts1[i]); }
  HB_TRY(check_acc(in, sets, 2, nd, ndig_evk, acc0, acc1, nitems, who));
  // ---- every argument is checked: nothing was launched before this point
  const std::vector<int32_t>& Sp = K.Sp;
  const int nSp = (int)Sp.size();
  const std::vector<u64>& scp = K.scp;
  const std::vector<u64> scx(Sp.size(), 1);   // the per-leaf sums are over S | special: extended form
  const int T = bad ? 2 * nleaves : nleaves;   // norm entries per item
  // chunks: at least 4 leaves (a thread's k_ks_leafmap<4> group) where the call has them, at most HB_LEAF_PAIRS pairs
  const int lc = std::min(nleaves, std::max(4, HB_LEAF_PAIRS / std::min(nitems, HB_LEAF_PAIRS)));
  const int ic = std::max(1, std::min(nitems, HB_LEAF_PAIRS / lc));
  const int G = ic * lc;
  const size_t need = (size_t)G * (2 + nd) + (bad ? 2 * (size_t)G : 0) + (bad && seeded_f ? nd : 0);
  while (c->leaf.size() < need) { hb_poly* p; HB_TRY(hb_poly_create(c, &p)); c->leaf.push_back(p); }
  hb_poly* const* XC0 = c->leaf.data();               // cleaned leaves; in a bad dimension then sigma_kfinal of the sums
  hb_poly* const* XC1 = XC0 + G;
  hb_poly* const* DG = XC1 + G;                        // digits, slot s at DG[s*nd ..]
  hb_poly* const* Y0 = DG + (size_t)G * nd;            // the per-leaf sums of the bad dimension
  hb_poly* const* Y1 = Y0 + G;
  hb_poly* const* KF = Y1 + G;                         // kfinal's a_i, regenerated once per call when seeded
  std::vector<hb_poly*> fa, fb;                        // kfinal's matrix once per leaf of a chunk (bsgs_finish's layout)
  if (bad && kfinal != 1) {
    std::vector<hb_poly*> ea(evkf_a, evkf_a + nd);
    if (seeded_f) {
      std::vector<hb_poly*> src; std::vector<u64*> dst;
      for (int i = 0; i < nd; i++) if (evkf_a[i]->sched) { ea[(size_t)i] = KF[i]; src.push_back(evkf_a[i]); dst.push_back(KF[i]->d); }
      HB_TRY(prg_expand(c, src.data(), dst.data(), (int)src.size(), Sp.data(), nSp, "key switch (evkf_a)"));
    }
    for (int l = 0; l < lc; l++) { fa.insert(fa.end(), ea.begin(), ea.end()); fb.insert(fb.end(), evkf_b, evkf_b + nd); }
  }
  const std::vector<uint64_t> kfv((size_t)lc, kfinal);
  const int tmax = bsgs_tmax(nd, false);
  const int achunk = seeded ? std::max(1, std::min(HB_LEAF_MAXAMT, HB_LINMAP_SEEDED / nd)) : HB_LEAF_MAXAMT;
  std::vector<hb_poly*> L0((size_t)G), L1((size_t)G), cp0, cp1, sd, part1, dg((size_t)G * nd), list, ka, ysrc0, ysrc1, ydst0, ydst1;
  std::vector<int> slot, sds;
  for (int i0 = 0; i0 < nitems; i0 += ic) {
    const int nit = std::min(ic, nitems - i0);
    bool acc_on = accumulate != 0;
    for (int l0 = 0; l0 < nleaves; l0 += lc) {
      const int nl = std::min(lc, nleaves - l0), np = nl * nit;
      // 1. cleanUp of the rotated leaves into scratch, and the digits of every leaf's part 1 over S
      cp0.clear(); cp1.clear(); sd.clear(); sds.clear(); part1.clear();
      for (int l = 0; l < nl; l++)
        for (int it = 0; it < nit; it++) {
          const int s = l * nit + it;
          const size_t e = (size_t)(i0 + it) * nleaves + l0 + l;
          if (ext && ext[l0 + l]) {
            L0[(size_t)s] = XC0[s]; L1[(size_t)s] = XC1[s];
            cp0.push_back(x0[e]); cp0.push_back(x1[e]); cp1.push_back(XC0[s]); cp1.push_back(XC1[s]); sds.push_back(s);
          } else {
            L0[(size_t)s] = x0[e]; L1[(size_t)s] = x1[e];
          }
          part1.push_back(L1[(size_t)s]);
          for (int i = 0; i < nd; i++) dg[(size_t)s * nd + i] = DG[(size_t)s * nd + i];
        }
      std::vector<double> sdn(norms ? cp1.size() : 0), ldn(norms ? (size_t)np * nd : 0);
      if (!cp1.empty()) {
        HB_TRY(pw_simple(HB_PW_COPY, cp1.data(), cp0.data(), (int)cp1.size(), Sp.data(), nSp, nullptr, c));
        HB_TRY(scale_down_impl(cp1.data(), (int)cp1.size(), Sp.data(), nSp, S, nS, ptxt_space, norms ? sdn.data() : nullptr));
      }
      int ndo = 0;
      HB_TRY(break_into_digits_impl(part1.data(), np, S, nS, dg.data(), nd, &ndo, norms ? ldn.data() : nullptr));
      if (norms) {
        for (int s = 0; s < np; s++) {
          double* o = norms + ((size_t)(i0 + s % nit) * T + l0 + s / nit) * (HB_MAXDIG + 2);
          for (int i = 0; i < nd; i++) o[i] = ldn[(size_t)s * nd + i];
        }
        for (size_t r = 0; r < sds.size(); r++) {
          const int s = sds[r];
          double* o = norms + ((size_t)(i0 + s % nit) * T + l0 + s / nit) * (HB_MAXDIG + 2);
          o[HB_MAXDIG] = sdn[2 * r]; o[HB_MAXDIG + 1] = sdn[2 * r + 1];
        }
      }
      // 2. every leaf's rotations, weighted by its constants, into the accumulators (and the per-leaf sums)
      for (int a0 = 0; a0 < namt; a0 += achunk) {
        const int na = std::min(achunk, namt - a0);
        list.clear(); slot.assign((size_t)na, -1);
        for (int a = 0; a < na; a++)
          if (k[a0 + a] != 1) { slot[(size_t)a] = (int)list.size(); list.insert(list.end(), evk_a + (size_t)(a0 + a) * ndig_evk, evk_a + (size_t)(a0 + a) * ndig_evk + nd); }
        if (!list.empty()) HB_TRY(ks_expand_a(c, list.data(), (int)list.size(), Sp.data(), nSp, ka));
        u64 item_rows = 0, shared_rows = 0;   // rows read (and written) per item and shared by the items, per row of the launch
        for (int a = 0; a < na; a++) {
          item_rows += (u64)nl * (k[a0 + a] == 1 ? 2 : nd + 1);
          shared_rows += k[a0 + a] == 1 ? 0 : 2 * nd;
          for (int l = 0; l < nl; l++) {
            const size_t e = (size_t)(l0 + l) * namt + a0 + a;
            shared_rows += (consts[e] != nullptr) + (bad && consts1[e] != nullptr);
          }
        }
        item_rows += (acc_on ? 4 : 2) + (bad ? (u64)nl * (a0 > 0 ? 4 : 2) : 0);
        for (int r0 = 0; r0 < nSp; r0 += HB_MAXROWS) {
          const int nr = std::min(HB_MAXROWS, nSp - r0);
          HbLeafJob J; memset(&J, 0, sizeof(J));
          J.N = c->N; J.m = c->m;
          if (c->gen.on) { J.rep = c->gen.d_rep; J.irep = c->gen.d_irep; }
          J.ndig = nd; J.nitems = nit; J.nleaves = nl; J.namt = na; J.accumulate = acc_on ? 1 : 0; J.accumulate1 = a0 > 0 ? 1 : 0;
          fill_rows(J.rows, Sp.data() + r0, nr);
          for (int i = 0; i < nr; i++) J.scal[i] = scp[(size_t)(r0 + i)];
          for (int a = 0; a < na; a++) {
            const int t = a0 + a;
            J.k[a] = k[t];
            if (slot[(size_t)a] >= 0)
              for (int i = 0; i < nd; i++) { J.evk_a[a][i] = ka[(size_t)slot[(size_t)a] + i]->d; J.evk_b[a][i] = evk_b[(size_t)t * ndig_evk + i]->d; }
            for (int l = 0; l < nl; l++) {
              const size_t e = (size_t)(l0 + l) * namt + t;
              J.cst[l * na + a] = consts[e] ? consts[e]->d : nullptr;
              if (bad) J.cst1[l * na + a] = consts1[e] ? consts1[e]->d : nullptr;
            }
          }
          for (int s = 0; s < np; s++) {
            J.c0[s] = L0[(size_t)s]->d; J.c1[s] = L1[(size_t)s]->d;
            for (int i = 0; i < nd; i++) J.dig[s][i] = DG[(size_t)s * nd + i]->d;
            if (bad) { J.y0[s] = Y0[s]->d; J.y1[s] = Y1[s]->d; }
          }
          for (int it = 0; it < nit; it++) { J.acc0[it] = acc0[i0 + it]->d; J.acc1[it] = acc1[i0 + it]->d; }
          const int li = nl >= 4 ? 4 : nl >= 2 ? 2 : 1;
          const dim3 g((unsigned)((c->N + HB_THREADS - 1) / HB_THREADS), (unsigned)nr, (unsigned)nit);
          pre_launch(c);
          if (bad) leaf_launch<true>(c, li, g, J); else leaf_launch<false>(c, li, g, J);
          HB_TRY(post_launch(c, "k_ks_leafmap", (item_rows * nit + shared_rows) * nr * c->N * 8));
        }
        acc_on = true;
      }
      if (!bad) continue;
      // 3. every leaf's sum rotated by kfinal (smartAutomorph), added to its item's accumulators
      double* nf = norms ? norms + ((size_t)i0 * T + nleaves + l0) * (HB_MAXDIG + 2) : nullptr;
      if (kfinal == 1) {
        HB_TRY(bsgs_finish(c, Y0, Y1, DG, nit, nl, kfv.data(), evkf_a, evkf_b, 0, nd, S, nS, Sp, 1, ptxt_space, scp, scx, tmax, false,
                           acc0 + i0, acc1 + i0, acc_on, nf, (size_t)T));
        continue;
      }
      ysrc0.assign(Y0, Y0 + np); ysrc1.assign(Y1, Y1 + np); ydst0.assign(XC0, XC0 + np); ydst1.assign(XC1, XC1 + np);
      HB_TRY(hb_automorph(ydst0.data(), ysrc0.data(), np, Sp.data(), nSp, kfinal));
      HB_TRY(hb_automorph(ydst1.data(), ysrc1.data(), np, Sp.data(), nSp, kfinal));
      HB_TRY(bsgs_finish(c, XC0, XC1, DG, nit, nl, kfv.data(), fa.data(), fb.data(), nd, nd, S, nS, Sp, 1, ptxt_space, scp, scx, tmax, false,
                         acc0 + i0, acc1 + i0, acc_on, nf, (size_t)T));
    }
  }
  return HB_OK;
}
extern "C" int hb_full_linear_map_leaves(hb_poly* const* x0, hb_poly* const* x1, int nleaves, int nitems, const int32_t* ext,
                                         const int32_t* S, int nS, uint64_t ptxt_space, int namt, const uint64_t* k,
                                         hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* consts, hb_poly* const* consts1,
                                         uint64_t kfinal, hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                                         hb_poly* const* acc0, hb_poly* const* acc1, int accumulate) {
  return full_leaves_impl(x0, x1, nleaves, nitems, ext, S, nS, ptxt_space, namt, k, evk_a, evk_b, consts, consts1, kfinal, evkf_a, evkf_b,
                          ndig_evk, acc0, acc1, accumulate, nullptr);
}
extern "C" int hb_full_linear_map_leaves_norm(hb_poly* const* x0, hb_poly* const* x1, int nleaves, int nitems, const int32_t* ext,
                                              const int32_t* S, int nS, uint64_t ptxt_space, int namt, const uint64_t* k,
                                              hb_poly* const* evk_a, hb_poly* const* evk_b, hb_poly* const* consts, hb_poly* const* consts1,
                                              uint64_t kfinal, hb_poly* const* evkf_a, hb_poly* const* evkf_b, int ndig_evk,
                                              hb_poly* const* acc0, hb_poly* const* acc1, int accumulate, double* norms) {
  if (!norms) return hb_fail(HB_ERR_BAD_ARG, "hb_full_linear_map_leaves_norm: null output");
  return full_leaves_impl(x0, x1, nleaves, nitems, ext, S, nS, ptxt_space, namt, k, evk_a, evk_b, consts, consts1, kfinal, evkf_a, evkf_b,
                          ndig_evk, acc0, acc1, accumulate, norms);
}

extern "C" int hb_tensor(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1,
                         hb_poly* const* o0, hb_poly* const* o1, hb_poly* const* o2, int nitems, const int32_t* idx, int n) {
  hb_ctx* c = nullptr;
  HB_TRY(check_polys(a0, nitems, &c, "hb_tensor")); HB_TRY(check_polys(a1, nitems, &c, "hb_tensor"));
  HB_TRY(check_polys(b0, nitems, &c, "hb_tensor")); HB_TRY(check_polys(b1, nitems, &c, "hb_tensor"));
  HB_TRY(check_polys(o0, nitems, &c, "hb_tensor")); HB_TRY(check_polys(o1, nitems, &c, "hb_tensor")); HB_TRY(check_polys(o2, nitems, &c, "hb_tensor"));
  HB_TRY(check_idx(c, idx, n, "hb_tensor"));
  return for_items(nitems, [&](int i0, int nit) {
    u64 *A0[HB_MAXB], *A1[HB_MAXB], *B0[HB_MAXB], *B1[HB_MAXB], *O0[HB_MAXB], *O1[HB_MAXB], *O2[HB_MAXB];
    ptrs_of(a0, i0, nit, A0); ptrs_of(a1, i0, nit, A1); ptrs_of(b0, i0, nit, B0); ptrs_of(b1, i0, nit, B1);
    ptrs_of(o0, i0, nit, O0); ptrs_of(o1, i0, nit, O1); ptrs_of(o2, i0, nit, O2);
    if (!c->gen.on && c->N % 512 == 0 && !c->force_v0) {   // streaming kernel: 128-bit accesses
      for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
        const int nr = std::min(HB_MAXROWS, n - r0);
        Hb1TensorJob J; memset(&J, 0, sizeof(J));
        J.N = c->N; J.nitems = nit;
        fill_rows(J.rows, idx + r0, nr);
        for (int i = 0; i < nit; i++) { J.a0[i] = A0[i]; J.a1[i] = A1[i]; J.b0[i] = B0[i]; J.b1[i] = B1[i]; J.o0[i] = O0[i]; J.o1[i] = O1[i]; J.o2[i] = O2[i]; }
        pre_launch(c);
        HB_LAUNCH(k1_tensor, dim3((unsigned)(c->N / 512), nr, nit), dim3(256), 0, c->stream, c->d_primes, J);
        HB_TRY(post_launch(c, "k1_tensor", (u64)7 * nr * nit * c->N * 8));
      }
      return HB_OK;
    }
    PwArgs A; memset(&A, 0, sizeof(A));
    A.op = HB_PW_TENSOR; A.dst = O0; A.dst1 = O1; A.dst2 = O2;
    A.a = (const u64* const*)A0; A.b = (const u64* const*)A1; A.cc = (const u64* const*)B0; A.d = (const u64* const*)B1;
    return launch_pw(c, A, nit, idx, n);
  });
}

// The summed tensor products of hb_tensor_sum on checked arguments.  Pair j of item t is [t*npairs + j].  Power-of-two m with
// N a multiple of 512 runs k1_tensor_sum, as many items per launch as fit HB_TSUM_SLOTS pair slots and, for more pairs than
// that, later pair groups accumulating into the outputs.  Otherwise (general m, small N, HB_FORCE_V0) every pair is an
// HB_PW_TENSOR pass into scratch (the first one straight into the outputs unless accumulating) and three ADDs, as hb_tensor's
// generic path; that path needs canonical inputs.
static int tensor_sum_impl(hb_ctx* c, hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1, int npairs,
                           int nitems, const int32_t* idx, int n, hb_poly* const* o0, hb_poly* const* o1, hb_poly* const* o2, int accumulate) {
  if (!c->gen.on && c->N % 512 == 0 && !c->force_v0) {
    const int ni = std::max(1, std::min(g_chunk, HB_TSUM_SLOTS / npairs));   // items per launch
    const int pp = std::min(npairs, HB_TSUM_SLOTS / ni);                       // pairs per launch
    for (int i0 = 0; i0 < nitems; i0 += ni) {
      const int nit = std::min(ni, nitems - i0);
      for (int j0 = 0; j0 < npairs; j0 += pp) {
        const int np = std::min(pp, npairs - j0);
        for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
          const int nr = std::min(HB_MAXROWS, n - r0);
          Hb1TensorSumJob J; memset(&J, 0, sizeof(J));
          J.N = c->N; J.npairs = np; J.nitems = nit; J.accumulate = accumulate || j0 > 0;
          fill_rows(J.rows, idx + r0, nr);
          for (int t = 0; t < nit; t++) {
            for (int j = 0; j < np; j++) {
              const size_t e = (size_t)(i0 + t) * npairs + j0 + j;
              const int s = t * np + j;
              J.a0[s] = a0[e]->d; J.a1[s] = a1[e]->d; J.b0[s] = b0[e]->d; J.b1[s] = b1[e]->d;
            }
            J.o0[t] = o0[i0 + t]->d; J.o1[t] = o1[i0 + t]->d; J.o2[t] = o2[i0 + t]->d;
          }
          pre_launch(c);
          HB_LAUNCH(k1_tensor_sum, dim3((unsigned)(c->N / 512), nr, nit), dim3(256), 0, c->stream, c->d_primes, J);
          HB_TRY(post_launch(c, "k1_tensor_sum", (u64)(4 * np + (J.accumulate ? 6 : 3)) * nr * nit * c->N * 8));
        }
      }
    }
    return HB_OK;
  }
  HB_TRY(ctx_scratch(c));
  const int per = std::max(1, std::min(g_chunk, HB_MAXB / 3));   // items per chunk: three scratch slots each
  for (int i0 = 0; i0 < nitems; i0 += per) {
    const int nit = std::min(per, nitems - i0);
    u64* O[3][HB_MAXB]; u64* T[HB_MAXB];
    ptrs_of(o0, i0, nit, O[0]); ptrs_of(o1, i0, nit, O[1]); ptrs_of(o2, i0, nit, O[2]);
    tmp_ptrs(c, c->tmpA, 3 * nit, T);
    for (int j = 0; j < npairs; j++) {
      u64 *A0[HB_MAXB], *A1[HB_MAXB], *B0[HB_MAXB], *B1[HB_MAXB];
      for (int t = 0; t < nit; t++) {
        const size_t e = (size_t)(i0 + t) * npairs + j;
        A0[t] = a0[e]->d; A1[t] = a1[e]->d; B0[t] = b0[e]->d; B1[t] = b1[e]->d;
      }
      const bool direct = j == 0 && !accumulate;
      PwArgs A; memset(&A, 0, sizeof(A));
      A.op = HB_PW_TENSOR; A.dst = direct ? O[0] : T; A.dst1 = direct ? O[1] : T + nit; A.dst2 = direct ? O[2] : T + 2 * nit;
      A.a = (const u64* const*)A0; A.b = (const u64* const*)A1; A.cc = (const u64* const*)B0; A.d = (const u64* const*)B1;
      HB_TRY(launch_pw(c, A, nit, idx, n));
      if (direct) continue;
      for (int k = 0; k < 3; k++) {
        PwArgs B; memset(&B, 0, sizeof(B));
        B.op = HB_PW_ADD; B.dst = O[k]; B.a = (const u64* const*)(T + k * nit);
        HB_TRY(launch_pw(c, B, nit, idx, n));
      }
    }
  }
  return HB_OK;
}
// outputs written while the inputs `in` are read: distinct, and aliasing none of them
static int check_outputs(const std::set<const hb_poly*>& in, std::initializer_list<hb_poly* const*> outs, int nitems, const char* who) {
  std::set<const hb_poly*> out;
  for (hb_poly* const* o : outs) out.insert(o, o + nitems);
  if (out.size() != outs.size() * (size_t)nitems) return hb_fail(HB_ERR_BAD_ARG, "%s: the outputs must be distinct polynomials", who);
  for (const hb_poly* p : out) if (in.count(p)) return hb_fail(HB_ERR_BAD_ARG, "%s: an output aliases an input", who);
  return HB_OK;
}
extern "C" int hb_tensor_sum(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1, int npairs, int nitems,
                             const int32_t* idx, int n, hb_poly* const* o0, hb_poly* const* o1, hb_poly* const* o2, int accumulate) {
  static const char* who = "hb_tensor_sum";
  if (npairs <= 0 || nitems <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: npairs and nitems must be positive", who);
  if (accumulate != 0 && accumulate != 1) return hb_fail(HB_ERR_BAD_ARG, "%s: accumulate must be 0 or 1", who);
  hb_ctx* c = nullptr;
  const int np = npairs * nitems;
  HB_TRY(check_polys(a0, np, &c, who)); HB_TRY(check_polys(a1, np, &c, who)); HB_TRY(check_polys(b0, np, &c, who)); HB_TRY(check_polys(b1, np, &c, who));
  HB_TRY(check_polys(o0, nitems, &c, who)); HB_TRY(check_polys(o1, nitems, &c, who)); HB_TRY(check_polys(o2, nitems, &c, who));
  HB_TRY(check_idx(c, idx, n, who));
  std::set<const hb_poly*> in(a0, a0 + np); in.insert(a1, a1 + np); in.insert(b0, b0 + np); in.insert(b1, b1 + np);
  HB_TRY(check_outputs(in, {o0, o1, o2}, nitems, who));
  return tensor_sum_impl(c, a0, a1, b0, b1, npairs, nitems, idx, n, o0, o1, o2, accumulate);
}

extern "C" int hb_automorph(hb_poly* const* dst, hb_poly* const* src, int nitems, const int32_t* idx, int n, uint64_t k) {
  hb_ctx* c = nullptr; HB_TRY(check_polys(dst, nitems, &c, "hb_automorph")); HB_TRY(check_polys(src, nitems, &c, "hb_automorph"));
  HB_TRY(check_idx(c, idx, n, "hb_automorph"));
  if (k == 0 || k >= c->m || h_gcd((long)k, (long)c->m) != 1) return hb_fail(HB_ERR_INDEX_SET, "DoubleCRT::automorph: k not in Zm*");  // src/DoubleCRT.cpp:1165-1167
  for (int i = 0; i < nitems; i++) if (dst[i] == src[i]) return hb_fail(HB_ERR_BAD_ARG, "hb_automorph: dst must differ from src");
  if (c->gen.on) return for_items(nitems, [&](int i0, int nit) {
    for (int r0 = 0; r0 < n; r0 += HB_MAXROWS) {
      int nr = std::min(HB_MAXROWS, n - r0);
      HbGenAutoJob J; memset(&J, 0, sizeof(J));
      J.m = c->gen.m; J.phim = c->gen.phim; J.k = k; J.rep = c->gen.d_rep; J.irep = c->gen.d_irep; J.nitems = nit;
      fill_rows(J.rows, idx + r0, nr);
      for (int i = 0; i < nit; i++) { J.src[i] = src[i0 + i]->d; J.dst[i] = dst[i0 + i]->d; }
      pre_launch(c);
      HB_LAUNCH(k_gen_automorph, dim3((unsigned)std::max<size_t>(1, c->N / HB_THREADS), nr, nit), dim3(HB_THREADS), 0, c->stream, J);
      HB_TRY(post_launch(c, "k_gen_automorph", (u64)2 * nr * nit * c->N * 8));
    }
    return HB_OK;
  });
  return for_items(nitems, [&](int i0, int nit) {
    u64* D[HB_MAXB]; u64* S[HB_MAXB]; ptrs_of(dst, i0, nit, D); ptrs_of(src, i0, nit, S);
    PwArgs A; memset(&A, 0, sizeof(A));
    A.op = HB_PW_AUTOMORPH; A.dst = D; A.a = (const u64* const*)S; A.k = k; A.m = c->m;
    return launch_pw(c, A, nit, idx, n);
  });
}

// ------------------------------------------------------------------------------------------
// fused ciphertext-level paths

// reLinearize for the register kernels: breakIntoDigits (src/DoubleCRT.cpp:479-561) without the two copy passes and without the
// separate mixed-radix pointwise pass.  The switched part c2 is updated in place (the ABI says it is consumed): digit i's own rows
// ARE c2's rows at the time digit i is reached, the digit polynomials only receive the base-extended rows, and the forward blk phase
// of digit i's extension applies  c2 <- (c2 - E_i) * Q_i^-1  on the rows of the later digits in its epilogue.  Values handed from
// kernel to kernel stay lazy; the inner product (src/Ctxt.cpp:191-230, with the addPrimesAndScale of src/Ctxt.cpp:764-768 folded in)
// reduces exactly.  Everything runs chunk by chunk so that a chunk's scratch is re-read while still in L2.
// The caller has checked the arguments and the key, and sends sets with more than four digits (the largest instantiation of
// the fused inner product) to the step-by-step path.
static int relin_fused_v1(hb_ctx* c, hb_poly* const* c0, hb_poly* const* c1, hb_poly* const* c2, int nitems, const int32_t* S, int nS,
                          const KsSets& K, hb_poly* const* evk_a, hb_poly* const* evk_b, const std::vector<hb_poly*>& dig) {
  const int maxdig = c->ndigits, nd = K.nd;
  const std::vector<int32_t>& Sp = K.Sp;
  std::vector<std::vector<int32_t>> dset, notin, full; ks_digits(c, S, nS, K, dset, notin, full);
  // per digit: epilogue scalars on the rows of notin[i]: Q_i^-1 mod q_r for rows of later digits, 0 elsewhere
  std::vector<std::vector<u64>> esc(nd);
  for (int i = 0; i < nd; i++) {
    esc[i].assign(notin[i].size(), 0);
    for (size_t r = 0; r < notin[i].size(); r++) {
      const int dj = c->digit_of[notin[i][r]];
      if (dj > i && dj < nd) {
        u64 inv; if (!h_invmod(prod_mod(c, full[i].data(), (int)full[i].size(), c->q[notin[i][r]]), c->q[notin[i][r]], &inv)) return hb_fail(HB_ERR_BAD_ARG, "digit product not invertible");
        esc[i][r] = inv;
      }
    }
  }
  std::vector<int> own_dig(Sp.size());   // the digit of each row of S, -1 on the special rows
  for (size_t r = 0; r < Sp.size(); r++) own_dig[r] = c->digit_of[Sp[r]];
  HB_TRY(ctx_scratch(c));
  return for_items(nitems, [&](int i0, int nit) {
    u64* R[HB_MAXB]; u64* tB[HB_MAXB]; u64* D[HB_MAXB];
    ptrs_of(c2, i0, nit, R); tmp_ptrs(c, c->tmpB, nit, tB);
    for (int i = 0; i < nd; i++) {
      for (int it = 0; it < nit; it++) D[it] = dig[(size_t)(i0 + it) * maxdig + i]->d;
      HB_TRY(conv_chunk(c, R, nit, dset[i].data(), (int)dset[i].size(), notin[i].data(), (int)notin[i].size(), 1));
      HB_TRY(launch_blk(c, +1, (const u64* const*)tB, D, nit, notin[i].data(), (int)notin[i].size(), 3, esc[i].data(), 1, R));
    }
    const int saved = g_chunk; g_chunk = HB_MAXB;   // already inside a chunk: one inner-product launch for it
    int rc = keyswitch_digits_impl(dig.data() + (size_t)i0 * maxdig, maxdig, nd, nit, Sp.data(), (int)Sp.size(), evk_a, evk_b, c0 + i0, c1 + i0, K.scp.data(), 0, nullptr, c2 + i0, own_dig.data());
    g_chunk = saved;
    return rc;
  });
}

// The checks of the key and the regeneration of a seeded evk_a for a relinearisation over K: the matrix must have a column
// for every digit of S, and only those columns are read.
static int relin_key(hb_ctx* c, const KsSets& K, hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk, const char* who,
                     std::vector<hb_poly*>& ka) {
  const KsKeys key = {1, nullptr, evk_a, evk_b, "evk"};
  HB_TRY(ks_check_keys(c, &key, 1, K.nd, ndig_evk, K.Sp, who));
  // ---- every argument is checked: nothing was launched before this point
  return ks_expand_a(c, evk_a, K.nd, K.Sp.data(), (int)K.Sp.size(), ka);
}
extern "C" int hb_relinearize(hb_poly* const* c0, hb_poly* const* c1, hb_poly* const* c2, int nitems,
                              const int32_t* S, int nS, hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk) {
  hb_ctx* c = nullptr;
  HB_TRY(check_polys(c0, nitems, &c, "hb_relinearize")); HB_TRY(check_polys(c1, nitems, &c, "hb_relinearize")); HB_TRY(check_polys(c2, nitems, &c, "hb_relinearize"));
  HB_TRY(check_idx(c, S, nS, "hb_relinearize"));
  if (c->special.empty()) return hb_fail(HB_ERR_BAD_ARG, "hb_relinearize: context has no special primes");
  const int maxdig = c->ndigits;
  std::vector<hb_poly*> dig; HB_TRY(pool_get(c, nitems * maxdig, dig));
  KsSets K; HB_TRY(ks_sets(c, S, nS, "breakIntoDigits", K));
  // a seeded key: its a_i are regenerated once for the whole call, on the rows S | special, before either path below
  std::vector<hb_poly*> ka; HB_TRY(relin_key(c, K, evk_a, evk_b, ndig_evk, "hb_relinearize", ka)); evk_a = ka.data();
  // a digit below the last live one may have no live prime (an index set with a hole): the reference then carries a zero digit
  // and still divides the later ones by that digit's full product (src/DoubleCRT.cpp:488-493,509-561); the fused path converts
  // from the digit's own rows and has nothing to convert from, so such sets take the step-by-step path below
  bool hole = false;
  {
    int last = -1; std::vector<char> live(c->ndigits > 0 ? c->ndigits : 1, 0);
    for (int i = 0; i < nS; i++) { const int d = c->digit_of[S[i]]; if (d >= 0) { live[d] = 1; last = std::max(last, d); } }
    for (int d = 0; d < last; d++) if (!live[d]) hole = true;
    if (last + 1 > 4) hole = true;   // the fused inner product is instantiated for up to four digits (c <= 4)
  }
  if (v1_blk_ok(c) && v1_cols_ok(c) && !c->gen.on && !hole && !getenv("HB_NO_FUSED_RELIN"))
    return relin_fused_v1(c, c0, c1, c2, nitems, S, nS, K, evk_a, evk_b, dig);
  // keySwitchPart (src/Ctxt.cpp:805-842)
  int nd = 0;
  HB_TRY(hb_break_into_digits(c2, nitems, S, nS, dig.data(), maxdig, &nd));
  return keyswitch_digits_impl(dig.data(), maxdig, nd, nitems, K.Sp.data(), (int)K.Sp.size(), evk_a, evk_b, c0, c1, K.scp.data(), 0, nullptr);
}

// bringToSet(S) of each item's parts fused with their product on the register kernels (power-of-two m, something dropped):
// per chunk of items, the inverse blk phase and the conversion of every part into adjacent scratch slots (np*i .. np*i+np-1),
// then one k1_fwd_blk_tensor pass (parts a0, a1, b0, b1 of an operand pair: the products over (a0, a1, b0) and b1's rescaled
// rows, as the separate rescale leaves them) or k1_fwd_blk_square pass (parts a0, a1 of a ciphertext: a0^2 and 2*a0*a1 over
// (a0, a1), a1^2 into o2).  The rescaled parts never make a round trip through HBM.  norms (optional): ||delta/P|| of each part,
// from the same conversion and norm_chunk as hb_scale_down_norm.
static int rescale_product_v1(hb_ctx* c, std::initializer_list<hb_poly* const*> parts, hb_poly* const* o2, int nitems,
                              const int32_t* S_in, int nS_in, const int32_t* S, int nS, uint64_t ptxt_space, double* norms) {
  const int np = (int)parts.size();
  std::vector<int32_t> diff, kept; std::vector<u64> sc;
  HB_TRY(scale_down_sets(c, S_in, nS_in, S, nS, ptxt_space, diff, kept, sc));
  if (diff.empty()) return hb_fail(HB_ERR_INDEX_SET, "the fused rescale needs a dropped prime");
  // ---- the rescale's arguments are checked (as scale_down_impl checks them) before its first launch
  HB_TRY(ctx_scratch(c));
  const int per = std::max(1, g_chunk / np);   // items per chunk (the scratch holds HB_MAXB >= 4 parts)
  for (int i0 = 0; i0 < nitems; i0 += per) {
    const int nit = std::min(per, nitems - i0);
    u64* P[HB_MAXB]; u64* tB[HB_MAXB]; u64* O2[HB_MAXB];
    for (int i = 0; i < nit; i++) {
      int k = 0;
      for (hb_poly* const* x : parts) P[np * i + k++] = x[i0 + i]->d;
      if (o2) O2[i] = o2[i0 + i]->d;
    }
    tmp_ptrs(c, c->tmpB, np * nit, tB);
    HB_TRY(conv_chunk(c, P, np * nit, diff.data(), (int)diff.size(), kept.data(), (int)kept.size(), ptxt_space, 0, norms != nullptr));
    HB_TRY(launch_blk_parts_v1(c, np, (const u64* const*)tB, P, o2 ? O2 : nullptr, nit, kept.data(), (int)kept.size(), sc.data()));
    if (norms) HB_TRY(norm_chunk(c, np * nit, norms + np * (size_t)i0));
  }
  return HB_OK;
}

// Operands over S_in are brought to S (bringToSet, src/Ctxt.cpp:373-389): S must lie within S_in.  what names S for the message.
static int check_subset(const int32_t* S_in, int nS_in, const int32_t* S, int nS, const char* who, const char* what) {
  for (int i = 0; i < nS; i++)
    if (std::find(S_in, S_in + nS_in, S[i]) == S_in + nS_in)
      return hb_fail(HB_ERR_INDEX_SET, "%s: the %s set must be a subset of the operands' set (prime %d)", who, what, S[i]);
  return HB_OK;
}

// reLinearize (src/Ctxt.cpp:720-786) of (c0, c1, c2) over S | special through hb_relinearize's fused or step-by-step path,
// then, with moddown, drop the special primes again: modDownToSet of (c0, c1) to S (src/Ctxt.cpp:589-593).
static int relin_moddown(hb_poly* const* c0, hb_poly* const* c1, hb_poly* const* c2, int nitems, const int32_t* S, int nS,
                         const KsSets& K, uint64_t ptxt_space, hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk, bool moddown) {
  HB_TRY(hb_relinearize(c0, c1, c2, nitems, S, nS, evk_a, evk_b, ndig_evk));
  if (!moddown) return HB_OK;
  std::vector<hb_poly*> two;
  for (int i = 0; i < nitems; i++) { two.push_back(c0[i]); two.push_back(c1[i]); }
  return hb_scale_down(two.data(), (int)two.size(), K.Sp.data(), (int)K.Sp.size(), S, nS, ptxt_space);
}

// Chunks of at most c->chunk items for the entry points that relinearise chunk by chunk: c->ip grows to one s^2 scratch poly
// per item of a chunk, and f(i0, nit) runs per chunk with g_chunk = c->chunk.
template <class F> static int ip_chunks(hb_ctx* c, int nitems, F f) {
  const int G = std::min(nitems, c->chunk);
  while ((int)c->ip.size() < G) { hb_poly* p; HB_TRY(hb_poly_create(c, &p)); c->ip.push_back(p); }
  for (int i0 = 0; i0 < nitems; i0 += G) {
    g_chunk = c->chunk;
    HB_TRY(f(i0, std::min(G, nitems - i0)));
  }
  return HB_OK;
}

extern "C" int hb_mul_relin_moddown(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1, int nitems,
                                    const int32_t* S_in, int nS_in, const int32_t* S, int nS, uint64_t ptxt_space,
                                    hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk) {
  hb_ctx* c = nullptr;
  HB_TRY(check_polys(a0, nitems, &c, "hb_mul_relin_moddown")); HB_TRY(check_polys(a1, nitems, &c, "hb_mul_relin_moddown"));
  HB_TRY(check_polys(b0, nitems, &c, "hb_mul_relin_moddown")); HB_TRY(check_polys(b1, nitems, &c, "hb_mul_relin_moddown"));
  {   // the product is formed in place over four distinct polys: a repeated one would receive two results
    std::set<const hb_poly*> ops(a0, a0 + nitems); ops.insert(a1, a1 + nitems); ops.insert(b0, b0 + nitems); ops.insert(b1, b1 + nitems);
    if (ops.size() != 4 * (size_t)nitems)
      return hb_fail(HB_ERR_BAD_ARG, "hb_mul_relin_moddown: the operand polys must be distinct (to square a ciphertext, use hb_square_relin_moddown)");
  }
  // bringToSet(common) on both operands: modDownToSet -> scaleDownToSet per part (src/Ctxt.cpp:393-562)
  HB_TRY(check_subset(S_in, nS_in, S, nS, "hb_mul_relin_moddown", "common"));
  HB_TRY(check_idx(c, S, nS, "hb_mul_relin_moddown"));
  KsSets K; HB_TRY(ks_sets(c, S, nS, "breakIntoDigits", K));
  std::vector<hb_poly*> ka; HB_TRY(relin_key(c, K, evk_a, evk_b, ndig_evk, "hb_mul_relin_moddown", ka)); evk_a = ka.data();
  // tensorProduct in place: (a0,a1,b0) <- (a0*b0, a0*b1+a1*b0, a1*b1)   (src/Ctxt.cpp:1563-1608)
  if (v1_blk_ok(c) && !c->gen.on && nS < nS_in) {   // S is a subset of S_in: something is dropped
    HB_TRY(rescale_product_v1(c, {a0, a1, b0, b1}, nullptr, nitems, S_in, nS_in, S, nS, ptxt_space, nullptr));
  } else {
    std::vector<hb_poly*> allp;
    for (int i = 0; i < nitems; i++) { allp.push_back(a0[i]); allp.push_back(a1[i]); allp.push_back(b0[i]); allp.push_back(b1[i]); }
    HB_TRY(scale_down_impl(allp.data(), (int)allp.size(), S_in, nS_in, S, nS, ptxt_space, nullptr, c->gen.on ? 0 : 1));   // lazy rows: the tensor product reduces exactly
    HB_TRY(hb_tensor(a0, a1, b0, b1, a0, a1, b0, nitems, S, nS));
  }
  return relin_moddown(a0, a1, b0, nitems, S, nS, K, ptxt_space, evk_a, evk_b, ndig_evk, true);
}

// innerProduct (src/Ctxt.cpp:2878-2893) of operands already brought to one prime set: sum_j multLowLvl(a_j, b_j), then one
// reLinearize and, if asked, the mod-down of hb_mul_relin_moddown.  Per chunk of items, k1_tensor_sum writes the summed
// s^0 and s^1 parts straight into out0/out1 and the s^2 part into one scratch poly per item, which the relinearisation
// consumes.  Operands over S_in with S a strict subset are brought to S first by the lazy scale-down, in place (each distinct
// operand poly once, so a == b is allowed).
extern "C" int hb_inner_product(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* b0, hb_poly* const* b1, int npairs, int nitems,
                                const int32_t* S_in, int nS_in, const int32_t* S, int nS, uint64_t ptxt_space,
                                hb_poly* const* evk_a, hb_poly* const* evk_b, int ndig_evk, hb_poly* const* out0, hb_poly* const* out1, int moddown) {
  static const char* who = "hb_inner_product";
  if (npairs <= 0 || nitems <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: npairs and nitems must be positive", who);
  if (moddown != 0 && moddown != 1) return hb_fail(HB_ERR_BAD_ARG, "%s: moddown must be 0 or 1", who);
  hb_ctx* c = nullptr;
  const int np = npairs * nitems;
  HB_TRY(check_polys(a0, np, &c, who)); HB_TRY(check_polys(a1, np, &c, who)); HB_TRY(check_polys(b0, np, &c, who)); HB_TRY(check_polys(b1, np, &c, who));
  HB_TRY(check_polys(out0, nitems, &c, who)); HB_TRY(check_polys(out1, nitems, &c, who));
  HB_TRY(check_idx(c, S_in, nS_in, who)); HB_TRY(check_idx(c, S, nS, who));
  HB_TRY(check_subset(S_in, nS_in, S, nS, who, "common"));
  if (ptxt_space < 1) return hb_fail(HB_ERR_BAD_ARG, "%s: ptxt_space must be at least 1", who);
  if (c->special.empty()) return hb_fail(HB_ERR_BAD_ARG, "%s: context has no special primes", who);
  KsSets K; HB_TRY(ks_sets(c, S, nS, who, K));
  const KsKeys key = {1, nullptr, evk_a, evk_b, "evk"};
  HB_TRY(ks_check_keys(c, &key, 1, K.nd, ndig_evk, K.Sp, who));
  std::set<const hb_poly*> in(a0, a0 + np); in.insert(a1, a1 + np); in.insert(b0, b0 + np); in.insert(b1, b1 + np);
  HB_TRY(check_acc(in, &key, 1, K.nd, ndig_evk, out0, out1, nitems, who));
  // ---- every argument is checked: nothing was launched before this point
  std::vector<hb_poly*> ka; HB_TRY(ks_expand_a(c, evk_a, K.nd, K.Sp.data(), (int)K.Sp.size(), ka)); evk_a = ka.data();
  if (nS < nS_in) {   // bringToSet(S) of every operand part (src/Ctxt.cpp:373-389), lazy rows: the tensor sum reduces on load
    std::vector<hb_poly*> parts; std::set<const hb_poly*> seen;
    for (hb_poly* const* x : {a0, a1, b0, b1})
      for (int i = 0; i < np; i++) if (seen.insert(x[i]).second) parts.push_back(x[i]);
    HB_TRY(scale_down_impl(parts.data(), (int)parts.size(), S_in, nS_in, S, nS, ptxt_space, nullptr, c->gen.on ? 0 : 1));
  }
  return ip_chunks(c, nitems, [&](int i0, int nit) {
    const size_t e = (size_t)i0 * npairs;
    HB_TRY(tensor_sum_impl(c, a0 + e, a1 + e, b0 + e, b1 + e, npairs, nit, S, nS, out0 + i0, out1 + i0, c->ip.data(), 0));
    return relin_moddown(out0 + i0, out1 + i0, c->ip.data(), nit, S, nS, K, ptxt_space, evk_a, evk_b, ndig_evk, moddown != 0);
  });
}

// bringToSet(S) of each ciphertext's two parts and its self-tensor: HElib's squaring multLowLvl (src/Ctxt.cpp:1704-1708,
// 1748-1751) before reLinearize, on checked arguments.  (a0, a1) over S_in become (a0^2, 2*a0*a1) over S and o2 receives
// a1^2, all canonical.  norms (optional, [2*nitems]): norms[2i + k] = ||delta/P|| of part k of item i, from the same
// conversion and norm_chunk as hb_scale_down_norm (0 when nothing is dropped).
// Register path (power-of-two m, something dropped): rescale_product_v1 of the two parts, one k1_fwd_blk_square pass per
// chunk.  Otherwise scale_down_impl of the parts (lazy rows only where k1_tensor follows) and
// hb_tensor(a0, a1, a0, a1 -> a0, a1, o2): k1_tensor and HB_PW_TENSOR read all four inputs of a position before they write
// any output there, so the in-place self-tensor is exact.
static int square_tensor_impl(hb_ctx* c, hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* o2, int nitems,
                              const int32_t* S_in, int nS_in, const int32_t* S, int nS, uint64_t ptxt_space, double* norms) {
  if (norms) std::fill(norms, norms + 2 * (size_t)nitems, 0.0);
  if (v1_blk_ok(c) && !c->gen.on && nS < nS_in)   // S is a strict subset of S_in: something is dropped
    return rescale_product_v1(c, {a0, a1}, o2, nitems, S_in, nS_in, S, nS, ptxt_space, norms);
  std::vector<hb_poly*> parts;
  for (int i = 0; i < nitems; i++) { parts.push_back(a0[i]); parts.push_back(a1[i]); }
  HB_TRY(scale_down_impl(parts.data(), (int)parts.size(), S_in, nS_in, S, nS, ptxt_space, norms, c->gen.on ? 0 : 1));
  return hb_tensor(a0, a1, a0, a1, a0, a1, o2, nitems, S, nS);
}
// The checks shared by the squaring entry points: the operand polys and S within S_in.  The operands are rescaled in place,
// so each poly may appear once only.
static int square_check_args(hb_poly* const* a0, hb_poly* const* a1, int nitems, const int32_t* S_in, int nS_in, const int32_t* S, int nS,
                             uint64_t ptxt_space, const char* who, hb_ctx** c, std::set<const hb_poly*>& in) {
  if (nitems <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: nitems must be positive", who);
  HB_TRY(check_polys(a0, nitems, c, who)); HB_TRY(check_polys(a1, nitems, c, who));
  HB_TRY(check_idx(*c, S_in, nS_in, who)); HB_TRY(check_idx(*c, S, nS, who));
  HB_TRY(check_subset(S_in, nS_in, S, nS, who, "target"));
  if (ptxt_space < 1) return hb_fail(HB_ERR_BAD_ARG, "%s: ptxt_space must be at least 1", who);
  in.clear(); in.insert(a0, a0 + nitems); in.insert(a1, a1 + nitems);
  if (in.size() != 2 * (size_t)nitems) return hb_fail(HB_ERR_BAD_ARG, "%s: the operand polys must be distinct", who);
  return HB_OK;
}
static int square_tensor_entry(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* o2, int nitems, const int32_t* S_in, int nS_in,
                               const int32_t* S, int nS, uint64_t ptxt_space, double* norms, const char* who) {
  hb_ctx* c = nullptr;
  std::set<const hb_poly*> in;
  HB_TRY(square_check_args(a0, a1, nitems, S_in, nS_in, S, nS, ptxt_space, who, &c, in));
  HB_TRY(check_polys(o2, nitems, &c, who));
  HB_TRY(check_outputs(in, {o2}, nitems, who));
  // ---- every argument is checked: nothing was launched before this point
  return square_tensor_impl(c, a0, a1, o2, nitems, S_in, nS_in, S, nS, ptxt_space, norms);
}
extern "C" int hb_square_tensor(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* o2, int nitems, const int32_t* S_in, int nS_in,
                                const int32_t* S, int nS, uint64_t ptxt_space) {
  return square_tensor_entry(a0, a1, o2, nitems, S_in, nS_in, S, nS, ptxt_space, nullptr, "hb_square_tensor");
}
extern "C" int hb_square_tensor_norm(hb_poly* const* a0, hb_poly* const* a1, hb_poly* const* o2, int nitems, const int32_t* S_in, int nS_in,
                                     const int32_t* S, int nS, uint64_t ptxt_space, double* norms) {
  if (!norms) return hb_fail(HB_ERR_BAD_ARG, "hb_square_tensor_norm: null output");
  return square_tensor_entry(a0, a1, o2, nitems, S_in, nS_in, S, nS, ptxt_space, norms, "hb_square_tensor_norm");
}

// Ctxt::square (multiplyBy(*this), src/Ctxt.cpp:1757-1774 with the squaring branch of multLowLvl) of nitems ciphertexts
// already at the target set's level, the squaring counterpart of hb_mul_relin_moddown: per chunk of items, the fused
// rescale and self-tensor into (a0, a1) and one s^2 scratch poly per item (c->ip, shared with hb_inner_product), then
// hb_relinearize's fused or step-by-step path over S | special, then the mod-down to S.
extern "C" int hb_square_relin_moddown(hb_poly* const* a0, hb_poly* const* a1, int nitems, const int32_t* S_in, int nS_in,
                                       const int32_t* S, int nS, uint64_t ptxt_space, hb_poly* const* evk_a, hb_poly* const* evk_b,
                                       int ndig_evk) {
  static const char* who = "hb_square_relin_moddown";
  hb_ctx* c = nullptr;
  std::set<const hb_poly*> in;
  HB_TRY(square_check_args(a0, a1, nitems, S_in, nS_in, S, nS, ptxt_space, who, &c, in));
  if (c->special.empty()) return hb_fail(HB_ERR_BAD_ARG, "%s: context has no special primes", who);
  KsSets K; HB_TRY(ks_sets(c, S, nS, who, K));
  const KsKeys key = {1, nullptr, evk_a, evk_b, "evk"};
  HB_TRY(ks_check_keys(c, &key, 1, K.nd, ndig_evk, K.Sp, who));
  for (int i = 0; i < K.nd; i++)   // the operands are written while the key is read
    if (in.count(evk_a[i]) || in.count(evk_b[i])) return hb_fail(HB_ERR_BAD_ARG, "%s: an operand aliases a key polynomial", who);
  // ---- every argument is checked: nothing was launched before this point
  std::vector<hb_poly*> ka; HB_TRY(ks_expand_a(c, evk_a, K.nd, K.Sp.data(), (int)K.Sp.size(), ka)); evk_a = ka.data();
  return ip_chunks(c, nitems, [&](int i0, int nit) {
    HB_TRY(square_tensor_impl(c, a0 + i0, a1 + i0, c->ip.data(), nit, S_in, nS_in, S, nS, ptxt_space, nullptr));
    return relin_moddown(a0 + i0, a1 + i0, c->ip.data(), nit, S, nS, K, ptxt_space, evk_a, evk_b, ndig_evk, true);
  });
}

// ------------------------------------------------------------------------------------------
// hb_ctxt_scaled_sums: k1_scaled_sums on checked arguments.  The tables travel to the context's device buffer in one
// stream-ordered copy (pageable: cudaMemcpyAsync has staged them when it returns, so the caller may free its arrays); the
// buffer only grows.  A launch covers at most HB_MAXROWS rows and HB_MAXB item-output pairs (one item at least, with all
// its outputs, so that every input row is read once); more than HB_SSUM_MAXIN inputs (the shared-memory stage of one
// thread group) run as input groups, the later ones accumulating into the outputs.
static int scaled_sums_impl(hb_ctx* c, hb_poly* const* in0, hb_poly* const* in1, int nin, hb_poly* const* out0, hb_poly* const* out1,
                            int nout, int nitems, const int32_t* U, int nU, const uint64_t* scal, const uint64_t* cst, int accumulate) {
  const size_t nsc = (size_t)nout * nin * nU, ncst = cst ? (size_t)nout * nU : 0;
  const size_t npi = (size_t)nitems * nin, npo = (size_t)nitems * nout;
  const size_t words = nsc + ncst + 2 * npi + 2 * npo;
  if (words > c->ssum_cap) {
    if (c->ssum) { HB_CUDA(cudaStreamSynchronize(c->stream)); cudaFree(c->ssum); c->bytes -= c->ssum_cap * 8; c->ssum = nullptr; c->ssum_cap = 0; }
    HB_TRY(ctx_alloc(c, (void**)&c->ssum, words * 8));
    c->ssum_cap = words;
  }
  std::vector<u64> h(words);
  memcpy(h.data(), scal, nsc * 8);
  if (cst) memcpy(h.data() + nsc, cst, ncst * 8);
  u64* pt = h.data() + nsc + ncst;
  for (size_t e = 0; e < npi; e++) { pt[e] = (u64)(uintptr_t)in0[e]->d; pt[npi + e] = (u64)(uintptr_t)in1[e]->d; }
  for (size_t e = 0; e < npo; e++) { pt[2 * npi + e] = (u64)(uintptr_t)out0[e]->d; pt[2 * npi + npo + e] = (u64)(uintptr_t)out1[e]->d; }
  HB_CUDA(cudaMemcpyAsync(c->ssum, h.data(), words * 8, cudaMemcpyHostToDevice, c->stream));
  const u64* d = c->ssum;
  const int per = std::max(1, HB_MAXB / nout);   // items per launch
  for (int g0 = 0; g0 < nin; g0 += HB_SSUM_MAXIN) {
    const int ni = std::min(HB_SSUM_MAXIN, nin - g0);
    int T = 256;   // threads per block: the largest whose stage fits HB_SSUM_SMEM / 3 (HB_SSUM_SMEM for 32 threads)
    while (T > 32 && (size_t)ni * (16 * T + 1) > HB_SSUM_SMEM / 3) T >>= 1;
    const size_t smem = (size_t)ni * (16 * T + 1);
    for (int t0 = 0; t0 < nitems; t0 += per) {
      const int nt = std::min(per, nitems - t0);
      for (int r0 = 0; r0 < nU; r0 += HB_MAXROWS) {
        const int nr = std::min(HB_MAXROWS, nU - r0);
        Hb1ScaledSumsJob J; memset(&J, 0, sizeof(J));
        J.N = c->N; fill_rows(J.rows, U + r0, nr); J.r0 = r0;
        J.nU = nU; J.nin = nin; J.nout = nout; J.i0 = g0; J.ni = ni; J.item0 = t0;
        J.accumulate = accumulate || g0 > 0; J.with_cst = cst != nullptr && g0 == 0;
        J.scal = d; J.cst = cst ? d + nsc : nullptr;
        J.in0 = (const u64* const*)(d + nsc + ncst); J.in1 = J.in0 + npi;
        J.out0 = (u64* const*)(d + nsc + ncst + 2 * npi); J.out1 = J.out0 + npo;
        u64 rd = 0;   // algorithmic bytes: the input rows some output reads, the outputs written (and read back)
        for (int k = 0; k < nr; k++)
          for (int i = g0; i < g0 + ni; i++)
            for (int j = 0; j < nout; j++) if (scal[((size_t)j * nin + i) * nU + r0 + k]) { rd += 2; break; }
        const u64 bytes = (rd + (u64)2 * nout * nr * (J.accumulate ? 2 : 1)) * nt * c->N * 8;
        pre_launch(c);
        HB_LAUNCH(k1_scaled_sums, dim3((unsigned)((c->N + T - 1) / T), nr, nt), dim3(T), smem, c->stream, c->d_primes, J);
        HB_TRY(post_launch(c, "k1_scaled_sums", bytes));
      }
    }
  }
  return HB_OK;
}
extern "C" int hb_ctxt_scaled_sums(hb_poly* const* in0, hb_poly* const* in1, int nin, hb_poly* const* out0, hb_poly* const* out1,
                                   int nout, int nitems, const int32_t* U, int nU, const uint64_t* scal, const uint64_t* cst,
                                   int accumulate) {
  static const char* who = "hb_ctxt_scaled_sums";
  if (nin <= 0 || nout <= 0 || nitems <= 0 || nU <= 0) return hb_fail(HB_ERR_BAD_ARG, "%s: nin, nout, nitems and nU must be positive", who);
  if (accumulate != 0 && accumulate != 1) return hb_fail(HB_ERR_BAD_ARG, "%s: accumulate must be 0 or 1", who);
  if (!U || !scal) return hb_fail(HB_ERR_BAD_ARG, "%s: null row set or scalar table", who);
  hb_ctx* c = nullptr;
  const int np = nin * nitems, no = nout * nitems;
  HB_TRY(check_polys(in0, np, &c, who)); HB_TRY(check_polys(in1, np, &c, who));
  HB_TRY(check_polys(out0, no, &c, who)); HB_TRY(check_polys(out1, no, &c, who));
  for (int r = 0; r < nU; r++) {
    if (U[r] < 0 || U[r] >= c->nprimes) return hb_fail(HB_ERR_INDEX_SET, "%s: prime index %d outside the chain", who, U[r]);
    if (r > 0 && U[r] <= U[r - 1]) return hb_fail(HB_ERR_INDEX_SET, "%s: the row set must be sorted without repeats", who);
  }
  for (int j = 0; j < nout; j++)
    for (int r = 0; r < nU; r++) {
      const u64 q = c->q[U[r]];
      if (cst && cst[(size_t)j * nU + r] >= q) return hb_fail(HB_ERR_BAD_ARG, "%s: constant %d of row %d is not below its prime", who, j, r);
      for (int i = 0; i < nin; i++)
        if (scal[((size_t)j * nin + i) * nU + r] >= q) return hb_fail(HB_ERR_BAD_ARG, "%s: scalar (%d, %d) of row %d is not below its prime", who, j, i, r);
    }
  std::set<const hb_poly*> in(in0, in0 + np); in.insert(in1, in1 + np);
  HB_TRY(check_outputs(in, {out0, out1}, no, who));
  return scaled_sums_impl(c, in0, in1, nin, out0, out1, nout, nitems, U, nU, scal, cst, accumulate);
}
