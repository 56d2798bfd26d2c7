// hb_device_prg.cuh -- device expansion of a PRG seed into uniform DoubleCRT rows (DoubleCRT::randomize after
// NTL::SetSeed, src/DoubleCRT.cpp:1258-1378; src/keys.cpp:1199-1206 and src/Ctxt.cpp:191-230 call it with prgSeed).
//
// The stream: key = DeriveKey(32, seed bytes) (HMAC-SHA256, host code below), then ChaCha20 (20 rounds,
// "expand 32-byte k", 64-bit block counter in words 12-13 from 0, zero nonce).  DoubleCRT::randomize consumes it in
// 2048-byte buffers, so buffer b is exactly the key-stream blocks 32b .. 32b+31 and can be generated on its own.
// Per row: a fresh buffer at the start, nb = ceil(k/8) little-endian bytes per candidate (k = bits(q-1)), masked to
// k bits, accepted when < q, floor(2048/nb) candidates per buffer (the tail bytes are skipped); once the row holds N
// values the rest of its last buffer is discarded.  Rows are filled in index order, polys one after another.
//
// The only serial dependency is where each row starts: B_{t+1} = B_t + need_t.  Two kernels:
//   k_prg_count  one launch per row t: one warp per buffer B_t + w (w < window_t) counts the accepted candidates;
//                the last CTA to finish (atomic ticket; no spin waits, no grid-wide barrier) scans the counts into
//                per-buffer row offsets and writes B_{t+1} to device memory, which the next launch reads.  A row that
//                needs more than window_t buffers is finished by that CTA itself, 8 buffers at a time (slow path).
//   k_prg_fill   one launch over all (row, buffer): regenerates each buffer, compacts its accepted candidates with a
//                ballot prefix sum and writes them to row[offset + rank] for positions < N.  Each launch row names the
//                schedule row it reads, so a kept schedule (hb_poly_create_seeded) refills any subset of its rows later.
// A warp makes one buffer, one 64-byte block per lane; the ChaCha state stays in registers and the candidates are read
// back through the warp's 2 KB slice of shared memory.
#pragma once

#include <cmath>
#include <cstring>
#include <vector>

#define HB_PRG_BUF 2048                      // bytes per refill of DoubleCRT::randomize
#define HB_PRG_WORDS (HB_PRG_BUF / 8)        // u64 words per buffer
#define HB_PRG_WARPS 8
#define HB_PRG_THREADS (32 * HB_PRG_WARPS)
#define HB_PRG_MAXT 256                      // rows per k_prg_fill launch (job descriptor: 8 KB of row records)
#define HB_PRG_WARP_SMEM (HB_PRG_WORDS + 1 + 16)   // buffer + one zero word (candidates read two words) + 32 u32 lane scratch
#define HB_PRG_SMEM_BYTES ((HB_PRG_WARPS * HB_PRG_WARP_SMEM + 8) * 8)

#ifdef HB_SIM
#define HB_PRG_FENCE() ((void)0)
#define HB_PRG_LDCG(p) (*(p))
static inline unsigned hb_prg_popc(unsigned x) { return (unsigned)__builtin_popcount(x); }
// the simulator has no warp vote: the lanes exchange their values through the warp's scratch words
static inline unsigned hb_prg_ballot(bool p, unsigned* scr, unsigned lane) {
  scr[lane] = p ? 1u : 0u;
  __syncwarp();
  unsigned m = 0;
  for (unsigned i = 0; i < 32; i++) m |= scr[i] << i;
  __syncwarp();
  return m;
}
static inline unsigned hb_prg_wsum(unsigned v, unsigned* scr, unsigned lane) {
  scr[lane] = v;
  __syncwarp();
  unsigned s = 0;
  for (unsigned i = 0; i < 32; i++) s += scr[i];
  __syncwarp();
  return s;
}
#else
#define HB_PRG_FENCE() __threadfence()
#define HB_PRG_LDCG(p) __ldcg(p)
__device__ __forceinline__ unsigned hb_prg_popc(unsigned x) { return (unsigned)__popc(x); }
__device__ __forceinline__ unsigned hb_prg_ballot(bool p, unsigned*, unsigned) { return __ballot_sync(0xffffffffu, p); }
__device__ __forceinline__ unsigned hb_prg_wsum(unsigned v, unsigned*, unsigned) { return __reduce_add_sync(0xffffffffu, v); }
#endif

struct HbPrgKey { unsigned k[8]; };   // the ChaCha20 key as little-endian words

// one row of the expansion: prime, its candidate format and where its values go
struct HbPrgRow {
  u64 q, mask;       // mask = 2^k - 1, k = bits(q-1)
  u64* row;          // N residues; nullptr in a count that only builds a schedule (hb_poly_create_seeded)
  int nb;            // bytes per candidate, ceil(k/8)
  int window;        // buffers counted in parallel for this row
};

struct HbPrgCountJob {
  HbPrgKey key;
  HbPrgRow r;
  u64 N;
  u64* start;                      // start[t] = first buffer of row t (read), start[t+1] (written)
  unsigned* off;                   // [window] accepted counts, then exclusive row offsets of the buffers
  unsigned long long* ticket;      // CTAs finished; the last one resets it
  int t;
};

// launch row y fills r[y].row from schedule row sr[y]: any subset of a schedule's rows, in any order
struct HbPrgFillJob {
  HbPrgKey key;
  u64 N;
  const u64* start;
  const unsigned* off;             // schedule row s's offsets at off + s*wstride
  int wstride;
  HbPrgRow r[HB_PRG_MAXT];
  unsigned sr[HB_PRG_MAXT];
};

__device__ __forceinline__ unsigned hb_rotl32(unsigned x, int n) { return (x << n) | (x >> (32 - n)); }

#define HB_CHACHA_QR(a, b, c, d)                                   \
  a += b; d ^= a; d = hb_rotl32(d, 16); c += d; b ^= c; b = hb_rotl32(b, 12); \
  a += b; d ^= a; d = hb_rotl32(d, 8);  c += d; b ^= c; b = hb_rotl32(b, 7);

// ChaCha20 block `ctr` (20 rounds, "expand 32-byte k", zero nonce), stored as 8 little-endian u64 at dst.
// Named scalars, so no index into the state is left to the unroller.
__device__ __forceinline__ void hb_chacha_block(const HbPrgKey& K, u64 ctr, u64* dst) {
  const unsigned s0 = 0x61707865u, s1 = 0x3320646Eu, s2 = 0x79622D32u, s3 = 0x6B206574u;
  const unsigned s4 = K.k[0], s5 = K.k[1], s6 = K.k[2], s7 = K.k[3], s8 = K.k[4], s9 = K.k[5], s10 = K.k[6], s11 = K.k[7];
  const unsigned s12 = (unsigned)ctr, s13 = (unsigned)(ctr >> 32);
  unsigned x0 = s0, x1 = s1, x2 = s2, x3 = s3, x4 = s4, x5 = s5, x6 = s6, x7 = s7;
  unsigned x8 = s8, x9 = s9, x10 = s10, x11 = s11, x12 = s12, x13 = s13, x14 = 0, x15 = 0;
#pragma unroll 2
  for (int i = 0; i < 10; i++) {
    HB_CHACHA_QR(x0, x4, x8, x12) HB_CHACHA_QR(x1, x5, x9, x13) HB_CHACHA_QR(x2, x6, x10, x14) HB_CHACHA_QR(x3, x7, x11, x15)
    HB_CHACHA_QR(x0, x5, x10, x15) HB_CHACHA_QR(x1, x6, x11, x12) HB_CHACHA_QR(x2, x7, x8, x13) HB_CHACHA_QR(x3, x4, x9, x14)
  }
  dst[0] = (u64)(x0 + s0) | (u64)(x1 + s1) << 32;
  dst[1] = (u64)(x2 + s2) | (u64)(x3 + s3) << 32;
  dst[2] = (u64)(x4 + s4) | (u64)(x5 + s5) << 32;
  dst[3] = (u64)(x6 + s6) | (u64)(x7 + s7) << 32;
  dst[4] = (u64)(x8 + s8) | (u64)(x9 + s9) << 32;
  dst[5] = (u64)(x10 + s10) | (u64)(x11 + s11) << 32;
  dst[6] = (u64)(x12 + s12) | (u64)(x13 + s13) << 32;
  dst[7] = (u64)x14 | (u64)x15 << 32;
}

// buffer b of the stream into the warp's shared slice (lane L makes block 32b + L)
__device__ __forceinline__ void hb_prg_gen(const HbPrgKey& K, u64 b, u64* buf, unsigned lane) {
  hb_chacha_block(K, b * 32 + lane, buf + 8 * lane);
  if (lane == 0) buf[HB_PRG_WORDS] = 0;
  __syncwarp();
}

// candidate j: nb little-endian bytes at byte j*nb, masked to k bits
__device__ __forceinline__ u64 hb_prg_cand(const u64* buf, unsigned j, int nb, u64 mask) {
  const unsigned o = j * (unsigned)nb, w = o >> 3, sh = (o & 7) * 8;
  u64 v = buf[w] >> sh;
  if (sh) v |= buf[w + 1] << (64 - sh);
  return v & mask;
}

// accepted candidates of the buffer (every lane gets the total)
__device__ __forceinline__ unsigned hb_prg_count_buf(const u64* buf, unsigned lane, const HbPrgRow& R, unsigned* scr) {
  const unsigned c = HB_PRG_BUF / R.nb;
  unsigned n = 0;
  for (unsigned j = lane; j < c; j += 32) n += hb_prg_cand(buf, j, R.nb, R.mask) < R.q ? 1u : 0u;
  return hb_prg_wsum(n, scr, lane);
}

// the accepted candidates of the buffer, in stream order, to row[pos ...] for positions < N (pos is warp-uniform)
__device__ __forceinline__ void hb_prg_emit(const u64* buf, unsigned lane, const HbPrgRow& R, u64 pos, u64 N, unsigned* scr) {
  const unsigned c = HB_PRG_BUF / R.nb;
  for (unsigned j0 = 0; j0 < c && pos < N; j0 += 32) {
    const unsigned j = j0 + lane;
    const u64 v = j < c ? hb_prg_cand(buf, j, R.nb, R.mask) : R.q;
    const bool ok = v < R.q;
    const unsigned m = hb_prg_ballot(ok, scr, lane);
    const u64 p = pos + hb_prg_popc(m & ((1u << lane) - 1u));
    if (ok && p < N) R.row[p] = v;
    pos += hb_prg_popc(m);
  }
}

__global__ void __launch_bounds__(HB_PRG_THREADS) k_prg_count(const HB_GRID_CONSTANT HbPrgCountJob J) {
  HB_SMEM_DECL
  u64* sm = HB_SMEM;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u64* buf = sm + warp * HB_PRG_WARP_SMEM;
  unsigned* scr = (unsigned*)(buf + HB_PRG_WORDS + 1);
  unsigned* flag = (unsigned*)(sm + HB_PRG_WARPS * HB_PRG_WARP_SMEM);
  const u64 B = HB_PRG_LDCG(J.start + J.t);
  const unsigned W = (unsigned)J.r.window;
  const unsigned w = blockIdx.x * HB_PRG_WARPS + warp;
  if (w < W) {
    hb_prg_gen(J.key, B + w, buf, lane);
    const unsigned n = hb_prg_count_buf(buf, lane, J.r, scr);
    if (lane == 0) J.off[w] = n;
  }
  HB_PRG_FENCE();
  __syncthreads();
  if (threadIdx.x == 0) {
    const bool last = atomicAdd(J.ticket, 1ULL) == (unsigned long long)gridDim.x - 1;
    if (last) *J.ticket = 0;
    flag[0] = last ? 1u : 0u;
  }
  __syncthreads();
  if (!flag[0]) return;
  HB_PRG_FENCE();

  // the last CTA: exclusive scan of the W counts (a contiguous chunk per thread, Hillis-Steele over the chunk sums)
  const unsigned tid = threadIdx.x, per = (W + HB_PRG_THREADS - 1) / HB_PRG_THREADS;
  const unsigned a = tid * per < W ? tid * per : W, e = a + per < W ? a + per : W;
  u64 s = 0;
  for (unsigned i = a; i < e; i++) s += HB_PRG_LDCG(J.off + i);
  u64* part = sm;
  part[tid] = s;
  __syncthreads();
  for (unsigned d = 1; d < HB_PRG_THREADS; d <<= 1) {
    const u64 v = tid >= d ? part[tid] + part[tid - d] : part[tid];
    __syncthreads();
    part[tid] = v;
    __syncthreads();
  }
  const u64 N = J.N, total = part[HB_PRG_THREADS - 1];
  u64 acc = part[tid] - s;
  for (unsigned i = a; i < e; i++) {
    const unsigned cnt = HB_PRG_LDCG(J.off + i);
    if (acc < N && acc + cnt >= N) J.start[J.t + 1] = B + i + 1;
    J.off[i] = (unsigned)acc;
    acc += cnt;
  }
  __syncthreads();
  if (total >= N) return;   // block-uniform

  // slow path: the window held fewer than N values; this CTA writes the rest of the row, 8 buffers per round (or, when it
  // only builds a schedule, just finds the next row's start)
  unsigned* wc = flag + 2;
  u64 base = total, b = B + W;
  while (base < N) {
    hb_prg_gen(J.key, b + warp, buf, lane);
    const unsigned n = hb_prg_count_buf(buf, lane, J.r, scr);
    if (lane == 0) wc[warp] = n;
    __syncthreads();
    u64 pos = base, tot = 0;
    for (unsigned i = 0; i < HB_PRG_WARPS; i++) { if (i < warp) pos += wc[i]; tot += wc[i]; }
    if (J.r.row) hb_prg_emit(buf, lane, J.r, pos, N, scr);   // grid-uniform
    if (lane == 0 && pos < N && pos + n >= N) J.start[J.t + 1] = b + warp + 1;
    __syncthreads();
    base += tot;
    b += HB_PRG_WARPS;
  }
}

// grid = (ceil(largest window / 8), rows of this launch)
__global__ void __launch_bounds__(HB_PRG_THREADS) k_prg_fill(const HB_GRID_CONSTANT HbPrgFillJob J) {
  HB_SMEM_DECL
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const HbPrgRow& R = J.r[blockIdx.y];
  const unsigned w = blockIdx.x * HB_PRG_WARPS + warp;
  if (w >= (unsigned)R.window) return;   // warp-uniform; the kernel has no CTA barrier
  const size_t t = J.sr[blockIdx.y];
  const u64 pos = J.off[t * J.wstride + w];
  if (pos >= J.N) return;                 // past the buffer that completes the row
  u64* buf = HB_SMEM + warp * HB_PRG_WARP_SMEM;
  unsigned* scr = (unsigned*)(buf + HB_PRG_WORDS + 1);
  hb_prg_gen(J.key, J.start[t] + w, buf, lane);
  hb_prg_emit(buf, lane, R, pos, J.N, scr);
}

// ---- host: NTL's DeriveKey(32, seed) = HMAC-SHA256(HMAC-SHA256("", seed), le64(0)) -------------------------------
// SHA-256 (FIPS 180-4) and HMAC (RFC 2104), written out so the library links nothing new.
namespace hbprg {
static const unsigned K256[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
    0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
    0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
    0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
    0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
    0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
static inline unsigned rotr(unsigned x, int n) { return (x >> n) | (x << (32 - n)); }
static void sha256(const unsigned char* msg, size_t len, unsigned char out[32]) {
  unsigned h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
  std::vector<unsigned char> m(msg, msg + len);
  m.push_back(0x80);
  while (m.size() % 64 != 56) m.push_back(0);
  const unsigned long long bits = (unsigned long long)len * 8;
  for (int i = 7; i >= 0; i--) m.push_back((unsigned char)(bits >> (8 * i)));
  for (size_t blk = 0; blk < m.size(); blk += 64) {
    unsigned w[64];
    for (int i = 0; i < 16; i++)
      w[i] = (unsigned)m[blk + 4 * i] << 24 | (unsigned)m[blk + 4 * i + 1] << 16 | (unsigned)m[blk + 4 * i + 2] << 8 | m[blk + 4 * i + 3];
    for (int i = 16; i < 64; i++) {
      const unsigned s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
      const unsigned s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
      w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    unsigned a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
    for (int i = 0; i < 64; i++) {
      const unsigned t1 = hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K256[i] + w[i];
      const unsigned t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
      hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
  }
  for (int i = 0; i < 8; i++)
    for (int j = 0; j < 4; j++) out[4 * i + j] = (unsigned char)(h[i] >> (24 - 8 * j));
}
static void hmac_sha256(const unsigned char* key, size_t klen, const unsigned char* msg, size_t len, unsigned char out[32]) {
  unsigned char k0[64] = {0};
  if (klen > 64) sha256(key, klen, k0);
  else if (klen) std::memcpy(k0, key, klen);
  std::vector<unsigned char> in(64 + len);
  for (int i = 0; i < 64; i++) in[i] = k0[i] ^ 0x36;
  if (len) std::memcpy(in.data() + 64, msg, len);
  unsigned char ih[32];
  sha256(in.data(), in.size(), ih);
  unsigned char o[96];
  for (int i = 0; i < 64; i++) o[i] = k0[i] ^ 0x5c;
  std::memcpy(o + 64, ih, 32);
  sha256(o, 96, out);
}
}  // namespace hbprg

// NTL::SetSeed(const ZZ&) on the magnitude bytes `seed` (little-endian; high-order zero bytes do not count)
static HbPrgKey hb_prg_derive_key(const unsigned char* seed, int seedlen) {
  while (seedlen > 0 && seed[seedlen - 1] == 0) seedlen--;
  unsigned char K[32], key[32];
  hbprg::hmac_sha256(nullptr, 0, seed, (size_t)seedlen, K);
  const unsigned char ctr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  hbprg::hmac_sha256(K, 32, ctr, 8, key);
  HbPrgKey r;
  for (int i = 0; i < 8; i++) r.k[i] = (unsigned)key[4 * i] | (unsigned)key[4 * i + 1] << 8 | (unsigned)key[4 * i + 2] << 16 | (unsigned)key[4 * i + 3] << 24;
  return r;
}

// buffers counted in parallel for a row: the mean count per buffer under q/2^k, less 8 standard deviations of the total,
// must reach N; one buffer of slack on top.  Rows that still run short finish on the slow path.
static int hb_prg_window(u64 q, int k, int nb, u64 N) {
  const double p = std::ldexp((double)q, -k), c = (double)(HB_PRG_BUF / nb);
  const double mu = c * p, var = c * p * (1.0 - p);
  long W = (long)((double)N / mu);
  if (W < 1) W = 1;
  while ((double)W * mu - 8.0 * std::sqrt((double)W * var) < (double)N) W++;
  return (int)(W + 1);
}
