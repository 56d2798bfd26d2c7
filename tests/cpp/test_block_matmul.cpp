// Block linear maps through the C++ mirror: hb::BlockMatMul1D, BlockMatMul1DExec::mul's non-iterative branches (FULL
// strategies, one thread; src/matmul.cpp:1663-1976) in one hb_block_linear_map_norm call.  Checks:
//  - the result equals a literal transcription of the loop (BasicAutomorphPrecon rotations, MulAdd into d1 sums, the outer
//    smartAutomorphs, +=, and the bad dimension's second sum rotated by gen^-D) bit for bit, with equal metadata, for
//    strategies +1 and -1, native and bad, with NULL blocks and a whole zero output;
//  - it decrypts to sum_j sigma_{k1_j}( sum_i C_ij(X) * m(X^{k0_i}) ) (+ the second set's sum rotated by gen^-D), mod p;
//  - the tracked noise bound dominates the decrypted polynomial's largest coefficient;
//  - an outer amount without a direct matrix takes the loop and still matches;
//  - CKKS is refused with LogicError.
// Exit codes: 0 ok, 3 no CUDA device, 1 failure.
#include <algorithm>
#include <cstdio>
#include <random>

#include "helib_b200_ctxt.hpp"

using namespace hb;

static std::vector<long> sample_ternary(std::mt19937_64& g, long n) { std::vector<long> v(n); for (auto& x : v) x = (long)(g() % 3) - 1; return v; }
static std::vector<long> sample_gauss(std::mt19937_64& g, long n, double sigma) { std::normal_distribution<double> d(0, sigma); std::vector<long> v(n); for (auto& x : v) x = std::lround(d(g)); return v; }
static DoubleCRT random_rows(const Context& ctx, const IndexSet& s, std::mt19937_64& g) {
  const long N = ctx.getPhiM();
  std::vector<uint64_t> dense((size_t)ctx.numPrimes() * N, 0);
  for (long i : s) for (long k = 0; k < N; k++) dense[(size_t)i * N + k] = g() % (uint64_t)ctx.ithPrime(i);
  return DoubleCRT::fromRows(ctx, s, dense);
}
static bool same_rows(const DoubleCRT& x, const DoubleCRT& y) {
  if (!(x.getIndexSet() == y.getIndexSet())) return false;
  for (long i : x.getIndexSet()) if (x.getOneRow(i) != y.getOneRow(i)) return false;
  return true;
}
static bool same_xd(const XD& a, const XD& b) { return a.m == b.m && a.e == b.e; }
static const char* differs(const Ctxt& x, const Ctxt& y) {
  if (x.parts.size() != y.parts.size()) return "number of parts";
  for (size_t j = 0; j < x.parts.size(); j++) {
    const long k = y.getPartIndexByHandle(x.parts[j].skHandle);
    if (k < 0 || !same_rows(x.parts[j].dcrt, y.parts[k].dcrt)) return "part rows";
  }
  if (!(x.primeSet == y.primeSet)) return "primeSet";
  if (x.ptxtSpace != y.ptxtSpace) return "ptxtSpace";
  if (x.intFactor != y.intFactor) return "intFactor";
  if (!same_xd(x.noiseBound, y.noiseBound)) return "noiseBound";
  if (!same_xd(x.ratFactor, y.ratFactor)) return "ratFactor";
  if (!same_xd(x.ptxtMag, y.ptxtMag)) return "ptxtMag";
  return nullptr;
}
static long double limbs_to_ld(const uint64_t* w, int L) {
  const bool neg = w[L - 1] >> 63;
  long double mag = 0;
  for (int l = L - 1; l >= 0; l--) mag = mag * 18446744073709551616.0L + (long double)(neg ? ~w[l] : w[l]);
  return neg ? -(mag + 1) : mag;
}
// f(X^k) mod X^N + 1
static std::vector<long> rotate(const std::vector<long>& f, long k, long N) {
  std::vector<long> out(N, 0);
  for (long i = 0; i < N; i++) { const long j = (i * k) % (2 * N); if (j < N) out[j] += f[i]; else out[j - N] -= f[i]; }
  return out;
}
// coefficient t of a*b mod X^N + 1
static long negacyclic_at(const std::vector<long>& a, const std::vector<long>& b, long t, long N) {
  long acc = 0;
  for (long i = 0; i < N; i++) { const long j = t - i; acc += j >= 0 ? a[i] * b[j] : -(a[i] * b[j + N]); }
  return acc;
}

struct Keys {
  KeyInfo pk;
  DoubleCRT S;
  std::vector<DoubleCRT> sKeys;
};

// s(X^k) -> s for every k in rots; the key-switching map then reaches products of them through several matrices
static void make_keys(Keys& K, const Context& ctx, const std::vector<long>& rots, long p, bool ckks, std::mt19937_64& gen) {
  const long N = ctx.getPhiM();
  K.pk.context = &ctx; K.pk.ckks = ckks; K.pk.scale = 10.0; K.pk.hwt = 0;
  K.pk.skBound = K.pk.scale * std::sqrt(double(N) * 2.0 / 3.0);
  for (long r : rots) {
    DoubleCRT sr(K.S); sr.automorph(r);
    std::vector<uint8_t> seed(32);
    for (auto& b : seed) b = (uint8_t)(gen() & 0xff);
    seed[31] |= 1;
    K.pk.keySwitching.push_back(genKeySWmatrix(ctx, sr, SKHandle(1, r, 0), 0, K.S, p, ckks, 3.2, gen, seed));
  }
  K.pk.setKeySwitchMap(0);
  K.sKeys.push_back(K.S);
}


// f(X^k) * c(X) mod (X^N + 1, p) for a sparse c
static std::vector<long> mul_sparse(const std::vector<long>& c, const std::vector<long>& f, long N, long p) {
  std::vector<long> out(N, 0);
  for (long a = 0; a < N; a++) {
    if (!c[a]) continue;
    for (long b = 0; b < N; b++) { const long t = a + b, v = c[a] * f[b]; if (t < N) out[t] = (out[t] + v) % p; else out[t - N] = (out[t - N] - v) % p; }
  }
  return out;
}
static void add_into(std::vector<long>& a, const std::vector<long>& b, long p) { for (size_t i = 0; i < a.size(); i++) a[i] = (a[i] + b[i]) % p; }

// the plaintext map: sum_j sigma_{k1_j}( sum_i C_ij * sigma_{k0_i}(m) ) for one set of blocks
static std::vector<long> want_set(const std::vector<std::vector<long>>& C, const std::vector<long>& msg, const std::vector<long>& k0,
                                  const std::vector<long>& k1, long N, long p) {
  const long d0 = (long)k0.size(), d1 = (long)k1.size();
  std::vector<long> out(N, 0);
  for (long j = 0; j < d1; j++) {
    std::vector<long> a(N, 0);
    for (long i = 0; i < d0; i++)
      if (!C[(size_t)(i * d1 + j)].empty()) add_into(a, mul_sparse(C[(size_t)(i * d1 + j)], rotate(msg, k0[(size_t)i], N), N, p), p);
    add_into(out, rotate(a, k1[(size_t)j], N), p);
  }
  return out;
}

static int bgv_case(long D, long d, bool bad, bool direct_outer) {
  const long m = 2048, p = 257, gen = 3;
  Context ctx(m, p, 1, /*bits=*/200, /*c=*/2);
  const long N = ctx.getPhiM();
  std::mt19937_64 gen64(20261016 + 10 * D + d + 100 * bad);
  const double sigma = 3.2;
  const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
  Keys K{KeyInfo(), DoubleCRT(sample_ternary(gen64, N), ctx, allq), {}};
  const bool plus = D >= d;
  const long d0 = plus ? D : d, d1 = plus ? d : D;
  std::vector<long> k0(d0), k1(d1);
  for (long i = 0; i < d0; i++) k0[i] = plus ? genToPow(gen, i, m) : genToPow(p, i, m);
  for (long j = 0; j < d1; j++) k1[j] = plus ? genToPow(p, j, m) : genToPow(gen, j, m);
  const long kf = genToPow(gen, -D, m);
  // the FULL key set: every inner and outer amount and gen^-D; without direct_outer, k1_2 is reached through k1_1 twice
  std::vector<long> rots;
  for (long k : k0) if (k != 1) rots.push_back(k);
  for (long j = 1; j < d1; j++) if (direct_outer || j != 2) rots.push_back(k1[j]);
  if (bad) rots.push_back(kf);
  std::sort(rots.begin(), rots.end()); rots.erase(std::unique(rots.begin(), rots.end()), rots.end());
  make_keys(K, ctx, rots, p, false, gen64);
  Ctxt pubEncrKey(K.pk, p);
  pubEncrKey.primeSet = ctx.getCtxtPrimes();
  DoubleCRT c1 = random_rows(ctx, pubEncrKey.primeSet, gen64);
  DoubleCRT c0(sample_gauss(gen64, N, sigma), ctx, pubEncrKey.primeSet); c0 *= p;
  DoubleCRT t(c1); t.Mul(K.S, false); c0 -= t;
  pubEncrKey.parts.emplace_back(c0, SKHandle());
  pubEncrKey.parts.emplace_back(c1, SKHandle(1, 1, 0));
  pubEncrKey.noiseBound = XD(double(p) * K.pk.noiseBoundForGaussian(sigma, N));
  std::vector<long> msg(N);
  for (auto& x : msg) x = (long)(gen64() % p);
  Ctxt c(K.pk, p);
  hb::EncryptionSample smp = hb::drawEncryptionSample(ctx, sigma, gen64);
  hb::Encrypt(c, pubEncrKey, msg, p, smp);
  // blocks: every fifth NULL, and set 0's output j = 1 without any block
  std::vector<std::vector<long>> cf(d0 * d1), cf1(bad ? d0 * d1 : 0);
  std::vector<DoubleCRT> store;
  store.reserve(2 * d0 * d1);
  std::vector<BsgsDiag> cache(d0 * d1), cache1(bad ? d0 * d1 : 0);
  auto block = [&](std::vector<long>& co, BsgsDiag& b, long e, bool none) {
    b = BsgsDiag{nullptr, e % 3 ? -1.0 : 30.0, XD(), XD(), 0.0};
    if (none || e % 5 == 4) return;
    co.assign(N, 0);
    for (long s = 0; s < 6; s++) co[(size_t)(gen64() % N)] = (long)(gen64() % 5) - 2;
    store.emplace_back(co, ctx, allq);
    b.c = &store.back();
  };
  for (long e = 0; e < d0 * d1; e++) { block(cf[e], cache[e], e, e % d1 == 1); if (bad) block(cf1[e], cache1[e], e + 1, false); }
  // the literal loop of src/matmul.cpp:1782-1868 / 1869-1974 (FULL, one thread), for the bits and the metadata
  Ctxt loop(c);
  {
    loop.cleanUp();
    BasicAutomorphPrecon precon(loop);
    auto mulAdd = [&](Ctxt& acc, const BsgsDiag& b, const Ctxt& r) { if (!b.c) return; Ctxt tmp(r); tmp.multByConstant(*b.c, b.size); acc += tmp; };
    std::vector<Ctxt> acc(d1, Ctxt(K.pk, p)), acc1(bad ? d1 : 0, Ctxt(K.pk, p));
    for (long i = 0; i < d0; i++) {
      auto r = precon.automorph(k0[i]);
      for (long j = 0; j < d1; j++) { mulAdd(acc[j], cache[i * d1 + j], *r); if (bad) mulAdd(acc1[j], cache1[i * d1 + j], *r); }
    }
    Ctxt sum(K.pk, p), sum1(K.pk, p);
    for (long j = 0; j < d1; j++) {
      if (j > 0) { acc[j].smartAutomorph(k1[j]); if (bad) acc1[j].smartAutomorph(k1[j]); }
      sum += acc[j];
      if (bad) sum1 += acc1[j];
    }
    if (bad) { sum1.smartAutomorph(kf); sum += sum1; }
    loop = sum;
  }
  Ctxt got(c);
  const uint64_t l0 = [&] { uint64_t s[3]; check(hb_ctx_stats(ctx.handle(), s)); return s[1]; }();
  BlockMatMul1D(got, gen, D, d, cache, cache1);
  const uint64_t l1 = [&] { uint64_t s[3]; check(hb_ctx_stats(ctx.handle(), s)); return s[1]; }();
  const char* tag = plus ? "+1" : "-1";
  if (const char* what = differs(got, loop)) { std::printf("BGV D=%ld d=%ld %s bad=%d: BlockMatMul1D differs from the loop in its %s\n", D, d, tag, (int)bad, what); return 1; }
  std::vector<long> out; std::vector<uint64_t> limbs; int L = 0;
  hb::Decrypt(out, got, K.sKeys, &limbs, &L);
  std::vector<long> want = want_set(cf, msg, k0, k1, N, p);
  if (bad) add_into(want, rotate(want_set(cf1, msg, k0, k1, N, p), kf, N), p);
  long double worst = 0;
  for (long idx = 0; idx < N; idx++) {
    const long w = ((want[idx] % p) + p) % p;
    if (out[idx] != w) { std::printf("BGV D=%ld d=%ld %s bad=%d: coefficient %ld decrypts to %ld, want %ld\n", D, d, tag, (int)bad, idx, out[idx], w); return 1; }
    worst = std::max(worst, std::fabs(limbs_to_ld(&limbs[(size_t)idx * L], L)));
  }
  const double lnw = std::log((double)worst), lnb = got.noiseBound.ln();
  if (lnw > lnb) { std::printf("BGV D=%ld d=%ld %s bad=%d: measured noise e^%.2f exceeds the tracked bound e^%.2f\n", D, d, tag, (int)bad, lnw, lnb); return 1; }
  std::printf("BGV D=%ld d=%ld strategy %s %s%s: bits and metadata of the loop, decrypts, noise e^%.1f <= bound e^%.1f; %llu launches\n", D, d, tag,
              bad ? "bad dimension" : "native", direct_outer ? "" : " (non-direct outer amount: the loop)", lnw, lnb, (unsigned long long)(l1 - l0));
  return 0;
}

static int ckks_refused() {
  Context ctx(2048, /*p=*/-1, /*r=*/20, /*bits=*/200, /*c=*/2);
  KeyInfo pk; pk.context = &ctx; pk.ckks = true;
  Ctxt c(pk, 1);
  try { BlockMatMul1D(c, 5, 4, 4, std::vector<BsgsDiag>(16)); }
  catch (const LogicError&) { std::printf("CKKS: refused (LogicError)\n"); return 0; }
  std::printf("CKKS: BlockMatMul1D did not throw LogicError\n");
  return 1;
}

int main() {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  try {
    if (bgv_case(4, 4, false, true) != 0 || bgv_case(3, 4, false, true) != 0 || bgv_case(4, 4, true, true) != 0 ||
        bgv_case(3, 4, true, true) != 0 || bgv_case(3, 4, false, false) != 0 || ckks_refused() != 0) return 1;
    std::printf("block matmul OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
