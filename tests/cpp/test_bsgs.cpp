// BSGS linear maps through the C++ mirror: hb::MatMul1DBSGS, MatMul1DExec::mul's non-iterative baby-step/giant-step
// branches (src/matmul.cpp:989-1142) with the giant steps in one hb_bsgs_linear_map call.  Checks:
//  - the result equals a literal transcription of the loop (GenBabySteps, MulAdd, smartAutomorph, +=, one partition) bit for
//    bit, with equal metadata, in the native and the bad-dimension form, D = g^2 and D not a multiple of g, with a key set
//    made like add1Dmats4dim's BSGS branch;
//  - BGV: it decrypts to sum_i c_i(X) * m(X^{gen^i}) (+ c1_i(X) * m(X^{gen^(i-D)}));
//  - a giant amount without a direct matrix takes the loop and still matches;
//  - CKKS: it decodes within its tracked noise bound.
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


// Sum_i c_i(X) * m(X^{gen^i}) (+ c1_i(X) * m(X^{gen^(i-D)})) at coefficient idx, mod p, where c_i is cache[i] rotated by
// giant step k = i / g's amount gen^(g k): the giant step's smartAutomorph rotates the diagonals with the baby steps, which is
// why MatMul1DExec's cache holds them pre-rotated
static long want_at(const std::vector<std::vector<long>>& c, const std::vector<std::vector<long>>& c1, const std::vector<long>& msg,
                    long gen, long D, long g, long m, long idx, long p) {
  const long N = (long)msg.size();
  long want = 0;
  for (long i = 0; i < D; i++) {
    const long kg = genToPow(gen, g * (i / g), m);
    if (!c[i].empty()) want = (want + negacyclic_at(rotate(c[i], kg, N), rotate(msg, genToPow(gen, i, m), N), idx, N)) % p;
    if (!c1.empty() && !c1[i].empty()) want = (want + negacyclic_at(rotate(c1[i], kg, N), rotate(msg, genToPow(gen, i - D, m), N), idx, N)) % p;
  }
  return (want % p + p) % p;
}

static int bgv_case(long D, bool bad, bool all_giant_keys) {
  const long m = 2048, p = 257, gen = 3;
  Context ctx(m, p, 1, /*bits=*/200, /*c=*/2);
  const long N = ctx.getPhiM();
  std::mt19937_64 gen64(20261015 + D);
  const double sigma = 3.2;
  const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
  Keys K{KeyInfo(), DoubleCRT(sample_ternary(gen64, N), ctx, allq), {}};
  long g = 1; while (g * g < D) g++;
  const long h = (D + g - 1) / g;
  // add1Dmats4dim's BSGS key set (src/keySwitching.cpp:546-559): baby steps gen^j, giant steps gen^(g k), gen^-D
  std::vector<long> rots;
  for (long j = 1; j < g; j++) rots.push_back(genToPow(gen, j, m));
  for (long k = 1; k < h; k++) if (all_giant_keys || k == 1) rots.push_back(genToPow(gen, g * k, m));
  if (bad) rots.push_back(genToPow(gen, -D, m));
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
  std::vector<std::vector<long>> cf(D), cf1(bad ? D : 0);
  std::vector<DoubleCRT> store;
  store.reserve(2 * D);
  std::vector<BsgsDiag> cache(D), cache1(bad ? D : 0);
  auto diag = [&](std::vector<long>& co, BsgsDiag& d, long i) {
    d = BsgsDiag{nullptr, i % 3 ? -1.0 : 30.0, XD(), XD(), 0.0};
    if (i % 5 == 4) return;   // a zero diagonal
    co.assign(N, 0);
    for (long s = 0; s < 6; s++) co[(size_t)(gen64() % N)] = (long)(gen64() % 5) - 2;
    store.emplace_back(co, ctx, allq);
    d.c = &store.back();
  };
  for (long i = 0; i < D; i++) { diag(cf[i], cache[i], i); if (bad) diag(cf1[i], cache1[i], i + 1); }
  // the literal loop of src/matmul.cpp:1022-1057 / 1097-1142 (one partition), for the bits and the metadata
  Ctxt loop(c);
  {
    std::vector<std::shared_ptr<Ctxt>> bs = GenBabySteps(c, gen, g, !bad), bs1;
    if (bad) { Ctxt cc(c); cc.smartAutomorph(genToPow(gen, -D, m)); bs1 = GenBabySteps(cc, gen, g, false); }
    auto mulAdd = [&](Ctxt& acc, const BsgsDiag& d, const Ctxt& b) { if (!d.c) return; Ctxt tmp(b); tmp.multByConstant(*d.c, d.size); acc += tmp; };
    Ctxt acc(K.pk, p);
    for (long k = 0; k < h; k++) {
      Ctxt inner(K.pk, p);
      for (long j = 0; j < g; j++) {
        const long i = j + g * k;
        if (i >= D) break;
        mulAdd(inner, cache[i], *bs[j]);
        if (bad) mulAdd(inner, cache1[i], *bs1[j]);
      }
      if (k > 0) inner.smartAutomorph(genToPow(gen, g * k, m));
      acc += inner;
    }
    loop = acc;
  }
  Ctxt got(c);
  const uint64_t l0 = [&] { uint64_t s[3]; check(hb_ctx_stats(ctx.handle(), s)); return s[1]; }();
  MatMul1DBSGS(got, gen, D, cache, cache1);
  const uint64_t l1 = [&] { uint64_t s[3]; check(hb_ctx_stats(ctx.handle(), s)); return s[1]; }();
  if (const char* what = differs(got, loop)) { std::printf("BGV D=%ld bad=%d: MatMul1DBSGS differs from the loop in its %s\n", D, (int)bad, what); return 1; }
  std::vector<long> out;
  hb::Decrypt(out, got, K.sKeys);
  for (long s = 0; s < 24; s++) {
    const long idx = (s * 173 + 11) % N;
    const long want = want_at(cf, cf1, msg, gen, D, g, m, idx, p);
    if (out[idx] != want) { std::printf("BGV D=%ld bad=%d: coefficient %ld decrypts to %ld, want %ld\n", D, (int)bad, idx, out[idx], want); return 1; }
  }
  std::printf("BGV D=%ld g=%ld h=%ld %s%s: bits and metadata of the loop, decrypts; %llu launches\n", D, g, h, bad ? "bad dimension" : "native",
              all_giant_keys ? "" : " (non-direct giant amounts: the loop)", (unsigned long long)(l1 - l0));
  return 0;
}

static int ckks_case() {
  const long m = 2048, gen = 5, D = 9;
  Context ctx(m, /*p=*/-1, /*r=*/20, /*bits=*/200, /*c=*/2);
  const long N = ctx.getPhiM();
  std::mt19937_64 gen64(7);
  const double sigma = 3.2;
  const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
  Keys K{KeyInfo(), DoubleCRT(sample_ternary(gen64, N), ctx, allq), {}};
  const long g = 3, h = 3;
  std::vector<long> rots;
  for (long j = 1; j < g; j++) rots.push_back(genToPow(gen, j, m));
  for (long k = 1; k < h; k++) rots.push_back(genToPow(gen, g * k, m));
  make_keys(K, ctx, rots, 1, true, gen64);
  const double Delta = std::ldexp(1.0, 30);
  std::vector<long> msg(N);
  for (auto& x : msg) x = (long)(gen64() % 7) - 3;
  Ctxt c(K.pk, 1);
  c.primeSet = ctx.getCtxtPrimes();
  {
    std::vector<long> e = sample_gauss(gen64, N, sigma), pt(N);
    for (long k = 0; k < N; k++) pt[k] = (long)(Delta * msg[k]) + e[k];
    DoubleCRT c1 = random_rows(ctx, c.primeSet, gen64);
    DoubleCRT c0(pt, ctx, c.primeSet);
    DoubleCRT t(c1); t.Mul(K.S, false); c0 -= t;
    c.parts.emplace_back(c0, SKHandle());
    c.parts.emplace_back(c1, SKHandle(1, 1, 0));
    c.noiseBound = XD(K.pk.noiseBoundForGaussian(sigma, N));
    c.ratFactor = XD(Delta);
    c.ptxtMag = XD(embeddingLargestCoeff(msg, m));
  }
  const double dc = std::ldexp(1.0, 20);
  std::vector<std::vector<long>> cf(D);
  std::vector<DoubleCRT> store;
  store.reserve(D);
  std::vector<BsgsDiag> cache(D);
  for (long i = 0; i < D; i++) {
    std::vector<long> cs(N, 0);
    cf[i].assign(N, 0); cf[i][i] = 2; cf[i][(i * 7 + 3) % N] = -1;
    for (long k = 0; k < N; k++) cs[k] = (long)(dc * cf[i][k]);
    store.emplace_back(cs, ctx, allq);
    cache[i] = BsgsDiag{&store.back(), 0.0, XD(embeddingLargestCoeff(cf[i], m)), XD(dc), 0.0};
  }
  Ctxt got(c);
  MatMul1DBSGS(got, gen, D, cache);
  std::vector<long> dummy; std::vector<uint64_t> limbs; int L = 0;
  hb::Decrypt(dummy, got, K.sKeys, &limbs, &L);
  const long double rf = std::ldexp((long double)got.ratFactor.m, (int)got.ratFactor.e);
  const double tol = std::exp2(got.noiseBound.ln() / std::log(2.0) - (std::log2((double)got.ratFactor.m) + (double)got.ratFactor.e));
  double worst = 0;
  for (long s = 0; s < 24; s++) {
    const long idx = (s * 173 + 11) % N;
    long want = 0;
    for (long i = 0; i < D; i++) want += negacyclic_at(rotate(cf[i], genToPow(gen, g * (i / g), m), N), rotate(msg, genToPow(gen, i, m), N), idx, N);
    worst = std::max(worst, std::fabs((double)(limbs_to_ld(&limbs[(size_t)idx * L], L) / rf) - (double)want));
  }
  if (worst > tol) { std::printf("CKKS: error %.3g exceeds the tracked bound %.3g\n", worst, tol); return 1; }
  std::printf("CKKS D=%ld: error %.3g <= bound %.3g\n", D, worst, tol);
  return 0;
}

int main() {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  try {
    if (bgv_case(9, false, true) != 0 || bgv_case(10, false, true) != 0 || bgv_case(9, true, true) != 0 ||
        bgv_case(10, true, true) != 0 || bgv_case(9, false, false) != 0 || ckks_case() != 0) return 1;
    std::printf("bsgs OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
