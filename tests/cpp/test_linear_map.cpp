// Hoisted linear maps through the C++ mirror: BasicAutomorphPrecon::linearCombination (BGV) and linearCombinationCKKS,
// the loop body of MatMul1DExec::mul's native FULL branch (src/matmul.cpp:1226-1252) in one hb_hoisted_linear_map call.
// Checks:
//  - the result equals the composed loop (automorph -> multByConstant -> +=) bit for bit in every part, with equal
//    metadata (primeSet, noiseBound, intFactor, ratFactor, ptxtMag, ptxtSpace);
//  - BGV: it decrypts to sum_j c_j(X) * m(X^k_j) mod (X^N + 1, p), also with an amount whose matrix is not direct (that
//    amount takes the composed path);
//  - CKKS: it decodes within its tracked noise bound.
// Exit codes: 0 ok, 3 no CUDA device, 1 failure.
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

static int bgv() {
  const long m = 8192, p = 257;
  Context ctx(m, p, 1, /*bits=*/300, /*c=*/2);
  const long N = ctx.getPhiM();
  std::mt19937_64 gen(20261015);
  const double sigma = 3.2;
  const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
  Keys K{KeyInfo(), DoubleCRT(sample_ternary(gen, N), ctx, allq), {}};
  make_keys(K, ctx, {3, 5, 9, m - 1}, p, false, gen);
  // a public encryption key, then an encryption of a random message
  Ctxt pubEncrKey(K.pk, p);
  pubEncrKey.primeSet = ctx.getCtxtPrimes();
  DoubleCRT c1 = random_rows(ctx, pubEncrKey.primeSet, gen);
  DoubleCRT c0(sample_gauss(gen, N, sigma), ctx, pubEncrKey.primeSet); c0 *= p;
  DoubleCRT t(c1); t.Mul(K.S, false); c0 -= t;
  pubEncrKey.parts.emplace_back(c0, SKHandle());
  pubEncrKey.parts.emplace_back(c1, SKHandle(1, 1, 0));
  pubEncrKey.noiseBound = XD(double(p) * K.pk.noiseBoundForGaussian(sigma, N));
  std::vector<long> msg(N);
  for (auto& x : msg) x = (long)(gen() % p);
  Ctxt c(K.pk, p);
  hb::EncryptionSample smp = hb::drawEncryptionSample(ctx, sigma, gen);
  hb::Encrypt(c, pubEncrKey, msg, p, smp);
  BasicAutomorphPrecon pre(c);
  // amounts: k = 1, direct ones (one repeated, m - 1), and 15 = 3 * 5, which has no direct matrix
  const std::vector<std::vector<long>> cases = {{1, 3, 5, 3, m - 1, 9}, {3, 15, 1, 5}};
  for (const auto& ks : cases) {
    std::vector<std::vector<long>> coefs;
    std::vector<DoubleCRT> consts;
    std::vector<const DoubleCRT*> cp;
    std::vector<double> sizes;
    for (size_t j = 0; j < ks.size(); j++) {
      std::vector<long> cj(N, 0);
      for (long i = 0; i < 8; i++) cj[(size_t)(gen() % N)] = (long)(gen() % 5) - 2;
      coefs.push_back(cj);
      consts.emplace_back(cj, ctx, allq);
      sizes.push_back(j % 2 ? -1.0 : 40.0);
    }
    for (auto& d : consts) cp.push_back(&d);
    Ctxt loop(K.pk, p);
    for (size_t j = 0; j < ks.size(); j++) { auto tmp = pre.automorph(ks[j]); tmp->multByConstant(consts[j], sizes[j]); loop += *tmp; }
    const uint64_t launches0 = [&] { uint64_t s[3]; check(hb_ctx_stats(ctx.handle(), s)); return s[1]; }();
    auto got = pre.linearCombination(ks, cp, sizes);
    const uint64_t launches1 = [&] { uint64_t s[3]; check(hb_ctx_stats(ctx.handle(), s)); return s[1]; }();
    if (const char* what = differs(*got, loop)) { std::printf("BGV: linearCombination differs from the loop in its %s\n", what); return 1; }
    std::vector<long> out;
    hb::Decrypt(out, *got, K.sKeys);
    for (long s = 0; s < 48; s++) {
      const long idx = (s * 173 + 11) % N;
      long want = 0;
      for (size_t j = 0; j < ks.size(); j++) want = (want + negacyclic_at(coefs[j], rotate(msg, ks[j], N), idx, N)) % p;
      want = (want % p + p) % p;
      if (out[idx] != want) { std::printf("BGV: coefficient %ld decrypts to %ld, want %ld\n", idx, out[idx], want); return 1; }
    }
    std::printf("BGV: %zu amounts, bits and metadata of the loop, decrypts; %llu launches\n", ks.size(), (unsigned long long)(launches1 - launches0));
  }
  return 0;
}

static int ckks() {
  const long m = 8192;
  Context ctx(m, /*p=*/-1, /*r=*/20, /*bits=*/300, /*c=*/2);
  const long N = ctx.getPhiM();
  std::mt19937_64 gen(7);
  const double sigma = 3.2;
  const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
  Keys K{KeyInfo(), DoubleCRT(sample_ternary(gen, N), ctx, allq), {}};
  make_keys(K, ctx, {3, 5, m - 1}, 1, true, gen);
  const double Delta = std::ldexp(1.0, 30);
  std::vector<long> msg(N);
  for (auto& x : msg) x = (long)(gen() % 7) - 3;
  Ctxt c(K.pk, 1);
  c.primeSet = ctx.getCtxtPrimes();
  {
    std::vector<long> e = sample_gauss(gen, N, sigma), pt(N);
    for (long k = 0; k < N; k++) pt[k] = (long)(Delta * msg[k]) + e[k];
    DoubleCRT c1 = random_rows(ctx, c.primeSet, gen);
    DoubleCRT c0(pt, ctx, c.primeSet);
    DoubleCRT t(c1); t.Mul(K.S, false); c0 -= t;
    c.parts.emplace_back(c0, SKHandle());
    c.parts.emplace_back(c1, SKHandle(1, 1, 0));
    c.noiseBound = XD(K.pk.noiseBoundForGaussian(sigma, N));
    c.ratFactor = XD(Delta);
    c.ptxtMag = XD(embeddingLargestCoeff(msg, m));
  }
  BasicAutomorphPrecon pre(c);
  const double dc = std::ldexp(1.0, 20);
  const std::vector<long> ks = {3, 5, m - 1, 3};
  std::vector<std::vector<long>> coefs;
  std::vector<DoubleCRT> consts;
  std::vector<const DoubleCRT*> cp;
  std::vector<XD> sizes, factors;
  std::vector<double> errs;
  for (size_t j = 0; j < ks.size(); j++) {
    std::vector<long> cj(N, 0), cs(N, 0);
    cj[j] = 2; cj[(j * 7 + 3) % N] = -1;
    for (long k = 0; k < N; k++) cs[k] = (long)(dc * cj[k]);
    coefs.push_back(cj);
    consts.emplace_back(cs, ctx, allq);
    sizes.push_back(XD(embeddingLargestCoeff(cj, m))); factors.push_back(XD(dc)); errs.push_back(0.0);
  }
  for (auto& d : consts) cp.push_back(&d);
  Ctxt loop(K.pk, 1);
  for (size_t j = 0; j < ks.size(); j++) { auto tmp = pre.automorph(ks[j]); tmp->multByConstantCKKS(consts[j], sizes[j], factors[j], errs[j]); loop += *tmp; }
  auto got = pre.linearCombinationCKKS(ks, cp, sizes, factors, errs);
  if (const char* what = differs(*got, loop)) { std::printf("CKKS: linearCombinationCKKS differs from the loop in its %s\n", what); return 1; }
  std::vector<long> dummy; std::vector<uint64_t> limbs; int L = 0;
  hb::Decrypt(dummy, *got, K.sKeys, &limbs, &L);
  const long double rf = std::ldexp((long double)got->ratFactor.m, (int)got->ratFactor.e);
  const double tol = std::exp2(got->noiseBound.ln() / std::log(2.0) - (std::log2((double)got->ratFactor.m) + (double)got->ratFactor.e));
  double worst = 0;
  for (long s = 0; s < 48; s++) {
    const long idx = (s * 173 + 11) % N;
    long want = 0;
    for (size_t j = 0; j < ks.size(); j++) want += negacyclic_at(coefs[j], rotate(msg, ks[j], N), idx, N);
    worst = std::max(worst, std::fabs((double)(limbs_to_ld(&limbs[(size_t)idx * L], L) / rf) - (double)want));
  }
  if (worst > tol) { std::printf("CKKS: error %.3g exceeds the tracked bound %.3g\n", worst, tol); return 1; }
  if (tol > 1.0) { std::printf("CKKS: tracked bound %.3g is useless for integer sums\n", tol); return 1; }
  std::printf("CKKS: %zu amounts, bits and metadata of the loop, error %.3g <= bound %.3g\n", ks.size(), worst, tol);
  return 0;
}

int main() {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  try {
    if (bgv() != 0 || ckks() != 0) return 1;
    std::printf("linear map OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
