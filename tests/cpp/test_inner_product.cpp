// innerProduct through the C++ mirror: hb::innerProduct (src/Ctxt.cpp:2878-2893) with the pairs' summed tensor products in one
// hb_tensor_sum call.  Checks, for BGV (p = 257, p = 2) and CKKS with n = 1, 2, 5, 17 pairs:
//  - the result equals a literal transcription of the loop (multLowLvl, +=, reLinearize) bit for bit, with equal metadata;
//  - BGV: it decrypts to sum_i mu_i * nu_i; CKKS: it decodes to that sum within its tracked noise bound;
//  - the fused call ran (k1_tensor_sum in the launch profile).
// And the cases that take the loop and must still match it: pairs at different levels, different intFactors, a 3-part
// operand, empty and unequal-length vectors.
// Exit codes: 0 ok, 3 no CUDA device, 1 failure.
#include <cstdio>
#include <cstring>
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
// Phi_m(X) = (X^m - 1) / prod_{d | m, d < m} Phi_d(X), low coefficient first (monic, degree phi(m))
static std::vector<long> cyclotomic(long m) {
  std::vector<long> a(m + 1, 0); a[0] = -1; a[m] = 1;
  for (long d = 1; d < m; d++) {
    if (m % d) continue;
    const std::vector<long> b = cyclotomic(d);
    const long db = (long)b.size() - 1;
    std::vector<long> q(a.size() - db, 0);
    for (long k = (long)a.size() - 1; k >= db; k--) { const long c = a[k]; q[k - db] = c; for (long j = 0; j <= db; j++) a[k - db + j] -= c * b[j]; }
    a = q;
  }
  return a;
}
// a*b mod Phi_m(X)
static std::vector<long> mul_mod_phi(const std::vector<long>& a, const std::vector<long>& b, const std::vector<long>& phi) {
  const long N = (long)phi.size() - 1;
  std::vector<long> r(2 * N, 0);
  for (long i = 0; i < N; i++) if (a[i]) for (long j = 0; j < N; j++) r[i + j] += a[i] * b[j];
  for (long k = 2 * N - 1; k >= N; k--) { const long c = r[k]; if (c) for (long j = 0; j <= N; j++) r[k - N + j] -= c * phi[j]; }
  r.resize(N);
  return r;
}
// the literal loop of src/Ctxt.cpp:2878-2893
static void loop_reference(Ctxt& result, const std::vector<Ctxt>& v1, const std::vector<Ctxt>& v2) {
  const size_t n = std::min(v1.size(), v2.size());
  if (n == 0) {
    result.parts.clear(); result.primeSet = result.context.getCtxtPrimes(); result.noiseBound = XD(0.0);
    result.intFactor = 1; result.ratFactor = XD(1.0); result.ptxtMag = XD(1.0);
    return;
  }
  result = v1[0];
  result.multLowLvl(v2[0]);
  for (size_t i = 1; i < n; i++) { Ctxt tmp = v1[i]; tmp.multLowLvl(v2[i]); result += tmp; }
  result.reLinearize();
}
// hb::innerProduct with the launch profile on: did the one tensor-sum call run (k1_tensor_sum, or for general m k_pw_tensor)?
static bool inner_product_fused(const Context& ctx, Ctxt& result, const std::vector<Ctxt>& v1, const std::vector<Ctxt>& v2) {
  check(hb_ctx_profile(ctx.handle(), 1));
  innerProduct(result, v1, v2);
  bool ran = false;
  char name[64]; uint64_t launches = 0, bytes = 0; double ms = 0;
  for (int i = 0; hb_ctx_profile_get(ctx.handle(), i, name, sizeof name, &launches, &ms, &bytes) == 0; i++) ran = ran || !std::strcmp(name, "k1_tensor_sum") || !std::strcmp(name, "k_pw_tensor");
  check(hb_ctx_profile(ctx.handle(), 0));
  return ran;
}

static KeyInfo key_info(const Context& ctx, bool ckks) {
  KeyInfo pk;
  pk.context = &ctx; pk.ckks = ckks; pk.scale = 10.0; pk.hwt = 0;
  pk.skBound = pk.scale * std::sqrt(double(ctx.getPhiM()) * 2.0 / 3.0);
  return pk;
}

struct Setup {
  Context ctx;
  KeyInfo pk;
  DoubleCRT S;
  std::vector<DoubleCRT> sKeys;
  Ctxt pubEncrKey;
  long p;
  std::mt19937_64 gen;
  Setup(long m, long p_, long r, uint64_t rng_seed)
      : ctx(m, p_, r, /*bits=*/200, /*c=*/2), pk(key_info(ctx, p_ < 0)), S(ctx, ctx.getCtxtPrimes() | ctx.getSpecialPrimes()), pubEncrKey(pk, p_ < 0 ? 1 : p_), p(p_), gen(rng_seed) {
    const long N = ctx.getPhiM();
    const bool ckks = p < 0;
    const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
    S = DoubleCRT(sample_ternary(gen, N), ctx, allq);
    std::vector<uint8_t> seed(32);
    for (auto& b : seed) b = (uint8_t)(gen() & 0xff);
    seed[31] |= 1;
    DoubleCRT s2(S); s2 *= S;   // s^2 -> s, its a_i kept as their PRG seed
    if ((m & (m - 1)) == 0) {
      pk.keySwitching.push_back(genKeySWmatrix(ctx, s2, SKHandle(2, 1, 0), 0, S, ckks ? 1 : p, ckks, 3.2, gen, seed));
    } else {   // general m (the mirror's bounded samplers are for power-of-two m): GenKeySWmatrix with plain Gaussian errors
      KeySwitch W; W.fromKey = SKHandle(2, 1, 0); W.toKeyID = 0; W.ptxtSpace = p;
      s2.multiplyByPrimes(ctx.getSpecialPrimes());
      for (size_t i = 0; i < ctx.getDigits().size(); i++) {
        W.a.push_back(random_rows(ctx, allq, gen));
        DoubleCRT b(sample_gauss(gen, N, 3.2), ctx, allq); b *= p;
        DoubleCRT t(W.a.back()); t *= S; b -= t;
        b += s2;
        W.b.push_back(b);
        s2.multiplyByPrimes(ctx.getDigit((long)i));
      }
      W.noiseBound = XD(double(p) * pk.noiseBoundForGaussian(3.2, N));
      pk.keySwitching.push_back(W);
    }
    pk.setKeySwitchMap(0);
    sKeys.push_back(S);
    if (ckks) return;
    pubEncrKey.primeSet = ctx.getCtxtPrimes();
    DoubleCRT c1 = random_rows(ctx, pubEncrKey.primeSet, gen);
    DoubleCRT c0(sample_gauss(gen, N, 3.2), ctx, pubEncrKey.primeSet); c0 *= p;
    DoubleCRT t(c1); t.Mul(S, false); c0 -= t;
    pubEncrKey.parts.emplace_back(c0, SKHandle());
    pubEncrKey.parts.emplace_back(c1, SKHandle(1, 1, 0));
    pubEncrKey.noiseBound = XD(double(p) * pk.noiseBoundForGaussian(3.2, N));
  }
  Ctxt encrypt(const std::vector<long>& msg) {
    const long N = ctx.getPhiM();
    if (p > 0 && (ctx.getM() & (ctx.getM() - 1)) != 0) {   // general m: symmetric encryption c0 = msg + p*e - c1*s
      Ctxt c(pk, p);
      c.primeSet = ctx.getCtxtPrimes();
      std::vector<long> e = sample_gauss(gen, N, 3.2), pt(N);
      for (long k = 0; k < N; k++) pt[k] = msg[k] + p * e[k];
      DoubleCRT c1 = random_rows(ctx, c.primeSet, gen);
      DoubleCRT c0(pt, ctx, c.primeSet);
      DoubleCRT t(c1); t.Mul(S, false); c0 -= t;
      c.parts.emplace_back(c0, SKHandle());
      c.parts.emplace_back(c1, SKHandle(1, 1, 0));
      c.noiseBound = XD(double(p) * pk.noiseBoundForGaussian(3.2, N));
      return c;
    }
    if (p > 0) {
      Ctxt c(pk, p);
      EncryptionSample smp = drawEncryptionSample(ctx, 3.2, gen);
      Encrypt(c, pubEncrKey, msg, p, smp);
      return c;
    }
    const double Delta = std::ldexp(1.0, 30);   // symmetric CKKS encryption of Delta*msg (SecKey::Encrypt, CKKS branch)
    Ctxt c(pk, 1);
    c.primeSet = ctx.getCtxtPrimes();
    std::vector<long> e = sample_gauss(gen, N, 3.2), pt(N);
    for (long k = 0; k < N; k++) pt[k] = (long)(Delta * msg[k]) + e[k];
    DoubleCRT c1 = random_rows(ctx, c.primeSet, gen);
    DoubleCRT c0(pt, ctx, c.primeSet);
    DoubleCRT t(c1); t.Mul(S, false); c0 -= t;
    c.parts.emplace_back(c0, SKHandle());
    c.parts.emplace_back(c1, SKHandle(1, 1, 0));
    c.noiseBound = XD(pk.noiseBoundForGaussian(3.2, N));
    c.ratFactor = XD(Delta);
    c.ptxtMag = XD(embeddingLargestCoeff(msg, ctx.getM()));
    return c;
  }
  std::vector<long> message() {
    std::vector<long> v(ctx.getPhiM());
    for (auto& x : v) x = p > 0 ? (long)(gen() % p) : (long)(gen() % 7) - 3;
    return v;
  }
};

static int sum_case(long p, long n) {
  const long m = p == 2 ? 105 : 2048;   // p = 2 needs an odd m: the general-m path
  Setup T(m, p, p < 0 ? 20 : 1, 20261016 + 31 * n + (p < 0 ? 7 : p));
  const std::vector<long> phi = cyclotomic(m);
  const long N = T.ctx.getPhiM();
  std::vector<std::vector<long>> mu, nu;
  std::vector<Ctxt> v1, v2;
  for (long i = 0; i < n; i++) {
    mu.push_back(T.message()); nu.push_back(T.message());
    v1.push_back(T.encrypt(mu.back())); v2.push_back(T.encrypt(nu.back()));
  }
  Ctxt loop(T.pk, T.pubEncrKey.ptxtSpace), got(T.pk, T.pubEncrKey.ptxtSpace);
  loop_reference(loop, v1, v2);
  const bool fused = inner_product_fused(T.ctx, got, v1, v2);
  if (const char* what = differs(got, loop)) { std::printf("p=%ld n=%ld: innerProduct differs from the loop in its %s\n", p, n, what); return 1; }
  if (!fused) { std::printf("p=%ld n=%ld: the fused call did not run\n", p, n); return 1; }
  std::vector<long> out; std::vector<uint64_t> limbs; int L = 0;
  Decrypt(out, got, T.sKeys, p < 0 ? &limbs : nullptr, &L);
  double worst = 0, tol = 0;
  if (p < 0) {
    tol = std::exp2(got.noiseBound.ln() / std::log(2.0) - (std::log2((double)got.ratFactor.m) + (double)got.ratFactor.e));
    if (tol > 0.5) { std::printf("CKKS n=%ld: tracked bound %.3g is useless\n", n, tol); return 1; }
  }
  const long double rf = std::ldexp((long double)got.ratFactor.m, (int)got.ratFactor.e);
  std::vector<long> sum(N, 0);
  for (long i = 0; i < n; i++) { const std::vector<long> t = mul_mod_phi(mu[i], nu[i], phi); for (long k = 0; k < N; k++) sum[k] += t[k]; }
  for (long s = 0; s < 24; s++) {
    const long idx = (s * 173 + 11) % N;
    long want = sum[idx];
    if (p > 0) {
      want = ((want % p) + p) % p;
      if (out[idx] != want) { std::printf("p=%ld n=%ld: coefficient %ld decrypts to %ld, want %ld\n", p, n, idx, out[idx], want); return 1; }
    } else {
      worst = std::max(worst, std::fabs((double)(limbs_to_ld(&limbs[(size_t)idx * L], L) / rf) - (double)want));
    }
  }
  if (p < 0 && worst > tol) { std::printf("CKKS n=%ld: error %.3g exceeds the tracked bound %.3g\n", n, worst, tol); return 1; }
  std::printf("%s n=%ld: bits and metadata of the loop, %s\n", p < 0 ? "CKKS" : p == 2 ? "BGV p=2" : "BGV p=257", n,
              p < 0 ? "decodes within the tracked bound" : "decrypts to the sum");
  return 0;
}

// the cases the fused call cannot reproduce, and the degenerate lengths: the loop's result either way
static int loop_cases() {
  Setup T(2048, 257, 1, 99);
  std::vector<Ctxt> v1, v2;
  for (int i = 0; i < 3; i++) { v1.push_back(T.encrypt(T.message())); v2.push_back(T.encrypt(T.message())); }
  auto run = [&](const char* what, const std::vector<Ctxt>& a, const std::vector<Ctxt>& b, int want_fused) {
    Ctxt loop(T.pk, 257), got(T.pk, 257);
    loop_reference(loop, a, b);
    const bool fused = inner_product_fused(T.ctx, got, a, b);
    if (const char* d = differs(got, loop)) { std::printf("%s: innerProduct differs from the loop in its %s\n", what, d); return 1; }
    if (want_fused >= 0 && fused != (want_fused != 0)) { std::printf("%s: the fused call %s\n", what, fused ? "ran" : "did not run"); return 1; }
    std::printf("%s: the loop's result (%s)\n", what, fused ? "one call" : "loop");
    return 0;
  };
  {   // pairs at different levels: pair 1 two primes lower
    std::vector<Ctxt> a = v1, b = v2;
    IndexSet low = T.ctx.getCtxtPrimes(); low.remove(low.last()); low.remove(low.last());
    a[1].modDownToSet(low); b[1].modDownToSet(low);
    if (run("different levels", a, b, -1)) return 1;
  }
  {   // a pair with another intFactor
    std::vector<Ctxt> a = v1;
    a[1].mulIntFactor(3);
    if (run("different intFactors", a, v2, 0)) return 1;
  }
  {   // a 3-part operand (an unrelinearised product) times a 1-part one (the constant part of a fresh ciphertext)
    std::vector<Ctxt> a = v1, b = v2;
    a[0].multLowLvl(v2[2]);
    Ctxt k(T.pk, 257);
    k.primeSet = v2[0].primeSet; k.noiseBound = v2[0].noiseBound;
    k.parts.push_back(v2[0].parts[0]);
    b[0] = k;
    if (run("3-part operand", a, b, 0)) return 1;
  }
  if (run("empty vectors", {}, {}, 0)) return 1;
  {
    std::vector<Ctxt> b(v2.begin(), v2.begin() + 2);
    if (run("unequal lengths", v1, b, 1)) return 1;
  }
  return 0;
}

int main() {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  try {
    for (long p : {257L, 2L, -1L})
      for (long n : {1L, 2L, 5L, 17L})
        if (sum_case(p, n) != 0) return 1;
    if (loop_cases() != 0) return 1;
    std::printf("inner product OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
