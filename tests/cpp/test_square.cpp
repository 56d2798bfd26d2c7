// Squaring through the C++ mirror: Ctxt::square / power / cube / multiplyBy2 (src/Ctxt.cpp:1681-1828, src/polyEval.cpp:18-29,
// 392-413) with multLowLvl's squaring branch as one hb_square_tensor_norm call.  Checks, for BGV p = 257 on a power-of-two
// ring (the fused k1_fwd_blk_square pass), BGV p = 2 on a general-m ring and CKKS:
//  - square(), power(e) for e in {1, 2, 3, 4, 5, 8}, cube() and each ordering branch of multiplyBy2 equal a literal
//    transcription of HElib's code bit for bit, with equal primeSet, noiseBound, intFactor, ratFactor, ptxtMag and
//    mod-switch statistic;
//  - each result decrypts to the plaintext power (BGV) or decodes to it within its tracked bound (CKKS);
//  - x.multiplyBy(x) equals x.multiplyBy(copy of x);
//  - the cases the call cannot reproduce (a 3-part input, a natural set that needs a mod-up, an empty ciphertext) take
//    the transcribed branch with the same results.
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
static long bits_of(long m, long p) { return p < 0 ? 300 : (m & (m - 1)) == 0 ? 360 : 200; }

// ---- the transcribed HElib code, with the squaring branch spelled out step by step
static void ref_multLowLvl(Ctxt& x, const Ctxt& o) {   // src/Ctxt.cpp:1681-1752
  if (&x != &o || x.isEmpty()) { x.multLowLvl(o); return; }   // real multiplication: unchanged code
  x.bringToSet(x.naturalPrimeSet());
  Ctxt tmp(x.pubKey, x.ptxtSpace);
  tmp.tensorProduct(x, x);
  x = tmp;
}
static void ref_multiplyBy(Ctxt& x, const Ctxt& o) {   // src/Ctxt.cpp:1757-1774
  if (x.isEmpty()) return;
  if (o.isEmpty()) { x = o; return; }
  ref_multLowLvl(x, o);
  x.reLinearize();
}
static void ref_multiplyBy2(Ctxt& x, const Ctxt& other1, const Ctxt& other2) {   // src/Ctxt.cpp:1776-1828
  if (x.isEmpty()) return;
  if (other1.isEmpty()) { x = other1; return; }
  if (other2.isEmpty()) { x = other2; return; }
  const double cap = x.capacity(), cap1 = other1.capacity(), cap2 = other2.capacity();
  if (cap < cap1 && cap < cap2) {
    Ctxt tmp = other1;
    if (&other1 == &other2) ref_multLowLvl(tmp, tmp);
    else ref_multLowLvl(tmp, other2);
    ref_multLowLvl(x, tmp);
    x.reLinearize();
    return;
  }
  const Ctxt *first, *second;
  if (cap < cap2 || cap1 < cap2) { first = &other2; second = &other1; }
  else { first = &other1; second = &other2; }
  if (&x == second) { Ctxt tmp = *second; ref_multLowLvl(x, *first); ref_multLowLvl(x, tmp); }
  else { ref_multLowLvl(x, *first); ref_multLowLvl(x, *second); }
  x.reLinearize();
}
static void ref_power(Ctxt& x, long e) {   // src/polyEval.cpp:392-413 and DynamicCtxtPowers::getPower (:18-29)
  if (e < 1) throw InvalidArgument("Cannot raise a ctxt to a non positive exponent");
  if (e == 1) return;
  if ((e & (e - 1)) == 0) { for (long k = e; k > 1; k >>= 1) ref_multiplyBy(x, x); return; }
  std::vector<Ctxt> v((size_t)e, Ctxt(x.pubKey, x.ptxtSpace));
  v[0] = x;
  std::function<Ctxt&(long)> get = [&](long k) -> Ctxt& {
    if (v[(size_t)k - 1].isEmpty()) {
      long h = 1;
      while (2 * h < k) h *= 2;
      v[(size_t)k - 1] = get(k - h);
      v[(size_t)k - 1].multiplyBy(get(h));   // two distinct stored powers: a real multiply
    }
    return v[(size_t)k - 1];
  };
  x = get(e);
}

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
  if (x.lastModSwitchRatio != y.lastModSwitchRatio) return "mod-switch statistic";
  return nullptr;
}
// did one squaring call run?  k1_fwd_blk_square on the register kernels, the in-place k1_tensor / k_pw_tensor otherwise
// (the transcribed branch multiplies part by part)
struct Launches {
  const Context& ctx;
  explicit Launches(const Context& c) : ctx(c) { check(hb_ctx_profile(ctx.handle(), 1)); }
  std::string stop() {
    std::string ran;
    char name[64]; uint64_t launches = 0, bytes = 0; double ms = 0;
    for (int i = 0; hb_ctx_profile_get(ctx.handle(), i, name, sizeof name, &launches, &ms, &bytes) == 0; i++) { ran += name; ran += ' '; }
    check(hb_ctx_profile(ctx.handle(), 0));
    return ran;
  }
};
static bool square_call(const std::string& ran) {
  return ran.find("k1_fwd_blk_square") != std::string::npos || ran.find("k1_tensor ") != std::string::npos || ran.find("k_pw_tensor") != std::string::npos;
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
      : ctx(m, p_, r, /*bits=*/bits_of(m, p_), /*c=*/2), pk(key_info(ctx, p_ < 0)), S(ctx, ctx.getCtxtPrimes() | ctx.getSpecialPrimes()), pubEncrKey(pk, p_ < 0 ? 1 : p_), p(p_), gen(rng_seed) {
    const long N = ctx.getPhiM();
    const bool ckks = p < 0;
    const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
    S = DoubleCRT(sample_ternary(gen, N), ctx, allq);
    std::vector<uint8_t> seed(32);
    for (auto& b : seed) b = (uint8_t)(gen() & 0xff);
    seed[31] |= 1;
    DoubleCRT s2(S); s2 *= S;   // s^2 -> s and s^3 -> s (cube), their a_i kept as their PRG seed
    DoubleCRT s3(s2); s3 *= S;
    for (long e : {2L, 3L}) {
    DoubleCRT se(e == 2 ? s2 : s3);
    seed[0] ^= (uint8_t)e;
    if ((m & (m - 1)) == 0) {
      pk.keySwitching.push_back(genKeySWmatrix(ctx, se, SKHandle(e, 1, 0), 0, S, ckks ? 1 : p, ckks, 3.2, gen, seed));
    } else {   // general m (the mirror's bounded samplers are for power-of-two m): GenKeySWmatrix with plain Gaussian errors
      KeySwitch W; W.fromKey = SKHandle(e, 1, 0); W.toKeyID = 0; W.ptxtSpace = p;
      DoubleCRT& s2 = se;
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
    for (auto& x : v) x = p > 0 ? (long)(gen() % p) : (long)(gen() % 3) - 1;
    return v;
  }
};

// x^e mod (Phi_m, p) or, for CKKS, over the integers
static std::vector<long> ptxt_power(const std::vector<long>& mu, long e, const std::vector<long>& phi, long p) {
  std::vector<long> r = mu;
  for (long k = 1; k < e; k++) {
    r = mul_mod_phi(r, mu, phi);
    if (p > 0) for (auto& c : r) c = ((c % p) + p) % p;
  }
  return r;
}
static int check_decrypt(Setup& T, const Ctxt& got, const std::vector<long>& want, const char* what) {
  const long p = T.p, N = T.ctx.getPhiM();
  std::vector<long> out; std::vector<uint64_t> limbs; int L = 0;
  Decrypt(out, got, T.sKeys, p < 0 ? &limbs : nullptr, &L);
  double worst = 0, tol = 0;
  if (p < 0) {
    tol = std::exp2(got.noiseBound.ln() / std::log(2.0) - (std::log2((double)got.ratFactor.m) + (double)got.ratFactor.e));
    if (tol > 0.5) { std::printf("%s: tracked bound %.3g is useless\n", what, tol); return 1; }
  }
  const long double rf = std::ldexp((long double)got.ratFactor.m, (int)got.ratFactor.e);
  for (long s = 0; s < 32; s++) {
    const long idx = (s * 173 + 11) % N;
    if (p > 0) {
      const long w = ((want[idx] % p) + p) % p;
      if (out[idx] != w) { std::printf("%s: coefficient %ld decrypts to %ld, want %ld\n", what, idx, out[idx], w); return 1; }
    } else {
      worst = std::max(worst, std::fabs((double)(limbs_to_ld(&limbs[(size_t)idx * L], L) / rf) - (double)want[idx]));
    }
  }
  if (p < 0 && worst > tol) { std::printf("%s: error %.3g exceeds the tracked bound %.3g\n", what, worst, tol); return 1; }
  return 0;
}

static int ring_case(long m, long p) {
  Setup T(m, p, p < 0 ? 20 : 1, 20261017 + m + (p < 0 ? 7 : p));
  const std::vector<long> phi = cyclotomic(m);
  const char* ring = p < 0 ? "CKKS" : p == 2 ? "BGV p=2" : "BGV p=257";
  const std::vector<long> mu = T.message();
  const Ctxt x = T.encrypt(mu);
  char what[128];
  // square(): one call, the transcription's bits and metadata, the plaintext square.  The input is one whose natural set
  // needs no mod-up (a fresh natural set often takes small primes): x or x times an encryption of 1 (over S | special
  // after its reLinearize, so that special primes are dropped with ctxt primes), with its bound raised 4^k-fold
  // (bumpNoiseBound) for the first k that gives one; on the BGV power-of-two ring one that drops primes.
  {
    std::vector<long> one(T.ctx.getPhiM(), 0); one[0] = 1;
    Ctxt xo = x; xo.multiplyBy(T.encrypt(one));
    Ctxt in = x;
    bool found = false;
    for (int k = 0; k < 24 && !found; k++)
      for (const Ctxt* c : {(const Ctxt*)&xo, &x}) {
        in = *c;
        in.noiseBound = in.noiseBound * XD(std::ldexp(1.0, 2 * k));
        const IndexSet nat = in.naturalPrimeSet();
        if (nat <= in.primeSet && (p != 257 || !(nat == in.primeSet))) { found = true; break; }
      }
    if (!found) { std::printf("%s: no square input without a mod-up\n", ring); return 1; }
    Ctxt got = in, ref = in;
    Launches L(T.ctx);
    got.square();
    const std::string ran = L.stop();
    ref_multiplyBy(ref, ref);
    std::snprintf(what, sizeof what, "%s square", ring);
    if (const char* d = differs(got, ref)) { std::printf("%s differs from the transcription in its %s\n", what, d); return 1; }
    if (!square_call(ran)) { std::printf("%s: the squaring call did not run (%s)\n", what, ran.c_str()); return 1; }
    if (p == 257 && ran.find("k1_fwd_blk_square") == std::string::npos) {
      std::printf("%s: k1_fwd_blk_square did not run (%s)\n", what, ran.c_str()); return 1;
    }
    if (check_decrypt(T, got, ptxt_power(mu, 2, phi, p), what)) return 1;
    Ctxt self = x, copy = x;   // x.multiplyBy(x) == x.multiplyBy(copy of x)
    self.multiplyBy(self);
    Ctxt other = x;
    copy.multiplyBy(other);
    if (const char* d = differs(self, copy)) { std::printf("%s: x.multiplyBy(x) differs from x.multiplyBy(copy) in its %s\n", ring, d); return 1; }
    std::printf("%s: square() is one call with the transcription's bits and metadata (%ld -> %ld primes), decrypts to x^2\n", ring,
                (long)in.primeSet.card(), (long)got.primeSet.card());
  }
  // power(e)
  for (long e : {1L, 2L, 3L, 4L, 5L, 8L}) {
    Ctxt got = x, ref = x;
    got.power(e);
    ref_power(ref, e);
    std::snprintf(what, sizeof what, "%s power(%ld)", ring, e);
    if (const char* d = differs(got, ref)) { std::printf("%s differs from the transcription in its %s\n", what, d); return 1; }
    if (p > 0 || e <= 3) { if (check_decrypt(T, got, ptxt_power(mu, e, phi, p), what)) return 1; }
  }
  std::printf("%s: power(1, 2, 3, 4, 5, 8) match the transcription%s\n", ring, p > 0 ? " and decrypt to the powers" : ", e <= 3 decode within the bound");
  // cube() and the orderings of multiplyBy2: y, z fresh; lo one prime lower (a lower capacity)
  const std::vector<long> nu = T.message(), rho = T.message();
  const Ctxt y = T.encrypt(nu), z = T.encrypt(rho);
  Ctxt lo = T.encrypt(mu);
  { IndexSet s = lo.primeSet; s.remove(s.last()); lo.modDownToSet(s); }
  struct Case { const char* name; int kind; };
  const Case cases[] = {{"cube", 0}, {"this lowest", 1}, {"this lowest, other1 == other2", 2}, {"other2 first", 3},
                        {"other1 first", 4}, {"pointer collision", 5}};
  for (const Case& c : cases) {
    Ctxt got = c.kind == 1 || c.kind == 2 ? lo : x, ref = got;
    std::vector<long> want;
    switch (c.kind) {
      case 0: got.cube(); ref_multiplyBy2(ref, ref, ref); want = ptxt_power(mu, 3, phi, p); break;
      case 1: got.multiplyBy2(y, z); ref_multiplyBy2(ref, y, z); want = mul_mod_phi(mul_mod_phi(mu, nu, phi), rho, phi); break;
      case 2: got.multiplyBy2(y, y); ref_multiplyBy2(ref, y, y); want = mul_mod_phi(mul_mod_phi(mu, nu, phi), nu, phi); break;
      case 3: got.multiplyBy2(lo, got); ref_multiplyBy2(ref, lo, ref); want = mul_mod_phi(mul_mod_phi(mu, mu, phi), mu, phi); break;
      case 4: got.multiplyBy2(y, lo); ref_multiplyBy2(ref, y, lo); want = mul_mod_phi(mul_mod_phi(mu, nu, phi), mu, phi); break;
      default: got.multiplyBy2(y, got); ref_multiplyBy2(ref, y, ref); want = mul_mod_phi(mul_mod_phi(mu, nu, phi), mu, phi); break;
    }
    std::snprintf(what, sizeof what, "%s multiplyBy2 (%s)", ring, c.name);
    if (const char* d = differs(got, ref)) { std::printf("%s differs from the transcription in its %s\n", what, d); return 1; }
    // CKKS: lo's mod-down of a fresh ciphertext leaves a scale below one prime, so only the cube is decoded
    if ((p > 0 || c.kind == 0) && check_decrypt(T, got, want, what)) return 1;
  }
  std::printf("%s: cube() and the multiplyBy2 orderings match the transcription, %s\n", ring,
              p > 0 ? "and decrypt to the products" : "the cube decodes within the bound");
  return 0;
}

// the cases one call cannot reproduce: the transcribed branch, the same results
static int fallback_cases() {
  Setup T(8192, 257, 1, 77);
  const Ctxt x = T.encrypt(T.message()), y = T.encrypt(T.message());
  {   // a 3-part input (an unrelinearised product), squared by multLowLvl
    Ctxt got = x; got.multLowLvl(y);
    Ctxt ref = got;
    Launches L(T.ctx);
    got.multLowLvl(got);
    const std::string ran = L.stop();
    ref_multLowLvl(ref, ref);
    if (const char* d = differs(got, ref)) { std::printf("3-part input: differs from the transcription in its %s\n", d); return 1; }
    if (square_call(ran)) { std::printf("3-part input: the squaring call ran\n"); return 1; }
  }
  {   // a natural set above the current one (a tracked noise far below the level): bringToSet mods up
    Ctxt got = x;
    IndexSet s = got.primeSet; s.remove(s.last()); s.remove(s.last()); got.modDownToSet(s);
    got.noiseBound = XD(1.0);
    const IndexSet nat = got.naturalPrimeSet();
    if (nat <= got.primeSet) { std::printf("mod-up case: the natural set needs no mod-up\n"); return 1; }
    Ctxt ref = got;
    Launches L(T.ctx);
    got.square();
    const std::string ran = L.stop();
    ref_multiplyBy(ref, ref);
    if (const char* d = differs(got, ref)) { std::printf("mod-up case: differs from the transcription in its %s\n", d); return 1; }
    if (square_call(ran)) { std::printf("mod-up case: the squaring call ran\n"); return 1; }
  }
  {   // an empty ciphertext: square() and power(2^k) do nothing, power(3) throws as DynamicCtxtPowers does
    Ctxt got(T.pk, 257), ref(T.pk, 257);
    got.square(); got.power(4); ref_power(ref, 4);
    if (const char* d = differs(got, ref)) { std::printf("empty: differs in its %s\n", d); return 1; }
    bool threw = false;
    try { got.power(3); } catch (const InvalidArgument&) { threw = true; }
    if (!threw) { std::printf("empty: power(3) did not throw\n"); return 1; }
    threw = false;
    try { Ctxt t = x; t.power(0); } catch (const InvalidArgument&) { threw = true; }
    if (!threw) { std::printf("power(0) did not throw\n"); return 1; }
  }
  std::printf("fallbacks: 3-part input, mod-up and empty ciphertexts take the transcribed branch\n");
  return 0;
}

int main() {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  try {
    if (ring_case(8192, 257) != 0) return 1;
    if (ring_case(105, 2) != 0) return 1;
    if (ring_case(8192, -1) != 0) return 1;
    if (fallback_cases() != 0) return 1;
    std::printf("square OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
