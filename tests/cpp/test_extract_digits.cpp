// Digit extraction through the C++ mirror: hb::extractDigits, hb::extendExtractDigits and hb::extractDigitsThin
// (src/extractDigits.cpp, src/recryption.cpp:793-909), with each round's subtract-and-divide chain and the thin final
// combination formed in one hb_ctxt_scaled_sums call.  Checks:
//  - the fused forms equal the transcribed step-by-step loops (fused = false) bit for bit: every part's rows, primeSet,
//    ptxtSpace, intFactor, noiseBound, ratFactor, ptxtMag and the mod-switch statistic, for p = 2, p = 3 and p = 17 with
//    r = 2..4, and p = 257 (the run with "full" also requires digits that end at different prime sets);
//  - the fused forms make one k1_scaled_sums launch per chain more than the loops;
//  - decrypted, digit j holds the j-th balanced base-p digit of every slot (slots Z/p^r on m = 16, p = 17 and m = 32,
//    p = 257; constant plaintexts on the p = 2 and p = 3 rings), Chen and Han's digits hold it at their whole plaintext
//    space, and extractDigitsThin leaves -(the selected digits) plus the bottom ones times p^e', mod p^r;
//  - divideByP and multByP alone, decrypted, and divideByP's asserts;
//  - a chain over digits brought down to two lower prime sets: the fused replay's mod-up, bit for bit and decrypted;
//  - a non-canonical input takes the loop, with the same result and no k1_scaled_sums launch.
// With the argument "full", also r = 4 for p = 17, p = 3 on m = 1024, config 5's ring (m = 21845, p = 2) and config 3's (m = 2^17, p = 257).
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
  if (x.lastModSwitchRatio != y.lastModSwitchRatio) return "mod-switch statistic";
  return nullptr;
}
static long sums_launches(const Context& ctx) {   // k1_scaled_sums launches since hb_ctx_profile(1)
  char name[64]; uint64_t launches = 0, bytes = 0; double ms = 0; long n = 0;
  for (int i = 0; hb_ctx_profile_get(ctx.handle(), i, name, sizeof name, &launches, &ms, &bytes) == 0; i++)
    if (std::strcmp(name, "k1_scaled_sums") == 0) n += (long)launches;
  check(hb_ctx_profile(ctx.handle(), 0));
  return n;
}
static long ipow(long p, long e) { long r = 1; while (e-- > 0) r *= p; return r; }
static long md(long a, long q) { long r = a % q; return r < 0 ? r + q : r; }
static long mulm(long a, long b, long q) { return (long)((__int128)md(a, q) * md(b, q) % q); }
static long bal(long a, long p) { long r = md(a, p); return r > p / 2 ? r - p : r; }
// the balanced base-p digits of v mod p^n (digits in [0, 1] for p = 2), as the digit polynomials and squaring produce them
static std::vector<long> digits_of(long v, long p, long n) {
  std::vector<long> d;
  v = md(v, ipow(p, n));
  for (long j = 0; j < n; j++) { const long x = p == 2 ? md(v, 2) : bal(v, p); d.push_back(x); v = (v - x) / p; }
  return d;
}

static KeyInfo key_info(const Context& ctx) {
  KeyInfo pk;
  pk.context = &ctx; pk.ckks = false; pk.scale = 10.0; pk.hwt = 0;
  pk.skBound = pk.scale * std::sqrt(double(ctx.getPhiM()) * 2.0 / 3.0);
  return pk;
}
// keys and symmetric encryption at plaintext space P = p^r
struct Setup {
  Context ctx;
  KeyInfo pk;
  DoubleCRT S;
  long p, r, P;
  std::mt19937_64 gen;
  Setup(long m, long p_, long r_, long bits, uint64_t seed, long c = 2)
      : ctx(m, p_, r_, bits, c), pk(key_info(ctx)), S(ctx, ctx.getCtxtPrimes() | ctx.getSpecialPrimes()), p(p_), r(r_), P(ipow(p_, r_)), gen(seed) {
    const long N = ctx.getPhiM();
    const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
    S = DoubleCRT(sample_ternary(gen, N), ctx, allq);
    DoubleCRT se(S);
    for (long e : {2L, 3L}) {   // s^2 -> s, and s^3 -> s for cube()
      se *= S;
      DoubleCRT s2(se);
      KeySwitch W; W.fromKey = SKHandle(e, 1, 0); W.toKeyID = 0; W.ptxtSpace = P;
      s2.multiplyByPrimes(ctx.getSpecialPrimes());
      for (size_t i = 0; i < ctx.getDigits().size(); i++) {
        W.a.push_back(random_rows(ctx, allq, gen));
        DoubleCRT b(sample_gauss(gen, N, 3.2), ctx, allq); b *= P;
        DoubleCRT t(W.a.back()); t *= S; b -= t;
        b += s2;
        W.b.push_back(b);
        s2.multiplyByPrimes(ctx.getDigit((long)i));
      }
      W.noiseBound = XD(double(P) * pk.noiseBoundForGaussian(3.2, N));
      pk.keySwitching.push_back(W);
    }
    pk.setKeySwitchMap(0);
  }
  Ctxt encrypt(const std::vector<long>& msg) {
    const long N = ctx.getPhiM();
    Ctxt c(pk, P);
    c.primeSet = ctx.getCtxtPrimes();
    std::vector<long> e = sample_gauss(gen, N, 3.2), pt(N);
    for (long k = 0; k < N; k++) pt[k] = msg[k] + P * e[k];
    DoubleCRT c1 = random_rows(ctx, c.primeSet, gen);
    DoubleCRT c0(pt, ctx, c.primeSet);
    DoubleCRT t(c1); t.Mul(S, false); c0 -= t;
    c.parts.emplace_back(c0, SKHandle());
    c.parts.emplace_back(c1, SKHandle(1, 1, 0));
    c.noiseBound = XD(double(P) * pk.noiseBoundForGaussian(3.2, N));
    if (P > 2) {   // the rows hold msg itself: intFactor = Q^-1 mod P makes decryption's (intFactor*Q)^-1 one
      long q = 1;
      for (long i : c.primeSet) q = (long)((__int128)q * (ctx.ithPrime(i) % P) % P);
      c.intFactor = Ctxt::invMod(q, P);
    }
    return c;
  }
  std::vector<long> decrypt(const Ctxt& c) { std::vector<long> out; Decrypt(out, c, {S}); return out; }
};

// the slots of a power-of-two ring with p = 1 mod m: mu evaluated at the primitive m-th roots of unity mod p^n, each a
// root of X^(m/2) + 1 found mod p and lifted by Newton's iteration
struct Slots {
  long m, p, n, q;
  std::vector<long> roots;
  Slots(long m_, long p_, long n_) : m(m_), p(p_), n(n_), q(ipow(p_, n_)) {
    const long h = m / 2;
    auto powm = [&](long a, long e, long mod) { long r = 1 % mod; a = md(a, mod); for (; e; e >>= 1, a = mulm(a, a, mod)) if (e & 1) r = mulm(r, a, mod); return r; };
    long z = 0;
    for (long g = 2; g < p && !z; g++) if (powm(g, h, p) == p - 1) z = g;
    for (long k = 0; k < n; k++) {   // z <- z - (z^h + 1) / (h z^(h-1)) mod p^n
      const long f = md(powm(z, h, q) + 1, q), d = mulm(h, powm(z, h - 1, q), q);
      z = md(z - mulm(f, Ctxt::invMod(d, q), q), q);
    }
    for (long k = 1; k < m; k += 2) roots.push_back(powm(z, k, q));
  }
  std::vector<long> of(const std::vector<long>& mu, long mod) const {
    std::vector<long> s;
    for (long z : roots) { long v = 0; for (size_t t = mu.size(); t-- > 0;) v = md(mulm(v, z, mod) + mu[t], mod); s.push_back(v); }
    return s;
  }
};

// ---- cases

static bool g_different_sets = false;   // some case's digits ended at different prime sets
static bool g_lower_digits = false;     // a chain modded digits at lower prime sets up
static int compare(const std::vector<Ctxt>& got, const std::vector<Ctxt>& want, const char* what) {
  if (got.size() != want.size()) { std::printf("%s: %zu digits, want %zu\n", what, got.size(), want.size()); return 1; }
  for (size_t j = 0; j < got.size(); j++)
    if (const char* d = differs(got[j], want[j])) { std::printf("%s: digit %zu differs from the loop in its %s\n", what, j, d); return 1; }
  return 0;
}

// slot values (or a constant) of c, n digits: the basic and Chen-Han extractions against the loops and the digits of
// every slot; the thin extraction at (botHigh, r, e') with both methods
struct Ring {
  Setup& T;
  const Slots* slots;   // nullptr: constant plaintexts
  const char* name;
  std::vector<long> values(const Ctxt& c) {   // the slot values of c, or its constant coefficient
    std::vector<long> pt = T.decrypt(c);
    if (!slots) {
      for (size_t k = 1; k < pt.size(); k++) if (md(pt[k], c.ptxtSpace) != 0) return {};
      return {md(pt[0], c.ptxtSpace)};
    }
    return slots->of(pt, c.ptxtSpace);
  }
  Ctxt encryptValues(std::vector<long>& v, long R) {   // v: the slot values mod p^R (filled in)
    const long N = T.ctx.getPhiM(), Q = ipow(T.p, R);
    std::vector<long> mu(N, 0);
    if (!slots) { mu[0] = (long)(T.gen() % (uint64_t)Q); v = {mu[0]}; }
    else { for (auto& x : mu) x = (long)(T.gen() % (uint64_t)Q); v = slots->of(mu, Q); }
    return T.encrypt(mu);
  }
};

static int digits_case(Ring& R, long n, const char* tag) {
  Setup& T = R.T;
  std::vector<long> v;
  const Ctxt c = R.encryptValues(v, T.r);
  char what[160];
  std::snprintf(what, sizeof what, "%s extractDigits %s n=%ld", R.name, tag, n);
  std::vector<Ctxt> got, want;
  check(hb_ctx_profile(T.ctx.handle(), 1));
  extractDigits(got, c, n);
  const long lf = sums_launches(T.ctx);
  check(hb_ctx_profile(T.ctx.handle(), 1));
  extractDigits(want, c, n, false);
  const long ll = sums_launches(T.ctx);
  if (compare(got, want, what)) return 1;
  if (lf - ll != (long)got.size() - 1) { std::printf("%s: %ld k1_scaled_sums launches more than the loop, want %zu\n", what, lf - ll, got.size() - 1); return 1; }
  for (size_t j = 1; j < got.size(); j++) if (!(got[j].primeSet == got[0].primeSet)) g_different_sets = true;
  const long nd = (long)got.size();
  for (long j = 0; j < nd; j++) {   // digit j holds d_j mod p^(n-j): each later round lifts it by one digit
    const std::vector<long> s = R.values(got[(size_t)j]);
    if (s.size() != v.size()) { std::printf("%s: digit %ld is not a constant\n", what, j); return 1; }
    const long q = ipow(T.p, nd - j);
    for (size_t k = 0; k < v.size(); k++)
      if (md(s[k], q) != md(digits_of(v[k], T.p, T.r)[(size_t)j], q)) {
        std::printf("%s: digit %ld slot %zu holds %ld, want %ld mod %ld\n", what, j, k, s[k], digits_of(v[k], T.p, T.r)[(size_t)j], q);
        return 1;
      }
  }
  std::printf("%s: %ld digits match the loop bit for bit and decrypt to the base-%ld digits (%ld fused chains)\n", what, nd, T.p, lf - ll);
  return 0;
}

static int extend_case(Ring& R, long r, long e) {
  Setup& T = R.T;   // T.r = r + e
  std::vector<long> v;
  const Ctxt c = R.encryptValues(v, T.r);
  char what[160];
  std::snprintf(what, sizeof what, "%s extendExtractDigits r=%ld e=%ld", R.name, r, e);
  std::vector<Ctxt> got, want;
  check(hb_ctx_profile(T.ctx.handle(), 1));
  extendExtractDigits(got, c, r, e);
  const long lf = sums_launches(T.ctx);
  check(hb_ctx_profile(T.ctx.handle(), 1));
  extendExtractDigits(want, c, r, e, false);
  const long ll = sums_launches(T.ctx);
  if (compare(got, want, what)) return 1;
  if (lf - ll != r - 1) { std::printf("%s: %ld k1_scaled_sums launches more than the loop, want %ld\n", what, lf - ll, r - 1); return 1; }
  for (long j = 0; j < r; j++) {   // G(x) = (x mod p) mod p^(e+r-j): the digit at the whole plaintext space
    const std::vector<long> s = R.values(got[(size_t)j]);
    const long q = got[(size_t)j].ptxtSpace;
    if (q != ipow(T.p, e + r - j) || s.size() != v.size()) { std::printf("%s: digit %ld at plaintext space %ld\n", what, j, q); return 1; }
    for (size_t k = 0; k < v.size(); k++)
      if (s[k] != md(digits_of(v[k], T.p, T.r)[(size_t)j], q)) { std::printf("%s: digit %ld slot %zu holds %ld\n", what, j, k, s[k]); return 1; }
  }
  std::printf("%s: %ld digits match the loop bit for bit and decrypt to the digits mod p^(e+r-j)\n", what, r);
  return 0;
}

// extractDigitsThin's result by its formula (src/recryption.cpp:873-907) on exact digits: slots mod p^(botHigh+r)
static long thin_value(long v, long p, long botHigh, long r, long ePrime) {
  const std::vector<long> d = digits_of(v, p, botHigh + r);
  const long q = ipow(p, r);
  long u = 0;
  for (long j = botHigh + r - 1; j >= botHigh; --j) u = md(u * p + d[(size_t)j], q);
  if (p == 2 && botHigh > 0) u = md(u + d[(size_t)botHigh - 1], q);
  u = md(-u, q);
  if (r > ePrime) {
    long t = 0;
    for (long j = r - 1 - ePrime; j >= 0; --j) t = md(t * p + d[(size_t)j], q);
    u = md(u + mulm(t, ipow(p, ePrime), q), q);
  }
  return u;
}
static int thin_case(Ring& R, long botHigh, long r, long ePrime, long chenHan, bool semantic = true) {
  Setup& T = R.T;   // T.r = botHigh + r
  std::vector<long> v;
  const Ctxt c = R.encryptValues(v, T.r);
  char what[160];
  std::snprintf(what, sizeof what, "%s extractDigitsThin bot=%ld r=%ld e'=%ld %s", R.name, botHigh, r, ePrime, chenHan > 0 ? "chen-han" : chenHan < 0 ? "basic" : "by cost");
  Ctxt got = c, want = c;
  check(hb_ctx_profile(T.ctx.handle(), 1));
  extractDigitsThin(got, botHigh, r, ePrime, chenHan);
  const long lf = sums_launches(T.ctx);
  check(hb_ctx_profile(T.ctx.handle(), 1));
  extractDigitsThin(want, botHigh, r, ePrime, chenHan, false);
  const long ll = sums_launches(T.ctx);
  if (const char* d = differs(got, want)) { std::printf("%s: differs from the loop in its %s\n", what, d); return 1; }
  if (lf - ll < 1) { std::printf("%s: the fused form made no more k1_scaled_sums launches than the loop\n", what); return 1; }
  if (got.ptxtSpace != ipow(T.p, r)) { std::printf("%s: plaintext space %ld\n", what, got.ptxtSpace); return 1; }
  if (!semantic) { std::printf("%s: matches the loop bit for bit\n", what); return 0; }
  const std::vector<long> s = R.values(got);
  if (s.size() != v.size()) { std::printf("%s: not a constant\n", what); return 1; }
  for (size_t k = 0; k < v.size(); k++) {
    const long w = thin_value(v[k], T.p, botHigh, r, ePrime);
    if (s[k] != w) { std::printf("%s: slot %zu holds %ld, want %ld\n", what, k, s[k], w); return 1; }
  }
  std::printf("%s: matches the loop bit for bit and decrypts to the formula\n", what);
  return 0;
}

static int divide_mult_by_p(Ring& R) {
  Setup& T = R.T;
  std::vector<long> v;
  Ctxt c = R.encryptValues(v, T.r - 1);   // values mod p^(r-1), times p below
  const char* what = R.name;
  c.multByP();
  if (c.ptxtSpace != T.P * T.p) { std::printf("%s multByP: plaintext space %ld\n", what, c.ptxtSpace); return 1; }
  c.reducePtxtSpace(T.P);
  std::vector<long> s = R.values(c);
  for (size_t k = 0; k < v.size(); k++) if (s[k] != md(v[k] * T.p, T.P)) { std::printf("%s multByP: slot %zu\n", what, k); return 1; }
  check(hb_ctx_profile(T.ctx.handle(), 1));
  c.divideByP();
  char name[64]; uint64_t launches = 0, bytes = 0; double ms = 0; long nl = 0;
  for (int i = 0; hb_ctx_profile_get(T.ctx.handle(), i, name, sizeof name, &launches, &ms, &bytes) == 0; i++) nl += (long)launches;
  check(hb_ctx_profile(T.ctx.handle(), 0));
  if (nl != 1) { std::printf("%s divideByP: %ld launches, want one for both parts\n", what, nl); return 1; }
  if (c.ptxtSpace != T.P / T.p) { std::printf("%s divideByP: plaintext space %ld\n", what, c.ptxtSpace); return 1; }
  s = R.values(c);
  for (size_t k = 0; k < v.size(); k++) if (s[k] != md(v[k], T.P / T.p)) { std::printf("%s divideByP: slot %zu\n", what, k); return 1; }
  auto throws = [&](Ctxt x, const char* why) {
    try { x.divideByP(); } catch (const LogicError&) { return 0; }
    std::printf("%s divideByP: no LogicError for %s\n", what, why);
    return 1;
  };
  Ctxt odd = c; odd.ptxtSpace = T.P / T.p + 1;
  if (throws(odd, "a plaintext space p does not divide")) return 1;
  Ctxt low = c; while (low.ptxtSpace > T.p) low.reducePtxtSpace(low.ptxtSpace / T.p);
  if (throws(low, "plaintext space p")) return 1;
  Ctxt empty(T.pk, T.P);
  empty.divideByP();   // an empty ciphertext is left as it is
  if (empty.ptxtSpace != T.P) { std::printf("%s divideByP: an empty ciphertext changed\n", what); return 1; }
  std::printf("%s: multByP and divideByP decrypt to p*v and v, divideByP in one launch, and its asserts hold\n", what);
  return 0;
}
static int effective_r(Setup& T) {
  Ctxt c(T.pk, T.P);
  if (c.effectiveR() != T.r) { std::printf("effectiveR: %ld, want %ld\n", c.effectiveR(), T.r); return 1; }
  Ctxt bad(T.pk, T.P + 1);
  try { bad.effectiveR(); } catch (const RuntimeError&) { return 0; }
  std::printf("effectiveR: no RuntimeError for a plaintext space not p^r\n");
  return 1;
}

// A chain over digits at lower prime sets than c, as the powerings leave them on larger rings: each digit is brought down
// by modDownToSet first, so the fused replay mods them up into c's set (addCtxt's addPrimesAndScale scalars and its
// noiseBound / ratFactor update).  Against the loop bit for bit, and decrypted: ((v - d0)/p - d1)/p mod p^(r-2).
static int lower_digits_chain_case(Ring& R) {
  Setup& T = R.T;
  std::vector<long> v;
  const Ctxt c = R.encryptValues(v, T.r);   // a constant v
  const long N = T.ctx.getPhiM();
  std::vector<long> mu0(N, 0), mu1(N, 0);   // d0 = v mod p, d1 = the next digit, so that both divisions are exact
  mu0[0] = md(v[0], T.p);
  mu1[0] = md((v[0] - mu0[0]) / T.p, T.p);
  Ctxt d0 = T.encrypt(mu0), d1 = T.encrypt(mu1);
  IndexSet s0 = d0.primeSet, s1 = d1.primeSet;
  s0.remove(s0.last()); s0.remove(s0.last()); s1.remove(s1.last());
  d0.modDownToSet(s0); d1.modDownToSet(s1);
  if (d0.primeSet == c.primeSet || d1.primeSet == c.primeSet || d0.primeSet == d1.primeSet) { std::printf("%s: the digits were not brought down\n", R.name); return 1; }
  Ctxt got(T.pk, T.P), want(T.pk, T.P);
  check(hb_ctx_profile(T.ctx.handle(), 1));
  detail::digitChain(got, c, {&d0, &d1}, true);
  const long lf = sums_launches(T.ctx);
  detail::digitChain(want, c, {&d0, &d1}, false);
  if (const char* d = differs(got, want)) { std::printf("%s lower digits: differs from the loop in its %s\n", R.name, d); return 1; }
  if (lf != 1) { std::printf("%s lower digits: %ld k1_scaled_sums launches, want 1\n", R.name, lf); return 1; }
  if (!(got.primeSet == c.primeSet)) { std::printf("%s lower digits: the chain did not end at c's prime set\n", R.name); return 1; }
  const long q = ipow(T.p, T.r - 2);
  const std::vector<long> s = R.values(got);
  if (got.ptxtSpace != q || s.size() != 1 || s[0] != md((v[0] - mu0[0] - T.p * mu1[0]) / (T.p * T.p), q)) { std::printf("%s lower digits: decrypts wrong\n", R.name); return 1; }
  g_lower_digits = true;
  std::printf("%s: a chain over digits at two lower prime sets matches the loop bit for bit in one launch and decrypts\n", R.name);
  return 0;
}

static int fallback_case(Ring& R) {
  Setup& T = R.T;
  std::vector<long> v;
  Ctxt c = R.encryptValues(v, T.r);
  std::swap(c.parts[0], c.parts[1]);   // parts in the order (s, 1): not canonical
  std::vector<Ctxt> got, want;
  check(hb_ctx_profile(T.ctx.handle(), 1));
  extractDigits(got, c, 3);
  const long lf = sums_launches(T.ctx);
  extractDigits(want, c, 3, false);
  if (compare(got, want, "non-canonical input")) return 1;
  if (lf != 0) { std::printf("non-canonical input: %ld k1_scaled_sums launches, want the loop's 0\n", lf); return 1; }
  std::printf("%s: a non-canonical input takes the loop with the same digits\n", R.name);
  return 0;
}

int main(int argc, char** argv) {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  const bool full = argc > 1 && std::strcmp(argv[1], "full") == 0;
  try {
    // the polynomial digit maps: the interpolation and Chen and Han's G, by their defining properties
    for (long p : {2L, 3L, 5L, 17L, 257L})
      for (long e = 2; e <= (p == 257 ? 3 : 4); e++) {
        const long q = ipow(p, e);
        const std::vector<long> f = xd::buildDigitPolynomial(p, e), G = xd::chenHanMagicPoly(p, e);
        auto ev = [&](const std::vector<long>& g, long x) { long r = 0; for (size_t t = g.size(); t-- > 0;) r = md(mulm(r, x, q) + g[t], q); return r; };
        for (long x = 0; x < std::min(q, 3000L); x++) {
          const long x0 = p == 2 ? md(x, 2) : bal(x, p);
          if (md(ev(G, x), q) != md(x0, q)) { std::printf("G(%ld) mod %ld^%ld is %ld\n", x, p, e, ev(G, x)); return 1; }
          if (p > 3 && md(ev(f, x), p * p) != md(bal(x, p), p * p)) { std::printf("digit polynomial at %ld mod %ld^%ld\n", x, p, e); return 1; }
        }
        if (p > 3 && (long)f.size() != p + 1) { std::printf("digit polynomial mod %ld^%ld has degree %zu\n", p, e, f.size() - 1); return 1; }
      }
    std::printf("the digit polynomials and Chen-Han's G have their defining properties\n");

    // slots Z/p^r: m = 16, p = 17 (r = 2..4) and m = 32, p = 257 (r = 2)
    for (long r = 2; r <= (full ? 4 : 3); r++) {
      Setup T(16, 17, r, 300 + 450 * r, 7100 + r);
      Slots sl(16, 17, r);
      Ring R{T, &sl, "m=16 p=17"};
      if (r == 2 && (effective_r(T) || divide_mult_by_p(R))) return 1;
      if (digits_case(R, r, "all")) return 1;
      if (r == 3 && digits_case(R, 2, "n<r")) return 1;
    }
    {
      Setup T(16, 17, 4, 1500, 7200);
      Slots sl(16, 17, 4);
      Ring R{T, &sl, "m=16 p=17"};
      if (extend_case(R, 2, 2)) return 1;
      if (extend_case(R, 3, 1)) return 1;
    }
    {
      Setup T(16, 17, 3, 1500, 7300);   // thin: p^(botHigh + r) = 17^3
      Slots sl(16, 17, 3);
      Ring R{T, &sl, "m=16 p=17"};
      for (long ch : {1L, -1L}) if (thin_case(R, 1, 2, 1, ch)) return 1;
      if (thin_case(R, 1, 2, 0, -1) || thin_case(R, 1, 2, 2, 0)) return 1;
    }
    {
      Setup T(32, 257, 2, 1200, 7400);
      Slots sl(32, 257, 2);
      Ring R{T, &sl, "m=32 p=257"};
      if (digits_case(R, 2, "all") || divide_mult_by_p(R)) return 1;
    }
    // p = 2 and p = 3 on rings with larger slots: constant plaintexts (p = 2 needs an odd m: a general-m ring)
    {
      Setup T(105, 2, 5, 700, 7500);
      Ring R{T, nullptr, "m=105 p=2"};
      if (digits_case(R, 5, "all") || digits_case(R, 3, "n<r") || divide_mult_by_p(R) || fallback_case(R) || lower_digits_chain_case(R)) return 1;
    }
    {
      Setup T(105, 2, 4, 700, 7550);
      Ring R{T, nullptr, "m=105 p=2"};
      if (extend_case(R, 2, 2)) return 1;
      for (long ch : {1L, -1L}) if (thin_case(R, 2, 2, 1, ch)) return 1;
      if (thin_case(R, 1, 3, 3, -1, false)) return 1;   // p = 2's free top bit: its value rests on thin recryption's input
    }
    {
      Setup T(105, 2, 4, 600, 7580);   // a general-m ring
      Ring R{T, nullptr, "m=105 p=2"};
      if (digits_case(R, 4, "all")) return 1;
    }
    {
      Setup T(64, 3, 3, 700, 7600);
      Ring R{T, nullptr, "m=64 p=3"};
      if (digits_case(R, 3, "all") || divide_mult_by_p(R)) return 1;
      Setup T4(64, 3, 3, 700, 7650);
      Ring R4{T4, nullptr, "m=64 p=3"};
      for (long ch : {1L, -1L}) if (thin_case(R4, 1, 2, 1, ch)) return 1;
    }
    if (full) {
      // p = 3 on m = 1024 and r = 4 for p = 17
      {
        Setup T(1024, 3, 3, 900, 7600);
        Ring R{T, nullptr, "m=1024 p=3"};
        if (digits_case(R, 3, "all") || divide_mult_by_p(R)) return 1;
        Setup T4(1024, 3, 3, 900, 7650);
        Ring R4{T4, nullptr, "m=1024 p=3"};
        for (long ch : {1L, -1L}) if (thin_case(R4, 1, 2, 1, ch)) return 1;
      }
      Setup T5(21845, 2, 8, 1200, 7700);   // config 5's ring (m = 21845, p = 2)
      Ring R5{T5, nullptr, "config 5"};
      if (digits_case(R5, 8, "all")) return 1;
      Setup T5t(21845, 2, 4, 1200, 7710);
      Ring R5t{T5t, nullptr, "config 5"};
      if (thin_case(R5t, 2, 2, 1, 0)) return 1;
      Setup T3(1 << 17, 257, 2, 1500, 7800, 3);   // config 3's ring and chain (m = 2^17, p = 257)
      Ring R3{T3, nullptr, "config 3"};
      if (digits_case(R3, 2, "all")) return 1;
    }
    if (!g_lower_digits || (full && !g_different_sets)) { std::printf("no case had digits at different prime sets\n"); return 1; }
    std::printf("digits at different prime sets: %s\n", g_different_sets ? "yes" : "no");
    std::printf("extract digits OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
