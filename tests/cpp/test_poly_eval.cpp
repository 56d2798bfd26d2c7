// Polynomial evaluation through the C++ mirror: hb::polyEval (src/polyEval.cpp:129-389) with every simplePolyEval leaf
// formed in one hb_ctxt_scaled_sums call.  Checks, for BGV p = 257 on a power-of-two ring, p = 17 with r = 2 (a plaintext
// space 289 where the top coefficient can be non-invertible and multByConstant has d > 1) and p = 2 on a general-m ring:
//  - polyEval equals a literal transcription of HElib's code kept below, bit for bit, with equal primeSet, noiseBound,
//    intFactor, ratFactor, ptxtMag and mod-switch statistic, for degrees 0 through 70 covering every branch of the
//    recursion (n a power of two, n = 2t - 1 with delta = 0, the general split), an explicit k, and zero, negative, >= p
//    and top = 0 mod p coefficients;
//  - on the fused path the evaluation makes exactly one k1_scaled_sums launch;
//  - each result decrypts to f(m(X)) mod (Phi_m, p^r);
//  - the cases one call cannot reproduce (a non-canonical x, plaintext spaces that differ, an empty x, CKKS) give the
//    transcription's results or its exception, with no k1_scaled_sums launch.
// With the argument "full", also a degree-257 polynomial on BASELINE config 3's ring and chain (m = 2^17, p = 257, 1500 bits,
// c = 3), decrypted.
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
static std::vector<long> cyclotomic(long m) {   // Phi_m(X), low coefficient first
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
// a*b mod (Phi_m(X), P), a and b reduced mod P
static std::vector<long> mul_mod_phi(const std::vector<long>& a, const std::vector<long>& b, const std::vector<long>& phi, long P) {
  const long N = (long)phi.size() - 1;
  std::vector<long> r(2 * N, 0);
  for (long i = 0; i < N; i++) if (a[i]) for (long j = 0; j < N; j++) r[i + j] = (r[i + j] + a[i] * b[j]) % P;
  for (long k = 2 * N - 1; k >= N; k--) { const long c = r[k] % P; if (c) for (long j = 0; j <= N; j++) r[k - N + j] = ((r[k - N + j] - c * phi[j]) % P + P) % P; }
  r.resize(N);
  for (auto& c : r) c = ((c % P) + P) % P;
  return r;
}

// ---- the transcribed HElib code (src/polyEval.cpp:18-29, 129-389, src/Ctxt.cpp:2033-2069, 2145-2185, 2264-2282)
namespace ref {
using ZZX = std::vector<long>;   // NTL's ZZX with word-sized coefficients, normalized
static long deg(const ZZX& a) { return (long)a.size() - 1; }
static void normalize(ZZX& a) { while (!a.empty() && a.back() == 0) a.pop_back(); }
static long coeff(const ZZX& a, long i) { return i >= 0 && i < (long)a.size() ? a[i] : 0; }
static long rem(long a, long p) { long r = a % p; return r < 0 ? r + p : r; }
static void SetCoeff(ZZX& x, long i, long a = 1) { if (i > deg(x)) { if (a == 0) return; x.resize(i + 1, 0); } x[i] = a; normalize(x); }
static ZZX trunc(const ZZX& a, long m) { ZZX r(a.begin(), a.begin() + std::min<long>(std::max(0L, m), a.size())); normalize(r); return r; }
static ZZX RightShift(const ZZX& a, long n) { return n >= (long)a.size() ? ZZX() : ZZX(a.begin() + n, a.end()); }
static long NextPowerOfTwo(long m) { long k = 0; while ((1L << k) < m) k++; return k; }
static long divc(long a, long b) { return (a + b - 1) / b; }
struct Powers {   // DynamicCtxtPowers
  std::vector<Ctxt> v;
  Powers(const Ctxt& c, long n) { if (c.isEmpty()) throw InvalidArgument("Ciphertext cannot be empty"); if (n <= 0) throw InvalidArgument("Must have positive nPowers"); v.assign(n, Ctxt(c.pubKey, c.ptxtSpace)); v[0] = c; }
  Ctxt& getPower(long e) {
    if (v.at(e - 1).isEmpty()) { long k = 1L << (NextPowerOfTwo(e) - 1); v[e - 1] = getPower(e - k); v[e - 1].multiplyBy(getPower(k)); }
    return v[e - 1];
  }
  long size() const { return (long)v.size(); }
};
static void multByConstant(Ctxt& c, long z) {
  if (c.isEmpty()) return;
  long c0 = rem(z, c.ptxtSpace);
  if (c0 == 1) return;
  if (c0 == 0) { c.clear(); return; }
  long d = std::gcd(c0, c.ptxtSpace), c1 = c0 / d, c1_inv = Ctxt::invMod(c1, c.ptxtSpace);
  c.intFactor = (long)((__int128)c.intFactor * c1_inv % c.ptxtSpace);
  if (d == 1) return;
  long cc = Ctxt::balRem(d, c.ptxtSpace);
  c.noiseBound = c.noiseBound * XD((double)std::abs(cc));
  for (auto& part : c.parts) part.dcrt *= cc;
}
static void addConstant(Ctxt& c, long z) {
  long cc = rem(z, c.ptxtSpace);
  if (cc > c.ptxtSpace / 2) cc -= c.ptxtSpace;
  if (cc == 0) return;
  double size = (double)cc;
  long f = 1;
  if (c.ptxtSpace > 2) {
    long q = 1;
    for (long i : c.primeSet) q = (long)((__int128)q * (c.context.ithPrime(i) % c.ptxtSpace) % c.ptxtSpace);
    f = Ctxt::balRem((long)((__int128)c.intFactor * q % c.ptxtSpace), c.ptxtSpace);
  }
  c.noiseBound = c.noiseBound + XD(size * std::abs(f));
  DoubleCRT d(std::vector<long>{cc}, c.context, c.primeSet);
  if (f != 1) d *= f;
  c.addPart(d, SKHandle(0, 1, 0));
}
static void simplePolyEval(Ctxt& ret, const ZZX& poly, Powers& babyStep) {
  ret.clear();
  if (deg(poly) < 0) return;
  if (!(deg(poly) <= babyStep.size())) throw LogicError("BabyStep has not enough powers");
  long p = babyStep.getPower(1).ptxtSpace, coef;
  for (long i = 1; i <= deg(poly); i++) {
    coef = rem(coeff(poly, i), p);
    if (coef > p / 2) coef -= p;
    Ctxt tmp = babyStep.getPower(i);
    multByConstant(tmp, coef);
    ret += tmp;
  }
  coef = rem(coeff(poly, 0), p);
  if (coef > p / 2) coef -= p;
  addConstant(ret, coef);
}
static void PatersonStockmeyer(Ctxt& ret, const ZZX& poly, long k, long t, long delta, Powers& babyStep, Powers& giantStep) {
  if (deg(poly) <= babyStep.size()) { simplePolyEval(ret, poly, babyStep); return; }
  ZZX r = trunc(poly, k * t);
  ZZX q = RightShift(poly, k * t);
  const long p = babyStep.getPower(1).ptxtSpace;
  const long coef = coeff(r, deg(q));
  SetCoeff(r, deg(q), coef - 1);
  // DivRem(c, s, r, q) over Z, then reduce mod p.  The integer quotient outgrows 128 bits, so the long division runs over
  // Z/MZ with M = p*1000003: q is monic, so it commutes with the reduction mod M and then mod p
  const long dq = deg(q), M = p * 1000003;
  std::vector<long> w, cq(deg(r) >= dq ? deg(r) - dq + 1 : 0, 0);
  for (long v : r) w.push_back(rem(v, M));
  for (long i = deg(r); i >= dq; i--) {
    const long tt = w[i]; cq[i - dq] = tt;
    for (long j = 0; j <= dq; j++) w[i - dq + j] = (long)((((__int128)w[i - dq + j] - (__int128)tt * rem(q[j], M)) % M + M) % M);
  }
  w.resize(std::max(0L, std::min<long>(dq, w.size())));
  ZZX c, s;
  for (long v : cq) c.push_back(v % p);
  for (long v : w) s.push_back(v % p);
  normalize(c); normalize(s);
  SetCoeff(s, deg(q));
  for (auto& v : s) v = rem(v, p);
  normalize(s);
  PatersonStockmeyer(ret, q, k, t / 2, delta, babyStep, giantStep);
  Ctxt tmp(ret.pubKey, ret.ptxtSpace);
  simplePolyEval(tmp, c, babyStep);
  tmp += giantStep.getPower(t);
  ret.multiplyBy(tmp);
  PatersonStockmeyer(tmp, s, k, t / 2, delta, babyStep, giantStep);
  ret += tmp;
}
static void degPowerOfTwo(Ctxt& ret, const ZZX& poly, long k, Powers& babyStep, Powers& giantStep) {
  if (deg(poly) <= babyStep.size()) { simplePolyEval(ret, poly, babyStep); return; }
  long n = deg(poly) / k;
  n = 1L << NextPowerOfTwo(n);
  ZZX r = trunc(poly, (n - 1) * k);
  ZZX q = RightShift(poly, (n - 1) * k);
  SetCoeff(r, (n - 1) * k);
  if (q.empty()) q.push_back(-1); else { q[0] -= 1; normalize(q); }
  PatersonStockmeyer(ret, r, k, n / 2, 0, babyStep, giantStep);
  Ctxt tmp(ret.pubKey, ret.ptxtSpace);
  simplePolyEval(tmp, q, babyStep);
  for (long i = 1; i < n; i *= 2) tmp.multiplyBy(giantStep.getPower(i));
  ret += tmp;
}
static void recursivePolyEval(Ctxt& ret, const ZZX& poly, long k, Powers& babyStep, Powers& giantStep) {
  if (deg(poly) <= babyStep.size()) { simplePolyEval(ret, poly, babyStep); return; }
  long delta = deg(poly) % k;
  long n = divc(deg(poly), k);
  long t = 1L << NextPowerOfTwo(n);
  if (n == t) { degPowerOfTwo(ret, poly, k, babyStep, giantStep); return; }
  if (n == t - 1 && delta == 0) { PatersonStockmeyer(ret, poly, k, t / 2, delta, babyStep, giantStep); return; }
  t = t / 2;
  long u = deg(poly) - k * (t - 1);
  ZZX r = trunc(poly, u);
  ZZX q = RightShift(poly, u);
  if (q.empty()) q.push_back(-1); else { q[0] -= 1; normalize(q); }
  SetCoeff(r, u);
  PatersonStockmeyer(ret, q, k, t / 2, 0, babyStep, giantStep);
  Ctxt tmp = giantStep.getPower(u / k);
  if (delta != 0) tmp.multiplyBy(babyStep.getPower(delta));
  ret.multiplyBy(tmp);
  recursivePolyEval(tmp, r, k, babyStep, giantStep);
  ret += tmp;
}
static void polyEval(Ctxt& ret, ZZX poly, const Ctxt& x, long k) {
  normalize(poly);
  if (deg(poly) <= 2) {
    if (deg(poly) < 1) { ret.clear(); addConstant(ret, coeff(poly, 0)); }
    else { Powers babyStep(x, deg(poly)); simplePolyEval(ret, poly, babyStep); }
    return;
  }
  if (k <= 0) {
    long kk = (long)sqrt(deg(poly) / 2.0);
    k = 1L << NextPowerOfTwo(kk);
    if ((k == 16 && deg(poly) > 167) || (k > 16 && k > (1.44 * kk))) k /= 2;
  }
  long n = divc(deg(poly), k);
  Powers babyStep(x, k);
  const Ctxt& x2k = babyStep.getPower(k);
  if (n == (1L << NextPowerOfTwo(n))) { Powers giantStep(x2k, n / 2); degPowerOfTwo(ret, poly, k, babyStep, giantStep); return; }
  const long p = x.ptxtSpace;
  long top = poly.back(), topInv = 0;
  bool divisible = (n * k == deg(poly));
  if (top < 0 || top >= p) throw LogicError("InvMod: first input out of range");   // NTL's InvModStatus takes 0 <= a < n
  long nonInvertible = std::gcd(top, p) != 1;
  if (!nonInvertible) topInv = Ctxt::invMod(top, p);
  long extra = 0;
  if (!divisible || nonInvertible) {
    top = 1; topInv = top;
    extra = top - coeff(poly, n * k); if (extra < 0) extra += p;   // SubMod
    SetCoeff(poly, n * k);
  }
  long t = extra == 0 ? divc(n, 2) : n;
  Powers giantStep(x2k, t);
  if (top != 1) {
    for (auto& c : poly) c = (long)((__int128)c * topInv % p);
    for (long i = 0; i <= n * k; i++) poly[i] = rem(poly[i], p);
    normalize(poly);
  }
  recursivePolyEval(ret, poly, k, babyStep, giantStep);
  if (top != 1) multByConstant(ret, top);
  if (extra != 0) { Ctxt topTerm = giantStep.getPower(n); multByConstant(topTerm, extra); ret -= topTerm; }
}
}  // namespace ref

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

static KeyInfo key_info(const Context& ctx, bool ckks) {
  KeyInfo pk;
  pk.context = &ctx; pk.ckks = ckks; pk.scale = 10.0; pk.hwt = 0;
  pk.skBound = pk.scale * std::sqrt(double(ctx.getPhiM()) * 2.0 / 3.0);
  return pk;
}
// keys and symmetric encryption at plaintext space P = p^r (CKKS: P = 1)
struct Setup {
  Context ctx;
  KeyInfo pk;
  DoubleCRT S;
  long P;
  std::mt19937_64 gen;
  Setup(long m, long p, long r, long bits, uint64_t seed, long c = 2)
      : ctx(m, p, r, bits, c), pk(key_info(ctx, p < 0)), S(ctx, ctx.getCtxtPrimes() | ctx.getSpecialPrimes()), P(1), gen(seed) {
    if (p > 0) for (long i = 0; i < r; i++) P *= p;
    const long N = ctx.getPhiM();
    const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
    S = DoubleCRT(sample_ternary(gen, N), ctx, allq);
    DoubleCRT s2(S); s2 *= S;
    KeySwitch W; W.fromKey = SKHandle(2, 1, 0); W.toKeyID = 0; W.ptxtSpace = P;
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
  std::vector<long> message() {   // small messages keep the coefficient sums of f(m) in range of mul_mod_phi
    std::vector<long> v(ctx.getPhiM());
    for (auto& x : v) x = (long)(gen() % 3) - 1 + P;
    for (auto& x : v) x %= P;
    return v;
  }
};
// f(mu) mod (Phi_m, P) by Horner
static std::vector<long> ptxt_eval(const std::vector<long>& f, const std::vector<long>& mu, const std::vector<long>& phi, long P) {
  const long N = (long)mu.size();
  std::vector<long> r(N, 0);
  for (long i = (long)f.size() - 1; i >= 0; i--) {
    r = mul_mod_phi(r, mu, phi, P);
    r[0] = ((r[0] + f[i]) % P + P) % P;
  }
  return r;
}
static int check_decrypt(Setup& T, const Ctxt& got, const std::vector<long>& want, const char* what) {
  std::vector<long> out;
  Decrypt(out, got, {T.S});
  for (long s = 0; s < 32; s++) {
    const long idx = (s * 173 + 11) % T.ctx.getPhiM();
    const long o = ((out[idx] % T.P) + T.P) % T.P;
    if (o != want[idx]) { std::printf("%s: coefficient %ld decrypts to %ld, want %ld\n", what, idx, o, want[idx]); return 1; }
  }
  return 0;
}

struct Case { long deg; long k; int top; };   // top: 0 random unit, 1 top = 0 mod P, 2 top = p (not invertible mod p^r)
static int run_case(Setup& T, const Ctxt& x, const std::vector<long>& mu, const std::vector<long>& phi, const Case& c, bool decrypt, const char* ring) {
  std::vector<long> f(c.deg + 1);
  for (long i = 0; i <= c.deg; i++) {
    const long v = (long)(T.gen() % 7);   // zero, small, negative, >= P and large coefficients
    f[i] = v == 0 ? 0 : v == 1 ? -(long)(T.gen() % (3 * T.P)) : v == 2 ? T.P + (long)(T.gen() % T.P) : v == 3 ? (long)(T.gen() % (1L << 40)) - (1L << 39) : (long)(T.gen() % T.P);
  }
  f[c.deg] = c.top == 1 ? T.P : c.top == 2 ? T.ctx.getP() : 1 + (long)(T.gen() % (T.P - 1));
  if (c.top == 0 && std::gcd(f[c.deg], T.P) != 1) f[c.deg] = 1;
  Ctxt got(T.pk, T.P), want(T.pk, T.P);
  check(hb_ctx_profile(T.ctx.handle(), 1));
  polyEval(got, f, x, c.k);
  const long launches = sums_launches(T.ctx);
  ref::polyEval(want, f, x, c.k);
  char what[160];
  std::snprintf(what, sizeof what, "%s degree %ld k %ld top %d", ring, c.deg, c.k, c.top);
  if (const char* d = differs(got, want)) { std::printf("%s: differs from the transcription in its %s\n", what, d); return 1; }
  long terms = 0;   // a leaf term exists when some non-constant coefficient is nonzero mod P (polyEval's leaves all take
  for (long i = 1; i <= c.deg; i++) terms += ref::rem(f[i], T.P) != 0;   // some power then; a degree >= 3 always has one)
  if (c.deg >= 1 && launches != 1 && (c.deg >= 3 || terms > 0)) { std::printf("%s: %ld k1_scaled_sums launches, want 1\n", what, launches); return 1; }
  if (decrypt) {
    std::vector<long> fr(f.size());
    for (size_t i = 0; i < f.size(); i++) fr[i] = ref::rem(f[i], T.P);
    if (check_decrypt(T, got, ptxt_eval(fr, mu, phi, T.P), what)) return 1;
  }
  return 0;
}

static int ring_cases(long m, long p, long r, long bits, const std::vector<Case>& cases, long maxdec, const char* ring) {
  Setup T(m, p, r, bits, 20261018 + m + p);
  const std::vector<long> phi = cyclotomic(m);
  const std::vector<long> mu = T.message();
  const Ctxt x = T.encrypt(mu);
  for (const Case& c : cases) if (run_case(T, x, mu, phi, c, c.deg <= maxdec, ring)) return 1;
  std::printf("%s: %zu polynomials match the transcription bit for bit in one k1_scaled_sums launch each, and decrypt to f(m)\n", ring, cases.size());
  return 0;
}

static int fallback_cases() {
  Setup T(1024, 257, 1, 300, 91);
  const std::vector<long> f = {3, -1, 0, 200, 5, 1, 7, 1};
  const Ctxt x = T.encrypt(T.message());
  auto same = [&](const char* what, const Ctxt& xin, long retP) {
    Ctxt got(T.pk, retP), want(T.pk, retP);
    check(hb_ctx_profile(T.ctx.handle(), 1));
    polyEval(got, f, xin, 0);
    if (sums_launches(T.ctx) != 0) { std::printf("%s: k1_scaled_sums ran\n", what); return 1; }
    ref::polyEval(want, f, xin, 0);
    if (const char* d = differs(got, want)) { std::printf("%s: differs from the transcription in its %s\n", what, d); return 1; }
    return 0;
  };
  if (same("ret at another plaintext space", x, 257 * 257)) return 1;
  Ctxt xr = x;   // x with its parts in the order (s, 1): not canonical
  std::swap(xr.parts[0], xr.parts[1]);
  if (same("non-canonical x", xr, 257)) return 1;
  bool threw = false;
  try { Ctxt e(T.pk, 257), out(T.pk, 257); polyEval(out, f, e); } catch (const InvalidArgument&) { threw = true; }
  if (!threw) { std::printf("empty x: no InvalidArgument\n"); return 1; }
  Setup C(1024, -1, 20, 300, 92);   // CKKS: the scalar forms are BGV only, in the mirror and the transcription alike
  const Ctxt xc = C.encrypt(std::vector<long>(C.ctx.getPhiM(), 0));
  bool a = false, b = false;
  try { Ctxt out(C.pk, 1); polyEval(out, f, xc); } catch (const LogicError&) { a = true; }
  try { Ctxt out(C.pk, 1); ref::polyEval(out, f, xc, 0); } catch (const LogicError&) { b = true; }
  if (!a || !b) { std::printf("CKKS: expected LogicError from both\n"); return 1; }
  std::printf("fallbacks: non-canonical x, differing plaintext spaces, empty x and CKKS behave as the transcription\n");
  return 0;
}

int main(int argc, char** argv) {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  const bool full = argc > 1 && std::strcmp(argv[1], "full") == 0;
  try {
    // degrees 0..2 (simple), 3..70: n a power of two (4, 8, 16, 33 at k = 1, 2, 4, 4 ...), n = 2t - 1 with delta = 0 (deg 12
    // at k = 4: n = 3), the general split (5, 10, 20, 45, 70), an explicit k, top = 0 mod p where n is a power of two
    const std::vector<Case> bgv = {{0, 0, 0}, {1, 0, 0}, {2, 0, 0}, {2, 0, 1}, {3, 0, 0}, {4, 0, 1}, {5, 0, 0}, {6, 0, 0},
                                   {8, 0, 1}, {12, 4, 0}, {10, 0, 0}, {16, 0, 0}, {20, 0, 0}, {20, 4, 0}, {28, 4, 0},
                                   {33, 0, 0}, {45, 0, 0}, {64, 0, 0}, {70, 0, 0}};
    if (ring_cases(1024, 257, 1, 600, bgv, 12, "BGV p=257 m=1024")) return 1;
    const std::vector<Case> pr = {{3, 0, 0}, {7, 0, 2}, {10, 0, 2}, {12, 4, 2}, {14, 0, 0}, {21, 0, 2}};
    if (ring_cases(1024, 17, 2, 600, pr, 12, "BGV p=17^2 m=1024")) return 1;
    const std::vector<Case> two = {{2, 0, 0}, {3, 0, 0}, {6, 0, 0}, {9, 0, 0}};
    if (ring_cases(105, 2, 1, 300, two, 9, "BGV p=2 m=105")) return 1;
    if (fallback_cases()) return 1;
    if (full) {   // config 3's chain (m = 2^17, p = 257, 1500 bits, c = 3) and a constant message, so that f(m) is the
                  // constant f(m_0) mod p and Horner's products mod Phi_m stay O(phi(m))
      Setup T(1 << 17, 257, 1, 1500, 93, 3);
      std::vector<long> mu(T.ctx.getPhiM(), 0), phi(T.ctx.getPhiM() + 1, 0);
      mu[0] = 2 + (long)(T.gen() % 250);
      phi[0] = 1; phi.back() = 1;   // Phi_m = X^(m/2) + 1
      const Ctxt x = T.encrypt(mu);
      if (run_case(T, x, mu, phi, {257, 0, 0}, true, "config 3")) return 1;
      std::printf("config 3: a degree-257 polynomial matches the transcription in one k1_scaled_sums launch and decrypts to f(m)\n");
    }
    std::printf("poly eval OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
