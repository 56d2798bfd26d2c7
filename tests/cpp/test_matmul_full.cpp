// Full-matrix linear maps through the C++ mirror: hb::MatMulFull, MatMulFullExec::mul (src/matmul.cpp:2132-2273, FULL
// strategies, one thread), whose leaves go through one hb_full_linear_map_leaves_norm call, and hb::MatMul1D's bad hoisted
// branch (src/matmul.cpp:1253-1283).  Checks:
//  - hb::MatMulFull equals a literal transcription of rec_mul (BasicAutomorphPrecon rotations, the bad outer dimension's
//    masks, MatMul1DExec leaves, +=) bit for bit, with equal metadata, for 2 and 3 dimensions, native and bad outer and
//    leaf dimensions, NULL diagonals and an all-NULL leaf;
//  - it decrypts to the same recursion on plaintext polynomials mod p (sigma_k and products mod X^N + 1);
//  - the tracked noise bound dominates the decrypted polynomial's largest coefficient;
//  - the fallbacks are taken and still match: a leaf amount without a direct matrix (the transcribed leaves) and a leaf
//    dimension above the BSGS threshold (hb::MatMul1DBSGS per leaf);
//  - hb::MatMul1D's bad branch equals its loop and hb::BlockMatMul1D with d = 1, bits and metadata;
//  - CKKS is refused with LogicError.
// Exit codes: 0 ok, 3 no CUDA device, 1 failure.
#include <algorithm>
#include <cstdio>
#include <random>
#include <string>

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
// f(X^k) mod (X^N + 1, p)
static std::vector<long> rotate(const std::vector<long>& f, long k, long N, long p) {
  std::vector<long> out(N, 0);
  for (long i = 0; i < N; i++) { const long j = (i * k) % (2 * N); if (j < N) out[j] = (out[j] + f[i]) % p; else out[j - N] = (out[j - N] - f[i]) % p; }
  return out;
}
// c(X) * f(X) mod (X^N + 1, p) for a sparse c
static std::vector<long> mul_sparse(const std::vector<long>& c, const std::vector<long>& f, long N, long p) {
  std::vector<long> out(N, 0);
  for (long a = 0; a < N; a++) {
    if (!c[a]) continue;
    for (long b = 0; b < N; b++) { const long t = a + b, v = c[a] * f[b]; if (t < N) out[t] = (out[t] + v) % p; else out[t - N] = (out[t - N] - v) % p; }
  }
  return out;
}
static void add_into(std::vector<long>& a, const std::vector<long>& b, long p, long sign = 1) { for (size_t i = 0; i < a.size(); i++) a[i] = (a[i] + sign * b[i]) % p; }

// whether k_ks_leafmap ran since profiling was enabled
static bool leafmap_ran(const Context& ctx) {
  char name[64]; uint64_t launches = 0, bytes = 0; double ms = 0;
  for (int i = 0; hb_ctx_profile_get(ctx.handle(), i, name, sizeof(name), &launches, &ms, &bytes) == 0; i++)
    if (std::string(name) == "k_ks_leafmap" && launches > 0) return true;
  return false;
}

struct Diag { std::vector<long> coeffs; BsgsDiag d; };   // a constant as a polynomial (empty: NULL) and as MulAdd takes it

struct Setup {
  Context ctx;
  KeyInfo pk;
  DoubleCRT S;
  std::vector<DoubleCRT> sKeys;
  std::mt19937_64 g;
  std::vector<DoubleCRT> store;
  long m, p, N;
  Setup(long seed) : ctx(2048, 257, 1, /*bits=*/200, /*c=*/2), S(std::vector<long>(ctx.getPhiM(), 0), ctx, ctx.getCtxtPrimes() | ctx.getSpecialPrimes()),
                     g((uint64_t)seed), m(2048), p(257), N(ctx.getPhiM()) {
    store.reserve(4096);
    S = DoubleCRT(sample_ternary(g, N), ctx, ctx.getCtxtPrimes() | ctx.getSpecialPrimes());
  }
  void keys(std::vector<long> rots) {
    pk.context = &ctx; pk.ckks = false; pk.scale = 10.0; pk.hwt = 0;
    pk.skBound = pk.scale * std::sqrt(double(N) * 2.0 / 3.0);
    std::sort(rots.begin(), rots.end()); rots.erase(std::unique(rots.begin(), rots.end()), rots.end());
    for (long r : rots) {
      if (r == 1) continue;
      DoubleCRT sr(S); sr.automorph(r);
      std::vector<uint8_t> seed(32);
      for (auto& b : seed) b = (uint8_t)(g() & 0xff);
      seed[31] |= 1;
      pk.keySwitching.push_back(genKeySWmatrix(ctx, sr, SKHandle(1, r, 0), 0, S, p, false, 3.2, g, seed));
    }
    pk.setKeySwitchMap(0);
    sKeys.push_back(S);
  }
  Ctxt encrypt(std::vector<long>& msg) {
    const double sigma = 3.2;
    Ctxt pubEncrKey(pk, p);
    pubEncrKey.primeSet = ctx.getCtxtPrimes();
    DoubleCRT c1 = random_rows(ctx, pubEncrKey.primeSet, g);
    DoubleCRT c0(sample_gauss(g, N, sigma), ctx, pubEncrKey.primeSet); c0 *= p;
    DoubleCRT t(c1); t.Mul(S, false); c0 -= t;
    pubEncrKey.parts.emplace_back(c0, SKHandle());
    pubEncrKey.parts.emplace_back(c1, SKHandle(1, 1, 0));
    pubEncrKey.noiseBound = XD(double(p) * pk.noiseBoundForGaussian(sigma, N));
    msg.assign(N, 0);
    for (auto& x : msg) x = (long)(g() % p);
    Ctxt c(pk, p);
    hb::EncryptionSample smp = hb::drawEncryptionSample(ctx, sigma, g);
    hb::Encrypt(c, pubEncrKey, msg, p, smp);
    return c;
  }
  Diag diag(bool none, long e) {
    Diag x;
    x.d = BsgsDiag{nullptr, e % 3 ? -1.0 : 30.0, XD(), XD(), 0.0};
    if (none) return x;
    x.coeffs.assign(N, 0);
    for (long s = 0; s < 6; s++) x.coeffs[(size_t)(g() % N)] = (long)(g() % 5) - 2;
    store.emplace_back(x.coeffs, ctx, ctx.getCtxtPrimes() | ctx.getSpecialPrimes());
    x.d.c = &store.back();
    return x;
  }
};

// ---- the literal transcription of MatMulFullExec::rec_mul and of MatMul1DExec::mul's hoisted branches
static void leaf_loop(Ctxt& c, const FullDim& d, const std::vector<BsgsDiag>& cache, const std::vector<BsgsDiag>* cache1) {
  const long m = c.context.getM();
  c.cleanUp();
  if (d.D > kBsgsMulThresh) { MatMul1DBSGS(c, d.gen, d.D, cache, cache1 ? *cache1 : std::vector<BsgsDiag>{}); return; }
  BasicAutomorphPrecon precon(c);
  Ctxt acc(c.pubKey, c.ptxtSpace), acc1(c.pubKey, c.ptxtSpace);
  for (long i = 0; i < d.D; i++) {
    if (!cache[i].c && !(cache1 && (*cache1)[i].c)) continue;
    auto tmp = precon.automorph(genToPow(d.gen, i, m));
    if (cache[i].c) { Ctxt t(*tmp); t.multByConstant(*cache[i].c, cache[i].size); acc += t; }
    if (cache1 && (*cache1)[i].c) { Ctxt t(*tmp); t.multByConstant(*(*cache1)[i].c, (*cache1)[i].size); acc1 += t; }
  }
  if (cache1 && !acc1.isEmpty()) { acc1.smartAutomorph(genToPow(d.gen, -d.D, m)); acc += acc1; }
  c = acc;
}
static long rec_mul(Ctxt& acc, const Ctxt& c, const std::vector<FullDim>& dims, size_t di, long idx,
                    const std::vector<std::vector<BsgsDiag>>& leaves, const std::vector<std::vector<BsgsDiag>>& leaves1) {
  const long m = c.context.getM();
  if (di + 1 == dims.size()) {
    Ctxt tmp = c;
    leaf_loop(tmp, dims[di], leaves[idx], dims[di].native ? nullptr : &leaves1[idx]);
    acc += tmp;
    return idx + 1;
  }
  const FullDim& d = dims[di];
  if (d.native) {
    BasicAutomorphPrecon precon(c);
    for (long i = 0; i < d.D; i++) idx = rec_mul(acc, *precon.automorph(genToPow(d.gen, i, m)), dims, di + 1, idx, leaves, leaves1);
    return idx;
  }
  Ctxt c1 = c;
  c1.smartAutomorph(genToPow(d.gen, -d.D, m));
  BasicAutomorphPrecon precon(c), precon1(c1);
  for (long i = 0; i < d.D; i++) {
    if (i == 0) { idx = rec_mul(acc, c, dims, di + 1, idx, leaves, leaves1); continue; }
    auto tmp = precon.automorph(genToPow(d.gen, i, m));
    auto tmp1 = precon1.automorph(genToPow(d.gen, i, m));
    tmp->multByConstant(*d.masks[i].c, d.masks[i].size);
    *tmp += *tmp1;
    tmp1->multByConstant(*d.masks[i].c, d.masks[i].size);
    tmp->addCtxt(*tmp1, true);
    idx = rec_mul(acc, *tmp, dims, di + 1, idx, leaves, leaves1);
  }
  return idx;
}
// the same recursion on plaintext polynomials mod p
static long want_rec(std::vector<long>& out, const std::vector<long>& f, const std::vector<FullDim>& dims, const std::vector<std::vector<std::vector<long>>>& mk,
                     size_t di, long idx, const std::vector<std::vector<Diag>>& lv, const std::vector<std::vector<Diag>>& lv1, long m, long N, long p) {
  const FullDim& d = dims[di];
  if (di + 1 == dims.size()) {
    std::vector<long> y(N, 0);
    if (d.D > kBsgsMulThresh) {   // HElib's BSGS branch: diagonal j + g*k multiplies baby step j inside giant step k
      long g = (long)std::sqrt((double)d.D); while (g * g < d.D) g++; while (g > 1 && (g - 1) * (g - 1) >= d.D) g--;
      for (long k = 0; k * g < d.D; k++) {
        std::vector<long> a(N, 0);
        for (long j = 0; j < g && j + g * k < d.D; j++)
          if (!lv[idx][j + g * k].coeffs.empty()) add_into(a, mul_sparse(lv[idx][j + g * k].coeffs, rotate(f, genToPow(d.gen, j, m), N, p), N, p), p);
        add_into(out, rotate(a, genToPow(d.gen, g * k, m), N, p), p);
      }
      return idx + 1;
    }
    for (long t = 0; t < d.D; t++) {
      const auto r = rotate(f, genToPow(d.gen, t, m), N, p);
      if (!lv[idx][t].coeffs.empty()) add_into(out, mul_sparse(lv[idx][t].coeffs, r, N, p), p);
      if (!d.native && !lv1[idx][t].coeffs.empty()) add_into(y, mul_sparse(lv1[idx][t].coeffs, r, N, p), p);
    }
    if (!d.native) add_into(out, rotate(y, genToPow(d.gen, -d.D, m), N, p), p);
    return idx + 1;
  }
  const auto f1 = rotate(f, genToPow(d.gen, -d.D, m), N, p);
  for (long i = 0; i < d.D; i++) {
    const auto r = rotate(f, genToPow(d.gen, i, m), N, p);
    if (d.native || i == 0) { idx = want_rec(out, d.native ? r : f, dims, mk, di + 1, idx, lv, lv1, m, N, p); continue; }
    const auto r1 = rotate(f1, genToPow(d.gen, i, m), N, p);
    std::vector<long> x = mul_sparse(mk[di][i], r, N, p);
    add_into(x, r1, p);
    add_into(x, mul_sparse(mk[di][i], r1, N, p), p, -1);
    idx = want_rec(out, x, dims, mk, di + 1, idx, lv, lv1, m, N, p);
  }
  return idx;
}

// given: the dimensions in any order (hb::MatMulFull sorts them); skip: an amount left without a direct matrix
static int full_case(const char* name, std::vector<FullDim> given, long skip = 0, bool fused = true) {
  Setup T(20261016 + (long)given.size() * 7 + given.back().D + skip);
  std::vector<FullDim> dims = given;
  std::stable_sort(dims.begin(), dims.end(), [](const FullDim& a, const FullDim& b) { return a.D < b.D || (a.D == b.D && a.native && !b.native); });
  std::vector<long> rots;
  for (const FullDim& d : dims) {
    for (long i = 0; i < d.D; i++) rots.push_back(genToPow(d.gen, i, T.m));
    if (!d.native) rots.push_back(genToPow(d.gen, -d.D, T.m));
  }
  if (skip) rots.erase(std::remove(rots.begin(), rots.end(), skip), rots.end());
  T.keys(rots);
  std::vector<long> msg;
  Ctxt c = T.encrypt(msg);
  // masks of the bad outer dimensions, and the leaves' diagonals: every fifth NULL, leaf 1 without any
  std::vector<std::vector<std::vector<long>>> mk(dims.size());
  for (size_t di = 0; di + 1 < dims.size(); di++) {
    if (dims[di].native) continue;
    mk[di].assign(dims[di].D, {});
    dims[di].masks.assign(dims[di].D, BsgsDiag{nullptr, -1.0, XD(), XD(), 0.0});
    for (long i = 1; i < dims[di].D; i++) { Diag x = T.diag(false, i); mk[di][i] = x.coeffs; dims[di].masks[i] = x.d; }
  }
  for (FullDim& gd : given) for (const FullDim& d : dims) if (gd.gen == d.gen && gd.D == d.D) gd.masks = d.masks;
  long nl = 1;
  for (size_t di = 0; di + 1 < dims.size(); di++) nl *= dims[di].D;
  const FullDim& last = dims.back();
  std::vector<std::vector<Diag>> lv(nl), lv1(last.native ? 0 : nl);
  std::vector<std::vector<BsgsDiag>> leaves(nl), leaves1(last.native ? 0 : nl);
  for (long l = 0; l < nl; l++)
    for (long t = 0; t < last.D; t++) {
      const long e = l * last.D + t;
      lv[l].push_back(T.diag(l == 1 || e % 5 == 4, e)); leaves[l].push_back(lv[l].back().d);
      if (!last.native) { lv1[l].push_back(T.diag(l == 1, e + 1)); leaves1[l].push_back(lv1[l].back().d); }
    }
  Ctxt loop(c);
  {
    loop.cleanUp();
    Ctxt acc(T.pk, T.p);
    rec_mul(acc, loop, dims, 0, 0, leaves, leaves1);
    loop = acc;
  }
  Ctxt got(c);
  check(hb_ctx_profile(T.ctx.handle(), 1));
  MatMulFull(got, given, leaves, leaves1);
  const bool ran = leafmap_ran(T.ctx);
  check(hb_ctx_profile(T.ctx.handle(), 0));
  if (const char* what = differs(got, loop)) { std::printf("%s: MatMulFull differs from rec_mul in its %s\n", name, what); return 1; }
  if (ran != fused) { std::printf("%s: the leaves %s through hb_full_linear_map_leaves\n", name, ran ? "went" : "did not go"); return 1; }
  std::vector<long> out; std::vector<uint64_t> limbs; int L = 0;
  hb::Decrypt(out, got, T.sKeys, &limbs, &L);
  std::vector<long> want(T.N, 0);
  want_rec(want, msg, dims, mk, 0, 0, lv, lv1, T.m, T.N, T.p);
  long double worst = 0;
  for (long i = 0; i < T.N; i++) {
    const long w = ((want[i] % T.p) + T.p) % T.p;
    if (out[i] != w) { std::printf("%s: coefficient %ld decrypts to %ld, want %ld\n", name, i, out[i], w); return 1; }
    worst = std::max(worst, std::fabs(limbs_to_ld(&limbs[(size_t)i * L], L)));
  }
  const double lnw = std::log((double)worst), lnb = got.noiseBound.ln();
  if (lnw > lnb) { std::printf("%s: measured noise e^%.2f exceeds the tracked bound e^%.2f\n", name, lnw, lnb); return 1; }
  std::printf("%s: bits and metadata of rec_mul, decrypts, noise e^%.1f <= bound e^%.1f\n", name, lnw, lnb);
  return 0;
}

// hb::MatMul1D's bad hoisted branch against its loop and hb::BlockMatMul1D with d = 1
static int matmul1d_bad() {
  Setup T(77);
  const long gen = 3, D = 5;
  std::vector<long> rots;
  for (long i = 0; i < D; i++) rots.push_back(genToPow(gen, i, T.m));
  rots.push_back(genToPow(gen, -D, T.m));
  T.keys(rots);
  std::vector<long> msg;
  Ctxt c = T.encrypt(msg);
  std::vector<BsgsDiag> cache, cache1;
  for (long i = 0; i < D; i++) { cache.push_back(T.diag(i == 2, i).d); cache1.push_back(T.diag(false, i + 1).d); }
  Ctxt got(c), loop(c), block(c);
  check(hb_ctx_profile(T.ctx.handle(), 1));
  MatMul1D(got, gen, D, cache, cache1);
  const bool ran = leafmap_ran(T.ctx);
  check(hb_ctx_profile(T.ctx.handle(), 0));
  if (!ran) { std::printf("MatMul1D bad: hb_full_linear_map_leaves did not run\n"); return 1; }
  leaf_loop(loop, FullDim{gen, D, false, {}}, cache, &cache1);
  BlockMatMul1D(block, gen, D, 1, cache, cache1);
  if (const char* what = differs(got, loop)) { std::printf("MatMul1D bad: differs from the loop in its %s\n", what); return 1; }
  if (const char* what = differs(got, block)) { std::printf("MatMul1D bad: differs from BlockMatMul1D(d = 1) in its %s\n", what); return 1; }
  std::printf("MatMul1D bad dimension: bits and metadata of the loop and of BlockMatMul1D with d = 1\n");
  return 0;
}

static int ckks_refused() {
  Context ctx(2048, /*p=*/-1, /*r=*/20, /*bits=*/200, /*c=*/2);
  KeyInfo pk; pk.context = &ctx; pk.ckks = true;
  Ctxt c(pk, 1);
  try { MatMulFull(c, {FullDim{5, 2, true, {}}, FullDim{3, 2, true, {}}}, std::vector<std::vector<BsgsDiag>>(2, std::vector<BsgsDiag>(2))); }
  catch (const LogicError&) { std::printf("CKKS: refused (LogicError)\n"); return 0; }
  std::printf("CKKS: MatMulFull did not throw LogicError\n");
  return 1;
}

int main() {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  try {
    const long m = 2048;
    if (full_case("2 dims, native outer, native leaf", {{5, 2, true, {}}, {3, 3, true, {}}}) != 0 ||
        full_case("2 dims, bad outer, bad leaf", {{5, 3, false, {}}, {3, 3, false, {}}}) != 0 ||
        full_case("3 dims, native, native, bad leaf (given out of order)", {{3, 3, false, {}}, {5, 2, true, {}}, {7, 3, true, {}}}) != 0 ||
        full_case("3 dims, bad outer, native leaf", {{5, 2, true, {}}, {7, 2, false, {}}, {3, 3, true, {}}}) != 0 ||
        full_case("fallback: leaf amount without a direct matrix", {{5, 2, true, {}}, {3, 3, true, {}}}, genToPow(3, 2, m), false) != 0 ||
        full_case("fallback: leaf dimension above the BSGS threshold", {{5, 2, true, {}}, {3, 52, true, {}}}, 0, false) != 0 ||
        matmul1d_bad() != 0 || ckks_refused() != 0)
      return 1;
    std::printf("matmul full OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
