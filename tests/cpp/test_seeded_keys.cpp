// Key-switching matrices held as HElib holds them (b_i rows plus prgSeed) through the C++ mirror.  KeySwitch::compress()
// drops the expanded a_i and keeps the seeded form (hb_poly_create_seeded); every key switch regenerates the rows it reads.
//   argv[1] = prgSeed of the relinearisation matrix as hex (little-endian magnitude bytes).
// Checks, all bit for bit against the same operations with the expanded matrices:
//  - relinearise (multiplyBy) and decrypt with compressed matrices, with matrices read by readFrom(..., false), and with a
//    copy of a compressed KeySwitch (which shares the seeded rows instead of copying them);
//  - hoisted rotations through BasicAutomorphPrecon;
//  - writeTo writes the same bytes for both forms;
//  - compress() without a seed throws InvalidArgument; compressing halves the device memory of a matrix.
// Exit codes: 0 ok, 3 no CUDA device, 1 failure.
#include <cstdio>
#include <random>
#include <sstream>
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
static bool same_ctxt(const Ctxt& x, const Ctxt& y) {
  if (x.parts.size() != y.parts.size()) return false;
  for (size_t j = 0; j < x.parts.size(); j++)
    if (!(x.parts[j].skHandle == y.parts[j].skHandle) || !same_rows(x.parts[j].dcrt, y.parts[j].dcrt)) return false;
  return true;
}
static std::string bytes_of(const KeySwitch& W) { std::ostringstream os; W.writeTo(os); return os.str(); }
static uint64_t device_bytes(const Context& ctx) { uint64_t s[3]; check(hb_ctx_stats(ctx.handle(), s)); return s[2]; }

// one key set: what a user computes with it, from the same randomness
struct Run {
  Ctxt product, rotated;
};

int main(int argc, char** argv) {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  if (argc < 2) { std::printf("usage: %s seed_hex\n", argv[0]); return 1; }
  try {
    std::vector<uint8_t> seed;
    for (const char* h = argv[1]; h[0] && h[1]; h += 2) seed.push_back((uint8_t)std::stoul(std::string(h, 2), nullptr, 16));
    std::vector<uint8_t> seedRot = seed;
    seedRot[0] ^= 0x5a;

    const long m = 8192, p = 257, rot = 3;
    Context ctx(m, p, 1, /*bits=*/300, /*c=*/2);
    const long N = ctx.getPhiM();
    std::mt19937_64 gen(20261015);
    const double sigma = 3.2;
    const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
    DoubleCRT S(sample_ternary(gen, N), ctx, allq);
    DoubleCRT s2(S); s2 *= S;
    DoubleCRT sRot(S); sRot.automorph(rot);

    // expanded matrices: s^2 -> s and s(X^3) -> s, a_i from their seeds
    const KeySwitch W = genKeySWmatrix(ctx, s2, SKHandle(2, 1, 0), 0, S, p, false, sigma, gen, seed);
    const KeySwitch Wr = genKeySWmatrix(ctx, sRot, SKHandle(1, rot, 0), 0, S, p, false, sigma, gen, seedRot);

    // compressed copies: the seeded form holds no rows of a
    const uint64_t before = device_bytes(ctx);
    KeySwitch Wc = W, Wrc = Wr;
    const uint64_t copied = device_bytes(ctx);
    Wc.compress(); Wrc.compress();
    const uint64_t compressed = device_bytes(ctx);
    if (!Wc.a.empty() || !Wc.aSeeded || Wc.aSeeded->size() != W.a.size()) { std::printf("compress() kept the expanded a\n"); return 1; }
    if (!(compressed - before < (copied - before) / 2 + (copied - before) / 20)) {
      std::printf("compressed matrices hold %llu bytes, expanded %llu\n", (unsigned long long)(compressed - before), (unsigned long long)(copied - before));
      return 1;
    }
    std::printf("device bytes per matrix: expanded %llu, compressed %llu\n", (unsigned long long)((copied - before) / 2), (unsigned long long)((compressed - before) / 2));
    // a copy of a compressed matrix shares its seeded rows
    const KeySwitch Wcc = Wc;
    if (Wcc.aSeeded.get() != Wc.aSeeded.get()) { std::printf("copying a compressed KeySwitch copied its a\n"); return 1; }

    // writeTo: the same bytes for both forms; readFrom(..., false) builds the seeded form only
    if (bytes_of(Wc) != bytes_of(W) || bytes_of(Wrc) != bytes_of(Wr)) { std::printf("writeTo differs between the forms\n"); return 1; }
    KeySwitch R, Rr;
    { std::istringstream is(bytes_of(W)); R = KeySwitch::readFrom(is, ctx, false); }
    { std::istringstream is(bytes_of(Wr)); Rr = KeySwitch::readFrom(is, ctx, false); }
    if (!R.a.empty() || !R.aSeeded || bytes_of(R) != bytes_of(W)) { std::printf("readFrom(..., false) did not keep the seeded form\n"); return 1; }

    // compress() needs the seed
    {
      KeySwitch Wn = genKeySWmatrix(ctx, s2, SKHandle(2, 1, 0), 0, S, p, false, sigma, gen, [&](DoubleCRT& a) { a.randomize(seed); });
      bool threw = false;
      try { Wn.compress(); } catch (const InvalidArgument&) { threw = true; }
      if (!threw) { std::printf("compress() without a prgSeed did not throw\n"); return 1; }
    }

    std::vector<long> ma(N), mb(N);
    for (long k = 0; k < N; k++) { ma[k] = (long)(gen() % p); mb[k] = (long)(gen() % p); }
    std::vector<DoubleCRT> sKeys; sKeys.push_back(S);
    // the same encryptions, product and rotation under a given pair of matrices
    auto run = [&](const KeySwitch& relin, const KeySwitch& rotation) {
      KeyInfo pk; pk.context = &ctx; pk.ckks = false; pk.scale = 10.0; pk.hwt = 0;
      pk.skBound = pk.scale * std::sqrt(double(N) * 2.0 / 3.0);
      pk.keySwitching.push_back(relin);
      pk.keySwitching.push_back(rotation);
      pk.setKeySwitchMap(0);
      std::mt19937_64 g(777);
      Ctxt pubEncrKey(pk, p);
      pubEncrKey.primeSet = ctx.getCtxtPrimes();
      std::vector<long> e = sample_gauss(g, N, sigma);
      DoubleCRT c1 = random_rows(ctx, pubEncrKey.primeSet, g);
      DoubleCRT c0(e, ctx, pubEncrKey.primeSet); c0 *= p;
      DoubleCRT t(c1); t.Mul(S, false); c0 -= t;
      pubEncrKey.parts.emplace_back(c0, SKHandle());
      pubEncrKey.parts.emplace_back(c1, SKHandle(1, 1, 0));
      pubEncrKey.noiseBound = XD(double(p) * pk.noiseBoundForGaussian(sigma, N));
      auto encrypt = [&](const std::vector<long>& msg) {
        Ctxt c(pk, p);
        hb::EncryptionSample smp = hb::drawEncryptionSample(ctx, sigma, g);
        hb::Encrypt(c, pubEncrKey, msg, p, smp);
        return c;
      };
      Ctxt ca = encrypt(ma), cb = encrypt(mb);
      Ctxt fresh = ca;
      ca.multiplyBy(cb);
      BasicAutomorphPrecon pre(fresh);
      std::shared_ptr<Ctxt> r = pre.automorph(rot);
      std::vector<long> out;
      hb::Decrypt(out, ca, sKeys);
      std::vector<long> outRot;
      hb::Decrypt(outRot, *r, sKeys);
      return std::make_tuple(ca, *r, out, outRot);
    };
    auto ref = run(W, Wr);
    const std::vector<long>& out = std::get<2>(ref);
    for (long t = 0; t < 64; t++) {
      const long k = (t * 131 + 7) % N;
      long acc = 0;
      for (long i = 0; i < N; i++) { long j = k - i; long term = j >= 0 ? ma[i] * mb[j] : -(ma[i] * mb[j + N]); acc = (acc + term) % p; }
      if (out[k] != ((acc % p) + p) % p) { std::printf("product mismatch at %ld\n", k); return 1; }
    }
    // X -> X^3 maps coefficient i to 3i mod 2N with the sign of the wrap
    const std::vector<long>& outRot = std::get<3>(ref);
    for (long i = 0; i < N; i += 97) {
      const long j = (i * rot) % (2 * N);
      const long want = j < N ? ma[i] : (p - ma[i]) % p;
      if (outRot[j % N] != want) { std::printf("rotation mismatch at %ld\n", i); return 1; }
    }
    const struct { const char* name; const KeySwitch* relin; const KeySwitch* rotation; } forms[] = {
        {"compressed", &Wc, &Wrc}, {"copied compressed", &Wcc, &Wrc}, {"readFrom(..., false)", &R, &Rr}};
    for (const auto& f : forms) {
      auto got = run(*f.relin, *f.rotation);
      if (!same_ctxt(std::get<0>(got), std::get<0>(ref))) { std::printf("%s: product differs\n", f.name); return 1; }
      if (!same_ctxt(std::get<1>(got), std::get<1>(ref))) { std::printf("%s: hoisted rotation differs\n", f.name); return 1; }
      if (std::get<2>(got) != out || std::get<3>(got) != outRot) { std::printf("%s: decryption differs\n", f.name); return 1; }
    }
    std::printf("seeded keys OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
