// Key-switching matrices from a PRG seed through the C++ mirror: genKeySWmatrix(prgSeed) expands the a_i on the device
// (SetSeed + DoubleCRT::randomize, src/keys.cpp:1189-1206) and KeySwitch::writeTo / readFrom (src/keySwitching.cpp:195-240)
// store b + seed only; readFrom expands a again.
//   argv[1] = prgSeed as hex (little-endian magnitude bytes), argv[2] = a file holding NTL's key stream for that seed
//   (written by the Python oracle), fed to the byte-stream overload genKeySWmatrix(drawA).
// Checks: both overloads give the same a_i; writeTo -> readFrom -> writeTo reproduces the bytes and the re-expanded a;
// a product relinearised with the read-back matrix decrypts; truncated or corrupted records throw.
// Exit codes: 0 ok, 3 no CUDA device, 1 failure.
#include <cstdio>
#include <fstream>
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
static bool same_a(const KeySwitch& u, const KeySwitch& v) {
  if (u.a.size() != v.a.size()) return false;
  for (size_t i = 0; i < u.a.size(); i++) if (!same_rows(u.a[i], v.a[i])) return false;
  return true;
}
static std::string bytes_of(const KeySwitch& W) { std::ostringstream os; W.writeTo(os); return os.str(); }
static bool read_throws(const std::string& rec, const Context& ctx) {
  std::istringstream is(rec);
  try { KeySwitch::readFrom(is, ctx); } catch (const std::exception&) { return true; }
  return false;
}

int main(int argc, char** argv) {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  if (argc < 3) { std::printf("usage: %s seed_hex stream_file\n", argv[0]); return 1; }
  try {
    std::vector<uint8_t> seed;
    for (const char* h = argv[1]; h[0] && h[1]; h += 2) seed.push_back((uint8_t)std::stoul(std::string(h, 2), nullptr, 16));
    std::ifstream stream(argv[2], std::ios::binary);
    if (!stream) { std::printf("cannot open %s\n", argv[2]); return 1; }

    const long m = 8192, p = 257;
    Context ctx(m, p, 1, /*bits=*/300, /*c=*/2);
    const long N = ctx.getPhiM();
    std::mt19937_64 gen(20261015);
    const double sigma = 3.2;
    const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
    std::vector<long> s = sample_ternary(gen, N);
    DoubleCRT S(s, ctx, allq);
    DoubleCRT s2(S); s2 *= S;

    // ---- the seed overload against the byte-stream overload fed with NTL's stream for the same seed
    KeySwitch W = genKeySWmatrix(ctx, s2, SKHandle(2, 1, 0), 0, S, p, false, sigma, gen, seed);
    auto get = [&](unsigned char* b, long n) { stream.read(reinterpret_cast<char*>(b), n); if (!stream) throw RuntimeError("key stream file too short"); };
    KeySwitch Wb = genKeySWmatrix(ctx, s2, SKHandle(2, 1, 0), 0, S, p, false, sigma, gen, [&](DoubleCRT& a) { a.randomize(get); });
    if (W.a.size() != ctx.getDigits().size() || !same_a(W, Wb)) { std::printf("seeded a_i differ from the byte-stream a_i\n"); return 1; }
    { std::vector<uint8_t> t = seed; while (!t.empty() && t.back() == 0) t.pop_back(); if (W.prgSeed != t) { std::printf("prgSeed not kept\n"); return 1; } }
    { DoubleCRT a0(ctx, allq); a0.randomize(seed); if (!same_rows(a0, W.a[0])) { std::printf("DoubleCRT::randomize(seed) != a_0\n"); return 1; } }

    // ---- round trip
    const std::string rec = bytes_of(W);
    KeySwitch R;
    { std::istringstream is(rec); R = KeySwitch::readFrom(is, ctx); }
    if (bytes_of(R) != rec) { std::printf("writeTo(readFrom(writeTo(W))) differs\n"); return 1; }
    if (!same_a(R, W)) { std::printf("re-expanded a differs\n"); return 1; }
    if (!(R.fromKey == W.fromKey) || R.toKeyID != W.toKeyID || R.ptxtSpace != W.ptxtSpace || R.b.size() != W.b.size()) { std::printf("fields differ\n"); return 1; }
    if (std::fabs(R.noiseBound.ln() - W.noiseBound.ln()) > 1e-12) { std::printf("noiseBound differs\n"); return 1; }

    // ---- truncated and corrupted records
    for (size_t cut : {(size_t)0, (size_t)3, (size_t)30, rec.size() / 2, rec.size() - 30, rec.size() - 1})
      if (!read_throws(rec.substr(0, cut), ctx)) { std::printf("truncated record (%zu bytes) accepted\n", cut); return 1; }
    const size_t seed_field = rec.size() - 4 - 16 - W.prgSeed.size() - 8;   // int64 byte count of the seed
    auto patched = [&](size_t off, int64_t v) { std::string r = rec; std::memcpy(&r[off], &v, 8); return r; };
    { std::string r = rec; r[0] = 'X'; if (!read_throws(r, ctx)) { std::printf("bad leading eye catcher accepted\n"); return 1; } }
    { std::string r = rec; r[r.size() - 1] = 'X'; if (!read_throws(r, ctx)) { std::printf("bad trailing eye catcher accepted\n"); return 1; } }
    if (!read_throws(patched(seed_field, 0), ctx)) { std::printf("zero seed length accepted\n"); return 1; }
    if (!read_throws(patched(seed_field, -5), ctx)) { std::printf("negative seed length accepted\n"); return 1; }
    if (!read_throws(patched(seed_field, (int64_t)1 << 40), ctx)) { std::printf("huge seed length accepted\n"); return 1; }
    if (!read_throws(patched(4 + 5 * 8, (int64_t)W.b.size() + 1), ctx)) { std::printf("wrong b count accepted\n"); return 1; }
    if (!read_throws(patched(4 + 5 * 8, 0), ctx)) { std::printf("zero b count accepted\n"); return 1; }

    // ---- a product relinearised with the read-back matrix decrypts to the product
    KeyInfo pk; pk.context = &ctx; pk.ckks = false; pk.scale = 10.0; pk.hwt = 0;
    pk.skBound = pk.scale * std::sqrt(double(N) * 2.0 / 3.0);
    pk.keySwitching.push_back(std::move(R));
    pk.setKeySwitchMap(0);
    Ctxt pubEncrKey(pk, p);
    {
      pubEncrKey.primeSet = ctx.getCtxtPrimes();
      std::vector<long> e = sample_gauss(gen, N, sigma);
      DoubleCRT c1 = random_rows(ctx, pubEncrKey.primeSet, gen);
      DoubleCRT c0(e, ctx, pubEncrKey.primeSet); c0 *= p;
      DoubleCRT t(c1); t.Mul(S, false); c0 -= t;
      pubEncrKey.parts.emplace_back(c0, SKHandle());
      pubEncrKey.parts.emplace_back(c1, SKHandle(1, 1, 0));
      pubEncrKey.noiseBound = XD(double(p) * pk.noiseBoundForGaussian(sigma, N));
    }
    std::vector<DoubleCRT> sKeys; sKeys.push_back(S);
    auto encrypt = [&](const std::vector<long>& msg) {
      Ctxt c(pk, p);
      hb::EncryptionSample smp = hb::drawEncryptionSample(ctx, sigma, gen);
      hb::Encrypt(c, pubEncrKey, msg, p, smp);
      return c;
    };
    std::vector<long> ma(N), mb(N);
    for (long k = 0; k < N; k++) { ma[k] = (long)(gen() % p); mb[k] = (long)(gen() % p); }
    Ctxt ca = encrypt(ma), cb = encrypt(mb);
    ca.multiplyBy(cb);
    if (ca.parts.size() != 2) { std::printf("not relinearised\n"); return 1; }
    std::vector<long> out;
    hb::Decrypt(out, ca, sKeys);
    for (long t = 0; t < 64; t++) {
      const long k = (t * 131 + 7) % N;
      long acc = 0;
      for (long i = 0; i < N; i++) { long j = k - i; long term = j >= 0 ? ma[i] * mb[j] : -(ma[i] * mb[j + N]); acc = (acc + term) % p; }
      if (out[k] != ((acc % p) + p) % p) { std::printf("product mismatch at %ld\n", k); return 1; }
    }
    std::printf("keyswitch io OK\n");
    return 0;
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 1;
  }
}
