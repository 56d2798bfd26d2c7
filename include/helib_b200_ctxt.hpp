// helib_b200_ctxt.hpp -- header-only C++17 mirror of the hot subset of helib::Ctxt over hb::DoubleCRT.
//
// Host orchestration stays on the host exactly as in the reference (SURVEY.md section 8a rows 15-17):
// noise estimates in extended-range floating point, the choice of the prime set for a product
// (computeIntervalForMul + ModuliSizes::getSet4Size), when to mod-switch and when to key-switch.  Every data
// operation goes to the engine through hb::DoubleCRT.  Method names, argument meaning and failure behaviour
// follow the reference (citations: paths in the HElib tree):
//   SKHandle::mul                  include/helib/Ctxt.h:155-185
//   modUpToSet / bringToSet        src/Ctxt.cpp:346-389
//   modDownToSet                   src/Ctxt.cpp:393-562      (added noise from the device-computed ||delta/P||)
//   dropSmallAndSpecialPrimes      src/Ctxt.cpp:589-662
//   relin_CKKS_adjust              src/Ctxt.cpp:664-716
//   reLinearize / keySwitchPart    src/Ctxt.cpp:720-842
//   keySwitchDigits                src/Ctxt.cpp:191-230
//   tensorProduct                  src/Ctxt.cpp:1563-1608
//   computeIntervalForMul          src/Ctxt.cpp:1610-1656
//   multLowLvl / multiplyBy        src/Ctxt.cpp:1681-1774
//   modSwitchAddedNoiseBound       src/Ctxt.cpp:2560-2582
//   polyEval / DynamicCtxtPowers   src/polyEval.cpp:18-29, 129-389   (every simplePolyEval leaf in one hb_ctxt_scaled_sums call)
//   divideByP / multByP            src/Ctxt.cpp:2415-2435, include/helib/Ctxt.h:1216-1221
//   extractDigits / extendExtract  src/extractDigits.cpp:28-308       (each round's subtract-and-divide chain in one call)
//   extractDigitsThin              src/recryption.cpp:793-909        (its final combination in one call)
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <complex>
#include <functional>
#include <memory>
#include <numeric>
#include <random>
#include <string>
#include <ostream>
#include <istream>
#include <cstring>
#include <type_traits>

#include "helib_b200_doublecrt.hpp"

namespace hb {

// NTL::xdouble stand-in: value = m * 2^e, enough range for noise bounds of 2^2000 and beyond.
struct XD {
  double m = 0; long e = 0;
  XD() = default;
  XD(double v) { int ex = 0; m = std::frexp(v, &ex); e = ex; }
  static XD make(double m_, long e_) { XD r; int ex = 0; r.m = std::frexp(m_, &ex); r.e = e_ + ex; if (r.m == 0) r.e = 0; return r; }
  static XD exp(double lnv) {
    if (!(lnv > -1e300)) return XD();   // ln 0 = -inf (the engine's answer for a zero polynomial) or ln() of a zero XD
    double l2 = lnv / std::log(2.0); long fl = (long)std::floor(l2); return make(std::exp2(l2 - fl), fl);
  }
  double ln() const { return m <= 0 ? -DBL_MAX : std::log(m) + e * std::log(2.0); }
  double to_double() const { return std::ldexp(m, (int)std::max(-2000L, std::min(2000L, e))); }
  XD operator*(const XD& o) const { return make(m * o.m, e + o.e); }
  XD operator/(const XD& o) const { return make(m / o.m, e - o.e); }
  XD operator+(const XD& o) const {
    if (m == 0) return o;
    if (o.m == 0) return *this;
    if (e >= o.e) { long d = e - o.e; return d > 1100 ? *this : make(m + std::ldexp(o.m, (int)-d), e); }
    return o + *this;
  }
  XD operator-() const { XD r = *this; r.m = -r.m; return r; }
  XD operator-(const XD& o) const { return *this + (-o); }
  XD abs() const { XD r = *this; r.m = std::fabs(r.m); return r; }
  // exact integer value floor(v) of a non-negative XD as mant * 2^shift (mant < 2^63)
  void floorParts(uint64_t& mant, long& shift) const {
    if (m <= 0 || e <= 0) { mant = 0; shift = 0; return; }
    if (e <= 62) { mant = (uint64_t)std::floor(std::ldexp(m, (int)e)); shift = 0; return; }
    mant = (uint64_t)std::ldexp(m, 53); shift = e - 53;      // 53-bit mantissa: already an integer
  }
  bool operator<(const XD& o) const { if (m <= 0 || o.m <= 0) return m < o.m; return e != o.e ? e < o.e : m < o.m; }
  bool operator>(const XD& o) const { return o < *this; }
  bool operator<=(const XD& o) const { return !(o < *this); }
};

// include/helib/Ctxt.h:82-260
struct SKHandle {
  long powerOfS = 0, powerOfX = 1, secretKeyID = 0;
  SKHandle() = default;
  SKHandle(long s, long x, long id) : powerOfS(s), powerOfX(x), secretKeyID(id) {}
  bool isOne() const { return powerOfS == 0; }
  bool isBase(long id = 0) const { return powerOfS == 1 && powerOfX == 1 && (id < 0 || secretKeyID == id); }
  bool operator==(const SKHandle& o) const { return powerOfS == o.powerOfS && powerOfX == o.powerOfX && secretKeyID == o.secretKeyID; }
  bool mul(const SKHandle& a, const SKHandle& b) {   // include/helib/Ctxt.h:155-185
    if (a.isOne()) { *this = b; return b.secretKeyID >= 0; }
    if (b.isOne()) { *this = a; return a.secretKeyID >= 0; }
    if (a.secretKeyID == -1 || b.secretKeyID == -1 || a.secretKeyID != b.secretKeyID || a.powerOfX != b.powerOfX) { secretKeyID = -1; return false; }
    secretKeyID = a.secretKeyID; powerOfX = a.powerOfX; powerOfS = a.powerOfS + b.powerOfS;
    return true;
  }
};

struct CtxtPart {
  DoubleCRT dcrt;
  SKHandle skHandle;
  CtxtPart(const DoubleCRT& d, const SKHandle& h) : dcrt(d), skHandle(h) {}
  CtxtPart(const Context& ctx, const IndexSet& s, const SKHandle& h) : dcrt(ctx, s), skHandle(h) {}   // rows to be written
};

// The a_i of a key-switching matrix held as HElib holds them: the seed and its row schedule over ctxt | special
// (hb_poly_create_seeded), no rows.  Every key switch that reads them regenerates the rows it needs on the device.
// Immutable; KeySwitch shares it, so copying a compressed matrix copies a pointer.
class SeededRows {
  std::vector<hb_poly*> h_;
 public:
  SeededRows(const Context& context, const std::vector<uint8_t>& seed, size_t n) : h_(n, nullptr) {
    const auto idx = (context.getCtxtPrimes() | context.getSpecialPrimes()).vec();
    if (n) check(hb_poly_create_seeded(context.handle(), (int)n, idx.data(), (int)idx.size(), seed.data(), (int)seed.size(), h_.data()));
  }
  ~SeededRows() { for (hb_poly* p : h_) if (p) hb_poly_destroy(p); }
  SeededRows(const SeededRows&) = delete;
  SeededRows& operator=(const SeededRows&) = delete;
  size_t size() const { return h_.size(); }
  hb_poly* handle(size_t i) const { return h_.at(i); }
};

// helib::KeySwitch (include/helib/keySwitching.h:86-100).  prgSeed holds the NumBytes little-endian magnitude bytes of the
// reference's ZZ prgSeed (empty when a came from another source).  a is held in one of two forms:
//  - expanded: the rows of a_i in `a` (genKeySWmatrix, readFrom(..., true));
//  - seeded: `aSeeded` only, as HElib keeps it (compress(), readFrom(..., false)); half the device memory of the expanded form.
struct KeySwitch {
  SKHandle fromKey; long toKeyID = 0; long ptxtSpace = 0;
  std::vector<DoubleCRT> a, b;
  std::shared_ptr<const SeededRows> aSeeded;
  std::vector<uint8_t> prgSeed;
  XD noiseBound;
  // the handle of a_i for the key-switching entry points, from either form
  hb_poly* aHandle(size_t i) const { return aSeeded ? aSeeded->handle(i) : a.at(i).handle(); }
  // drop the expanded a and keep the seed form; needs prgSeed (InvalidArgument otherwise)
  void compress() {
    if (aSeeded) return;
    if (prgSeed.empty()) throw InvalidArgument("KeySwitch::compress: no prgSeed to regenerate a from");
    if (b.empty()) throw InvalidArgument("KeySwitch::compress: empty matrix");
    aSeeded = std::make_shared<const SeededRows>(b[0].getContext(), prgSeed, b.size());
    a.clear();
  }
  // KeySwitch::writeTo / readFrom (src/keySwitching.cpp:195-240), defined after Ctxt (they share its field writers).
  // expandA = false builds the seeded form and never allocates the rows of a.
  void writeTo(std::ostream& str) const;
  static KeySwitch readFrom(std::istream& str, const Context& context, bool expandA = true);
};

// a_0 .. a_{n-1} of W from W.prgSeed over ctxt | special: SetSeed(prgSeed); a[i].randomize() (src/keys.cpp:1199-1206),
// one device call for all of them
inline void expandKeySWmatrixA(KeySwitch& W, const Context& context, size_t n) {
  const IndexSet all = context.getCtxtPrimes() | context.getSpecialPrimes();
  W.a.clear();
  for (size_t i = 0; i < n; i++) W.a.emplace_back(context, all);
  std::vector<hb_poly*> ap;
  for (auto& x : W.a) ap.push_back(x.handle());
  auto idx = all.vec();
  if (n && !idx.empty()) check(hb_poly_randomize(ap.data(), (int)n, idx.data(), (int)idx.size(), W.prgSeed.data(), (int)W.prgSeed.size()));
}

// the part of helib::PubKey / Context the ciphertext logic consults
struct KeyInfo {
  const Context* context;
  bool ckks = false;
  double scale = 10.0;           // Context::scale (include/helib/Context.h:151)
  long hwt = 0;                  // Context::getHwt()
  double skBound = 0;            // PubKey::getSKeyBound (src/keys.cpp:280)
  std::vector<KeySwitch> keySwitching;
  const KeySwitch* getKeySWmatrix(const SKHandle& from, long toID) const {
    for (auto& w : keySwitching) if (w.fromKey == from && w.toKeyID == toID) return &w;
    return nullptr;
  }
  // PubKey::setKeySwitchMap / getNextKSWmatrix / isReachable (src/keys.cpp:122-172,310-319): BFS from 1 over the
  // automorphism matrices W[s(X^n) -> s(X)]; map[k] = matrix of the first step towards k
  std::vector<std::vector<long>> keySwitchMap;
  void setKeySwitchMap(long keyId = 0) {
    const long m = context->getM();
    std::vector<std::pair<long, long>> edges;
    for (size_t i = 0; i < keySwitching.size(); i++) {
      const KeySwitch& mat = keySwitching[i];
      if (mat.toKeyID == keyId && mat.fromKey.powerOfS == 1 && mat.fromKey.secretKeyID == keyId) edges.emplace_back(mat.fromKey.powerOfX, (long)i);
    }
    if (keyId >= (long)keySwitchMap.size()) keySwitchMap.resize(keyId + 1);
    keySwitchMap[keyId].assign((size_t)m, -1);
    std::vector<long> queue{1};
    for (size_t h = 0; h < queue.size(); h++)
      for (auto& e : edges) {
        long next = (long)(((unsigned __int128)(unsigned long)queue[h] * (unsigned long)e.first) % (unsigned long)m);
        if (keySwitchMap[keyId][next] == -1) { keySwitchMap[keyId][next] = e.second; queue.push_back(next); }
      }
  }
  bool isReachable(long k, long keyID) const { return keyID < (long)keySwitchMap.size() && keySwitchMap[keyID].at((size_t)k) >= 0; }
  const KeySwitch* getNextKSWmatrix(long fromXPower, long fromID) const {
    long i = keySwitchMap.at((size_t)fromID).at((size_t)fromXPower);
    return i >= 0 ? &keySwitching[(size_t)i] : nullptr;
  }
  double noiseBoundForUniform(double mag, long deg) const { return scale * std::sqrt(double(deg) / 3.0) * mag; }   // include/helib/Context.h:475-478
  double noiseBoundForMod(long modulus, long deg) const {   // include/helib/Context.h:517-524
    double var = double(modulus) * double(modulus) / 12.0; if (modulus % 2 == 0) var += 1.0 / 6.0;
    return scale * std::sqrt(deg * var);
  }
  double noiseBoundForGaussian(double sigma, long deg) const { return scale * std::sqrt(double(deg)) * sigma; }   // include/helib/Context.h:541-544
  double logOfProduct(const IndexSet& s) const { double x = 0; for (long i : s) x += std::log((double)context->ithPrime(i)); return x; }
};

class Ctxt {
 public:
  const KeyInfo& pubKey;
  const Context& context;
  std::vector<CtxtPart> parts;
  IndexSet primeSet;
  long ptxtSpace;
  XD noiseBound;
  long intFactor = 1;
  XD ratFactor = XD(1.0), ptxtMag = XD(1.0);
  static constexpr double safety = 0.6931471805599453;   // log 2, top of src/Ctxt.cpp

  Ctxt(const KeyInfo& pk, long ptxtSp) : pubKey(pk), context(*pk.context), ptxtSpace(ptxtSp), noiseBound(0.0) {}
  Ctxt& operator=(const Ctxt& o) {
    parts = o.parts; primeSet = o.primeSet; ptxtSpace = o.ptxtSpace; noiseBound = o.noiseBound;
    intFactor = o.intFactor; ratFactor = o.ratFactor; ptxtMag = o.ptxtMag;
    if (o.lastKSNoiseRatio != 0) lastKSNoiseRatio = o.lastKSNoiseRatio;
    if (o.lastModSwitchRatio != 0) lastModSwitchRatio = o.lastModSwitchRatio;
    return *this;
  }
  Ctxt(const Ctxt&) = default;
  bool isCKKS() const { return pubKey.ckks; }
  bool isEmpty() const { return parts.empty(); }
  double logOfPrimeSet() const { return pubKey.logOfProduct(primeSet); }
  long getPartIndexByHandle(const SKHandle& h) const { for (size_t i = 0; i < parts.size(); i++) if (parts[i].skHandle == h) return (long)i; return -1; }
  bool inCanonicalForm(long keyID = 0) const {
    if (parts.size() > 2) return false;
    if (parts.size() > 0 && !parts[0].skHandle.isOne()) return false;
    if (parts.size() > 1 && !parts[1].skHandle.isBase(keyID)) return false;
    return true;
  }
  XD totalNoiseBound() const { return isCKKS() ? ptxtMag * ratFactor + noiseBound : noiseBound; }   // include/helib/Ctxt.h:1358-1364
  // src/Ctxt.cpp:116-127; polyNormBnd = 1 for power-of-two m (PAlgebra::getPolyNormBnd), else supplied by the caller
  bool isCorrect(double polyNormBnd = 1.0) const { return (totalNoiseBound() * XD(polyNormBnd)).ln() <= std::log(0.48) + logOfPrimeSet(); }
  bool verifyPrimeSet() const {   // src/Ctxt.cpp:177-186
    IndexSet s = primeSet & context.getSpecialPrimes();
    if (!empty(s) && s != context.getSpecialPrimes()) return false;
    return (primeSet & context.getCtxtPrimes()).isInterval();
  }
  XD modSwitchAddedNoiseBound() const {   // src/Ctxt.cpp:2560-2582
    XD added(0.0);
    for (auto& part : parts) {
      if (part.skHandle.isOne()) added = added + XD(1.0);
      else added = added + XD::exp(part.skHandle.powerOfS * std::log(pubKey.skBound));
    }
    return added * XD(pubKey.noiseBoundForUniform(double(ptxtSpace) / 2.0, context.getPhiM()));
  }

  void modUpToSet(const IndexSet& s) {   // src/Ctxt.cpp:346-371
    IndexSet setDiff = s / primeSet;
    if (empty(setDiff)) return;
    double f = 0;
    for (auto& part : parts) f = part.dcrt.addPrimesAndScale(setDiff);
    noiseBound = noiseBound * XD::exp(f);
    ratFactor = ratFactor * XD::exp(f);
    primeSet.insert(setDiff);
    if (!verifyPrimeSet()) throw LogicError("primeSet is no longer valid");
  }
  void modDownToSet(const IndexSet& s) {   // src/Ctxt.cpp:393-562 ("real mod switching" branch)
    HB_TIMER_START(context.handle());
    IndexSet intersection = primeSet & s;
    if (empty(intersection)) throw RuntimeError("modDownToSet called with a disjoint set");
    IndexSet setDiff = primeSet / intersection;
    if (empty(setDiff)) return;
    std::vector<double> norms;
    for (auto& part : parts) norms.push_back(part.dcrt.scaleDownToSetNorm(intersection, ptxtSpace));   // ||delta/P||_canon, computed on the device
    modDownToSetMeta(setDiff, norms.data());
  }
  // the metadata half of modDownToSet: setDiff dropped, with norms[j] = ||delta/P||_canon of parts[j] (the rows are already
  // scaled down; the parts' handles are what the added noise depends on)
  void modDownToSetMeta(const IndexSet& setDiff, const double* norms) {
    XD addedNoiseBound = modSwitchAddedNoiseBound();
    XD addedNoise(0.0);
    for (size_t j = 0; j < parts.size(); j++) {
      const CtxtPart& part = parts[j];
      if (part.skHandle.isOne()) addedNoise = addedNoise + XD(norms[j]);
      else addedNoise = addedNoise + XD(norms[j]) * XD::exp(part.skHandle.powerOfS * std::log(pubKey.skBound));
    }
    XD f = XD::exp(pubKey.logOfProduct(setDiff));
    ratFactor = ratFactor / f;
    noiseBound = noiseBound / f;
    noiseBound = noiseBound + addedNoise;
    lastModSwitchRatio = (addedNoise / addedNoiseBound).to_double();   // the reference's "mod-switch-added-noise" statistic
    HB_STATS_UPDATE("mod-switch-added-noise", lastModSwitchRatio);      // src/Ctxt.cpp:537
    primeSet.remove(setDiff);
    if (!verifyPrimeSet()) throw LogicError("primeSet is no longer valid");
  }
  void bringToSet(const IndexSet& s) {   // src/Ctxt.cpp:373-389
    if (empty(s)) { IndexSet tmp(context.getCtxtPrimes().first()); modUpToSet(tmp); modDownToSet(tmp); }
    else { modUpToSet(s); modDownToSet(s); }
  }
  void dropSmallAndSpecialPrimes() {   // src/Ctxt.cpp:589-662
    if (primeSet.disjointFrom(context.getSmallPrimes())) { modDownToSet(context.getCtxtPrimes()); return; }
    IndexSet target = primeSet & context.getCtxtPrimes();
    IndexSet dropping = primeSet / target;
    double log_dropping = pubKey.logOfProduct(dropping);
    double log_modswitch_noise = modSwitchAddedNoiseBound().ln();
    double log_noise = noiseBound.m <= 0 ? -DBL_MAX : noiseBound.ln();
    double log_compensation = 0;
    log_modswitch_noise += 3 * std::log(2.0);
    if (log_noise - log_dropping + log_compensation < log_modswitch_noise) {
      IndexSet candidates = context.getCtxtPrimes() / target;
      for (long i : candidates) {
        target.insert(i);
        log_compensation += std::log((double)context.ithPrime(i));
        if (log_noise - log_dropping + log_compensation >= log_modswitch_noise) break;
      }
    }
    bringToSet(target);
  }
  void relin_CKKS_adjust() {   // src/Ctxt.cpp:664-716
    if (!isCKKS()) return;
    long phim = context.getPhiM();
    double h = pubKey.hwt == 0 ? phim / 2.0 : (double)pubKey.hwt;
    double log_phim = std::max(1.0, std::log((double)phim));
    double beta = pubKey.scale * std::sqrt(phim * log_phim * h / 12.0);
    double gamma = beta * 8;
    if (XD(gamma) > noiseBound) {
      long xf = (long)std::ceil(gamma / noiseBound.to_double());
      for (auto& part : parts) part.dcrt *= xf;
      noiseBound = noiseBound * XD((double)xf);
      ratFactor = ratFactor * XD((double)xf);
    }
  }
  void addPart(const DoubleCRT& part, const SKHandle& handle, bool negative = false) {   // src/Ctxt.cpp:851-893 (matchPrimeSet)
    if (!(primeSet <= part.getIndexSet())) throw RuntimeError("Ctxt::addPart: ctxt has primes not in part");
    long j = getPartIndexByHandle(handle);
    if (j >= 0) { if (negative) parts[j].dcrt.Sub(part, /*matchIndexSets=*/false); else parts[j].dcrt.Add(part, /*matchIndexSets=*/false); }
    else {
      parts.emplace_back(part, handle);
      if (part.getIndexSet() != primeSet) parts.back().dcrt.removePrimes(part.getIndexSet() / primeSet);
      if (negative) parts.back().dcrt.Negate();
    }
  }
  // src/Ctxt.cpp:191-230 -- the two products per digit and their accumulation run as ONE engine launch
  void keySwitchDigits(const KeySwitch& W, std::vector<DoubleCRT>& digits) {
    HB_NTIMER_START(KS_loop, context.handle());   // src/Ctxt.cpp:205
    long j0 = getPartIndexByHandle(SKHandle()), j1 = getPartIndexByHandle(SKHandle(1, 1, W.toKeyID));
    if (j0 < 0) { parts.emplace_back(DoubleCRT(context, primeSet), SKHandle()); j0 = (long)parts.size() - 1; }
    if (j1 < 0) { parts.emplace_back(DoubleCRT(context, primeSet), SKHandle(1, 1, W.toKeyID)); j1 = (long)parts.size() - 1; }
    std::vector<hb_poly*> dg, ea, eb;
    for (size_t i = 0; i < digits.size(); i++) { dg.push_back(digits[i].handle()); ea.push_back(W.aHandle(i)); eb.push_back(W.b[i].handle()); }
    hb_poly* o0[1] = {parts[j0].dcrt.handle()}; hb_poly* o1[1] = {parts[j1].dcrt.handle()};
    auto idx = primeSet.vec();
    check(hb_keyswitch_digits(dg.data(), (int)digits.size(), (int)digits.size(), 1, idx.data(), (int)idx.size(), ea.data(), eb.data(), o0, o1));
  }
  void keySwitchPart(const CtxtPart& p, const KeySwitch& W) {   // src/Ctxt.cpp:805-842
    HB_TIMER_START(context.handle());
    if (!context.getSpecialPrimes().disjointFrom(p.dcrt.getIndexSet())) throw LogicError("Special primes and CtxtPart's index set have non-empty intersection");
    if (p.skHandle.isOne() || p.skHandle.isBase(W.toKeyID)) {
      CtxtPart pp = p;
      pp.dcrt.addPrimesAndScale(context.getSpecialPrimes());
      addPart(pp.dcrt, pp.skHandle);
      return;
    }
    if (!(W.fromKey == p.skHandle)) throw LogicError("Secret key handles do not match");
    std::vector<DoubleCRT> polyDigits;
    XD addedNoise(0.0);
    for (double ln : p.dcrt.breakIntoDigitsLogNorms(polyDigits)) addedNoise = addedNoise + XD::exp(ln);   // sum of ||E_i||, computed on the device
    addedNoise = addedNoise * W.noiseBound;
    keySwitchDigits(W, polyDigits);
    lastKSNoiseRatio = (addedNoise / noiseBound).to_double();   // "KS-noise-ratio"
    HB_STATS_UPDATE("KS-noise-ratio", lastKSNoiseRatio);         // src/Ctxt.cpp:835
    noiseBound = noiseBound + addedNoise;
  }
  void reLinearize(long keyID = 0) {   // src/Ctxt.cpp:720-786
    HB_TIMER_START(context.handle());
    if (isEmpty() || inCanonicalForm(keyID)) return;
    dropSmallAndSpecialPrimes();
    relin_CKKS_adjust();
    long g = ptxtSpace;
    double logProd = pubKey.logOfProduct(context.getSpecialPrimes());
    Ctxt tmp(pubKey, ptxtSpace);
    tmp.intFactor = intFactor; tmp.ptxtMag = ptxtMag;
    tmp.noiseBound = noiseBound * XD::exp(logProd);
    tmp.primeSet = primeSet | context.getSpecialPrimes();
    tmp.ratFactor = ratFactor * XD::exp(logProd);
    for (CtxtPart& part : parts) {
      if (part.skHandle.isOne() || part.skHandle.isBase(keyID)) {
        part.dcrt.addPrimesAndScale(context.getSpecialPrimes());
        tmp.addPart(part.dcrt, part.skHandle);
        continue;
      }
      const KeySwitch* W = pubKey.getKeySWmatrix(part.skHandle, keyID);
      if (!W) throw LogicError("No key-switching matrix exists");
      if (g > 1) { tmp.reducePtxtSpace(W->ptxtSpace); g = tmp.ptxtSpace; }   // g == 1 for CKKS (src/Ctxt.cpp:771-775)
      tmp.keySwitchPart(part, *W);
    }
    *this = tmp;
  }
  void tensorProduct(const Ctxt& c1, const Ctxt& c2) {   // src/Ctxt.cpp:1563-1608
    HB_TIMER_START(context.handle());
    parts.clear();
    primeSet = c1.primeSet;
    long ptxtSp = c1.ptxtSpace;
    if (ptxtSp > 2) {
      unsigned long q = 1;
      for (long i : c1.primeSet) q = (unsigned long)(((unsigned __int128)q * (unsigned long)(context.ithPrime(i) % ptxtSp)) % (unsigned long)ptxtSp);
      intFactor = (long)(((unsigned __int128)c1.intFactor * c2.intFactor) % ptxtSp);
      intFactor = (long)(((unsigned __int128)intFactor * q) % ptxtSp);
    }
    for (auto& p1 : c1.parts)
      for (auto& p2 : c2.parts) {
        CtxtPart tmpPart = p2;
        if (!tmpPart.skHandle.mul(p1.skHandle, tmpPart.skHandle)) throw LogicError("Ctxt::tensorProduct: cannot multiply secret-key handles");
        tmpPart.dcrt *= p1.dcrt;
        long k = getPartIndexByHandle(tmpPart.skHandle);
        if (k >= 0) parts[k].dcrt += tmpPart.dcrt;
        else parts.push_back(tmpPart);
      }
    if (isCKKS()) {
      noiseBound = c1.noiseBound * c2.ptxtMag * c2.ratFactor + c2.noiseBound * c1.ptxtMag * c1.ratFactor + c1.noiseBound * c2.noiseBound;
      ratFactor = c1.ratFactor * c2.ratFactor;
      ptxtMag = c1.ptxtMag * c2.ptxtMag;
    } else noiseBound = c1.noiseBound * c2.noiseBound;
  }
  static void computeIntervalForMul(double& lo, double& hi, const Ctxt& c1, const Ctxt& c2) {   // src/Ctxt.cpp:1610-1656
    const double slack = 4 * std::log(2.0);
    double cap1 = c1.logOfPrimeSet() - std::max(c1.noiseBound, XD(1.0)).ln();
    double cap2 = c2.logOfPrimeSet() - std::max(c2.noiseBound, XD(1.0)).ln();
    double adn1 = c1.modSwitchAddedNoiseBound().ln(), adn2 = c2.modSwitchAddedNoiseBound().ln();
    if (c1.isCKKS()) { lo = std::max(cap1 + adn1, cap2 + adn2) + safety; hi = lo + slack; }
    else { hi = std::min(cap1 + adn1, cap2 + adn2) - safety; lo = hi - slack; }
  }
  // capacity (include/helib/Ctxt.h:1314-1319): log2 of the modulus over the total noise bound
  double capacity() const { return (logOfPrimeSet() - std::max(totalNoiseBound(), XD(1.0)).ln()) / std::log(2.0); }
  // naturalPrimeSet (src/Ctxt.cpp:1673-1678): getSet4Size's one-set form on computeIntervalForSqr's interval
  IndexSet naturalPrimeSet() const {
    double lo, hi;
    computeIntervalForMul(lo, hi, *this, *this);   // computeIntervalForSqr (src/Ctxt.cpp:1658-1661)
    auto f1 = primeSet.vec();
    std::vector<int32_t> out(context.numPrimes()); int nout = 0;
    check(hb_chain_set4size(context.chain(), lo, hi, f1.data(), (int)f1.size(), nullptr, 0, isCKKS() ? 1 : 0, out.data(), &nout));
    return IndexSet(out.begin(), out.begin() + nout);
  }
  // multLowLvl(*this) (src/Ctxt.cpp:1704-1708, 1748-1751) as one hb_square_tensor_norm call: a 2-part canonical ciphertext
  // under one key whose natural set needs no mod-up (bringToSet is then modDownToSet alone).  modDownToSet's metadata is
  // replayed from the returned norms and tensorProduct's from the metadata of the brought-down operand.  Returns false, with
  // nothing changed, where the call cannot reproduce the branch.
  bool squareFused() {
    const long keyID = getKeyID();
    if (parts.size() != 2 || !inCanonicalForm(keyID)) return false;
    const IndexSet nat = naturalPrimeSet();
    if (empty(nat) || !(nat <= primeSet)) return false;   // bringToSet would mod up first
    const IndexSet setDiff = primeSet / nat;
    auto Sin = primeSet.vec(), Sv = nat.vec();
    DoubleCRT o2(context, nat);
    hb_poly* a0[1] = {parts[0].dcrt.handle()}; hb_poly* a1[1] = {parts[1].dcrt.handle()}; hb_poly* p2[1] = {o2.handle()};
    double norms[2] = {0.0, 0.0};
    check(hb_square_tensor_norm(a0, a1, p2, 1, Sin.data(), (int)Sin.size(), Sv.data(), (int)Sv.size(), (uint64_t)ptxtSpace, norms));
    for (auto& part : parts) part.dcrt.removePrimes(setDiff);
    if (!empty(setDiff)) modDownToSetMeta(setDiff, norms);   // bringToSet(nat) (src/Ctxt.cpp:373-389)
    Ctxt x(pubKey, ptxtSpace);   // tensorProduct(*this, *this)'s metadata (its part loop has nothing to do on metadata only)
    x.primeSet = primeSet; x.noiseBound = noiseBound; x.intFactor = intFactor; x.ratFactor = ratFactor; x.ptxtMag = ptxtMag;
    Ctxt t(pubKey, ptxtSpace);
    t.tensorProduct(x, x);
    primeSet = t.primeSet; noiseBound = t.noiseBound; intFactor = t.intFactor; ratFactor = t.ratFactor; ptxtMag = t.ptxtMag;
    SKHandle s2; s2.mul(parts[1].skHandle, parts[1].skHandle);
    parts.emplace_back(o2, s2);
    return true;
  }
  void multLowLvl(const Ctxt& other_orig) {   // src/Ctxt.cpp:1681-1753 (non-destructive)
    HB_TIMER_START(context.handle());
    if (isEmpty()) return;
    if (other_orig.isEmpty()) { *this = other_orig; return; }
    if (isCKKS() != other_orig.isCKKS()) throw LogicError("Scheme mismatch");
    if (&context != &other_orig.context) throw LogicError("Context mismatch");
    if (&pubKey != &other_orig.pubKey) throw LogicError("Public key mismatch");
    if (isCKKS() && (ptxtSpace != 1 || other_orig.ptxtSpace != 1)) throw LogicError("Plaintext spaces incompatible");
    if (this == &other_orig) {   // squaring: drop to the "natural" primeSet (src/Ctxt.cpp:1704-1706)
      if (squareFused()) return;
      bringToSet(naturalPrimeSet());
      Ctxt tmp(pubKey, ptxtSpace);
      tmp.tensorProduct(*this, *this);
      *this = tmp;
      return;
    }
    Ctxt other = other_orig;
    bringToCommonSet(other);
    Ctxt tmp(pubKey, ptxtSpace);
    tmp.tensorProduct(*this, other);
    *this = tmp;
  }
  // multLowLvl's preparation of the two operands (src/Ctxt.cpp:1717-1747): equal plaintext spaces, then both brought to the
  // common prime set that getSet4Size picks for the product
  void bringToCommonSet(Ctxt& other) {
    if (!isCKKS()) {   // equalize plaintext spaces (src/Ctxt.cpp:1717-1725); reducePtxtSpace also reduces intFactor
      long g = std::gcd(ptxtSpace, other.ptxtSpace);
      if (g <= 1) throw LogicError("Plaintext spaces are co-prime");
      reducePtxtSpace(g);
      other.reducePtxtSpace(g);
    }
    double lo, hi;
    computeIntervalForMul(lo, hi, *this, other);
    auto f1 = primeSet.vec(), f2 = other.primeSet.vec();
    std::vector<int32_t> out(context.numPrimes()); int nout = 0;
    check(hb_chain_set4size(context.chain(), lo, hi, f1.data(), (int)f1.size(), f2.data(), (int)f2.size(), isCKKS() ? 1 : 0, out.data(), &nout));
    IndexSet common(out.begin(), out.begin() + nout);
    lastCommonPrimeSet = common; lastLo = lo; lastHi = hi;
    bringToSet(common);
    other.bringToSet(common);
  }
  // ---- linear operations (addConstant / multByConstant: BGV branches only)
  void negate() { for (auto& part : parts) part.dcrt.Negate(); }   // src/Ctxt.cpp:1190-1194
  void reducePtxtSpace(long newPtxtSpace) {   // src/Ctxt.cpp:576-584
    long g = std::gcd(ptxtSpace, newPtxtSpace);
    if (g <= 1) throw LogicError("New and old plaintext spaces are coprime");
    ptxtSpace = g; intFactor %= g;
  }
  static long balRem(long a, long q) { return a > q / 2 ? a - q : a; }   // include/helib/NumbTh.h:140-146
  void mulIntFactor(long e) {   // src/Ctxt.cpp:331-340
    if (e == 1) return;
    intFactor = (long)(((unsigned __int128)(unsigned long)intFactor * (unsigned long)e) % (unsigned long)ptxtSpace);
    long bal_e = balRem(e, ptxtSpace);
    for (auto& part : parts) part.dcrt *= bal_e;
    noiseBound = noiseBound * XD((double)std::labs(bal_e));
  }
  void addCtxt(const Ctxt& other, bool negative = false) {   // src/Ctxt.cpp:1406-1556
    if (&context != &other.context) throw LogicError("Context mismatch");
    if (&pubKey != &other.pubKey) throw LogicError("Public key mismatch");
    if (other.isEmpty()) return;
    if (isEmpty()) { *this = other; if (negative) negate(); return; }
    if (isCKKS()) { if (ptxtSpace != 1 || other.ptxtSpace != 1) throw LogicError("Plaintext spaces incompatible"); }
    else reducePtxtSpace(other.ptxtSpace);
    Ctxt tmp(pubKey, other.ptxtSpace);
    const Ctxt* other_pt = &other;
    if (ptxtSpace != other_pt->ptxtSpace) { tmp = other; tmp.reducePtxtSpace(ptxtSpace); other_pt = &tmp; }
    IndexSet s = other_pt->primeSet / primeSet;
    if (!empty(s)) modUpToSet(s);
    s = primeSet / other_pt->primeSet;
    if (!empty(s)) { if (other_pt != &tmp) { tmp = other; other_pt = &tmp; } tmp.modUpToSet(s); }
    if (isCKKS()) { if (other_pt != &tmp) { tmp = other; other_pt = &tmp; } equalizeRationalFactors(*this, tmp, context.getR()); }
    long e1 = 1, e2 = 1;
    if (!isCKKS() && intFactor != other_pt->intFactor) harmoniseIntFactors(*this, *other_pt, e1, e2);
    if (e2 != 1) { if (other_pt != &tmp) { tmp = other; other_pt = &tmp; } tmp.mulIntFactor(e2); }
    if (e1 != 1) mulIntFactor(e1);
    for (const CtxtPart& part : other_pt->parts) {
      long j = getPartIndexByHandle(part.skHandle);
      if (j >= 0) { if (negative) parts[j].dcrt -= part.dcrt; else parts[j].dcrt += part.dcrt; }
      else { parts.push_back(part); if (negative) parts.back().dcrt.Negate(); }
    }
    ptxtMag = ptxtMag + other_pt->ptxtMag;
    noiseBound = noiseBound + other_pt->noiseBound;
  }
  // addCtxt's harmonisation of two BGV intFactors (src/Ctxt.cpp:1475-1527): e1*f1 == e2*f2 (mod ptxtSpace) with the least
  // noise growth, a and b at one plaintext space
  static void harmoniseIntFactors(const Ctxt& a, const Ctxt& b, long& e1, long& e2) {
    const long P = a.ptxtSpace, f1 = a.intFactor, f2 = b.intFactor;
    const long ratio = (long)(((unsigned __int128)(unsigned long)f2 * (unsigned long)invMod(f1, P)) % (unsigned long)P);
    auto noiseNorm = [&](long x, long y) { return a.noiseBound * XD((double)std::labs(balRem(x, P))) + b.noiseBound * XD((double)std::labs(balRem(y, P))); };
    auto mc = [&](long x) { x %= P; return x < 0 ? x + P : x; };
    long r0 = P, t0 = 0, r1 = ratio, t1 = 1;
    long e1_best = r1, e2_best = t1;
    XD noise_best = noiseNorm(e1_best, e2_best);
    const long pp = a.context.getP();
    while (r1 != 0) {
      long q = r0 / r1, r2 = r0 % r1, t2 = t0 - t1 * q;
      r0 = r1; r1 = r2; t0 = t1; t1 = t2;
      long e1_try = mc(r1), e2_try = mc(t1);
      if (e1_try % pp != 0) { XD n = noiseNorm(e1_try, e2_try); if (n < noise_best) { e1_best = e1_try; e2_best = e2_try; noise_best = n; } }
    }
    e1 = e1_best; e2 = e2_best;
  }
  // src/Ctxt.cpp:1199-1351 ("NEW VERSION"): bring two CKKS ciphertexts to a common scaling factor by multiplying them by
  // the numerator / denominator of a continued-fraction approximation of the ratio, stopping as soon as the
  // discretisation error is within sqrt(2) of the unavoidable one.  r = Context::getPrecision().
  static void equalizeRationalFactors(Ctxt& c1, Ctxt& c2, long r) {
    Ctxt& big = (c1.ratFactor > c2.ratFactor) ? c1 : c2;
    Ctxt& small = (c1.ratFactor > c2.ratFactor) ? c2 : c1;
    const XD x = big.ratFactor / small.ratFactor;
    const double denomBound = std::ldexp(1.0, (int)r + 1);
    const double epsilon = 0.125 / denomBound;
    auto calc_err = [](const XD& f, const XD& m1, const XD& f1, const XD& e1, const XD& m2, const XD& f2, const XD& e2) {
      return m1 * (f1 / f - XD(1.0)).abs() + m2 * (f2 / f - XD(1.0)).abs() + (e1 + e2) / f;
    };
    auto floorXD = [](const XD& v) { uint64_t mant; long sh; v.floorParts(mant, sh); return XD::make((double)mant, sh); };
    XD xi = x - floorXD(x + XD(epsilon));
    double prevDenom = 0, denom = 1;
    XD numer = floorXD(XD(denom) * x + XD(0.5));
    const XD m1 = big.ptxtMag, of1 = big.ratFactor, oe1 = big.noiseBound;
    const XD m2 = small.ptxtMag, of2 = small.ratFactor, oe2 = small.noiseBound;
    const XD target_error = oe1 / of1 + oe2 / of2;
    XD f, fe1, fe2;
    for (;;) {
      const XD xdenom(denom);
      const XD f1 = of1 * xdenom, e1 = oe1 * xdenom, f2 = of2 * numer, e2 = oe2 * numer;
      const XD err1 = calc_err(f1, m1, f1, e1, m2, f2, e2), err2 = calc_err(f2, m1, f1, e1, m2, f2, e2);
      XD err;
      if (err1 < err2) { f = f1; fe1 = e1; fe2 = e2 + m2 * (f2 - f1).abs(); err = err1; }
      else { f = f2; fe1 = e1 + m1 * (f2 - f1).abs(); fe2 = e2; err = err2; }
      if (err < XD(std::sqrt(2.0)) * target_error) break;
      if (xi.m <= 0) break;
      xi = XD(1.0) / xi;
      const XD ai = floorXD(xi + XD(epsilon));
      xi = xi - ai;
      const double tmpDenom = denom * ai.to_double() + prevDenom;
      if (tmpDenom > denomBound) break;
      prevDenom = denom; denom = tmpDenom;
      numer = floorXD(XD(denom) * x + XD(0.5));
    }
    if (denom != 1) for (auto& part : big.parts) part.dcrt *= (long)denom;
    big.ratFactor = f; big.noiseBound = fe1;
    uint64_t nm; long nsh; numer.floorParts(nm, nsh);
    if (!(nm == 1 && nsh == 0)) for (auto& part : small.parts) part.dcrt.mulByPow2Scaled(nm, nsh);
    small.ratFactor = f; small.noiseBound = fe2;
  }
  Ctxt& operator+=(const Ctxt& o) { addCtxt(o); return *this; }
  Ctxt& operator-=(const Ctxt& o) { addCtxt(o, true); return *this; }
  // src/Ctxt.cpp:896-935 (BGV): the constant is scaled by intFactor*Q mod p so that it decrypts unscaled
  void addConstant(const DoubleCRT& dcrt, double size = -1.0) {
    if (isCKKS()) throw LogicError("Ctxt::addConstant: use addConstantCKKS (explicit size and factor)");
    if (size < 0.0) size = pubKey.noiseBoundForMod(ptxtSpace, context.getPhiM());
    const long f = constantFactor();
    noiseBound = noiseBound + XD(size * (double)std::labs(f));
    if (f == 1) addPart(dcrt, SKHandle(0, 1, 0));
    else { DoubleCRT tmp = dcrt; tmp *= f; addPart(tmp, SKHandle(0, 1, 0)); }
  }
  // multByConstantCKKS (src/Ctxt.cpp:1905-1938): dcrt encodes slots of magnitude <= size at scaling factor `factor`;
  // roundingErr = the encoding's rounding error.  The reference's defaults come from EncryptedArrayCx (the encoding layer,
  // out of scope here), so the three values are explicit arguments.
  void multByConstantCKKS(const DoubleCRT& dcrt, const XD& size, const XD& factor, double roundingErr) {
    if (isEmpty()) return;
    if (!isCKKS()) throw LogicError("multByConstantCKKS on a BGV ciphertext");
    noiseBound = noiseBound * factor * size + XD(roundingErr) * ratFactor * ptxtMag + noiseBound * XD(roundingErr);   // must come first
    ptxtMag = ptxtMag * size;
    ratFactor = ratFactor * factor;
    for (auto& part : parts) part.dcrt.Mul(dcrt, /*matchIndexSets=*/false);
  }
  // addConstantCKKS (src/Ctxt.cpp:941-1052): the constant (scaling factor `factor`) is multiplied by round(ratFactor/factor)
  // so that it matches the ciphertext's factor.  The reference adds primes (addSomePrimes) when that rounding alone would
  // cost more than 2^-precision of accuracy; the mirror reports that case instead.
  void addConstantCKKS(const DoubleCRT& dcrt, const XD& size_in, const XD& factor) {
    if (!isCKKS()) throw LogicError("addConstantCKKS on a BGV ciphertext");
    const XD size = size_in.m <= 0 ? XD(1.0) : size_in;
    if (factor.m <= 0) throw InvalidArgument("addConstantCKKS: the scaling factor of the constant must be given");
    XD ratio = ratFactor / factor + XD(0.5);
    uint64_t mant; long sh; ratio.floorParts(mant, sh);
    const XD r = XD::make((double)mant, sh);
    const double inaccuracy = std::fabs((r * factor / ratFactor).to_double() - 1.0);
    if (inaccuracy * std::ldexp(1.0, (int)context.getR()) > 1.0) throw LogicError("addConstantCKKS: scaling factors too far apart (the reference calls addSomePrimes here)");
    ptxtMag = ptxtMag + size;
    noiseBound = noiseBound + XD(0.5);
    IndexSet delta = primeSet / dcrt.getIndexSet();
    if (mant == 1 && sh == 0 && empty(delta)) { addPart(dcrt, SKHandle(0, 1, 0)); return; }
    DoubleCRT tmp = dcrt;
    if (!empty(delta)) tmp.addPrimes(delta);
    if (!(mant == 1 && sh == 0)) tmp.mulByPow2Scaled(mant, sh);
    addPart(tmp, SKHandle(0, 1, 0));
  }
  // src/Ctxt.cpp:1832-1856 (BGV)
  void multByConstant(const DoubleCRT& dcrt, double size = -1.0) {
    if (isEmpty()) return;
    if (isCKKS()) throw LogicError("Ctxt::multByConstant: use multByConstantCKKS (explicit size, factor and rounding error)");
    if (size < 0.0) size = pubKey.noiseBoundForMod(ptxtSpace, context.getPhiM());
    for (auto& part : parts) part.dcrt.Mul(dcrt, /*matchIndexSets=*/false);
    noiseBound = noiseBound * XD(size);
  }
  // Ctxt::clear (include/helib/Ctxt.h:1347-1355); the plaintext space stays
  void clear() { parts.clear(); primeSet = context.getCtxtPrimes(); noiseBound = XD(0.0); intFactor = 1; ratFactor = ptxtMag = XD(1.0); }
  // multByConstant(ZZ) for a word-sized c, BGV branch (src/Ctxt.cpp:2033-2069): c = c1*d with d = gcd(c, ptxtSpace); the
  // rows are multiplied by balRem(d) and intFactor by c1^-1.  The CKKS branch encodes through the slot layer, which the
  // mirror does not have.
  void multByConstant(long c) {
    if (isCKKS()) throw LogicError("Ctxt::multByConstant(long): BGV only (the CKKS branch encodes the scalar)");
    if (isEmpty()) return;
    long c0 = c % ptxtSpace; if (c0 < 0) c0 += ptxtSpace;
    if (c0 == 1) return;
    if (c0 == 0) { clear(); return; }
    const long d = std::gcd(c0, ptxtSpace);
    const long c1_inv = invMod(c0 / d, ptxtSpace);
    intFactor = (long)(((unsigned __int128)(unsigned long)intFactor * (unsigned long)c1_inv) % (unsigned long)ptxtSpace);
    if (d == 1) return;
    const long cc = balRem(d, ptxtSpace);
    noiseBound = noiseBound * XD((double)std::labs(cc));
    for (auto& part : parts) part.dcrt *= cc;
  }
  // addConstant(ZZ) for a word-sized c, BGV branch (src/Ctxt.cpp:2264-2282), through addConstant(FatEncodedPtxt_BGV)
  // (:2145-2185) with the constant polynomial cc = balRem(c mod ptxtSpace) of size cc (negative sizes lower the bound, as
  // there); the constant is scaled by intFactor*Q mod ptxtSpace so that it decrypts unscaled.
  void addConstant(long c, bool neg = false) {
    if (isCKKS()) throw LogicError("Ctxt::addConstant(long): BGV only (the CKKS branch encodes the scalar)");
    long cc = c % ptxtSpace; if (cc < 0) cc += ptxtSpace;
    if (cc > ptxtSpace / 2) cc -= ptxtSpace;
    if (cc == 0) return;
    const long f = constantFactor();
    noiseBound = noiseBound + XD((double)cc * (double)std::labs(f));
    DoubleCRT d(std::vector<long>{cc}, context, primeSet);
    if (f != 1) d *= f;
    addPart(d, SKHandle(0, 1, 0), neg);
  }
  // the factor addConstant scales a BGV constant by: balRem(intFactor * prod(primeSet) mod ptxtSpace), 1 for ptxtSpace <= 2
  long constantFactor() const {
    if (ptxtSpace <= 2) return 1;
    unsigned long q = 1;
    for (long i : primeSet) q = (unsigned long)(((unsigned __int128)q * (unsigned long)(context.ithPrime(i) % ptxtSpace)) % (unsigned long)ptxtSpace);
    return balRem((long)(((unsigned __int128)(unsigned long)intFactor * q) % (unsigned long)ptxtSpace), ptxtSpace);
  }
  // effectiveR (src/Ctxt.cpp:103-114): r with ptxtSpace = p^r
  long effectiveR() const {
    const long p = context.getP();
    for (long r = 1, p2r = p; r < 60; r++, p2r *= p) {   // HELIB_SP_NBITS
      if (p2r == ptxtSpace) return r;
      if (p2r > ptxtSpace) break;
    }
    throw RuntimeError("ctxt.ptxtSpace is not of the form p^r");
  }
  // divideByP (src/Ctxt.cpp:2415-2435): every part times p^-1 mod Q, in one hb_scale_rows call over the parts; the
  // plaintext space drops from p^r to p^(r-1).  The ciphertext must encrypt a multiple of p.
  void divideByP() {
    if (isEmpty()) return;
    divideByPMeta();
    const std::vector<int32_t> idx = primeSet.vec();
    std::vector<uint64_t> sc;
    for (int32_t i : idx) sc.push_back((uint64_t)invMod(context.getP(), context.ithPrime(i)));
    std::vector<hb_poly*> d;   // every part is over primeSet (addPart and matchPrimeSet keep it so)
    for (auto& part : parts) d.push_back(part.dcrt.handle());
    if (!idx.empty()) check(hb_scale_rows(d.data(), (int)d.size(), idx.data(), (int)idx.size(), sc.data()));
  }
  // divideByP's asserts and metadata, the part the fused digit chains replay
  void divideByPMeta() {
    const long p = context.getP();
    if (ptxtSpace % p != 0) throw LogicError("p must divide ptxtSpace");
    if (!(ptxtSpace > p)) throw LogicError("ptxtSpace must be strictly greater than p");
    noiseBound = noiseBound / XD((double)p);
    ptxtSpace /= p;
    intFactor %= ptxtSpace;
  }
  // multByP (include/helib/Ctxt.h:1216-1221): times p^e, the plaintext space grows to p^(r+e)
  void multByP(long e = 1) {
    long p2e = 1;
    for (long i = 0; i < e; i++) p2e *= context.getP();
    ptxtSpace *= p2e;
    multByConstant(p2e);
  }
  long getKeyID() const { for (auto& part : parts) if (!part.skHandle.isOne()) return part.skHandle.secretKeyID; return 0; }   // src/Ctxt.cpp:2550-2557
  void cleanUp() {   // src/Ctxt.cpp:788-797
    reLinearize();
    if (!primeSet.disjointFrom(context.getSpecialPrimes()) || !primeSet.disjointFrom(context.getSmallPrimes())) dropSmallAndSpecialPrimes();
  }
  static long invMod(long a, long m) {
    long b = m, x0 = 1, x1 = 0; a %= m; if (a < 0) a += m;
    while (b) { long q = a / b, t = a - q * b; a = b; b = t; t = x0 - q * x1; x0 = x1; x1 = t; }
    if (a != 1) throw InvalidArgument("InvMod: not invertible");
    x0 %= m; return x0 < 0 ? x0 + m : x0;
  }
  void automorph(long k) {   // src/Ctxt.cpp:2437-2457: F(X) -> F(X^k), no change in the noise bound
    if (isEmpty()) return;
    const long m = context.getM();
    if (k <= 0 || k >= m || std::gcd(k, m) != 1) throw LogicError("k must be in Zm*");
    for (auto& part : parts) {
      part.dcrt.automorph(k);
      if (!part.skHandle.isOne()) part.skHandle.powerOfX = (long)(((unsigned __int128)(unsigned long)part.skHandle.powerOfX * (unsigned long)k) % (unsigned long)m);
    }
  }
  void complexConj() { automorph(context.getM() - 1); }   // src/Ctxt.cpp:2517-2523
  void smartAutomorph(long k) {   // src/Ctxt.cpp:2462-2515: automorphism then re-linearisation, in the steps the key-switching map allows
    const long m = context.getM();
    k %= m; if (k < 0) k += m;
    if (isEmpty() || k == 1) return;
    if (std::gcd(k, m) != 1) throw LogicError("k must be in Zm*");
    const long keyID = getKeyID();
    if (!pubKey.isReachable(k, keyID)) throw LogicError("no key-switching matrices for k=" + std::to_string(k) + ", keyID=" + std::to_string(keyID));
    if (!inCanonicalForm(keyID)) { reLinearize(keyID); if (!inCanonicalForm(keyID)) throw LogicError("Re-linearization failed: not in canonical form"); }
    while (k != 1) {
      const KeySwitch* matrix = pubKey.getNextKSWmatrix(k, keyID);
      const long amt = matrix->fromKey.powerOfX;
      automorph(amt);
      reLinearize(keyID);
      k = (long)(((unsigned __int128)(unsigned long)k * (unsigned long)invMod(amt, m)) % (unsigned long)m);
    }
  }
  // Phi_m(X) over Z (Cyclotomic(m)): Phi_1 = X - 1; Phi_{np}(X) = Phi_n(X^p) / Phi_n(X) for p not dividing n, Phi_n(X^p) otherwise
  static std::vector<long> cyclotomic(long m) {
    std::vector<long> phi{-1, 1};
    long n = 1;
    for (long p = 2; m > 1; p++) {
      bool first = true;
      while (m % p == 0) {
        m /= p;
        std::vector<long> up((phi.size() - 1) * p + 1, 0);
        for (size_t i = 0; i < phi.size(); i++) up[i * p] = phi[i];
        if (first && n % p != 0) {   // exact division of up by the monic phi
          std::vector<long> quo(up.size() - phi.size() + 1, 0);
          for (long i = (long)up.size() - 1; i >= (long)phi.size() - 1; i--) {
            const long c = up[i]; quo[i - (phi.size() - 1)] = c;
            if (c) for (size_t j = 0; j < phi.size(); j++) up[i - (phi.size() - 1) + j] -= c * phi[j];
          }
          phi = quo;
        } else phi = up;
        n *= p; first = false;
      }
    }
    return phi;
  }
  // Ctxt::rawModSwitch (src/Ctxt.cpp:2949-3046): mod-switch to an external modulus q for bootstrapping.  The scaling and
  // rounding run on the device in the powerful basis (hb_raw_mod_switch); the small result is brought back to the
  // polynomial basis here (PowerfulDCRT::powerfulToZZX, src/powerful.cpp:355-391).  Returns the scaled noise estimate.
  double rawModSwitch(std::vector<std::vector<long>>& zzParts, long q) const {
    if (q <= 1) throw InvalidArgument("q must be greater than 1");
    if (ptxtSpace <= 1) throw LogicError("Plaintext space must be greater than 1 for mod switching");
    if (std::gcd(q, ptxtSpace) != 1) throw LogicError("New modulus and current plaintext space must be co-prime");
    const long phim = context.getPhiM(), m = context.getM();
    int32_t nf = 0; std::vector<int32_t> toPoly((size_t)phim);
    check(hb_ctx_powerful_info(context.handle(), &nf, nullptr, toPoly.data()));
    std::vector<long> phimx;
    if (nf > 1) phimx = cyclotomic(m);
    zzParts.assign(parts.size(), std::vector<long>());
    auto idx = primeSet.vec();
    for (size_t i = 0; i < parts.size(); i++) {
      std::vector<int64_t> pw((size_t)phim);
      check(hb_raw_mod_switch(parts[i].dcrt.handle(), idx.data(), (int)idx.size(), (uint64_t)q, (uint64_t)ptxtSpace, pw.data()));
      if (nf <= 1) { zzParts[i].assign(pw.begin(), pw.end()); continue; }
      std::vector<long> tmp((size_t)m, 0);
      for (long k = 0; k < phim; k++) tmp[toPoly[k]] = pw[k];
      for (long k = m - 1; k >= phim; k--) {   // rem(tmp, Phi_m): Phi_m is monic of degree phi(m)
        const long c = tmp[k];
        if (c) for (long j = 0; j <= phim; j++) tmp[k - phim + j] -= c * phimx[j];
      }
      zzParts[i].assign(tmp.begin(), tmp.begin() + phim);
    }
    return (noiseBound * XD::exp(std::log((double)q) - logOfPrimeSet())).to_double();
  }
  // ---- binary wire format, Ctxt::writeTo / read (src/Ctxt.cpp:2584-2641, src/binio.h:91-137, src/binio.cpp:75-178):
  //   24-byte SerializeHeader<Ctxt> ("|HE[", format version 0.0.1.0, library version, struct id 20, 7 reserved, "]HE|"),
  //   "|CX[", ptxtSpace, intFactor, ptxtMag, ratFactor, noiseBound (xdouble = raw double mantissa + int64 exponent),
  //   primeSet, vector<CtxtPart> (count, then DoubleCRT + SKHandle each), "]CX|".  All integers little-endian int64.
  // NTL's xdouble is x * (2^114)^e with 2^-57 <= |x| <= 2^57 (NTL 11.4.3 xdouble.h, NTL_XD_BOUND); NTL is not in the
  // reference tree, so this split is restated from its documentation: parity unpinned for those 16-byte fields.
  static void writeXD(std::ostream& str, const XD& v) {
    double x = 0; int64_t e = 0;
    if (v.m != 0) {
      long E = v.e;                      // v = m * 2^E, 0.5 <= |m| < 1
      e = E > 57 ? (E - 57 + 113) / 114 : (E < -56 ? -((-56 - E + 113) / 114) : 0);
      x = std::ldexp(v.m, (int)(E - 114 * e));
    }
    str.write(reinterpret_cast<const char*>(&x), 8); str.write(reinterpret_cast<const char*>(&e), 8);
  }
  static XD readXD(std::istream& str) {
    double x = 0; int64_t e = 0;
    str.read(reinterpret_cast<char*>(&x), 8); str.read(reinterpret_cast<char*>(&e), 8);
    return XD::make(x, 114 * (long)e);
  }
  static void writeInt(std::ostream& str, int64_t v) { str.write(reinterpret_cast<const char*>(&v), 8); }
  static int64_t readInt(std::istream& str) { int64_t v = 0; str.read(reinterpret_cast<char*>(&v), 8); return v; }
  void writeTo(std::ostream& str) const {
    const char header[24] = {'|', 'H', 'E', '[', 0, 0, 1, 0, 2, 2, 0, 0, 20, 0, 0, 0, 0, 0, 0, 0, ']', 'H', 'E', '|'};
    str.write(header, 24);
    str.write("|CX[", 4);
    writeInt(str, ptxtSpace); writeInt(str, intFactor);
    writeXD(str, ptxtMag); writeXD(str, ratFactor); writeXD(str, noiseBound);
    writeInt(str, primeSet.card());
    for (long i : primeSet) writeInt(str, i);
    writeInt(str, (int64_t)parts.size());
    for (const CtxtPart& part : parts) {
      part.dcrt.writeTo(str);
      writeInt(str, part.skHandle.powerOfS); writeInt(str, part.skHandle.powerOfX); writeInt(str, part.skHandle.secretKeyID);
    }
    str.write("]CX|", 4);
  }
  void read(std::istream& str) {
    char header[24];
    str.read(header, 24);
    if (!str || std::memcmp(header, "|HE[", 4) != 0 || std::memcmp(header + 20, "]HE|", 4) != 0) throw RuntimeError("Eye catchers for header mismatch");
    const char ver[4] = {0, 0, 1, 0};
    if (std::memcmp(header + 4, ver, 4) != 0) throw RuntimeError("Header: version not supported");
    char eye[4];
    str.read(eye, 4);
    if (std::memcmp(eye, "|CX[", 4) != 0) throw RuntimeError("Could not find pre-ciphertext eye catcher");
    ptxtSpace = readInt(str); intFactor = readInt(str);
    ptxtMag = readXD(str); ratFactor = readXD(str); noiseBound = readXD(str);
    const int64_t card = readInt(str);
    if (!str || card < 0 || card > context.numPrimes()) throw RuntimeError("Ctxt::read: bad prime set");
    primeSet = IndexSet();
    for (int64_t i = 0; i < card; i++) primeSet.insert(readInt(str));
    const int64_t np = readInt(str);
    if (!str || np < 0 || np > 64) throw RuntimeError("Ctxt::read: bad part count");
    parts.clear();
    for (int64_t i = 0; i < np; i++) {
      DoubleCRT d(context, IndexSet::emptySet());
      d.read(str);
      SKHandle h; h.powerOfS = readInt(str); h.powerOfX = readInt(str); h.secretKeyID = readInt(str);
      parts.emplace_back(d, h);
    }
    str.read(eye, 4);
    if (!str || std::memcmp(eye, "]CX|", 4) != 0) throw RuntimeError("Could not find post-ciphertext eye catcher");
  }
  void multiplyBy(const Ctxt& other) {   // src/Ctxt.cpp:1757-1774
    HB_TIMER_START(context.handle());
    if (isEmpty()) return;
    if (other.isEmpty()) { *this = other; return; }
    multLowLvl(other);
    reLinearize();
  }
  // multiplyBy2 (src/Ctxt.cpp:1776-1828): this * other1 * other2, the two lower-capacity factors first, relinearised once
  void multiplyBy2(const Ctxt& other1, const Ctxt& other2) {
    HB_TIMER_START(context.handle());
    if (isEmpty()) return;
    if (other1.isEmpty()) { *this = other1; return; }
    if (other2.isEmpty()) { *this = other2; return; }
    const double cap = capacity(), cap1 = other1.capacity(), cap2 = other2.capacity();
    if (cap < cap1 && cap < cap2) {   // both others at higher levels than this: multiply them first, then by this
      Ctxt tmp = other1;
      if (&other1 == &other2) tmp.multLowLvl(tmp);   // squaring rather than multiplication
      else tmp.multLowLvl(other2);
      multLowLvl(tmp);
      reLinearize();
      return;
    }
    const Ctxt *first, *second;
    if (cap < cap2 || cap1 < cap2) { first = &other2; second = &other1; }
    else { first = &other1; second = &other2; }
    if (this == second) {   // pointer collision
      Ctxt tmp = *second;
      multLowLvl(*first);
      multLowLvl(tmp);
    } else {
      multLowLvl(*first);
      multLowLvl(*second);
    }
    reLinearize();
  }
  void square() { multiplyBy(*this); }        // include/helib/Ctxt.h:1230
  void cube() { multiplyBy2(*this, *this); }  // include/helib/Ctxt.h:1231
  void power(long e);   // src/polyEval.cpp:392-413, defined after DynamicCtxtPowers
  // statistics the reference records through HELIB_STATS_UPDATE (src/Ctxt.cpp:537,835)
  double lastModSwitchRatio = 0, lastKSNoiseRatio = 0, lastLo = 0, lastHi = 0;
  IndexSet lastCommonPrimeSet;
};

// DynamicCtxtPowers (include/helib/polyEval.h:45-75, src/polyEval.cpp:18-29): the powers X^1..X^n of a ciphertext, each
// computed on first use as X^e = X^(e-k) * X^k, k the largest power of two below e -- a product of two stored powers, never
// a square -- so that every power sits as high as it can.
class DynamicCtxtPowers {
  std::vector<Ctxt> v;
 public:
  DynamicCtxtPowers(const Ctxt& c, long nPowers) {
    if (c.isEmpty()) throw InvalidArgument("Ciphertext cannot be empty");
    if (nPowers <= 0) throw InvalidArgument("Must have positive nPowers");
    v.assign((size_t)nPowers, Ctxt(c.pubKey, c.ptxtSpace));
    v[0] = c;
  }
  Ctxt& getPower(long e) {
    if (v.at((size_t)e - 1).isEmpty()) {
      long np2 = 0;
      while ((1L << np2) < e) np2++;   // NTL::NextPowerOfTwo(e)
      const long k = 1L << (np2 - 1);
      v[(size_t)e - 1] = getPower(e - k);
      v[(size_t)e - 1].multiplyBy(getPower(k));
    }
    return v[(size_t)e - 1];
  }
  Ctxt& at(long i) { return getPower(i + 1); }
  Ctxt& operator[](long i) { return getPower(i + 1); }
  long size() const { return (long)v.size(); }
  bool isPowerComputed(long i) const { return i > 0 && i <= (long)v.size() && !v[(size_t)i - 1].isEmpty(); }
};

// power (src/polyEval.cpp:392-413): repeated squaring for a power of two, DynamicCtxtPowers otherwise
inline void Ctxt::power(long e) {
  if (e < 1) throw InvalidArgument("Cannot raise a ctxt to a non positive exponent");
  if (e == 1) return;
  long ell = 0;
  for (unsigned long x = (unsigned long)e; x; x >>= 1) ell++;   // NTL::NumBits(e): e < 2^ell <= 2e
  if ((unsigned long)e == (1UL << (ell - 1))) {
    while (--ell > 0) square();
    return;
  }
  DynamicCtxtPowers pwrs(*this, e);
  *this = pwrs.getPower(e);
}

// BasicAutomorphPrecon (src/matmul.cpp:60-184): hoisting -- one breakIntoDigits shared by many automorphisms of the
// same ciphertext.  Each automorph(k) is ONE engine launch for power-of-two m (sigma_k applied in the load stage of
// the evaluation-key inner product, hb_automorph_keyswitch_digits); general m permutes the digits first.
class BasicAutomorphPrecon {
  Ctxt ctxt;
  XD noise;
  std::vector<DoubleCRT> polyDigits;
 public:
  double lastKSNoiseRatioHoist = 0;   // "KS-noise-ratio-hoist" (src/matmul.cpp:101)
  // the cleaned ciphertext, the noise bound of every hoisted rotation and the digits of its part 1 (hb::BlockMatMul1D
  // hands them to one engine call)
  const Ctxt& cleaned() const { return ctxt; }
  const XD& hoistNoise() const { return noise; }
  const std::vector<DoubleCRT>& digits() const { return polyDigits; }
  explicit BasicAutomorphPrecon(const Ctxt& c) : ctxt(c), noise(1.0) {
    if (ctxt.parts.size() >= 1 && !ctxt.parts[0].skHandle.isOne()) throw LogicError("Invalid ciphertext (secret key handle for part 0 is not one)");
    if (ctxt.parts.size() <= 1) return;
    ctxt.cleanUp();
    if (!ctxt.inCanonicalForm(ctxt.getKeyID())) throw LogicError("Ciphertext is not in canonical form");
    ctxt.relin_CKKS_adjust();
    XD addedNoise(0.0);
    for (double ln : ctxt.parts[1].dcrt.breakIntoDigitsLogNorms(polyDigits)) addedNoise = addedNoise + XD::exp(ln);
    XD max_ks_noise(0.0);
    for (const KeySwitch& ks : ctxt.pubKey.keySwitching) if (max_ks_noise < ks.noiseBound) max_ks_noise = ks.noiseBound;
    addedNoise = addedNoise * max_ks_noise;
    noise = ctxt.noiseBound * XD::exp(ctxt.pubKey.logOfProduct(ctxt.context.getSpecialPrimes()));
    lastKSNoiseRatioHoist = (addedNoise / noise).to_double();
    noise = noise + addedNoise;
  }
  std::shared_ptr<Ctxt> automorph(long k) const {
    if (k == 1 || ctxt.isEmpty()) return std::make_shared<Ctxt>(ctxt);
    const Context& context = ctxt.context;
    const KeyInfo& pubKey = ctxt.pubKey;
    const long m = context.getM();
    auto result = std::make_shared<Ctxt>(pubKey, ctxt.ptxtSpace);
    result->noiseBound = noise;
    result->intFactor = ctxt.intFactor;
    result->primeSet = ctxt.primeSet | context.getSpecialPrimes();
    if (ctxt.isCKKS()) {
      result->ptxtMag = ctxt.ptxtMag;
      result->ratFactor = ctxt.ratFactor * XD::exp(pubKey.logOfProduct(context.getSpecialPrimes()));
    }
    if (ctxt.parts.size() == 1) {   // only the constant part: no key switch
      DoubleCRT tmp = ctxt.parts[0].dcrt;
      tmp.automorph(k);
      tmp.addPrimesAndScale(context.getSpecialPrimes());
      result->addPart(tmp, ctxt.parts[0].skHandle);
      return result;
    }
    const long keyID = ctxt.getKeyID();
    if (!pubKey.isReachable(k, keyID)) throw LogicError("no key-switching matrices for k=" + std::to_string(k) + ", keyID=" + std::to_string(keyID));
    const KeySwitch& W = *pubKey.getNextKSWmatrix(k, keyID);
    const long amt = W.fromKey.powerOfX;
    const bool pow2 = (m & (m - 1)) == 0;
    if (pow2) {
      DoubleCRT o0(context, result->primeSet), o1(context, result->primeSet);
      std::vector<hb_poly*> dg, ea, eb;
      for (size_t i = 0; i < polyDigits.size(); i++) { dg.push_back(polyDigits[i].handle()); ea.push_back(W.aHandle(i)); eb.push_back(W.b[i].handle()); }
      hb_poly* c0[1] = {ctxt.parts[0].dcrt.handle()}; hb_poly* p0[1] = {o0.handle()}; hb_poly* p1[1] = {o1.handle()};
      auto S = ctxt.primeSet.vec();
      check(hb_automorph_keyswitch_digits(dg.data(), (int)dg.size(), (int)dg.size(), 1, S.data(), (int)S.size(), c0, (uint64_t)amt, ea.data(), eb.data(), p0, p1));
      result->parts.emplace_back(o0, SKHandle());
      result->parts.emplace_back(o1, SKHandle(1, 1, W.toKeyID));
    } else {
      DoubleCRT tmp = ctxt.parts[0].dcrt;
      tmp.automorph(amt);
      tmp.addPrimesAndScale(context.getSpecialPrimes());
      result->addPart(tmp, ctxt.parts[0].skHandle);
      std::vector<DoubleCRT> tmpDigits = polyDigits;
      for (auto& d : tmpDigits) d.automorph(amt);
      result->keySwitchDigits(W, tmpDigits);
    }
    if ((amt - k) % m != 0) result->smartAutomorph((long)(((unsigned __int128)(unsigned long)k * (unsigned long)Ctxt::invMod(amt, m)) % (unsigned long)m));
    return result;
  }
  // The hoisted linear map of MatMul1DExec::mul's native FULL branch (src/matmul.cpp:1226-1252):
  //   acc = 0;  for j: tmp = automorph(k[j]); tmp->multByConstant(*consts[j], sizes[j]); acc += *tmp;  return acc
  // The amounts whose matrix is direct (getNextKSWmatrix(k).fromKey.powerOfX == k), and k == 1, are summed by one
  // hb_hoisted_linear_map call over S | special, without intermediate ciphertexts; the rest, and a ciphertext with one
  // part, take the loop above.  Bits and metadata are those of the loop.  BGV; CKKS: linearCombinationCKKS.
  std::shared_ptr<Ctxt> linearCombination(const std::vector<long>& k, const std::vector<const DoubleCRT*>& consts, const std::vector<double>& sizes) const {
    if (ctxt.isCKKS()) throw LogicError("linearCombination: use linearCombinationCKKS (explicit size, factor and rounding error)");
    std::vector<Coef> cf;
    for (size_t j = 0; j < consts.size(); j++) cf.push_back({consts[j], j < sizes.size() ? sizes[j] : -1.0, XD(), XD(), 0.0});
    return combine(k, cf);
  }
  // CKKS: each constant's (size, factor, roundingErr) as multByConstantCKKS takes them.  Terms are fused when their matrix is
  // direct, k != 1, and their factor equals the first such term's; if any term cannot be fused, every term takes the loop,
  // because equalizeRationalFactors scales the partial sum it meets and that sum then depends on the order of the terms.
  std::shared_ptr<Ctxt> linearCombinationCKKS(const std::vector<long>& k, const std::vector<const DoubleCRT*>& consts, const std::vector<XD>& sizes,
                                              const std::vector<XD>& factors, const std::vector<double>& roundingErrs) const {
    if (!ctxt.isCKKS()) throw LogicError("linearCombinationCKKS on a BGV ciphertext");
    std::vector<Coef> cf;
    for (size_t j = 0; j < consts.size(); j++) cf.push_back({consts[j], 0.0, sizes.at(j), factors.at(j), roundingErrs.at(j)});
    return combine(k, cf);
  }

  // a constant as multByConstant (BGV: size, < 0 for the default) or multByConstantCKKS (csize, factor, err) takes it
  struct Coef { const DoubleCRT* c; double size; XD csize, factor; double err; };
  static void mulConst(Ctxt& t, const Coef& c) {
    if (t.isCKKS()) t.multByConstantCKKS(*c.c, c.csize, c.factor, c.err); else t.multByConstant(*c.c, c.size);
  }
  // the metadata the loop's multByConstant / multByConstantCKKS gives a term (Ctxt::multByConstant returns early for a
  // ciphertext without parts, so the metadata-only terms below are updated here)
  static void mulConstMeta(Ctxt& t, const Coef& c) {
    if (t.isCKKS()) {
      t.noiseBound = t.noiseBound * c.factor * c.csize + XD(c.err) * t.ratFactor * t.ptxtMag + t.noiseBound * XD(c.err);
      t.ptxtMag = t.ptxtMag * c.csize;
      t.ratFactor = t.ratFactor * c.factor;
    } else {
      const double size = c.size < 0.0 ? t.pubKey.noiseBoundForMod(t.ptxtSpace, t.context.getPhiM()) : c.size;
      t.noiseBound = t.noiseBound * XD(size);
    }
  }
  // Ctxt::modUpToSet / addCtxt on metadata only, for terms with one intFactor: f is what DoubleCRT::addPrimesAndScale returns
  static void modUpMeta(Ctxt& c, const IndexSet& s) {
    IndexSet d = s / c.primeSet;
    if (empty(d)) return;
    const double f = c.pubKey.logOfProduct(d);
    c.noiseBound = c.noiseBound * XD::exp(f);
    c.ratFactor = c.ratFactor * XD::exp(f);
    c.primeSet.insert(d);
  }
  static void addMeta(Ctxt& a, bool& first, Ctxt o) {
    if (first) { a = o; first = false; return; }
    if (!a.isCKKS()) a.reducePtxtSpace(o.ptxtSpace);
    if (a.ptxtSpace != o.ptxtSpace) o.reducePtxtSpace(a.ptxtSpace);
    modUpMeta(a, o.primeSet);
    modUpMeta(o, a.primeSet);
    if (a.isCKKS()) Ctxt::equalizeRationalFactors(a, o, a.context.getR());
    a.ptxtMag = a.ptxtMag + o.ptxtMag;
    a.noiseBound = a.noiseBound + o.noiseBound;
  }
 private:
  std::shared_ptr<Ctxt> combine(const std::vector<long>& ks, const std::vector<Coef>& cf) const {
    if (ks.size() != cf.size()) throw InvalidArgument("linearCombination: one constant per amount");
    const Context& context = ctxt.context;
    const KeyInfo& pubKey = ctxt.pubKey;
    const long m = context.getM();
    const size_t n = ks.size();
    const bool ckks = ctxt.isCKKS();
    auto term = [&](size_t j) { auto t = automorph(ks[j]); mulConst(*t, cf[j]); return t; };
    auto loop = [&](std::vector<std::shared_ptr<Ctxt>>& done) {
      auto acc = std::make_shared<Ctxt>(pubKey, ctxt.ptxtSpace);
      for (size_t j = 0; j < n; j++) *acc += *(done[j] ? done[j] : term(j));
      return acc;
    };
    std::vector<std::shared_ptr<Ctxt>> done(n);
    // which amounts one call can sum
    std::vector<long> kk(n);
    std::vector<const KeySwitch*> W(n, nullptr);
    std::vector<char> fuse(n, 0);
    size_t nk = 0, nf = 0;
    const long keyID = ctxt.getKeyID();
    const Coef* first = nullptr;
    for (size_t j = 0; j < n && ctxt.parts.size() == 2; j++) {
      kk[j] = ((ks[j] % m) + m) % m;
      if (kk[j] == 1) { fuse[j] = !ckks; continue; }
      if (std::gcd(kk[j], m) != 1 || !pubKey.isReachable(kk[j], keyID)) continue;
      const KeySwitch* w = pubKey.getNextKSWmatrix(kk[j], keyID);
      if (w->fromKey.powerOfX != kk[j] || w->toKeyID != keyID) continue;
      if (ckks && first && (first->factor < cf[j].factor || cf[j].factor < first->factor)) continue;
      if (!first) first = &cf[j];
      W[j] = w; fuse[j] = 1; nk++;
    }
    for (size_t j = 0; j < n; j++) nf += fuse[j];
    if (nk == 0 || (ckks && nf < n)) return loop(done);
    // the other terms first: summing the fused ones apart reorders additions, which is exact only for one intFactor
    for (size_t j = 0; j < n; j++)
      if (!fuse[j]) { done[j] = term(j); if (!ckks && done[j]->intFactor != ctxt.intFactor) return loop(done); }
    // the fused terms: one call
    const IndexSet full = ctxt.primeSet | context.getSpecialPrimes();
    DoubleCRT a0(context, full), a1(context, full);
    {
      std::vector<hb_poly*> dg, cs, ea, eb;
      std::vector<uint64_t> kv;
      for (auto& d : polyDigits) dg.push_back(d.handle());
      const size_t nd = polyDigits.size();
      for (size_t j = 0; j < n; j++) {
        if (!fuse[j]) continue;
        kv.push_back((uint64_t)kk[j]); cs.push_back(cf[j].c->handle());
        for (size_t i = 0; i < nd; i++) { ea.push_back(W[j] ? W[j]->aHandle(i) : nullptr); eb.push_back(W[j] ? W[j]->b[i].handle() : nullptr); }
      }
      hb_poly* c0[1] = {ctxt.parts[0].dcrt.handle()}; hb_poly* c1[1] = {ctxt.parts[1].dcrt.handle()};
      hb_poly* o0[1] = {a0.handle()}; hb_poly* o1[1] = {a1.handle()};
      auto S = ctxt.primeSet.vec();
      check(hb_hoisted_linear_map(dg.data(), (int)nd, (int)nd, 1, S.data(), (int)S.size(), c0, c1, (int)kv.size(), kv.data(), cs.data(),
                                  ea.data(), eb.data(), o0, o1, 0));
    }
    auto acc = std::make_shared<Ctxt>(pubKey, ctxt.ptxtSpace);
    acc->primeSet = full;
    acc->intFactor = ctxt.intFactor;
    acc->parts.emplace_back(a0, SKHandle());
    acc->parts.emplace_back(a1, ctxt.parts[1].skHandle);
    for (size_t j = 0; j < n; j++) if (!fuse[j]) *acc += *done[j];   // data only: the metadata is replayed below
    // metadata: the loop's, term by term in its order
    Ctxt meta(pubKey, ctxt.ptxtSpace);
    bool empty_acc = true;
    for (size_t j = 0; j < n; j++) {
      Ctxt t(pubKey, ctxt.ptxtSpace);
      if (!fuse[j]) t = *done[j];
      else {
        if (kk[j] == 1) t = ctxt;
        else {
          t.noiseBound = noise; t.intFactor = ctxt.intFactor; t.primeSet = full;
          if (ckks) { t.ptxtMag = ctxt.ptxtMag; t.ratFactor = ctxt.ratFactor * XD::exp(pubKey.logOfProduct(context.getSpecialPrimes())); }
        }
        mulConstMeta(t, cf[j]);
      }
      t.parts.clear();
      addMeta(meta, empty_acc, t);
    }
    acc->primeSet = meta.primeSet; acc->ptxtSpace = meta.ptxtSpace; acc->noiseBound = meta.noiseBound;
    acc->intFactor = meta.intFactor; acc->ratFactor = meta.ratFactor; acc->ptxtMag = meta.ptxtMag;
    return acc;
  }
};

// ---- MatMul1DExec::mul's non-iterative baby-step/giant-step branches (src/matmul.cpp:989-1142) ------------------------
// genToPow(dim, e) of a dimension with generator gen: gen^e mod m, a negative e through the inverse
inline long genToPow(long gen, long e, long m) {
  unsigned long b = (unsigned long)(e < 0 ? Ctxt::invMod(gen, m) : ((gen % m) + m) % m), r = 1, x = (unsigned long)(e < 0 ? -e : e);
  for (; x; x >>= 1) { if (x & 1) r = (unsigned long)(((unsigned __int128)r * b) % (unsigned long)m); b = (unsigned long)(((unsigned __int128)b * b) % (unsigned long)m); }
  return (long)r;
}
// GenBabySteps (src/matmul.cpp:925-980), its hoisted branch: v[j] = automorph(gen^j) of one BasicAutomorphPrecon, cleaned if asked
inline std::vector<std::shared_ptr<Ctxt>> GenBabySteps(const Ctxt& ctxt, long gen, long g, bool clean) {
  std::vector<std::shared_ptr<Ctxt>> v((size_t)g);
  if (g == 1) { v[0] = std::make_shared<Ctxt>(ctxt); if (clean) v[0]->cleanUp(); return v; }
  BasicAutomorphPrecon precon(ctxt);
  for (long j = 0; j < g; j++) { v[(size_t)j] = precon.automorph(genToPow(gen, j, ctxt.context.getM())); if (clean) v[(size_t)j]->cleanUp(); }
  return v;
}
// A diagonal of the matrix as MatMul1DExec's cache holds it: c == nullptr is a zero diagonal (MulAdd skips it); BGV takes
// size (< 0: the default of multByConstant), CKKS csize, factor and err (multByConstantCKKS).
using BsgsDiag = BasicAutomorphPrecon::Coef;
// hb_bsgs_linear_map_norm: per giant step, 8 digit log-norms then the two mod-down norms
constexpr long kNormStride8 = 8;
// The metadata smartAutomorph gives a rotated term with a direct matrix W, replayed from the norms the device returned
// (nr: nd digit log-norms, then at kNormStride8 the two mod-down norms): if extended (over S | special), modDownToSet(S);
// then relin_CKKS_adjust and keySwitchPart.
inline void relinTermMeta(Ctxt& t, const double* nr, bool extended, const KeySwitch& W, long nd, const IndexSet& S) {
  const KeyInfo& pubKey = t.pubKey;
  const IndexSet special = t.context.getSpecialPrimes();
  const double logP = pubKey.logOfProduct(special);
  if (extended) {      // modDownToSet(S): parts 1 and s, the noise of delta/P from the device
    const XD addedNoise = XD(nr[kNormStride8]) + XD(nr[kNormStride8 + 1]) * XD::exp(std::log(pubKey.skBound));
    const XD f = XD::exp(logP);
    t.ratFactor = t.ratFactor / f;
    t.noiseBound = t.noiseBound / f;
    t.noiseBound = t.noiseBound + addedNoise;
    t.primeSet = S;
  }
  t.relin_CKKS_adjust();
  Ctxt tmp(pubKey, t.ptxtSpace);
  tmp.intFactor = t.intFactor; tmp.ptxtMag = t.ptxtMag;
  tmp.noiseBound = t.noiseBound * XD::exp(logP);
  tmp.primeSet = t.primeSet | special;
  tmp.ratFactor = t.ratFactor * XD::exp(logP);
  if (!t.isCKKS()) tmp.reducePtxtSpace(W.ptxtSpace);
  XD addedNoise(0.0);
  for (long i = 0; i < nd; i++) addedNoise = addedNoise + XD::exp(nr[i]);
  addedNoise = addedNoise * W.noiseBound;
  tmp.noiseBound = tmp.noiseBound + addedNoise;
  t = tmp;
}
// MatMul1DExec::mul for a dimension of size D > HELIB_KEYSWITCH_THRESH with generator gen, not iterative: ctxt becomes
// sum_i cache[i] * rot_i(ctxt) (+ cache1[i] * rot_{i-D}(ctxt) for a bad dimension, cache1 non-empty).  g = KSGiantStepSize(D).
// The baby steps are built as GenBabySteps builds them; every giant step is then summed by one hb_bsgs_linear_map call,
// with the loop's bits and its metadata (noise, factors, prime set), replayed from the norms the call returns.  The loop
// below runs instead wherever one call cannot reproduce it: a giant amount whose matrix is not direct, baby steps whose
// prime sets or factors differ (so that addCtxt would rescale, or dropSmallAndSpecialPrimes would keep a set other than S),
// a CKKS bad dimension, giant steps whose sum would not be a plain add (different intFactor or ratFactor), or no rotated
// giant step at all.
inline void MatMul1DBSGS(Ctxt& ctxt, long gen, long D, const std::vector<BsgsDiag>& cache, const std::vector<BsgsDiag>& cache1 = {}) {
  using P = BasicAutomorphPrecon;
  if (D <= 0 || (long)cache.size() != D || (!cache1.empty() && (long)cache1.size() != D)) throw InvalidArgument("MatMul1DBSGS: one diagonal per index");
  const bool native = cache1.empty();
  const Context& context = ctxt.context;
  const KeyInfo& pubKey = ctxt.pubKey;
  const long m = context.getM();
  long g = (long)std::sqrt((double)D); while (g * g < D) g++; while (g > 1 && (g - 1) * (g - 1) >= D) g--;
  const long h = (D + g - 1) / g;
  std::vector<std::shared_ptr<Ctxt>> bs = GenBabySteps(ctxt, gen, g, native), bs1;
  if (!native) { Ctxt c1(ctxt); c1.smartAutomorph(genToPow(gen, -D, m)); bs1 = GenBabySteps(c1, gen, g, false); }
  auto mulAdd = [&](Ctxt& acc, const BsgsDiag& d, const Ctxt& b) { if (!d.c) return; Ctxt tmp(b); P::mulConst(tmp, d); acc += tmp; };
  auto loop = [&]() {   // src/matmul.cpp:1022-1057 and 1097-1142, one partition
    Ctxt acc(pubKey, ctxt.ptxtSpace);
    for (long k = 0; k < h; k++) {
      Ctxt inner(pubKey, ctxt.ptxtSpace);
      for (long j = 0; j < g; j++) {
        const long i = j + g * k;
        if (i >= D) break;
        mulAdd(inner, cache[(size_t)i], *bs[(size_t)j]);
        if (!native) mulAdd(inner, cache1[(size_t)i], *bs1[(size_t)j]);
      }
      if (k > 0) inner.smartAutomorph(genToPow(gen, g * k, m));
      acc += inner;
    }
    ctxt = acc;
  };
  auto meta_of = [&](const Ctxt& c) {
    Ctxt t(pubKey, c.ptxtSpace);
    t.primeSet = c.primeSet; t.noiseBound = c.noiseBound; t.intFactor = c.intFactor; t.ratFactor = c.ratFactor; t.ptxtMag = c.ptxtMag;
    return t;
  };
  // ---- can one call reproduce the loop?
  const bool ckks = ctxt.isCKKS();
  const long keyID = ctxt.getKeyID();
  const IndexSet special = context.getSpecialPrimes();
  std::vector<const Ctxt*> all;
  for (auto& b : bs) all.push_back(b.get());
  for (auto& b : bs1) all.push_back(b.get());
  const IndexSet S = bs[0]->primeSet;
  bool ok = !(ckks && !native) && S <= context.getCtxtPrimes() && S.disjointFrom(context.getSmallPrimes()) && S.disjointFrom(special);
  for (size_t a = 0; ok && a < all.size(); a++) {
    const Ctxt& b = *all[a];
    const bool j0 = a % (size_t)g == 0;
    ok = b.parts.size() == 2 && b.getPartIndexByHandle(SKHandle()) >= 0 && b.getPartIndexByHandle(SKHandle(1, 1, keyID)) >= 0 &&
         b.primeSet == (native || j0 ? S : (S | special)) && b.ptxtSpace == bs[0]->ptxtSpace && b.intFactor == bs[0]->intFactor;
  }
  std::vector<uint64_t> kg((size_t)h, 1), scal((size_t)h, 1);
  std::vector<const KeySwitch*> W((size_t)h, nullptr);
  std::vector<Ctxt> inner;   // metadata of each giant step's acc_inner; empty ones are skipped as addCtxt skips them
  std::vector<char> nonempty((size_t)h, 0);
  bool anyrot = false;
  long nd = 0;   // the digits of S (src/DoubleCRT.cpp:485-493)
  for (IndexSet rem = S; !empty(rem) && nd < (long)context.getDigits().size(); nd++) rem.remove(context.getDigit(nd));
  for (long k = 0; ok && k < h; k++) {
    Ctxt im(pubKey, ctxt.ptxtSpace);
    bool first = true, high = false;
    for (long j = 0; ok && j < g && j + g * k < D; j++)
      for (int list = 0; list < (native ? 1 : 2); list++) {
        const BsgsDiag& d = (list ? cache1 : cache)[(size_t)(j + g * k)];
        if (!d.c) continue;
        Ctxt t = meta_of(*(list ? bs1 : bs)[(size_t)j]);
        P::mulConstMeta(t, d);
        if (!first && ckks) { Ctxt x = meta_of(im); P::modUpMeta(x, t.primeSet); Ctxt y = t; P::modUpMeta(y, im.primeSet); if (x.ratFactor < y.ratFactor || y.ratFactor < x.ratFactor) ok = false; }
        P::addMeta(im, first, t);
        high = high || j > 0;
      }
    inner.push_back(im);
    nonempty[(size_t)k] = !first;
    if (first) continue;
    if (!native && !high) ok = false;   // acc_inner over S alone would be relinearised as the native form's
    const long kk = genToPow(gen, g * k, m);
    if (k == 0 || kk == 1) continue;
    if (!pubKey.isReachable(kk, keyID)) { ok = false; break; }
    const KeySwitch* w = pubKey.getNextKSWmatrix(kk, keyID);
    if (w->fromKey.powerOfX != kk || w->toKeyID != keyID || (long)w->b.size() < nd) { ok = false; break; }
    kg[(size_t)k] = (uint64_t)kk; W[(size_t)k] = w; anyrot = true;
    Ctxt x = im;
    x.relin_CKKS_adjust();   // metadata only: the native form has no mod-down before it
    if (ckks) { const XD r = x.ratFactor / im.ratFactor; scal[(size_t)k] = (uint64_t)std::llround(r.to_double()); }
  }
  if (!ok || !anyrot) { loop(); return; }
  // ---- the call
  const long nb = native ? g : 2 * g;
  std::vector<DoubleCRT> up;   // the extended form's j = 0 baby steps, brought to S | special (addCtxt's scaling by P)
  if (!native)
    for (const Ctxt* b : {bs[0].get(), bs1[0].get()})
      for (int pt = 0; pt < 2; pt++) { up.push_back(b->parts[(size_t)b->getPartIndexByHandle(pt ? SKHandle(1, 1, keyID) : SKHandle())].dcrt); up.back().addPrimesAndScale(special); }
  std::vector<hb_poly*> b0, b1, cs((size_t)(h * nb), nullptr), ea((size_t)(h * nd), nullptr), eb((size_t)(h * nd), nullptr);
  for (long a = 0; a < nb; a++) {
    const Ctxt& b = *(a < g ? bs : bs1)[(size_t)(a % g)];
    const long ui = a == 0 ? 0 : a == g ? 2 : -1;
    b0.push_back(!native && ui >= 0 ? up[(size_t)ui].handle() : b.parts[(size_t)b.getPartIndexByHandle(SKHandle())].dcrt.handle());
    b1.push_back(!native && ui >= 0 ? up[(size_t)ui + 1].handle() : b.parts[(size_t)b.getPartIndexByHandle(SKHandle(1, 1, keyID))].dcrt.handle());
  }
  for (long k = 0; k < h; k++) {
    for (long j = 0; j < g && j + g * k < D; j++) {
      if (cache[(size_t)(j + g * k)].c) cs[(size_t)(k * nb + j)] = cache[(size_t)(j + g * k)].c->handle();
      if (!native && cache1[(size_t)(j + g * k)].c) cs[(size_t)(k * nb + g + j)] = cache1[(size_t)(j + g * k)].c->handle();
    }
    if (W[(size_t)k]) for (long i = 0; i < nd; i++) { ea[(size_t)(k * nd + i)] = W[(size_t)k]->aHandle((size_t)i); eb[(size_t)(k * nd + i)] = W[(size_t)k]->b[(size_t)i].handle(); }
  }
  const IndexSet full = S | special;
  DoubleCRT a0(context, full), a1(context, full);
  std::vector<double> norms((size_t)h * (kNormStride8 + 2), 0.0);
  {
    hb_poly* o0[1] = {a0.handle()}; hb_poly* o1[1] = {a1.handle()};
    auto Sv = S.vec();
    check(hb_bsgs_linear_map_norm(b0.data(), b1.data(), (int)nb, 1, Sv.data(), (int)Sv.size(), native ? 0 : 1, (uint64_t)bs[0]->ptxtSpace,
                                  (int)h, kg.data(), cs.data(), scal.data(), ea.data(), eb.data(), (int)nd, o0, o1, 0, norms.data()));
  }
  // ---- metadata: the loop's, giant step by giant step in its order
  Ctxt meta(pubKey, ctxt.ptxtSpace);
  bool first = true;
  for (long k = 0; k < h; k++) {
    if (!nonempty[(size_t)k]) continue;
    Ctxt t = inner[(size_t)k];
    if (W[(size_t)k]) relinTermMeta(t, &norms[(size_t)k * (kNormStride8 + 2)], !native, *W[(size_t)k], nd, S);
    if (!first) {   // acc += term must be a plain add
      Ctxt x = meta, y = t;
      P::modUpMeta(x, t.primeSet); P::modUpMeta(y, meta.primeSet);
      if (x.ptxtSpace != y.ptxtSpace || x.intFactor != y.intFactor || (ckks && (x.ratFactor < y.ratFactor || y.ratFactor < x.ratFactor))) { loop(); return; }
    }
    P::addMeta(meta, first, t);
  }
  Ctxt out(pubKey, meta.ptxtSpace);
  out.primeSet = meta.primeSet; out.noiseBound = meta.noiseBound; out.intFactor = meta.intFactor;
  out.ratFactor = meta.ratFactor; out.ptxtMag = meta.ptxtMag;
  out.parts.emplace_back(a0, SKHandle());
  out.parts.emplace_back(a1, SKHandle(1, 1, keyID));
  ctxt = out;
}

// ---- innerProduct (src/Ctxt.cpp:2878-2893) ----------------------------------------------------------------------------
// result = sum_i v1[i] * v2[i] over the first min(|v1|, |v2|) pairs, relinearised once at the end.  Every pair is prepared as
// multLowLvl prepares it (copies brought to the common prime set getSet4Size picks).  When every prepared operand is a 2-part
// canonical ciphertext under one key, every pair lands on one prime set with one ptxtSpace, and the terms sum as a plain add
// (BGV: one intFactor; CKKS: one ratFactor), one hb_tensor_sum call forms the 3-part sum and the loop's metadata is replayed
// term by term through tensorProduct and addCtxt's metadata steps.  Otherwise the transcribed loop (multLowLvl, +=) runs.
// Either way the mirror's own reLinearize finishes, so the result has the loop's bits and metadata.
inline void innerProduct(Ctxt& result, const std::vector<Ctxt>& v1, const std::vector<Ctxt>& v2) {
  using P = BasicAutomorphPrecon;
  const size_t n = std::min(v1.size(), v2.size());
  if (n == 0) {   // Ctxt::clear (include/helib/Ctxt.h:1347-1355)
    result.parts.clear(); result.primeSet = result.context.getCtxtPrimes(); result.noiseBound = XD(0.0);
    result.intFactor = 1; result.ratFactor = XD(1.0); result.ptxtMag = XD(1.0);
    return;
  }
  auto loop = [&]() {
    result = v1[0];
    result.multLowLvl(v2[0]);
    for (size_t i = 1; i < n; i++) { Ctxt tmp = v1[i]; tmp.multLowLvl(v2[i]); result += tmp; }
    result.reLinearize();
  };
  auto meta_of = [](const Ctxt& c) {
    Ctxt t(c.pubKey, c.ptxtSpace);
    t.primeSet = c.primeSet; t.noiseBound = c.noiseBound; t.intFactor = c.intFactor; t.ratFactor = c.ratFactor; t.ptxtMag = c.ptxtMag;
    return t;
  };
  // ---- the prepared pairs, and can one call reproduce the loop?
  const KeyInfo& pubKey = result.pubKey;
  const bool ckks = v1[0].isCKKS();
  const long keyID = v1[0].getKeyID();
  std::vector<Ctxt> x, y;
  x.reserve(n); y.reserve(n);
  Ctxt meta(pubKey, v1[0].ptxtSpace);
  bool ok = true, first = true;
  for (size_t i = 0; ok && i < n; i++) {
    const Ctxt& a = v1[i];
    const Ctxt& b = v2[i];
    // the cases where multLowLvl returns early or throws take the loop
    if (&a.pubKey != &pubKey || &b.pubKey != &pubKey || a.isEmpty() || b.isEmpty() || a.isCKKS() != ckks || b.isCKKS() != ckks ||
        (ckks ? (a.ptxtSpace != 1 || b.ptxtSpace != 1) : std::gcd(a.ptxtSpace, b.ptxtSpace) <= 1)) { ok = false; break; }
    x.push_back(a); y.push_back(b);
    x.back().bringToCommonSet(y.back());
    for (const Ctxt* c : {&x.back(), &y.back()})
      ok = ok && c->parts.size() == 2 && c->inCanonicalForm(keyID) && c->getKeyID() == keyID;
    if (!ok) break;
    Ctxt t(pubKey, x.back().ptxtSpace);   // tensorProduct's metadata (its part loop has nothing to do on metadata-only operands)
    t.tensorProduct(meta_of(x.back()), meta_of(y.back()));
    if (!first && (!(t.primeSet == meta.primeSet) || t.ptxtSpace != meta.ptxtSpace || (!ckks && t.intFactor != meta.intFactor) ||
                   (ckks && (t.ratFactor < meta.ratFactor || meta.ratFactor < t.ratFactor)))) { ok = false; break; }
    P::addMeta(meta, first, t);
  }
  if (!ok) { loop(); return; }
  // ---- the call
  const IndexSet S = meta.primeSet;
  std::vector<hb_poly*> a0, a1, b0, b1;
  for (size_t i = 0; i < n; i++) {
    a0.push_back(x[i].parts[0].dcrt.handle()); a1.push_back(x[i].parts[1].dcrt.handle());
    b0.push_back(y[i].parts[0].dcrt.handle()); b1.push_back(y[i].parts[1].dcrt.handle());
  }
  DoubleCRT o0(result.context, S), o1(result.context, S), o2(result.context, S);
  {
    hb_poly* p0[1] = {o0.handle()}; hb_poly* p1[1] = {o1.handle()}; hb_poly* p2[1] = {o2.handle()};
    auto Sv = S.vec();
    check(hb_tensor_sum(a0.data(), a1.data(), b0.data(), b1.data(), (int)n, 1, Sv.data(), (int)Sv.size(), p0, p1, p2, 0));
  }
  const SKHandle s1(1, 1, keyID);
  SKHandle s2; s2.mul(s1, s1);
  Ctxt out = meta;
  out.parts.emplace_back(o0, SKHandle());
  out.parts.emplace_back(o1, s1);
  out.parts.emplace_back(o2, s2);
  result = out;
  result.reLinearize();
}

// ---- BlockMatMul1DExec::mul's non-iterative branches (src/matmul.cpp:1663-1976) ------------------------------------
// A GF(p)-linear map on slots of degree d along a dimension of size D with generator gen, both dimensions' strategy FULL
// and one thread (one PartitionInfo interval): ctxt becomes sum_j sigma_{k1_j}( sum_i cache[i*d1 + j] * rot_{k0_i}(ctxt) )
// (+ the same sum over cache1, rotated by gen^-D, for a bad dimension: cache1 non-empty).  Strategy +1 (D >= d) hoists
// k0_i = gen^i, i < D, and rotates by the Frobenius k1_j = p^j, j < d; strategy -1 the other way round.  The map runs as one
// hb_block_linear_map_norm call, with the loop's bits and its metadata (noise, factors, prime set) replayed term by term
// from the norms the call returns.  The transcribed loop runs instead wherever one call cannot reproduce it: a ciphertext
// that is not 2-part canonical after cleanUp, an amount whose matrix is not direct, an outer sum that is not over
// S | special (so smartAutomorph would not mod down), sums that would not be a plain add, or no term at all.  The
// iterative (HELIB_KSS_MIN) branches are not taken.  BGV only: HElib has no CKKS block executor.
inline void BlockMatMul1D(Ctxt& ctxt, long gen, long D, long d, const std::vector<BsgsDiag>& cache, const std::vector<BsgsDiag>& cache1 = {}) {
  using P = BasicAutomorphPrecon;
  if (ctxt.isCKKS()) throw LogicError("BlockMatMul1DExec: not implemented for CKKS");
  if (D <= 0 || d <= 0 || (long)cache.size() != D * d || (!cache1.empty() && (long)cache1.size() != D * d))
    throw InvalidArgument("BlockMatMul1D: one block per (i, j)");
  const bool bad = !cache1.empty();
  const Context& context = ctxt.context;
  const KeyInfo& pubKey = ctxt.pubKey;
  const long m = context.getM();
  const long p = context.getP();
  const bool plus = D >= d;
  const long d0 = plus ? D : d, d1 = plus ? d : D;
  std::vector<long> k0((size_t)d0), k1((size_t)d1);
  for (long i = 0; i < d0; i++) k0[(size_t)i] = plus ? genToPow(gen, i, m) : genToPow(p, i, m);
  for (long j = 0; j < d1; j++) k1[(size_t)j] = plus ? genToPow(p, j, m) : genToPow(gen, j, m);
  const long kf = genToPow(gen, -D, m);
  ctxt.cleanUp();
  auto mulAdd = [&](Ctxt& acc, const BsgsDiag& c, const Ctxt& r) { if (!c.c) return; Ctxt tmp(r); P::mulConst(tmp, c); acc += tmp; };
  auto loop = [&]() {   // src/matmul.cpp:1782-1868 and 1869-1974, FULL strategies, one thread
    BasicAutomorphPrecon precon(ctxt);
    std::vector<Ctxt> acc((size_t)d1, Ctxt(pubKey, ctxt.ptxtSpace)), acc1(bad ? (size_t)d1 : 0, Ctxt(pubKey, ctxt.ptxtSpace));
    for (long i = 0; i < d0; i++) {
      std::shared_ptr<Ctxt> r = precon.automorph(k0[(size_t)i]);
      for (long j = 0; j < d1; j++) {
        mulAdd(acc[(size_t)j], cache[(size_t)(i * d1 + j)], *r);
        if (bad) mulAdd(acc1[(size_t)j], cache1[(size_t)(i * d1 + j)], *r);
      }
    }
    Ctxt sum(pubKey, ctxt.ptxtSpace), sum1(pubKey, ctxt.ptxtSpace);
    for (long j = 0; j < d1; j++) {
      if (j > 0) { acc[(size_t)j].smartAutomorph(k1[(size_t)j]); if (bad) acc1[(size_t)j].smartAutomorph(k1[(size_t)j]); }
      sum += acc[(size_t)j];
      if (bad) sum1 += acc1[(size_t)j];
    }
    if (bad) { sum1.smartAutomorph(kf); sum += sum1; }
    ctxt = sum;
  };
  // ---- can one call reproduce the loop?
  const long keyID = ctxt.getKeyID();
  const IndexSet special = context.getSpecialPrimes();
  const IndexSet S = ctxt.primeSet;
  const IndexSet full = S | special;
  bool ok = ctxt.parts.size() == 2 && ctxt.getPartIndexByHandle(SKHandle()) >= 0 && ctxt.getPartIndexByHandle(SKHandle(1, 1, keyID)) >= 0 &&
            S <= context.getCtxtPrimes() && S.disjointFrom(context.getSmallPrimes()) && S.disjointFrom(special);
  if (!ok) { loop(); return; }
  long nd = 0;   // the digits of S (src/DoubleCRT.cpp:485-493)
  for (IndexSet rem = S; !empty(rem) && nd < (long)context.getDigits().size(); nd++) rem.remove(context.getDigit(nd));
  auto direct = [&](long k) -> const KeySwitch* {
    if (k == 1) return nullptr;
    if (!pubKey.isReachable(k, keyID)) { ok = false; return nullptr; }
    const KeySwitch* w = pubKey.getNextKSWmatrix(k, keyID);
    if (w->fromKey.powerOfX != k || w->toKeyID != keyID || (long)w->b.size() < nd) ok = false;
    return w;
  };
  std::vector<const KeySwitch*> W0((size_t)d0), W1((size_t)d1);
  for (long i = 0; i < d0; i++) W0[(size_t)i] = direct(k0[(size_t)i]);
  for (long j = 1; j < d1; j++) W1[(size_t)j] = direct(k1[(size_t)j]);
  const KeySwitch* Wf = bad ? direct(kf) : nullptr;
  if (!ok) { loop(); return; }
  BasicAutomorphPrecon precon(ctxt);
  const Ctxt& cl = precon.cleaned();
  auto meta_of = [&](const Ctxt& c) {
    Ctxt t(pubKey, c.ptxtSpace);
    t.primeSet = c.primeSet; t.noiseBound = c.noiseBound; t.intFactor = c.intFactor; t.ratFactor = c.ratFactor; t.ptxtMag = c.ptxtMag;
    return t;
  };
  auto rot_meta = [&](long i) {   // BasicAutomorphPrecon::automorph(k0_i), metadata only
    if (k0[(size_t)i] == 1) return meta_of(cl);
    Ctxt t(pubKey, cl.ptxtSpace);
    t.noiseBound = precon.hoistNoise(); t.intFactor = cl.intFactor; t.primeSet = full;
    return t;
  };
  // the outer sums' metadata before their smartAutomorph: set 1 at n1 + j
  const int nsets = bad ? 2 : 1;
  std::vector<Ctxt> outer;
  std::vector<char> nonempty;
  bool any = false;
  for (int set = 0; set < nsets; set++)
    for (long j = 0; j < d1; j++) {
      Ctxt a(pubKey, cl.ptxtSpace);
      bool first = true;
      for (long i = 0; i < d0; i++) {
        const BsgsDiag& c = (set ? cache1 : cache)[(size_t)(i * d1 + j)];
        if (!c.c) continue;
        Ctxt t = rot_meta(i);
        P::mulConstMeta(t, c);
        P::addMeta(a, first, t);
      }
      outer.push_back(a); nonempty.push_back(!first);
      any = any || !first;
      if (!first && j > 0 && k1[(size_t)j] != 1 && !(a.primeSet == full)) ok = false;
    }
  if (!ok || !any) { loop(); return; }
  // ---- the call
  std::vector<hb_poly*> dg, cs((size_t)(d0 * d1), nullptr), cs1(bad ? (size_t)(d0 * d1) : 0, nullptr);
  std::vector<hb_poly*> e0a((size_t)(d0 * nd), nullptr), e0b((size_t)(d0 * nd), nullptr), e1a((size_t)(d1 * nd), nullptr), e1b((size_t)(d1 * nd), nullptr);
  std::vector<hb_poly*> efa((size_t)nd, nullptr), efb((size_t)nd, nullptr);
  for (const DoubleCRT& x : precon.digits()) dg.push_back(x.handle());
  for (long i = 0; i < d0 * d1; i++) {
    if (cache[(size_t)i].c) cs[(size_t)i] = cache[(size_t)i].c->handle();
    if (bad && cache1[(size_t)i].c) cs1[(size_t)i] = cache1[(size_t)i].c->handle();
  }
  auto keys = [&](const KeySwitch* w, hb_poly** a, hb_poly** b) { if (w) for (long i = 0; i < nd; i++) { a[i] = w->aHandle((size_t)i); b[i] = w->b[(size_t)i].handle(); } };
  for (long i = 0; i < d0; i++) keys(W0[(size_t)i], &e0a[(size_t)(i * nd)], &e0b[(size_t)(i * nd)]);
  for (long j = 0; j < d1; j++) keys(W1[(size_t)j], &e1a[(size_t)(j * nd)], &e1b[(size_t)(j * nd)]);
  keys(Wf, efa.data(), efb.data());
  std::vector<uint64_t> u0(k0.begin(), k0.end()), u1(k1.begin(), k1.end());
  const long T = bad ? 2 * d1 + 1 : d1;
  std::vector<double> norms((size_t)T * (kNormStride8 + 2), 0.0);
  DoubleCRT a0(context, full), a1(context, full);
  {
    hb_poly* c0[1] = {cl.parts[(size_t)cl.getPartIndexByHandle(SKHandle())].dcrt.handle()};
    hb_poly* c1[1] = {cl.parts[(size_t)cl.getPartIndexByHandle(SKHandle(1, 1, keyID))].dcrt.handle()};
    hb_poly* o0[1] = {a0.handle()}; hb_poly* o1[1] = {a1.handle()};
    auto Sv = S.vec();
    check(hb_block_linear_map_norm(dg.data(), (int)dg.size(), 1, Sv.data(), (int)Sv.size(), c0, c1, (uint64_t)cl.ptxtSpace,
                                   (int)d0, u0.data(), e0a.data(), e0b.data(), (int)d1, u1.data(), e1a.data(), e1b.data(),
                                   cs.data(), bad ? cs1.data() : nullptr, (uint64_t)kf, efa.data(), efb.data(), (int)nd, o0, o1, 0, norms.data()));
  }
  // ---- metadata: the loop's, term by term in its order
  auto plain = [&](const Ctxt& a, const Ctxt& b) {   // a += b must be a plain add
    Ctxt x = a, y = b;
    P::modUpMeta(x, b.primeSet); P::modUpMeta(y, a.primeSet);
    return x.ptxtSpace == y.ptxtSpace && x.intFactor == y.intFactor;
  };
  Ctxt sums[2] = {Ctxt(pubKey, cl.ptxtSpace), Ctxt(pubKey, cl.ptxtSpace)};
  bool firsts[2] = {true, true};
  for (int set = 0; set < nsets; set++)
    for (long j = 0; j < d1; j++) {
      const size_t e = (size_t)(set * d1 + j);
      if (!nonempty[e]) continue;
      Ctxt t = outer[e];
      if (j > 0 && W1[(size_t)j]) relinTermMeta(t, &norms[e * (kNormStride8 + 2)], true, *W1[(size_t)j], nd, S);
      if (!firsts[set] && !plain(sums[set], t)) { loop(); return; }
      P::addMeta(sums[set], firsts[set], t);
    }
  Ctxt meta = sums[0];
  bool first = firsts[0];
  if (bad && !firsts[1]) {
    Ctxt t = sums[1];
    if (Wf) {
      if (!(t.primeSet == full)) { loop(); return; }
      relinTermMeta(t, &norms[(size_t)(2 * d1) * (kNormStride8 + 2)], true, *Wf, nd, S);
    }
    if (!first && !plain(meta, t)) { loop(); return; }
    P::addMeta(meta, first, t);
  }
  if (!(meta.primeSet == full)) { loop(); return; }   // only unrotated terms over S: the loop's result stays over S
  Ctxt out(pubKey, meta.ptxtSpace);
  out.primeSet = meta.primeSet; out.noiseBound = meta.noiseBound; out.intFactor = meta.intFactor;
  out.ratFactor = meta.ratFactor; out.ptxtMag = meta.ptxtMag;
  out.parts.emplace_back(a0, SKHandle());
  out.parts.emplace_back(a1, SKHandle(1, 1, keyID));
  ctxt = out;
}

// ---- MatMulFullExec::mul (src/matmul.cpp:2132-2273) and MatMul1DExec::mul's hoisted branches (:1226-1283) ----------
constexpr long kBsgsMulThresh = 50;   // HELIB_BSGS_MUL_THRESH (= HELIB_KEYSWITCH_THRESH): larger dimensions take BSGS
// One dimension of a full-matrix map: its generator, order D and whether it is native.  A bad outer dimension also has the
// masks getMask_zzX(dim, i) as constants with their sizes, masks[i] for 1 <= i < D (masks[0] is not used).
struct FullDim { long gen; long D; bool native; std::vector<BsgsDiag> masks; };

namespace detail {
// MatMul1DExec::mul's hoisted branches transcribed (FULL strategy, one thread): cleanUp, then
//   acc = sum_i cache[i] * automorph(gen^i)  (+ smartAutomorph(gen^-D) of sum_i cache1[i] * automorph(gen^i), bad)
inline void matmul1dLoop(Ctxt& ctxt, long gen, long D, const std::vector<BsgsDiag>& cache, const std::vector<BsgsDiag>* cache1) {
  const long m = ctxt.context.getM();
  ctxt.cleanUp();
  BasicAutomorphPrecon precon(ctxt);
  Ctxt acc(ctxt.pubKey, ctxt.ptxtSpace), acc1(ctxt.pubKey, ctxt.ptxtSpace);
  for (long i = 0; i < D; i++) {
    const BsgsDiag& c = cache[(size_t)i];
    const BsgsDiag* c1 = cache1 ? &(*cache1)[(size_t)i] : nullptr;
    if (!c.c && !(c1 && c1->c)) continue;
    std::shared_ptr<Ctxt> r = precon.automorph(genToPow(gen, i, m));
    if (c.c) { Ctxt t(*r); BasicAutomorphPrecon::mulConst(t, c); acc += t; }
    if (c1 && c1->c) { Ctxt t(*r); BasicAutomorphPrecon::mulConst(t, *c1); acc1 += t; }
  }
  if (cache1 && !acc1.isEmpty()) { acc1.smartAutomorph(genToPow(gen, -D, m)); acc += acc1; }
  ctxt = acc;
}
// The metadata modDownToSet(S) gives a ciphertext over S | special, from the device's ||delta/P|| of its two parts
// (nr[kNormStride8], nr[kNormStride8 + 1])
inline void modDownMeta(Ctxt& t, const double* nr, const IndexSet& S) {
  const XD addedNoise = XD(nr[kNormStride8]) + XD(nr[kNormStride8 + 1]) * XD::exp(std::log(t.pubKey.skBound));
  const XD f = XD::exp(t.pubKey.logOfProduct(t.context.getSpecialPrimes()));
  t.ratFactor = t.ratFactor / f;
  t.noiseBound = t.noiseBound / f;
  t.noiseBound = t.noiseBound + addedNoise;
  t.primeSet = S;
}
// sum_l MatMul1DExec::mul(leaves[l]) for leaves of one hoisted dimension (D <= kBsgsMulThresh), the cache of leaf l at
// cache[l] (cache1[l] for a bad dimension): one hb_full_linear_map_leaves_norm call, and the loop's metadata replayed term
// by term, leaf by leaf, from the norms it returns.  Returns false, with out untouched, where one call cannot reproduce the
// loop: CKKS, a leaf that is not 2-part canonical under the first leaf's key or whose cleanUp would not land on the common
// set S, an amount without a direct matrix, sums that would not be a plain add, or a result not over S | special.
inline bool leavesFused(Ctxt& out, const std::vector<const Ctxt*>& leaves, long gen, long D,
                        const std::vector<const std::vector<BsgsDiag>*>& cache, const std::vector<const std::vector<BsgsDiag>*>& cache1) {
  using P = BasicAutomorphPrecon;
  if (leaves.empty() || D > kBsgsMulThresh) return false;
  const Ctxt& c0 = *leaves[0];
  if (c0.isCKKS()) return false;
  const Context& context = c0.context;
  const KeyInfo& pubKey = c0.pubKey;
  const long m = context.getM();
  const bool bad = !cache1.empty();
  const long keyID = c0.getKeyID();
  const IndexSet special = context.getSpecialPrimes();
  const IndexSet S = c0.primeSet / special;
  const IndexSet full = S | special;
  if (empty(S) || !(S <= context.getCtxtPrimes()) || !S.disjointFrom(context.getSmallPrimes())) return false;
  const long nl = (long)leaves.size();
  std::vector<int32_t> ext((size_t)nl);
  for (long l = 0; l < nl; l++) {
    const Ctxt& x = *leaves[(size_t)l];
    if (&x.pubKey != &pubKey || x.ptxtSpace != c0.ptxtSpace || x.parts.size() != 2 || x.getPartIndexByHandle(SKHandle()) < 0 ||
        x.getPartIndexByHandle(SKHandle(1, 1, keyID)) < 0 || !(x.primeSet == S || x.primeSet == full))
      return false;
    ext[(size_t)l] = x.primeSet == full;
  }
  long nd = 0;   // the digits of S (src/DoubleCRT.cpp:485-493)
  for (IndexSet rem = S; !empty(rem) && nd < (long)context.getDigits().size(); nd++) rem.remove(context.getDigit(nd));
  bool ok = true;
  auto direct = [&](long k) -> const KeySwitch* {
    if (k == 1) return nullptr;
    if (!pubKey.isReachable(k, keyID)) { ok = false; return nullptr; }
    const KeySwitch* w = pubKey.getNextKSWmatrix(k, keyID);
    if (w->fromKey.powerOfX != k || w->toKeyID != keyID || (long)w->b.size() < nd) ok = false;
    return w;
  };
  std::vector<long> k((size_t)D);
  std::vector<const KeySwitch*> W((size_t)D);
  for (long t = 0; t < D; t++) { k[(size_t)t] = genToPow(gen, t, m); W[(size_t)t] = direct(k[(size_t)t]); }
  const long kf = genToPow(gen, -D, m);
  const KeySwitch* Wf = bad ? direct(kf) : nullptr;
  if (!ok) return false;
  // ---- the call
  std::vector<hb_poly*> x0((size_t)nl), x1((size_t)nl), cs((size_t)(nl * D), nullptr), cs1(bad ? (size_t)(nl * D) : 0, nullptr);
  std::vector<hb_poly*> ea((size_t)(D * nd), nullptr), eb((size_t)(D * nd), nullptr), efa((size_t)nd, nullptr), efb((size_t)nd, nullptr);
  for (long l = 0; l < nl; l++) {
    const Ctxt& x = *leaves[(size_t)l];
    x0[(size_t)l] = x.parts[(size_t)x.getPartIndexByHandle(SKHandle())].dcrt.handle();
    x1[(size_t)l] = x.parts[(size_t)x.getPartIndexByHandle(SKHandle(1, 1, keyID))].dcrt.handle();
    for (long t = 0; t < D; t++) {
      if ((*cache[(size_t)l])[(size_t)t].c) cs[(size_t)(l * D + t)] = (*cache[(size_t)l])[(size_t)t].c->handle();
      if (bad && (*cache1[(size_t)l])[(size_t)t].c) cs1[(size_t)(l * D + t)] = (*cache1[(size_t)l])[(size_t)t].c->handle();
    }
  }
  auto keys = [&](const KeySwitch* w, hb_poly** a, hb_poly** b) { if (w) for (long i = 0; i < nd; i++) { a[i] = w->aHandle((size_t)i); b[i] = w->b[(size_t)i].handle(); } };
  for (long t = 0; t < D; t++) keys(W[(size_t)t], &ea[(size_t)(t * nd)], &eb[(size_t)(t * nd)]);
  keys(Wf, efa.data(), efb.data());
  std::vector<uint64_t> ku(k.begin(), k.end());
  const long T = bad ? 2 * nl : nl;
  std::vector<double> norms((size_t)T * (kNormStride8 + 2), 0.0);
  DoubleCRT a0(context, full), a1(context, full);
  {
    hb_poly* o0[1] = {a0.handle()}; hb_poly* o1[1] = {a1.handle()};
    auto Sv = S.vec();
    check(hb_full_linear_map_leaves_norm(x0.data(), x1.data(), (int)nl, 1, ext.data(), Sv.data(), (int)Sv.size(), (uint64_t)c0.ptxtSpace,
                                         (int)D, ku.data(), ea.data(), eb.data(), cs.data(), bad ? cs1.data() : nullptr, (uint64_t)kf,
                                         efa.data(), efb.data(), (int)nd, o0, o1, 0, norms.data()));
  }
  // ---- metadata: the loop's, leaf by leaf and term by term in its order
  auto meta_of = [&](const Ctxt& c) {
    Ctxt t(pubKey, c.ptxtSpace);
    t.primeSet = c.primeSet; t.noiseBound = c.noiseBound; t.intFactor = c.intFactor; t.ratFactor = c.ratFactor; t.ptxtMag = c.ptxtMag;
    return t;
  };
  auto plain = [&](const Ctxt& a, const Ctxt& b) {   // a += b must be a plain add
    Ctxt x = a, y = b;
    P::modUpMeta(x, b.primeSet); P::modUpMeta(y, a.primeSet);
    return x.ptxtSpace == y.ptxtSpace && x.intFactor == y.intFactor;
  };
  XD max_ks_noise(0.0);
  for (const KeySwitch& ks : pubKey.keySwitching) if (max_ks_noise < ks.noiseBound) max_ks_noise = ks.noiseBound;
  const double logP = pubKey.logOfProduct(special);
  Ctxt meta(pubKey, c0.ptxtSpace);
  bool first = true;
  for (long l = 0; l < nl; l++) {
    const double* nr = &norms[(size_t)l * (kNormStride8 + 2)];
    Ctxt cl = meta_of(*leaves[(size_t)l]);   // cleanUp
    if (ext[(size_t)l]) modDownMeta(cl, nr, S);
    XD addedNoise(0.0);                        // BasicAutomorphPrecon's hoisting noise
    for (long i = 0; i < nd; i++) addedNoise = addedNoise + XD::exp(nr[i]);
    addedNoise = addedNoise * max_ks_noise;
    XD hn = cl.noiseBound * XD::exp(logP);
    hn = hn + addedNoise;
    Ctxt sums[2] = {Ctxt(pubKey, cl.ptxtSpace), Ctxt(pubKey, cl.ptxtSpace)};
    bool firsts[2] = {true, true};
    for (long t = 0; t < D; t++)
      for (int set = 0; set < (bad ? 2 : 1); set++) {
        const BsgsDiag& c = (*(set ? cache1 : cache)[(size_t)l])[(size_t)t];
        if (!c.c) continue;
        Ctxt r = meta_of(cl);
        if (k[(size_t)t] != 1) { r = Ctxt(pubKey, cl.ptxtSpace); r.noiseBound = hn; r.intFactor = cl.intFactor; r.primeSet = full; }
        P::mulConstMeta(r, c);
        if (!firsts[set] && !plain(sums[set], r)) return false;
        P::addMeta(sums[set], firsts[set], r);
      }
    if (bad && !firsts[1]) {
      Ctxt t = sums[1];
      if (Wf) {
        if (!(t.primeSet == full)) return false;
        relinTermMeta(t, &norms[(size_t)(nl + l) * (kNormStride8 + 2)], true, *Wf, nd, S);
      }
      if (!firsts[0] && !plain(sums[0], t)) return false;
      P::addMeta(sums[0], firsts[0], t);
    }
    if (firsts[0]) continue;   // an empty leaf: acc += 0 changes nothing
    if (!first && !plain(meta, sums[0])) return false;
    P::addMeta(meta, first, sums[0]);
  }
  if (first || !(meta.primeSet == full)) return false;
  Ctxt res(pubKey, meta.ptxtSpace);
  res.primeSet = meta.primeSet; res.noiseBound = meta.noiseBound; res.intFactor = meta.intFactor;
  res.ratFactor = meta.ratFactor; res.ptxtMag = meta.ptxtMag;
  res.parts.emplace_back(a0, SKHandle());
  res.parts.emplace_back(a1, SKHandle(1, 1, keyID));
  out = res;
  return true;
}
}  // namespace detail

// MatMul1DExec::mul's hoisted branches (FULL strategy, one thread; src/matmul.cpp:1226-1283): ctxt becomes
// sum_i cache[i] * rot_{gen^i}(ctxt) (+ smartAutomorph(gen^-D) of sum_i cache1[i] * rot_{gen^i}(ctxt) for a bad dimension,
// cache1 non-empty).  The native branch is BasicAutomorphPrecon::linearCombination; the bad branch is one
// hb_full_linear_map_leaves_norm call with a single leaf, with the loop's bits and metadata, or the transcribed loop where
// one call cannot reproduce it.  D > kBsgsMulThresh takes HElib's BSGS branch, hb::MatMul1DBSGS.  BGV only.
inline void MatMul1D(Ctxt& ctxt, long gen, long D, const std::vector<BsgsDiag>& cache, const std::vector<BsgsDiag>& cache1 = {}) {
  if (ctxt.isCKKS()) throw LogicError("hb::MatMul1D: BGV only (CKKS takes linearCombinationCKKS or MatMul1DBSGS)");
  if (D <= 0 || (long)cache.size() != D || (!cache1.empty() && (long)cache1.size() != D)) throw InvalidArgument("MatMul1D: one diagonal per index");
  if (D > kBsgsMulThresh) { ctxt.cleanUp(); MatMul1DBSGS(ctxt, gen, D, cache, cache1); return; }
  const long m = ctxt.context.getM();
  ctxt.cleanUp();
  if (cache1.empty()) {
    std::vector<long> k; std::vector<const DoubleCRT*> cs; std::vector<double> sz;
    for (long i = 0; i < D; i++) if (cache[(size_t)i].c) { k.push_back(genToPow(gen, i, m)); cs.push_back(cache[(size_t)i].c); sz.push_back(cache[(size_t)i].size); }
    if (k.empty()) { ctxt = Ctxt(ctxt.pubKey, ctxt.ptxtSpace); return; }
    ctxt = *BasicAutomorphPrecon(ctxt).linearCombination(k, cs, sz);
    return;
  }
  Ctxt out(ctxt.pubKey, ctxt.ptxtSpace);
  if (detail::leavesFused(out, {&ctxt}, gen, D, {&cache}, {&cache1})) { ctxt = out; return; }
  detail::matmul1dLoop(ctxt, gen, D, cache, &cache1);
}

// MatMulFullExec::mul (src/matmul.cpp:2132-2273, BGV; FULL key strategy in every dimension, one thread): cleanUp, then
// rec_mul over the dimensions sorted as MatMulDimComp sorts them (smaller order first, native before bad on ties).  The
// outer levels run as rec_mul does, with BasicAutomorphPrecon rotations (hb_automorph_keyswitch_digits) and, for a bad
// outer dimension, tmp*mask + tmp1 - tmp1*mask with tmp1 rotated from smartAutomorph(gen^-D).  leaves[idx] (leaves1[idx]
// for a bad last dimension) is the cache of leaf idx in rec_mul's order, one diagonal per index of the last dimension.
// The leaves then go through one hb_full_linear_map_leaves_norm call (hb::detail::leavesFused, shared with hb::MatMul1D),
// so the result has the transcribed loop's bits and metadata; the transcribed leaves run instead where that call cannot
// reproduce them, and a last dimension above kBsgsMulThresh takes hb::MatMul1DBSGS per leaf, as HElib's BSGS branch.
// CKKS: LogicError, as HElib (HELIB_NO_CKKS_IMPL).
inline void MatMulFull(Ctxt& ctxt, std::vector<FullDim> dims, const std::vector<std::vector<BsgsDiag>>& leaves,
                       const std::vector<std::vector<BsgsDiag>>& leaves1 = {}) {
  if (ctxt.isCKKS()) throw LogicError("MatMulFullExec: not implemented for CKKS");
  if (dims.empty()) throw InvalidArgument("MatMulFull: no dimensions");
  std::stable_sort(dims.begin(), dims.end(), [](const FullDim& a, const FullDim& b) { return a.D < b.D || (a.D == b.D && a.native && !b.native); });
  size_t nl = 1;
  for (size_t i = 0; i + 1 < dims.size(); i++) {
    nl *= (size_t)dims[i].D;
    if (!dims[i].native && (long)dims[i].masks.size() != dims[i].D) throw InvalidArgument("MatMulFull: a bad dimension needs D masks");
  }
  const FullDim& last = dims.back();
  if (leaves.size() != nl || (!last.native && leaves1.size() != nl) || (last.native && !leaves1.empty())) throw InvalidArgument("MatMulFull: one cache per leaf");
  for (size_t l = 0; l < nl; l++)
    if ((long)leaves[l].size() != last.D || (!last.native && (long)leaves1[l].size() != last.D)) throw InvalidArgument("MatMulFull: one diagonal per index");
  const long m = ctxt.context.getM();
  ctxt.cleanUp();
  // the outer levels of rec_mul; the leaf inputs in its order
  std::vector<Ctxt> L;
  L.reserve(nl);
  std::function<void(const Ctxt&, size_t)> rec = [&](const Ctxt& c, size_t di) {
    if (di + 1 == dims.size()) { L.push_back(c); return; }
    const FullDim& d = dims[di];
    if (d.native) {
      BasicAutomorphPrecon precon(c);
      for (long i = 0; i < d.D; i++) rec(*precon.automorph(genToPow(d.gen, i, m)), di + 1);
      return;
    }
    Ctxt c1(c);
    c1.smartAutomorph(genToPow(d.gen, -d.D, m));
    BasicAutomorphPrecon precon(c), precon1(c1);
    for (long i = 0; i < d.D; i++) {
      if (i == 0) { rec(c, di + 1); continue; }
      std::shared_ptr<Ctxt> tmp = precon.automorph(genToPow(d.gen, i, m)), tmp1 = precon1.automorph(genToPow(d.gen, i, m));
      const BsgsDiag& mk = d.masks[(size_t)i];
      tmp->multByConstant(*mk.c, mk.size);
      *tmp += *tmp1;
      tmp1->multByConstant(*mk.c, mk.size);
      tmp->addCtxt(*tmp1, /*negative=*/true);
      rec(*tmp, di + 1);
    }
  };
  rec(ctxt, 0);
  // the leaves
  Ctxt acc(ctxt.pubKey, ctxt.ptxtSpace);
  if (last.D <= kBsgsMulThresh) {
    std::vector<const Ctxt*> lp; std::vector<const std::vector<BsgsDiag>*> cp, cp1;
    for (size_t l = 0; l < nl; l++) { lp.push_back(&L[l]); cp.push_back(&leaves[l]); if (!last.native) cp1.push_back(&leaves1[l]); }
    if (detail::leavesFused(acc, lp, last.gen, last.D, cp, cp1)) { ctxt = acc; return; }
  }
  for (size_t l = 0; l < nl; l++) {   // transforms[idx].mul(tmp); acc += tmp
    Ctxt tmp(L[l]);
    if (last.D > kBsgsMulThresh) { tmp.cleanUp(); MatMul1DBSGS(tmp, last.gen, last.D, leaves[l], last.native ? std::vector<BsgsDiag>{} : leaves1[l]); }
    else detail::matmul1dLoop(tmp, last.gen, last.D, leaves[l], last.native ? nullptr : &leaves1[l]);
    acc += tmp;
  }
  ctxt = acc;
}

// ---- SURVEY 8f-2: the steps either side of the path ------------------------------------------------------------
// Sampling follows the reference's DISTRIBUTIONS (src/sample.cpp); its bit stream (NTL's PRG) is not restated, so
// the sampled values are an input of Encrypt below and "parity unpinned" is confined to them.
struct EncryptionSample {
  std::vector<long> r, e0, e1;
  double r_bound = 0, e0_bound = 0, e1_bound = 0;   // what sampleSmallBounded / sampleGaussianBounded return
};
// max_j |f(zeta^(2j+1))| for power-of-two m (embeddingLargestCoeff, src/norms.cpp:204-261): twist + N-point FFT on the host
inline double embeddingLargestCoeff(const std::vector<long>& f, long m) {
  const long N = m / 2;
  if (m < 4 || (m & (m - 1)) != 0) throw LogicError("embeddingLargestCoeff: host version is for power-of-two m");
  std::vector<std::complex<double>> z((size_t)N);
  const double pi = 3.14159265358979323846;
  for (long k = 0; k < N; k++) z[k] = (k < (long)f.size() ? double(f[k]) : 0.0) * std::polar(1.0, pi * double(k) / double(N));
  for (long i = 1, j = 0; i < N; i++) { long bit = N >> 1; for (; j & bit; bit >>= 1) j ^= bit; j ^= bit; if (i < j) std::swap(z[i], z[j]); }
  for (long len = 2; len <= N; len <<= 1) {
    const std::complex<double> wl = std::polar(1.0, 2 * pi / double(len));
    for (long i = 0; i < N; i += len) { std::complex<double> w(1.0, 0.0);
      for (long k = 0; k < len / 2; k++) { auto u = z[i + k], v = z[i + k + len / 2] * w; z[i + k] = u + v; z[i + k + len / 2] = u - v; w *= wl; } }
  }
  double mx = 0; for (auto& c : z) mx = std::max(mx, std::abs(c));
  return mx;
}
template <class Gen> void sampleSmall(std::vector<long>& poly, long n, Gen& g) {   // src/sample.cpp:67-103 (prob = 1/2)
  poly.assign((size_t)n, 0);
  for (long i = 0; i < n; i++) { unsigned u = (unsigned)(g() & 3u); poly[i] = (u & 1u) ? long(u & 2u) - 1 : 0; }
}
template <class Gen> void sampleGaussian(std::vector<long>& poly, long n, double stdev, Gen& g) {   // src/sample.cpp:140-187
  std::normal_distribution<double> d(0.0, stdev);
  poly.assign((size_t)n, 0);
  for (long i = 0; i < n; i++) poly[i] = std::lround(d(g));
}
template <class Gen> double sampleSmallBounded(std::vector<long>& poly, const Context& ctx, Gen& g) {   // src/sample.cpp:342-396
  const long phim = ctx.getPhiM();
  const double bound = std::sqrt(phim * std::log(double(phim)) / 2.0);
  double val; long count = 0;
  do { sampleSmall(poly, phim, g); val = embeddingLargestCoeff(poly, ctx.getM()); } while (++count < 1000 && val > bound);
  if (val > bound) throw RuntimeError("Error: sampleSmallBounded, after 1000 trials, still val > bound");
  return bound;
}
template <class Gen> double sampleGaussianBounded(std::vector<long>& poly, const Context& ctx, double stdev, Gen& g) {   // src/sample.cpp:459-512
  const long phim = ctx.getPhiM();
  const double bound = stdev * std::sqrt(phim * std::log(double(phim)));
  double val; long count = 0;
  do { sampleGaussian(poly, phim, stdev, g); val = embeddingLargestCoeff(poly, ctx.getM()); } while (++count < 1000 && val > bound);
  if (val > bound) throw RuntimeError("Error: sampleGaussianBounded, after 1000 trials, still val > bound");
  return bound;
}
template <class Gen> EncryptionSample drawEncryptionSample(const Context& ctx, double stdev, Gen& g) {
  EncryptionSample s;
  s.r_bound = sampleSmallBounded(s.r, ctx, g);
  s.e0_bound = sampleGaussianBounded(s.e0, ctx, stdev, g);
  s.e1_bound = sampleGaussianBounded(s.e1, ctx, stdev, g);
  return s;
}

// PubKey::Encrypt, BGV branch (src/keys.cpp:358-488): ctxt = r*pk + p*(e0,e1) + (ptxt_fixed, 0).  Three polynomials
// cross the bus as phi(m) words each; the products, sums and transforms run on the device.
// tieCoin stands for NTL::RandomBnd(2) in balanced_MulMod (src/NumbTh.cpp:876-892, even ptxtSpace only).
inline long Encrypt(Ctxt& ctxt, const Ctxt& pubEncrKey, const std::vector<long>& ptxt, long ptxtSpace,
                    const EncryptionSample& smp, const std::function<bool()>& tieCoin = [] { return false; }) {
  const Context& context = pubEncrKey.context;
  if (&ctxt.pubKey != &pubEncrKey.pubKey) throw LogicError("Public key and context public key mismatch");
  if (pubEncrKey.isCKKS()) throw LogicError("Encrypt: BGV only (CKKSencrypt is separate in the reference)");
  if (pubEncrKey.parts.size() != 2) throw LogicError("Encrypt: public encryption key must have two parts");
  if (ptxtSpace != pubEncrKey.ptxtSpace) {
    ptxtSpace = std::gcd(ptxtSpace, pubEncrKey.ptxtSpace);
    if (ptxtSpace <= 1) throw RuntimeError("Plaintext-space mismatch on encryption");
  }
  const long phim = context.getPhiM();
  if ((long)ptxt.size() > phim) throw InvalidArgument("plaintext degree >= phi(m)");
  ctxt = pubEncrKey;
  const IndexSet& S = ctxt.primeSet;
  DoubleCRT r(smp.r, context, S);
  ctxt.noiseBound = XD(smp.r_bound) * pubEncrKey.noiseBound;
  unsigned long QmodP = 1;
  for (long i : S) QmodP = (unsigned long)(((unsigned __int128)QmodP * (unsigned long)(context.ithPrime(i) % ptxtSpace)) % (unsigned long)ptxtSpace);
  for (size_t i = 0; i < ctxt.parts.size(); i++) {
    const std::vector<long>& ei = i == 0 ? smp.e0 : smp.e1;
    std::vector<long> c((size_t)phim, 0);
    for (long k = 0; k < phim && k < (long)ei.size(); k++) {
      const __int128 v = (__int128)ei[k] * ptxtSpace;
      if (v > ((__int128)1 << 61) || v < -((__int128)1 << 61)) throw InvalidArgument("Encrypt: ptxtSpace * e does not fit a word");
      c[k] = (long)v;
    }
    if (i == 0)
      for (long k = 0; k < (long)ptxt.size(); k++) {   // ptxt_fixed = balanced(ptxt * (Q mod p) mod p)  (:453-455)
        long t = ptxt[k] % ptxtSpace; if (t < 0) t += ptxtSpace;
        long f = (long)(((unsigned __int128)(unsigned long)t * QmodP) % (unsigned long)ptxtSpace);
        if (f > ptxtSpace / 2 || (ptxtSpace % 2 == 0 && f == ptxtSpace / 2 && tieCoin())) f -= ptxtSpace;
        c[k] += f;
      }
    DoubleCRT e(c, context, S);                    // p*e_i (+ ptxt_fixed)
    e.mulAdd(ctxt.parts[i].dcrt, r);               // + pk_i * r      (:416,443)
    ctxt.parts[i].dcrt = e;
    XD e_bound = XD((i == 0 ? smp.e0_bound : smp.e1_bound) * double(ptxtSpace));
    if (i == 1) e_bound = e_bound * XD(pubEncrKey.pubKey.skBound);
    ctxt.noiseBound = ctxt.noiseBound + e_bound;
  }
  ctxt.noiseBound = ctxt.noiseBound + XD(pubEncrKey.pubKey.noiseBoundForMod(ptxtSpace, phim));   // (:462,476)
  ctxt.ptxtSpace = ptxtSpace;
  ctxt.intFactor = 1;
  return ptxtSpace;
}

// SecKey::Decrypt (src/keys.cpp:1327-1400).  sKeys[id] = the secret key polynomials in DoubleCRT form.
// BGV: plaintxt in [0, ptxtSpace).  CKKS (or f_limbs != nullptr): the integer polynomial before reduction is
// returned as phi(m) x L two's-complement limbs.
inline void Decrypt(std::vector<long>& plaintxt, const Ctxt& c, const std::vector<DoubleCRT>& sKeys,
                    std::vector<uint64_t>* f_limbs = nullptr, int* L = nullptr, double polyNormBnd = 1.0) {
  if (!c.isCorrect(polyNormBnd)) throw LogicError("Decrypting with too much noise");
  const Context& context = c.context;
  const IndexSet& P = c.primeSet;
  DoubleCRT ptxt(context, P);
  for (const CtxtPart& part : c.parts) {
    if (part.skHandle.isOne()) { ptxt.Add(part.dcrt, false); continue; }
    DoubleCRT key = sKeys.at((size_t)part.skHandle.secretKeyID);
    key.addPrimes(P / key.getIndexSet());              // key.setPrimes(ptxtPrimes)  (include/helib/DoubleCRT.h:275-279)
    key.removePrimes(key.getIndexSet() / P);
    if (part.skHandle.powerOfX > 1) key.automorph(part.skHandle.powerOfX);
    if (part.skHandle.powerOfS > 1) { DoubleCRT base(key); for (long e = 1; e < part.skHandle.powerOfS; e++) key *= base; }   // Exp (src/DoubleCRT.cpp:1142-1156)
    ptxt.mulAdd(key, part.dcrt);
  }
  if (c.isCKKS() || f_limbs) {
    int l = 0; std::vector<uint64_t> limbs = ptxt.toPoly(P, false, l);
    if (f_limbs) *f_limbs = std::move(limbs);
    if (L) *L = l;
    if (c.isCKKS()) return;
  }
  const long p = c.ptxtSpace;
  long factor = 1;
  if (p > 2) {   // multiply by (intFactor * Q)^-1 mod p  (:1388-1398)
    unsigned long f = 1;
    for (long i : P) f = (unsigned long)(((unsigned __int128)f * (unsigned long)(context.ithPrime(i) % p)) % (unsigned long)p);
    long jf = c.intFactor % p; if (jf < 0) jf += p;
    f = (unsigned long)(((unsigned __int128)f * (unsigned long)jf) % (unsigned long)p);
    if (f != 1) {   // InvMod by extended Euclid
      long a = (long)f, b = p, x0 = 1, x1 = 0;
      while (b) { long q = a / b, t = a - q * b; a = b; b = t; t = x0 - q * x1; x0 = x1; x1 = t; }
      if (a != 1) throw LogicError("Decrypt: intFactor*Q not invertible mod ptxtSpace");
      factor = x0 % p; if (factor < 0) factor += p;
    }
  }
  plaintxt = ptxt.toPolyModP(P, p, factor);
}

// RLWE1 (src/keys.cpp:39-72): c0 = p*e - c1*s for a short e; returns the high-probability bound on the canonical
// embedding of the decryption.  e is drawn by sampleGaussianBounded above (the reference's distribution and rejection bound).
template <class Gen> double RLWE1(DoubleCRT& c0, const DoubleCRT& c1, const DoubleCRT& s, long p, double stdev, Gen& g) {
  if (p <= 0) throw InvalidArgument("Cannot generate RLWE instance with nonpositive p");
  const Context& context = s.getContext();
  if ((context.getM() & (context.getM() - 1)) != 0) stdev *= std::sqrt((double)context.getM());
  std::vector<long> e;
  double bound = sampleGaussianBounded(e, context, stdev, g);
  c0 = DoubleCRT(e, context, c0.getIndexSet());
  if (p > 1) { c0 *= p; bound *= p; }
  DoubleCRT tmp(c1);
  tmp.Mul(s, /*matchIndexSets=*/false);
  c0 -= tmp;
  return bound;
}
// SecKey::GenKeySWmatrix (src/keys.cpp:1159-1256): W[fromKey -> toKey] over ctxt | special primes,
// b_i = p*e_i - a_i*s + P*(prod_{j<i} Q_j)*fromKey.  fromKey = s^r(X^t) is passed in already transformed;
// drawA(a_i) fills a_i with uniform rows (the reference: a[i].randomize() under SetSeed(prgSeed); DoubleCRT::randomize here).
namespace detail {
inline KeySwitch keySWmatrixHead(const SKHandle& fromHandle, long toKeyID, long p, bool ckks) {
  KeySwitch W; W.fromKey = fromHandle; W.toKeyID = toKeyID;
  if (ckks) p = 1;
  else if (p < 2) throw LogicError("Invalid p value found generating BGV key-switching matrix");
  W.ptxtSpace = p;
  return W;
}
// b_i = p*e_i - a_i*s + P*(prod_{j<i} Q_j)*fromKey for the a_i already in W (src/keys.cpp:1208-1245)
template <class Gen>
void keySWmatrixB(KeySwitch& W, const Context& context, DoubleCRT fromKey, const DoubleCRT& toKey, double stdev, Gen& g) {
  const IndexSet all = context.getCtxtPrimes() | context.getSpecialPrimes();
  const size_t n = W.a.size();
  for (size_t i = 0; i < n; i++) { W.b.emplace_back(context, all); W.noiseBound = XD(RLWE1(W.b[i], W.a[i], toKey, W.ptxtSpace, stdev, g)); }
  fromKey.addPrimes(all / fromKey.getIndexSet());
  fromKey.multiplyByPrimes(context.getSpecialPrimes());
  for (size_t i = 0; i < n; i++) { W.b[i] += fromKey; fromKey.multiplyByPrimes(context.getDigit((long)i)); }
}
}  // namespace detail

template <class Gen, class DrawA, std::enable_if_t<!std::is_same<std::decay_t<DrawA>, std::vector<uint8_t>>::value, int> = 0>
KeySwitch genKeySWmatrix(const Context& context, DoubleCRT fromKey, const SKHandle& fromHandle, long toKeyID,
                         const DoubleCRT& toKey, long p, bool ckks, double stdev, Gen& g, DrawA&& drawA) {
  KeySwitch W = detail::keySWmatrixHead(fromHandle, toKeyID, p, ckks);
  const IndexSet all = context.getCtxtPrimes() | context.getSpecialPrimes();
  const size_t n = context.getDigits().size();
  for (size_t i = 0; i < n; i++) { W.a.emplace_back(context, all); drawA(W.a.back()); }
  detail::keySWmatrixB(W, context, std::move(fromKey), toKey, stdev, g);
  return W;
}
// The same with the a_i drawn as the reference draws them: prgSeed is what RandomBits(prgSeed, 256) gave
// (little-endian magnitude bytes); SetSeed(prgSeed) and a[i].randomize() for all i in one device call
// (src/keys.cpp:1189-1206).  The matrix keeps the seed, so writeTo can store b + seed only.
template <class Gen>
KeySwitch genKeySWmatrix(const Context& context, DoubleCRT fromKey, const SKHandle& fromHandle, long toKeyID,
                         const DoubleCRT& toKey, long p, bool ckks, double stdev, Gen& g, const std::vector<uint8_t>& prgSeed) {
  KeySwitch W = detail::keySWmatrixHead(fromHandle, toKeyID, p, ckks);
  W.prgSeed = prgSeed;
  while (!W.prgSeed.empty() && W.prgSeed.back() == 0) W.prgSeed.pop_back();   // NumBytes(prgSeed)
  expandKeySWmatrixA(W, context, context.getDigits().size());
  detail::keySWmatrixB(W, context, std::move(fromKey), toKey, stdev, g);
  return W;
}

// KeySwitch::writeTo / readFrom (src/keySwitching.cpp:195-240), the v2.2.0 binary layout:
//   "|KM[", SKHandle (powerOfS, powerOfX, secretKeyID), toKeyID, ptxtSpace, b (int64 count, then DoubleCRT records),
//   prgSeed (write_raw_ZZ: int64 byte count, then the little-endian magnitude bytes, src/binio.cpp:180-203),
//   noiseBound (xdouble), "]KM|".  All integers little-endian int64.  a is not stored (both forms write the same bytes):
//   readFrom expands it on the device, or with expandA = false keeps the seeded form.
inline void KeySwitch::writeTo(std::ostream& str) const {
  if (prgSeed.empty()) throw InvalidArgument("KeySwitch::writeTo: no prgSeed (write_raw_ZZ needs a positive byte count)");
  str.write("|KM[", 4);
  Ctxt::writeInt(str, fromKey.powerOfS); Ctxt::writeInt(str, fromKey.powerOfX); Ctxt::writeInt(str, fromKey.secretKeyID);
  Ctxt::writeInt(str, toKeyID); Ctxt::writeInt(str, ptxtSpace);
  Ctxt::writeInt(str, (int64_t)b.size());
  for (const DoubleCRT& d : b) d.writeTo(str);
  Ctxt::writeInt(str, (int64_t)prgSeed.size());
  str.write(reinterpret_cast<const char*>(prgSeed.data()), (std::streamsize)prgSeed.size());
  Ctxt::writeXD(str, noiseBound);
  str.write("]KM|", 4);
}
inline KeySwitch KeySwitch::readFrom(std::istream& str, const Context& context, bool expandA) {
  char eye[4];
  str.read(eye, 4);
  if (!str || std::memcmp(eye, "|KM[", 4) != 0) throw RuntimeError("Could not find pre-secret key eyecatcher");
  KeySwitch W;
  W.fromKey.powerOfS = Ctxt::readInt(str); W.fromKey.powerOfX = Ctxt::readInt(str); W.fromKey.secretKeyID = Ctxt::readInt(str);
  W.toKeyID = Ctxt::readInt(str); W.ptxtSpace = Ctxt::readInt(str);
  const int64_t nb = Ctxt::readInt(str);
  if (!str || nb != (int64_t)context.getDigits().size()) throw RuntimeError("KeySwitch::readFrom: b count does not match the context's digits");
  for (int64_t i = 0; i < nb; i++) {
    DoubleCRT d(context, IndexSet::emptySet());
    d.read(str);
    W.b.push_back(std::move(d));
  }
  const int64_t len = Ctxt::readInt(str);
  if (!str || len <= 0 || len > 4096) throw InvalidArgument("KeySwitch::readFrom: bad prgSeed byte count");
  W.prgSeed.resize((size_t)len);
  str.read(reinterpret_cast<char*>(W.prgSeed.data()), (std::streamsize)len);
  W.noiseBound = Ctxt::readXD(str);
  str.read(eye, 4);
  if (!str || std::memcmp(eye, "]KM|", 4) != 0) throw RuntimeError("Could not find post-secret key eyecatcher");
  while (!W.prgSeed.empty() && W.prgSeed.back() == 0) W.prgSeed.pop_back();   // ZZFromBytes
  if (expandA) expandKeySWmatrixA(W, context, (size_t)nb);
  else W.aSeeded = std::make_shared<const SeededRows>(context, W.prgSeed, (size_t)nb);
  return W;
}

// ---- polyEval (src/polyEval.cpp:129-389): a cleartext polynomial on a ciphertext, by Paterson-Stockmeyer --------------
// The polynomial is NTL's ZZX with word-sized coefficients, low first; the mirror accepts |c| <= 2^62, so that the
// recursion's few decrements (q -= 1, r - X^deg(q)) stay within a long.  Every deg() is taken on the unreduced
// polynomial, as NTL does: a leading coefficient = 0 mod p still counts.
namespace pe {
using Poly = std::vector<long>;
inline long deg(const Poly& a) { return (long)a.size() - 1; }
inline void normalize(Poly& a) { while (!a.empty() && a.back() == 0) a.pop_back(); }
inline long coeff(const Poly& a, long i) { return i >= 0 && i < (long)a.size() ? a[(size_t)i] : 0; }
inline long remp(long c, long p) { long r = c % p; return r < 0 ? r + p : r; }                          // NTL rem, p > 0
inline long balanced(long c, long p) { long r = remp(c, p); return r > p / 2 ? r - p : r; }            // simplePolyEval's coef
inline void setCoeff(Poly& a, long i, long c = 1) {   // NTL::SetCoeff
  if (i > deg(a)) { if (c == 0) return; a.resize((size_t)i + 1, 0); }
  a[(size_t)i] = c;
  normalize(a);
}
inline Poly trunc(const Poly& a, long m) { Poly r(a.begin(), a.begin() + std::max(0L, std::min(m, (long)a.size()))); normalize(r); return r; }
inline Poly rightShift(const Poly& a, long n) { return n >= (long)a.size() ? Poly() : Poly(a.begin() + n, a.end()); }
inline void minusOne(Poly& a) { if (a.empty()) a.push_back(-1); else { a[0] -= 1; normalize(a); } }
inline long nextPowerOfTwo(long m) { long k = 0; while ((1L << k) < m) k++; return k; }                    // NTL::NextPowerOfTwo
inline long divc(long a, long b) { return (a + b - 1) / b; }
// NTL::DivRem(c, s, r, q) followed by the coefficient reduction mod p that PatersonStockmeyer applies to both: q is monic,
// so division over Z and reduction mod p commute, and the mirror divides mod p (the quotient over Z outgrows a long)
inline void divRemModP(Poly& c, Poly& s, const Poly& r, const Poly& q, long p) {
  const long dq = deg(q);
  s.assign(r.size(), 0);
  for (size_t i = 0; i < r.size(); i++) s[i] = remp(r[i], p);
  c.assign(deg(r) >= dq ? (size_t)(deg(r) - dq + 1) : 0, 0);
  for (long i = deg(r); i >= dq; i--) {
    const long t = s[(size_t)i];
    c[(size_t)(i - dq)] = t;
    if (t == 0) continue;
    for (long j = 0; j <= dq; j++)
      s[(size_t)(i - dq + j)] = (long)(((__int128)s[(size_t)(i - dq + j)] - (__int128)t * remp(q[(size_t)j], p)) % p + p) % p;
  }
  s.resize((size_t)std::max(0L, std::min(dq, (long)s.size())));
  normalize(c); normalize(s);
}
}  // namespace pe

// The recursion of polyEval over one DynamicCtxtPowers of baby steps, its giant steps built from X^k on first use.  A
// dry run walks the recursion's shape (it depends on the polynomial, k and p only) and records every simplePolyEval
// leaf; a run with `sums` takes each leaf's result from there, in the walk's order, instead of evaluating it.
class PolyEvalRun {
 public:
  using Poly = pe::Poly;
  struct Leaf { int kind = 0; Ctxt* sum = nullptr; };   // kind 0: the loop leaves ret empty; 1: run the loop; 2: *sum
  DynamicCtxtPowers& baby;
  const long p, k, nGiant;
  bool dry = false;
  std::vector<Poly> leaves;            // dry: every simplePolyEval polynomial, in order
  const std::vector<Leaf>* sums = nullptr;
  size_t next = 0;
  PolyEvalRun(DynamicCtxtPowers& b, long p_, long k_, long nGiant_) : baby(b), p(p_), k(k_), nGiant(nGiant_) {}
  DynamicCtxtPowers& giant() {
    if (!giant_) giant_ = std::make_unique<DynamicCtxtPowers>(baby.getPower(k), nGiant);
    return *giant_;
  }

  // simplePolyEval (src/polyEval.cpp:223-255): sum_i f_i X^i + f_0, the coefficients balanced mod p
  void simple(Ctxt& ret, const Poly& poly) {
    if (dry) { leaves.push_back(poly); return; }
    if (sums) {
      const Leaf& L = (*sums)[next++];
      if (L.kind == 2) { ret.clear(); assign(ret, *L.sum); return; }
      if (L.kind == 0) { ret.clear(); return; }
    }
    ret.clear();
    if (pe::deg(poly) < 0) return;
    if (pe::deg(poly) > baby.size()) throw LogicError("BabyStep has not enough powers (required more than deg(poly))");
    for (long i = 1; i <= pe::deg(poly); i++) {
      Ctxt tmp = baby.getPower(i);
      tmp.multByConstant(pe::balanced(poly[(size_t)i], p));
      ret += tmp;
    }
    ret.addConstant(pe::balanced(poly[0], p));
  }
  // PatersonStockmeyer (:261-311): poly monic, deg(poly) = k(2t-1) + delta
  void patersonStockmeyer(Ctxt& ret, const Poly& poly, long t, long delta) {
    if (pe::deg(poly) <= baby.size()) { simple(ret, poly); return; }
    Poly r = pe::trunc(poly, k * t), q = pe::rightShift(poly, k * t);
    pe::setCoeff(r, pe::deg(q), pe::coeff(r, pe::deg(q)) - 1);   // r' = r - X^deg(q)
    Poly c, s;
    pe::divRemModP(c, s, r, q, p);                                 // r' = c*q + s, both reduced mod p
    if (!(pe::deg(s) < pe::deg(q))) throw LogicError("Degree of s is not less than degree of q");
    if (!(c.empty() || pe::deg(c) < k - delta)) throw LogicError("Nonzero c has not degree smaller than k - delta");
    pe::setCoeff(s, pe::deg(q));                                   // s' = s + X^deg(q)
    patersonStockmeyer(ret, q, t / 2, delta);
    Ctxt tmp(ret.pubKey, ret.ptxtSpace);
    simple(tmp, c);
    if (!dry) { tmp += giant().getPower(t); ret.multiplyBy(tmp); }
    patersonStockmeyer(tmp, s, t / 2, delta);
    if (!dry) ret += tmp;
  }
  // degPowerOfTwo (:315-344): k(2^e + 1) > deg(poly) > k(2^e - 1)
  void degPowerOfTwo(Ctxt& ret, const Poly& poly) {
    if (pe::deg(poly) <= baby.size()) { simple(ret, poly); return; }
    long n = pe::deg(poly) / k;
    n = 1L << pe::nextPowerOfTwo(n);
    Poly r = pe::trunc(poly, (n - 1) * k), q = pe::rightShift(poly, (n - 1) * k);
    pe::setCoeff(r, (n - 1) * k);
    pe::minusOne(q);
    patersonStockmeyer(ret, r, n / 2, 0);
    Ctxt tmp(ret.pubKey, ret.ptxtSpace);
    simple(tmp, q);
    if (dry) return;
    for (long i = 1; i < n; i *= 2) tmp.multiplyBy(giant().getPower(i));
    ret += tmp;
  }
  // recursivePolyEval (:346-389)
  void recursive(Ctxt& ret, const Poly& poly) {
    if (pe::deg(poly) <= baby.size()) { simple(ret, poly); return; }
    const long delta = pe::deg(poly) % k, n = pe::divc(pe::deg(poly), k);
    long t = 1L << pe::nextPowerOfTwo(n);
    if (n == t) { degPowerOfTwo(ret, poly); return; }
    if (n == t - 1 && delta == 0) { patersonStockmeyer(ret, poly, t / 2, delta); return; }
    t = t / 2;
    const long u = pe::deg(poly) - k * (t - 1);
    Poly r = pe::trunc(poly, u), q = pe::rightShift(poly, u);
    pe::minusOne(q);
    pe::setCoeff(r, u);
    patersonStockmeyer(ret, q, t / 2, 0);
    Ctxt tmp(ret.pubKey, ret.ptxtSpace);
    if (!dry) {
      tmp = giant().getPower(u / k);
      if (delta != 0) tmp.multiplyBy(baby.getPower(delta));
      ret.multiplyBy(tmp);
    }
    recursive(tmp, r);
    if (!dry) ret += tmp;
  }

 private:
  std::unique_ptr<DynamicCtxtPowers> giant_;
  // ret = a leaf sum, as the loop's first `ret += tmp` (a copy into the cleared ret) and the rest of it leave ret
  static void assign(Ctxt& ret, Ctxt& sum) {
    ret.parts.swap(sum.parts);
    ret.primeSet = sum.primeSet; ret.ptxtSpace = sum.ptxtSpace; ret.noiseBound = sum.noiseBound;
    ret.intFactor = sum.intFactor; ret.ratFactor = sum.ratFactor; ret.ptxtMag = sum.ptxtMag;
    if (sum.lastKSNoiseRatio != 0) ret.lastKSNoiseRatio = sum.lastKSNoiseRatio;
    if (sum.lastModSwitchRatio != 0) ret.lastModSwitchRatio = sum.lastModSwitchRatio;
  }
};

// Every leaf of a run as one hb_ctxt_scaled_sums call.  Each leaf the loop of simplePolyEval would evaluate to a 2-part
// ciphertext is sum_i s_{i,r} X^i + c_r on every row r: the loop's multByConstant (balRem(d) on the rows), modUpToSet
// (the product of the added primes on the old rows, zero on the new ones), addCtxt's intFactor harmonisation (balRem(e1),
// balRem(e2)) and addConstant (cc*f on part 0) are all linear and exact mod every prime.  The per-row scalars and each
// leaf's primeSet, noiseBound, intFactor, ratFactor and ptxtMag are replayed here from the metadata the loop would compute.
// Leaves the loop leaves empty need nothing; a leaf of only a constant (a 1-part result) runs the loop.  Returns false, with
// nothing launched, where one call cannot reproduce the loop: CKKS (the loop reduces mod ptxtSpace = 1 and encodes its
// scalars), plaintext spaces that differ, a baby step that is not a 2-part canonical ciphertext under x's key, or a prime
// set the loop's verifyPrimeSet would reject.
inline bool polyEvalLeafSums(PolyEvalRun& run, const Ctxt& ret, std::vector<PolyEvalRun::Leaf>& plan, std::vector<Ctxt>& sums) {
  using u64 = uint64_t;
  const Ctxt& x = run.baby.getPower(1);
  const Context& ctx = x.context;
  const KeyInfo& pubKey = x.pubKey;
  const long P = x.ptxtSpace;
  if (x.isCKKS() || ret.ptxtSpace != P || &ret.pubKey != &pubKey) return false;
  long maxdeg = 0;
  for (const auto& L : run.leaves) maxdeg = std::max(maxdeg, pe::deg(L));
  if (maxdeg > run.baby.size()) return false;   // the loop throws
  const long keyID = x.getKeyID();
  for (long i = 1; i <= maxdeg; i++) {   // the powers the loop takes, computed as it computes them
    const Ctxt& c = run.baby.getPower(i);
    if (&c.pubKey != &pubKey || c.ptxtSpace != P || c.parts.size() != 2 || !c.inCanonicalForm(keyID) || c.getKeyID() != keyID) return false;
  }
  const long np = ctx.numPrimes();
  auto mulmod = [](u64 a, u64 b, u64 q) { return (u64)((unsigned __int128)a * b % q); };
  auto resid = [&](long v, long i) { const long q = ctx.ithPrime(i); long r = v % q; return (u64)(r < 0 ? r + q : r); };
  auto prodMod = [&](const IndexSet& s, long i) { u64 r = 1; for (long j : s) r = mulmod(r, (u64)ctx.ithPrime(j) % (u64)ctx.ithPrime(i), (u64)ctx.ithPrime(i)); return r; };
  auto modUp = [&](Ctxt& m, std::vector<std::vector<u64>*> rows, const IndexSet& s) {   // Ctxt::modUpToSet's arithmetic
    const IndexSet d = s / m.primeSet;
    if (empty(d)) return true;
    for (auto* v : rows) for (long i : m.primeSet) (*v)[(size_t)i] = mulmod((*v)[(size_t)i], prodMod(d, i), (u64)ctx.ithPrime(i));
    const double f = pubKey.logOfProduct(d);
    m.noiseBound = m.noiseBound * XD::exp(f);
    m.ratFactor = m.ratFactor * XD::exp(f);
    m.primeSet.insert(d);
    return m.verifyPrimeSet();
  };
  auto mulInt = [&](Ctxt& m, std::vector<std::vector<u64>*> rows, long e) {   // Ctxt::mulIntFactor's arithmetic
    if (e == 1) return;
    m.intFactor = (long)(((unsigned __int128)(unsigned long)m.intFactor * (unsigned long)e) % (unsigned long)P);
    const long b = Ctxt::balRem(e, P);
    for (auto* v : rows) for (long i : m.primeSet) (*v)[(size_t)i] = mulmod((*v)[(size_t)i], resid(b, i), (u64)ctx.ithPrime(i));
    m.noiseBound = m.noiseBound * XD((double)std::labs(b));
  };
  struct Acc { Ctxt meta; std::vector<std::vector<u64>> s; std::vector<u64> cst; long nterms = 0; };
  std::vector<Acc> acc;
  plan.assign(run.leaves.size(), PolyEvalRun::Leaf());
  IndexSet U;
  long nin = 0;
  for (size_t l = 0; l < run.leaves.size(); l++) {
    const pe::Poly& poly = run.leaves[l];
    if (pe::deg(poly) < 0) continue;   // kind 0
    Acc A{Ctxt(pubKey, P), std::vector<std::vector<u64>>((size_t)pe::deg(poly) + 1, std::vector<u64>((size_t)np, 0)), {}, 0};
    bool empty_acc = true;
    for (long i = 1; i <= pe::deg(poly); i++) {
      const long c0 = pe::remp(pe::balanced(poly[(size_t)i], run.p), P);   // multByConstant: 0 clears the term, 1 leaves it
      if (c0 == 0) continue;
      const Ctxt& X = run.baby.getPower(i);
      Ctxt T(pubKey, P);
      T.primeSet = X.primeSet; T.noiseBound = X.noiseBound; T.intFactor = X.intFactor; T.ratFactor = X.ratFactor; T.ptxtMag = X.ptxtMag;
      std::vector<u64> t((size_t)np, 0);
      for (long r : X.primeSet) t[(size_t)r] = 1;
      if (c0 != 1) {
        const long d = std::gcd(c0, P);
        T.intFactor = (long)(((unsigned __int128)(unsigned long)T.intFactor * (unsigned long)Ctxt::invMod(c0 / d, P)) % (unsigned long)P);
        if (d != 1) {
          const long cc = Ctxt::balRem(d, P);
          T.noiseBound = T.noiseBound * XD((double)std::labs(cc));
          for (long r : T.primeSet) t[(size_t)r] = resid(cc, r);
        }
      }
      if (empty_acc) {   // addCtxt's copy into the empty ret
        A.meta = T;
        if (X.lastKSNoiseRatio != 0) A.meta.lastKSNoiseRatio = X.lastKSNoiseRatio;
        if (X.lastModSwitchRatio != 0) A.meta.lastModSwitchRatio = X.lastModSwitchRatio;
        A.s[(size_t)i] = t;
        empty_acc = false;
      } else {
        std::vector<std::vector<u64>*> rows;
        for (auto& v : A.s) rows.push_back(&v);
        if (!modUp(A.meta, rows, T.primeSet) || !modUp(T, {&t}, A.meta.primeSet)) return false;
        long e1 = 1, e2 = 1;
        if (A.meta.intFactor != T.intFactor) Ctxt::harmoniseIntFactors(A.meta, T, e1, e2);
        mulInt(T, {&t}, e2);
        mulInt(A.meta, rows, e1);
        A.s[(size_t)i] = t;
        A.meta.ptxtMag = A.meta.ptxtMag + T.ptxtMag;
        A.meta.noiseBound = A.meta.noiseBound + T.noiseBound;
      }
      A.nterms = i;
    }
    const long cc = pe::balanced(pe::balanced(poly[0], run.p), P);   // addConstant
    if (empty_acc) { if (cc != 0) plan[l].kind = 1; continue; }
    A.cst.assign((size_t)np, 0);
    if (cc != 0) {
      const long f = A.meta.constantFactor();
      A.meta.noiseBound = A.meta.noiseBound + XD((double)cc * (double)std::labs(f));
      for (long r : A.meta.primeSet) A.cst[(size_t)r] = mulmod(resid(cc, r), resid(f, r), (u64)ctx.ithPrime(r));
    }
    plan[l].kind = 2;
    U.insert(A.meta.primeSet);
    nin = std::max(nin, A.nterms);
    acc.push_back(std::move(A));
  }
  if (acc.empty()) return true;
  // ---- the call: input i is X^(i+1), output j the j-th summed leaf
  const std::vector<long> Uv(U.begin(), U.end());
  const size_t nU = Uv.size(), nout = acc.size();
  std::vector<u64> scal(nout * (size_t)nin * nU, 0), cst(nout * nU, 0);
  for (size_t j = 0; j < nout; j++)
    for (size_t r = 0; r < nU; r++) {
      cst[j * nU + r] = acc[j].cst[(size_t)Uv[r]];
      for (long i = 1; i <= acc[j].nterms; i++) scal[(j * (size_t)nin + (size_t)(i - 1)) * nU + r] = acc[j].s[(size_t)i][(size_t)Uv[r]];
    }
  // the leaf ciphertexts get their two parts first, unwritten, and the call writes straight into them
  sums.clear();
  sums.reserve(nout);
  std::vector<hb_poly*> in0, in1, out0, out1;
  for (long i = 1; i <= nin; i++) { const Ctxt& X = run.baby.getPower(i); in0.push_back(X.parts[0].dcrt.handle()); in1.push_back(X.parts[1].dcrt.handle()); }
  for (size_t j = 0; j < nout; j++) {
    sums.push_back(acc[j].meta);
    std::vector<CtxtPart>& pt = sums.back().parts;
    pt.reserve(2);
    pt.emplace_back(ctx, acc[j].meta.primeSet, SKHandle());
    pt.emplace_back(ctx, acc[j].meta.primeSet, SKHandle(1, 1, keyID));
    out0.push_back(pt[0].dcrt.handle()); out1.push_back(pt[1].dcrt.handle());
  }
  std::vector<int32_t> Ui(Uv.begin(), Uv.end());
  check(hb_ctxt_scaled_sums(in0.data(), in1.data(), (int)nin, out0.data(), out1.data(), (int)nout, 1, Ui.data(), (int)nU,
                            scal.data(), cst.data(), 0));
  for (size_t l = 0, j = 0; l < plan.size(); l++) if (plan[l].kind == 2) plan[l].sum = &sums[j++];
  return true;
}

// Runs body (the recursion from its top call) once dry, then with every leaf summed in one call, or, where the call
// cannot reproduce the loop, as transcribed.
template <class Body>
inline void polyEvalRun(PolyEvalRun& run, Ctxt& ret, Body body) {
  Ctxt scratch(ret.pubKey, ret.ptxtSpace);
  run.dry = true;
  body(scratch);
  run.dry = false;
  std::vector<PolyEvalRun::Leaf> plan;
  std::vector<Ctxt> sums;
  if (polyEvalLeafSums(run, ret, plan, sums)) { run.sums = &plan; run.next = 0; }
  body(ret);
  run.sums = nullptr;
}

// hb::polyEval(ret, poly, x, k): helib::polyEval(Ctxt&, ZZX, const Ctxt&, long) (src/polyEval.cpp:129-221), poly low
// coefficient first with |c| <= 2^62, k <= 0 for polyEval's choice.  The ciphertext operations are HElib's; the
// simplePolyEval leaves are formed together by polyEvalLeafSums in one hb_ctxt_scaled_sums call where it can.  BGV only
// (the CKKS branch of the scalar operations encodes through the slot layer): a CKKS x throws LogicError from
// multByConstant / addConstant, as a transcription over the mirror does.  The top coefficient of a polynomial whose n is
// not a power of two goes to NTL's InvModStatus, which takes 0 <= top < p.
inline void polyEval(Ctxt& ret, std::vector<long> poly, const Ctxt& x, long k = 0) {
  for (long c : poly) if (c > (1L << 62) || c < -(1L << 62)) throw InvalidArgument("polyEval: coefficients must be within +-2^62");
  pe::normalize(poly);
  const long dg = pe::deg(poly);
  if (dg <= 2) {
    if (dg < 1) { ret.clear(); ret.addConstant(pe::coeff(poly, 0)); return; }
    DynamicCtxtPowers babyStep(x, dg);
    PolyEvalRun run(babyStep, x.ptxtSpace, 1, 1);
    polyEvalRun(run, ret, [&](Ctxt& r) { run.simple(r, poly); });
    return;
  }
  if (k <= 0) {
    const long kk = (long)std::sqrt(dg / 2.0);
    k = 1L << pe::nextPowerOfTwo(kk);
    if ((k == 16 && dg > 167) || (k > 16 && k > (1.44 * kk))) k /= 2;
  }
  const long n = pe::divc(dg, k);
  DynamicCtxtPowers babyStep(x, k);
  if (n == (1L << pe::nextPowerOfTwo(n))) {
    if (n / 2 <= 0) throw InvalidArgument("Must have positive nPowers");   // DynamicCtxtPowers giantStep(x2k, n/2)
    PolyEvalRun run(babyStep, x.ptxtSpace, k, n / 2);
    polyEvalRun(run, ret, [&](Ctxt& r) { run.degPowerOfTwo(r, poly); });
    return;
  }
  // make poly monic of degree n*k: topInv, or an added term extra*X^(n*k) for a non-divisible degree or a top that is not
  // invertible mod p (src/polyEval.cpp:178-219)
  const long p = x.ptxtSpace;
  long top = poly.back();
  if (top < 0 || top >= p) throw LogicError(top < 0 ? "InvMod: first input negative" : "InvMod: first input too big");
  long topInv = 0;
  const bool divisible = n * k == dg;
  const bool nonInvertible = std::gcd(top, p) != 1;
  if (!nonInvertible) topInv = Ctxt::invMod(top, p);
  long extra = 0;
  if (!divisible || nonInvertible) {
    top = 1; topInv = 1;
    extra = 1 - pe::coeff(poly, n * k);   // SubMod(1, c, p), c in [0, p)
    if (extra < 0) extra += p;
    pe::setCoeff(poly, n * k);
  }
  const long t = extra == 0 ? pe::divc(n, 2) : n;
  if (top != 1) {
    for (long i = 0; i <= n * k; i++) poly[(size_t)i] = (long)(((__int128)pe::remp(poly[(size_t)i], p) * topInv) % p);
    pe::normalize(poly);
  }
  PolyEvalRun run(babyStep, p, k, t);
  polyEvalRun(run, ret, [&](Ctxt& r) { run.recursive(r, poly); });
  if (top != 1) ret.multByConstant(top);
  if (extra != 0) {
    Ctxt topTerm = run.giant().getPower(n);
    topTerm.multByConstant(extra);
    ret -= topTerm;
  }
}

// ---- digit extraction (src/extractDigits.cpp, src/recryption.cpp:793-909) ----------------------------------------------
// The polynomials are computed on the host from their definitions: arithmetic mod p^e (p^e < 2^30) and, for Chen and Han's
// a(m), mod p^(2e) < 2^60, in 128-bit products.
namespace xd {
using Poly = std::vector<long>;
inline long mulmod(long a, long b, long q) { return (long)((unsigned __int128)(uint64_t)a * (uint64_t)b % (uint64_t)q); }
inline long power(long p, long e) { long r = 1; for (long i = 0; i < e; i++) r *= p; return r; }
inline long powmod(long a, long e, long q) { long r = 1 % q; for (a %= q; e; e >>= 1, a = mulmod(a, a, q)) if (e & 1) r = mulmod(r, a, q); return r; }
inline Poly mulTrunc(const Poly& a, const Poly& b, long len, long q) {   // a*b mod (X^len, q)
  Poly r((size_t)len, 0);
  for (size_t i = 0; i < a.size() && (long)i < len; i++)
    if (a[i]) for (size_t j = 0; j < b.size() && (long)(i + j) < len; j++) r[i + j] = (r[i + j] + mulmod(a[i], b[j], q)) % q;
  return r;
}
// The unique f of degree < #x with f(x_j) = y_j mod p^e, coefficients in [0, p^e), for x_j distinct mod p
// (interpolateMod, src/NumbTh.cpp:1043): its p-adic digits are interpolated one at a time mod p, lowest first.
inline Poly interpolateMod(const std::vector<long>& x, std::vector<long> y, long p, long e) {
  const size_t n = x.size();
  const long p2e = power(p, e);
  Poly res(n, 0);
  for (auto& v : y) { v %= p2e; if (v < 0) v += p2e; }
  std::vector<long> xm(n);
  for (size_t j = 0; j < n; j++) { xm[j] = x[j] % p; if (xm[j] < 0) xm[j] += p; }
  Poly M{1};   // prod_k (X - x_k) mod p
  for (size_t k = 0; k < n; k++) {
    Poly nb(M.size() + 1, 0);
    for (size_t t = 0; t < M.size(); t++) { nb[t + 1] = (nb[t + 1] + M[t]) % p; nb[t] = (nb[t] + mulmod(M[t], (p - xm[k]) % p, p)) % p; }
    M = nb;
  }
  std::vector<Poly> basis(n, Poly(n, 0));   // M / (X - x_j), scaled to 1 at x_j
  for (size_t j = 0; j < n; j++) {
    Poly& b = basis[j];
    for (size_t t = n; t-- > 0;) b[t] = t + 1 == n ? M[n] : (M[t + 1] + mulmod(xm[j], b[t + 1], p)) % p;
    long den = 0;
    for (size_t t = n; t-- > 0;) den = (mulmod(den, xm[j], p) + b[t]) % p;
    const long s = Ctxt::invMod(den, p);
    for (auto& c : b) c = mulmod(c, s, p);
  }
  for (long pl = 1, mod = p2e; mod > 1; pl *= p, mod /= p) {
    Poly g(n, 0);   // the lowest p-adic digits of y, interpolated mod p
    for (size_t j = 0; j < n; j++) for (size_t t = 0; t < n; t++) g[t] = (g[t] + mulmod(basis[j][t], y[j] % p, p)) % p;
    for (size_t t = 0; t < n; t++) res[t] += g[t] * pl;
    for (size_t j = 0; j < n; j++) {   // y_j = (y_j - g(x_j) mod p^(e-lvl)) / p
      long v = 0, xj = x[j] % mod; if (xj < 0) xj += mod;
      for (size_t t = n; t-- > 0;) v = (mulmod(v, xj, mod) + g[t]) % mod;
      long d = y[j] - v; if (d < 0) d += mod;
      y[j] = d / p;
    }
  }
  pe::normalize(res);
  return res;
}
// buildDigitPolynomial (src/extractDigits.cpp:28-58): f = X^p + f' with f'(z) = z - z^p mod p^e for |z| <= p/2, so that
// f(z0 + p^t z1) = z0 mod p^(t+1) for t < e.  Empty for p < 2 or e <= 1.
inline Poly buildDigitPolynomial(long p, long e) {
  if (p < 2 || e <= 1) return {};
  const long p2e = power(p, e);
  std::vector<long> x((size_t)p), y((size_t)p);
  for (long j = 0; j < p; j++) {
    const long z = -(p / 2) + j;
    x[(size_t)j] = z;
    long v = z - powmod(z < 0 ? z + p2e : z, p, p2e);
    while (v > p2e / 2) v -= p2e;
    while (v < -(p2e / 2)) v += p2e;
    y[(size_t)j] = v;
  }
  Poly f = interpolateMod(x, y, p, e);
  if (pe::deg(f) >= p) throw LogicError("Interpolation error.  Degree too high.");
  pe::setCoeff(f, p);
  return f;
}
// compute_a_vals (src/extractDigits.cpp:131-172): a[m] = a(m)/m! mod p^e for m = p .. (e-1)(p-1)+1, where the a(m) are the
// coefficients of p (X+1)^p / ((X+1)^p - X^p) as a power series mod p^(2e)
inline std::vector<long> chenHanA(long p, long e) {
  const long pe_ = power(p, e), p2e = pe_ * pe_;
  const long len = (e - 1) * (p - 1) + 2;
  Poly xp1{1}, b{1, 1};   // (X+1)^p mod (X^len, p^(2e))
  for (long k = p; k; k >>= 1) { if (k & 1) xp1 = mulTrunc(xp1, b, len, p2e); b = mulTrunc(b, b, len, p2e); }
  Poly den = xp1;
  if (p < len) den[(size_t)p] = (den[(size_t)p] - 1 + p2e) % p2e;
  Poly inv((size_t)len, 0);   // 1/den mod X^len: den(0) = 1
  for (long i = 0; i < len; i++) {
    long s = i == 0 ? 1 : 0;
    for (long j = 1; j <= i; j++) s = (s - mulmod(den[(size_t)j], inv[(size_t)(i - j)], p2e) + p2e) % p2e;
    inv[(size_t)i] = s;
  }
  Poly poly = mulTrunc(xp1, inv, len, p2e);
  for (auto& c : poly) c = mulmod(c, p, p2e);
  std::vector<long> a((size_t)len, 0);
  long mfac = 1;
  for (long m = 2; m < p; m++) mfac = mulmod(mfac, m, p2e);
  for (long m = p; m < len; m++) {
    mfac = mulmod(mfac, m, p2e);
    const long c = poly[(size_t)m];
    long d = 1;   // gcd(mfac, p^(2e)), p^(2e) for mfac = 0
    for (long t = mfac; d < p2e && t % p == 0; t /= p) { d *= p; if (t == 0) { d = p2e; break; } }
    if (d > pe_ || c % d != 0) throw RuntimeError("cannot divide");
    a[(size_t)m] = mulmod((c / d) % pe_, Ctxt::invMod((mfac / d) % pe_, pe_), pe_);
  }
  return a;
}
// compute_magic_poly (src/extractDigits.cpp:178-222): Chen and Han's G with G(x) = (x mod p) mod p^e, x mod p in [0, 1]
// for p = 2 and in (-p/2, p/2) otherwise; coefficients in [0, p^e)
inline Poly chenHanMagicPoly(long p, long e) {
  const std::vector<long> a = chenHanA(p, e);
  const long q = power(p, e), len = (e - 1) * (p - 1) + 2;
  auto mulLin = [&](Poly& t, long m) {   // t *= (X - m)
    Poly r(t.size() + 1, 0);
    const long mm = (q - m % q) % q;
    for (size_t i = 0; i < t.size(); i++) { r[i + 1] = (r[i + 1] + t[i]) % q; r[i] = (r[i] + mulmod(t[i], mm, q)) % q; }
    t = r;
  };
  Poly term{1 % q}, poly;
  for (long m = 0; m < p; m++) mulLin(term, m);
  for (long m = p; m < len; m++) {
    if (poly.size() < term.size()) poly.resize(term.size(), 0);
    for (size_t i = 0; i < term.size(); i++) poly[i] = (poly[i] + mulmod(term[i], a[(size_t)m], q)) % q;
    mulLin(term, m);
  }
  if (p % 2 == 1) {   // poly(X + (p-1)/2), by Horner
    Poly p2;
    for (long i = (long)poly.size() - 1; i >= 0; i--) {
      mulLin(p2, -((p - 1) / 2));
      if (p2.empty()) p2.push_back(0);
      p2[0] = (p2[0] + poly[(size_t)i]) % q;
    }
    poly = p2;
  }
  for (auto& c : poly) c = (q - c) % q;   // X - poly
  if (poly.size() < 2) poly.resize(2, 0);
  poly[1] = (poly[1] + 1) % q;
  pe::normalize(poly);
  return poly;
}
}  // namespace xd

// One linear combination of 2-part ciphertexts, formed in one hb_ctxt_scaled_sums call.  The operations of the digit
// chains (addCtxt, divideByP, multByP, negate, reducePtxtSpace) are linear and exact on every row: the mod-up of addCtxt
// multiplies the old rows by the added primes and leaves zero on the new ones, the intFactor harmonisation and multByP
// multiply by small signed integers, divideByP by p^-1 mod q_r.  A Term replays them on the metadata (primeSet, ptxtSpace,
// intFactor, noiseBound, ratFactor, ptxtMag) as the mirror's methods compute it, and keeps each input's scalar on every row.
// `ok` turns false where the loop would throw; the caller then runs the loop, which throws as HElib does.
class LinearChain {
 public:
  using u64 = uint64_t;
  struct Term { Ctxt meta; std::vector<std::vector<u64>> s; };   // s[input][row]
  bool ok = true;

  // ok is false unless the inputs are BGV, non-empty, 2-part canonical under one key, with their parts over their primeSet
  explicit LinearChain(std::vector<const Ctxt*> inputs) : in_(std::move(inputs)), ctx_(in_.at(0)->context), np_(ctx_.numPrimes()) {
    const Ctxt& c0 = *in_[0];
    keyID_ = c0.getKeyID();
    for (const Ctxt* c : in_) {
      if (c->isCKKS() || &c->pubKey != &c0.pubKey || c->parts.size() != 2 || !c->inCanonicalForm(keyID_) || c->getKeyID() != keyID_) ok = false;
      else for (const auto& part : c->parts) if (!(part.dcrt.getIndexSet() == c->primeSet)) ok = false;
    }
  }
  Term term(size_t k) const {
    const Ctxt& c = *in_.at(k);
    Term t{metaOf(c), std::vector<std::vector<u64>>(in_.size(), std::vector<u64>(np_, 0))};
    for (long r : c.primeSet) t.s[k][(size_t)r] = 1;
    return t;
  }
  // a += b or a -= b: Ctxt::addCtxt (src/Ctxt.cpp:1406-1556), BGV
  void add(Term& a, Term b, bool negative = false) {
    if (!ok) return;
    const long g = std::gcd(a.meta.ptxtSpace, b.meta.ptxtSpace);
    if (g <= 1) { ok = false; return; }
    a.meta.reducePtxtSpace(b.meta.ptxtSpace);
    if (b.meta.ptxtSpace != a.meta.ptxtSpace) b.meta.reducePtxtSpace(a.meta.ptxtSpace);
    if (!modUp(a, b.meta.primeSet / a.meta.primeSet) || !modUp(b, a.meta.primeSet / b.meta.primeSet)) return;
    long e1 = 1, e2 = 1;
    if (a.meta.intFactor != b.meta.intFactor) Ctxt::harmoniseIntFactors(a.meta, b.meta, e1, e2);
    mulInt(b, e2);
    mulInt(a, e1);
    for (size_t k = 0; k < in_.size(); k++)
      for (long r : a.meta.primeSet) {
        const u64 q = (u64)ctx_.ithPrime(r), x = b.s[k][(size_t)r];
        a.s[k][(size_t)r] = negative ? (a.s[k][(size_t)r] + q - x) % q : (a.s[k][(size_t)r] + x) % q;
      }
    a.meta.ptxtMag = a.meta.ptxtMag + b.meta.ptxtMag;
    a.meta.noiseBound = a.meta.noiseBound + b.meta.noiseBound;
  }
  void divideByP(Term& a) {   // Ctxt::divideByP
    if (!ok) return;
    const long p = ctx_.getP();
    if (a.meta.ptxtSpace % p != 0 || !(a.meta.ptxtSpace > p)) { ok = false; return; }
    a.meta.divideByPMeta();
    for (long r : a.meta.primeSet) scaleRow(a, r, (u64)Ctxt::invMod(p, ctx_.ithPrime(r)));
  }
  void multByP(Term& a, long e = 1) {   // Ctxt::multByP, through multByConstant(long)'s BGV branch
    if (!ok) return;
    const long p2e = xd::power(ctx_.getP(), e);
    Ctxt& m = a.meta;
    m.ptxtSpace *= p2e;
    const long c0 = p2e % m.ptxtSpace;
    if (c0 == 1) return;
    if (c0 == 0) { ok = false; return; }   // multByConstant clears the ciphertext
    const long d = std::gcd(c0, m.ptxtSpace);
    m.intFactor = (long)(((unsigned __int128)(unsigned long)m.intFactor * (unsigned long)Ctxt::invMod(c0 / d, m.ptxtSpace)) % (unsigned long)m.ptxtSpace);
    if (d == 1) return;
    const long cc = Ctxt::balRem(d, m.ptxtSpace);
    m.noiseBound = m.noiseBound * XD((double)std::labs(cc));
    for (long r : m.primeSet) scaleRow(a, r, resid(cc, r));
  }
  void negate(Term& a) {   // Ctxt::negate
    for (auto& v : a.s) for (long r : a.meta.primeSet) { const u64 q = (u64)ctx_.ithPrime(r); v[(size_t)r] = (q - v[(size_t)r]) % q; }
  }
  void reducePtxtSpace(Term& a, long P) {   // Ctxt::reducePtxtSpace
    if (!ok) return;
    if (std::gcd(a.meta.ptxtSpace, P) <= 1) { ok = false; return; }
    a.meta.reducePtxtSpace(P);
  }
  // dst = the combination, in one call: dst's parts are replaced by new ones over the term's primeSet and its metadata
  // set as Ctxt::operator= sets it from the loop's result (the mod-switch and key-switch statistics only where nonzero)
  bool form(const Term& a, Ctxt& dst) {
    if (!ok || &dst.pubKey != &a.meta.pubKey) return false;
    const std::vector<int32_t> U = a.meta.primeSet.vec();
    const size_t nU = U.size(), nin = in_.size();
    std::vector<u64> scal(nin * nU, 0);
    for (size_t k = 0; k < nin; k++) for (size_t r = 0; r < nU; r++) scal[k * nU + r] = a.s[k][(size_t)U[r]];
    std::vector<hb_poly*> in0, in1;
    for (const Ctxt* c : in_) { in0.push_back(c->parts[0].dcrt.handle()); in1.push_back(c->parts[1].dcrt.handle()); }
    std::vector<CtxtPart> out;
    out.reserve(3);   // a later product adds a third part: no reallocation, which would copy the two parts through the device
    out.emplace_back(ctx_, a.meta.primeSet, SKHandle());
    out.emplace_back(ctx_, a.meta.primeSet, SKHandle(1, 1, keyID_));
    hb_poly* o0[1] = {out[0].dcrt.handle()}; hb_poly* o1[1] = {out[1].dcrt.handle()};
    check(hb_ctxt_scaled_sums(in0.data(), in1.data(), (int)nin, o0, o1, 1, 1, U.data(), (int)nU, scal.data(), nullptr, 0));
    dst.parts.swap(out);
    const Ctxt& m = a.meta;
    dst.primeSet = m.primeSet; dst.ptxtSpace = m.ptxtSpace; dst.noiseBound = m.noiseBound;
    dst.intFactor = m.intFactor; dst.ratFactor = m.ratFactor; dst.ptxtMag = m.ptxtMag;
    if (m.lastKSNoiseRatio != 0) dst.lastKSNoiseRatio = m.lastKSNoiseRatio;
    if (m.lastModSwitchRatio != 0) dst.lastModSwitchRatio = m.lastModSwitchRatio;
    return true;
  }

 private:
  std::vector<const Ctxt*> in_;
  const Context& ctx_;
  size_t np_;
  long keyID_ = 0;
  static Ctxt metaOf(const Ctxt& c) {
    Ctxt m(c.pubKey, c.ptxtSpace);
    m.primeSet = c.primeSet; m.noiseBound = c.noiseBound; m.intFactor = c.intFactor; m.ratFactor = c.ratFactor; m.ptxtMag = c.ptxtMag;
    m.lastKSNoiseRatio = c.lastKSNoiseRatio; m.lastModSwitchRatio = c.lastModSwitchRatio;
    return m;
  }
  u64 resid(long v, long r) const { const long q = ctx_.ithPrime(r); long x = v % q; return (u64)(x < 0 ? x + q : x); }
  void scaleRow(Term& a, long r, u64 f) {
    const u64 q = (u64)ctx_.ithPrime(r);
    for (auto& v : a.s) v[(size_t)r] = (u64)((unsigned __int128)v[(size_t)r] * f % q);
  }
  bool modUp(Term& a, const IndexSet& d) {   // Ctxt::modUpToSet's arithmetic
    if (empty(d)) return true;
    for (long r : a.meta.primeSet) {
      u64 f = 1;
      const u64 q = (u64)ctx_.ithPrime(r);
      for (long j : d) f = (u64)((unsigned __int128)f * ((u64)ctx_.ithPrime(j) % q) % q);
      scaleRow(a, r, f);
    }
    const double f = a.meta.pubKey.logOfProduct(d);
    a.meta.noiseBound = a.meta.noiseBound * XD::exp(f);
    a.meta.ratFactor = a.meta.ratFactor * XD::exp(f);
    a.meta.primeSet.insert(d);
    if (!a.meta.verifyPrimeSet()) ok = false;
    return ok;
  }
  void mulInt(Term& a, long e) {   // Ctxt::mulIntFactor's arithmetic
    if (e == 1) return;
    Ctxt& m = a.meta;
    m.intFactor = (long)(((unsigned __int128)(unsigned long)m.intFactor * (unsigned long)e) % (unsigned long)m.ptxtSpace);
    const long b = Ctxt::balRem(e, m.ptxtSpace);
    for (long r : m.primeSet) scaleRow(a, r, resid(b, r));
    m.noiseBound = m.noiseBound * XD((double)std::labs(b));
  }
};

namespace detail {
// the powerings of extractDigits: x^p in spirit (src/extractDigits.cpp:91-97)
inline void powerDigit(Ctxt& d, const std::vector<long>& x2p) {
  HB_NTIMER_START(digit_power, d.context.handle());
  const long p = d.context.getP();
  if (p == 2) d.square();
  else if (p == 3) d.cube();
  else polyEval(d, x2p, d);
}
// tmp = c - sum_j in[j] with a divideByP after each step (src/extractDigits.cpp:90-109), as transcribed
inline void digitChainLoop(Ctxt& dst, const Ctxt& c, const std::vector<const Ctxt*>& sub) {
  Ctxt tmp(c.pubKey, c.ptxtSpace);
  tmp = c;
  for (const Ctxt* d : sub) { tmp -= *d; tmp.divideByP(); }
  dst = tmp;
}
// the same chain in one hb_ctxt_scaled_sums call; false, with nothing launched, where one call cannot reproduce it
inline bool digitChainFused(Ctxt& dst, const Ctxt& c, const std::vector<const Ctxt*>& sub) {
  std::vector<const Ctxt*> in{&c};
  in.insert(in.end(), sub.begin(), sub.end());
  LinearChain L(in);
  if (!L.ok) return false;
  LinearChain::Term t = L.term(0);
  for (size_t j = 0; j < sub.size(); j++) { L.add(t, L.term(j + 1), true); L.divideByP(t); }
  return L.form(t, dst);
}
// Chen and Han's digit: G(tmp) (src/extractDigits.cpp:283)
inline void liftDigit(Ctxt& d, const std::vector<long>& G, const Ctxt& tmp) {
  HB_NTIMER_START(digit_lift, d.context.handle());
  polyEval(d, G, tmp);
}
inline void digitChain(Ctxt& dst, const Ctxt& c, const std::vector<const Ctxt*>& sub, bool fused) {
  if (sub.empty()) { dst = c; return; }
  HB_NTIMER_START(digit_chain, c.context.handle());
  if (!fused || !digitChainFused(dst, c, sub)) digitChainLoop(dst, c, sub);
}
}  // namespace detail

// hb::extractDigits (src/extractDigits.cpp:70-129): digits[j] holds the j-th base-p digit of the slots of c (integers mod
// p^r), at plaintext space p^(r-j).  Round i powers digits 0..i-1 (square for p = 2, cube for p = 3, the digit polynomial
// through polyEval otherwise) and forms c minus them, divided by p after each, in one hb_ctxt_scaled_sums call.
// fused = false runs the chains as transcribed (the reference the tests compare against).
inline void extractDigits(std::vector<Ctxt>& digits, const Ctxt& c, long r = 0, bool fused = true) {
  const long rr = c.effectiveR();
  if (r <= 0 || r > rr) r = rr;
  const long p = c.context.getP();
  std::vector<long> x2p;
  if (p > 3) x2p = xd::buildDigitPolynomial(p, r);
  Ctxt tmp(c.pubKey, c.ptxtSpace);
  digits.resize((size_t)r, tmp);
  for (long i = 0; i < r; i++) {
    std::vector<const Ctxt*> sub;
    for (long j = 0; j < i; j++) { detail::powerDigit(digits[(size_t)j], x2p); sub.push_back(&digits[(size_t)j]); }
    detail::digitChain(digits[(size_t)i], c, sub, fused);
  }
}

// hb::extendExtractDigits (src/extractDigits.cpp:225-308), Chen and Han's variant: c holds integers mod p^(r+e) in its
// slots; digits[i] = G_{e+r-i}(the i-th chain), at plaintext space p^(e+r-i).  Each chain subtracts whichever of digits[j]
// and the powered digits0[j] has more capacity, as HElib does, in one hb_ctxt_scaled_sums call.
inline void extendExtractDigits(std::vector<Ctxt>& digits, const Ctxt& c, long r, long e, bool fused = true) {
  const long p = c.context.getP();
  std::vector<long> x2p;
  if (p > 3) x2p = xd::buildDigitPolynomial(p, r);
  std::vector<std::vector<long>> G((size_t)std::max(0L, r));
  for (long i = 0; i < r; i++) G[(size_t)i] = xd::chenHanMagicPoly(p, e + r - i);
  Ctxt tmp(c.pubKey, c.ptxtSpace);
  digits.resize((size_t)r, tmp);
  std::vector<Ctxt> digits0((size_t)r, tmp);
  for (long i = 0; i < r; i++) {
    std::vector<const Ctxt*> sub;
    for (long j = 0; j < i; j++) {
      if (digits[(size_t)j].capacity() >= digits0[(size_t)j].capacity()) sub.push_back(&digits[(size_t)j]);
      else { detail::powerDigit(digits0[(size_t)j], x2p); sub.push_back(&digits0[(size_t)j]); }
    }
    detail::digitChain(digits0[(size_t)i], c, sub, fused);
    detail::liftDigit(digits[(size_t)i], G[(size_t)i], digits0[(size_t)i]);
  }
}

namespace detail {
// extractDigitsThin's final combination (src/recryption.cpp:852-867 and 881-907): from `top` (the Chen-Han branch's
// chain, or the highest selected digit) down, then the p = 2 bit, the negation and the bottom digits, mod p^r
struct ThinPlan {
  long start = -1;   // -1: top = unpacked - scratch[0..botHigh) with a divideByP after each (Chen-Han); else scratch[start]
  long lo = 0;       // the basic branch's digits start-1 .. lo, each after a multByP
  long botHigh = 0, r = 0, ePrime = 0, p = 0;
};
inline void thinCombineLoop(Ctxt& unpacked, const std::vector<Ctxt>& s, const ThinPlan& P) {
  if (P.start < 0) {
    for (long j = 0; j < P.botHigh; j++) { unpacked -= s[(size_t)j]; unpacked.divideByP(); }
  } else {
    unpacked = s[(size_t)P.start];
    for (long j = P.start - 1; j >= P.lo; --j) { unpacked.multByP(); unpacked += s[(size_t)j]; }
  }
  if (P.p == 2 && P.botHigh > 0) unpacked += s[(size_t)P.botHigh - 1];
  unpacked.negate();
  if (P.r > P.ePrime) {
    const long topLow = P.r - 1 - P.ePrime;
    Ctxt tmp = s.at((size_t)topLow);
    for (long j = topLow - 1; j >= 0; --j) { tmp.multByP(); tmp += s[(size_t)j]; }
    if (P.ePrime > 0) tmp.multByP(P.ePrime);
    unpacked += tmp;
  }
  unpacked.reducePtxtSpace(xd::power(P.p, P.r));
}
inline bool thinCombineFused(Ctxt& unpacked, const std::vector<Ctxt>& s, const ThinPlan& P) {
  std::vector<const Ctxt*> in;
  if (P.start < 0) in.push_back(&unpacked);
  for (const Ctxt& x : s) in.push_back(&x);
  LinearChain L(in);
  if (!L.ok) return false;
  const size_t o = P.start < 0 ? 1 : 0;   // input index of scratch[0]
  auto S = [&](long j) { return L.term(o + (size_t)j); };
  LinearChain::Term t = P.start < 0 ? L.term(0) : S(P.start);
  if (P.start < 0) for (long j = 0; j < P.botHigh; j++) { L.add(t, S(j), true); L.divideByP(t); }
  else for (long j = P.start - 1; j >= P.lo; --j) { L.multByP(t); L.add(t, S(j)); }
  if (P.p == 2 && P.botHigh > 0) L.add(t, S(P.botHigh - 1));
  L.negate(t);
  if (P.r > P.ePrime) {
    const long topLow = P.r - 1 - P.ePrime;
    LinearChain::Term b = S(topLow);
    for (long j = topLow - 1; j >= 0; --j) { L.multByP(b); L.add(b, S(j)); }
    if (P.ePrime > 0) L.multByP(b, P.ePrime);
    L.add(t, b);
  }
  L.reducePtxtSpace(t, xd::power(P.p, P.r));
  return L.form(t, unpacked);
}
}  // namespace detail

// hb::extractDigitsThin (src/recryption.cpp:793-909): ctxt's slots hold integers mod p^(botHigh+r); ctxt becomes
// -(digits botHigh .. botHigh+r-1, as one integer mod p^r) plus, for r > ePrime, the digits below r-ePrime times p^ePrime,
// at plaintext space p^r.  The cost rule picks Chen and Han's method or the basic one; chenHan > 0 forces the former and
// chenHan < 0 the latter (HElib's global fhe_force_chen_han).  The final combination is one hb_ctxt_scaled_sums call.
inline void extractDigitsThin(Ctxt& ctxt, long botHigh, long r, long ePrime, long chenHan = 0, bool fused = true) {
  Ctxt unpacked(ctxt);
  unpacked.cleanUp();
  std::vector<Ctxt> scratch;
  const long p = ctxt.context.getP();
  long topHigh = botHigh + r - 1;
  bool useChenHan = false;
  if (r > 1) {   // degree of Chen-Han p^(bot-1)(p-1)r; of the basic method p^(bot-1)p^r, or p^(bot-1)p^(r-1) for a free bit
    const double chenHanCost = std::log((double)(p - 1)) + std::log((double)r);
    const double basicCost = (p == 2 && r > 2 && botHigh + r > 2) ? (r - 1) * std::log((double)p) : r * std::log((double)p);
    const double thresh = p == 2 ? 1.75 : 1.5;   // squaring is cheaper: p = 2 leans to the basic method
    if (basicCost > thresh * chenHanCost) useChenHan = true;
  }
  if (chenHan > 0) useChenHan = true;
  else if (chenHan < 0) useChenHan = false;
  detail::ThinPlan plan;
  plan.botHigh = botHigh; plan.r = r; plan.ePrime = ePrime; plan.p = p;
  if (useChenHan) {
    extendExtractDigits(scratch, unpacked, botHigh, r, fused);
  } else {
    if (p == 2 && r > 2 && topHigh + 1 > 2) topHigh--;   // for p = 2 the top bit comes for free
    extractDigits(scratch, unpacked, topHigh + 1, fused);
    if (topHigh >= (long)scratch.size()) topHigh = (long)scratch.size() - 1;   // not enough digits: HElib warns and goes on
    plan.start = topHigh;
    plan.lo = botHigh;
  }
  {
    HB_NTIMER_START(thin_combine, ctxt.context.handle());
    if (!fused || !detail::thinCombineFused(unpacked, scratch, plan)) detail::thinCombineLoop(unpacked, scratch, plan);
  }
  ctxt = unpacked;
}

}  // namespace hb
