// helib_b200_doublecrt.hpp -- header-only C++17 mirror of helib::DoubleCRT over the C ABI.
//
// Same method names, argument meaning and error behaviour as the reference class
// (include/helib/DoubleCRT.h:120-463), so that a maintainer can alias `helib::DoubleCRT` to
// `hb::DoubleCRT` inside an NTL-equipped HElib build (INTEGRATION.md).  NTL types are replaced by
// plain C++ ones here (ZZX -> vector of two's-complement limbs, IndexSet -> hb::IndexSet) because
// this repository cannot link NTL; the shim in INTEGRATION.md shows the two conversions.
//
// Value semantics like the reference: copying a DoubleCRT copies its rows (device-to-device).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <memory>
#include <set>
#include <stdexcept>
#include <string>
#include <vector>
#include <ostream>
#include <istream>
#include <cstring>
#include <chrono>
#include <map>
#include <mutex>
#include <type_traits>

#include "helib_b200.h"
#include "helib_b200_chain.h"

namespace hb {

// helib's exception taxonomy (include/helib/exceptions.h:52-139)
struct RuntimeError : std::runtime_error { using std::runtime_error::runtime_error; };
struct LogicError : std::logic_error { using std::logic_error::logic_error; };
struct InvalidArgument : std::invalid_argument { using std::invalid_argument::invalid_argument; };

inline void check(int rc) {
  if (rc == HB_OK) return;
  std::string msg = hb_last_error();
  if (rc == HB_ERR_INDEX_SET) throw RuntimeError(msg);
  if (rc == HB_ERR_BAD_ARG) throw InvalidArgument(msg);
  if (rc == HB_ERR_UNSUPPORTED) throw LogicError(msg);
  throw RuntimeError(msg);
}


// helib's timers and statistics (include/helib/timing.h:44-128, src/timing.cpp:21-110, include/helib/fhe_stats.h:38-52) under the
// reference's own names on the host wrappers (FFT, toPoly, addPrimes, breakIntoDigits, scaleDownToSet, KS_loop, reLinearize, ...):
// getTimerByName / printAllTimers / fhe_stats keep working for a caller that reads them.  Engine calls are asynchronous, so a
// timer measures real time only in timing mode (setTimersOn(): every timed wrapper synchronises its context before it stops --
// a profiling mode, like the reference's always-on CPU timers); off by default (call counts only, no synchronisation).
// Per-kernel device times come from hb_ctx_profile.
struct FHEtimer {
  const char* name; const char* loc;
  long counter = 0;      // microseconds
  long numCalls = 0;
  FHEtimer(const char* n, const char* l);
  double getTime() const { return counter / 1e6; }
  long getNumCalls() const { return numCalls; }
};
inline std::vector<FHEtimer*>& timerMap() { static std::vector<FHEtimer*> v; return v; }
inline std::mutex& timerMutex() { static std::mutex m; return m; }
inline FHEtimer::FHEtimer(const char* n, const char* l) : name(n), loc(l) { std::lock_guard<std::mutex> g(timerMutex()); timerMap().push_back(this); }
inline bool& timersOn() { static bool on = false; return on; }
inline void setTimersOn() { timersOn() = true; }
inline void setTimersOff() { timersOn() = false; }
inline const FHEtimer* getTimerByName(const char* name) {
  std::lock_guard<std::mutex> g(timerMutex());
  for (FHEtimer* t : timerMap()) if (std::strcmp(t->name, name) == 0) return t;
  return nullptr;
}
inline void resetAllTimers() { std::lock_guard<std::mutex> g(timerMutex()); for (FHEtimer* t : timerMap()) { t->counter = 0; t->numCalls = 0; } }
inline void printAllTimers(std::ostream& str) {   // name: total / calls = avg [location]   (src/timing.cpp:92-110)
  std::lock_guard<std::mutex> g(timerMutex());
  for (const FHEtimer* t : timerMap())
    if (t->numCalls > 0)
      str << "  " << t->name << ": " << t->getTime() << " / " << t->numCalls << " = " << t->getTime() / t->numCalls << "   [" << t->loc << "]\n";
}
struct auto_timer {
  FHEtimer* t; hb_ctx* ctx; std::chrono::steady_clock::time_point t0; bool running;
  auto_timer(FHEtimer* t_, hb_ctx* c) : t(t_), ctx(c), running(true) { t->numCalls++; if (timersOn()) t0 = std::chrono::steady_clock::now(); }
  void stop() {
    if (!running) return;
    running = false;
    if (!timersOn()) return;
    if (ctx) hb_ctx_sync(ctx);
    t->counter += (long)std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count();
  }
  ~auto_timer() { stop(); }
};
#define HB_STR2(x) #x
#define HB_STR(x) HB_STR2(x)
#define HB_AT __FILE__ ":" HB_STR(__LINE__)
#define HB_TIMER_START(ctx) static hb::FHEtimer _local_timer(__func__, HB_AT); hb::auto_timer _local_auto_timer(&_local_timer, (ctx))
#define HB_NTIMER_START(n, ctx) static hb::FHEtimer _named_local_timer##n(#n, HB_AT); hb::auto_timer _named_local_auto_timer##n(&_named_local_timer##n, (ctx))
// HELIB_STATS_UPDATE (include/helib/fhe_stats.h:38-52): gated by the global switch, keeps count / sum / max per name
struct fhe_stats_record { long count = 0; double sum = 0, max = 0; };
inline bool& fhe_stats() { static bool on = false; return on; }
inline std::map<std::string, fhe_stats_record>& fhe_stats_map() { static std::map<std::string, fhe_stats_record> m; return m; }
inline void stats_update(const char* name, double val) {
  if (!fhe_stats()) return;
  std::lock_guard<std::mutex> g(timerMutex());
  fhe_stats_record& r = fhe_stats_map()[name];
  r.count++; r.sum += val; if (val > r.max) r.max = val;
}
#define HB_STATS_UPDATE(name, val) hb::stats_update((name), (val))

// helib::IndexSet (include/helib/IndexSet.h) restricted to what the hot path uses
class IndexSet {
  std::set<long> s_;
 public:
  IndexSet() = default;
  IndexSet(long lo, long hi) { for (long i = lo; i <= hi; i++) s_.insert(i); }
  explicit IndexSet(long i) { s_.insert(i); }
  IndexSet(std::initializer_list<long> l) : s_(l) {}
  template <class It> IndexSet(It a, It b) : s_(a, b) {}
  static IndexSet emptySet() { return IndexSet(); }
  long card() const { return (long)s_.size(); }
  bool contains(long i) const { return s_.count(i) != 0; }
  bool contains(const IndexSet& o) const { return std::includes(s_.begin(), s_.end(), o.s_.begin(), o.s_.end()); }
  bool disjointFrom(const IndexSet& o) const { for (long i : o.s_) if (s_.count(i)) return false; return true; }
  void insert(long i) { s_.insert(i); }
  void insert(const IndexSet& o) { s_.insert(o.s_.begin(), o.s_.end()); }
  void remove(long i) { s_.erase(i); }
  void remove(const IndexSet& o) { for (long i : o.s_) s_.erase(i); }
  void retain(const IndexSet& o) { for (auto it = s_.begin(); it != s_.end();) it = o.s_.count(*it) ? std::next(it) : s_.erase(it); }
  long first() const { return s_.empty() ? 0 : *s_.begin(); }
  long last() const { return s_.empty() ? -1 : *s_.rbegin(); }
  bool isInterval() const { return s_.empty() || last() - first() + 1 == card(); }
  auto begin() const { return s_.begin(); }
  auto end() const { return s_.end(); }
  bool operator==(const IndexSet& o) const { return s_ == o.s_; }
  bool operator!=(const IndexSet& o) const { return s_ != o.s_; }
  bool operator<=(const IndexSet& o) const { return o.contains(*this); }
  bool operator>=(const IndexSet& o) const { return contains(o); }
  IndexSet operator|(const IndexSet& o) const { IndexSet r = *this; r.insert(o); return r; }
  IndexSet operator&(const IndexSet& o) const { IndexSet r = *this; r.retain(o); return r; }
  IndexSet operator/(const IndexSet& o) const { IndexSet r = *this; r.remove(o); return r; }  // set minus
  std::vector<int32_t> vec() const { return std::vector<int32_t>(s_.begin(), s_.end()); }
};
inline bool empty(const IndexSet& s) { return s.card() == 0; }
inline bool disjoint(const IndexSet& a, const IndexSet& b) { return a.disjointFrom(b); }

// helib::Context reduced to the chain + its device image (include/helib/Context.h)
class Context {
  hb_chain* chain_ = nullptr;
  hb_ctx* ctx_ = nullptr;
  std::vector<uint64_t> primes_;
  IndexSet small_, ctxt_, special_;
  std::vector<IndexSet> digits_;
  long m_, phim_, p_, r_;
 public:
  // psi (optional, one per chain prime): the primitive m-th root every row is evaluated at.  A build of the reference derives its
  // roots from NTL's zz_pContext tables (src/CModulus.cpp:93-119): hand them over (Cmodulus::FFT of the monomial X yields psi in
  // y[0]) to make rows and the writeTo/read bytes interchangeable with that build; without it the engine picks its own root.
  Context(long m, long p, long r, long bits, long c, int device = 0, const std::vector<uint64_t>* psi = nullptr) : m_(m), p_(p), r_(r) {
    if (hb_chain_build(&chain_, (uint64_t)m, p, (int)r, (int)bits, (int)c, 0, 3, 0, 3.2) != HB_OK)
      throw InvalidArgument(hb_chain_last_error());
    int np, ns, nc, nsp, nd; int64_t phim;
    hb_chain_info(chain_, &np, &ns, &nc, &nsp, &nd, &phim);
    phim_ = (long)phim;
    primes_.resize(np);
    std::vector<int32_t> kind(np), dig(np);
    hb_chain_get(chain_, primes_.data(), kind.data(), dig.data());
    digits_.resize(nd);
    std::vector<int32_t> sp;
    for (int i = 0; i < np; i++) {
      if (kind[i] == 0) small_.insert(i);
      else if (kind[i] == 1) { ctxt_.insert(i); if (dig[i] >= 0) digits_[dig[i]].insert(i); }
      else { special_.insert(i); sp.push_back(i); }
    }
    if (psi && (int)psi->size() != np) throw InvalidArgument("Context: one root per chain prime expected");
    check(hb_ctx_create(&ctx_, device, (uint64_t)m, np, primes_.data(), psi ? psi->data() : nullptr));
    check(hb_ctx_set_chain(ctx_, dig.data(), nd, sp.data(), (int)sp.size()));
  }
  ~Context() { if (ctx_) hb_ctx_destroy(ctx_); if (chain_) hb_chain_destroy(chain_); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
  long getM() const { return m_; }
  long getP() const { return p_; }
  long getR() const { return r_; }
  long getPhiM() const { return phim_; }
  long numPrimes() const { return (long)primes_.size(); }
  long ithPrime(long i) const { return (long)primes_.at(i); }
  const IndexSet& getSmallPrimes() const { return small_; }
  const IndexSet& getCtxtPrimes() const { return ctxt_; }
  const IndexSet& getSpecialPrimes() const { return special_; }
  const std::vector<IndexSet>& getDigits() const { return digits_; }
  const IndexSet& getDigit(long i) const { return digits_.at(i); }
  hb_ctx* handle() const { return ctx_; }
  hb_chain* chain() const { return chain_; }
  void sync() const { check(hb_ctx_sync(ctx_)); }
};

class DoubleCRT {
  const Context* context_;
  IndexSet set_;
  hb_poly* p_ = nullptr;
  void alloc() { check(hb_poly_create(context_->handle(), &p_)); }
 public:
  // DoubleCRT(context, indexSet): zero object on the given primes (DoubleCRT.h:153-158)
  DoubleCRT(const Context& ctx, const IndexSet& s) : context_(&ctx), set_(s) { alloc(); }
  // DoubleCRT(zzX poly, context, indexSet): small-coefficient polynomial (DoubleCRT.h:140-151)
  // One copy of the coefficients crosses the bus; the per-prime reduction and the transforms run on the device.
  DoubleCRT(const std::vector<long>& poly, const Context& ctx, const IndexSet& s) : context_(&ctx), set_(s) {
    HB_NTIMER_START(FFT, ctx.handle());   // DoubleCRT::FFT (src/DoubleCRT.cpp:68-105)
    alloc();
    const long N = ctx.getPhiM();
    if ((long)poly.size() > N) throw InvalidArgument("polynomial degree >= phi(m)");
    std::vector<int64_t> c(poly.begin(), poly.end()); c.resize((size_t)N, 0);
    auto idx = s.vec();
    hb_poly* arr[1] = {p_};
    if (!idx.empty()) check(hb_poly_from_i64(arr, 1, idx.data(), (int)idx.size(), c.data()));
  }
  // DoubleCRT(ZZX poly, context, indexSet) (DoubleCRT.h:129-138): big coefficients as N x L little-endian
  // two's-complement limbs (the layout toPoly returns; NTL side: BytesFromZZ + sign, see INTEGRATION.md)
  static DoubleCRT fromLimbs(const Context& ctx, const IndexSet& s, const std::vector<uint64_t>& limbs, int L) {
    if (L < 1 || limbs.size() != (size_t)ctx.getPhiM() * L) throw InvalidArgument("fromLimbs: expected phi(m) x L limbs");
    DoubleCRT r(ctx, s);
    auto idx = s.vec();
    hb_poly* arr[1] = {r.p_};
    if (!idx.empty()) check(hb_poly_from_limbs(arr, 1, idx.data(), (int)idx.size(), limbs.data(), L));
    return r;
  }
  DoubleCRT(const DoubleCRT& o) : context_(o.context_), set_(o.set_) {
    alloc();
    auto idx = set_.vec();
    if (!idx.empty()) { hb_poly* d[1] = {p_}; hb_poly* s[1] = {o.p_}; check(hb_pointwise(HB_OP_COPY, d, s, 1, idx.data(), (int)idx.size())); }
  }
  DoubleCRT& operator=(const DoubleCRT& o) {
    if (this == &o) return *this;
    if (context_ != o.context_) throw RuntimeError("DoubleCRT assignment: incompatible contexts");
    set_ = o.set_;
    auto idx = set_.vec();
    if (!idx.empty()) { hb_poly* d[1] = {p_}; hb_poly* s[1] = {o.p_}; check(hb_pointwise(HB_OP_COPY, d, s, 1, idx.data(), (int)idx.size())); }
    return *this;
  }
  ~DoubleCRT() { if (p_) hb_poly_destroy(p_); }

  const Context& getContext() const { return *context_; }
  const IndexSet& getIndexSet() const { return set_; }
  hb_poly* handle() const { return p_; }

  // Op<Add/Sub/Mul> (src/DoubleCRT.cpp:216-337): other must cover this's primes
  DoubleCRT& Op(const DoubleCRT& other, int op, bool matchIndexSets) {
    HB_TIMER_START(context_->handle());
    if (context_ != other.context_) throw RuntimeError("DoubleCRT::Op: incompatible objects");
    if (matchIndexSets && !(set_ >= other.set_)) throw RuntimeError("DoubleCRT::Op: matchIndexSets not honored");
    if (!(set_ <= other.set_)) throw RuntimeError("DoubleCRT::Op: !(map.getIndexSet() <= other.map.getIndexSet())");
    auto idx = set_.vec();
    if (idx.empty()) return *this;
    hb_poly* d[1] = {p_}; hb_poly* s[1] = {other.p_};
    check(hb_pointwise(op, d, s, 1, idx.data(), (int)idx.size()));
    return *this;
  }
  DoubleCRT& Add(const DoubleCRT& o, bool matchIndexSets = true) { return Op(o, HB_OP_ADD, matchIndexSets); }
  DoubleCRT& Sub(const DoubleCRT& o, bool matchIndexSets = true) { return Op(o, HB_OP_SUB, matchIndexSets); }
  DoubleCRT& Mul(const DoubleCRT& o, bool matchIndexSets = true) { return Op(o, HB_OP_MUL, matchIndexSets); }
  DoubleCRT& operator+=(const DoubleCRT& o) { return Add(o); }
  DoubleCRT& operator-=(const DoubleCRT& o) { return Sub(o); }
  DoubleCRT& operator*=(const DoubleCRT& o) { return Mul(o); }
  DoubleCRT& Negate() {
    auto idx = set_.vec();
    if (!idx.empty()) { hb_poly* d[1] = {p_}; check(hb_pointwise(HB_OP_NEG, d, d, 1, idx.data(), (int)idx.size())); }
    return *this;
  }
  // Op(ZZ, MulFun) for a word-sized scalar (src/DoubleCRT.cpp:339-361)
  DoubleCRT& operator*=(long num) {
    auto idx = set_.vec();
    std::vector<uint64_t> sc;
    for (int i : idx) { long q = context_->ithPrime(i); long v = num % q; sc.push_back((uint64_t)(v < 0 ? v + q : v)); }
    if (!idx.empty()) { hb_poly* d[1] = {p_}; check(hb_scale_rows(d, 1, idx.data(), (int)idx.size(), sc.data())); }
    return *this;
  }
  // Op(ZZ, MulFun) for a big non-negative scalar given as mant * 2^shift (the integers NTL converts out of an xdouble)
  DoubleCRT& mulByPow2Scaled(uint64_t mant, long shift) {
    auto idx = set_.vec();
    std::vector<uint64_t> sc;
    for (int i : idx) {
      const uint64_t q = (uint64_t)context_->ithPrime(i);
      unsigned __int128 r = mant % q, b = 2 % q;
      for (long e = shift; e > 0; e >>= 1) { if (e & 1) r = r * b % q; b = b * b % q; }
      sc.push_back((uint64_t)r);
    }
    if (!idx.empty()) { hb_poly* d[1] = {p_}; check(hb_scale_rows(d, 1, idx.data(), (int)idx.size(), sc.data())); }
    return *this;
  }
  // operator/= by the product of a set of chain primes (what the hot path divides by; src/DoubleCRT.cpp:1122-1139)
  DoubleCRT& divideByPrimes(const IndexSet& f) {
    auto idx = set_.vec(), fi = f.vec();
    if (!idx.empty()) { hb_poly* d[1] = {p_}; check(hb_scale_by_primes(d, 1, idx.data(), (int)idx.size(), fi.data(), (int)fi.size(), 1)); }
    return *this;
  }
  // automorph / complexConj (src/DoubleCRT.cpp:1160-1255)
  void automorph(long k) {
    HB_TIMER_START(context_->handle());
    DoubleCRT tmp(*this);
    auto idx = set_.vec();
    if (idx.empty()) return;
    hb_poly* d[1] = {p_}; hb_poly* s[1] = {tmp.p_};
    check(hb_automorph(d, s, 1, idx.data(), (int)idx.size(), (uint64_t)k));
  }
  void complexConj() { automorph(context_->getM() - 1); }
  // removePrimes / addPrimes / addPrimesAndScale (src/DoubleCRT.cpp:565-647)
  void removePrimes(const IndexSet& s) { set_.remove(s); }
  void addPrimes(const IndexSet& s1) {
    HB_TIMER_START(context_->handle());
    if (empty(s1)) return;
    auto cur = set_.vec(), add = s1.vec();
    hb_poly* d[1] = {p_};
    check(hb_add_primes(d, 1, cur.data(), (int)cur.size(), add.data(), (int)add.size()));
    set_.insert(s1);
  }
  double addPrimesAndScale(const IndexSet& s1) {
    if (empty(s1)) return 0.0;
    auto cur = set_.vec(), add = s1.vec();
    hb_poly* d[1] = {p_};
    check(hb_add_primes_and_scale(d, 1, cur.data(), (int)cur.size(), add.data(), (int)add.size()));
    bool was_empty = empty(set_);
    set_.insert(s1);
    if (was_empty) return 0.0;
    double lf = 0; for (long i : s1) lf += std::log((double)context_->ithPrime(i));
    return lf;
  }
  // scaleDownToSet (src/DoubleCRT.cpp:1464-1516)
  void scaleDownToSet(const IndexSet& s, long ptxtSpace) {
    HB_TIMER_START(context_->handle());
    IndexSet diff = set_ / s;
    if (empty(diff)) return;
    if (ptxtSpace < 1) throw InvalidArgument("ptxtSpace must be at least 1");
    auto cur = set_.vec(), keep = (set_ & s).vec();
    hb_poly* d[1] = {p_};
    check(hb_scale_down(d, 1, cur.data(), (int)cur.size(), keep.data(), (int)keep.size(), (uint64_t)ptxtSpace));
    set_.remove(diff);
  }
  // breakIntoDigits (src/DoubleCRT.cpp:479-561); the FP64 noise norm it returns is host metadata (not computed)
  void breakIntoDigits(std::vector<DoubleCRT>& digits) const {
    HB_TIMER_START(context_->handle());
    const long maxdig = (long)context_->getDigits().size();
    digits.clear();
    IndexSet all = set_ | context_->getSpecialPrimes();
    for (long i = 0; i < maxdig; i++) digits.emplace_back(*context_, all);
    std::vector<hb_poly*> dp;
    for (auto& d : digits) dp.push_back(d.p_);
    auto cur = set_.vec();
    hb_poly* s[1] = {p_};
    int nd = 0;
    check(hb_break_into_digits(s, 1, cur.data(), (int)cur.size(), dp.data(), (int)maxdig, &nd));
    digits.erase(digits.begin() + nd, digits.end());
  }
  // scaleDownToSet that also returns ||delta/P||_canon, the quantity Ctxt::modDownToSet derives from the
  // returned delta (src/Ctxt.cpp:476-505); computed on the device.
  double scaleDownToSetNorm(const IndexSet& s, long ptxtSpace) {
    IndexSet diff = set_ / s;
    if (empty(diff)) return 0.0;
    if (ptxtSpace < 1) throw InvalidArgument("ptxtSpace must be at least 1");
    auto cur = set_.vec(), keep = (set_ & s).vec();
    hb_poly* d[1] = {p_};
    double norm = 0;
    check(hb_scale_down_norm(d, 1, cur.data(), (int)cur.size(), keep.data(), (int)keep.size(), (uint64_t)ptxtSpace, &norm));
    set_.remove(diff);
    return norm;
  }
  // breakIntoDigits returning ln ||E_i||_canon per digit (the reference returns their sum, src/DoubleCRT.cpp:542-545)
  std::vector<double> breakIntoDigitsLogNorms(std::vector<DoubleCRT>& digits) const {
    const long maxdig = (long)context_->getDigits().size();
    digits.clear();
    IndexSet all = set_ | context_->getSpecialPrimes();
    for (long i = 0; i < maxdig; i++) digits.emplace_back(*context_, all);
    std::vector<hb_poly*> dp;
    for (auto& d : digits) dp.push_back(d.p_);
    auto cur = set_.vec();
    hb_poly* s[1] = {p_};
    int nd = 0;
    std::vector<double> ln(maxdig);
    check(hb_break_into_digits_norm(s, 1, cur.data(), (int)cur.size(), dp.data(), (int)maxdig, &nd, ln.data()));
    digits.erase(digits.begin() + nd, digits.end());
    ln.resize(nd);
    return ln;
  }
  // multiply by the product of a set of chain primes (DoubleCRT::Op(ZZ, MulFun) with that ZZ, src/DoubleCRT.cpp:339-361)
  DoubleCRT& multiplyByPrimes(const IndexSet& f) {
    auto idx = set_.vec(), fi = f.vec();
    if (!idx.empty() && !fi.empty()) { hb_poly* d[1] = {p_}; check(hb_scale_by_primes(d, 1, idx.data(), (int)idx.size(), fi.data(), (int)fi.size(), 0)); }
    return *this;
  }
  // evaluation rows given directly (what DoubleCRT::randomize fills, src/DoubleCRT.cpp:1258-1378): dense [nprimes][N]
  static DoubleCRT fromRows(const Context& ctx, const IndexSet& s, const std::vector<uint64_t>& dense) {
    DoubleCRT r(ctx, s);
    auto idx = s.vec();
    if (!idx.empty()) check(hb_poly_upload(r.p_, idx.data(), (int)idx.size(), dense.data()));
    check(hb_ctx_sync(ctx.handle()));
    return r;
  }
  // DoubleCRT::randomize (src/DoubleCRT.cpp:1258-1378): uniform rows by rejection sampling from a byte stream --
  // get(buf, 2048) stands for NTL::RandomStream::get (the ChaCha20 stream keyed by SetSeed; not restated).  A fresh 2048-byte
  // buffer per refill and per row, nb = ceil(bits(q-1)/8) little-endian bytes per candidate, masked, accepted when < q.
  // Runs on the host (once per key-switching matrix) and uploads the rows.
  template <class GetBytes, std::enable_if_t<!std::is_same<std::decay_t<GetBytes>, std::vector<uint8_t>>::value, int> = 0>
  void randomize(GetBytes&& get) {
    const long N = context_->getPhiM(), bufsz = 2048;
    std::vector<uint64_t> dense((size_t)context_->numPrimes() * N, 0);
    std::vector<unsigned char> buf((size_t)bufsz);
    for (long i : set_) {
      const uint64_t q = (uint64_t)context_->ithPrime(i);
      long k = 0; for (uint64_t t = q - 1; t; t >>= 1) k++;
      const long nb = (k + 7) / 8;
      const uint64_t mask = k >= 64 ? ~0ULL : ((1ULL << k) - 1ULL);
      uint64_t* row = &dense[(size_t)i * N];
      long j = 0;
      while (j < N) {
        get(buf.data(), bufsz);
        for (long pos = 0; pos <= bufsz - nb && j < N; pos += nb) {
          uint64_t u = 0;
          for (long c = nb - 1; c >= 0; c--) u = (u << 8) | buf[(size_t)(pos + c)];
          u &= mask;
          row[j] = u;
          j += (u < q);
        }
      }
    }
    auto idx = set_.vec();
    if (!idx.empty()) check(hb_poly_upload(p_, idx.data(), (int)idx.size(), dense.data()));
    check(hb_ctx_sync(context_->handle()));
  }
  // randomize(&seed) (src/DoubleCRT.cpp:1258-1378 after NTL::SetSeed(seed)): the same rows from NTL's own stream, expanded
  // on the device.  seed = the little-endian magnitude bytes of the ZZ (high-order zero bytes do not count; empty = 0).
  void randomize(const std::vector<uint8_t>& seed) {
    auto idx = set_.vec();
    hb_poly* d[1] = {p_};
    if (!idx.empty()) check(hb_poly_randomize(d, 1, idx.data(), (int)idx.size(), seed.data(), (int)seed.size()));
  }
  // toPoly (src/DoubleCRT.cpp:925-1113): N x L little-endian two's-complement limbs
  std::vector<uint64_t> toPoly(const IndexSet& s, bool positive, int& L) const {
    HB_TIMER_START(context_->handle());
    auto idx = (set_ & s).vec();
    L = (int)idx.size() + 1;
    std::vector<uint64_t> out((size_t)context_->getPhiM() * L);
    check(hb_to_poly(p_, idx.data(), (int)idx.size(), positive ? 1 : 0, out.data(), L));
    return out;
  }
  // *this += a * b on this object's primes (both operands must cover them): `key *= part; ptxt += key`
  // (src/keys.cpp:1373-1374) and `parts[i] *= r; parts[i] += e` (src/keys.cpp:416,443) without the temporary
  DoubleCRT& mulAdd(const DoubleCRT& a, const DoubleCRT& b) {
    if (context_ != a.context_ || context_ != b.context_) throw RuntimeError("DoubleCRT::Op: incompatible objects");  // src/DoubleCRT.cpp:222-223
    if (!(set_ <= a.set_) || !(set_ <= b.set_)) throw RuntimeError("DoubleCRT::Op: !(map.getIndexSet() <= other.map.getIndexSet())");
    auto idx = set_.vec();
    hb_poly* d[1] = {p_}; hb_poly* x[1] = {a.p_}; hb_poly* y[1] = {b.p_};
    if (!idx.empty()) check(hb_muladd(d, x, y, 1, idx.data(), (int)idx.size()));
    return *this;
  }
  // PolyRed(toPoly(s), ptxtSpace, abs=true) * factor mod ptxtSpace: the tail of SecKey::Decrypt (src/keys.cpp:1381-1399)
  std::vector<long> toPolyModP(const IndexSet& s, long ptxtSpace, long factor = 1) const {
    auto idx = (set_ & s).vec();
    std::vector<int64_t> out((size_t)context_->getPhiM());
    check(hb_to_poly_mod_p(p_, idx.data(), (int)idx.size(), (uint64_t)ptxtSpace, (uint64_t)factor, out.data()));
    return std::vector<long>(out.begin(), out.end());
  }
  // DoubleCRT::writeTo / read (src/DoubleCRT.cpp:1530-1561): IndexSet, then per row int32 length, int32 intSize, LE values
  void writeTo(std::ostream& str) const {
    auto idx = set_.vec();
    uint64_t bytes = 0;
    check(hb_poly_serialized_size(p_, (int)idx.size(), &bytes));
    std::vector<char> buf((size_t)bytes);
    check(hb_poly_serialize(p_, idx.data(), (int)idx.size(), buf.data(), bytes));
    str.write(buf.data(), (std::streamsize)buf.size());
  }
  void read(std::istream& str) {
    // the record is self-delimiting: read the index set first, then the rows it announces
    std::vector<char> buf(8);
    str.read(buf.data(), 8);
    int64_t card = 0; std::memcpy(&card, buf.data(), 8);
    if (!str || card < 0 || card > context_->numPrimes()) throw RuntimeError("DoubleCRT::read: bad index set");
    buf.resize(8 + 8 * (size_t)card);
    str.read(buf.data() + 8, 8 * card);
    for (int64_t r = 0; r < card; r++) {
      size_t off = buf.size(); buf.resize(off + 8);
      str.read(buf.data() + off, 8);
      int32_t len = 0, isz = 0; std::memcpy(&len, buf.data() + off, 4); std::memcpy(&isz, buf.data() + off + 4, 4);
      if (!str || len < 0 || (isz != 4 && isz != 8)) throw RuntimeError("DoubleCRT::read: bad row header");
      size_t off2 = buf.size(); buf.resize(off2 + (size_t)len * isz);
      str.read(buf.data() + off2, (std::streamsize)len * isz);
    }
    if (!str) throw RuntimeError("DoubleCRT::read: truncated input");
    std::vector<int32_t> idx((size_t)context_->numPrimes()); int n = 0;
    check(hb_poly_deserialize(p_, buf.data(), buf.size(), idx.data(), &n));
    set_ = IndexSet(idx.begin(), idx.begin() + n);
  }
  // getOneRow (DoubleCRT.h:332-336)
  std::vector<long> getOneRow(long i) const {
    if (!set_.contains(i)) throw RuntimeError("getOneRow: prime not in index set");
    const long N = context_->getPhiM();
    std::vector<uint64_t> dense((size_t)context_->numPrimes() * N);
    int32_t idx[1] = {(int32_t)i};
    check(hb_poly_download(p_, idx, 1, dense.data()));
    return std::vector<long>(dense.begin() + (size_t)i * N, dense.begin() + (size_t)(i + 1) * N);
  }
};

// helib::Cmodulus (include/helib/CModulus.h:104-157): the transform of ONE chain prime -- the row-level view of the engine.
// FFT / iFFT run on the device through the same kernels as DoubleCRT (a one-row DoubleCRT per call); this is the surface the
// reference's own per-row seams use (src/CModulus.cpp:358-578), kept for callers that hold a Cmodulus (tests, PAlgebraMod).
class Cmodulus {
  const Context* context_ = nullptr;
  long idx_ = -1;
 public:
  Cmodulus() = default;
  Cmodulus(const Context& ctx, long primeIdx) : context_(&ctx), idx_(primeIdx) {
    if (primeIdx < 0 || primeIdx >= ctx.numPrimes()) throw InvalidArgument("Cmodulus: prime index out of range");
  }
  unsigned long getM() const { return (unsigned long)context_->getM(); }
  unsigned long getPhiM() const { return (unsigned long)context_->getPhiM(); }
  long getQ() const { return context_->ithPrime(idx_); }
  // the primitive m-th root the rows are evaluated at (Cmodulus::getRoot)
  long getRoot() const {
    std::vector<uint64_t> psi((size_t)context_->numPrimes());
    check(hb_ctx_get_psi(context_->handle(), psi.data()));
    return (long)psi[(size_t)idx_];
  }
  // y = FFT(x): x a polynomial with small signed coefficients (zzX), y[j] = x(psi^(rep(j)))   (src/CModulus.cpp:358-443)
  void FFT(std::vector<long>& y, const std::vector<long>& x) const {
    IndexSet s; s.insert(idx_);
    DoubleCRT d(x, *context_, s);
    y = d.getOneRow(idx_);
  }
  // x = FFT^-1(y): coefficients in [0, q)   (src/CModulus.cpp:486-577)
  void iFFT(std::vector<long>& x, const std::vector<long>& y) const {
    const long N = context_->getPhiM();
    if ((long)y.size() != N) throw InvalidArgument("iFFT: row length must be phi(m)");
    hb_poly* p = nullptr;
    check(hb_poly_create(context_->handle(), &p));
    std::vector<uint64_t> dense((size_t)context_->numPrimes() * N, 0);
    for (long k = 0; k < N; k++) dense[(size_t)idx_ * N + k] = (uint64_t)y[k];
    int32_t idx[1] = {(int32_t)idx_};
    int rc = hb_poly_upload(p, idx, 1, dense.data());
    if (rc == HB_OK) rc = hb_ntt_inv(&p, 1, idx, 1);
    if (rc == HB_OK) rc = hb_poly_download(p, idx, 1, dense.data());
    hb_poly_destroy(p);
    check(rc);
    x.assign(dense.begin() + (size_t)idx_ * N, dense.begin() + (size_t)(idx_ + 1) * N);
  }
};

}  // namespace hb
