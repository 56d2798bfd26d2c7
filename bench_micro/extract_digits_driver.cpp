// The timing driver of bench_extract_digits.py: one workload of hb::extractDigits or hb::extractDigitsThin, fused against
// the transcribed step-by-step chains (fused = false), alternated in one process on the same input.
//   extract_digits_driver digits m p bits c n runs
//   extract_digits_driver thin   m p bits c botHigh r ePrime runs
// Prints one JSON line.  Each run calls both forms, in alternating order, each on a fresh output as a user would:
//  - the whole call, timed by CUDA events on the context's stream (hb_ctx_mark_begin / hb_ctx_mark_end);
//  - the same call again with the mirror's timers on (every timed step synchronises before it stops), which splits it
//    into the powerings (digit_power, and Chen and Han's digit_lift) and the chains (digit_chain, thin_combine).
// A last, profiled call of the fused form counts k1_scaled_sums launches, their time and algorithmic bytes.
#include <cstdio>
#include <cstring>
#include <random>
#include <string>

#include "helib_b200_ctxt.hpp"

using namespace hb;

static long ipow(long p, long e) { long r = 1; while (e-- > 0) r *= p; return r; }
static DoubleCRT random_rows(const Context& ctx, const IndexSet& s, std::mt19937_64& g) {
  const long N = ctx.getPhiM();
  std::vector<uint64_t> dense((size_t)ctx.numPrimes() * N, 0);
  for (long i : s) for (long k = 0; k < N; k++) dense[(size_t)i * N + k] = g() % (uint64_t)ctx.ithPrime(i);
  return DoubleCRT::fromRows(ctx, s, dense);
}
static std::vector<long> small(std::mt19937_64& g, long n, long range) { std::vector<long> v(n); for (auto& x : v) x = (long)(g() % (uint64_t)(2 * range + 1)) - range; return v; }

struct Setup {   // relinearisation keys (s^2 and s^3) and a symmetric encryption of a constant at plaintext space p^r
  Context ctx;
  KeyInfo pk;
  DoubleCRT S;
  long P;
  std::mt19937_64 gen;
  Setup(long m, long p, long r, long bits, long c) : ctx(m, p, r, bits, c), S(ctx, ctx.getCtxtPrimes() | ctx.getSpecialPrimes()), P(ipow(p, r)), gen(20261019) {
    pk.context = &ctx; pk.ckks = false; pk.scale = 10.0; pk.hwt = 0;
    pk.skBound = pk.scale * std::sqrt(double(ctx.getPhiM()) * 2.0 / 3.0);
    const long N = ctx.getPhiM();
    const IndexSet allq = ctx.getCtxtPrimes() | ctx.getSpecialPrimes();
    S = DoubleCRT(small(gen, N, 1), ctx, allq);
    DoubleCRT se(S);
    for (long e : {2L, 3L}) {
      se *= S;
      DoubleCRT s2(se);
      KeySwitch W; W.fromKey = SKHandle(e, 1, 0); W.toKeyID = 0; W.ptxtSpace = P;
      s2.multiplyByPrimes(ctx.getSpecialPrimes());
      for (size_t i = 0; i < ctx.getDigits().size(); i++) {
        W.a.push_back(random_rows(ctx, allq, gen));
        DoubleCRT b(small(gen, N, 8), ctx, allq); b *= P;
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
  Ctxt encrypt(long value) {
    const long N = ctx.getPhiM();
    Ctxt c(pk, P);
    c.primeSet = ctx.getCtxtPrimes();
    std::vector<long> pt = small(gen, N, 8);
    for (auto& x : pt) x *= P;
    pt[0] += value;
    DoubleCRT c1 = random_rows(ctx, c.primeSet, gen);
    DoubleCRT c0(pt, ctx, c.primeSet);
    DoubleCRT t(c1); t.Mul(S, false); c0 -= t;
    c.parts.emplace_back(c0, SKHandle());
    c.parts.emplace_back(c1, SKHandle(1, 1, 0));
    c.noiseBound = XD(double(P) * pk.noiseBoundForGaussian(3.2, N));
    return c;
  }
};

static bool same(const Ctxt& x, const Ctxt& y) {
  if (x.parts.size() != y.parts.size() || !(x.primeSet == y.primeSet) || x.ptxtSpace != y.ptxtSpace || x.intFactor != y.intFactor) return false;
  if (x.noiseBound.m != y.noiseBound.m || x.noiseBound.e != y.noiseBound.e || x.ptxtMag.m != y.ptxtMag.m || x.ptxtMag.e != y.ptxtMag.e) return false;
  for (size_t j = 0; j < x.parts.size(); j++)
    for (long i : x.primeSet) if (x.parts[j].dcrt.getOneRow(i) != y.parts[j].dcrt.getOneRow(i)) return false;
  return true;
}
static double timerSeconds(const char* name) { const FHEtimer* t = getTimerByName(name); return t ? t->getTime() : 0.0; }
static long timerCalls(const char* name) { const FHEtimer* t = getTimerByName(name); return t ? t->getNumCalls() : 0; }

static std::string list(const std::vector<double>& v) {
  std::string s = "[";
  for (size_t i = 0; i < v.size(); i++) { char b[32]; std::snprintf(b, sizeof b, "%s%.3f", i ? ", " : "", v[i]); s += b; }
  return s + "]";
}

int main(int argc, char** argv) {
  if (hb_device_count() <= 0) { std::printf("no CUDA device\n"); return 3; }
  const bool thin = argc > 1 && std::strcmp(argv[1], "thin") == 0;
  if (argc < (thin ? 10 : 8)) { std::fprintf(stderr, "usage: see the top of extract_digits_driver.cpp\n"); return 2; }
  const long m = std::atol(argv[2]), p = std::atol(argv[3]), bits = std::atol(argv[4]), c = std::atol(argv[5]);
  long n = 0, bot = 0, r = 0, ep = 0, runs = 0;
  if (thin) { bot = std::atol(argv[6]); r = std::atol(argv[7]); ep = std::atol(argv[8]); runs = std::atol(argv[9]); }
  else { n = std::atol(argv[6]); runs = std::atol(argv[7]); }
  try {
    Setup T(m, p, thin ? bot + r : n, bits, c);
    const Ctxt x = T.encrypt((long)(T.gen() % (uint64_t)T.P));
    // one call of form f (0 fused, 1 composed) on a fresh output; result[f] keeps the last one for the comparison
    std::vector<Ctxt> result[2];
    auto call = [&](int f) {
      std::vector<Ctxt> out;
      if (thin) { Ctxt t = x; extractDigitsThin(t, bot, r, ep, 0, f == 0); out.push_back(t); }
      else extractDigits(out, x, n, f == 0);
      result[f] = std::move(out);
    };
    std::vector<double> total[2], power[2], chains[2];
    for (int f = 0; f < 2; f++) call(f);   // warm-up: every shape once
    for (long i = 0; i < runs; i++)
      for (int k = 0; k < 2; k++) {
        const int f = (int)((i + k) % 2);   // fused first in even runs, composed first in odd ones
        check(hb_ctx_sync(T.ctx.handle()));
        check(hb_ctx_mark_begin(T.ctx.handle()));
        call(f);
        float ms = 0;
        check(hb_ctx_mark_end(T.ctx.handle(), &ms));
        total[f].push_back(ms);
        resetAllTimers();
        setTimersOn();
        call(f);
        setTimersOff();
        power[f].push_back(1e3 * (timerSeconds("digit_power") + timerSeconds("digit_lift")));
        chains[f].push_back(1e3 * (timerSeconds("digit_chain") + timerSeconds("thin_combine")));
      }
    bool identical = result[0].size() == result[1].size();
    for (size_t j = 0; identical && j < result[0].size(); j++) identical = same(result[0][j], result[1][j]);
    // profiled call of the fused form: k1_scaled_sums launches, time and algorithmic bytes, and the calls they come from
    resetAllTimers();
    check(hb_ctx_profile(T.ctx.handle(), 1));
    call(0);
    check(hb_ctx_sync(T.ctx.handle()));
    char name[64]; uint64_t launches = 0, bytes = 0, sl = 0, sb = 0; double ms = 0, sms = 0;
    for (int i = 0; hb_ctx_profile_get(T.ctx.handle(), i, name, sizeof name, &launches, &ms, &bytes) == 0; i++)
      if (std::strcmp(name, "k1_scaled_sums") == 0) { sl += launches; sms += ms; sb += bytes; }
    check(hb_ctx_profile(T.ctx.handle(), 0));
    std::printf("{\"primes\": %ld, \"fused_ms\": %s, \"composed_ms\": %s, \"fused_power_ms\": %s, \"composed_power_ms\": %s, "
                "\"fused_chain_ms\": %s, \"composed_chain_ms\": %s, \"chain_calls\": %ld, \"powerings\": %ld, "
                "\"sums_launches\": %lu, \"sums_ms\": %.4f, \"sums_bytes\": %lu, \"identical\": %s}\n",
                (long)T.ctx.getCtxtPrimes().card(), list(total[0]).c_str(), list(total[1]).c_str(), list(power[0]).c_str(),
                list(power[1]).c_str(), list(chains[0]).c_str(), list(chains[1]).c_str(),
                timerCalls("digit_chain") + timerCalls("thin_combine"), timerCalls("digit_power") + timerCalls("digit_lift"),
                (unsigned long)sl, sms, (unsigned long)sb, identical ? "true" : "false");
    return identical ? 0 : 1;
  } catch (const std::exception& e) {
    std::printf("{\"error\": \"%s\"}\n", e.what());
    return 1;
  }
}
