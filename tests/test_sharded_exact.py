"""The prime-sharded key switch against exact references, for every owner layout, both exchange forms and CKKS.

helib_b200/sharded.py splits a ciphertext's rows by RNS prime over R ranks and moves only y rows between them
(hb_conv_make_y / hb_conv_make_y_bcast, then hb_conv_from_y into the rows each rank owns).  Its layouts are what break
sharded code: a rank that owns no special prime, no prime of some digit or no row of S at all, a digit with no live prime,
a batch that the engine splits into chunks while peer buffers are indexed by item.  Here R ranks run as R threads of one
process, driving the real ShardedKeySwitch through an in-process stand-in for torch.distributed (the collectives copy
tensors between the ranks' buffers; on the GPU they are ordered with the kernels by the one stream every rank uses), and
the p2p form's peer stores land in the other ranks' y buffers directly.  Every row a rank does not own holds a poison
value in every input, key, scratch and output poly; it must still hold it afterwards (a stray write) and the owned rows
must equal the oracle's unsharded step-by-step key switch and mod-down bit for bit (a stray read).  The entry points
run on their own as well, against the oracle's step, and with bad arguments, which must come back before any launch.

Every body runs on the CPU simulator build and, marked gpu, on the H100; the full-size chains of BASELINE configs 3 and 4
only on the GPU.
"""
import gc
import threading
import zlib

import numpy as np
import pytest
import torch

import orc
import pyoracle as po
from helib_b200 import sharded
from helib_b200.engine import Engine, HbError
from helib_b200.sharded import ShardedKeySwitch
from test_norms import to_limbs
from test_value_ranges import largest_primes

R17 = 1 << 17
MAXROWS, MAXPEERS = 64, 8     # HB_MAXROWS, HB_MAXPEERS (hb_device.cuh)


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def backend(request):
    return request.param


@pytest.fixture
def lib(backend, request):
    return request.getfixturevalue("sim_lib" if backend == "sim" else "cuda_lib")


# ---- one lock around the library, a stand-in for torch.distributed

class LockedLib:
    """The loaded library with every hb_* call under one lock: the simulator keeps global fiber state and ctypes releases
    the GIL, so two ranks must never be inside the library at once.  Re-entrant, because a Poly's finaliser may run
    (and call hb_poly_destroy) while its thread holds the lock."""

    def __init__(self, lib, lock):
        self._lib, self._lock = lib, lock

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if not name.startswith("hb_"):
            return f

        def call(*args):
            with self._lock:
                return f(*args)
        return call


class Group:
    def __init__(self, ranks, timeout):
        self.ranks = list(ranks)
        self.barrier = threading.Barrier(len(self.ranks), timeout=timeout)
        self.slots = [None] * len(self.ranks)


class FakeDist:
    """get_rank, get_world_size, all_gather_into_tensor, all_gather_object, all_reduce and barrier over threads.  Each
    collective publishes the caller's object, waits for the group, combines, and waits again before a slot is reused, so
    a rank's send buffer is never overwritten while another rank still reads it.  A rank that raises aborts every barrier,
    and the others fail with BrokenBarrierError instead of waiting forever."""

    def __init__(self, world, timeout=900):
        self.timeout = timeout
        self.world = Group(range(world), timeout)
        self.groups = [self.world]
        self.local = threading.local()

    def new_group(self, ranks):
        g = Group(ranks, self.timeout)
        self.groups.append(g)
        return g

    def abort(self):
        for g in self.groups:
            g.barrier.abort()

    def _g(self, group):
        return self.world if group is None else group

    def get_rank(self, group=None):
        return self._g(group).ranks.index(self.local.rank)

    def get_world_size(self, group=None):
        return len(self._g(group).ranks)

    def _collective(self, group, obj, combine):
        g = self._g(group)
        g.slots[g.ranks.index(self.local.rank)] = obj
        g.barrier.wait()
        out = combine(list(g.slots))
        g.barrier.wait()
        return out

    def all_gather_into_tensor(self, out, inp, group=None):
        self._collective(group, inp, lambda vals: out.copy_(torch.cat([v.reshape(-1) for v in vals])))

    def all_gather_object(self, out, obj, group=None):
        out[:] = self._collective(group, obj, lambda vals: vals)

    def all_reduce(self, t, group=None):
        s = self._collective(group, t, lambda vals: sum(v.clone() for v in vals))
        t.copy_(s)

    def barrier(self, group=None):
        self._g(group).barrier.wait()


def run_ranks(fd, R, body):
    """body(r) on R threads, rank r on thread r; re-raises the first real failure."""
    errs = [None] * R

    def run(r):
        fd.local.rank = r
        try:
            body(r)
        except BaseException as e:    # noqa: B902 -- any failure must reach the test, and release the other ranks
            errs[r] = e
            fd.abort()
    th = [threading.Thread(target=run, args=(r,)) for r in range(R)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    real = [e for e in errs if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if real:
        raise real[0]
    if any(e is not None for e in errs):
        raise next(e for e in errs if e is not None)


# ---- chains, engines, poison

def chain_of(m, p, primes, digit_sizes, nspecial):
    digits, i = [], 0
    for n in digit_sizes:
        digits.append(list(range(i, i + n)))
        i += n
    return po.Chain(m=m, p=p, r=1, phim=po.euler_phi(m), primes=list(primes), ctxt=list(range(i)),
                    special=list(range(i, i + nspecial)), digits=digits)


def top_primes_chain(m, p, form, digit_sizes, nspecial):
    """The largest primes below 2^60 (test_value_ranges), in the shift form ('sp') or the generic one ('gen')."""
    return chain_of(m, p, largest_primes(form, sum(digit_sizes) + nspecial, m), digit_sizes, nspecial)


def config_chain(name):
    """BASELINE config 3 (BGV, p = 257) and config 4 (CKKS) at N = 2^16."""
    return {"cfg3": lambda: po.build_mod_chain(R17, 257, 1, 1500, 3),
            "cfg4": lambda: po.build_mod_chain(R17, -1, 1, 1700, 2)}[name]()


def oracle(ch):
    return orc.Oracle(ch.phim, ch.m, ch.primes, [po.find_psi(q, ch.m) for q in ch.primes], ch.digits, ch.special, nthreads=8)


@pytest.fixture
def cluster(lib, backend):
    """cluster(ch, R, shared) -> (lock, engines): one engine per rank (or one shared engine), all through one locked
    library; closed when the test ends, pass or fail, after the test's Polys."""
    gc.collect()     # engines of earlier tests that are only held by reference cycles: their device memory first
    made = []

    def make(ch, R, shared=False):
        lock = threading.RLock()
        L = LockedLib(lib, lock)
        psis = [po.find_psi(q, ch.m) for q in ch.primes]
        engines = [Engine(ch.m, ch.primes, psis, ch.digits, ch.special, lib=L) for _ in range(1 if shared else R)]
        if backend == "cuda":
            for E in engines:
                E.set_stream(torch.cuda.current_stream().cuda_stream)
        made.extend(engines)
        return lock, engines
    yield make
    gc.collect()
    for E in made:
        E.close()


def poison_rows(ch):
    """The value every row a rank does not own holds: q_i - 2 (distinct from the q_i - 1 of the worst-case words)."""
    return np.array([[q - 2] * ch.phim for q in ch.primes], dtype=np.uint64)


def poisoned(ch, x, owned):
    out = poison_rows(ch)
    if x is not None:
        out[owned] = x[owned]
    return out


def device_of(backend):
    return "cpu" if backend == "sim" else "cuda"


def kernels(engines):
    out = set()
    for E in engines:
        out |= {r["kernel"] for r in E.profile_results()}
    return out


def fallbacks(engines):
    return sum(E.stats()["exact_fallbacks"] for E in engines)


def sync(engines, backend):
    if backend == "cuda":
        torch.cuda.synchronize()


# ---- the in-process R-rank run of ShardedKeySwitch

def install_ybuf(KS, fd, ch):
    """Every y buffer starts poisoned.  gather: the class's own torch-owned buffer; p2p: the same kind of buffer, with the
    peers as plain polys over the other ranks' buffers instead of CUDA-IPC mappings (hb_conv_make_y_bcast only stores
    through the pointers it is given; IPC export and open stay with the multi-process tests)."""
    orig = KS._ybuf
    pz = torch.from_numpy(poison_rows(ch).view(np.int64)).to(KS.device)

    def ybuf(key):
        if key in KS._bufs:
            return KS._bufs[key]
        if not KS.p2p:
            t, y, _ = orig(key)
            t.copy_(pz)
            return KS._bufs[key]
        t = pz.clone()
        mine = KS.E.wrap(t.data_ptr())
        every = [None] * KS.world
        fd.all_gather_object(every, t, group=KS.group)
        KS._bufs[key] = (t, mine, [KS.E.wrap(o.data_ptr()) for r, o in enumerate(every) if r != KS.rank])
        return KS._bufs[key]
    KS._ybuf = ybuf


def sharded_run(monkeypatch, cluster, backend, ch, R, items, sets, ptxt, p2p, evk, group_size=0, shared=False,
                mod_down_only=False):
    """items[it] = (c0, c1, c2) dense arrays over S (for mod_down_only: (c0, c1) over S | special); sets: the index sets S.
    Runs relinearize + mod_down (or mod_down alone) on R ranks per S and checks every rank's owned rows against the
    oracle and its non-owned rows against the poison.  Returns (engines, kernels that ran, exact fallbacks)."""
    lock, engines = cluster(ch, R, shared)
    fd = FakeDist(R)
    monkeypatch.setattr(sharded, "dist", fd)
    groups = [fd.new_group(range(i, i + group_size)) for i in range(0, R, group_size)] if group_size else None
    O = oracle(ch)
    full = ch.ctxt + ch.special
    allrows = list(range(len(ch.primes)))
    nd_all = len(ch.digits)
    evk_a, evk_b = evk
    for E in engines:
        E.profile(False)
        E.profile(True)
        E.reset_stats()
    dev = device_of(backend)
    for S in sets:
        Sp = sorted(set(S) | set(ch.special))
        out = [None] * R

        def body(r):
            E = engines[0 if shared else r]
            group = groups[r // group_size] if groups else None
            KS = ShardedKeySwitch(E, ch.ctxt, ch.special, ch.digits, device=dev, p2p=p2p, group=group)
            install_ybuf(KS, fd, ch)
            own_full = KS.owned(full)
            EA = [E.poly(poisoned(ch, evk_a[i], own_full), allrows) for i in range(nd_all)]
            EB = [E.poly(poisoned(ch, evk_b[i], own_full), allrows) for i in range(nd_all)]
            if mod_down_only:
                oSp = KS.owned(Sp)
                C = [[E.poly(poisoned(ch, x[k], oSp), allrows) for x in items] for k in range(2)]
                KS.mod_down(C[0] + C[1], Sp, S, ptxt)
                DIG, C2 = [], []
            else:
                oS = KS.owned(S)
                C = [[E.poly(poisoned(ch, x[k], oS), allrows) for x in items] for k in range(3)]
                DIG = [[E.poly(poison_rows(ch), allrows) for _ in range(nd_all)] for _ in items]
                got = KS.relinearize(C[0], C[1], C[2], S, EA, EB, dig_polys=DIG)
                assert got == Sp
                KS.mod_down(C[0] + C[1], Sp, S, ptxt)
                C2 = C[2]
            out[r] = (KS, C[0], C[1], C2, DIG, EA, EB)
        run_ranks(fd, R, body)
        sync(engines, backend)
        # references: the oracle's unsharded step-by-step key switch and mod-down
        refs = []
        for x in items:
            if mod_down_only:
                r0, r1 = x[0].copy(), x[1].copy()
            else:
                r0, r1 = O.relinearize(x[0], x[1], x[2], S, evk_a, evk_b)
            O.scale_down(r0, Sp, S, ptxt)
            O.scale_down(r1, Sp, S, ptxt)
            refs.append((r0, r1))
        pz = poison_rows(ch)
        covered = set()
        for r in range(R):
            KS, C0, C1, C2, DIG, EA, EB = out[r]
            own = set(KS.owned(full))
            oS = KS.owned(S)
            covered |= set(oS) if not groups else set()
            other = [i for i in allrows if i not in own]
            for it, (r0, r1) in enumerate(refs):
                g0, g1 = C0[it].download(allrows), C1[it].download(allrows)
                assert (g0[oS] == r0[oS]).all() and (g1[oS] == r1[oS]).all(), ("rank", r, "item", it, "S", len(S))
                for what, g in (("c0", g0), ("c1", g1)):
                    assert (g[other] == pz[other]).all(), ("stray write", what, "rank", r, "item", it)
            for it in range(len(C2)):
                for what, P in [("c2", C2[it])] + [(f"digit {d}", D) for d, D in enumerate(DIG[it])]:
                    g = P.download(allrows)
                    assert (g[other] == pz[other]).all(), ("stray write", what, "rank", r, "item", it)
            # y buffers: the digit exchanges read rows of S only, the mod-down's the special rows only
            for key, buf in KS._bufs.items():
                if key[0] in ("dig", "md"):
                    src = S if key[0] == "dig" else [i for i in Sp if i not in S]
                    g = buf[0].cpu().numpy().view(np.uint64)
                    rest = [i for i in allrows if i not in src]
                    assert (g[rest] == pz[rest]).all(), ("stray write into a y buffer", key, "rank", r)
            for i in range(nd_all):
                for what, P, ref in (("evk_a", EA[i], evk_a[i]), ("evk_b", EB[i], evk_b[i])):
                    assert (P.download(allrows) == poisoned(ch, ref, sorted(own & set(full)))).all(), ("key written", what, r)
        if not groups:
            assert covered == set(S)
        if backend == "cuda" and not mod_down_only:
            # the unsharded engine path on the same data
            E = engines[0]
            EA = [E.poly(evk_a[i], full) for i in range(nd_all)]
            EB = [E.poly(evk_b[i], full) for i in range(nd_all)]
            C = [[E.poly(x[k], S) for x in items] for k in range(3)]
            E.relinearize(C[0], C[1], C[2], S, EA, EB)
            E.scale_down(C[0] + C[1], Sp, S, ptxt)
            for it, (r0, r1) in enumerate(refs):
                assert (C[0][it].download(S)[S] == r0[S]).all() and (C[1][it].download(S)[S] == r1[S]).all(), it
    ran = kernels(engines)
    fb = fallbacks(engines)
    for E in engines:
        E.profile(False)
    return engines, ran, fb


def random_items(O, rng, S, nit, parts=3):
    return [tuple(O.random(rng, S) for _ in range(parts)) for _ in range(nit)]


def random_keys(O, rng, ch):
    full = ch.ctxt + ch.special
    nd = len(ch.digits)
    return np.stack([O.random(rng, full) for _ in range(nd)]), np.stack([O.random(rng, full) for _ in range(nd)])


def hole(ch, d=1):
    return [i for i in ch.ctxt if i not in ch.digits[d]]


def expect_kernels(ran, N, p2p, R, fused_conv=True):
    """The forms the case must have run: the register kernels at N = 2^16 (k1_inv_cols with the folded factor, k1_conv
    from y rows), the generic ones below."""
    if N == 1 << 16:
        assert ("k1_inv_cols_bcast" if p2p and R > 1 else "k1_inv_cols") in ran, ran
        assert "k1_conv" in ran and "k_conv" not in ran and "k_scale_bcast" not in ran, ran
    else:
        assert "k_conv" in ran and "k1_conv" not in ran, ran
        if p2p and R > 1:
            assert "k_scale_bcast" in ran and "k1_inv_cols_bcast" not in ran, ran
        else:
            assert "k_pw_scale" in ran and "k_scale_bcast" not in ran, ran


# ---- 1. owner layouts, exchange forms, plaintext spaces and batches on the small rings

# (m, form, digit sizes, special primes, R, ptxt_space, group size, items)
SMALL = {
    # m = 64: five ctxt primes over four digits, two special primes.  R = 3..5 exceed the special primes and the
    # one-prime digits; R = 5 = #ctxt leaves rank 4 with no row of S once the last prime is dropped
    "64-R1-bgv": (64, "gen", [1, 2, 1, 1], 2, 1, 257, 0, 2),
    "64-R2-p2": (64, "sp", [1, 2, 1, 1], 2, 2, 2, 0, 2),
    "64-R3-ckks": (64, "gen", [1, 2, 1, 1], 2, 3, 1, 0, 2),
    "64-R4-p289": (64, "sp", [1, 2, 1, 1], 2, 4, 289, 0, 2),
    "64-R5-bgv": (64, "gen", [1, 2, 1, 1], 2, 5, 257, 0, 2),
    # four digits (the fused limit) and five (the step-by-step branch of relinearize)
    "4096-R3-fused4-p2": (4096, "gen", [1, 1, 1, 1], 2, 3, 2, 0, 2),
    "4096-R2-unfused5-ckks": (4096, "sp", [1, 1, 1, 1, 1], 2, 2, 1, 0, 1),
    # two groups of two ranks inside R = 4 (bench.py's p2p_groups_of_2)
    "8192-R4-groups2-p289": (8192, "sp", [2, 1, 2], 3, 4, 289, 2, 2),
    # batches past the 64-item chunk: the peer buffers are indexed by item across chunks
    "64-R3-65items": (64, "gen", [1, 1, 1], 2, 3, 257, 0, 65),
    "64-R4-130items-ckks": (64, "sp", [1, 1, 1], 2, 4, 1, 0, 130),
}


@pytest.mark.parametrize("case,mode", [(c, md) for c in SMALL for md in ("gather", "p2p") if md == "gather" or SMALL[c][4] > 1])
def test_sharded_key_switch_owner_layouts(monkeypatch, cluster, backend, case, mode):
    """relinearize + mod_down on R ranks over the full ctxt set, the set without its last prime and (with three or more
    digits) a hole, against the oracle on every owned row; poison intact on every other row.  (One rank has no peers, so
    R = 1 runs the gather form only.)"""
    m, form, sizes, nsp, R, ptxt, gsz, nit = SMALL[case]
    p2p = mode == "p2p"
    ch = top_primes_chain(m, 257 if ptxt > 1 else -1, form, sizes, nsp)
    O = oracle(ch)
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    sets = [ch.ctxt, ch.ctxt[:-1]] + ([hole(ch)] if len(ch.digits) >= 3 and nit <= 2 else [])
    evk = random_keys(O, rng, ch)
    for S in sets:
        items = random_items(O, rng, S, nit)
        _, ran, _ = sharded_run(monkeypatch, cluster, backend, ch, R, items, [S], ptxt, p2p, evk, group_size=gsz)
        expect_kernels(ran, ch.phim, p2p, gsz or R)
    if case == "64-R5-bgv":
        own = sharded.owner_map(ch.ctxt, ch.special, R)
        assert not [i for i in ch.ctxt[:-1] if own[i] == R - 1]       # the layout this case is for


def test_sim_register_kernels_on_a_short_chain(monkeypatch, cluster, backend):
    """N = 2^16 on a short chain: k1_inv_cols with the per-row factor folded in and its peer stores, k1_conv from y rows,
    with the items split into chunks of two (HB_CHUNK) so the chunked peer indexing runs without 65 items.  Three ctxt
    primes in two digits: each of three ranks owns one, so every peer slot a producer stores to is read by its rank."""
    monkeypatch.setenv("HB_CHUNK", "2")
    ch = top_primes_chain(R17, 257, "sp", [1, 2], 1)
    O = oracle(ch)
    rng = np.random.default_rng(17)
    evk = random_keys(O, rng, ch)
    for mode, R, ptxt in (("p2p", 3, 2), ("gather", 2, 1)):
        items = random_items(O, rng, ch.ctxt, 3)
        _, ran, _ = sharded_run(monkeypatch, cluster, backend, ch, R, items, [ch.ctxt], ptxt, mode == "p2p", evk)
        expect_kernels(ran, ch.phim, mode == "p2p", R)


@pytest.mark.parametrize("world,cfg,port", [(2, "4096,-1,1,160,3", 29619), (5, "64,257,1,200,3", 29620)])
def test_sharded_keyswitch_processes_ckks_and_five_ranks(sim_lib, world, cfg, port):
    """The class over real torch.distributed (gloo, one process per rank; tests/mp/sharded_worker.py): a CKKS chain
    (plaintext space 1 in the mod-down) and five ranks."""
    from test_sharded import run
    run("sim", world, cfg, port)


# ---- 2. worst-case words at the largest primes below 2^60

def planted_digits(ch, S, N):
    """Coefficients whose balanced mixed-radix digits over the digits of S are chosen: each digit cycles through 0, +-1,
    +-(Q_d-1)/2 and the 4n-ulp band next to both ends (n = the digit's live primes), with its own period so that the
    digits combine differently at each coefficient."""
    parts = [[i for i in d if i in S] for d in ch.digits]
    parts = [p for p in parts if p]
    out = [0] * N
    Qp = 1
    for d, part in enumerate(parts):
        Qd = ch.product(part)
        A = (Qd - 1) // 2
        n = len(part)
        pat = [0, 1, -1, A, -A] + [-A + j for j in range(4 * n + 1)] + [A - j for j in range(4 * n + 1)]
        for k in range(N):
            out[k] += pat[(k * (d + 1) + d) % len(pat)] * Qp
        Qp *= Qd
    return out


def rows_of(O, ch, coeffs, idx):
    x = np.zeros((len(ch.primes), ch.phim), dtype=np.uint64)
    O.fft_bigpoly(to_limbs(coeffs), idx, x)
    return x


def all_minus_one(ch, S):
    c, Qp = 0, 1
    for d in ch.digits:
        part = [i for i in d if i in S]
        if part:
            c -= Qp
            Qp *= ch.product(part)
    return c


def const(ch, idx, v):
    x = np.zeros((len(ch.primes), ch.phim), dtype=np.uint64)
    for i in idx:
        x[i] = v % ch.primes[i]
    return x


@pytest.mark.parametrize("mode", ["gather", "p2p"])
@pytest.mark.parametrize("ring", ["4096-sp", "4096-gen", "r17-sp", "r17-gen"])
def test_sharded_worst_case_words(monkeypatch, cluster, backend, ring, mode):
    """Digits of two primes at the largest primes below 2^60: c2 with planted digits (+-(Q_d-1)/2 and the band beside it,
    so the y-row conversions reach the exact fallback of k_conv / k1_conv) and c2 whose balanced digits are all -1, with
    c0, c1 and the keys at q-1; CKKS and p = 2."""
    m, form = ring.split("-")
    m = 4096 if m == "4096" else R17
    sizes = [2, 2] if m == R17 else [2, 2, 2]
    ch = top_primes_chain(m, 2, form, sizes, 2)
    O = oracle(ch)
    full = ch.ctxt + ch.special
    top = const(ch, full, -1)
    evk = (np.stack([top] * len(ch.digits)), np.stack([top] * len(ch.digits)))
    R = 3
    for S, ptxt in ((ch.ctxt, 1), (ch.ctxt[:-1], 2)):
        planted = rows_of(O, ch, planted_digits(ch, S, ch.phim), S)
        items = [(const(ch, S, -1), const(ch, S, -1), planted),
                 (const(ch, S, -1), planted, const(ch, S, all_minus_one(ch, S)))]
        engines, ran, fb = sharded_run(monkeypatch, cluster, backend, ch, R, items, [S], ptxt, mode == "p2p", evk)
        expect_kernels(ran, ch.phim, mode == "p2p", R)
        assert fb > 0, "the planted digits never reached the exact fallback"


def delta_plants(P, p, N):
    """Special-prime coefficients d (the delta of the mod-down is d + P*u): 0, +-1, +-(P-1)/2 and the band next to
    both ends, and for p > 1 values near both ends whose u = d*P^-1 mod p sits on either side of p/2 (for even p the tie
    u = p/2, decided by the sign of d)."""
    A = (P - 1) // 2
    vals = [0, 1, -1, 2, -2, A, -A] + [-A + j for j in range(9)] + [A - j for j in range(9)]
    if p > 1:
        for u in {p // 2, p // 2 + 1 if p > 2 else 1}:
            for base, step in ((-A, 1), (A, -1), (-1, -1), (1, 1)):
                d = base
                while (d * pow(P % p, -1, p) - u) % p:
                    d += step
                vals.append(d)
    return [vals[k % len(vals)] for k in range(N)]


@pytest.mark.parametrize("p", [1, 2, 257, 289])
@pytest.mark.parametrize("ring", ["4096-gen", "r17-sp"])
def test_sharded_mod_down_at_the_delta_boundaries(monkeypatch, cluster, backend, ring, p):
    """mod_down alone, the special-prime rows planted with deltas at the rounding boundary and at the tie of p = 2, the
    ctxt rows random; p2p on three ranks (two special primes: one rank owns none)."""
    m, form = ring.split("-")
    m = 4096 if m == "4096" else R17
    ch = top_primes_chain(m, p if p != 289 else 17, form, [1, 1] if m == R17 else [1, 1, 1], 2)
    O = oracle(ch)
    rng = np.random.default_rng(p)
    S = ch.ctxt
    Sp = sorted(S + ch.special)
    Pd = ch.product(ch.special)
    items = []
    for it in range(2):
        x = O.random(rng, S)
        sp = rows_of(O, ch, delta_plants(Pd, p, ch.phim)[it:] + delta_plants(Pd, p, ch.phim)[:it], ch.special)
        x[ch.special] = sp[ch.special]
        y = O.random(rng, Sp)
        items.append((x, y))
    evk = random_keys(O, rng, ch)
    engines, ran, fb = sharded_run(monkeypatch, cluster, backend, ch, 3, items, [S], p, True, evk, mod_down_only=True)
    assert fb > 0
    assert ("k1_conv" if ch.phim == 1 << 16 else "k_conv") in ran, ran


# ---- 3. full-size chains on the GPU

@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["cuda"])
@pytest.mark.parametrize("R,nit,mode", [(R, 2, md) for R in (2, 4, 8) for md in ("gather", "p2p")] + [(4, 3, "p2p")])
def test_config4_chain_sharded(monkeypatch, cluster, backend, R, nit, mode):
    """BASELINE config 4 (CKKS, 29 + 15 primes, 2 digits) over 2, 4 and 8 ranks of one shared engine, and three items in
    chunks of two (HB_CHUNK) on four ranks with the peer stores: the chunked peer indexing at full size, without the
    ~15 GB that 65 full-size items take (65 and 130 items run on the small rings)."""
    if nit == 3:
        monkeypatch.setenv("HB_CHUNK", "2")
    ch = config_chain("cfg4")
    O = oracle(ch)
    rng = np.random.default_rng(R)
    evk = random_keys(O, rng, ch)
    sets = [ch.ctxt, ch.ctxt[:-1]] if nit <= 2 else [ch.ctxt]
    for S in sets:
        items = random_items(O, rng, S, nit)
        _, ran, _ = sharded_run(monkeypatch, cluster, backend, ch, R, items, [S], 1, mode == "p2p", evk, shared=True)
        expect_kernels(ran, ch.phim, mode == "p2p", R)


@pytest.mark.gpu
@pytest.mark.parametrize("backend", ["cuda"])
@pytest.mark.parametrize("mode", ["gather", "p2p"])
def test_config3_chain_sharded_with_a_hole(monkeypatch, cluster, backend, mode):
    """BASELINE config 3's BGV chain (p = 257, 3 digits) on 4 ranks: the full set, the last prime dropped and a hole."""
    ch = config_chain("cfg3")
    O = oracle(ch)
    rng = np.random.default_rng(3)
    evk = random_keys(O, rng, ch)
    for S in (ch.ctxt, ch.ctxt[:-1], hole(ch)):
        items = random_items(O, rng, S, 2)
        _, ran, _ = sharded_run(monkeypatch, cluster, backend, ch, 4, items, [S], 257, mode == "p2p", evk, shared=True)
        expect_kernels(ran, ch.phim, mode == "p2p", 4)


# ---- 4. the entry points on their own

@pytest.fixture
def one(lib, backend):
    """one(ch) -> engine; closed at the end of the test."""
    gc.collect()
    made = []

    def make(ch):
        psis = [po.find_psi(q, ch.m) for q in ch.primes] if ch.m & (ch.m - 1) == 0 else None
        E = Engine(ch.m, ch.primes, psis, ch.digits, ch.special, lib=lib)
        made.append(E)
        return E
    yield make
    gc.collect()
    for E in made:
        E.close()


def y_rows(O, ch, x, D):
    """y_j = iNTT(row_j) * (Q_D/q_j)^-1 mod q_j for j in D."""
    y = x.copy()
    O.ntt_inv_rows(y, D)
    for j in D:
        q = ch.primes[j]
        s = pow(ch.product([i for i in D if i != j]) % q, -1, q)
        O.scale_by_word(y, [j], s)
    return y


ENTRY_RINGS = {"64": (64, "gen"), "8192": (8192, "sp"), "r17": (R17, "sp")}


@pytest.mark.parametrize("ring", list(ENTRY_RINGS))
def test_conv_make_y_for_any_owned_subset(one, ring):
    m, form = ENTRY_RINGS[ring]
    ch = top_primes_chain(m, 257, form, [3, 1], 2)
    O, E = oracle(ch), one(ch)
    allrows = list(range(len(ch.primes)))
    rng = np.random.default_rng(5)
    D = [0, 1, 2, 4]
    pz = poison_rows(ch)
    for owned in ([], [1], [0, 4], D):
        x = [O.random(rng, allrows) for _ in range(2)]
        ref = [y_rows(O, ch, xi, D) for xi in x]
        Y = [E.poly(pz, allrows) for _ in x]
        E.profile(False); E.profile(True)
        E.conv_make_y([E.poly(xi, allrows) for xi in x], D, owned, Y)
        ran = {r["kernel"] for r in E.profile_results()}
        if not owned:
            assert not ran, ran
        elif ch.phim == 1 << 16:
            assert "k1_inv_cols" in ran and "k_pw_scale" not in ran, ran
        else:
            assert "k_pw_scale" in ran, ran
        other = [i for i in allrows if i not in owned]
        for it in range(2):
            g = Y[it].download(allrows)
            assert (g[owned] == ref[it][owned]).all(), (owned, it)
            assert (g[other] == pz[other]).all(), ("stray write", owned, it)


@pytest.mark.parametrize("npeers", [0, 1, 3, 8])
@pytest.mark.parametrize("ring", list(ENTRY_RINGS))
def test_conv_make_y_bcast_stores_exactly_the_owned_rows(one, ring, npeers):
    m, form = ENTRY_RINGS[ring]
    ch = top_primes_chain(m, 257, form, [3, 1], 2)
    O, E = oracle(ch), one(ch)
    allrows = list(range(len(ch.primes)))
    rng = np.random.default_rng(npeers)
    D = [0, 1, 2, 4]
    pz = poison_rows(ch)
    for owned in ([2], [0, 1, 4]):
        x = [O.random(rng, allrows) for _ in range(2)]
        ref = [y_rows(O, ch, xi, D) for xi in x]
        Y = [E.poly(pz, allrows) for _ in x]
        PE = [[E.poly(pz, allrows) for _ in x] for _ in range(npeers)]
        E.profile(False); E.profile(True)
        E.conv_make_y_bcast([E.poly(xi, allrows) for xi in x], D, owned, Y, PE)
        ran = {r["kernel"] for r in E.profile_results()}
        assert ("k1_inv_cols_bcast" if npeers else "k1_inv_cols") in ran if ch.phim == 1 << 16 else "k_scale_bcast" in ran, ran
        other = [i for i in allrows if i not in owned]
        for it in range(2):
            for who, P in [("local", Y[it])] + [(f"peer {p}", PE[p][it]) for p in range(npeers)]:
                g = P.download(allrows)
                assert (g[owned] == ref[it][owned]).all(), (who, owned, it)
                assert (g[other] == pz[other]).all(), ("stray write", who, owned, it)


@pytest.mark.parametrize("ptxt", [1, 2, 257])
@pytest.mark.parametrize("ring", list(ENTRY_RINGS))
def test_conv_from_y_into_a_strict_subset_of_targets(one, ring, ptxt):
    """Mode 0 (addPrimes) and mode 1 (scaleDownToSet's (dst - x)/Q_D) from y rows of D into targets that are a strict subset
    of the complement of D; the other rows keep their poison."""
    m, form = ENTRY_RINGS[ring]
    ch = top_primes_chain(m, 257, form, [3, 1], 2)
    O, E = oracle(ch), one(ch)
    allrows = list(range(len(ch.primes)))
    rng = np.random.default_rng(ptxt)
    D = [1, 4]
    tgt = [0, 3, 5]
    pz = poison_rows(ch)
    x = [O.random(rng, allrows) for _ in range(2)]
    Yd = [y_rows(O, ch, xi, D) for xi in x]
    other = [i for i in allrows if i not in tgt]
    for mode in (0, 1):
        if mode == 0 and ptxt != 1:
            continue
        dst = [E.poly(poisoned(ch, xi, tgt), allrows) for xi in x]
        E.profile(False); E.profile(True)
        E.conv_from_y([E.poly(poisoned(ch, y, D), allrows) for y in Yd], D, tgt, ptxt, dst, mode)
        ran = {r["kernel"] for r in E.profile_results()}
        assert ("k1_conv" if ch.phim == 1 << 16 else "k_conv") in ran, ran
        for it in range(2):
            ref = x[it].copy()
            if mode == 0:
                O.add_primes(ref, D, tgt)
            else:
                O.scale_down(ref, sorted(D + tgt), tgt, ptxt)
            g = dst[it].download(allrows)
            assert (g[tgt] == ref[tgt]).all(), (mode, it)
            assert (g[other] == pz[other]).all(), ("stray write", mode, it)


def test_sub_div_by_primes_by_full_digit_products(one, backend):
    """dst = (dst - src) / prod(digit) on the rows of a later digit, with the divisor the full product of an earlier digit,
    also of one that has no live prime (the hole of relinearize)."""
    ch = top_primes_chain(64, 257, "gen", [2, 2, 2], 2)
    O, E = oracle(ch), one(ch)
    allrows = list(range(len(ch.primes)))
    rng = np.random.default_rng(11)
    pz = poison_rows(ch)
    for rows, fac in (([2, 3], ch.digits[0]), ([4], ch.digits[1]), ([4, 5, 6], ch.digits[0] + ch.digits[1])):
        a, b = O.random(rng, allrows), O.random(rng, allrows)
        dst = E.poly(poisoned(ch, a, rows), allrows)
        E.sub_div_by_primes([dst], [E.poly(b, allrows)], rows, fac)
        ref = a.copy()
        O.pointwise("sub", ref, b, rows)
        O.scale_by_primes(ref, rows, fac, inv=True)
        other = [i for i in allrows if i not in rows]
        g = dst.download(allrows)
        assert (g[rows] == ref[rows]).all(), (rows, fac)
        assert (g[other] == pz[other]).all()


# ---- 5. argument errors: refused before anything is launched

def refused(E, fn):
    E.profile(False)
    E.profile(True)
    with pytest.raises(HbError):
        fn()
    ran = [r["kernel"] for r in E.profile_results()]
    E.profile(False)
    assert not ran, ran


@pytest.mark.parametrize("ring", ["64", "r17"])
def test_sharded_entry_points_refuse_bad_arguments(one, ring):
    m, form = ENTRY_RINGS[ring]
    ch = top_primes_chain(m, 257, form, [3, 1], 2)
    E = one(ch)
    X, Y = [E.poly(), E.poly()], [E.poly(), E.poly()]
    D = [0, 1, 2]
    peers = [[E.poly(), E.poly()] for _ in range(MAXPEERS + 1)]
    refused(E, lambda: E.conv_make_y(X, D, [1, 3], Y))                          # owned prime outside D
    refused(E, lambda: E.conv_make_y_bcast(X, D, [4], Y, peers[:1]))            # the same, with a peer
    refused(E, lambda: E.conv_make_y_bcast(X, D, [1], Y, peers))                # more than HB_MAXPEERS peers
    refused(E, lambda: E.conv_from_y(Y, D, [2, 3], 1, X, 0))                    # D and the targets overlap
    refused(E, lambda: E.conv_from_y(Y, D, [3], 0, X, 1))                       # ptxt_space 0
    refused(E, lambda: E.conv_from_y(Y, D, [3], 257, X, 2))                     # no mode 2
    refused(E, lambda: E.conv_from_y(Y, D, [3], 257, X, -1))
    # a null peer handle
    import ctypes as C
    from helib_b200.engine import _arr, _idx
    a, pd, nd = _idx(D)
    b, po_, no = _idx([1])
    flat = (C.c_void_p * 2)(peers[0][0].h, None)
    refused(E, lambda: E._ck(E.lib.hb_conv_make_y_bcast(_arr(X), 2, pd, nd, po_, no, _arr(Y), flat, 1)))


def test_bcast_refuses_more_than_maxrows_owned_rows(one):
    ch = chain_of(64, 257, largest_primes("gen", MAXROWS + 3, 64), [MAXROWS + 1], 2)
    E = one(ch)
    X, Y = [E.poly()], [E.poly()]
    D = ch.digits[0]
    refused(E, lambda: E.conv_make_y_bcast(X, D, D, Y, [[E.poly()]]))


def test_sharded_entry_points_refuse_a_general_m_context(one):
    ch = chain_of(105, 2, largest_primes("gen", 4, 105), [1, 1], 2)
    E = one(ch)
    X, Y = [E.poly()], [E.poly()]
    refused(E, lambda: E.conv_make_y(X, [0, 1], [0], Y))
    refused(E, lambda: E.conv_make_y_bcast(X, [0, 1], [0], Y, [[E.poly()]]))
    refused(E, lambda: E.conv_from_y(Y, [0, 1], [2], 1, X, 0))
