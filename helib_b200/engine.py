"""ctypes binding of the C ABI in include/helib_b200.h (plumbing for tests and bench)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
u64p = C.POINTER(C.c_uint64)
i32p = C.POINTER(C.c_int32)
vpp = C.POINTER(C.c_void_p)

OPS = {"add": 0, "sub": 1, "mul": 2, "neg": 3, "copy": 7}


class HbError(RuntimeError):
    """Raised for a negative return code of the C ABI; .code holds HB_ERR_*."""

    def __init__(self, code, msg):
        super().__init__(f"helib_b200 error {code}: {msg}")
        self.code = code


def library_path() -> str:
    return os.path.join(_HERE, "libhelib_b200.so")


def _declare(lib):
    lib.hb_last_error.restype = C.c_char_p
    lib.hb_poly_destroy.restype = None
    lib.hb_ctx_destroy.restype = None
    lib.hb_poly_destroy.argtypes = [C.c_void_p]
    lib.hb_ctx_destroy.argtypes = [C.c_void_p]
    return lib


_LIB = None


def load_library(path: str | None = None):
    """Load the CUDA engine.  Fails loudly if the library has not been built."""
    global _LIB
    if path is not None:
        return _declare(C.CDLL(path))
    if _LIB is None:
        p = library_path()
        if not os.path.exists(p):
            raise HbError(-3, f"{p} not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                              "the engine has no CPU fallback")
        _LIB = _declare(C.CDLL(p))
    return _LIB


def _euler_phi(m):
    r, n, p = m, m, 2
    while p * p <= n:
        if n % p == 0:
            while n % p == 0:
                n //= p
            r -= r // p
        p += 1
    if n > 1:
        r -= r // n
    return r


def _idx(idx):
    a = np.ascontiguousarray(np.asarray(list(idx), dtype=np.int32))
    return a, a.ctypes.data_as(i32p), len(a)


class Poly:
    """A device DoubleCRT matrix [nprimes][N] (hb_poly)."""

    def __init__(self, eng):
        self.eng = eng
        h = C.c_void_p()
        eng._ck(eng.lib.hb_poly_create(eng.h, C.byref(h)))
        self.h = h

    def __del__(self):
        try:
            if self.h and self.eng.h:
                self.eng.lib.hb_poly_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def upload(self, dense, idx):
        assert dense.dtype == np.uint64 and dense.flags["C_CONTIGUOUS"] and dense.shape == (self.eng.np, self.eng.N)
        a, p, n = _idx(idx)
        if n:
            self.eng._ck(self.eng.lib.hb_poly_upload(self.h, p, n, dense.ctypes.data_as(u64p)))
        return self

    def upload_ptr(self, ptr, idx):
        """Upload from a raw host pointer to a dense [nprimes][N] matrix (e.g. pinned memory)."""
        a, p, n = _idx(idx)
        self.eng._ck(self.eng.lib.hb_poly_upload(self.h, p, n, C.cast(ptr, u64p)))

    def download_async_ptr(self, ptr, idx):
        a, p, n = _idx(idx)
        self.eng._ck(self.eng.lib.hb_poly_download_async(self.h, p, n, C.cast(ptr, u64p)))

    def download(self, idx, out=None):
        if out is None:
            out = np.zeros((self.eng.np, self.eng.N), dtype=np.uint64)
        a, p, n = _idx(idx)
        if n:
            self.eng._ck(self.eng.lib.hb_poly_download(self.h, p, n, out.ctypes.data_as(u64p)))
        return out


def _arr(polys):
    arr = (C.c_void_p * len(polys))(*[p.h for p in polys])
    return arr


class Engine:
    """Device image of a prime chain + the DoubleCRT operations of the hot path."""

    def __init__(self, m, primes, psis=None, digits=None, special=None, device=0, lib=None):
        self.lib = lib if lib is not None else load_library()
        self.m = int(m)
        self.N = _euler_phi(self.m)      # row length phi(m) (= m/2 for the power-of-two rings)
        self.primes = [int(q) for q in primes]
        self.np = len(self.primes)
        self.h = C.c_void_p()
        q = np.array(self.primes, dtype=np.uint64)
        ps = np.array([int(x) for x in psis], dtype=np.uint64) if psis is not None else None
        self._ck(self.lib.hb_ctx_create(C.byref(self.h), int(device), C.c_uint64(self.m), self.np,
                                        q.ctypes.data_as(u64p), ps.ctypes.data_as(u64p) if ps is not None else None))
        out = np.zeros(self.np, dtype=np.uint64)
        self._ck(self.lib.hb_ctx_get_psi(self.h, out.ctypes.data_as(u64p)))
        self.psis = [int(x) for x in out]
        self.digits = [list(d) for d in (digits or [])]
        self.special = list(special or [])
        if self.digits or self.special:
            digit_of = np.full(self.np, -1, dtype=np.int32)
            for d, lst in enumerate(self.digits):
                for i in lst:
                    digit_of[i] = d
            sp = np.ascontiguousarray(np.array(self.special, dtype=np.int32))
            self._ck(self.lib.hb_ctx_set_chain(self.h, digit_of.ctypes.data_as(i32p), len(self.digits),
                                               sp.ctypes.data_as(i32p), len(sp)))

    def close(self):
        if self.h:
            self.lib.hb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        # every Poly holds its engine, so an engine is collected only after its polys: the context's device memory (the
        # phase scratch alone is 2 x 64 x nprimes x N words) goes with it instead of staying allocated until the process exits
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise HbError(rc, self.lib.hb_last_error().decode())

    # ---- plumbing
    def poly(self, dense=None, idx=None):
        p = Poly(self)
        if dense is not None:
            p.upload(dense, idx)
        return p

    def sync(self):
        self._ck(self.lib.hb_ctx_sync(self.h))

    def stats(self):
        out = np.zeros(3, dtype=np.uint64)
        self._ck(self.lib.hb_ctx_stats(self.h, out.ctypes.data_as(u64p)))
        return {"exact_fallbacks": int(out[0]), "launches": int(out[1]), "device_bytes": int(out[2])}

    def reset_stats(self):
        self._ck(self.lib.hb_ctx_reset_stats(self.h))

    def mark_begin(self):
        self._ck(self.lib.hb_ctx_mark_begin(self.h))

    def mark_end(self) -> float:
        ms = C.c_float()
        self._ck(self.lib.hb_ctx_mark_end(self.h, C.byref(ms)))
        return ms.value

    def profile(self, enable: bool):
        self._ck(self.lib.hb_ctx_profile(self.h, int(enable)))

    def profile_results(self):
        out, i = [], 0
        while True:
            name = C.create_string_buffer(64)
            n, ms, by = C.c_uint64(), C.c_double(), C.c_uint64()
            if self.lib.hb_ctx_profile_get(self.h, i, name, 64, C.byref(n), C.byref(ms), C.byref(by)) != 0:
                break
            out.append({"kernel": name.value.decode(), "launches": n.value, "ms": ms.value, "bytes": by.value})
            i += 1
        return out

    # ---- operations (lists of Poly = batch items)
    def ntt_fwd(self, polys, idx):
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_ntt_fwd(_arr(polys), len(polys), p, n))

    def ntt_inv(self, polys, idx):
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_ntt_inv(_arr(polys), len(polys), p, n))

    def pointwise(self, op, dst, src, idx):
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_pointwise(OPS[op], _arr(dst), _arr(src), len(dst), p, n))

    def scale_rows(self, polys, idx, scalars):
        a, p, n = _idx(idx)
        sc = np.array([int(s) for s in scalars], dtype=np.uint64)
        self._ck(self.lib.hb_scale_rows(_arr(polys), len(polys), p, n, sc.ctypes.data_as(u64p)))

    def scale_by_primes(self, polys, idx, fidx, inv=False):
        a, p, n = _idx(idx)
        b, pf, nf = _idx(fidx)
        self._ck(self.lib.hb_scale_by_primes(_arr(polys), len(polys), p, n, pf, nf, int(inv)))

    def zero_rows(self, polys, idx):
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_zero_rows(_arr(polys), len(polys), p, n))

    def add_primes_and_scale(self, polys, cur, add):
        a, pc, nc = _idx(cur)
        b, pa, na = _idx(add)
        self._ck(self.lib.hb_add_primes_and_scale(_arr(polys), len(polys), pc, nc, pa, na))

    def add_primes(self, polys, cur, add):
        a, pc, nc = _idx(cur)
        b, pa, na = _idx(add)
        self._ck(self.lib.hb_add_primes(_arr(polys), len(polys), pc, nc, pa, na))

    def scale_down(self, polys, cur, keep, ptxt_space=1):
        a, pc, nc = _idx(cur)
        b, pk, nk = _idx(keep)
        self._ck(self.lib.hb_scale_down(_arr(polys), len(polys), pc, nc, pk, nk, C.c_uint64(int(ptxt_space))))

    def to_poly(self, poly, idx, positive=False, L=None):
        a, p, n = _idx(idx)
        L = L or (n + 1)
        out = np.zeros((self.N, L), dtype=np.uint64)
        self._ck(self.lib.hb_to_poly(poly.h, p, n, int(positive), out.ctypes.data_as(u64p), L))
        return out

    def set_powerful(self, mvec):
        arr = (C.c_int64 * len(mvec))(*[int(f) for f in mvec])
        self._ck(self.lib.hb_ctx_set_powerful(self.h, arr, len(mvec)))

    def powerful_info(self):
        nf = C.c_int32()
        mv = (C.c_int64 * 32)()
        to_poly = np.zeros(self.N, dtype=np.int32)
        self._ck(self.lib.hb_ctx_powerful_info(self.h, C.byref(nf), mv, to_poly.ctypes.data_as(C.POINTER(C.c_int32))))
        return [int(mv[i]) for i in range(nf.value)], to_poly

    def dcrt_to_powerful(self, poly, idx, L=None):
        a, p, n = _idx(idx)
        L = L or (n + 1)
        out = np.zeros((self.N, L), dtype=np.uint64)
        self._ck(self.lib.hb_dcrt_to_powerful(poly.h, p, n, out.ctypes.data_as(u64p), L))
        return out

    def raw_mod_switch(self, poly, idx, q, ptxt_space):
        a, p, n = _idx(idx)
        out = np.zeros(self.N, dtype=np.int64)
        self._ck(self.lib.hb_raw_mod_switch(poly.h, p, n, C.c_uint64(int(q)), C.c_uint64(int(ptxt_space)),
                                            out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def to_poly_mod_p(self, poly, idx, ptxt_space, factor=1):
        a, p, n = _idx(idx)
        out = np.zeros(self.N, dtype=np.int64)
        self._ck(self.lib.hb_to_poly_mod_p(poly.h, p, n, C.c_uint64(int(ptxt_space)), C.c_uint64(int(factor)),
                                           out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def from_i64(self, polys, idx, coeffs):
        """coeffs: [len(polys)][N] signed integers -> evaluation rows idx of each poly."""
        a, p, n = _idx(idx)
        buf = np.ascontiguousarray(np.asarray(coeffs, dtype=np.int64).reshape(len(polys), self.N))
        self._ck(self.lib.hb_poly_from_i64(_arr(polys), len(polys), p, n, buf.ctypes.data_as(C.POINTER(C.c_int64))))

    def from_limbs(self, polys, idx, limbs):
        """limbs: [len(polys)][N][L] two's-complement uint64 limbs (hb_to_poly layout)."""
        a, p, n = _idx(idx)
        buf = np.ascontiguousarray(np.asarray(limbs, dtype=np.uint64))
        L = buf.shape[-1]
        assert buf.size == len(polys) * self.N * L
        self._ck(self.lib.hb_poly_from_limbs(_arr(polys), len(polys), p, n, buf.ctypes.data_as(u64p), L))

    def muladd(self, dst, a_, b_, idx):
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_muladd(_arr(dst), _arr(a_), _arr(b_), len(dst), p, n))

    def break_into_digits(self, src, cur, digits=None):
        """digits: list (per item) of lists (per digit) of Poly; allocated if None."""
        a, pc, nc = _idx(cur)
        maxdig = len(self.digits)
        if digits is None:
            digits = [[Poly(self) for _ in range(maxdig)] for _ in src]
        flat = [d for item in digits for d in item]
        nd = C.c_int()
        self._ck(self.lib.hb_break_into_digits(_arr(src), len(src), pc, nc, _arr(flat), maxdig, C.byref(nd)))
        return [item[:nd.value] for item in digits]

    def keyswitch_digits(self, digits, idx, evk_a, evk_b, out0, out1):
        a, p, n = _idx(idx)
        nd = len(digits[0])
        flat = [d for item in digits for d in item]
        self._ck(self.lib.hb_keyswitch_digits(_arr(flat), nd, nd, len(digits), p, n, _arr(evk_a), _arr(evk_b), _arr(out0), _arr(out1)))

    def keyswitch_digits_fused(self, digits, idx, evk_a, evk_b, out0, out1, scal, own=None, own_dig=None):
        """out = scal[r]*out + sum_i D_i*evk_i on rows idx (scal 0 => pure output); rows with own_dig[r] = i take digit i
        from own[item] (hb_keyswitch_digits_fused)."""
        a, p, n = _idx(idx)
        nd = len(digits[0])
        flat = [d for item in digits for d in item]
        sc = np.array([int(x) for x in scal], dtype=np.uint64)
        od = np.ascontiguousarray(np.array(own_dig, dtype=np.int32)) if own_dig is not None else None
        self._ck(self.lib.hb_keyswitch_digits_fused(_arr(flat), nd, nd, len(digits), p, n, _arr(evk_a), _arr(evk_b), _arr(out0), _arr(out1),
                                                    sc.ctypes.data_as(u64p), _arr(own) if own is not None else None,
                                                    od.ctypes.data_as(i32p) if od is not None else None))

    def sub_div_by_primes(self, dst, src, idx, fidx):
        """dst = (dst - src) / prod(q_f) on rows idx (hb_sub_div_by_primes)."""
        a, p, n = _idx(idx)
        b, pf, nf = _idx(fidx)
        self._ck(self.lib.hb_sub_div_by_primes(_arr(dst), _arr(src), len(dst), p, n, pf, nf))

    def tensor(self, a0, a1, b0, b1, o0, o1, o2, idx):
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_tensor(_arr(a0), _arr(a1), _arr(b0), _arr(b1), _arr(o0), _arr(o1), _arr(o2), len(a0), p, n))

    def automorph(self, dst, src, idx, k):
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_automorph(_arr(dst), _arr(src), len(dst), p, n, C.c_uint64(int(k))))

    def relinearize(self, c0, c1, c2, S, evk_a, evk_b):
        a, p, n = _idx(S)
        self._ck(self.lib.hb_relinearize(_arr(c0), _arr(c1), _arr(c2), len(c0), p, n, _arr(evk_a), _arr(evk_b), len(evk_a)))

    def mul_relin_moddown(self, a0, a1, b0, b1, S_in, S, ptxt_space, evk_a, evk_b):
        x, pi, ni = _idx(S_in)
        y, ps, ns = _idx(S)
        self._ck(self.lib.hb_mul_relin_moddown(_arr(a0), _arr(a1), _arr(b0), _arr(b1), len(a0), pi, ni, ps, ns,
                                               C.c_uint64(int(ptxt_space)), _arr(evk_a), _arr(evk_b), len(evk_a)))

    def tensor_sum(self, a0, a1, b0, b1, o0, o1, o2, idx, accumulate=False):
        """Per item t: the tensor products of its pairs (a0[t][j], a1[t][j]) x (b0[t][j], b1[t][j]), summed into
        (o0[t], o1[t], o2[t]) on rows idx (hb_tensor_sum).  a0..b1: one list of pairs per item, all of one length."""
        npairs = len(a0[0])
        fl = [[p for item in x for p in item] for x in (a0, a1, b0, b1)]
        assert all(len(item) == npairs for x in (a0, a1, b0, b1) for item in x)
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_tensor_sum(_arr(fl[0]), _arr(fl[1]), _arr(fl[2]), _arr(fl[3]), npairs, len(a0), p, n,
                                        _arr(o0), _arr(o1), _arr(o2), int(bool(accumulate))))

    def ctxt_scaled_sums(self, in0, in1, out0, out1, U, scal, cst=None, accumulate=False):
        """Per item t and output j, on every row r of U: (out0, out1)[t][j] (+)= sum_i scal[j, i, r] * (in0, in1)[t][i],
        plus cst[j, r] on part 0 (hb_ctxt_scaled_sums).  in0/in1: one list of nin inputs per item; out0/out1: one list of
        nout outputs per item; scal: (nout, nin, len(U)) canonical residues; cst: (nout, len(U)) or None."""
        nin = len(in0[0]) if in0 else 0
        nout = len(out0[0]) if out0 else 0
        fi = [[p for item in x for p in item] for x in (in0, in1)]
        fo = [[p for item in x for p in item] for x in (out0, out1)]
        a, p, n = _idx(U)
        sc = np.ascontiguousarray(np.asarray(scal, dtype=np.uint64))
        cs = None if cst is None else np.ascontiguousarray(np.asarray(cst, dtype=np.uint64))
        self._ck(self.lib.hb_ctxt_scaled_sums(_arr(fi[0]), _arr(fi[1]), nin, _arr(fo[0]), _arr(fo[1]), nout, len(in0), p, n,
                                              sc.ctypes.data_as(u64p), cs.ctypes.data_as(u64p) if cs is not None else None,
                                              int(bool(accumulate))))

    def inner_product(self, a0, a1, b0, b1, S_in, S, ptxt_space, evk_a, evk_b, out0, out1, moddown=True):
        """Per item t: sum_j (a0,a1)[t][j] * (b0,b1)[t][j] brought to S, relinearised once into (out0[t], out1[t]) over
        S | special, and with moddown over S (hb_inner_product).  Operands over S_in are brought to S in place."""
        npairs = len(a0[0])
        fl = [[p for item in x for p in item] for x in (a0, a1, b0, b1)]
        assert all(len(item) == npairs for x in (a0, a1, b0, b1) for item in x)
        x, pi, ni = _idx(S_in)
        y, ps, ns = _idx(S)
        self._ck(self.lib.hb_inner_product(_arr(fl[0]), _arr(fl[1]), _arr(fl[2]), _arr(fl[3]), npairs, len(a0), pi, ni, ps, ns,
                                           C.c_uint64(int(ptxt_space)), _arr(evk_a), _arr(evk_b), len(evk_a),
                                           _arr(out0), _arr(out1), int(bool(moddown))))

    def square_tensor(self, a0, a1, o2, S_in, S, ptxt_space, norms=False):
        """Per item i: (a0[i], a1[i]) over S_in brought to S and squared in place, a1[i]^2 into o2[i] (hb_square_tensor).
        norms=True returns ||delta/P|| of each part, [item][part] (hb_square_tensor_norm)."""
        x, pi, ni = _idx(S_in)
        y, ps, ns = _idx(S)
        if not norms:
            self._ck(self.lib.hb_square_tensor(_arr(a0), _arr(a1), _arr(o2), len(a0), pi, ni, ps, ns, C.c_uint64(int(ptxt_space))))
            return None
        out = np.zeros(2 * len(a0), dtype=np.float64)
        self._ck(self.lib.hb_square_tensor_norm(_arr(a0), _arr(a1), _arr(o2), len(a0), pi, ni, ps, ns, C.c_uint64(int(ptxt_space)),
                                                out.ctypes.data_as(C.POINTER(C.c_double))))
        return out.reshape(len(a0), 2)

    def square_relin_moddown(self, a0, a1, S_in, S, ptxt_space, evk_a, evk_b):
        """Per item i: (a0[i], a1[i]) over S_in squared, relinearised and modded down to S in place (hb_square_relin_moddown)."""
        x, pi, ni = _idx(S_in)
        y, ps, ns = _idx(S)
        self._ck(self.lib.hb_square_relin_moddown(_arr(a0), _arr(a1), len(a0), pi, ni, ps, ns, C.c_uint64(int(ptxt_space)),
                                                  _arr(evk_a), _arr(evk_b), len(evk_a)))

    def randomize(self, polys, idx, seed):
        """NTL::SetSeed(seed), then p.randomize() over rows idx for each p in polys, expanded on the device
        (hb_poly_randomize).  seed: the ZZ's little-endian magnitude bytes, or a non-negative int."""
        if isinstance(seed, int):
            if seed < 0:
                raise ValueError("seed must be non-negative")
            seed = seed.to_bytes((seed.bit_length() + 7) // 8, "little")
        seed = bytes(seed)
        a, p, n = _idx(idx)
        buf = (C.c_uint8 * max(1, len(seed))).from_buffer_copy(seed or b"\0")
        self._ck(self.lib.hb_poly_randomize(_arr(polys), len(polys), p, n, buf, len(seed)))

    def seeded(self, npolys, idx, seed):
        """The rows randomize(npolys polys, idx, seed) would write, kept as the seed plus a row schedule
        (hb_poly_create_seeded).  The returned Polys have no rows: they go in any evk_a list, where the key switch
        regenerates the rows it reads, and to expand()."""
        if isinstance(seed, int):
            if seed < 0:
                raise ValueError("seed must be non-negative")
            seed = seed.to_bytes((seed.bit_length() + 7) // 8, "little")
        seed = bytes(seed)
        a, p, n = _idx(idx)
        buf = (C.c_uint8 * max(1, len(seed))).from_buffer_copy(seed or b"\0")
        hs = (C.c_void_p * max(1, npolys))()
        self._ck(self.lib.hb_poly_create_seeded(self.h, int(npolys), p, n, buf, len(seed), hs))
        out = []
        for h in hs[:npolys]:
            q = Poly.__new__(Poly)
            q.eng, q.h = self, C.c_void_p(h)
            out.append(q)
        return out

    def expand(self, seeded, dst, idx):
        """Rows idx of each seeded Poly into the ordinary Poly beside it in dst (hb_poly_expand)."""
        a, p, n = _idx(idx)
        self._ck(self.lib.hb_poly_expand(_arr(seeded), _arr(dst), len(seeded), p, n))


class Chain:
    """Host-side prime chain (hb_chain): helib::Context::buildModChain reproduced in C++."""

    def __init__(self, m, p, r, bits, c, sk_hwt=0, resolution=3, bits_in_special=0, stdev=3.2, lib=None, bootstrappable=False, scale=10.0):
        self.lib = lib if lib is not None else load_library()
        self.lib.hb_chain_last_error.restype = C.c_char_p
        self.lib.hb_chain_destroy.restype = None
        self.lib.hb_chain_destroy.argtypes = [C.c_void_p]
        self.h = C.c_void_p()
        rc = self.lib.hb_chain_build_ex(C.byref(self.h), C.c_uint64(m), C.c_int64(p), int(r), int(bits), int(c),
                                        int(sk_hwt), int(resolution), int(bits_in_special), C.c_double(stdev),
                                        int(bool(bootstrappable)), C.c_double(scale))
        if rc != 0:
            raise HbError(rc, self.lib.hb_chain_last_error().decode())
        n = [C.c_int() for _ in range(5)]
        phim = C.c_int64()
        self.lib.hb_chain_info(self.h, *[C.byref(x) for x in n], C.byref(phim))
        self.m, self.p, self.r, self.phim = int(m), int(p), int(r), phim.value
        npr = n[0].value
        primes = np.zeros(npr, dtype=np.uint64)
        kind = np.zeros(npr, dtype=np.int32)
        dig = np.zeros(npr, dtype=np.int32)
        self.lib.hb_chain_get(self.h, primes.ctypes.data_as(u64p), kind.ctypes.data_as(i32p), dig.ctypes.data_as(i32p))
        self.primes = [int(q) for q in primes]
        self.small = [i for i in range(npr) if kind[i] == 0]
        self.ctxt = [i for i in range(npr) if kind[i] == 1]
        self.special = [i for i in range(npr) if kind[i] == 2]
        self.digits = [[i for i in range(npr) if dig[i] == d] for d in range(n[4].value)]
        e, ep, hw = C.c_int64(), C.c_int64(), C.c_int64()
        self.lib.hb_chain_recrypt_params(self.h, C.byref(e), C.byref(ep), C.byref(hw))
        self.e_param, self.e_prime_param, self.sk_hwt = e.value, ep.value, hw.value

    def __del__(self):
        try:
            if self.h:
                self.lib.hb_chain_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set4size(self, low, high, from1, from2=None, reverse=False):
        a, p1, n1 = _idx(from1)
        out = np.zeros(len(self.primes), dtype=np.int32)
        nout = C.c_int()
        if from2 is None:
            rc = self.lib.hb_chain_set4size(self.h, C.c_double(low), C.c_double(high), p1, n1, None, 0, int(reverse), out.ctypes.data_as(i32p), C.byref(nout))
        else:
            b, p2, n2 = _idx(from2)
            rc = self.lib.hb_chain_set4size(self.h, C.c_double(low), C.c_double(high), p1, n1, p2, n2, int(reverse), out.ctypes.data_as(i32p), C.byref(nout))
        if rc != 0:
            raise HbError(rc, "hb_chain_set4size")
        return [int(x) for x in out[:nout.value]]


def _engine_extra(cls):
    def wrap(self, ptr):
        """Alias caller-owned device memory (uint64[nprimes][N]) as a Poly (hb_poly_wrap)."""
        p = Poly.__new__(Poly)
        p.eng = self
        p.h = C.c_void_p()
        self._ck(self.lib.hb_poly_wrap(self.h, C.c_void_p(ptr), C.byref(p.h)))
        return p

    def set_stream(self, cuda_stream):
        self._ck(self.lib.hb_ctx_set_stream(self.h, C.c_void_p(cuda_stream)))

    def conv_make_y(self, polys, D, owned, ypolys):
        a, pd, nd = _idx(D)
        b, po_, no = _idx(owned)
        self._ck(self.lib.hb_conv_make_y(_arr(polys), len(polys), pd, nd, po_, no, _arr(ypolys)))

    def conv_from_y(self, ypolys, D, tgt, ptxt_space, dst, mode):
        a, pd, nd = _idx(D)
        b, pt, nt = _idx(tgt)
        self._ck(self.lib.hb_conv_from_y(_arr(ypolys), len(ypolys), pd, nd, pt, nt, C.c_uint64(int(ptxt_space)), _arr(dst), int(mode)))

    cls.wrap, cls.set_stream, cls.conv_make_y, cls.conv_from_y = wrap, set_stream, conv_make_y, conv_from_y
    return cls


_engine_extra(Engine)


def _engine_norms(cls):
    def add_primes_norm(self, polys, cur, add):
        a, pc, nc = _idx(cur)
        b, pa, na = _idx(add)
        out = np.zeros(len(polys), dtype=np.float64)
        self._ck(self.lib.hb_add_primes_norm(_arr(polys), len(polys), pc, nc, pa, na, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def scale_down_norm(self, polys, cur, keep, ptxt_space=1):
        a, pc, nc = _idx(cur)
        b, pk, nk = _idx(keep)
        out = np.zeros(len(polys), dtype=np.float64)
        self._ck(self.lib.hb_scale_down_norm(_arr(polys), len(polys), pc, nc, pk, nk, C.c_uint64(int(ptxt_space)), out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def break_into_digits_norm(self, src, cur, digits=None):
        a, pc, nc = _idx(cur)
        maxdig = len(self.digits)
        if digits is None:
            digits = [[Poly(self) for _ in range(maxdig)] for _ in src]
        flat = [d for item in digits for d in item]
        nd = C.c_int()
        out = np.zeros(len(src) * maxdig, dtype=np.float64)
        self._ck(self.lib.hb_break_into_digits_norm(_arr(src), len(src), pc, nc, _arr(flat), maxdig, C.byref(nd), out.ctypes.data_as(C.POINTER(C.c_double))))
        return [item[:nd.value] for item in digits], out.reshape(len(src), maxdig)[:, :nd.value]

    cls.add_primes_norm, cls.scale_down_norm, cls.break_into_digits_norm = add_primes_norm, scale_down_norm, break_into_digits_norm
    return cls


_engine_norms(Engine)


def _engine_p2p(cls):
    def ipc_export(self, poly) -> bytes:
        buf = C.create_string_buffer(64)
        self._ck(self.lib.hb_poly_ipc_export(poly.h, buf))
        return buf.raw

    def ipc_open(self, handle: bytes):
        p = Poly.__new__(Poly)
        p.eng = self
        p.h = C.c_void_p()
        self._ck(self.lib.hb_poly_ipc_open(self.h, C.c_char_p(handle), C.byref(p.h)))
        return p

    def conv_make_y_bcast(self, polys, D, owned, ypolys, peer_ypolys):
        """peer_ypolys: list (per peer) of lists (per item) of Poly opened with ipc_open."""
        a, pd, nd = _idx(D)
        b, po_, no = _idx(owned)
        flat = [p for peer in peer_ypolys for p in peer]
        self._ck(self.lib.hb_conv_make_y_bcast(_arr(polys), len(polys), pd, nd, po_, no, _arr(ypolys),
                                               _arr(flat) if flat else None, len(peer_ypolys)))

    cls.ipc_export, cls.ipc_open, cls.conv_make_y_bcast = ipc_export, ipc_open, conv_make_y_bcast
    return cls


_engine_p2p(Engine)


def _engine_hoist(cls):
    def automorph_keyswitch_digits(self, digits, S, c0, k, evk_a, evk_b, out0, out1):
        a, p, n = _idx(S)
        nd = len(digits[0])
        flat = [d for item in digits for d in item]
        self._ck(self.lib.hb_automorph_keyswitch_digits(_arr(flat), nd, nd, len(digits), p, n, _arr(c0), C.c_uint64(int(k)),
                                                        _arr(evk_a), _arr(evk_b), _arr(out0), _arr(out1)))

    def hoisted_linear_map(self, digits, S, c0, c1, ks, consts, evk_a, evk_b, acc0, acc1, accumulate=False):
        """acc (+)= sum_j consts[j] * (hoisted automorph by ks[j]) over S | special, for every item (hb_hoisted_linear_map).
        digits: per item, the digit Polys of c1; c1 may be None when no k is 1; evk_a / evk_b: per amount, the list of
        ndig matrix Polys (None where k == 1)."""
        a, p, n = _idx(S)
        nd = len(digits[0])
        flat = [d for item in digits for d in item]
        kk = np.ascontiguousarray(np.array([int(x) for x in ks], dtype=np.uint64))
        na = len(kk)

        def keys(evk):
            arr = (C.c_void_p * max(1, na * nd))()
            for j, mat in enumerate(evk):
                for i in range(nd):
                    arr[j * nd + i] = mat[i].h if mat is not None else None
            return arr
        self._ck(self.lib.hb_hoisted_linear_map(_arr(flat), nd, nd, len(digits), p, n, _arr(c0), _arr(c1) if c1 is not None else None,
                                                na, kk.ctypes.data_as(u64p), _arr(consts), keys(evk_a), keys(evk_b),
                                                _arr(acc0), _arr(acc1), int(bool(accumulate))))

    def bsgs_linear_map(self, baby0, baby1, S, ks, consts, evk_a, evk_b, acc0, acc1, extended=False, ptxt_space=1,
                        scal=None, accumulate=False, norms=False):
        """acc (+)= the giant steps of a BSGS linear map over S | special, for every item (hb_bsgs_linear_map).
        baby0 / baby1: per item, the list of the baby steps' parts; consts: per giant step, one Poly (or None) per baby
        step; ks: the giant amounts; evk_a / evk_b: per giant step, the list of matrix Polys (None where k == 1).
        norms=True calls hb_bsgs_linear_map_norm and returns its norms as [item][giant step][10] (NaN where not written)."""
        a, p, n = _idx(S)
        nb = len(baby0[0])
        kk = np.ascontiguousarray(np.array([int(x) for x in ks], dtype=np.uint64))
        ng = len(kk)
        nd = max([len(m_) for m_ in evk_a if m_ is not None] or [1])
        cs = (C.c_void_p * (ng * nb))(*[c_.h if c_ is not None else None for row in consts for c_ in row])

        def keys(evk):
            arr = (C.c_void_p * (ng * nd))()
            for j, mat in enumerate(evk):
                for i in range(nd):
                    arr[j * nd + i] = mat[i].h if mat is not None else None
            return arr
        sc = np.ascontiguousarray(np.array([int(x) for x in scal], dtype=np.uint64)) if scal is not None else None
        args = (_arr([x for it in baby0 for x in it]), _arr([x for it in baby1 for x in it]), nb, len(baby0),
                p, n, int(bool(extended)), C.c_uint64(int(ptxt_space)), ng, kk.ctypes.data_as(u64p), cs,
                sc.ctypes.data_as(u64p) if sc is not None else None, keys(evk_a), keys(evk_b), nd,
                _arr(acc0), _arr(acc1), int(bool(accumulate)))
        if not norms:
            self._ck(self.lib.hb_bsgs_linear_map(*args))
            return None
        out = np.full((len(baby0), ng, 10), np.nan, dtype=np.float64)
        self._ck(self.lib.hb_bsgs_linear_map_norm(*args, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def block_linear_map(self, digits, S, c0, c1, k0, evk0_a, evk0_b, k1, evk1_a, evk1_b, consts, acc0, acc1,
                         consts1=None, kfinal=1, evkf_a=None, evkf_b=None, ptxt_space=1, accumulate=False, norms=False):
        """acc (+)= BlockMatMul1DExec's non-iterative branches over S | special, for every item (hb_block_linear_map).
        digits: per item, the digit Polys of c1; consts / consts1: per inner amount, one Poly (or None) per outer amount;
        consts1 (with kfinal and its matrix evkf_a / evkf_b) selects the bad dimension; evk*_a / evk*_b: per amount, the list
        of matrix Polys (None where the amount is 1).  norms=True calls hb_block_linear_map_norm and returns its norms as
        [item][entry][10] (entry j: set 0's term j; n1 + j: set 1's; 2*n1: the final term; NaN where not written)."""
        a, p, n = _idx(S)
        nd = len(digits[0])
        n0, n1 = len(k0), len(k1)

        def amounts(ks):
            return np.ascontiguousarray(np.array([int(x) for x in ks], dtype=np.uint64))

        def blocks(cs):
            return (C.c_void_p * (n0 * n1))(*[c_.h if c_ is not None else None for row in cs for c_ in row])

        def keys(evk, cnt):
            arr = (C.c_void_p * max(1, cnt * nd))()
            for j, mat in enumerate(evk):
                for i in range(nd):
                    arr[j * nd + i] = mat[i].h if mat is not None else None
            return arr
        kk0, kk1 = amounts(k0), amounts(k1)
        bad = consts1 is not None
        args = (_arr([d for item in digits for d in item]), nd, len(digits), p, n, _arr(c0), _arr(c1),
                C.c_uint64(int(ptxt_space)), n0, kk0.ctypes.data_as(u64p), keys(evk0_a, n0), keys(evk0_b, n0),
                n1, kk1.ctypes.data_as(u64p), keys(evk1_a, n1), keys(evk1_b, n1), blocks(consts),
                blocks(consts1) if bad else None, C.c_uint64(int(kfinal)),
                keys([evkf_a], 1) if bad else None, keys([evkf_b], 1) if bad else None, nd,
                _arr(acc0), _arr(acc1), int(bool(accumulate)))
        if not norms:
            self._ck(self.lib.hb_block_linear_map(*args))
            return None
        T = 2 * n1 + 1 if bad else n1
        out = np.full((len(digits), T, 10), np.nan, dtype=np.float64)
        self._ck(self.lib.hb_block_linear_map_norm(*args, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    def full_linear_map_leaves(self, x0, x1, S, ks, evk_a, evk_b, consts, acc0, acc1, ext=None, consts1=None, kfinal=1,
                               evkf_a=None, evkf_b=None, ptxt_space=1, accumulate=False, norms=False):
        """acc (+)= the leaves of MatMulFullExec::rec_mul over S | special, for every item (hb_full_linear_map_leaves).
        x0 / x1: per item, one Poly per leaf; ext: per leaf, whether it is over S | special (None: all over S); consts /
        consts1: per leaf, one Poly (or None) per amount; consts1 (with kfinal and its matrix evkf_a / evkf_b) selects a
        bad leaf dimension; evk_a / evk_b: per amount, the list of matrix Polys (None where the amount is 1).  norms=True
        calls hb_full_linear_map_leaves_norm and returns its norms as [item][entry][10] (entry l: leaf l's cleanUp and
        digits; nleaves + l: its final term; NaN where not written)."""
        a, p, n = _idx(S)
        nl, nit = len(x0[0]), len(x0)
        kk = np.ascontiguousarray(np.array([int(x) for x in ks], dtype=np.uint64))
        na = len(kk)
        nd = max([len(m_) for m_ in list(evk_a) + [evkf_a] if m_ is not None] or [1])

        def cst(cs):
            return (C.c_void_p * (nl * na))(*[c_.h if c_ is not None else None for row in cs for c_ in row])

        def keys(evk, cnt):
            arr = (C.c_void_p * max(1, cnt * nd))()
            for j, mat in enumerate(evk):
                for i in range(nd):
                    arr[j * nd + i] = mat[i].h if mat is not None else None
            return arr
        ex = np.ascontiguousarray(np.array([int(bool(e)) for e in ext], dtype=np.int32)) if ext is not None else None
        bad = consts1 is not None
        args = (_arr([x for it in x0 for x in it]), _arr([x for it in x1 for x in it]), nl, nit,
                ex.ctypes.data_as(C.POINTER(C.c_int32)) if ex is not None else None, p, n, C.c_uint64(int(ptxt_space)),
                na, kk.ctypes.data_as(u64p), keys(evk_a, na), keys(evk_b, na), cst(consts), cst(consts1) if bad else None,
                C.c_uint64(int(kfinal)), keys([evkf_a], 1) if bad else None, keys([evkf_b], 1) if bad else None, nd,
                _arr(acc0), _arr(acc1), int(bool(accumulate)))
        if not norms:
            self._ck(self.lib.hb_full_linear_map_leaves(*args))
            return None
        T = 2 * nl if bad else nl
        out = np.full((nit, T, 10), np.nan, dtype=np.float64)
        self._ck(self.lib.hb_full_linear_map_leaves_norm(*args, out.ctypes.data_as(C.POINTER(C.c_double))))
        return out

    cls.automorph_keyswitch_digits = automorph_keyswitch_digits
    cls.hoisted_linear_map = hoisted_linear_map
    cls.bsgs_linear_map = bsgs_linear_map
    cls.block_linear_map = block_linear_map
    cls.full_linear_map_leaves = full_linear_map_leaves
    return cls


_engine_hoist(Engine)


def _poly_io(cls):
    def serialize(self, idx) -> bytes:
        a, p, n = _idx(idx)
        need = C.c_uint64()
        self.eng._ck(self.eng.lib.hb_poly_serialized_size(self.h, n, C.byref(need)))
        buf = C.create_string_buffer(need.value)
        self.eng._ck(self.eng.lib.hb_poly_serialize(self.h, p, n, buf, need))
        return buf.raw

    def deserialize(self, data: bytes):
        out = np.zeros(self.eng.np, dtype=np.int32)
        n = C.c_int()
        self.eng._ck(self.eng.lib.hb_poly_deserialize(self.h, data, C.c_uint64(len(data)), out.ctypes.data_as(i32p), C.byref(n)))
        return [int(x) for x in out[:n.value]]

    cls.serialize, cls.deserialize = serialize, deserialize
    return cls


_poly_io(Poly)
