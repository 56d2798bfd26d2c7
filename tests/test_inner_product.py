"""Encrypted inner products on the device: hb_tensor_sum (k1_tensor_sum) and hb_inner_product.

innerProduct (src/Ctxt.cpp:2878-2893) sums the tensor products of its pairs and relinearises once.  hb_tensor_sum must equal
the oracle's tensorProduct summed per item, on the register path (k1_tensor_sum) and on the generic one (general m, small N,
HB_FORCE_V0), also with lazy operands and worst-case words at the largest primes; hb_inner_product must equal the oracle's
scale-down + tensor sum + reLinearize (+ scale-down to S) and, bit for bit, the composition of the existing entry points.
Every body runs on the CPU simulator build and, marked gpu, on the H100; the code generation of the kernel is checked on
sm_90a without a GPU."""
import os
import re
import subprocess

import numpy as np
import pytest

import pyoracle as po
from common import make, ptxt_space, rows_equal
from helib_b200.engine import Engine, HbError
from test_codegen import CSRC, _depots, _frames, _nvcc
from test_value_ranges import top_chain

HB_ERR_BAD_ARG = -1
HB_ERR_INDEX_SET = -2
SEED = 0x243F6A8885A308D313198A2E03707344


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


def kernels(E):
    return {r["kernel"]: r["launches"] for r in E.profile_results()}


def rand(ch, rng, idx, N):
    out = np.zeros((len(ch.primes), N), dtype=np.uint64)
    for i in idx:
        out[i] = rng.integers(0, ch.primes[i], size=N, dtype=np.uint64)
    return out


def ref_tensor_sum(ch, O, ops, idx, old=None):
    """sum over the pairs (a0, a1, b0, b1) of the oracle's tensorProduct (python integers without an oracle), mod q."""
    acc = [np.zeros_like(ops[0][0]) for _ in range(3)] if old is None else [x.copy() for x in old]
    for a0, a1, b0, b1 in ops:
        if O is not None:
            t = O.tensor(*(x % np.array(ch.primes, dtype=np.uint64)[:, None] for x in (a0, a1, b0, b1)), idx)
        else:
            t = [np.zeros_like(a0) for _ in range(3)]
            for i in idx:
                q = ch.primes[i]
                A0, A1, B0, B1 = ([int(v) % q for v in x[i]] for x in (a0, a1, b0, b1))
                t[0][i] = [x * y % q for x, y in zip(A0, B0)]
                t[1][i] = [(x * y + z * w) % q for x, y, z, w in zip(A0, B1, A1, B0)]
                t[2][i] = [x * y % q for x, y in zip(A1, B1)]
        for k in range(3):
            for i in idx:
                acc[k][i] = (acc[k][i] % ch.primes[i] + t[k][i]) % ch.primes[i]
    return acc


def run_tensor_sum(E, ch, O, ops, nitems, npairs, idx, accumulate, old=None):
    """ops[t][j] = (a0, a1, b0, b1) arrays; identical arrays in one pair share one Poly (a == b)."""
    P = []
    for item in ops:
        row = []
        for a0, a1, b0, b1 in item:
            pa0, pa1 = E.poly(a0, idx), E.poly(a1, idx)
            same = a0 is b0 and a1 is b1
            row.append((pa0, pa1, pa0 if same else E.poly(b0, idx), pa1 if same else E.poly(b1, idx)))
        P.append(row)
    outs = [[E.poly(old[t][k], idx) if old else E.poly() for t in range(nitems)] for k in range(3)]
    E.profile(True)
    E.tensor_sum(*([[pr[k] for pr in item] for item in P] for k in range(4)), *outs, idx, accumulate)
    E.profile(False)
    for t in range(nitems):
        ref = ref_tensor_sum(ch, O, ops[t], idx, old[t] if old else None)
        for k in range(3):
            assert rows_equal(outs[k][t].download(idx), ref[k], idx), (t, k)
    return kernels(E)


# ---- 1. hb_tensor_sum against the oracle

@pytest.mark.parametrize("m, npairs, nitems, accumulate, alias", [
    (8192, 1, 3, False, False),
    (8192, 3, 4, True, True),            # a == b: sums of squares
    (8192, 130, 2, True, False),         # two reduction groups and two launches per item
    (1 << 17, 3, 2, False, False),       # N = 2^16
], ids=["n4096-1pair", "n4096-3pairs-alias", "n4096-130pairs", "n65536-3pairs"])
def test_tensor_sum_matches_oracle(lib, m, npairs, nitems, accumulate, alias):
    ch, psis, O, E = make(lib, m, -1, 1, 119, 2)
    rng = np.random.default_rng(201)
    idx = ch.ctxt[:2] if npairs > 10 else ch.ctxt
    ops = []
    for _ in range(nitems):
        item = []
        for _ in range(npairs):
            a0, a1 = rand(ch, rng, idx, E.N), rand(ch, rng, idx, E.N)
            item.append((a0, a1, a0, a1) if alias else (a0, a1, rand(ch, rng, idx, E.N), rand(ch, rng, idx, E.N)))
        ops.append(item)
    old = [[rand(ch, rng, idx, E.N) for _ in range(3)] for _ in range(nitems)] if accumulate else None
    ran = run_tensor_sum(E, ch, O, ops, nitems, npairs, idx, accumulate, old)
    assert set(ran) == {"k1_tensor_sum"}, ran
    if npairs == 130:   # 128 pair slots per launch: each item takes a launch of 128 pairs and one of 2
        assert ran["k1_tensor_sum"] == 2 * nitems, ran


@pytest.mark.parametrize("case", ["general-m", "small-n", "force-v0"])
def test_tensor_sum_generic_path(lib, monkeypatch, case):
    """General m, N not a multiple of 512 and HB_FORCE_V0 compose k_pw_tensor and k_pw_add."""
    if case == "force-v0":
        monkeypatch.setenv("HB_FORCE_V0", "1")
    if case == "general-m":
        ch = po.build_mod_chain(105, 2, 1, 120, 2)
        O, E = None, Engine(105, ch.primes, None, ch.digits, ch.special, lib=lib)
    else:
        ch, psis, O, E = make(lib, 256 if case == "small-n" else 8192, -1, 1, 119, 2)
    rng = np.random.default_rng(202)
    idx = ch.ctxt
    ops = [[tuple(rand(ch, rng, idx, E.N) for _ in range(4)) for _ in range(3)] for _ in range(2)]
    for accumulate in (False, True):
        old = [[rand(ch, rng, idx, E.N) for _ in range(3)] for _ in range(2)] if accumulate else None
        ran = run_tensor_sum(E, ch, O, ops, 2, 3, idx, accumulate, old)
        assert "k1_tensor_sum" not in ran and {"k_pw_tensor", "k_pw_add"} <= set(ran), ran


# ---- 2. worst-case words at the largest primes

@pytest.mark.parametrize("form", ["sp", "gen"])
@pytest.mark.parametrize("npairs", [127, 128])
@pytest.mark.parametrize("word", ["q-1", "lazy"])
def test_tensor_sum_worst_case(lib, form, npairs, word):
    """Chains of the largest primes below 2^60 (test_value_ranges.largest_primes, both modulus forms).  Every operand word
    at q-1, or lazy at 8q + 2^32 - 1 (= 2^32 - 1 mod q), at the reduction-group limit (127 pairs:
    254 products of (q-1)^2 in o1's 128-bit sum, plus the old output) and one past it.  Old outputs at q-1."""
    ch, O, E = top_chain(lib, 2048, -1, form, [2, 1], 1)
    idx = ch.ctxt
    x = np.zeros((len(ch.primes), E.N), dtype=np.uint64)
    for i in idx:
        q = ch.primes[i]
        x[i] = q - 1 if word == "q-1" else 8 * q + (1 << 32) - 1
    old = [[np.where(x > 0, np.array(ch.primes, dtype=np.uint64)[:, None] - 1, 0).astype(np.uint64) for _ in range(3)]]
    ops = [[(x, x, x, x)] * npairs]
    ran = run_tensor_sum(E, ch, O, ops, 1, npairs, idx, True, old)
    assert set(ran) == {"k1_tensor_sum"}, ran


# ---- 3. hb_inner_product against the oracle and the composition of the existing entry points

def keys(E, ch, rng, seeded):
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    if seeded:
        SA = E.seeded(nd, full, SEED)
        EA = [E.poly() for _ in range(nd)]
        E.randomize(EA, full, SEED)
    else:
        EA = [E.poly(rand(ch, rng, full, E.N), full) for _ in range(nd)]
        SA = EA
    EB = [E.poly(rand(ch, rng, full, E.N), full) for _ in range(nd)]
    ea = np.stack([p.download(full) for p in EA])
    eb = np.stack([p.download(full) for p in EB])
    return SA, EA, EB, ea, eb


def oracle_inner_product(O, ch, pairs, S_in, S, p, evk_a, evk_b, moddown):
    """innerProduct restated: every part scaled down to S, the tensor products summed, relinearised, scaled down to S."""
    parts = []
    for pr in pairs:
        xs = [x.copy() for x in pr]
        for x in xs:
            O.scale_down(x, S_in, S, p)
        parts.append(xs)
    t = ref_tensor_sum(ch, O, parts, S)
    r0, r1 = O.relinearize(t[0], t[1], t[2], S, evk_a, evk_b)
    if moddown:
        Sp = sorted(S + ch.special)
        O.scale_down(r0, Sp, S, p)
        O.scale_down(r1, Sp, S, p)
    return r0, r1


def composed(E, ch, P, S_in, S, p, EA, EB, moddown):
    """The same with the existing entry points: hb_scale_down, hb_tensor and ADDs per pair, hb_relinearize, hb_scale_down."""
    outs = []
    for item in P:
        cp = [[E.poly(x.download(S_in), S_in) for x in pr] for pr in item]
        if S != S_in:
            E.scale_down([x for pr in cp for x in pr], S_in, S, p)
        acc = [E.poly() for _ in range(3)]
        E.tensor(*([x] for x in cp[0]), *([a] for a in acc), S)
        for pr in cp[1:]:
            t = [E.poly() for _ in range(3)]
            E.tensor(*([x] for x in pr), *([a] for a in t), S)
            for k in range(3):
                E.pointwise("add", [acc[k]], [t[k]], S)
        E.relinearize([acc[0]], [acc[1]], [acc[2]], S, EA, EB)
        if moddown:
            E.scale_down([acc[0], acc[1]], sorted(S + ch.special), S, p)
        outs.append((acc[0], acc[1]))
    return outs


def inner_case(E, ch, O, S_in, S, p, npairs, nitems, moddown, seeded, alias=False, rng_seed=203, check=None):
    rng = np.random.default_rng(rng_seed)
    SA, EA, EB, ea, eb = keys(E, ch, rng, seeded)
    ops = []
    for _ in range(nitems):
        item = []
        for _ in range(npairs):
            a0, a1 = rand(ch, rng, S_in, E.N), rand(ch, rng, S_in, E.N)
            item.append((a0, a1, a0, a1) if alias else (a0, a1, rand(ch, rng, S_in, E.N), rand(ch, rng, S_in, E.N)))
        ops.append(item)
    P = []
    for item in ops:
        row = []
        for a0, a1, b0, b1 in item:
            pa0, pa1 = E.poly(a0, S_in), E.poly(a1, S_in)
            row.append((pa0, pa1, pa0, pa1) if alias else (pa0, pa1, E.poly(b0, S_in), E.poly(b1, S_in)))
        P.append(row)
    comp = composed(E, ch, P, S_in, S, p, EA, EB, moddown)
    out0, out1 = [E.poly() for _ in range(nitems)], [E.poly() for _ in range(nitems)]
    E.profile(True)
    E.inner_product(*([[pr[k] for pr in item] for item in P] for k in range(4)), S_in, S, p, SA, EB, out0, out1, moddown)
    E.profile(False)
    ran = kernels(E)
    R = S if moddown else sorted(S + ch.special)
    for t in (range(nitems) if check is None else check):
        if O is not None:
            r0, r1 = oracle_inner_product(O, ch, ops[t], S_in, S, p, ea, eb, moddown)
            assert rows_equal(out0[t].download(R), r0, R) and rows_equal(out1[t].download(R), r1, R), t
        assert rows_equal(out0[t].download(R), comp[t][0].download(R), R), t
        assert rows_equal(out1[t].download(R), comp[t][1].download(R), R), t
    return ran, P, (SA, EB), (out0, out1)


@pytest.mark.parametrize("cfg, drop, moddown, seeded, alias", [
    ((8192, 257, 1, 119, 2), 1, True, False, False),
    ((8192, 257, 1, 119, 2), 0, False, True, False),
    ((8192, -1, 1, 119, 2), 1, False, True, False),
    ((8192, -1, 1, 119, 2), 0, True, False, False),
    ((8192, 257, 1, 119, 2), 1, True, True, True),
], ids=["bgv-drop-moddown", "bgv-same-seeded", "ckks-drop-seeded", "ckks-same-moddown", "bgv-squares-seeded"])
def test_inner_product_matches_oracle_and_composition(lib, cfg, drop, moddown, seeded, alias):
    ch, psis, O, E = make(lib, *cfg, nthreads=8)
    S_in = ch.ctxt
    S = ch.ctxt[:len(ch.ctxt) - drop]
    ran, P, key, outs = inner_case(E, ch, O, S_in, S, ptxt_space(ch), 3, 2, moddown, seeded, alias)
    assert "k1_tensor_sum" in ran and "k1_tensor" not in ran and "k_pw_tensor" not in ran, ran
    # a second call of the same shape allocates nothing
    before = E.stats()["device_bytes"]
    E.inner_product(*([[pr[k] for pr in item] for item in P] for k in range(4)), S, S, ptxt_space(ch), *key, *outs, moddown)
    assert E.stats()["device_bytes"] == before


@pytest.mark.parametrize("case", ["general-m", "force-v0"])
def test_inner_product_generic_paths_match_composition(sim_lib, monkeypatch, case):
    """General m (Bluestein rows) and HB_FORCE_V0: the generic tensor sum, bit for bit the composed entry points."""
    if case == "force-v0":
        monkeypatch.setenv("HB_FORCE_V0", "1")
        ch, psis, O, E = make(sim_lib, 8192, 257, 1, 119, 2)
    else:
        ch = po.build_mod_chain(105, 2, 1, 120, 2)
        O, E = None, Engine(105, ch.primes, None, ch.digits, ch.special, lib=sim_lib)
    ran, *_ = inner_case(E, ch, O, ch.ctxt, ch.ctxt[:-1], ptxt_space(ch), 2, 2, True, False)
    assert "k1_tensor_sum" not in ran and "k_pw_tensor" in ran, ran


@pytest.mark.gpu
def test_inner_product_full_size_config2(cuda_lib):
    """BASELINE config 2 (m = 2^17, 20 ctxt primes, CKKS): two inner products of 17 pairs, one prime dropped."""
    ch, psis, O, E = make(cuda_lib, 1 << 17, -1, 1, 1190, 2, nthreads=8)
    assert len(ch.ctxt) == 20
    ran, *_ = inner_case(E, ch, O, ch.ctxt, ch.ctxt[:-1], 1, 17, 2, True, False)
    assert "k1_tensor_sum" in ran, ran


# ---- 4. argument errors: the code, and nothing launched

def test_errors_are_reported_before_any_launch(lib):
    ch, psis, O, E = make(lib, 8192, 257, 1, 119, 2)
    rng = np.random.default_rng(204)
    S = ch.ctxt
    full = sorted(ch.ctxt + ch.special)
    nd = len(ch.digits)
    EA = [E.poly(rand(ch, rng, full, E.N), full) for _ in range(nd)]
    EB = [E.poly(rand(ch, rng, full, E.N), full) for _ in range(nd)]
    ops = [[[E.poly(rand(ch, rng, S, E.N), S)] for _ in range(1)] for _ in range(4)]   # [part][item][pair]
    o = [E.poly() for _ in range(3)]

    def expect(code, f):
        E.profile(True)
        with pytest.raises(HbError) as e:
            f()
        E.profile(False)
        assert e.value.code == code, e.value
        assert E.profile_results() == [], E.profile_results()

    ip = lambda a, S_in, S_, out0, out1, ea=EA, eb=EB: E.inner_product(*a, S_in, S_, 257, ea, eb, out0, out1)
    ts = lambda a, o0, o1, o2: E.tensor_sum(*a, [o0], [o1], [o2], S)
    empty = [[[]] for _ in range(4)]
    expect(HB_ERR_BAD_ARG, lambda: ts(empty, *o))
    expect(HB_ERR_BAD_ARG, lambda: ip(empty, S, S, [o[0]], [o[1]]))
    expect(HB_ERR_BAD_ARG, lambda: ts(ops, ops[0][0][0], o[1], o[2]))        # an output aliasing an input
    expect(HB_ERR_BAD_ARG, lambda: ts(ops, o[0], o[0], o[2]))                # two outputs alike
    expect(HB_ERR_BAD_ARG, lambda: ip(ops, S, S, [ops[3][0][0]], [o[1]]))
    expect(HB_ERR_BAD_ARG, lambda: ip(ops, S, S, [o[0]], [o[0]]))
    expect(HB_ERR_BAD_ARG, lambda: ip(ops, S, S, [EB[0]], [o[1]]))           # an output aliasing a key
    expect(HB_ERR_INDEX_SET, lambda: ip(ops, S[:-1], S, [o[0]], [o[1]]))     # S not within S_in
    expect(HB_ERR_INDEX_SET, lambda: ip(ops, full, [ch.special[0]], [o[0]], [o[1]]))   # S not within the ctxt primes
    expect(HB_ERR_BAD_ARG, lambda: ip(ops, S, S, [o[0]], [o[1]], EA[:1], EB[:1]))      # too few matrix columns


# ---- 5. code generation on sm_90a

def test_tensor_sum_kernel_has_no_local_array_stack_frame_or_spill(tmp_path):
    """k1_tensor_sum keeps its six 128-bit sums in registers and reads the pairs' pointers from the parameter space: no local
    array in the PTX, and a (0, 0, 0) frame in `ptxas -v`."""
    nvcc = _nvcc()
    ptx = str(tmp_path / "hb_engine.ptx")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ptx",
                    os.path.join(CSRC, "hb_engine.cu"), "-o", ptx], check=True, capture_output=True, text=True)
    r = subprocess.run([os.path.join(os.path.dirname(nvcc), "ptxas"), "-arch=sm_90a", "-O3", "-v", ptx,
                        "-o", str(tmp_path / "hb_engine.cubin")], check=True, capture_output=True, text=True)
    mine = lambda k: re.match(r"_Z\d+k1_tensor_sum[A-Z]", k) is not None
    depots = {k: v for k, v in _depots(open(ptx).read()).items() if mine(k)}
    frames = {k: v for k, v in _frames(r.stdout + r.stderr).items() if mine(k)}
    assert len(frames) == 1, frames
    assert not depots, depots
    assert all(v == (0, 0, 0) for v in frames.values()), frames


# ---- 6. the C++ mirror (tests/cpp/test_inner_product.cpp): hb::innerProduct against the transcribed loop

def test_mirror_inner_product_on_simulator():
    from test_cpp_shim import build_exe
    r = subprocess.run([build_exe("test_inner_product", sim=True)], capture_output=True, text=True)
    assert r.returncode == 0 and "inner product OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_inner_product_on_gpu():
    from test_cpp_shim import build_exe
    r = subprocess.run([build_exe("test_inner_product")], capture_output=True, text=True)
    assert r.returncode == 0 and "inner product OK" in r.stdout, r.stdout + r.stderr
