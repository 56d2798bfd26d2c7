"""Polynomial evaluation on the device: hb_ctxt_scaled_sums (k1_scaled_sums) and the mirror's hb::polyEval.

polyEval (src/polyEval.cpp:129-389) spends its additions in simplePolyEval, whose every leaf is sum_i s_{i,r} X^i + c_r on
every row r.  hb_ctxt_scaled_sums must equal per-row big-integer arithmetic on power-of-two and general-m rings, for any N,
across the 128-bit carry group, across launches and input groups, and with worst-case words at the largest primes below
2^60; its errors come before any launch; its kernel has no local memory.  hb::polyEval must equal a literal transcription
of HElib's code (tests/cpp/test_poly_eval.cpp).  Every body runs on the CPU simulator build and, marked gpu, on the H100."""
import os
import re
import subprocess

import numpy as np
import pytest

import pyoracle as po
from common import make
from helib_b200.engine import Engine, HbError
from test_codegen import CSRC, _depots, _frames, _nvcc
from test_value_ranges import top_chain

HB_ERR_BAD_ARG = -1
HB_ERR_INDEX_SET = -2
ONES = np.uint64(0xFFFFFFFFFFFFFFFF)
HB_SSUM_MAXIN = (96 * 1024) // (16 * 32 + 1)


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


def kernels(E):
    return {r["kernel"]: r["launches"] for r in E.profile_results()}


def engine(lib, ring):
    if ring == "general-m":
        ch = po.build_mod_chain(105, 2, 1, 120, 2)
        return ch, Engine(105, ch.primes, None, ch.digits, ch.special, lib=lib)
    m = {"n4096": 8192, "n128": 256}[ring]
    ch, psis, O, E = make(lib, m, -1, 1, 119, 2)
    return ch, E


def reference(ch, U, ins, scal, cst, old):
    """out_k[j] = old_k[j] + sum_i scal[j, i, r] * in_k[i] (+ cst[j, r] on part 0) mod q, in Python integers."""
    nout = scal.shape[0]
    outs = []
    for j in range(nout):
        parts = []
        for k in range(2):
            o = np.zeros((len(ch.primes), ins[0][0].shape[1]), dtype=np.uint64)
            for r, row in enumerate(U):
                q = ch.primes[row]
                acc = [0] * o.shape[1] if old is None else [int(v) for v in old[j][k][row]]
                if k == 0 and cst is not None:
                    acc = [a + int(cst[j, r]) for a in acc]
                for i in range(scal.shape[1]):
                    s = int(scal[j, i, r])
                    if s:
                        acc = [a + s * int(v) for a, v in zip(acc, ins[i][k][row])]
                o[row] = [a % q for a in acc]
            parts.append(o)
        outs.append(parts)
    return outs


def run(E, ch, U, nin, nout, nitems, accumulate, with_cst, rng, absent=None):
    """Random inputs (any 64-bit words), scalars and constants; absent[i] = the rows of U input i does not have: they are
    poisoned with all-ones words and take zero scalars.  Returns the launches."""
    N = E.N
    qU = np.array([ch.primes[r] for r in U], dtype=np.uint64)
    scal = np.stack([np.stack([rng.integers(0, qU, dtype=np.uint64) for _ in range(nin)]) for _ in range(nout)])
    scal[:, ::3, :] = np.where(rng.random((nout, len(range(0, nin, 3)), len(U))) < 0.3, 0, scal[:, ::3, :])
    cst = np.stack([rng.integers(0, qU, dtype=np.uint64) for _ in range(nout)]) if with_cst else None
    items = []
    for _ in range(nitems):
        ins = []
        for i in range(nin):
            pr = []
            for _ in range(2):
                x = np.zeros((len(ch.primes), N), dtype=np.uint64)
                for row in U:
                    x[row] = rng.integers(0, 1 << 64, size=N, dtype=np.uint64)
                pr.append(x)
            ins.append(pr)
        items.append(ins)
    for i, rows in (absent or {}).items():
        for r, row in enumerate(U):
            if row in rows:
                scal[:, i, r] = 0
                for ins in items:
                    ins[i][0][row] = ONES
                    ins[i][1][row] = ONES
    old = [[[rng.integers(0, 1 << 64, size=(len(ch.primes), N), dtype=np.uint64) for _ in range(2)] for _ in range(nout)]
           for _ in range(nitems)] if accumulate else None
    P_in = [[[E.poly(ins[i][k], U) for i in range(nin)] for ins in items] for k in range(2)]
    P_out = [[[E.poly(old[t][j][k], U) if accumulate else E.poly() for j in range(nout)] for t in range(nitems)] for k in range(2)]
    E.profile(True)
    E.ctxt_scaled_sums(P_in[0], P_in[1], P_out[0], P_out[1], U, scal, cst, accumulate)
    E.profile(False)
    ran = kernels(E)
    if ran == {"k1_scaled_sums": 1}:
        # the launch's algorithmic bytes count an input row only where some output's scalar is nonzero: the poisoned rows of
        # an absent input, and every row whose scalars are all zero, are not among the rows it reads
        read = sum(int(scal[:, i, r].any()) for i in range(nin) for r in range(len(U)))
        assert read < nin * len(U) or not absent
        want = (2 * read + 2 * nout * len(U) * (2 if accumulate else 1)) * nitems * N * 8
        assert [r["bytes"] for r in E.profile_results()] == [want]
    for t in range(nitems):
        want = reference(ch, U, items[t], scal, cst, old[t] if accumulate else None)
        for j in range(nout):
            for k in range(2):
                got = P_out[k][t][j].download(U)
                assert (got[U] == want[j][k][U]).all(), (t, j, k)
    before = E.stats()["device_bytes"]
    E.ctxt_scaled_sums(P_in[0], P_in[1], P_out[0], P_out[1], U, scal, cst, True)   # the same shape allocates nothing
    assert E.stats()["device_bytes"] == before
    return ran


# ---- 1. the entry point against per-row big-integer arithmetic

@pytest.mark.parametrize("ring, nin, nout, nitems, accumulate, with_cst", [
    ("n4096", 5, 3, 2, False, True),
    ("n4096", 4, 2, 3, True, False),
    ("n128", 3, 2, 2, True, True),        # N not a multiple of 512
    ("general-m", 3, 2, 2, False, True),  # m = 105: N = 48
    ("general-m", 2, 2, 1, True, False),
], ids=["n4096", "n4096-acc-nocst", "n128-acc", "general-m", "general-m-acc-nocst"])
def test_scaled_sums_match_reference(lib, ring, nin, nout, nitems, accumulate, with_cst):
    ch, E = engine(lib, ring)
    rng = np.random.default_rng(301)
    U = ch.ctxt
    absent = {1: set(U[len(U) // 2:])}   # input 1 is over a smaller set: its other rows are poisoned and never weigh in
    ran = run(E, ch, U, nin, nout, nitems, accumulate, with_cst, rng, absent)
    assert set(ran) == {"k1_scaled_sums"}, ran
    assert ran["k1_scaled_sums"] == 1, ran


@pytest.mark.parametrize("nin", [127, 128, HB_SSUM_MAXIN + 2])
def test_scaled_sums_carry_groups_and_input_groups(lib, nin):
    """127 products per 128-bit sum, then a carry; more inputs than one launch stages run as accumulating input groups."""
    ch, E = engine(lib, "n128")
    rng = np.random.default_rng(302)
    ran = run(E, ch, ch.ctxt[:1], nin, 2, 1, False, True, rng)
    assert ran == {"k1_scaled_sums": 1 if nin <= HB_SSUM_MAXIN else 2}, ran


def test_scaled_sums_outputs_past_one_launch(lib):
    """70 outputs per item (past HB_MAXB = 64 item-output pairs): one launch per item, every output of it in one pass."""
    ch, E = engine(lib, "n128")
    rng = np.random.default_rng(303)
    ran = run(E, ch, ch.ctxt[:1], 2, 70, 2, True, True, rng)
    assert ran == {"k1_scaled_sums": 2}, ran


# ---- 2. worst-case words at the largest primes

@pytest.mark.parametrize("form", ["sp", "gen"])
@pytest.mark.parametrize("nin", [127, 128])
def test_scaled_sums_worst_case(lib, form, nin):
    """Chains of the largest primes below 2^60 (test_value_ranges.largest_primes, both modulus forms): every input word
    all-ones, every scalar and constant q-1, old outputs all-ones, at the carry-group limit and one past it."""
    ch, O, E = top_chain(lib, 2048, -1, form, [2, 1], 1)
    U = ch.ctxt
    N = E.N
    ones = np.full((len(ch.primes), N), ONES, dtype=np.uint64)
    qU = np.array([ch.primes[r] for r in U], dtype=np.uint64)
    nout = 2
    scal = np.broadcast_to(qU - 1, (nout, nin, len(U))).copy()
    cst = np.broadcast_to(qU - 1, (nout, len(U))).copy()
    P_in = [[[E.poly(ones, U) for _ in range(nin)]] for _ in range(2)]
    P_out = [[[E.poly(ones, U) for _ in range(nout)]] for _ in range(2)]
    E.profile(True)
    E.ctxt_scaled_sums(P_in[0], P_in[1], P_out[0], P_out[1], U, scal, cst, True)
    E.profile(False)
    assert kernels(E) == {"k1_scaled_sums": 1}
    for r, row in enumerate(U):
        q = ch.primes[row]
        w = (1 << 64) - 1
        base = (w + nin * (q - 1) * w) % q
        for j in range(nout):
            assert (P_out[0][0][j].download(U)[row] == (base + q - 1) % q).all(), (row, j)
            assert (P_out[1][0][j].download(U)[row] == base).all(), (row, j)


# ---- 3. argument errors: the code, nothing launched, the outputs untouched

def test_errors_are_reported_before_any_launch(lib):
    ch, E = engine(lib, "n4096")
    rng = np.random.default_rng(304)
    U = ch.ctxt
    qU = np.array([ch.primes[r] for r in U], dtype=np.uint64)
    x = np.zeros((len(ch.primes), E.N), dtype=np.uint64)
    for r in U:
        x[r] = rng.integers(0, ch.primes[r], size=E.N, dtype=np.uint64)
    i0, i1 = [[E.poly(x, U), E.poly(x, U)]], [[E.poly(x, U), E.poly(x, U)]]
    o0, o1 = [[E.poly(x, U)]], [[E.poly(x, U)]]
    scal = np.ones((1, 2, len(U)), dtype=np.uint64)
    cst = np.zeros((1, len(U)), dtype=np.uint64)
    seeded = E.seeded(1, U, 0x1234)

    def expect(code, f):
        E.profile(True)
        with pytest.raises(HbError) as e:
            f()
        E.profile(False)
        assert e.value.code == code, e.value
        assert E.profile_results() == [], E.profile_results()
        for o in (o0[0][0], o1[0][0]):
            assert (o.download(U)[U] == x[U]).all()

    call = lambda a=i0, b=i1, c=o0, d=o1, u=U, s=scal, k=cst: E.ctxt_scaled_sums(a, b, c, d, u, s, k)
    expect(HB_ERR_BAD_ARG, lambda: call(a=[[]], b=[[]], s=np.ones((1, 0, len(U)), dtype=np.uint64)))   # nin = 0
    expect(HB_ERR_BAD_ARG, lambda: call(c=[[]], d=[[]], s=np.ones((0, 2, len(U)), dtype=np.uint64)))   # nout = 0
    expect(HB_ERR_BAD_ARG, lambda: call(a=[], b=[], c=[], d=[]))                                         # nitems = 0
    big = scal.copy()
    big[0, 1, -1] = qU[-1]
    expect(HB_ERR_BAD_ARG, lambda: call(s=big))                                 # a scalar not below its prime
    bigc = cst.copy()
    bigc[0, 0] = qU[0]
    expect(HB_ERR_BAD_ARG, lambda: call(k=bigc))                                # a constant not below its prime
    expect(HB_ERR_BAD_ARG, lambda: call(c=[[i0[0][1]]]))                        # an output aliasing an input
    expect(HB_ERR_BAD_ARG, lambda: call(d=o0))                                  # two outputs alike
    expect(HB_ERR_BAD_ARG, lambda: call(a=[[i0[0][0], seeded[0]]]))             # a seeded handle
    expect(HB_ERR_INDEX_SET, lambda: call(u=U[::-1]))                           # U unsorted
    expect(HB_ERR_INDEX_SET, lambda: call(u=[U[0], U[0]] + U[2:]))              # U repeated
    expect(HB_ERR_INDEX_SET, lambda: call(u=U[:-1] + [len(ch.primes)]))        # U outside the chain


# ---- 4. code generation on sm_90a

def test_scaled_sums_kernel_has_no_local_array_stack_frame_or_spill(tmp_path):
    """k1_scaled_sums keeps its sums in registers and its inputs in shared memory: no local array in the PTX, and a
    (0, 0, 0) frame in `ptxas -v`."""
    nvcc = _nvcc()
    ptx = str(tmp_path / "hb_engine.ptx")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ptx",
                    os.path.join(CSRC, "hb_engine.cu"), "-o", ptx], check=True, capture_output=True, text=True)
    r = subprocess.run([os.path.join(os.path.dirname(nvcc), "ptxas"), "-arch=sm_90a", "-O3", "-v", ptx,
                        "-o", str(tmp_path / "hb_engine.cubin")], check=True, capture_output=True, text=True)
    mine = lambda k: re.match(r"_Z\d+k1_scaled_sums[A-Z]", k) is not None
    depots = {k: v for k, v in _depots(open(ptx).read()).items() if mine(k)}
    frames = {k: v for k, v in _frames(r.stdout + r.stderr).items() if mine(k)}
    assert len(frames) == 1, frames
    assert not depots, depots
    assert all(v == (0, 0, 0) for v in frames.values()), frames


# ---- 5. the C++ mirror (tests/cpp/test_poly_eval.cpp): hb::polyEval against the transcribed HElib code

def test_mirror_poly_eval_on_simulator():
    from test_cpp_shim import build_exe
    r = subprocess.run([build_exe("test_poly_eval", sim=True)], capture_output=True, text=True)
    assert r.returncode == 0 and "poly eval OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_poly_eval_on_gpu():
    """The same cases, and a degree-257 polynomial on BASELINE config 3's ring (m = 2^17, p = 257)."""
    from test_cpp_shim import build_exe
    r = subprocess.run([build_exe("test_poly_eval"), "full"], capture_output=True, text=True)
    assert r.returncode == 0 and "poly eval OK" in r.stdout and "config 3" in r.stdout, r.stdout + r.stderr
