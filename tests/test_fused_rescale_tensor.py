"""The operands' rescale fused with the tensor product (k1_fwd_blk_tensor) inside hb_mul_relin_moddown.

On the register kernels (power-of-two m, N >= 2^12) a multiplication that drops primes runs the forward blk phase of its
four operand parts in one pass that also forms the tensor product; everything else keeps the separate rescale and
tensor kernels.  Results must equal the oracle's scaleDownToSet + tensorProduct + reLinearize + modDownToSet bit for bit,
and the launch profile shows which path ran.  Every body runs on the simulator and (-m gpu) on the H100; the code
generation of the kernel is checked on sm_90a without a GPU."""
import os
import subprocess

import numpy as np
import pytest

import pyoracle as po
from common import make, ptxt_space, rows_equal
from helib_b200.engine import Engine
from test_codegen import CSRC, _depots, _frames, _nvcc, _short
from test_engine_parity import oracle_mul_relin_moddown


def test_fused_kernel_has_no_local_array_stack_frame_or_spill(tmp_path):
    """k1_fwd_blk_tensor holds its 16 residues and second-pass twiddles in registers and the results of the earlier parts in
    shared memory: both instantiations must have no local array in the PTX and no stack frame or spill in `ptxas -v`."""
    nvcc = _nvcc()
    ptx = str(tmp_path / "hb_engine.ptx")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ptx",
                    os.path.join(CSRC, "hb_engine.cu"), "-o", ptx], check=True, capture_output=True, text=True)
    r = subprocess.run([os.path.join(os.path.dirname(nvcc), "ptxas"), "-arch=sm_90a", "-O3", "-v", ptx,
                        "-o", str(tmp_path / "hb_engine.cubin")], check=True, capture_output=True, text=True)
    text = open(ptx).read()
    depots = {k: v for k, v in _depots(text).items() if _short(k) == "k1_fwd_blk_tensor"}
    frames = {k: v for k, v in _frames(r.stdout + r.stderr).items() if _short(k) == "k1_fwd_blk_tensor"}
    assert len(frames) == 2, frames                      # SP = false / true
    assert not depots, depots
    assert all(v == (0, 0, 0) for v in frames.values()), frames


def backends():
    return [pytest.param("sim", id="sim"), pytest.param("cuda", id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(params=backends())
def lib(request):
    return request.getfixturevalue("sim_lib" if request.param == "sim" else "cuda_lib")


def keys(O, E, ch, rng):
    full = ch.ctxt + ch.special
    nd = len(ch.digits)
    evk_a = np.stack([O.random(rng, full) for _ in range(nd)])
    evk_b = np.stack([O.random(rng, full) for _ in range(nd)])
    return evk_a, evk_b, [E.poly(evk_a[i], full) for i in range(nd)], [E.poly(evk_b[i], full) for i in range(nd)]


def run(E, O, ch, rng, S_in, S, p, nitems, check=None):
    """mul_relin_moddown of nitems random pairs with profiling on; returns the kernel names that ran.  check: the items
    compared against the oracle (all by default)."""
    evk_a, evk_b, EA, EB = keys(O, E, ch, rng)
    ops = [[O.random(rng, S_in) for _ in range(4)] for _ in range(nitems)]
    A0, A1, B0, B1 = ([E.poly(o[k], S_in) for o in ops] for k in range(4))
    E.profile(True)
    E.mul_relin_moddown(A0, A1, B0, B1, S_in, S, p, EA, EB)
    E.profile(False)
    for it in (range(nitems) if check is None else check):
        r0, r1 = oracle_mul_relin_moddown(O, ch, *ops[it], S_in, S, p, evk_a, evk_b)
        assert rows_equal(A0[it].download(S), r0, S) and rows_equal(A1[it].download(S), r1, S), it
    return {r["kernel"] for r in E.profile_results()}


@pytest.mark.parametrize("cfg, ndrop", [
    ((8192, -1, 1, 119, 2), 1),          # CKKS, N = 4096: generic conversion, then the fused pass
    ((1 << 17, 257, 1, 230, 2), 1),      # BGV p = 257, N = 2^16: k1_conv with the plaintext correction
    ((8192, -1, 1, 200, 2), 2),          # two primes dropped
    ((1 << 17, -1, 1, 330, 3), 2),       # two primes dropped at N = 2^16: k1_conv
], ids=["ckks-n4096", "bgv-n65536", "drop2-n4096", "drop2-n65536"])
def test_fused_path_matches_oracle(lib, cfg, ndrop):
    ch, psis, O, E = make(lib, *cfg, nthreads=8)
    rng = np.random.default_rng(101)
    S_in = ch.ctxt
    S = ch.ctxt[:-ndrop]
    ran = run(E, O, ch, rng, S_in, S, ptxt_space(ch), 2)
    assert "k1_fwd_blk_tensor" in ran and "k1_tensor" not in ran, ran


def test_fused_path_over_several_chunks(sim_lib, monkeypatch):
    """HB_CHUNK = 8 parts per launch: two pairs per chunk, so three pairs take two conversion + fused launches."""
    monkeypatch.setenv("HB_CHUNK", "8")
    ch, psis, O, E = make(sim_lib, 8192, -1, 1, 119, 2)
    rng = np.random.default_rng(102)
    ran = run(E, O, ch, rng, ch.ctxt, ch.ctxt[:-1], 1, 3)
    assert "k1_fwd_blk_tensor" in ran, ran
    st = {r["kernel"]: r["launches"] for r in E.profile_results()}
    assert st["k1_fwd_blk_tensor"] == 2, st


def test_nothing_dropped_keeps_the_tensor_kernel(lib):
    """S == S_in: no rescale, the tensor product runs alone in k1_tensor."""
    ch, psis, O, E = make(lib, 8192, -1, 1, 119, 2)
    rng = np.random.default_rng(103)
    ran = run(E, O, ch, rng, ch.ctxt, ch.ctxt, 1, 2)
    assert "k1_tensor" in ran and "k1_fwd_blk_tensor" not in ran, ran


def test_general_m_keeps_the_separate_kernels(sim_lib):
    """General m (Bluestein rows): the rescale and the tensor product stay separate launches (the results of this path
    are checked in test_general_m.py; here only the kernel selection)."""
    ch = po.build_mod_chain(105, 2, 1, 120, 2)
    E = Engine(105, ch.primes, None, ch.digits, ch.special, lib=sim_lib)
    rng = np.random.default_rng(104)
    full = ch.ctxt + ch.special

    def rand(idx):
        out = np.zeros((len(ch.primes), ch.phim), dtype=np.uint64)
        for i in idx:
            out[i] = rng.integers(0, ch.primes[i], size=ch.phim, dtype=np.uint64)
        return E.poly(out, idx)

    EA = [rand(full) for _ in ch.digits]
    EB = [rand(full) for _ in ch.digits]
    A0, A1, B0, B1 = ([rand(ch.ctxt)] for _ in range(4))
    E.profile(True)
    E.mul_relin_moddown(A0, A1, B0, B1, ch.ctxt, ch.ctxt[:-1], 2, EA, EB)
    E.profile(False)
    ran = {r["kernel"] for r in E.profile_results()}
    assert "k1_fwd_blk_tensor" not in ran and "k_pw_tensor" in ran, ran


@pytest.mark.gpu
def test_full_size_config2_batch_over_one_chunk(cuda_lib):
    """BASELINE config 2 (m = 2^17, 20 ctxt primes, CKKS) with 17 pairs: more than the 16 pairs of one chunk.  The pairs
    at the chunk edges (0, 15, 16) are checked against the oracle."""
    ch, psis, O, E = make(cuda_lib, 1 << 17, -1, 1, 1190, 2, nthreads=8)
    assert len(ch.ctxt) == 20
    rng = np.random.default_rng(105)
    ran = run(E, O, ch, rng, ch.ctxt, ch.ctxt[:-1], 1, 17, check=(0, 15, 16))
    assert "k1_fwd_blk_tensor" in ran and "k1_tensor" not in ran, ran
    st = {r["kernel"]: r["launches"] for r in E.profile_results()}
    assert st["k1_fwd_blk_tensor"] == 2, st
