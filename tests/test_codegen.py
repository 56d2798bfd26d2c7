"""Code generation of the register-blocked transform kernels on sm_90a (CPU only: nvcc and ptxas need no GPU).

Every k1_* / k2_* transform kernel keeps its 16 residues and its twiddle pairs in registers; the whole design (DESIGN §4)
rests on that.  When the network loops are left to the unroller, the sm_90a front end keeps them partly rolled and puts
u64 a[16] and the twiddle array in local memory: a 256-864 byte stack frame in every transform kernel that `-Xptxas -v`
reports with zero spill bytes.  These tests compile the engine as build() does and fail if a hot kernel has a local array
in its PTX, or a stack frame or spill count above the allowance stated for it below."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "helib_b200", "csrc")
HOT = ("k1_fwd_blk", "k1_inv_blk", "k1_fwd_cols", "k1_inv_cols", "k1_conv", "k1_conv1", "k2_fwd_blk", "k2_inv_blk")

# Local arrays (PTX __local_depot bytes) allowed per kernel.  k1_conv: the quotient phase passes the addresses of two
# scalars (the sign of the exact CRT fallback, a call that is not inlined, and the optional x/Q fraction) -- 16 bytes
# outside the transform network.
DEPOT_ALLOW = {"k1_conv": 16}
# ptxas stack frame / spill bytes allowed per kernel (the larger of the SP = false / true instantiations).  The blk and
# cols kernels hold 32 registers of residues and 30 of second-pass twiddles under the 128-register cap of
# __launch_bounds__(256, 2); the k2 kernels and k1_conv run under a 96-register cap (576 / 640 threads per CTA).
# ptxas spills a few scalars at those caps; the stack frame of k1_conv also holds the registers saved around the call
# of its exact CRT fallback.
FRAME_ALLOW = {
    "k1_fwd_blk": (144, 144, 344),
    "k1_inv_blk": (104, 104, 104),
    "k1_fwd_cols": (24, 24, 24),
    "k1_inv_cols": (32, 32, 32),
    "k1_conv": (584, 64, 64),
    "k1_conv1": (0, 0, 0),
    "k2_fwd_blk": (192, 224, 252),
    "k2_inv_blk": (184, 196, 244),
}


def _nvcc():
    from helib_b200.build import _nvcc
    return _nvcc()


def _short(mangled):
    m = re.match(r"_Z\d+(k[12]_\w+?)I", mangled)
    return m.group(1) if m else None


@pytest.fixture(scope="module")
def engine_codegen(tmp_path_factory):
    """PTX and `ptxas -v` report of hb_engine.cu for sm_90a, compiled once per module (about half a minute)."""
    d = tmp_path_factory.mktemp("codegen")
    ptx = str(d / "hb_engine.ptx")
    nvcc = _nvcc()
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ptx",
                    os.path.join(CSRC, "hb_engine.cu"), "-o", ptx], check=True, capture_output=True, text=True)
    ptxas = os.path.join(os.path.dirname(nvcc), "ptxas")
    r = subprocess.run([ptxas, "-arch=sm_90a", "-O3", "-v", ptx, "-o", str(d / "hb_engine.cubin")],
                       check=True, capture_output=True, text=True)
    return open(ptx).read(), r.stdout + r.stderr


def _depots(ptx):
    """{mangled entry name: local depot bytes} for every kernel with a local array."""
    out = {}
    for m in re.finditer(r"\.entry (\w+)\(", ptx):
        end = ptx.find("\n}\n", m.end())
        body = ptx[m.end():end]
        sizes = [int(s) for s in re.findall(r"__local_depot\d+\[(\d+)\]", body)]
        if sizes:
            out[m.group(1)] = sum(sizes)
    return out


def _frames(report):
    """{mangled entry name: (stack frame, spill stores, spill loads)} from a `ptxas -v` report."""
    out, cur = {}, None
    for ln in report.splitlines():
        m = re.search(r"Function properties for (\w+)", ln)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and cur:
            out[cur] = tuple(int(x) for x in m.groups())
            cur = None
    return out


def test_every_hot_kernel_is_compiled(engine_codegen):
    _, report = engine_codegen
    names = {_short(k) for k in _frames(report)}
    for k in HOT:
        assert k in names, k


def test_no_local_arrays_in_transform_kernels(engine_codegen):
    ptx, _ = engine_codegen
    bad = {}
    for mangled, size in _depots(ptx).items():
        k = _short(mangled)
        if k in HOT and size > DEPOT_ALLOW.get(k, 0):
            bad[mangled] = size
    assert not bad, f"local arrays in the PTX of register-blocked kernels (bytes): {bad}"


def test_stack_frames_and_spills_within_allowance(engine_codegen):
    _, report = engine_codegen
    bad = {}
    for mangled, got in _frames(report).items():
        k = _short(mangled)
        if k in HOT and any(g > a for g, a in zip(got, FRAME_ALLOW[k])):
            bad[mangled] = (got, FRAME_ALLOW[k])
    assert not bad, f"(stack frame, spill stores, spill loads) above the allowance: {bad}"


def test_butterfly_microbenchmark_has_no_stack_frame(tmp_path):
    """bench_micro/ubench_butterfly.cu measures the network's ceiling: a stack frame there measures local memory instead."""
    nvcc = _nvcc()
    src = os.path.join(ROOT, "bench_micro", "ubench_butterfly.cu")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", "-Xptxas", "-v",
                        src, "-o", str(tmp_path / "ub.cubin")], check=True, capture_output=True, text=True)
    frames = {k: v for k, v in _frames(r.stdout + r.stderr).items() if re.match(r"_Z2kbILi\d", k)}
    assert len(frames) == 4
    assert all(v == (0, 0, 0) for v in frames.values()), frames
