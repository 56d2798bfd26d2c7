"""Code generation of the seeded-expansion kernels on sm_90a (CPU only).  k_prg_count / k_prg_fill keep the ChaCha20 state
in registers (named scalars) and read candidates back through shared memory: no local array in their PTX, no stack frame
and no spills in the `ptxas -v` report of the engine compiled as build() compiles it."""
import re

from test_codegen import _depots, _frames, engine_codegen  # noqa: F401  (module-scoped compile fixture)

PRG = ("k_prg_count", "k_prg_fill")


def _name(mangled):
    m = re.match(r"_Z\d+(k_prg_\w+?)\d", mangled)
    return m.group(1) if m else None


def test_prg_kernels_keep_their_state_in_registers(engine_codegen):
    ptx, report = engine_codegen
    frames = {_name(k): v for k, v in _frames(report).items() if _name(k)}
    assert set(frames) == set(PRG), frames
    assert all(v == (0, 0, 0) for v in frames.values()), frames
    depots = {k: v for k, v in _depots(ptx).items() if _name(k)}
    assert not depots, depots
