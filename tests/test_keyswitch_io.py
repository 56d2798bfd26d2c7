"""Key-switching matrices held as b + prgSeed in the C++ mirror (tests/cpp/test_keyswitch_io.cpp): genKeySWmatrix(prgSeed)
against the byte-stream overload fed with the oracle's restatement of NTL's stream, the KeySwitch::writeTo / readFrom
round trip with a re-expanded on the device, relinearisation with the read-back matrix, and rejected records."""
import subprocess

import pytest

import ntl_prg_np as npg
from test_cpp_shim import build_exe
from prg_sim import drop_stale_sim_build

drop_stale_sim_build()

SEED = bytes.fromhex("7f3c19a2d05be8416c2e9db3f70815aa4c6e21d8930b5f7ee2a1c4d6089b3e51")


def _run(exe, tmp_path):
    # NTL's key stream for SEED, enough for both a_i of the m = 8192 chain (about 40 buffers per a_i)
    path = tmp_path / "stream.bin"
    path.write_bytes(npg.BufferStream(SEED).peek(400).tobytes())
    return subprocess.run([exe, SEED.hex(), str(path)], capture_output=True, text=True)


def test_keyswitch_seed_and_io_on_simulator(tmp_path):
    r = _run(build_exe("test_keyswitch_io", sim=True), tmp_path)
    assert r.returncode == 0 and "keyswitch io OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_keyswitch_seed_and_io_on_gpu(tmp_path):
    r = _run(build_exe("test_keyswitch_io"), tmp_path)
    assert r.returncode == 0 and "keyswitch io OK" in r.stdout, r.stdout + r.stderr
