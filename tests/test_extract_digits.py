"""Digit extraction on the device: the mirror's divideByP, multByP, extractDigits, extendExtractDigits and
extractDigitsThin (src/Ctxt.cpp:2415-2435, src/extractDigits.cpp, src/recryption.cpp:793-909).

Each round's subtract-and-divide chain and the thin final combination run as one hb_ctxt_scaled_sums call; they must equal
the transcribed step-by-step loops bit for bit, metadata included, and decrypt to the base-p digits of the slots
(tests/cpp/test_extract_digits.cpp).  The body runs on the CPU simulator build and, marked gpu, on the H100 with config 5's
and config 3's rings added."""
import subprocess

import pytest


def test_mirror_extract_digits_on_simulator():
    from test_cpp_shim import build_exe
    r = subprocess.run([build_exe("test_extract_digits", sim=True)], capture_output=True, text=True)
    assert r.returncode == 0 and "extract digits OK" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_mirror_extract_digits_on_gpu():
    """The same cases, and config 5's ring (m = 21845, p = 2) and config 3's (m = 2^17, p = 257)."""
    from test_cpp_shim import build_exe
    r = subprocess.run([build_exe("test_extract_digits"), "full"], capture_output=True, text=True)
    assert r.returncode == 0 and "extract digits OK" in r.stdout, r.stdout + r.stderr
    assert "config 5" in r.stdout and "config 3" in r.stdout, r.stdout
