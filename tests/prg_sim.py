"""Keeps the simulator build current for the seeded-expansion tests.

conftest.build_sim rebuilds tests/cusim/libhelib_b200_sim.so when a source it lists is newer than the library.
helib_b200/csrc/hb_device_prg.cuh, which hb_engine.cu includes, is not in that list, so an edit to it alone would leave the
simulator running the old kernels.  The test modules that exercise it call drop_stale_sim_build() at import: collection
happens before any test loads the library, and build_sim then compiles a current one."""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM_LIB = os.path.join(ROOT, "tests", "cusim", "libhelib_b200_sim.so")
PRG_HEADER = os.path.join(ROOT, "helib_b200", "csrc", "hb_device_prg.cuh")


def drop_stale_sim_build():
    if os.path.exists(SIM_LIB) and os.path.getmtime(PRG_HEADER) > os.path.getmtime(SIM_LIB):
        os.remove(SIM_LIB)
