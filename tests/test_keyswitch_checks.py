"""Argument checks of the hoisted rotation (hb_automorph_keyswitch_digits) on the CPU simulator build.

On a general-m ring the call runs its automorphisms before the key switch, so an argument error must be found before either:
a seeded matrix that lacks a row of S | special, and an S that holds a special prime (reported as HB_ERR_INDEX_SET, as the
linear maps report it), both return with nothing launched, on a power-of-two and on a general-m ring.
"""
import numpy as np
import pytest

import pyoracle as po
from common import chain
from helib_b200.engine import Engine, HbError

HB_ERR_INDEX_SET = -2


def _rand(ch, rng, idx, N):
    out = np.zeros((len(ch.primes), N), dtype=np.uint64)
    for i in idx:
        out[i] = rng.integers(0, ch.primes[i], size=N, dtype=np.uint64)
    return out


def _ring(sim_lib, m):
    if m & (m - 1) == 0:
        ch, psis = chain(m, 257, 1, 60, 2)
        return ch, Engine(ch.m, ch.primes, psis, ch.digits, ch.special, lib=sim_lib)
    ch = po.build_mod_chain(m, 2, 1, 120, 2)
    return ch, Engine(m, ch.primes, None, ch.digits, ch.special, lib=sim_lib)


@pytest.mark.parametrize("m,k", [(4096, 3), (105, 2)])
def test_hoisted_rotation_checks_before_launching(sim_lib, m, k):
    ch, E = _ring(sim_lib, m)
    rng = np.random.default_rng(2)
    nd = len(ch.digits)
    S, full = ch.ctxt, sorted(ch.ctxt + ch.special)
    short = E.seeded(nd, sorted(ch.ctxt[:-1] + ch.special), 3)    # lacks the top ctxt prime
    EA, EB = ([E.poly(_rand(ch, rng, full, E.N), full) for _ in range(nd)] for _ in range(2))
    digs = [[E.poly(_rand(ch, rng, full, E.N), full) for _ in range(nd)]]
    C0, O0, O1 = E.poly(_rand(ch, rng, S, E.N), S), E.poly(), E.poly()
    for S_, A in ((S, short), (S + ch.special[:1], EA)):
        E.sync()
        E.reset_stats()
        with pytest.raises(HbError) as ei:
            E.automorph_keyswitch_digits(digs, S_, [C0], k, A, EB, [O0], [O1])
        assert ei.value.code == HB_ERR_INDEX_SET, len(S_)
        assert E.stats()["launches"] == 0, len(S_)
    E.automorph_keyswitch_digits(digs, S, [C0], k, EA, EB, [O0], [O1])
    E.close()
