"""Constraint JIT (miden-vm_b200/csrc/jit.hpp): the lowering + NVRTC compile needs no device, so CPU CI checks
that every op of the vocabulary generates valid sm_90a code.  Execution parity is in test_gpu_parity.py."""
import numpy as np
import pytest

import helpers as H
import test_airs

B = H.B


def _check(prog):
    try:
        n = B.jit_compile_check(prog)
    except B.ProverError as e:
        if "NVRTC unavailable" in str(e):
            pytest.skip(str(e))
        raise
    assert n > 1000


def test_jit_compiles_every_leaf_kind():
    wl, _ = test_airs.fib_product_workload([5])                 # aux, challenges, publics, selectors, aux values
    _check(wl.programs[0])
    _check(test_airs.periodic_workload(5).programs[0])          # periodic columns
    _check(test_airs.preprocessed_workload().programs[0])       # preprocessed window
    wl, _ = test_airs.logup_workload(5)
    _check(wl.programs[0])                                      # mixed base/extension arithmetic
    _check(wl._lookups[0][1])                                   # lowered LookupAir -> generated row kernel


def test_jit_chunks_large_programs():
    # 2 k nodes -> several __noinline__ chunk functions with values spilled across them
    _check(test_airs.big_program_workload(5, n_terms=60).programs[0])


def test_jit_rejects_malformed_programs():
    good = test_airs.periodic_workload(5).programs[0]
    bad = good.copy(); bad[0] ^= 1
    with pytest.raises(B.ProverError):
        B.jit_compile_check(bad)
    bad = good.copy(); bad[5] = 99          # unknown op
    with pytest.raises(B.ProverError):
        B.jit_compile_check(bad)
    with pytest.raises(B.ProverError):
        B.jit_compile_check(good[:-1])
