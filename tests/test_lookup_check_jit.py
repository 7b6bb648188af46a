"""NVRTC-specialised lookup-check kernels (jit.hpp MODE_LOOKUP_CHECK: k_jit_balance, k_jit_fold, k_jit_fold_census)
against the op-list interpreter (k_balance_rows, k_fold_rows, k_fold_census_rows).

A session with set_jit(1) specialises every lookup program; one with set_jit(0) interprets every program.  On the same
calls the two must give equal mdn_check_trace_balance and mdn_check_lookup_folds reports (field by field, folds_out
included) and byte-equal mdn_lookup_fold_census outputs, truncated and not.  MDN_INFO_JIT_LOOKUP_CHECK (info 12) tells
which path ran.  The workloads and fault builders are those of tests/test_trace_balance.py, test_lookup_folds.py,
test_lookup_fold_census.py, test_lookup_preprocessed.py and test_lookup_registers.py; the Miden-shaped statement is the
one of tools/lookup_check_timing.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

import pkgload
import test_lookup_fold_census as TFC
import test_lookup_folds as TF
import test_lookup_preprocessed as TLP
import test_lookup_registers as TLR
import test_trace_balance as TB

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
P, RND = W.P, TB.RND
ROOT = pkgload.ROOT
gpu = pytest.mark.gpu
MODES = ["host", "device_rm", "device_cm"]
sys.path.insert(0, os.path.join(ROOT, "tools"))
import lookup_check_timing as LT  # noqa: E402


def new_pair():
    jit, interp = B.Session(W.fast_pcs_params(), 0), B.Session(W.fast_pcs_params(), 0)
    jit.set_jit(1)
    interp.set_jit(0)
    return jit, interp


@pytest.fixture(scope="module")
def pair():
    jit, interp = new_pair()
    yield jit, interp
    jit.close(); interp.close()


def used(s):
    return [int(x) for x in s.info(B.INFO_JIT_LOOKUP_CHECK)]


def lookups(wl):
    """info 12 of a session that specialised every lookup program: 1 for each AIR with one"""
    return [1 if wl.statement.airs[i].lookup else 0 for i in range(wl.k)]


def both(pair, fn):
    """fn(session) on the NVRTC session and the interpreter's; the results, and info 12 of each"""
    jit, interp = pair
    a, b = fn(jit), fn(interp)
    return a, b, used(jit), used(interp)


def same_balance(pair, wl, mats, flags, sites, bnd=()):
    for maxc in (1 << 16, 1):                       # contributions listed, and truncated
        a, b, uj, ui = both(pair, lambda s: s.check_trace_balance(wl.statement, mats, RND, bnd, sites, maxc, flags))
        assert a == b
        assert uj == lookups(wl) and ui == [0] * wl.k, (uj, ui)
    return a


def same_folds(pair, wl, marks, mode, auxs=None, finals=None):
    a, b, uj, ui = both(pair, lambda s: TF.run(s, wl, marks, mode, auxs, finals, want_folds=True))
    assert a[0] == b[0]
    assert len(a[1]) == len(b[1]) and all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a[1], b[1]))
    assert uj == lookups(wl) and ui == [0] * wl.k, (uj, ui)
    return a[0]


def same_census(pair, wl, marks, mode, auxs=None, finals=None):
    for mf, mt in ((TFC.ALL, TFC.ALL), (3, 1), (0, 0)):     # whole, truncated, counts only
        a, b, uj, ui = both(pair, lambda s: TFC.run(s, wl, marks, mode, auxs, finals, mf, mt, raw=True))
        assert a == b
        assert uj == lookups(wl) and ui == [0] * wl.k, (uj, ui)


# ---------------------------------------------------------------------------------------------------------------------
# the closed bus of tests/test_trace_balance.py and its faults
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", TB.CASES)
def test_balance_equals_the_interpreter(pair, name, mode):
    bus, bnd, _, _ = TB.case(name)
    wl, sites, _ = bus.workload()
    mats, flags, keep = TB.traces_for(wl, mode)
    rep = same_balance(pair, wl, mats, flags, sites, bnd)
    assert rep["holds"] == (name == "closed")
    same_balance(pair, wl, mats, flags, None, bnd)  # without mutex sites


@gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", TF.FAULTS)
def test_folds_equal_the_interpreter(pair, name, mode):
    _, wl, marks, _, auxs, finals, exp = TF.fault(name)
    rep = same_folds(pair, wl, marks, mode, auxs, finals)
    assert (rep["kind"], rep["instance"], rep["row"], rep["column"]) == exp[:4]
    same_folds(pair, wl, None, mode, auxs, finals)   # without marks: one group per interaction
    if name != "zero_denominator":                   # the device LogUp build refuses a zero denominator
        same_folds(pair, wl, marks, mode)


@gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", TF.FAULTS + TFC.MULTI)
def test_fold_census_equals_the_interpreter(pair, name, mode):
    wl, marks, _, auxs, finals, given = TFC.case(name)
    same_census(pair, wl, marks, mode, auxs if given else None, finals if given else None)
    same_census(pair, wl, None, mode, auxs if given else None, finals if given else None)


# ---------------------------------------------------------------------------------------------------------------------
# preprocessed reads, a version-2 program, a chunked program
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_preprocessed_reads(pair):
    case = TLP.Case(6, 9)
    for fault in (False, True):
        if fault:
            case.lut[20, 0] = (int(case.lut[20, 0]) + 2) % P
        wl = case.wl(True)
        for s in pair:
            TLP.install(s, wl)
        mats, flags, keep = TB.traces_for(wl, "host")
        assert same_balance(pair, wl, mats, flags, None)["holds"] == (not fault)
        same_folds(pair, wl, None, "host")
        same_census(pair, wl, None, "host")


@gpu
def test_version_2_program(pair):
    case = TLR.Case(7, 8)
    wl = case.wl(True)
    mats, flags, keep = TB.traces_for(wl, "host")
    assert same_balance(pair, wl, mats, flags, None)["holds"] == 1
    assert same_folds(pair, wl, None, "host")["holds"] == 1
    same_census(pair, wl, None, "host")
    full, fb, ffin = TLR.aux_matrices(case, wl, False)
    fb[TLR.STORE][9, 0] = (int(fb[TLR.STORE][9, 0]) + 1) % P
    a, b, uj, ui = both(pair, lambda s: s.check_lookup_folds(wl.statement, wl.matrices, RND, aux=full, aux_finals=ffin))
    assert a == b and a["holds"] == 0 and uj == lookups(wl)
    a, b, uj, ui = both(pair, lambda s: TFC._raw(*s.lookup_fold_census(wl.statement, wl.matrices, RND, aux=full, aux_finals=ffin)))
    assert a == b


@gpu
def test_chunked_program_with_spills(monkeypatch):
    """MDN_JIT_CHUNK=4 cuts the bus's lookup programs into many chunks whose values cross chunk boundaries."""
    monkeypatch.setenv("MDN_JIT_CHUNK", "4")
    pair = new_pair()
    try:
        for name in ("closed", "mutex", "flag"):
            bus, bnd, _, _ = TB.case(name)
            wl, sites, _ = bus.workload()
            mats, flags, keep = TB.traces_for(wl, "host")
            same_balance(pair, wl, mats, flags, sites, bnd)
        for name in ("fraction", "flag_two"):
            _, wl, marks, _, auxs, finals, _ = TF.fault(name)
            same_folds(pair, wl, marks, "host", auxs, finals)
            same_census(pair, wl, marks, "host", auxs, finals)
        assert "disagreed" not in pair[0].jit_status()
    finally:
        for s in pair:
            s.close()


# ---------------------------------------------------------------------------------------------------------------------
# the Miden-shaped statement of tools/lookup_check_timing.py
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("log_n", [16, 20])
@pytest.mark.parametrize("fault", [None, "scattered", "whole"])
def test_miden_shaped(pair, log_n, fault):
    wl, sites, marks = LT.statement(W, AP, P, log_n, fault)
    assert int(wl.statement.airs[0].lookup.contents.program[2]) >= 2000
    mats, flags, keep = TB.traces_for(wl, "host")
    rep = same_balance(pair, wl, mats, flags, sites)
    assert rep["holds"] == (fault is None)
    rep = same_folds(pair, wl, marks, "host")
    assert rep["holds"] == (fault is None)
    for mf, mt in ((TFC.ALL, TFC.ALL), (5, 2)):
        a, b, uj, ui = both(pair, lambda s: TFC._raw(*s.lookup_fold_census(wl.statement, mats, RND, marks, flags=flags,
                                                                           max_failures=mf, max_tallies=mt)))
        assert a == b and uj == [1, 1] and ui == [0, 0]
    assert "disagreed" not in pair[0].jit_status(), pair[0].jit_status()


@gpu
def test_self_check_with_torch_bundled_nvrtc():
    """tests/run_lookup_check_jit_old_nvrtc.py: torch's older NVRTC on the Miden-shaped program through the three checks."""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "run_lookup_check_jit_old_nvrtc.py")], capture_output=True,
                       text=True, timeout=1800, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "SELF-CHECK OK" in r.stdout or "NOTE" in r.stdout or "SKIP" in r.stdout, r.stdout[-3000:]
