"""The fallback of every NVRTC row pass, run on purpose.

MDN_JIT_FORCE_DISAGREE=1 makes every first-use comparison of an NVRTC-specialised kernel with the interpreter report a
disagreement, so each pass takes its real fallback: the interpreter's results are restored, the kernel is retired, the
pass's used flag is cleared and its note is set.  For each of the seven passes a set_jit(1) session under the variable
and a set_jit(0) session must give equal outputs on the same call, and a second call -- with the variable unset, so a
kernel left in use would run and set its flag -- must still be interpreted.  Both sides of a forced comparison hold
equal words, so these tests cannot show that a restore copies from the interpreter's side."""
import ctypes as C

import numpy as np
import pytest

import pkgload
import test_airs as TA
import test_check_constraints as TC
import test_constraint_census as TCC
import test_constraint_guard as TG
import test_device_resident as TDR
import test_lookup_fold_census as TFC
import test_lookup_folds as TF
import test_trace_balance as TB

pkg = pkgload.load_pkg()
W, B = pkg.workload, pkg.binding
gpu = pytest.mark.gpu
INFO_JIT, INFO_JIT_CHECK = 8, 11

PROOF = "NVRTC kernel disagreed with the interpreter on its first use; interpreter kept"
LOGUP = "NVRTC lookup kernel disagreed with the interpreter on its first use; interpreter kept"
CHECK = "NVRTC check kernel disagreed with the interpreter on its first use; interpreter kept"
LOOKUP_CHECK = "NVRTC lookup-check kernel disagreed with the interpreter on its first use; interpreter kept"


@pytest.fixture
def forced(monkeypatch):
    monkeypatch.setenv("MDN_JIT_FORCE_DISAGREE", "1")
    jit, interp = B.Session(W.fast_pcs_params(), 0), B.Session(W.fast_pcs_params(), 0)
    jit.set_jit(1)
    interp.set_jit(0)
    yield jit, interp, monkeypatch
    jit.close(); interp.close()


def flags(s, what):
    return [int(x) for x in s.info(what)]


def note(s):
    """the session's latest JIT note"""
    return s.jit_status().split("; ", 1)[1] if "; " in s.jit_status() else ""


def staged_proof(s, wl, params, aux_fn=None):
    """mdn_prove_begin / commit_aux (the device LogUp build, or test_constraint_guard.staged_aux's aux_fn, then the
    guard) / finish: the note after commit_aux, the proof, and the proof's kernel launches"""
    L = B.lib()
    m = max(wl._airs[i].num_randomness for i in range(wl.k))
    rnd = np.zeros(max(1, 2 * m), dtype=np.uint64)
    ch = TC.seed(params)
    assert L.mdn_prove_begin(s.handle, C.byref(wl.statement), wl.matrices, C.byref(ch), 0, B.ptr(np.zeros(4, dtype=np.uint64)), B.ptr(rnd)) == 0
    aux, vals = aux_fn([int(x) for x in rnd[: 2 * m]]) if aux_fn is not None else (None, None)
    assert L.mdn_prove_commit_aux(s.handle, aux, vals, B.ptr(np.zeros(4, dtype=np.uint64))) == 0, L.mdn_last_error(s.handle)
    logup_note = note(s)
    pf = B.Proof()
    assert L.mdn_prove_finish(s.handle, C.byref(pf)) == 0, L.mdn_last_error(s.handle)
    return logup_note, B.proof_to_numpy(pf), s.timings().kernel_launches


@gpu
def test_constraint_evaluation_and_logup_build(forced):
    jit, interp, mp = forced
    params = W.fast_pcs_params()
    wl, _ = TA.logup_workload(7, device=True)
    logup_note, got, _ = staged_proof(jit, wl, params)
    assert logup_note == LOGUP, jit.jit_status()
    assert flags(jit, INFO_JIT) == [0] * wl.k and note(jit) == PROOF, jit.jit_status()
    _, want, launches = staged_proof(interp, wl, params)
    assert TDR.same(got, want)
    mp.delenv("MDN_JIT_FORCE_DISAGREE")
    _, again, again_launches = staged_proof(jit, wl, params)
    assert TDR.same(again, want) and flags(jit, INFO_JIT) == [0] * wl.k
    assert again_launches == launches   # neither the constraint nor the LogUp kernel runs again


def census_call(s, wl, params, bld, mf, mt):
    cb = B.AUX_BUILDER(bld) if bld is not None else None
    c, f, t, _ = s.constraint_census(wl.statement, wl.matrices, TC.seed(params), aux_builder=cb, max_failures=mf, max_tallies=mt)
    return TCC.census_dict(c, f, t)


def check_call(s, wl, params, bld):
    cb = B.AUX_BUILDER(bld) if bld is not None else None
    rep, _ = s.check_constraints(wl.statement, wl.matrices, TC.seed(params), aux_builder=cb)
    return TC.report_dict(rep)


@gpu
@pytest.mark.parametrize("which", ["check", "census"])
def test_constraint_check_and_census(forced, which):
    jit, interp, mp = forced
    params = W.fast_pcs_params()
    wl, bld, _, _ = TCC.any_case("one_cell")
    run = (lambda s, mf, mt: check_call(s, wl, params, bld)) if which == "check" else \
          (lambda s, mf, mt: census_call(s, wl, params, bld, mf, mt))
    got = run(jit, 1 << 16, 1 << 16)
    assert flags(jit, INFO_JIT_CHECK) == [0] * wl.k and note(jit) == CHECK, jit.jit_status()
    assert got == run(interp, 1 << 16, 1 << 16)
    mp.delenv("MDN_JIT_FORCE_DISAGREE")
    assert run(jit, 3, 2) == run(interp, 3, 2)                   # truncated lists, for the census
    assert flags(jit, INFO_JIT_CHECK) == [0] * wl.k


@gpu
def test_guard(monkeypatch):
    """the check pass inside a guarded proof, which runs in commit_aux"""
    monkeypatch.setenv("MDN_JIT_FORCE_DISAGREE", "1")
    params = W.fast_pcs_params()
    wl, bld = TA.fib_product_workload([5, 6])
    jit, interp = TG.hash_session(params, guard=True), TG.hash_session(params, guard=True)
    jit.set_jit(1); interp.set_jit(0)
    try:
        guard_note, got, _ = staged_proof(jit, wl, params, TG.staged_aux(wl, bld))
        assert flags(jit, INFO_JIT_CHECK) == [0] * wl.k and guard_note == CHECK, jit.jit_status()
        _, want, _ = staged_proof(interp, wl, params, TG.staged_aux(wl, bld))
        assert TDR.same(got, want)
        monkeypatch.delenv("MDN_JIT_FORCE_DISAGREE")
        assert TDR.same(staged_proof(jit, wl, params, TG.staged_aux(wl, bld))[1], want)
        assert flags(jit, INFO_JIT_CHECK) == [0] * wl.k
    finally:
        jit.close(); interp.close()


@gpu
def test_balance(forced):
    jit, interp, mp = forced
    bus, bnd, _, _ = TB.case("mutex")
    wl, sites, _ = bus.workload()
    mats, fl, keep = TB.traces_for(wl, "host")
    call = lambda s, maxc: s.check_trace_balance(wl.statement, mats, TB.RND, bnd, sites, maxc, fl)
    got = call(jit, 1 << 16)
    assert flags(jit, B.INFO_JIT_LOOKUP_CHECK) == [0] * wl.k and note(jit) == LOOKUP_CHECK, jit.jit_status()
    assert got == call(interp, 1 << 16)
    mp.delenv("MDN_JIT_FORCE_DISAGREE")
    assert call(jit, 1) == call(interp, 1)
    assert flags(jit, B.INFO_JIT_LOOKUP_CHECK) == [0] * wl.k


@gpu
def test_folds(forced):
    jit, interp, mp = forced
    _, wl, marks, _, auxs, finals, _ = TF.fault("fraction")

    def call(s, given):
        rep, folds = TF.run(s, wl, marks, "host", auxs if given else None, finals if given else None, want_folds=True)
        return rep, [None if x is None else x.tobytes() for x in folds]
    got = call(jit, True)
    assert flags(jit, B.INFO_JIT_LOOKUP_CHECK) == [0] * wl.k and note(jit) == LOOKUP_CHECK, jit.jit_status()
    assert got == call(interp, True)
    mp.delenv("MDN_JIT_FORCE_DISAGREE")
    assert call(jit, False) == call(interp, False)                # the aux trace built on the device
    assert flags(jit, B.INFO_JIT_LOOKUP_CHECK) == [0] * wl.k


@gpu
def test_fold_census(forced):
    jit, interp, mp = forced
    wl, marks, _, auxs, finals, given = TFC.case("scattered")
    call = lambda s, mf, mt: TFC.run(s, wl, marks, "host", auxs if given else None, finals if given else None, mf, mt, raw=True)
    got = call(jit, TFC.ALL, TFC.ALL)
    assert flags(jit, B.INFO_JIT_LOOKUP_CHECK) == [0] * wl.k and note(jit) == LOOKUP_CHECK, jit.jit_status()
    assert got == call(interp, TFC.ALL, TFC.ALL)
    mp.delenv("MDN_JIT_FORCE_DISAGREE")
    assert call(jit, 3, 1) == call(interp, 3, 1)                  # truncated lists
    assert flags(jit, B.INFO_JIT_LOOKUP_CHECK) == [0] * wl.k
