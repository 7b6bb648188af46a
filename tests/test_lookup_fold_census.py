"""mdn_lookup_fold_census: every (instance, row, column) where a LogUp aux trace departs from the constraint-path fold of
its lookup program, listed in row order and tallied per column, without proving -- the census of mdn_check_lookup_folds.

Three implementations: the device kernels; the CPU oracle's handle-by-handle walk keeping every disagreement
(orc_lookup_fold_census, tests/oracle_fold_census); and `ref_census` below, built from the closed-form Python folds of
tests/test_lookup_folds.py.  The fixtures are those of tests/test_lookup_folds.py (the closed two-AIR bus), with single
faults and with traces that carry many faults at once.  The small -m gpu cases also run on the kernel emulator of
tests/emu (tests/test_lookup_fold_census_emulated.py)."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
import pkgload
import test_lookup_folds as TF
import test_trace_balance as TB

pkg = pkgload.load_pkg()
W, B = pkg.workload, pkg.binding
P, RND, ROOT = TB.P, TB.RND, TB.ROOT
ef_add, ef_mul, ef_inv, ef_sub = TB.ef_add, TB.ef_mul, TB.ef_inv, TF.ef_sub
gpu = pytest.mark.gpu
INFO_POOL = 9                                                           # MDN_INFO_POOL
ALL = 1 << 16


# ---------------------------------------------------------------------------------------------------------------------
# the census with Python integers, from the closed-form folds
# ---------------------------------------------------------------------------------------------------------------------
def ref_census(airs, rnd, marks, auxs, finals, max_failures=ALL, max_tallies=ALL):
    """(report, failures, tallies) as `census_tuple` gives them."""
    first = dict(holds=1, kind=0, instance=0, column=0, row=0, fold=(0,) * 4, expected=(0, 0), actual=(0, 0), failing_rows=0,
                 zero_u=0, n_skipped_airs=0)
    fails, tallies = [], []
    for i, a in enumerate(airs):
        if a["lookup"] is None:
            first["n_skipped_airs"] += 1
            continue
        folds = TF.ref_folds(a, rnd, marks[i])
        aux, n = auxs[i], len(folds)
        at = lambda r, c: tuple(int(x) for x in finals[i]) if r == n else (int(aux[r, 2 * c]), int(aux[r, 2 * c + 1]))
        cols = {}
        for r, row in enumerate(folds):
            zero = [u == (0, 0) for _, u in row]
            frac = [(0, 0) if z else ef_mul(v, ef_inv(u)) for (v, u), z in zip(row, zero)]
            total = (0, 0)
            for f in frac:
                total = ef_add(total, f)
            bad = False
            for c, (v, u) in enumerate(row):
                expected, actual = (frac[c], at(r, c)) if c else (total, ef_sub(at(r + 1, 0), at(r, 0)))
                kind = 3 if zero[c] else ((1 if c else 2) if expected != actual and (c or not any(zero)) else 0)
                if not kind:
                    continue
                bad = True
                fails.append((i, c, kind, r, v + u, expected, actual))
                t = cols.setdefault(c, [i, c, 0, 0, r, r, kind, expected, actual])
                t[2] += 1
                t[3] += kind == 3
                t[5] = r
            first["failing_rows"] += bad
        tallies += [tuple(cols[c]) for c in sorted(cols)]
    first["zero_u"] = sum(t[3] for t in tallies)
    if fails:
        i, c, kind, r, fold, expected, actual = fails[0]
        first.update(holds=0, kind=kind, instance=i, column=c, row=r, fold=fold, expected=expected, actual=actual)
    rep = dict(first=TB._norm(first), disagreements=len(fails), n_failures=min(len(fails), max_failures),
               failing_columns=len(tallies), n_tallies=min(len(tallies), max_tallies))
    return rep, fails[:max_failures], tallies[:max_tallies]


def census_tuple(out, fails, tallies):
    """A FoldCensus and its lists as plain Python values."""
    rep = dict(first=TB._norm(B.fold_report_dict(out.first)), disagreements=out.disagreements, n_failures=out.n_failures,
               failing_columns=out.failing_columns, n_tallies=out.n_tallies)
    fl = [(f.instance, f.column, f.kind, f.row, tuple(f.fold), tuple(f.expected), tuple(f.actual)) for f in fails]
    tl = [(t.instance, t.column, t.failing_rows, t.zero_u_rows, t.first_row, t.last_row, t.first_kind, tuple(t.first_expected),
           tuple(t.first_actual)) for t in tallies]
    return rep, fl, tl


def _raw(out, fails, tallies):
    """The bytes of everything a call returned."""
    return bytes(out) + b"".join(bytes(f) for f in fails) + b"".join(bytes(t) for t in tallies)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle (tests/oracle_fold_census/liboracle_fold_census.so)
# ---------------------------------------------------------------------------------------------------------------------
_ofc_lib = None


def _ofl():
    global _ofc_lib
    if _ofc_lib is None:
        d = os.path.join(ROOT, "tests", "oracle_fold_census")
        subprocess.check_call(["make", "-s", "-C", d])
        L = C.CDLL(os.path.join(d, "liboracle_fold_census.so"))
        L.orc_last_error.restype = C.c_char_p
        L.orc_lookup_fold_census.argtypes = [C.POINTER(ob.Statement), C.POINTER(ob.Matrix), ob.u64p, C.POINTER(ob.u32p),
                                             C.POINTER(ob.Matrix), C.POINTER(ob.u64p), C.POINTER(B.FoldFailure), C.c_uint64,
                                             C.POINTER(B.FoldTally), C.c_uint64, C.POINTER(B.FoldCensus)]
        L.orc_logup_aux.argtypes = [C.POINTER(ob.Statement), C.POINTER(ob.Matrix), ob.u64p, C.POINTER(ob.u64p), C.POINTER(ob.u64p)]
        _ofc_lib = L
    return _ofc_lib


def oracle_census(wl, rnd, marks, auxs, finals, max_failures=ALL, max_tallies=ALL):
    keep = []
    mats, fins = (ob.Matrix * wl.k)(), (ob.u64p * wl.k)()
    for i, a in enumerate(auxs):
        if a is not None:
            keep += [np.ascontiguousarray(a), np.array([int(x) for x in finals[i]], dtype=np.uint64)]
            mats[i] = ob.Matrix(ob.ptr(keep[-2]), wl.log_heights[i], a.shape[1])
            fins[i] = ob.ptr(keep[-1])
    out = B.FoldCensus()
    fails, tallies = (B.FoldFailure * max(1, max_failures))(), (B.FoldTally * max(1, max_tallies))()
    r = np.array(rnd, dtype=np.uint64)
    if _ofl().orc_lookup_fold_census(TB._cast(wl.statement, ob.Statement), TB._cast(wl.matrices, ob.Matrix), ob.ptr(r),
                                     TF._marks_arg(wl, marks, keep), mats, fins, fails, max_failures, tallies, max_tallies,
                                     C.byref(out)) != 0:
        raise RuntimeError(_ofl().orc_last_error().decode())
    return census_tuple(out, fails[: out.n_failures], tallies[: out.n_tallies])


def oracle_aux(wl, rnd):
    """The prover path's aux traces and closing values from the oracle (for traces too tall for ref_aux)."""
    auxs = [np.zeros((1 << wl.log_heights[i], 2 * wl.aux_widths[i]), dtype=np.uint64) if wl.aux_widths[i] else None for i in range(wl.k)]
    fins = [np.zeros(2, dtype=np.uint64) if a is not None else None for a in auxs]
    outs, fouts = (ob.u64p * wl.k)(), (ob.u64p * wl.k)()
    for i, a in enumerate(auxs):
        if a is not None:
            outs[i], fouts[i] = ob.ptr(a), ob.ptr(fins[i])
    r = np.array(rnd, dtype=np.uint64)
    if _ofl().orc_logup_aux(TB._cast(wl.statement, ob.Statement), TB._cast(wl.matrices, ob.Matrix), ob.ptr(r), outs, fouts) != 0:
        raise RuntimeError(_ofl().orc_last_error().decode())
    return auxs, [tuple(int(x) for x in f) if f is not None else None for f in fins]


# ---------------------------------------------------------------------------------------------------------------------
# traces with many faults at once
# ---------------------------------------------------------------------------------------------------------------------
def _bump(aux, r, word, by=1):
    aux[r, word] = (int(aux[r, word]) + by) % P


def multi(name):
    """(wl, marks, airs, auxs, finals); auxs is None where the case is checked on the device LogUp build (aux = NULL)."""
    bus, wl, marks, airs = TF.bus_case()
    auxs, finals = TF.all_aux(airs, RND)
    n = auxs[1].shape[0]
    rng = random.Random(name)
    if name == "column_2_every_row":               # one fraction column wrong throughout (a wrong encoding in one group)
        for r in range(n):
            _bump(auxs[1], r, 4)
    elif name == "column_0_shift":                 # the running sum off by a constant from row 37 on: one missing fraction
        for r in range(37, n):
            _bump(auxs[1], r, 0, 5)
        finals[1] = ((finals[1][0] + 5) % P, finals[1][1])
    elif name == "scattered":                      # flips in several columns of both lookup AIRs
        for r in rng.sample(range(auxs[0].shape[0]), 4):
            _bump(auxs[0], r, 1)
        for r in rng.sample(range(n), 12):
            _bump(auxs[1], r, rng.choice([0, 1, 2, 3, 4, 5]))
    elif name == "zero_u_and_fractions":           # zero denominators on rows 9, 21, 50 and kind 1 faults in column 1
        for r in (9, 21, 50):
            bus.sender[r, 9], bus.sender[r, 10] = 1, 0
        wl, marks, airs = TF.marked(bus)
        auxs, finals = TF.all_aux(airs, RND)
        for r in (3, 21, 77):
            _bump(auxs[1], r, 2)
    elif name == "boundary_rows":                  # row 0 of both AIRs, the last row and the closing value
        _bump(auxs[1], 0, 2)
        _bump(auxs[1], n - 1, 5)
        _bump(auxs[0], 0, 0)
        finals[0] = ((finals[0][0] + 1) % P, finals[0][1])
    elif name == "flags_two":                      # non-boolean flags on several rows, checked on the prover path
        for r in (5, 14, 63, 100):
            bus.sender[r, 2] = 2
        wl, marks, airs = TF.marked(bus)
        auxs, finals = TF.all_aux(airs, RND)
    else:
        raise KeyError(name)
    return wl, marks, airs, auxs, finals


MULTI = ["column_2_every_row", "column_0_shift", "scattered", "zero_u_and_fractions", "boundary_rows", "flags_two"]


def case(name):
    """(wl, marks, airs, auxs, finals, device aux: None when the device LogUp build is checked) of a single fault of
    tests/test_lookup_folds.py or of a multi-fault trace."""
    if name in TF.FAULTS:
        _, wl, marks, airs, auxs, finals, _ = TF.fault(name)
    else:
        wl, marks, airs, auxs, finals = multi(name)
    return wl, marks, airs, auxs, finals, name != "flags_two"


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle on the Python census
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", TF.FAULTS + MULTI)
def test_oracle_census_equals_the_python_census(name):
    wl, marks, airs, auxs, finals, _ = case(name)
    ref = ref_census(airs, RND, marks, auxs, finals)
    assert ref[0]["disagreements"] > 0 and ref[0]["first"]["holds"] == 0
    assert oracle_census(wl, RND, marks, auxs, finals) == ref
    # `first` is the fold check's report
    assert ref[0]["first"] == TB._norm(TF.ref_check(airs, RND, marks, auxs, finals))


def _ref(name):
    wl, marks, airs, auxs, finals, _ = case(name)
    return ref_census(airs, RND, marks, auxs, finals)


def test_the_multi_fault_cases_list_what_they_were_built_to_show():
    rep, fails, tallies = _ref("column_2_every_row")
    assert [(t[0], t[1], t[2]) for t in tallies] == [(1, 2, 1 << 7)] and rep["disagreements"] == 1 << 7
    _, fails, _ = _ref("column_0_shift")
    assert [(f[0], f[1], f[2], f[3]) for f in fails] == [(1, 0, 2, 36)]
    rep, fails, _ = _ref("zero_u_and_fractions")
    assert {(f[1], f[2], f[3]) for f in fails if f[3] in (9, 21, 50)} == {(2, 3, 9), (2, 3, 21), (1, 1, 21), (2, 3, 50)}
    assert rep["first"]["zero_u"] == 3 and {(f[1], f[3]) for f in fails if f[2] == 1} == {(1, 3), (1, 21), (1, 77)}
    _, fails, _ = _ref("boundary_rows")
    assert {(f[0], f[1], f[3]) for f in fails} == {(0, 0, 0), (0, 0, (1 << 5) - 1), (1, 1, 0), (1, 2, (1 << 7) - 1)}
    _, fails, _ = _ref("flags_two")
    assert {f[3] for f in fails} == {5, 14, 63, 100}


@pytest.mark.parametrize("name", ["scattered", "zero_u_and_fractions"])
def test_oracle_truncates_like_the_python_census(name):
    wl, marks, airs, auxs, finals, _ = case(name)
    full = ref_census(airs, RND, marks, auxs, finals)
    mf, mt = full[0]["disagreements"] - 3, full[0]["failing_columns"] - 1
    for f, t in ((mf, ALL), (ALL, mt), (mf, mt), (0, 0)):
        ref = ref_census(airs, RND, marks, auxs, finals, f, t)
        assert ref[0]["first"] == full[0]["first"] and ref[1] == full[1][:f] and ref[2] == full[2][:t]
        assert oracle_census(wl, RND, marks, auxs, finals, f, t) == ref


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def run(sess, wl, marks, mode="host", auxs=None, finals=None, max_failures=ALL, max_tallies=ALL, raw=False):
    mats, flags, keep = TB.traces_for(wl, mode)
    amats, akeep = TF.aux_for(wl, auxs, mode) if auxs is not None else (None, None)
    res = sess.lookup_fold_census(wl.statement, mats, RND, marks, amats, finals, flags, max_failures, max_tallies)
    return _raw(*res) if raw else census_tuple(*res)


@gpu
@pytest.mark.parametrize("mode", ["host", "device_rm", "device_cm"])
@pytest.mark.parametrize("name", TF.FAULTS + MULTI)
def test_device_census_equals_the_oracle_and_the_python_census(name, mode):
    wl, marks, airs, auxs, finals, explicit = case(name)
    got = run(TB.session(), wl, marks, mode, auxs if explicit else None, finals if explicit else None)
    assert got == ref_census(airs, RND, marks, auxs, finals)
    assert got == oracle_census(wl, RND, marks, auxs, finals)


@gpu
@pytest.mark.parametrize("name", ["scattered", "flags_two"])
def test_device_census_without_fold_marks(name):
    wl, marks, airs, auxs, finals, explicit = case(name)
    none = [None] * wl.k
    got = run(TB.session(), wl, None, "host", auxs if explicit else None, finals if explicit else None)
    assert got == ref_census(airs, RND, none, auxs, finals) == oracle_census(wl, RND, none, auxs, finals)


@gpu
def test_device_census_of_the_prover_path_holds_on_the_closed_bus():
    _, wl, marks, airs = TF.bus_case()
    rep, fails, tallies = run(TB.session(), wl, marks)
    assert rep["first"]["holds"] == 1 and rep["disagreements"] == 0 and fails == [] and tallies == []
    assert rep["first"]["n_skipped_airs"] == 1


@gpu
@pytest.mark.parametrize("mode", ["host", "device_cm"])
@pytest.mark.parametrize("name", TF.FAULTS + MULTI)
def test_first_is_the_fold_check_report(name, mode):
    wl, marks, airs, auxs, finals, explicit = case(name)
    a, f = (auxs, finals) if explicit else (None, None)
    got = run(TB.session(), wl, marks, mode, a, f)
    mats, flags, keep = TB.traces_for(wl, mode)
    amats, akeep = TF.aux_for(wl, a, mode) if a is not None else (None, None)
    assert got[0]["first"] == TB._norm(TB.session().check_lookup_folds(wl.statement, mats, RND, marks, amats, f, None, flags))


@gpu
@pytest.mark.parametrize("name", ["scattered", "zero_u_and_fractions", "column_2_every_row"])
def test_device_truncates_like_the_oracle_and_the_python_census(name):
    wl, marks, airs, auxs, finals, _ = case(name)
    full = ref_census(airs, RND, marks, auxs, finals)
    mf, mt = max(0, full[0]["disagreements"] - 3), max(0, full[0]["failing_columns"] - 1)
    for f, t in ((mf, ALL), (ALL, mt), (mf, mt), (0, 0), (1, 0)):
        got = run(TB.session(), wl, marks, "host", auxs, finals, f, t)
        assert got == ref_census(airs, RND, marks, auxs, finals, f, t) == oracle_census(wl, RND, marks, auxs, finals, f, t)


@gpu
def test_two_calls_give_byte_identical_outputs():
    for name in ("scattered", "column_2_every_row"):
        wl, marks, _, auxs, finals, _ = case(name)
        a = run(TB.session(), wl, marks, "host", auxs, finals, raw=True)
        b = run(TB.session(), wl, marks, "host", auxs, finals, raw=True)
        assert a == b


@gpu
def test_lookup_2_20_against_table_2_16_matches_the_oracle():
    bus = TB.Bus(log_t=16, log_l=20, seed=3, n_boundary=4)
    wl, marks, _ = TF.marked(bus)
    auxs, finals = oracle_aux(wl, RND)
    n = 1 << 20
    auxs[1][:, 2] = (auxs[1][:, 2] + np.uint64(1)) % np.uint64(P)          # column 1 wrong on every row: 2^20 disagreements
    rng = random.Random(20)
    for r in rng.sample(range(n), 1000):                                     # and about 1000 scattered faults in column 2
        _bump(auxs[1], r, 4)
    orc = oracle_census(wl, RND, marks, auxs, finals, 1 << 21, 64)
    assert orc[0]["disagreements"] == n + 1000 and orc[0]["failing_columns"] == 2
    for mode in ("host", "device_cm"):
        assert run(TB.session(), wl, marks, mode, auxs, finals, 1 << 21, 64) == orc
    assert run(TB.session(), wl, marks, "host", auxs, finals, 5000, 1) == oracle_census(wl, RND, marks, auxs, finals, 5000, 1)


@gpu
def test_error_paths_are_refused_and_launch_nothing():
    _, wl, marks, airs = TF.bus_case()
    auxs, finals = TF.all_aux(airs, RND)
    sess = B.Session(W.miden_pcs_params(), 0)
    run(sess, wl, marks)                          # the arena has its slabs from here on
    pool = sess.info(INFO_POOL).copy()
    keep = []

    def call(rnd=RND, marks=marks, auxs=auxs, finals=finals, flags=0, mf=ALL, mt=ALL, fails=True, tallies=True, out=True):
        amats, k = TF.aux_for(wl, auxs, "host") if auxs is not None else (None, None)
        keep.append(k)
        if fails and tallies and out:
            return sess.lookup_fold_census(wl.statement, wl.matrices, rnd, marks, amats, finals, flags, mf, mt)
        rnd_a, marks_a, fins_a, k2 = B._fold_inputs(wl.statement, rnd, marks, finals)
        keep.append(k2)
        rc = B.lib().mdn_lookup_fold_census(sess.handle, C.byref(wl.statement), wl.matrices, B.ptr(rnd_a), marks_a, amats, fins_a,
                                            flags, (B.FoldFailure * 4)() if fails else None, mf,
                                            (B.FoldTally * 4)() if tallies else None, mt, C.byref(B.FoldCensus()) if out else None)
        sess._check(rc)
    TB._expect_error(-1, lambda: call(fails=False, mf=4), "failures is NULL but max_failures is not 0")
    TB._expect_error(-1, lambda: call(tallies=False, mt=4), "tallies is NULL but max_tallies is not 0")
    TB._expect_error(-1, lambda: call(out=False, mf=4, mt=4), "null argument")
    TB._expect_error(-1, lambda: call(rnd=[P] + RND[1:]), "randomness word 0 is not a canonical")
    bad = [m.copy() if m is not None else None for m in marks]
    bad[1][0] = 1
    TB._expect_error(-1, lambda: call(marks=bad), "must open a group")
    bad[1][0], bad[1][4] = 3, 0
    TB._expect_error(-1, lambda: call(marks=bad), "do not share a flag node")
    TB._expect_error(-1, lambda: call(marks=[marks[0], marks[1], np.zeros(1, dtype=np.uint32)]), "without a lookup program")
    TB._expect_error(-1, lambda: call(auxs=None), "aux_finals given without aux")
    TB._expect_error(-1, lambda: call(finals=[finals[0], None, None]), "aux_finals is NULL")
    TB._expect_error(-1, lambda: call(auxs=[auxs[0], auxs[1][:, :4], None]), "the aux trace must be")
    TB._expect_error(-1, lambda: call(flags=B.FLAG_COLUMN_MAJOR), "MDN_FLAG_COLUMN_MAJOR is only valid")
    assert np.array_equal(sess.info(INFO_POOL), pool)
    # inside a staged proof: refused without disturbing it
    pw = W.Workload([10, 9, 8])
    obs = lambda c, f: B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(f, dtype=np.uint64)), len(f))
    ch = W.initial_challenger(W.miden_pcs_params(), obs)
    root, rnd = np.zeros(4, dtype=np.uint64), np.zeros(8, dtype=np.uint64)
    assert B.lib().mdn_prove_begin(sess.handle, C.byref(pw.statement), pw.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0
    staged_pool = sess.info(INFO_POOL).copy()
    TB._expect_error(-1, call, "mdn_lookup_fold_census called inside a proof")
    assert np.array_equal(sess.info(INFO_POOL), staged_pool)
    assert B.lib().mdn_prove_commit_aux(sess.handle, None, None, B.ptr(root)) == 0
    proof = B.Proof()
    assert B.lib().mdn_prove_finish(sess.handle, C.byref(proof)) == 0
    staged = B.proof_to_numpy(proof)
    fresh = B.Session(W.miden_pcs_params(), 0)
    ref = fresh.prove(pw.statement, pw.matrices, W.initial_challenger(W.miden_pcs_params(), obs))
    assert staged[0] == ref[0] and np.array_equal(staged[1], ref[1]) and np.array_equal(staged[2], ref[2])
    sess.close(); fresh.close()


@gpu
def test_proof_after_a_census_is_byte_identical():
    pw = W.Workload([10, 9, 8])
    params = W.miden_pcs_params()
    obs = lambda c, f: B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(f, dtype=np.uint64)), len(f))
    fresh = B.Session(params, 0)
    ref = fresh.prove(pw.statement, pw.matrices, W.initial_challenger(params, obs))
    a = B.Session(params, 0)
    before = a.prove(pw.statement, pw.matrices, W.initial_challenger(params, obs))
    t_before = (a.timings().total, a.timings().kernel_launches)
    info_before = a.info(0)
    wl, marks, _, auxs, finals, _ = case("scattered")
    run(a, wl, marks, "host", auxs, finals)
    run(a, wl, marks)
    assert (a.timings().total, a.timings().kernel_launches) == t_before and np.array_equal(a.info(0), info_before)
    after = a.prove(pw.statement, pw.matrices, W.initial_challenger(params, obs))
    for got in (before, after):
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])
    a.close(); fresh.close()


def test_new_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "miden_b200.h")).read()
    assert "int mdn_lookup_fold_census(" in header and "} mdn_fold_census_report;" in header
    assert "} mdn_fold_failure;" in header and "} mdn_fold_tally;" in header
    assert "mdn_lookup_fold_census" in B.EXPORTS
    assert C.sizeof(B.FoldFailure) == 88 and C.sizeof(B.FoldTally) == 80
    assert C.sizeof(B.FoldCensus) == C.sizeof(B.FoldReport) + 4 * 8


def test_oracle_aux_equals_the_python_prover_path():
    for name in ("fraction", "zero_denominator", "flag_two"):
        _, wl, _, airs, _, _, _ = TF.fault(name)
        auxs, finals = TF.all_aux(airs, RND)
        got, fins = oracle_aux(wl, RND)
        for i in (0, 1):
            assert np.array_equal(got[i], auxs[i]) and fins[i] == tuple(int(x) for x in finals[i])
