"""mdn_constraint_census: every violated AIR constraint of a statement, per constraint and in row order, without proving.

Two references besides the device:
  * `ref_census` below: a reduction over `test_check_constraints.constraint_rows` (the Python-integer evaluation of the
    op-list, row by row, constraints in emission order) with that file's challenges and aux traces;
  * the CPU oracle's census, orc_constraint_census (tests/oracle_census: the oracle's constraint checker keeping every
    violation).
The CPU tests pin the oracle on `ref_census`; the -m gpu tests require device = oracle = Python, field for field and in
order, and `census.first` = mdn_check_constraints' report of the same call.  The small -m gpu cases also run on the
kernel emulator (tests/test_constraint_census_emulated.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import helpers as H
import oracle_binding as ob
import pkgload
import test_airs as TA
import test_check_constraints as TC
import test_device_resident as TD

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
P = W.P
ROOT = pkgload.ROOT
gpu = pytest.mark.gpu
ALL = 1 << 40      # a capacity no case reaches


# ---------------------------------------------------------------------------------------------------------------------
# reference: a reduction over constraint_rows
# ---------------------------------------------------------------------------------------------------------------------
def ref_census(instances, publics, challenges, ext_failed=None, max_failures=ALL, max_tallies=ALL):
    """The census as a dict: first (the report of ref_check), violations, failing_constraints, failures [(instance,
    constraint, row, (c0, c1))] and tallies [(instance, constraint, failing_rows, first_row, last_row, first_value)]."""
    first = TC.ref_check(instances, publics, challenges, ext_failed)
    failures, tallies = [], []
    for i, a in enumerate(instances):
        t = {}
        for r, vals in enumerate(TC.constraint_rows(a["prog"], a["main"], a["aux"], a["aux_values"], publics, challenges,
                                                    a["periodic"], a["prep"])):
            for k, v in enumerate(vals):
                if v == (0, 0):
                    continue
                failures.append((i, k, r, v))
                if k not in t:
                    t[k] = [0, r, r, v]
                t[k][0] += 1
                t[k][2] = r
        tallies += [(i, k, n, lo, hi, v) for k, (n, lo, hi, v) in sorted(t.items())]
    return dict(first=first, violations=len(failures), failing_constraints=len(tallies),
                failures=failures[:max_failures], tallies=tallies[:max_tallies])


def instances_of(wl, params, builder=None):
    """(instances, challenges) as test_check_constraints.reference builds them."""
    chal = TC.oracle_challenges(wl, params)
    inst = []
    for i in range(wl.k):
        a = wl._airs[i]
        if builder is not None:
            aux, vals = TC.run_builder(builder, wl, i, chal)
        else:
            aux = np.zeros((1 << wl.log_heights[i]) * 2 * a.aux_width, dtype=np.uint64)
            vals = np.zeros(2 * a.num_aux_values, dtype=np.uint64)
        per = None
        if a.num_periodic_columns:
            per = np.ctypeslib.as_array(a.periodic_values, shape=((1 << a.log_max_period) * a.num_periodic_columns,))
            per = per.reshape(1 << a.log_max_period, a.num_periodic_columns)
        prep = wl.preprocessed[i] if wl.preprocessed is not None else None
        inst.append(dict(prog=wl.programs[i], main=wl.traces[i], aux=aux, aux_values=vals, periodic=per, prep=prep))
    return inst, chal


def reference(wl, params, builder=None, ext=None, **kw):
    inst, chal = instances_of(wl, params, builder)
    ext_failed = None
    if ext is not None:
        k = ext(np.array(chal, dtype=np.uint64), [np.asarray(d["aux_values"], dtype=np.uint64) for d in inst], bytes(wl.log_heights))
        ext_failed = None if k is None or k < 0 else k
    return ref_census(inst, wl.public_values, chal, ext_failed, **kw)


def census_dict(c, failures, tallies):
    return dict(first=TC.report_dict(c.first), violations=c.violations, failing_constraints=c.failing_constraints,
                failures=[(f.instance, f.constraint, f.row, (f.value[0], f.value[1])) for f in failures],
                tallies=[(t.instance, t.constraint, t.failing_rows, t.first_row, t.last_row, (t.first_value[0], t.first_value[1]))
                         for t in tallies])


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's census (tests/oracle_census/liboracle_census.so)
# ---------------------------------------------------------------------------------------------------------------------
class OrcCensus(C.Structure):
    _fields_ = B.ConstraintCensus._fields_


_lib = None


def _orc():
    global _lib
    if _lib is None:
        d = os.path.join(ROOT, "tests", "oracle_census")
        subprocess.check_call(["make", "-s", "-C", d])
        L = C.CDLL(os.path.join(d, "liboracle_census.so"))
        L.orc_last_error.restype = C.c_char_p
        L.orc_constraint_census.restype = C.c_int
        L.orc_constraint_census.argtypes = [C.POINTER(ob.Statement), C.POINTER(ob.Matrix), C.POINTER(ob.Matrix),
                                            C.POINTER(ob.Challenger), ob.AUX_BUILDER, C.c_void_p, B.EXTERNAL_CHECK, C.c_void_p,
                                            ob.u64p, C.POINTER(B.ConstraintFailure), C.c_uint64, C.POINTER(B.ConstraintTally),
                                            C.c_uint64, C.POINTER(OrcCensus)]
        _lib = L
    return _lib


def oracle_census(wl, params, builder=None, ext=None, max_failures=1 << 16, max_tallies=1 << 16):
    L = _orc()
    ch = TC.seed(params)
    m = max(wl._airs[i].num_randomness for i in range(wl.k))
    rnd = np.zeros(max(1, 2 * m), dtype=np.uint64)
    out = OrcCensus()
    fails = (B.ConstraintFailure * max(1, max_failures))()
    tallies = (B.ConstraintTally * max(1, max_tallies))()
    cb = ob.AUX_BUILDER(builder) if builder is not None else C.cast(None, ob.AUX_BUILDER)
    ecb = TC._ext_callback(ext) if ext is not None else C.cast(None, B.EXTERNAL_CHECK)
    prep = H.cast(wl.preprocessed_matrices, ob.Matrix) if wl.preprocessed is not None else None
    rc = L.orc_constraint_census(H.cast(wl.statement, ob.Statement), H.cast(wl.matrices, ob.Matrix), prep, H.cast(ch, ob.Challenger),
                                 cb, None, ecb, None, ob.ptr(rnd), fails, max_failures, tallies, max_tallies, C.byref(out))
    if rc != 0:
        raise RuntimeError(L.orc_last_error().decode())
    return census_dict(out, fails[: out.n_failures], tallies[: out.n_tallies])


# ---------------------------------------------------------------------------------------------------------------------
# multi-fault statements
# ---------------------------------------------------------------------------------------------------------------------
def _ext_fail(ch, av, lh):
    return 1


def _wide_program(n_cons):
    """n_cons constraints, constraint j = main[j mod 3] (base) or u * main[j mod 3] (extension, every 7th)."""
    b = AP.ProgramBuilder()
    for j in range(n_cons):
        x = b.main(0, j % 3)
        if j % 7 == 3:
            b.assert_zero_ext(b.ext_const(0, 1) * x)
        else:
            b.assert_zero(x)
    return b.serialize()


def multi_case(name):
    """(workload, host builder or None, external check or None) with several faults."""
    if name == "boundary_rows":                         # rows 0 and N-1: the selectors and the wrap to the next row
        wl, bld = TA.fib_product_workload([5])
        wl.traces[0][0, 0] = 5
        wl.traces[0][31, 2] = (int(wl.traces[0][31, 2]) + 1) % P
        return wl, bld, None
    if name == "one_cell":                              # the transitions into and out of row 17
        wl, bld = TA.fib_product_workload([6])
        wl.traces[0][17, 0] = (int(wl.traces[0][17, 0]) + 2) % P
        return wl, bld, None
    if name == "whole_column":                          # one constraint fails on every row, over many blocks
        wl = TC.dummy_workload([12])
        wl.traces[0][:, 0] = 3
        return wl, None, None
    if name == "two_heights":
        wl = TC.dummy_workload([7, 5])
        wl.traces[0][[3, 64, 127], 0] = 1
        wl.traces[1][[0, 9], 0] = 2
        return wl, None, None
    if name == "logup_main_cell":                       # device-built aux from a corrupted main trace
        wl, _ = TA.logup_workload(6, device=True)
        wl.traces[0][20, 4] = 2
        wl.traces[0][40, 5] = (int(wl.traces[0][40, 5]) + 1) % P
        return wl, None, None
    if name == "host_aux_cell":
        wl, bld = TA.fib_product_workload([5])
        return wl, TC._corrupt_aux(bld, 9, 0, 1), None
    if name == "external_and_rows":
        wl, bld = TA.fib_product_workload([5])
        wl.traces[0][6, 1] = 9
        return wl, bld, _ext_fail
    if name == "more_constraints_than_shared":          # 300 > CENSUS_SHARED_K: the global-atomic tally
        t = np.zeros((1 << 8, 3), dtype=np.uint64)
        t[[0, 5, 200], 0] = 4
        t[7, 1] = 1
        t[255, 2] = 6
        t[130:140, 1] = 2
        wl = W.Workload([8], widths=[3], aux_widths=[0], programs=[_wide_program(300)], traces=[t], log_quotient_degrees=[1],
                        num_aux_values=[0])
        return wl, None, None
    raise KeyError(name)


MULTI = ["boundary_rows", "one_cell", "whole_column", "two_heights", "logup_main_cell", "host_aux_cell", "external_and_rows",
         "more_constraints_than_shared"]


def any_case(name):
    """(workload, builder for the call, builder standing for the aux traces in the Python reference, external check)."""
    if name in TC.VALID:
        wl, bld = TC.valid_case(name)
        return wl, bld, TC.reference_builder(name, bld), None
    if name in TC.VIOLATIONS:
        wl, bld = TC.violation_case(name)
        return wl, bld, bld, None
    wl, bld, ext = multi_case(name)
    ref_bld = bld
    if name == "logup_main_cell":                       # the host twin of the device LogUp build, on the same traces
        ref_bld = TA.logup_workload(6, device=False)[1]
    return wl, bld, ref_bld, ext


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the layouts and the reference itself
# ---------------------------------------------------------------------------------------------------------------------
def test_struct_layouts():
    assert C.sizeof(B.ConstraintFailure) == 32 and C.sizeof(B.ConstraintTally) == 48
    assert [getattr(B.ConstraintFailure, f).offset for f in ("instance", "constraint", "row", "value")] == [0, 4, 8, 16]
    assert [getattr(B.ConstraintTally, f).offset for f in ("instance", "constraint", "failing_rows", "first_row", "last_row",
                                                            "first_value")] == [0, 4, 8, 16, 24, 32]
    assert C.sizeof(B.ConstraintCensus) == 48 + 32
    assert "mdn_constraint_census" in B.EXPORTS


def test_reference_on_hand_derived_faults():
    """fib/product constraints (test_check_constraints): 0 first*(a-p0), 1 first*(b-p1), 2 tr*(a'-b), 3 tr*(b'-(a+b)), ..."""
    params = W.fast_pcs_params()
    wl, bld, rb, _ = any_case("one_cell")               # a[17] += 2: a' = b fails at row 16, b' = a + b at row 17
    got = reference(wl, params, rb)
    assert [(f[1], f[2]) for f in got["failures"]] == [(2, 16), (3, 17)]
    wl, bld, rb, _ = any_case("whole_column")
    got = reference(wl, params, rb)
    n = 1 << 12
    assert got["tallies"][0][:5] == (0, 0, n, 0, n - 1) and got["first"]["failing_rows"] == n
    wl, bld, rb, _ = any_case("more_constraints_than_shared")
    got = reference(wl, params, rb)
    assert got["failing_constraints"] == 300 and got["first"]["failing_rows"] == 15


@pytest.mark.parametrize("name", TC.VALID + TC.VIOLATIONS + MULTI)
def test_oracle_census_agrees_with_python(name):
    params = W.fast_pcs_params()
    wl, bld, rb, ext = any_case(name)
    got = oracle_census(wl, params, bld, ext)
    want = reference(wl, params, rb, ext)
    assert got == want
    if name in TC.VALID:
        assert want["first"]["holds"] == 1 and want["violations"] == 0
    else:
        assert want["first"]["holds"] == 0
    if ext is None:
        assert sum(t[2] for t in want["tallies"]) == want["violations"]
        assert len({(f[0], f[2]) for f in want["failures"]}) == want["first"]["failing_rows"]


# ---------------------------------------------------------------------------------------------------------------------
# GPU (also run on the emulator, except the tests named h100)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sess():
    s = B.Session(W.fast_pcs_params(), 0)
    yield s
    s.close()


def device_census(sess, wl, params, bld=None, ext=None, max_failures=1 << 16, max_tallies=1 << 16, layout="host"):
    """(census dict, check_constraints report dict, randomness) of one call in one trace layout."""
    ch = TC.seed(params)
    prep = wl.preprocessed_matrices if wl.preprocessed is not None else None
    if ext is not None:
        sess.set_external_check(ext)
    try:
        if layout == "host":
            cb = B.AUX_BUILDER(bld) if bld is not None else None
            c, f, t, rnd = sess.constraint_census(wl.statement, wl.matrices, ch, aux_builder=cb, preprocessed=prep,
                                                  max_failures=max_failures, max_tallies=max_tallies)
            rep, rnd2 = sess.check_constraints(wl.statement, wl.matrices, ch, aux_builder=cb, preprocessed=prep)
        else:
            mats, bufs = TD.column_major_traces(wl)
            sess.set_device_aux_builder(TD.device_builder(wl, bld, bufs))
            try:
                c, f, t, rnd = sess.constraint_census(wl.statement, mats, ch, preprocessed=prep, flags=TD.CM,
                                                      max_failures=max_failures, max_tallies=max_tallies)
                rep, rnd2 = sess.check_constraints(wl.statement, mats, ch, preprocessed=prep, flags=TD.CM)
            finally:
                sess.set_device_aux_builder(None)
            for tr, b in zip(wl.traces, bufs):
                assert np.array_equal(TD.from_device(b), tr.T), "the caller's device trace changed"
    finally:
        if ext is not None:
            sess.set_external_check(None)
    assert np.array_equal(rnd, rnd2)
    return census_dict(c, f, t), TC.report_dict(rep), [int(x) for x in rnd]


def _row_major_device(sess, wl, params, **kw):
    mats, bufs = TD.row_major_device_traces(wl)
    c, f, t, rnd = sess.constraint_census(wl.statement, mats, TC.seed(params), flags=B.FLAG_DEVICE_TRACES, **kw)
    return census_dict(c, f, t)


@gpu
@pytest.mark.parametrize("name", TC.VALID + TC.VIOLATIONS + MULTI)
def test_census_matches_oracle_and_python(sess, name):
    params = W.fast_pcs_params()
    wl, bld, rb, ext = any_case(name)
    got, rep, rnd = device_census(sess, wl, params, bld, ext)
    want = reference(wl, params, rb, ext)
    assert got == want == oracle_census(wl, params, bld, ext)
    assert got["first"] == rep
    assert rnd == TC.oracle_challenges(wl, params)
    if name in TC.VALID:
        assert got["first"]["holds"] == 1 and got["violations"] == 0 and not got["failures"] and not got["tallies"]


@gpu
@pytest.mark.parametrize("name", ["two_heights", "logup_main_cell", "host_aux_cell", "more_constraints_than_shared",
                                  "periodic_value", "preprocessed_cell"])
def test_layouts_and_repeat_calls_agree(sess, name):
    """Host row-major, row-major device and column-major device traces give identical outputs; so do two calls."""
    params = W.fast_pcs_params()
    wl, bld, rb, ext = any_case(name)
    host, rep, _ = device_census(sess, wl, params, bld, ext)
    assert device_census(sess, wl, params, bld, ext)[0] == host
    assert device_census(sess, wl, params, bld, ext, layout="cm")[0] == host
    if bld is None and wl.preprocessed is None and ext is None:
        assert _row_major_device(sess, wl, params) == host
    assert host["violations"] > 0 and host["first"] == rep


@gpu
@pytest.mark.parametrize("name", ["more_constraints_than_shared", "boundary_rows", "two_in_one_row"])
def test_truncation(sess, name):
    """max_failures / max_tallies of 0, 1, exactly the total, and fewer than the first failing row's violations: the
    lists are prefixes of the full ones, the counts and `first` do not change."""
    params = W.fast_pcs_params()
    wl, bld, rb, ext = any_case(name)
    full, _, _ = device_census(sess, wl, params, bld, ext)
    v, fc = full["violations"], full["failing_constraints"]
    first_row = full["failures"][0][:1] + full["failures"][0][2:3]
    in_first_row = sum(1 for f in full["failures"] if (f[0], f[2]) == first_row)
    assert in_first_row >= 2
    for mf, mt in [(0, 0), (1, 1), (v, fc), (in_first_row - 1, fc - 1), (0, fc), (v, 0)]:
        got, _, _ = device_census(sess, wl, params, bld, ext, max_failures=mf, max_tallies=mt)
        assert got == dict(full, failures=full["failures"][:mf], tallies=full["tallies"][:mt])
        assert got == reference(wl, params, rb, ext, max_failures=mf, max_tallies=mt)
    assert oracle_census(wl, params, bld, ext, max_failures=1, max_tallies=1) == dict(full, failures=full["failures"][:1],
                                                                                      tallies=full["tallies"][:1])


@gpu
def test_error_paths_leave_the_session_usable(sess):
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    L = B.lib()
    wl0, bld0 = TA.fib_product_workload([5])
    want = sess.prove(wl0.statement, wl0.matrices, ch, aux_builder=B.AUX_BUILDER(bld0))

    def expect(rc, msg, fn):
        with pytest.raises(B.ProverError, match=msg) as e:
            fn()
        assert f"[{rc}]" in str(e.value)
        got = sess.prove(wl0.statement, wl0.matrices, ch, aux_builder=B.AUX_BUILDER(bld0))
        assert got[0] == want[0] and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])

    def raw(failures, max_failures, tallies, max_tallies, out=True):
        wl = TC.dummy_workload([5])
        o = B.ConstraintCensus()
        rc = L.mdn_constraint_census(sess.handle, C.byref(wl.statement), wl.matrices, None, C.byref(ch),
                                     C.cast(None, B.AUX_BUILDER), None, 0, None, failures, max_failures, tallies, max_tallies,
                                     C.byref(o) if out else None)
        if rc != 0:
            raise B.ProverError(f"[{rc}] {L.mdn_last_error(sess.handle).decode()}")

    f1, t1 = (B.ConstraintFailure * 1)(), (B.ConstraintTally * 1)()
    expect(-1, "failures is NULL", lambda: raw(None, 1, t1, 1))
    expect(-1, "tallies is NULL", lambda: raw(f1, 1, None, 1))
    expect(-1, "null argument", lambda: raw(f1, 1, t1, 1, out=False))
    wl = TC.dummy_workload([5])
    wl.traces[0][3, 2] = P
    expect(-1, "main trace contains a non-canonical", lambda: sess.constraint_census(wl.statement, wl.matrices, ch))
    wl = TA.preprocessed_workload((6, 8))
    expect(-1, "preprocessed presence mismatch", lambda: sess.constraint_census(wl.statement, wl.matrices, ch))
    wl = W.Workload([5], widths=[2], aux_widths=[0], programs=[TC._too_many_live_values()], log_quotient_degrees=[1], num_aux_values=[0])
    expect(-4, "live values", lambda: sess.constraint_census(wl.statement, wl.matrices, ch))
    wl = TC._zero_denominator_workload()
    expect(-1, "denominator must be non-zero", lambda: sess.constraint_census(wl.statement, wl.matrices, ch))
    wl, _ = TA.fib_product_workload([5])
    expect(-5, "aux builder failed", lambda: sess.constraint_census(wl.statement, wl.matrices, ch, aux_builder=B.AUX_BUILDER(lambda *a: 1)))

    def census_with_reduction_error():
        sess.set_external_check(TC._ext_raise)
        try:
            sess.constraint_census(wl0.statement, wl0.matrices, ch, aux_builder=B.AUX_BUILDER(bld0))
        finally:
            sess.set_external_check(None)
    expect(-7, "reduction error", census_with_reduction_error)


@gpu
def test_census_between_proofs_changes_nothing():
    """prove -> census -> prove: identical proof bytes, kernel launches, timings and introspection of the last proof."""
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    s = B.Session(params, 0)
    fresh = B.Session(params, 0)
    try:
        wl, bld = TA.fib_product_workload([6])
        cb = B.AUX_BUILDER(bld)
        p1 = s.prove(wl.statement, wl.matrices, ch, aux_builder=cb)
        launches1 = s.timings().kernel_launches
        t1 = TC._timings(s)
        info1 = [s.info(w).tolist() for w in (0, 1, 2, 3, 6, 7, 8)]
        bad, bbld, _, _ = any_case("one_cell")
        c, f, _, _ = s.constraint_census(bad.statement, bad.matrices, ch, aux_builder=B.AUX_BUILDER(bbld))
        assert c.first.holds == 0 and c.violations == 2 and len(f) == 2
        assert TC._timings(s) == t1
        assert [s.info(w).tolist() for w in (0, 1, 2, 3, 6, 7, 8)] == info1
        p2 = s.prove(wl.statement, wl.matrices, ch, aux_builder=cb)
        p3 = fresh.prove(wl.statement, wl.matrices, ch, aux_builder=cb)
        for q in (p2, p3):
            assert q[0] == p1[0] and np.array_equal(q[1], p1[1]) and np.array_equal(q[2], p1[2])
        assert s.timings().kernel_launches == launches1
    finally:
        s.close()
        fresh.close()


@gpu
def test_census_refused_inside_a_staged_proof():
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    wl = TC.dummy_workload([6, 5])
    s = B.Session(params, 0)
    try:
        want = s.prove(wl.statement, wl.matrices, ch)
        L = B.lib()
        root = np.zeros(4, dtype=np.uint64)
        rnd = np.zeros(4, dtype=np.uint64)
        assert L.mdn_prove_begin(s.handle, C.byref(wl.statement), wl.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0
        with pytest.raises(B.ProverError, match=r"\[-1\].*inside a proof"):
            s.constraint_census(wl.statement, wl.matrices, ch)
        assert L.mdn_prove_commit_aux(s.handle, None, None, None) == 0
        pf = B.Proof()
        assert L.mdn_prove_finish(s.handle, C.byref(pf)) == 0
        got = B.proof_to_numpy(pf)
        assert got[0] == want[0] and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
    finally:
        s.close()


def _miden_shape(fault):
    wl = W.Workload([20, 20, 20])
    if fault == "scattered":                            # about a thousand faults spread over the three AIRs
        rng = np.random.default_rng(20)
        for i, t in enumerate(wl.traces):
            rows = rng.choice(1 << 20, 333 + i, replace=False)
            t[rows, 0] = rng.integers(1, P, len(rows), dtype=np.uint64)
    elif fault == "column":                             # instance 1's constrained column wrong on every row
        wl.traces[1][:, 0] = 1
    return wl


@gpu
@pytest.mark.parametrize("fault", ["scattered", "column"])
def test_h100_miden_shape_2_20(fault):
    """The benchmark's statement (2^20 x (51, 22, 16)) with scattered faults and with a whole-column fault: GPU = oracle."""
    params = W.miden_pcs_params()
    s = B.Session(params, 0)
    try:
        wl = _miden_shape(fault)
        ch = W.initial_challenger(params, H.oracle_observe)
        c, f, t, dev_rnd = s.constraint_census(wl.statement, wl.matrices, ch, max_failures=1 << 12, max_tallies=64)
        got = census_dict(c, f, t)
        rep, _ = s.check_constraints(wl.statement, wl.matrices, ch)
        assert got["first"] == TC.report_dict(rep)
        L = _orc()
        m = max(wl._airs[i].num_randomness for i in range(wl.k))
        rnd = np.zeros(max(1, 2 * m), dtype=np.uint64)      # the oracle writes 2 * max num_randomness words
        o = OrcCensus()
        fo, to = (B.ConstraintFailure * (1 << 12))(), (B.ConstraintTally * 64)()
        assert L.orc_constraint_census(H.cast(wl.statement, ob.Statement), H.cast(wl.matrices, ob.Matrix), None, H.cast(ch, ob.Challenger),
                                       C.cast(None, ob.AUX_BUILDER), None, C.cast(None, B.EXTERNAL_CHECK), None, ob.ptr(rnd),
                                       fo, 1 << 12, to, 64, C.byref(o)) == 0
        assert got == census_dict(o, fo[: o.n_failures], to[: o.n_tallies])
        assert [int(x) for x in dev_rnd] == [int(x) for x in rnd]
        assert got["violations"] > 0 and sum(x[2] for x in got["tallies"]) == got["violations"]
        if fault == "column":
            assert got["tallies"][0][:5] == (1, 0, 1 << 20, 0, (1 << 20) - 1)
    finally:
        s.close()


def _cpp_census(target):
    d = os.path.join(ROOT, "tests", "cpp_census")
    if target.endswith("_emu"):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu")])
    subprocess.check_call(["make", "-s", "-C", d, target])
    r = subprocess.run([os.path.join(d, target)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "CENSUS_API_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@gpu
def test_h100_cpp_host_layer_constraint_census():
    """miden::constraint_census / ConstraintCensus (host/miden_prover.hpp) with the reference's panic texts."""
    _cpp_census("test_census_api")


def test_cpp_host_layer_constraint_census_on_the_emulator():
    _cpp_census("test_census_api_emu")


def test_census_refused_on_a_split_session_on_the_emulator():
    """A session split over 2 ranks refuses the census with MDN_ERR_UNSUPPORTED (tests/run_check_sharded.py's setup)."""
    import sys
    emu = os.path.join(ROOT, "tests", "emu")
    subprocess.check_call(["make", "-s", "-C", emu])
    env = dict(os.environ, MDN_LIB_PATH=os.path.join(emu, "libmiden_b200_emu.so"), MDN_ALLOW_EMULATOR="1", MDN_EMU_SHM="1",
               OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29753", os.path.join(ROOT, "tests", "run_census_sharded.py")],
                       env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.count("CENSUS_SHARD_REFUSED_OK") == 2, r.stdout[-2000:] + r.stderr[-3000:]
