"""The constraint guard (mdn_session_set_constraint_guard): every constraint of every AIR on every trace row, checked inside
the proof with the proof's own challenges, before the aux commitment.

What is pinned:
  * a statement that holds gets the byte-identical proof with the guard on and off, accepted by the oracle verifier,
    for every trace source, hash configuration, preprocessed / periodic columns, mixed heights and the staged API;
  * a single hand-made fault makes the proof fail with MDN_ERR_CONSTRAINT_VIOLATED, and the report equals, field for
    field, `ref_check` of tests/test_check_constraints.py (debug.rs restated with Python integers) evaluated with the
    proof's randomness -- taken from mdn_prove_begin's randomness_out on the same inputs (the proof is deterministic);
  * the same faulty statement with the guard off still proves, and the oracle verifier rejects that proof;
  * a challenge-dependent aux bug passes mdn_check_constraints (debug challenges) and is refused by the guard.
The small -m gpu cases also run on the kernel emulator (tests/test_constraint_guard_emulated.py)."""
import ctypes as C
import os

import numpy as np
import pytest

import pkgload
import test_airs as TA
import test_check_constraints as TC
import test_device_resident as TDR

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
P = W.P
gpu = pytest.mark.gpu
HASHES = TC.HASHES
HOLDS = dict(TC.NO_FAIL, holds=1, failing_rows=0)


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def hash_session(params, hash_kind=B.HASH_POSEIDON2, guard=False):
    s = TDR.session(params, hash_kind)
    s.set_constraint_guard(guard)
    return s


def proof_randomness(params, wl, hash_kind=B.HASH_POSEIDON2):
    """The proof's randomness (2 * max num_randomness u64): mdn_prove_begin's randomness_out on the same inputs, on a
    session of its own that is closed with the staged proof still open."""
    s = TDR.session(params, hash_kind)
    try:
        if wl.preprocessed is not None:
            s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
        m = max(wl._airs[i].num_randomness for i in range(wl.k))
        rnd = np.zeros(max(1, 2 * m), dtype=np.uint64)
        root = np.zeros(4, dtype=np.uint64)
        ch = TC.seed(params, hash_kind)
        rc = B.lib().mdn_prove_begin(s.handle, C.byref(wl.statement), wl.matrices, C.byref(ch) if ch is not None else None, 0,
                                     B.ptr(root), B.ptr(rnd))
        assert rc == 0, B.lib().mdn_last_error(s.handle).decode()
        return [int(x) for x in rnd[: 2 * m]]
    finally:
        s.close()


def restate(wl, builder, chal):
    """`ref_check` of debug.rs on the workload with challenges `chal` and the aux traces of `builder` (None: zeros)."""
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
    return TC.ref_check(inst, wl.public_values, chal)


def prove(s, wl, params, builder=None, hash_kind=B.HASH_POSEIDON2, traces=None, flags=0):
    """s.prove with the workload's preprocessed bundle installed (removed again afterwards); returns the proof and the
    bundle's commitment."""
    prep = None
    if wl.preprocessed is not None:
        prep = s.set_preprocessed(wl.statement, wl.preprocessed_matrices)
    try:
        cb = B.AUX_BUILDER(builder) if builder is not None else None
        return s.prove(wl.statement, wl.matrices if traces is None else traces, TC.seed(params, hash_kind), cb, flags), prep
    finally:
        if prep is not None:
            s.set_preprocessed(None, None)


def guarded_and_plain(wl, params, builder=None, hash_kind=B.HASH_POSEIDON2, traces=None, flags=0):
    """The proof with the guard on and with it off (two sessions): byte-equal and accepted by the oracle verifier."""
    on, off = hash_session(params, hash_kind, True), hash_session(params, hash_kind, False)
    try:
        got, prep = prove(on, wl, params, builder, hash_kind, traces, flags)
        want, _ = prove(off, wl, params, builder, hash_kind, traces, flags)
        assert TDR.same(got, want), "the guard changed the proof"
        assert TC.report_dict(on.last_constraint_report()) == HOLDS
        rc, err = TDR.oracle_verify(params, wl, hash_kind, got, prep)
        assert rc == 0, err
        return got
    finally:
        on.close(); off.close()


def refused(wl, params, builder=None, traces=None, flags=0):
    """Prove with the guard on: must fail with ConstraintViolation; returns (report dict, message)."""
    s = hash_session(params, guard=True)
    try:
        with pytest.raises(B.ConstraintViolation) as e:
            prove(s, wl, params, builder, traces=traces, flags=flags)
        rep = TC.report_dict(e.value.report)
        assert rep == TC.report_dict(s.last_constraint_report())
        assert str(e.value).startswith("[-8]") and isinstance(e.value, B.ProverError)
        return rep, str(e.value)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# statements
# ---------------------------------------------------------------------------------------------------------------------
def fault_case(name):
    """(workload, host builder or None) with one hand-made fault."""
    if name == "main_mid_trace":                       # b[13] += 1: b' = a + b fails at row 12, a' = b at row 13
        return TC.violation_case("main_row_interior")
    if name == "first_row_boundary_only":              # public 0: first * (a - p0) fails at row 0 only
        wl, bld = TA.fib_product_workload([5])
        wl.public_values[0] = 5
        return wl, bld
    if name == "last_row_boundary_only":               # public 2: last * (b - p2) fails at row N-1 only
        return TC.violation_case("public_value")
    if name == "transition":                           # a[20] += 1: a' = b fails at row 19 and b' = a + b at row 20
        wl, bld = TA.fib_product_workload([5])
        wl.traces[0][20, 0] = (int(wl.traces[0][20, 0]) + 1) % P
        return wl, bld
    if name == "host_aux_cell":
        return TC.violation_case("aux_cell")
    if name in ("preprocessed_cell", "periodic_value", "taller_first"):
        return TC.violation_case(name)
    raise KeyError(name)


FAULTS = ["main_mid_trace", "first_row_boundary_only", "last_row_boundary_only", "transition", "host_aux_cell",
          "preprocessed_cell", "periodic_value", "taller_first"]
NO_RANDOMNESS = ["preprocessed_cell", "periodic_value", "taller_first"]


def test_abi_surface():
    assert {"mdn_session_set_constraint_guard", "mdn_last_constraint_report"} <= set(B.EXPORTS)
    assert B.ERR_CONSTRAINT_VIOLATED == -8
    assert issubclass(B.ConstraintViolation, B.ProverError)
    hdr = open(os.path.join(pkgload.ROOT, "include", "miden_b200.h")).read()
    assert "MDN_ERR_CONSTRAINT_VIOLATED = -8" in hdr


@pytest.mark.parametrize("name", FAULTS)
def test_faults_are_single_and_where_expected(name):
    """The restatement with the debug challenges (any challenges would do for these) finds each fault where the case says."""
    wl, bld = fault_case(name)
    rep, _ = TC.reference(wl, W.fast_pcs_params(), bld)
    assert rep["holds"] == 0 and rep["kind"] == 1
    where = {"main_mid_trace": (0, 12, 3), "first_row_boundary_only": (0, 0, 0), "last_row_boundary_only": (0, 31, 6),
             "transition": (0, 19, 2)}
    if name in where:
        assert (rep["instance"], rep["row"], rep["constraint"]) == where[name]
    if name == "taller_first":                             # the taller instance 0 wins, though it is committed second
        assert (rep["instance"], rep["row"]) == (0, 100)
    if name in ("first_row_boundary_only", "last_row_boundary_only"):
        assert rep["failing_rows"] == 1


# ---------------------------------------------------------------------------------------------------------------------
# GPU: identical proofs on statements that hold
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("hash_kind", HASHES)
def test_identical_proof_every_hash(hash_kind):
    wl, bld = TA.fib_product_workload([5])
    guarded_and_plain(wl, W.fast_pcs_params(), bld, hash_kind)


@gpu
@pytest.mark.parametrize("name", TC.VALID)
def test_identical_proof_valid_statements(name):
    """LogUp built on the device and by a host builder, periodic and preprocessed columns, mixed heights, a large program."""
    wl, bld = TC.valid_case(name)
    guarded_and_plain(wl, W.fast_pcs_params(), bld)


@gpu
def test_identical_proof_row_major_device_traces():
    wl = TC.dummy_workload([6, 5])
    mats, bufs = TDR.row_major_device_traces(wl)
    guarded_and_plain(wl, W.fast_pcs_params(), traces=mats, flags=B.FLAG_DEVICE_TRACES)


@gpu
@pytest.mark.parametrize("name", ["logup_device", "dummy_device_builder"])
def test_identical_proof_column_major_device_traces(name):
    """Column-major device traces read in place, aux from the device aux builder or the device LogUp build."""
    params = W.fast_pcs_params()
    if name == "logup_device":
        wl, bld = TA.logup_workload(6, device=True)
    else:
        wl, bld = TDR.dummy_case([6, 4, 5], (11, 9, 10), (2, 0, 1))
    proofs = []
    for guard in (True, False):
        s = hash_session(params, guard=guard)
        mats, bufs = TDR.column_major_traces(wl)
        s.set_device_aux_builder(TDR.device_builder(wl, bld, bufs))
        try:
            proofs.append(s.prove(wl.statement, mats, TC.seed(params), None, TDR.CM))
        finally:
            s.set_device_aux_builder(None)
            s.close()
        for t, b in zip(wl.traces, bufs):
            assert np.array_equal(TDR.from_device(b), t.T), "the caller's device trace changed"
    assert TDR.same(*proofs)
    rc, err = TDR.oracle_verify(params, wl, B.HASH_POSEIDON2, proofs[0])
    assert rc == 0, err


def staged(s, wl, params, aux_fn=None):
    """mdn_prove_begin / commit_aux / finish; aux_fn(randomness) -> (aux matrices, aux value pointers) or None (zeros).
    Returns (status of commit_aux, proof or None)."""
    L = B.lib()
    m = max(wl._airs[i].num_randomness for i in range(wl.k))
    rnd = np.zeros(max(1, 2 * m), dtype=np.uint64)
    root = np.zeros(4, dtype=np.uint64)
    ch = TC.seed(params)
    assert L.mdn_prove_begin(s.handle, C.byref(wl.statement), wl.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0
    aux, vals = aux_fn([int(x) for x in rnd[: 2 * m]]) if aux_fn is not None else (None, None)
    rc = L.mdn_prove_commit_aux(s.handle, aux, vals, B.ptr(np.zeros(4, dtype=np.uint64)))
    if rc != 0:
        return rc, None
    pf = B.Proof()
    assert L.mdn_prove_finish(s.handle, C.byref(pf)) == 0
    return rc, B.proof_to_numpy(pf)


def staged_aux(wl, builder, corrupt=None):
    """aux_fn for `staged` from a host builder; `corrupt(aux list)` may change the built traces."""
    def fn(chal):
        bufs = [TC.run_builder(builder, wl, i, chal) for i in range(wl.k)]
        if corrupt is not None:
            corrupt(bufs)
        mats = (B.Matrix * wl.k)()
        vals = (B.u64p * wl.k)()
        for i, (a, v) in enumerate(bufs):
            mats[i] = B.Matrix(B.ptr(a), wl.log_heights[i], 2 * wl._airs[i].aux_width)
            vals[i] = B.ptr(v)
        mats._keep = bufs
        return mats, vals
    return fn


@gpu
def test_staged_api_identical_and_refused():
    params = W.fast_pcs_params()
    wl, bld = TA.fib_product_workload([5, 6])
    on, off = hash_session(params, guard=True), hash_session(params)
    try:
        rc1, p1 = staged(on, wl, params, staged_aux(wl, bld))
        rc2, p2 = staged(off, wl, params, staged_aux(wl, bld))
        assert rc1 == rc2 == 0 and TDR.same(p1, p2)
        rc, err = TDR.oracle_verify(params, wl, B.HASH_POSEIDON2, p1)
        assert rc == 0, err

        def corrupt(bufs):                                 # instance 0, row 9, the c1 coordinate of its EF aux column
            bufs[0][0][9 * 2 + 1] = (int(bufs[0][0][9 * 2 + 1]) + 1) % P
        rc, _ = staged(on, wl, params, staged_aux(wl, bld, corrupt))
        assert rc == B.ERR_CONSTRAINT_VIOLATED
        chal = proof_randomness(params, wl)
        rep = TC.report_dict(on.last_constraint_report())

        def bad_builder(ctx, inst, main, rnd, aux_out, aux_values):
            r = bld(ctx, inst, main, rnd, aux_out, aux_values)
            if inst == 0:
                aux_out[19] = (aux_out[19] + 1) % P
            return r
        assert rep == restate(wl, bad_builder, chal) and rep["kind"] == 1
        # the session is usable again, and commit_aux's caller-supplied zero aux is checked as well
        rc, p3 = staged(on, wl, params, staged_aux(wl, bld))
        assert rc == 0 and TDR.same(p3, p1)
        assert staged(on, wl, params, None)[0] == B.ERR_CONSTRAINT_VIOLATED     # zero aux: first * (p0 - 1) fails
        assert TC.report_dict(on.last_constraint_report())["constraint"] == 4
    finally:
        on.close(); off.close()


@gpu
def test_zero_aux_of_a_null_builder_is_checked():
    """No aux builder: the aux traces and values are zero; the dummy AIR does not constrain them (proved), the
    fib/product AIR does (refused at its first aux constraint, as the restatement with zero aux says)."""
    params = W.fast_pcs_params()
    wl = TC.dummy_workload([6, 5])
    guarded_and_plain(wl, params)
    wl, _ = TA.fib_product_workload([5])
    rep, _ = refused(wl, params)
    assert rep == restate(wl, None, proof_randomness(params, wl))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: refusals
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", FAULTS)
def test_refusal_report_matches_the_restatement(name):
    params = W.fast_pcs_params()
    wl, bld = fault_case(name)
    rep, msg = refused(wl, params, bld)
    want = restate(wl, bld, proof_randomness(params, wl))
    assert want["kind"] == 1 and rep == want
    assert f"constraint {rep['constraint']} of AIR {rep['instance']} is non-zero at row {rep['row']}" in msg
    if name in NO_RANDOMNESS:                              # no challenges: the same report as mdn_check_constraints
        s = B.Session(params, 0)
        try:
            prep = wl.preprocessed_matrices if wl.preprocessed is not None else None
            chk, _ = s.check_constraints(wl.statement, wl.matrices, TC.seed(params), preprocessed=prep)
            assert TC.report_dict(chk) == rep
        finally:
            s.close()
    # with the guard off the same statement proves, and the verifier rejects the proof: what the guard prevents
    s = hash_session(params)
    try:
        pf, prep = prove(s, wl, params, bld)
    finally:
        s.close()
    rc, _ = TDR.oracle_verify(params, wl, B.HASH_POSEIDON2, pf, prep)
    assert rc != 0, "the oracle verifier accepted a proof of a statement that does not hold"


@gpu
def test_refusal_logup_main_cell():
    """A LogUp AIR built on the device with the flag f = 2 at row 21: row 21 is the only failing row, and its first
    failing constraint is f * (f - 1) = 2 (the device build then also breaks the accumulator constraint of that row)."""
    params = W.fast_pcs_params()
    wl, _ = TA.logup_workload(6, device=True)
    wl.traces[0][21, 4] = 2
    rep, _ = refused(wl, params)
    assert rep == dict(holds=0, kind=1, instance=0, constraint=0, row=21, value=(2, 0), failing_rows=1)
    mats, bufs = TDR.column_major_traces(wl)              # the same from column-major device traces, read in place
    rep2, _ = refused(wl, params, traces=mats, flags=TDR.CM)
    assert rep2 == rep


@gpu
def test_refusal_device_aux_builder():
    """A column-major device trace whose device aux builder writes one wrong cell."""
    params = W.fast_pcs_params()
    wl, bld = TA.fib_product_workload([5])
    mats, bufs = TDR.column_major_traces(wl)

    def corrupt(aux):
        aux = aux.copy()
        aux[9, 1] = (int(aux[9, 1]) + 1) % P
        return aux
    s = hash_session(params, guard=True)
    s.set_device_aux_builder(TDR.device_builder(wl, bld, bufs, corrupt=corrupt))
    try:
        with pytest.raises(B.ConstraintViolation) as e:
            s.prove(wl.statement, mats, TC.seed(params), None, TDR.CM)
    finally:
        s.set_device_aux_builder(None)
        s.close()
    want = restate(wl, TC._corrupt_aux(bld, 9, 0, 1), proof_randomness(params, wl))
    assert TC.report_dict(e.value.report) == want and want["kind"] == 1


@gpu
def test_external_assertion_comes_first():
    params = W.fast_pcs_params()
    wl, bld = fault_case("main_mid_trace")
    s = hash_session(params, guard=True)
    try:
        before = TC.report_dict(s.last_constraint_report())
        s.set_external_check(lambda ch, av, lh: 2)
        with pytest.raises(B.ProverError, match=r"^\[-7\] external assertion 2 failed") as e:
            prove(s, wl, params, bld)
        assert not isinstance(e.value, B.ConstraintViolation)
        assert TC.report_dict(s.last_constraint_report()) == before == HOLDS      # the guard did not run
    finally:
        s.close()


@gpu
def test_next_proof_after_a_refusal_matches_a_fresh_session():
    params = W.fast_pcs_params()
    s, fresh = hash_session(params, guard=True), hash_session(params, guard=True)
    try:
        bad, bbld = fault_case("host_aux_cell")
        with pytest.raises(B.ConstraintViolation):
            prove(s, bad, params, bbld)
        wl, bld = TA.fib_product_workload([6])
        got, _ = prove(s, wl, params, bld)
        want, _ = prove(fresh, wl, params, bld)
        assert TDR.same(got, want)
        assert TC.report_dict(s.last_constraint_report()) == HOLDS                # a passing guard run resets the report
        s.set_constraint_guard(False)
        assert TDR.same(prove(s, wl, params, bld)[0], want)
    finally:
        s.close(); fresh.close()


@gpu
def test_challenge_dependent_aux_bug():
    """A host builder that corrupts an aux cell only when bit `b` of randomness[0] is set, with b chosen so that the
    proof's challenge has it and the debug challenge of mdn_check_constraints does not: the check passes, the guard
    refuses, and the unguarded proof is rejected by the verifier."""
    params = W.fast_pcs_params()
    wl, bld = TA.fib_product_workload([5])
    proof_r0 = proof_randomness(params, wl)[0]
    debug_r0 = TC.oracle_challenges(wl, params)[0]
    bit = next(b for b in range(64) if (proof_r0 >> b) & 1 and not (debug_r0 >> b) & 1)

    def sneaky(ctx, inst, main, rnd, aux_out, aux_values):
        r = bld(ctx, inst, main, rnd, aux_out, aux_values)
        if inst == 0 and (rnd[0] >> bit) & 1:
            aux_out[2 * 17] = (aux_out[2 * 17] + 1) % P
        return r
    s = hash_session(params, guard=True)
    try:
        chk, _ = s.check_constraints(wl.statement, wl.matrices, TC.seed(params), aux_builder=B.AUX_BUILDER(sneaky))
        assert TC.report_dict(chk) == HOLDS
        with pytest.raises(B.ConstraintViolation) as e:
            prove(s, wl, params, sneaky)
        rep = TC.report_dict(e.value.report)
        assert rep == restate(wl, sneaky, proof_randomness(params, wl)) and (rep["row"], rep["kind"]) == (16, 1)
        s.set_constraint_guard(False)
        pf, _ = prove(s, wl, params, sneaky)
    finally:
        s.close()
    assert TDR.oracle_verify(params, wl, B.HASH_POSEIDON2, pf)[0] != 0


@gpu
def test_error_paths():
    L = B.lib()
    params = W.fast_pcs_params()
    assert L.mdn_session_set_constraint_guard(None, 1) == -1
    assert L.mdn_last_constraint_report(None, C.byref(B.ConstraintReport())) == -1
    s = B.Session(params, 0)
    try:
        assert TC.report_dict(s.last_constraint_report()) == HOLDS                # before any guard run
        assert L.mdn_last_constraint_report(s.handle, None) == -1
        with pytest.raises(B.ProverError, match=r"\[-1\].*0 or 1"):
            s._check(L.mdn_session_set_constraint_guard(s.handle, 2))
        wl = TC.dummy_workload([5])
        rnd, root = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
        assert L.mdn_prove_begin(s.handle, C.byref(wl.statement), wl.matrices, C.byref(TC.seed(params)), 0, B.ptr(root), B.ptr(rnd)) == 0
        with pytest.raises(B.ProverError, match=r"\[-1\].*inside a proof"):
            s.set_constraint_guard(True)
        assert L.mdn_prove_commit_aux(s.handle, None, None, None) == 0
        pf = B.Proof()
        assert L.mdn_prove_finish(s.handle, C.byref(pf)) == 0
        s.set_constraint_guard(True)
        s.set_constraint_guard(False)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# H100 only
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_h100_benchmark_statement_identical():
    """The 2^20 x (51, 22, 16) benchmark statement: guard on and off give the same proof, accepted by the oracle."""
    params = W.miden_pcs_params()
    wl = W.Workload([20, 20, 20])
    ch = W.initial_challenger(params, TC.H.oracle_observe)
    on, off = hash_session(params, guard=True), hash_session(params)
    try:
        got = on.prove(wl.statement, wl.matrices, ch)
        want = off.prove(wl.statement, wl.matrices, ch)
        assert TDR.same(got, want)
        assert on.timings().kernel_launches > off.timings().kernel_launches
    finally:
        on.close(); off.close()
    rc, err = TC.H.oracle_verify(params, wl, ch, *got)
    assert rc == 0, err
