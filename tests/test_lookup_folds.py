"""mdn_check_lookup_folds: the constraint-path fold (V, U) of every LogUp column on every row, computed on the device and
compared with an aux trace, without proving (the reference's `collect_column_oracle_folds`,
air/src/lookup/debug/trace/mod.rs:191-207 with debug/trace/builder.rs, compared as `assert_prover_matches_oracle` does).

Three implementations: the device kernel; the CPU oracle's handle-by-handle restatement (tests/oracle_folds); and
`ref_folds` below, which evaluates every group in closed form with Python integers on the lowered op-list
(U_g = 1 + sum_calls flag * (prod d - 1), V_g = sum_calls flag * sum_i m_i * prod_{j != i} d_j).  The aux traces "from
elsewhere" come from `ref_aux`, a Python-integer prover path (sum of m / d over the active pushes, running sum in
column 0).  The fixture is the closed two-AIR bus of tests/test_trace_balance.py: a periodic flag, a flagged and an
unflagged interaction, batches and a cached-encoding group.  The small -m gpu cases also run on the kernel emulator of
tests/emu (tests/test_lookup_folds_emulated.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
import pkgload
import test_trace_balance as TB

pkg = pkgload.load_pkg()
W, B = pkg.workload, pkg.binding
P, RND, ROOT, EMU, NONE = TB.P, TB.RND, TB.ROOT, TB.EMU, TB.NONE
ef_add, ef_mul, ef_inv = TB.ef_add, TB.ef_mul, TB.ef_inv
gpu = pytest.mark.gpu
INFO_POOL = 9                                                           # MDN_INFO_POOL
HEIGHTS = [(3, 3), (3, 4), (4, 6), (5, 7), (6, 9), (8, 12)]          # (log table height, log lookup height)


def ef_sub(x, y):
    return ((x[0] - y[0]) % P, (x[1] - y[1]) % P)


def bus_case(log_t=5, log_l=7, seed=11):
    """(workload, fold marks per AIR, airs for the Python references) of the closed bus."""
    bus = TB.Bus(log_t=log_t, log_l=log_l, seed=seed)
    return bus, *marked(bus)


def marked(bus):
    wl, _, airs = bus.workload()
    return wl, [TB.table_lookup().fold_marks(), TB.sender_lookup().fold_marks(), None], airs


# ---------------------------------------------------------------------------------------------------------------------
# references with Python integers
# ---------------------------------------------------------------------------------------------------------------------
def _rows_of(a, rnd):
    """Per row the list of (column, flag, multiplicity, denominator) values of one AIR's interactions."""
    v, items = TB._nodes(a["lookup"], a["main"], a["periodic"], a.get("publics", ()), rnd)
    n = a["main"].shape[0]
    ncol = 1 + max(c for c, _, _, _ in items)
    rows = [[(c, 1 if f == NONE else v[f][0][r], v[m][0][r], (v[d][0][r], v[d][1][r] if v[d][1] is not None else 0))
             for c, f, m, d in items] for r in range(n)]
    return rows, ncol


def ref_folds(a, rnd, marks):
    """folds[r][c] = (V, U) of one AIR, every group in closed form."""
    rows, ncol = _rows_of(a, rnd)
    marks = [3] * len(rows[0]) if marks is None else [int(x) for x in marks]
    out = []
    for row in rows:
        groups = []                                   # (column, [calls]), a call = (flag, [(m, d)])
        for (c, f, m, d), mk in zip(row, marks):
            if mk == 3:
                groups.append((c, []))
            if mk & 1:
                groups[-1][1].append((f, []))
            groups[-1][1][-1][1].append((m, d))
        folds = [((0, 0), (1, 0)) for _ in range(ncol)]
        for c, calls in groups:
            ug, vg = (1, 0), (0, 0)
            for f, ins in calls:
                prod = (1, 0)
                for _, d in ins:
                    prod = ef_mul(prod, d)
                num = (0, 0)
                for i, (m, _) in enumerate(ins):
                    t = (m, 0)
                    for j, (_, d) in enumerate(ins):
                        if j != i:
                            t = ef_mul(t, d)
                    num = ef_add(num, t)
                ug = ef_add(ug, ef_mul(ef_sub(prod, (1, 0)), (f, 0)))
                vg = ef_add(vg, ef_mul(num, (f, 0)))
            v, u = folds[c]
            folds[c] = (ef_add(ef_mul(v, ug), ef_mul(vg, u)), ef_mul(u, ug))
        out.append(folds)
    return out


def ref_aux(a, rnd):
    """The prover path: (aux (N, 2 * columns) uint64, final (c0, c1)).  A zero denominator contributes nothing."""
    rows, ncol = _rows_of(a, rnd)
    aux = np.zeros((len(rows), 2 * ncol), dtype=np.uint64)
    acc = (0, 0)
    for r, row in enumerate(rows):
        frac = [(0, 0)] * ncol
        for c, f, m, d in row:
            if f and d != (0, 0):
                frac[c] = ef_add(frac[c], ef_mul((m, 0), ef_inv(d)))
        aux[r, 0:2] = acc
        for c in range(1, ncol):
            aux[r, 2 * c: 2 * c + 2] = frac[c]
        for c in range(ncol):
            acc = ef_add(acc, frac[c])
    return aux, acc


def ref_check(airs, rnd, marks, auxs, finals):
    """The report of mdn_check_lookup_folds as binding.fold_report_dict gives it."""
    rep = dict(holds=1, kind=0, instance=0, column=0, row=0, fold=(0,) * 4, expected=(0, 0), actual=(0, 0), failing_rows=0,
               zero_u=0, n_skipped_airs=0)
    for i, a in enumerate(airs):
        if a["lookup"] is None:
            rep["n_skipped_airs"] += 1
            continue
        folds = ref_folds(a, rnd, marks[i])
        aux, n = auxs[i], len(folds)
        at = lambda r, c: tuple(int(x) for x in finals[i]) if r == n else (int(aux[r, 2 * c]), int(aux[r, 2 * c + 1]))
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
                rep["zero_u"] += zero[c]
                if kind and rep["holds"]:
                    rep.update(holds=0, kind=kind, instance=i, column=c, row=r, fold=v + u, expected=expected, actual=actual)
                bad |= kind != 0
            rep["failing_rows"] += bad
    return rep


def flat(folds):
    return np.array([w for row in folds for v, u in row for w in v + u], dtype=np.uint64)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle (tests/oracle_folds/liboracle_folds.so)
# ---------------------------------------------------------------------------------------------------------------------
_of_lib = None


def _ofl():
    global _of_lib
    if _of_lib is None:
        d = os.path.join(ROOT, "tests", "oracle_folds")
        subprocess.check_call(["make", "-s", "-C", d])
        L = C.CDLL(os.path.join(d, "liboracle_folds.so"))
        L.orc_last_error.restype = C.c_char_p
        L.orc_collect_column_folds.argtypes = [C.POINTER(ob.Statement), C.POINTER(ob.Matrix), ob.u64p, C.POINTER(ob.u32p), C.POINTER(ob.u64p)]
        L.orc_check_lookup_folds.argtypes = [C.POINTER(ob.Statement), C.POINTER(ob.Matrix), ob.u64p, C.POINTER(ob.u32p),
                                             C.POINTER(ob.Matrix), C.POINTER(ob.u64p), C.POINTER(B.FoldReport)]
        _of_lib = L
    return _of_lib


def _marks_arg(wl, marks, keep):
    arr = (ob.u32p * wl.k)()
    for i, m in enumerate(marks):
        if m is not None:
            keep.append(np.ascontiguousarray(m, dtype=np.uint32))
            arr[i] = keep[-1].ctypes.data_as(ob.u32p)
    return arr


def fold_buffers(wl):
    return [np.zeros((1 << wl.log_heights[i]) * wl.aux_widths[i] * 4, dtype=np.uint64) if wl.aux_widths[i] else None for i in range(wl.k)]


def oracle_folds(wl, rnd, marks):
    keep, bufs = [], fold_buffers(wl)
    outs = (ob.u64p * wl.k)()
    for i, b in enumerate(bufs):
        if b is not None:
            outs[i] = ob.ptr(b)
    r = np.array(rnd, dtype=np.uint64)
    if _ofl().orc_collect_column_folds(TB._cast(wl.statement, ob.Statement), TB._cast(wl.matrices, ob.Matrix), ob.ptr(r),
                                       _marks_arg(wl, marks, keep), outs) != 0:
        raise RuntimeError(_ofl().orc_last_error().decode())
    return bufs


def oracle_check(wl, rnd, marks, auxs, finals):
    keep = []
    mats, fins = (ob.Matrix * wl.k)(), (ob.u64p * wl.k)()
    for i, a in enumerate(auxs):
        if a is not None:
            keep += [np.ascontiguousarray(a), np.array([int(x) for x in finals[i]], dtype=np.uint64)]
            mats[i] = ob.Matrix(ob.ptr(keep[-2]), wl.log_heights[i], a.shape[1])
            fins[i] = ob.ptr(keep[-1])
    rep = B.FoldReport()
    r = np.array(rnd, dtype=np.uint64)
    if _ofl().orc_check_lookup_folds(TB._cast(wl.statement, ob.Statement), TB._cast(wl.matrices, ob.Matrix), ob.ptr(r),
                                     _marks_arg(wl, marks, keep), mats, fins, C.byref(rep)) != 0:
        raise RuntimeError(_ofl().orc_last_error().decode())
    return B.fold_report_dict(rep)


def all_aux(airs, rnd):
    pairs = [ref_aux(a, rnd) if a["lookup"] is not None else (None, None) for a in airs]
    return [p[0] for p in pairs], [p[1] for p in pairs]


# ---------------------------------------------------------------------------------------------------------------------
# one fault at a time
# ---------------------------------------------------------------------------------------------------------------------
def fault(name):
    """(bus, wl, marks, airs, auxs, finals, expected (kind, instance, row, column, failing_rows, zero_u))."""
    bus, wl, marks, airs = bus_case()
    auxs, finals = all_aux(airs, RND)
    n = auxs[1].shape[0]
    if name == "fraction":                       # one flipped word in fraction column 2 of the lookup AIR
        auxs[1][40, 4] ^= 1
        exp = (1, 1, 40, 2, 1, 0)
    elif name == "accumulator":                  # one flipped word in column 0: the deltas of rows r - 1 and r
        auxs[1][33, 1] ^= 1
        exp = (2, 1, 32, 0, 2, 0)
    elif name == "final":                        # a wrong closing value: the last row's delta only
        finals[0] = ((finals[0][0] + 1) % P, finals[0][1])
        exp = (2, 0, auxs[0].shape[0] - 1, 0, 1, 0)
    elif name == "zero_denominator":             # h = 1 with q = 0 at row 9: U of column 2 is zero there
        bus.sender[9, 9], bus.sender[9, 10] = 1, 0
        wl, marks, airs = marked(bus)
        auxs, finals = all_aux(airs, RND)
        exp = (3, 1, 9, 2, 1, 1)
    elif name == "flag_two":                     # f = 2 at row 5: the prover pushes -1 / d, the group folds (-2, 1 + 2 (d - 1))
        bus.sender[5, 2] = 2
        wl, marks, airs = marked(bus)
        auxs, finals = all_aux(airs, RND)
        exp = (2, 1, 5, 0, 1, 0)
    else:
        raise KeyError(name)
    assert n == auxs[1].shape[0]
    return bus, wl, marks, airs, auxs, finals, exp


FAULTS = ["fraction", "accumulator", "final", "zero_denominator", "flag_two"]


def _two_flags():
    """s0 and s1 both set at row 0: the cached group adds the two denominators where separate groups multiply them.  Both
    carry the same denominator with multiplicities +1 and -1, so V is zero either way and every aux trace still holds."""
    bus = TB.Bus()
    bus.sender[0, 7] = 1
    return bus


def _norm(d):
    return TB._norm(d)


def _key(rep):
    return (rep["kind"], rep["instance"], rep["row"], rep["column"], rep["failing_rows"], rep["zero_u"])


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the builder's marks, the oracle on the Python reference
# ---------------------------------------------------------------------------------------------------------------------
def test_builder_marks_groups_and_batches():
    assert [int(x) for x in TB.sender_lookup().fold_marks()] == [3, 3, 0, 3, 1, 1, 0, 3]
    assert [int(x) for x in TB.table_lookup().fold_marks()] == [3]
    lb = pkg.air_program.LookupProgramBuilder(1)
    lb.insert(0, None, lb.const(1), lb.ext_const(5, 9))           # outside `group`: a group of its own
    lb.insert(0, None, lb.const(1), lb.ext_const(5, 9))
    assert [int(x) for x in lb.fold_marks()] == [3, 3]


@pytest.mark.parametrize("log_t,log_l", HEIGHTS)
def test_oracle_folds_equal_the_python_folds(log_t, log_l):
    _, wl, marks, airs = bus_case(log_t, log_l)
    got = oracle_folds(wl, RND, marks)
    for i in (0, 1):
        assert np.array_equal(got[i], flat(ref_folds(airs[i], RND, marks[i])))
    auxs, finals = all_aux(airs, RND)
    rep = oracle_check(wl, RND, marks, auxs, finals)
    assert rep["holds"] == 1 and rep["n_skipped_airs"] == 1 and rep["failing_rows"] == 0


def test_folds_without_marks_are_one_group_per_interaction():
    _, wl, marks, airs = bus_case()
    none = [None] * 3
    got = oracle_folds(wl, RND, none)
    assert np.array_equal(got[1], flat(ref_folds(airs[1], RND, None)))
    assert np.array_equal(got[1], oracle_folds(wl, RND, marks)[1])         # boolean flags, one per group: the same pairs
    wl, marks, _ = marked(_two_flags())
    assert not np.array_equal(oracle_folds(wl, RND, none)[1], oracle_folds(wl, RND, marks)[1])


@pytest.mark.parametrize("name", FAULTS)
def test_oracle_and_python_report_each_fault_where_it_was_made(name):
    _, wl, marks, airs, auxs, finals, exp = fault(name)
    ref = ref_check(airs, RND, marks, auxs, finals)
    assert _key(ref) == exp and ref["holds"] == 0
    assert _norm(oracle_check(wl, RND, marks, auxs, finals)) == _norm(ref)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def aux_for(wl, auxs, mode):
    """(mdn_matrix array, buffers to keep alive) of the aux traces in the layout of traces_for(wl, mode)."""
    mats, keep = (B.Matrix * wl.k)(), []
    for i, a in enumerate(auxs):
        if a is None:
            continue
        if mode == "host":
            keep.append(np.ascontiguousarray(a))
            mats[i] = B.Matrix(B.ptr(keep[-1]), wl.log_heights[i], a.shape[1])
        else:
            keep.append(TB._to_device(a if mode == "device_rm" else a.T))
            mats[i] = B.Matrix(C.cast(C.c_void_p(TB._addr(keep[-1])), B.u64p), wl.log_heights[i], a.shape[1])
    return mats, keep


def device_fold_buffers(wl, mode):
    """(folds_out argument, read-back function giving row-major numpy folds per AIR)."""
    host = fold_buffers(wl)
    if mode == "host":
        return host, lambda: host
    dev = [TB._to_device(b) if b is not None else None for b in host]

    def back():
        out = []
        for i, d in enumerate(dev):
            if d is None:
                out.append(None)
                continue
            a = d if EMU else d.cpu().numpy().view(np.uint64)
            n, c = 1 << wl.log_heights[i], wl.aux_widths[i]
            out.append(np.ascontiguousarray(a.reshape(4 * c, n).T).reshape(-1) if mode == "device_cm" else a.copy())
        return out
    return [TB._addr(d) if d is not None else None for d in dev], back, dev


def run(sess, wl, marks, mode="host", auxs=None, finals=None, want_folds=False):
    mats, flags, keep = TB.traces_for(wl, mode)
    amats, akeep = aux_for(wl, auxs, mode) if auxs is not None else (None, None)
    fb = device_fold_buffers(wl, mode) if want_folds else (None, None)
    rep = sess.check_lookup_folds(wl.statement, mats, RND, marks, amats, finals, fb[0], flags)
    return (rep, fb[1]()) if want_folds else rep


@gpu
@pytest.mark.parametrize("log_t,log_l", HEIGHTS)
def test_device_folds_equal_the_oracle_and_the_python_folds(log_t, log_l):
    _, wl, marks, airs = bus_case(log_t, log_l)
    rep, got = run(TB.session(), wl, marks, want_folds=True)            # aux == NULL: the device LogUp build is checked
    assert rep["holds"] == 1 and rep["kind"] == 0 and rep["n_skipped_airs"] == 1 and rep["zero_u"] == 0
    orc = oracle_folds(wl, RND, marks)
    for i in (0, 1):
        assert np.array_equal(got[i], orc[i])
        assert np.array_equal(got[i], flat(ref_folds(airs[i], RND, marks[i])))


@gpu
def test_device_folds_without_marks():
    _, wl, _, airs = bus_case()
    rep, got = run(TB.session(), wl, None, want_folds=True)
    assert rep["holds"] == 1                                              # boolean flags: one group per interaction holds too
    assert np.array_equal(got[1], flat(ref_folds(airs[1], RND, None)))


@gpu
@pytest.mark.parametrize("mode", ["host", "device_rm", "device_cm"])
def test_aux_from_the_python_builder_holds_in_every_layout(mode):
    _, wl, marks, airs = bus_case()
    auxs, finals = all_aux(airs, RND)
    rep, got = run(TB.session(), wl, marks, mode, auxs, finals, want_folds=True)
    assert _norm(rep) == _norm(ref_check(airs, RND, marks, auxs, finals)) and rep["holds"] == 1
    orc = oracle_folds(wl, RND, marks)
    for i in (0, 1):
        assert np.array_equal(got[i], orc[i])


@gpu
@pytest.mark.parametrize("mode", ["host", "device_rm", "device_cm"])
@pytest.mark.parametrize("name", FAULTS)
def test_each_fault_is_reported_at_its_first_row_and_column(name, mode):
    _, wl, marks, airs, auxs, finals, exp = fault(name)
    rep = run(TB.session(), wl, marks, mode, auxs, finals)
    assert _key(rep) == exp
    assert _norm(rep) == _norm(ref_check(airs, RND, marks, auxs, finals))
    assert _norm(rep) == _norm(oracle_check(wl, RND, marks, auxs, finals))


@gpu
def test_self_check_finds_a_flag_that_is_not_boolean_and_refuses_a_zero_denominator():
    _, wl, marks, airs, _, _, exp = fault("flag_two")
    rep = run(TB.session(), wl, marks)
    assert _key(rep) == exp                      # the device LogUp build pushes -1 / d whatever the non-zero flag is
    wl, marks, airs = marked(_two_flags())       # U differs between the groupings, V / U does not
    rep, got = run(TB.session(), wl, marks, want_folds=True)
    assert rep["holds"] == 1 and np.array_equal(got[1], flat(ref_folds(airs[1], RND, marks[1])))
    assert not np.array_equal(got[1], run(TB.session(), wl, None, want_folds=True)[1][1])
    _, wl, marks, _, _, _, _ = fault("zero_denominator")
    TB._expect_error(-1, lambda: run(TB.session(), wl, marks), "LogUp denominator must be non-zero")


@gpu
def test_lookup_2_20_against_table_2_16_matches_the_oracle():
    bus = TB.Bus(log_t=16, log_l=20, seed=3, n_boundary=4)
    wl, marks, _ = marked(bus)
    orc = oracle_folds(wl, RND, marks)
    for mode in ("host", "device_cm"):
        rep, got = run(TB.session(), wl, marks, mode, want_folds=True)
        assert rep["holds"] == 1
        assert np.array_equal(got[0], orc[0]) and np.array_equal(got[1], orc[1])


@gpu
def test_error_paths_are_refused_and_launch_nothing():
    _, wl, marks, airs = bus_case()
    auxs, finals = all_aux(airs, RND)
    sess = B.Session(W.miden_pcs_params(), 0)
    run(sess, wl, marks)                          # the arena has its slabs from here on
    pool = sess.info(INFO_POOL).copy()

    def call(rnd=RND, marks=marks, auxs=auxs, finals=finals, folds=None, flags=0):
        amats, keep = aux_for(wl, auxs, "host") if auxs is not None else (None, None)
        return sess.check_lookup_folds(wl.statement, wl.matrices, rnd, marks, amats, finals, folds, flags)
    TB._expect_error(-1, lambda: call(rnd=[P] + RND[1:]), "randomness word 0 is not a canonical")
    bad = [m.copy() if m is not None else None for m in marks]
    bad[1][0] = 1
    TB._expect_error(-1, lambda: call(marks=bad), "must open a group")
    bad[1][0], bad[1][4] = 3, 0                   # two inserts with different flags claimed as one batch
    TB._expect_error(-1, lambda: call(marks=bad), "do not share a flag node")
    bad[1][4] = 2
    TB._expect_error(-1, lambda: call(marks=bad), "fold mark 2")
    TB._expect_error(-1, lambda: call(marks=[marks[0], marks[1], np.zeros(1, dtype=np.uint32)]), "without a lookup program")
    TB._expect_error(-1, lambda: call(auxs=None), "aux_finals given without aux")
    TB._expect_error(-1, lambda: call(finals=[finals[0], None, None]), "aux_finals is NULL")
    TB._expect_error(-1, lambda: call(finals=[(P, 0), finals[1], None]), "not a canonical")
    TB._expect_error(-1, lambda: call(auxs=[auxs[0], auxs[1][:, :4], None]), "the aux trace must be")
    TB._expect_error(-1, lambda: call(flags=B.FLAG_COLUMN_MAJOR), "MDN_FLAG_COLUMN_MAJOR is only valid")
    assert np.array_equal(sess.info(INFO_POOL), pool)
    noncanon = [auxs[0], auxs[1].copy(), None]
    noncanon[1][3, 2] = P
    TB._expect_error(-1, lambda: call(auxs=noncanon), "an aux trace contains a non-canonical")
    # inside a staged proof: refused without disturbing it
    pw = W.Workload([10, 9, 8])
    obs = lambda c, f: B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(f, dtype=np.uint64)), len(f))
    ch = W.initial_challenger(W.miden_pcs_params(), obs)
    root, rnd = np.zeros(4, dtype=np.uint64), np.zeros(8, dtype=np.uint64)
    assert B.lib().mdn_prove_begin(sess.handle, C.byref(pw.statement), pw.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0
    TB._expect_error(-1, call, "inside a proof")
    assert B.lib().mdn_prove_commit_aux(sess.handle, None, None, B.ptr(root)) == 0
    proof = B.Proof()
    assert B.lib().mdn_prove_finish(sess.handle, C.byref(proof)) == 0
    staged = B.proof_to_numpy(proof)
    fresh = B.Session(W.miden_pcs_params(), 0)
    ref = fresh.prove(pw.statement, pw.matrices, W.initial_challenger(W.miden_pcs_params(), obs))
    assert staged[0] == ref[0] and np.array_equal(staged[1], ref[1]) and np.array_equal(staged[2], ref[2])
    sess.close(); fresh.close()


@gpu
def test_proof_after_a_fold_check_is_byte_identical():
    pw = W.Workload([10, 9, 8])
    params = W.miden_pcs_params()
    obs = lambda c, f: B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(f, dtype=np.uint64)), len(f))
    a = B.Session(params, 0)
    before = a.prove(pw.statement, pw.matrices, W.initial_challenger(params, obs))
    t_before = (a.timings().total, a.timings().kernel_launches)
    info_before = a.info(0)
    _, wl, marks, airs, auxs, finals, _ = fault("fraction")
    run(a, wl, marks, "host", auxs, finals, want_folds=True)
    run(a, wl, marks)
    assert (a.timings().total, a.timings().kernel_launches) == t_before and np.array_equal(a.info(0), info_before)
    after = a.prove(pw.statement, pw.matrices, W.initial_challenger(params, obs))
    assert before[0] == after[0] and np.array_equal(before[1], after[1]) and np.array_equal(before[2], after[2])
    a.close()


def test_new_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "miden_b200.h")).read()
    assert "int mdn_check_lookup_folds(" in header and "} mdn_fold_report;" in header
    assert "mdn_check_lookup_folds" in B.EXPORTS
    assert C.sizeof(B.FoldReport) == 4 * 4 + 8 + 8 * 8 + 2 * 8 + 2 * 4
