"""mdn_check_constraints: every AIR constraint on every trace row, without proving (the reference's
`debug::check_constraints`, crates/lifted-stark/src/debug.rs:70-214).

Two references:
  * `ref_check` below: debug.rs restated with Python integers directly on the op-list (node by node, row by row, the
    constraint ids in emission order), with the challenges derived by the oracle's challenger (orc_challenger_script:
    statement felts, instance count and log heights, no commitment) and the aux traces built by the workloads' own host
    builders;
  * the CPU oracle's checker, orc_check_constraints (tests/oracle_check: the oracle's C API plus its restatement of
    debug.rs, with the oracle's LogUp builder and its node evaluator).
The CPU tests pin the oracle's checker on `ref_check` (every case, every field, the challenges) and `ref_check` on
hand-derived faults; the -m gpu tests compare every field of the device report with both; the small -m gpu cases also
run on the kernel emulator of tests/emu."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
import oracle_binding as ob
import pkgload
import test_airs as TA

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
P = W.P
ROOT = pkgload.ROOT
gpu = pytest.mark.gpu
NO_FAIL = dict(kind=0, instance=0, constraint=0, row=0, value=(0, 0))


# ---------------------------------------------------------------------------------------------------------------------
# reference: debug.rs on the op-list, Python integers
# ---------------------------------------------------------------------------------------------------------------------
def _mul(x, y):
    return ((x[0] * y[0] + 7 * x[1] * y[1]) % P, (x[0] * y[1] + x[1] * y[0]) % P)


def constraint_rows(prog, main, aux, aux_values, publics, challenges, periodic, prep):
    """Per row r of the trace, the values (c0, c1) of the AIR's constraints in emission order."""
    w = [int(x) for x in prog]
    nn, nc, nk = w[2], w[3], w[4]
    nodes = [tuple(w[5 + 3 * j: 8 + 3 * j]) for j in range(nn)]
    cons = w[5 + 3 * nn: 5 + 3 * nn + nc]
    kw = w[5 + 3 * nn + nc:]
    consts = [kw[2 * j] | (kw[2 * j + 1] << 32) for j in range(nk)]
    n = main.shape[0]
    ml = main.tolist()
    al = aux.reshape(n, -1).tolist() if aux is not None and aux.size else None
    pl = prep.tolist() if prep is not None else None
    per = periodic.tolist() if periodic is not None else None
    pub = [int(x) for x in publics]
    ch = [int(x) for x in challenges]
    av = [int(x) for x in aux_values]
    for r in range(n):
        rn = (r + 1) % n
        v = [None] * nn
        for j, (op, a, b) in enumerate(nodes):
            if op == 0: x = (ml[rn if a else r][b], 0)
            elif op == 1: row = al[rn if a else r]; x = (row[2 * b], row[2 * b + 1])
            elif op == 2: x = (pub[a], 0)
            elif op == 3: x = (ch[2 * a], ch[2 * a + 1])
            elif op == 4: x = (av[2 * a], av[2 * a + 1])
            elif op == 5: x = (int(r == 0), 0)
            elif op == 6: x = (int(r == n - 1), 0)
            elif op == 7: x = (int(r != n - 1), 0)
            elif op == 8: x = (consts[a], 0)
            elif op == 9: x = (consts[a], consts[a + 1])
            elif op == 10: x = ((v[a][0] + v[b][0]) % P, (v[a][1] + v[b][1]) % P)
            elif op == 11: x = ((v[a][0] - v[b][0]) % P, (v[a][1] - v[b][1]) % P)
            elif op == 12: x = _mul(v[a], v[b])
            elif op == 13: x = ((-v[a][0]) % P, (-v[a][1]) % P)
            elif op == 14: x = (per[r % len(per)][a], 0)
            elif op == 15: x = (pl[rn if a else r][b], 0)
            else: raise ValueError(op)
            v[j] = x
        yield [v[c] for c in cons]


def ref_check(instances, publics, challenges, ext_failed=None):
    """instances: per AIR (instance order) dict(prog, main, aux, aux_values, periodic, prep).  Returns the report."""
    rep = dict(NO_FAIL, failing_rows=0)
    found = False
    for i, a in enumerate(instances):
        for r, vals in enumerate(constraint_rows(a["prog"], a["main"], a["aux"], a["aux_values"], publics, challenges,
                                                 a["periodic"], a["prep"])):
            bad = [k for k, c in enumerate(vals) if c != (0, 0)]
            if not bad:
                continue
            rep["failing_rows"] += 1
            if not found:
                found = True
                rep.update(kind=1, instance=i, row=r, constraint=bad[0], value=vals[bad[0]])
    if ext_failed is not None:
        rep.update(NO_FAIL, kind=2, constraint=ext_failed)
    rep["holds"] = int(rep["failing_rows"] == 0 and ext_failed is None)
    return rep


def report_dict(rep):
    return dict(holds=rep.holds, kind=rep.kind, instance=rep.instance, constraint=rep.constraint, row=rep.row,
                value=(rep.value[0], rep.value[1]), failing_rows=rep.failing_rows)


# ---------------------------------------------------------------------------------------------------------------------
# challenges (the oracle's challenger) and aux traces (the workloads' host builders)
# ---------------------------------------------------------------------------------------------------------------------
def _orc():
    L = ob.lib()
    L.orc_set_hash.restype = C.c_int
    L.orc_set_hash.argtypes = [C.c_int, C.c_char_p, C.c_size_t]
    return L


def seed(params, hash_kind=B.HASH_POSEIDON2):
    """The caller's duplex challenger: `config.challenger()` + `observe_protocol_params` with the configuration's
    permutation (None for the hash-challenger configurations, whose state is installed with set_hash)."""
    if hash_kind in (B.HASH_BLAKE3, B.HASH_KECCAK):
        return None
    L = _orc()
    assert L.orc_set_hash(hash_kind, None, 0) == 0
    try:
        return W.initial_challenger(params, H.oracle_observe)
    finally:
        L.orc_set_hash(0, None, 0)


def oracle_challenges(wl, params, hash_kind=B.HASH_POSEIDON2):
    """debug.rs:87-97 on the oracle's challenger: the seed (config.challenger() + observe_protocol_params here), the
    statement felts, the instance count and the log heights; then 2 * max num_randomness base samples."""
    L = _orc()
    init = W.initial_hash_challenger(params) if hash_kind in (B.HASH_BLAKE3, B.HASH_KECCAK) else b""
    assert L.orc_set_hash(hash_kind, init or None, len(init)) == 0
    try:
        ch = W.initial_challenger(params, H.oracle_observe)
        m = max(wl._airs[i].num_randomness for i in range(wl.k))
        obs = [int(x) for x in wl.observe_felts] + [wl.k] + list(wl.log_heights)
        ops = np.array([0] * len(obs) + [1] * (2 * m), dtype=np.uint32)
        args = np.array(obs + [0] * (2 * m), dtype=np.uint64)
        out = np.zeros(len(ops), dtype=np.uint64)
        L.orc_challenger_script(H.cast(ch, ob.Challenger), ops.ctypes.data_as(ob.u32p), ob.ptr(args), len(ops), ob.ptr(out))
        return [int(x) for x in out[len(obs):]]
    finally:
        L.orc_set_hash(0, None, 0)


def run_builder(fn, wl, i, challenges):
    a = wl._airs[i]
    n = 1 << wl.log_heights[i]
    m = B.Matrix(wl.traces[i].ctypes.data_as(B.u64p), wl.log_heights[i], wl.widths[i])
    aux = np.zeros(max(1, n * 2 * a.aux_width), dtype=np.uint64)
    vals = np.zeros(2 * a.num_aux_values + 1, dtype=np.uint64)
    r = np.array(challenges[: 2 * a.num_randomness] + [0], dtype=np.uint64)
    assert fn(None, i, C.pointer(m), r.ctypes.data_as(B.u64p), aux.ctypes.data_as(B.u64p), vals.ctypes.data_as(B.u64p)) == 0
    return aux[: n * 2 * a.aux_width], vals[: 2 * a.num_aux_values]


def reference(wl, params, builder=None, hash_kind=B.HASH_POSEIDON2, ext=None):
    """(report, challenges) of debug.rs for workload `wl`; `builder` is the host aux builder (python function) that
    stands for the aux traces -- for a device-built LogUp trace, the host builder of the same trace."""
    chal = oracle_challenges(wl, params, hash_kind)
    inst = []
    for i in range(wl.k):
        a = wl._airs[i]
        if builder is not None:
            aux, vals = run_builder(builder, wl, i, chal)
        else:
            aux = np.zeros((1 << wl.log_heights[i]) * 2 * a.aux_width, dtype=np.uint64)
            vals = np.zeros(2 * a.num_aux_values, dtype=np.uint64)
        per = None
        if a.num_periodic_columns:
            per = np.ctypeslib.as_array(a.periodic_values, shape=((1 << a.log_max_period) * a.num_periodic_columns,))
            per = per.reshape(1 << a.log_max_period, a.num_periodic_columns)
        prep = wl.preprocessed[i] if wl.preprocessed is not None else None
        inst.append(dict(prog=wl.programs[i], main=wl.traces[i], aux=aux, aux_values=vals, periodic=per, prep=prep))
    ext_failed = None
    if ext is not None:
        av = [np.asarray(d["aux_values"], dtype=np.uint64) for d in inst]
        k = ext(np.array(chal, dtype=np.uint64), av, bytes(wl.log_heights))
        ext_failed = None if k is None or k < 0 else k
    return ref_check(inst, wl.public_values, chal, ext_failed), chal


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's checker (tests/oracle_check/liboracle_check.so)
# ---------------------------------------------------------------------------------------------------------------------
class OrcReport(C.Structure):
    _fields_ = B.ConstraintReport._fields_


_occ_lib = None


def _occ():
    global _occ_lib
    if _occ_lib is None:
        d = os.path.join(ROOT, "tests", "oracle_check")
        subprocess.check_call(["make", "-s", "-C", d])
        L = C.CDLL(os.path.join(d, "liboracle_check.so"))
        L.orc_last_error.restype = C.c_char_p
        L.orc_set_hash.restype = C.c_int
        L.orc_set_hash.argtypes = [C.c_int, C.c_char_p, C.c_size_t]
        L.orc_check_constraints.restype = C.c_int
        L.orc_check_constraints.argtypes = [C.POINTER(ob.Statement), C.POINTER(ob.Matrix), C.POINTER(ob.Matrix),
                                            C.POINTER(ob.Challenger), ob.AUX_BUILDER, C.c_void_p, B.EXTERNAL_CHECK,
                                            C.c_void_p, ob.u64p, C.POINTER(OrcReport)]
        _occ_lib = L
    return _occ_lib


def _ext_callback(fn):
    """An mdn_external_check over fn(challenges, aux_values, log_heights) -> None | k (raises: ReductionError)."""
    def tramp(ctx, ch, n_ch, vals, n_vals, lh, n_airs, failed):
        try:
            chal = np.ctypeslib.as_array(ch, shape=(2 * n_ch,)).copy() if n_ch else np.zeros(0, np.uint64)
            av = [np.ctypeslib.as_array(vals[i], shape=(2 * n_vals[i],)).copy() if n_vals[i] else np.zeros(0, np.uint64)
                  for i in range(n_airs)]
            k = fn(chal, av, bytes(lh[:n_airs]))
        except Exception:
            return -1
        if k is None or k < 0:
            return 0
        failed[0] = k
        return 1
    return B.EXTERNAL_CHECK(tramp)


def oracle_check(wl, params, builder=None, hash_kind=B.HASH_POSEIDON2, ext=None):
    """(report, challenges) of orc_check_constraints for workload `wl`."""
    L = _occ()
    init = W.initial_hash_challenger(params) if hash_kind in (B.HASH_BLAKE3, B.HASH_KECCAK) else b""
    ch = seed(params, hash_kind) or B.Challenger()
    assert L.orc_set_hash(hash_kind, init or None, len(init)) == 0
    try:
        m = max(wl._airs[i].num_randomness for i in range(wl.k))
        rnd = np.zeros(max(1, 2 * m), dtype=np.uint64)
        rep = OrcReport()
        cb = ob.AUX_BUILDER(builder) if builder is not None else C.cast(None, ob.AUX_BUILDER)
        ecb = _ext_callback(ext) if ext is not None else C.cast(None, B.EXTERNAL_CHECK)
        prep = H.cast(wl.preprocessed_matrices, ob.Matrix) if wl.preprocessed is not None else None
        rc = L.orc_check_constraints(H.cast(wl.statement, ob.Statement), H.cast(wl.matrices, ob.Matrix), prep,
                                     H.cast(ch, ob.Challenger), cb, None, ecb, None, ob.ptr(rnd), C.byref(rep))
        if rc != 0:
            raise RuntimeError(L.orc_last_error().decode())
        return report_dict(rep), [int(x) for x in rnd[: 2 * m]]
    finally:
        L.orc_set_hash(0, None, 0)


def device_check(sess, wl, params, builder=None, hash_kind=B.HASH_POSEIDON2):
    ch = seed(params, hash_kind)
    cb = B.AUX_BUILDER(builder) if builder is not None else None
    prep = wl.preprocessed_matrices if wl.preprocessed is not None else None
    rep, rnd = sess.check_constraints(wl.statement, wl.matrices, ch, aux_builder=cb, preprocessed=prep)
    return report_dict(rep), [int(x) for x in rnd]


# ---------------------------------------------------------------------------------------------------------------------
# workloads: valid statements and single-fault variants
# ---------------------------------------------------------------------------------------------------------------------
def ext_program():
    """An EF constraint that is (0, x) when main[1] = x: u * main[1], with u the extension generator."""
    b = AP.ProgramBuilder()
    b.assert_zero(-b.main(0, 0))
    b.assert_zero_ext(b.ext_const(0, 1) * b.main(0, 1))
    return b.serialize()


def ext_workload(log_h):
    t = np.zeros((1 << log_h, 2), dtype=np.uint64)
    return W.Workload([log_h], widths=[2], aux_widths=[0], programs=[ext_program()], traces=[t],
                      log_quotient_degrees=[1], num_aux_values=[0])


def dummy_workload(log_heights, widths=None, seed=W.SEED):
    widths = widths or [9 + 3 * i for i in range(len(log_heights))]
    return W.Workload(log_heights, widths=widths, aux_widths=[1] * len(log_heights), seed=seed,
                      num_aux_values=[0] * len(log_heights))


def valid_case(name):
    """(workload, host builder or None); every one holds."""
    if name == "fib_product":
        return TA.fib_product_workload([5])
    if name == "periodic":
        return TA.periodic_workload(6), None
    if name == "preprocessed":
        return TA.preprocessed_workload((6, 8)), None
    if name == "logup_device":
        return TA.logup_workload(6, device=True)
    if name == "logup_host":
        return TA.logup_workload(6, device=False)
    if name == "big_program":
        return TA.big_program_workload(5), None
    if name == "dummy_mixed":
        return dummy_workload([6, 4, 5]), None
    raise KeyError(name)


VALID = ["fib_product", "periodic", "preprocessed", "logup_device", "logup_host", "big_program", "dummy_mixed"]


def reference_builder(name, builder):
    """The host builder standing for the aux traces of case `name` (the device LogUp build has its host twin)."""
    if name == "logup_device":
        return TA.logup_workload(6, device=False)[1]
    return builder


def _corrupt_aux(builder, row, col, coord):
    def fn(ctx, inst, main, rnd, aux_out, aux_values):
        rc = builder(ctx, inst, main, rnd, aux_out, aux_values)
        idx = row * 2 + 2 * col + coord          # the fib/product AIR has one EF aux column
        aux_out[idx] = (aux_out[idx] + 1) % P
        return rc
    return fn


def _corrupt_aux_value(builder):
    def fn(ctx, inst, main, rnd, aux_out, aux_values):
        rc = builder(ctx, inst, main, rnd, aux_out, aux_values)
        if inst == 0:
            aux_values[1] = (aux_values[1] + 3) % P
        return rc
    return fn


def violation_case(name):
    """(workload, builder) with one deliberate fault."""
    if name.startswith("main_row"):
        wl, bld = TA.fib_product_workload([5])
        n = 1 << 5
        r = {"main_row_first": 0, "main_row_interior": 13, "main_row_last": n - 1}[name]
        wl.traces[0][r, 1] = (int(wl.traces[0][r, 1]) + 1) % P
        return wl, bld
    if name == "aux_cell":
        wl, bld = TA.fib_product_workload([5])
        return wl, _corrupt_aux(bld, 9, 0, 1)
    if name == "aux_value":
        wl, bld = TA.fib_product_workload([5])
        return wl, _corrupt_aux_value(bld)
    if name == "public_value":
        wl, bld = TA.fib_product_workload([5])
        wl.public_values[2] = (int(wl.public_values[2]) + 1) % P
        return wl, bld
    if name == "periodic_value":
        wl = TA.periodic_workload(6)
        wl._periodic_keep[0][2, 1] = 6
        return wl, None
    if name == "preprocessed_cell":
        wl = TA.preprocessed_workload((6, 8))
        wl.preprocessed[1][77, 1] = (int(wl.preprocessed[1][77, 1]) + 5) % P
        return wl, None
    if name == "two_in_one_row":
        wl, bld = TA.fib_product_workload([5])
        wl.traces[0][0, 0] = 2                        # breaks the first-row boundary and the row-0 transition
        return wl, bld
    if name == "ext_c1_only":
        wl = ext_workload(6)
        wl.traces[0][21, 1] = 5
        return wl, None
    if name == "taller_first":
        wl = dummy_workload([7, 5])
        wl.traces[0][100, 0] = 1                      # instance 0 (height 2^7, proof position 1)
        wl.traces[0][100, 1:9] = 3
        wl.traces[1][3, :9] = 2                       # instance 1 (height 2^5, proof position 0)
        return wl, None
    if name == "random_traces":
        wl = dummy_workload([6, 5], widths=[9, 10], seed=77)
        rng = np.random.default_rng(77)
        for t in wl.traces:                           # column 0 random, zero on about half of the rows
            t[:, 0] = rng.integers(0, 2, t.shape[0], dtype=np.uint64) * rng.integers(1, P, t.shape[0], dtype=np.uint64)
        return wl, None
    raise KeyError(name)


def distinct_fields_workload():
    """Three AIRs (heights 2^5, 2^7, 2^6: instance order differs from proof order), faults only in instance 2: constraint
    3 = (2 + 3u) * main[1] is (8, 12) at row 37, constraint 2 = main[2] fails on rows 50..53."""
    b = AP.ProgramBuilder()
    b.assert_zero(-b.main(0, 0))
    b.assert_zero(b.main(0, 0) * b.main(0, 1))
    b.assert_zero(b.main(0, 2))
    b.assert_zero_ext(b.ext_const(2, 3) * b.main(0, 1))
    prog = b.serialize()
    hs = [5, 7, 6]
    ts = [np.zeros((1 << h, 3), dtype=np.uint64) for h in hs]
    ts[2][37, 1] = 4
    ts[2][50:54, 2] = 1
    return W.Workload(hs, widths=[3] * 3, aux_widths=[0] * 3, programs=[prog] * 3, traces=ts, log_quotient_degrees=[1] * 3,
                      num_aux_values=[0] * 3)


DISTINCT = dict(holds=0, kind=1, instance=2, constraint=3, row=37, value=(8, 12), failing_rows=5)
HASHES = [B.HASH_POSEIDON2, B.HASH_BLAKE3, B.HASH_KECCAK, B.HASH_RPO, B.HASH_RPX]

VIOLATIONS = ["main_row_first", "main_row_interior", "main_row_last", "aux_cell", "aux_value", "public_value",
              "periodic_value", "preprocessed_cell", "two_in_one_row", "ext_c1_only", "taller_first", "random_traces"]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the layout and the reference evaluator itself
# ---------------------------------------------------------------------------------------------------------------------
def test_report_layout():
    assert C.sizeof(B.ConstraintReport) == 48
    offs = [getattr(B.ConstraintReport, f).offset for f in ("holds", "kind", "instance", "constraint", "row", "value", "failing_rows")]
    assert offs == [0, 4, 8, 12, 16, 24, 40]
    assert "mdn_check_constraints" in B.EXPORTS


def test_reference_covers_every_op():
    ops = set()
    for name in VALID + ["ext_c1_only"]:
        wl = valid_case(name)[0] if name in VALID else violation_case(name)[0]
        for prog in wl.programs:
            nn = int(prog[2])
            ops |= {int(prog[5 + 3 * j]) for j in range(nn)}
    assert ops == set(range(16))


@pytest.mark.parametrize("name", VALID)
def test_reference_holds_on_valid_statements(name):
    wl, bld = valid_case(name)
    params = W.fast_pcs_params()
    rep, chal = reference(wl, params, reference_builder(name, bld))
    assert rep == dict(NO_FAIL, holds=1, failing_rows=0)
    assert len(chal) == 2 * max(wl._airs[i].num_randomness for i in range(wl.k))


def _ext_fail(ch, av, lh):
    return 3


def _ext_raise(ch, av, lh):
    raise ArithmeticError("reduction")


@pytest.mark.parametrize("name", VALID + VIOLATIONS + ["distinct_fields", "external_assertion"])
def test_oracle_checker_agrees_with_python_evaluator(name):
    """orc_check_constraints (the oracle's restatement of debug.rs) = ref_check, every field and the challenges."""
    params = W.fast_pcs_params()
    ext = None
    if name in VALID:
        wl, bld = valid_case(name)
    elif name == "distinct_fields":
        wl, bld = distinct_fields_workload(), None
    elif name == "external_assertion":
        (wl, bld), ext = violation_case("main_row_interior"), _ext_fail
    else:
        wl, bld = violation_case(name)
    got, rnd = oracle_check(wl, params, bld, ext=ext)
    want, chal = reference(wl, params, reference_builder(name, bld), ext=ext)
    assert (got, rnd) == (want, chal)
    if name == "distinct_fields":
        assert got == DISTINCT


@pytest.mark.parametrize("hash_kind", HASHES)
def test_oracle_checker_hash_configurations(hash_kind):
    params = W.fast_pcs_params()
    wl, bld = TA.fib_product_workload([5])
    wl.traces[0][7, 0] = 3
    assert oracle_check(wl, params, bld, hash_kind) == reference(wl, params, bld, hash_kind)


def test_oracle_checker_errors():
    params = W.fast_pcs_params()
    wl, bld = TA.fib_product_workload([5])
    with pytest.raises(RuntimeError, match="reduction error"):
        oracle_check(wl, params, bld, ext=_ext_raise)
    with pytest.raises(RuntimeError, match="aux builder failed"):
        oracle_check(wl, params, lambda *a: 1)
    with pytest.raises(RuntimeError, match="denominator must be non-zero"):
        oracle_check(_zero_denominator_workload(), params)


def test_reference_locates_hand_derived_faults():
    """Expected reports worked out by hand from the fib/product AIR (constraints: 0 first*(a-p0), 1 first*(b-p1),
    2 tr*(a'-b), 3 tr*(b'-(a+b)), 4 first*(p-1), 5 tr*(p'-p*f), 6 last*(b-p2), 7 last*(p*f-z), 8 0)."""
    params = W.fast_pcs_params()
    n = 32
    wl, bld = violation_case("main_row_first")          # b[0] += 1: constraint 1 at row 0 first
    rep, _ = reference(wl, params, bld)
    assert (rep["kind"], rep["instance"], rep["row"], rep["constraint"], rep["value"]) == (1, 0, 0, 1, (1, 0))
    wl, bld = violation_case("main_row_interior")       # b[13] += 1: b' = a + b fails at row 12
    rep, _ = reference(wl, params, bld)
    assert (rep["row"], rep["constraint"], rep["value"]) == (12, 3, (1, 0))
    wl, bld = violation_case("main_row_last")           # b[N-1] += 1: b' = a + b fails at row N-2 first
    rep, _ = reference(wl, params, bld)
    assert (rep["row"], rep["constraint"]) == (n - 2, 3)
    wl, bld = violation_case("two_in_one_row")
    rep, _ = reference(wl, params, bld)
    assert (rep["row"], rep["constraint"]) == (0, 0)
    wl, _ = violation_case("ext_c1_only")
    rep, _ = reference(wl, params)
    assert (rep["row"], rep["constraint"], rep["value"], rep["failing_rows"]) == (21, 1, (0, 5), 1)
    wl, _ = violation_case("taller_first")
    rep, _ = reference(wl, params)
    assert (rep["instance"], rep["row"], rep["failing_rows"]) == (0, 100, 2)
    wl, _ = violation_case("random_traces")
    rep, _ = reference(wl, params)
    assert all((t[:, 1:9] != 0).all() for t in wl.traces)      # the product fails exactly where column 0 is non-zero
    assert 0 < rep["failing_rows"] == sum(int((t[:, 0] != 0).sum()) for t in wl.traces)


# ---------------------------------------------------------------------------------------------------------------------
# GPU (also run on the emulator, except the tests named h100)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sess():
    s = B.Session(W.fast_pcs_params(), 0)
    yield s
    s.close()


@gpu
@pytest.mark.parametrize("name", VALID)
def test_valid_statements_hold(sess, name):
    wl, bld = valid_case(name)
    params = W.fast_pcs_params()
    got, rnd = device_check(sess, wl, params, bld)
    want, chal = reference(wl, params, reference_builder(name, bld))
    assert got == want == oracle_check(wl, params, bld)[0] == dict(NO_FAIL, holds=1, failing_rows=0)
    assert rnd == chal


@gpu
@pytest.mark.parametrize("hash_kind", HASHES)
def test_hash_configurations(hash_kind):
    params = W.fast_pcs_params()
    s = B.Session(params, 0)
    try:
        s.set_hash(hash_kind, W.initial_hash_challenger(params) if hash_kind in (B.HASH_BLAKE3, B.HASH_KECCAK) else b"")
        wl, bld = TA.fib_product_workload([5])
        got, rnd = device_check(s, wl, params, bld, hash_kind)
        want, chal = reference(wl, params, bld, hash_kind)
        assert rnd == chal
        assert got == want == oracle_check(wl, params, bld, hash_kind)[0] == dict(NO_FAIL, holds=1, failing_rows=0)
        wl.traces[0][7, 0] = 3                            # and a fault under this configuration
        got, rnd = device_check(s, wl, params, bld, hash_kind)
        want, chal = reference(wl, params, bld, hash_kind)
        assert rnd == chal and want["kind"] == 1 and got == want == oracle_check(wl, params, bld, hash_kind)[0]
    finally:
        s.close()


@gpu
@pytest.mark.parametrize("name", VIOLATIONS)
def test_violations_located_like_the_reference(sess, name):
    wl, bld = violation_case(name)
    params = W.fast_pcs_params()
    got, rnd = device_check(sess, wl, params, bld)
    want, chal = reference(wl, params, bld)
    assert rnd == chal
    assert want["kind"] == 1 and want["holds"] == 0
    assert got == want == oracle_check(wl, params, bld)[0]


@gpu
def test_report_fields_distinct_values(sess):
    """Every field of one failure report carries its own expected value (the fault is in instance 2)."""
    wl = distinct_fields_workload()
    got, _ = device_check(sess, wl, W.fast_pcs_params())
    assert got == DISTINCT == oracle_check(wl, W.fast_pcs_params())[0]


@gpu
def test_external_assertion_and_reduction_error(sess):
    params = W.fast_pcs_params()
    wl, bld = TA.fib_product_workload([5])
    wl.traces[0][4, 2] = 1          # column 2 is unconstrained: the rows hold

    def ext_fail(ch, av, lh):
        return 3

    def ext_raise(ch, av, lh):
        raise ArithmeticError("reduction")

    try:
        sess.set_external_check(ext_fail)
        got, _ = device_check(sess, wl, params, bld)
        want, _ = reference(wl, params, bld, ext=ext_fail)
        assert got == want == oracle_check(wl, params, bld, ext=ext_fail)[0] == dict(NO_FAIL, holds=0, kind=2, constraint=3, failing_rows=0)
        wl.traces[0][6, 1] = 9      # with failing rows too: kind 2 still wins, failing_rows is filled
        got, _ = device_check(sess, wl, params, bld)
        want, _ = reference(wl, params, bld, ext=ext_fail)
        assert got == want == oracle_check(wl, params, bld, ext=ext_fail)[0] and got["kind"] == 2 and got["failing_rows"] > 0
        sess.set_external_check(ext_raise)
        with pytest.raises(B.ProverError, match=r"\[-7\].*reduction error"):
            device_check(sess, wl, params, bld)
    finally:
        sess.set_external_check(None)
    wl2, bld2 = TA.fib_product_workload([5])
    assert device_check(sess, wl2, params, bld2)[0]["holds"] == 1


def _too_many_live_values():
    b = AP.ProgramBuilder()
    xs = [b.main(0, 0) for _ in range(1100)]
    acc = xs[0]
    for x in xs[1:]:
        acc = acc + x
    b.assert_zero(acc)
    return b.serialize()


def _zero_denominator_workload():
    lb = AP.LookupProgramBuilder(1)
    lb.insert(0, None, lb.const(1), lb.main(0, 0))            # column 0 of the trace is zero
    b = AP.ProgramBuilder()
    b.assert_zero_ext(b.aux(0, 0) * b.const(0))
    t = W.synthetic_trace(3, 5, 2)
    return W.Workload([5], widths=[2], aux_widths=[1], programs=[b.serialize()], traces=[t], log_quotient_degrees=[1],
                      num_aux_values=[1], lookups=[(1, lb.serialize())])


@gpu
def test_error_paths_leave_the_session_usable(sess):
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)

    def expect(rc, msg, fn):
        with pytest.raises(B.ProverError, match=msg) as e:
            fn()
        assert f"[{rc}]" in str(e.value)
        wl, bld = TA.fib_product_workload([5])
        assert device_check(sess, wl, params, bld)[0]["holds"] == 1

    wl = dummy_workload([5])
    wl.matrices[0].width = 8
    expect(-1, "width 8 does not match", lambda: sess.check_constraints(wl.statement, wl.matrices, ch))
    wl = dummy_workload([5])
    wl.traces[0][3, 2] = P
    expect(-1, "main trace contains a non-canonical", lambda: sess.check_constraints(wl.statement, wl.matrices, ch))
    wl = TA.preprocessed_workload((6, 8))
    expect(-1, "preprocessed presence mismatch", lambda: sess.check_constraints(wl.statement, wl.matrices, ch))
    wl.preprocessed_matrices[1].log_height = 7
    expect(-1, "preprocessed height", lambda: sess.check_constraints(wl.statement, wl.matrices, ch, preprocessed=wl.preprocessed_matrices))
    wl = W.Workload([5], widths=[2], aux_widths=[0], programs=[_too_many_live_values()], log_quotient_degrees=[1], num_aux_values=[0])
    expect(-4, "live values", lambda: sess.check_constraints(wl.statement, wl.matrices, ch))
    wl = _zero_denominator_workload()
    expect(-1, "denominator must be non-zero", lambda: sess.check_constraints(wl.statement, wl.matrices, ch))
    wl, _ = TA.fib_product_workload([5])
    bad = B.AUX_BUILDER(lambda *a: 1)
    expect(-5, "aux builder failed", lambda: sess.check_constraints(wl.statement, wl.matrices, ch, aux_builder=bad))


def _timings(s):
    t = s.timings()
    return bytes(memoryview(t).cast("B"))


@gpu
def test_check_between_proofs_changes_nothing():
    """prove -> check -> prove: identical proof bytes, kernel launches, timings and introspection of the last proof."""
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    s = B.Session(params, 0)
    fresh = B.Session(params, 0)
    try:
        wl, bld = TA.fib_product_workload([6])
        cb = B.AUX_BUILDER(bld)
        p1 = s.prove(wl.statement, wl.matrices, ch, aux_builder=cb)
        launches1 = s.timings().kernel_launches
        t1 = _timings(s)
        info1 = [s.info(w).tolist() for w in (0, 1, 2, 3, 6, 7, 8)]
        bad, bbld = violation_case("main_row_interior")
        rep, _ = s.check_constraints(bad.statement, bad.matrices, ch, aux_builder=B.AUX_BUILDER(bbld))
        assert rep.holds == 0
        assert _timings(s) == t1
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
def test_check_refused_inside_a_staged_proof():
    params = W.fast_pcs_params()
    ch = W.initial_challenger(params, H.oracle_observe)
    wl = dummy_workload([6, 5])
    s = B.Session(params, 0)
    try:
        want = s.prove(wl.statement, wl.matrices, ch)
        L = B.lib()
        root = np.zeros(4, dtype=np.uint64)
        rnd = np.zeros(4, dtype=np.uint64)
        assert L.mdn_prove_begin(s.handle, C.byref(wl.statement), wl.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0
        with pytest.raises(B.ProverError, match=r"\[-1\].*inside a proof"):
            s.check_constraints(wl.statement, wl.matrices, ch)
        assert L.mdn_prove_commit_aux(s.handle, None, None, None) == 0
        pf = B.Proof()
        assert L.mdn_prove_finish(s.handle, C.byref(pf)) == 0
        got = B.proof_to_numpy(pf)
        assert got[0] == want[0] and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
    finally:
        s.close()


@gpu
@pytest.mark.parametrize("log_h", range(16, 23))
def test_h100_last_row_fault_at_every_height(sess, log_h):
    """One non-zero cell at the last row of a narrow AIR, 2^16..2^22 rows: the atomicMin over many blocks finds it."""
    b = AP.ProgramBuilder()
    b.assert_zero(b.main(0, 1) * b.main(0, 0))
    b.assert_zero(b.main(0, 0))
    t = np.zeros((1 << log_h, 2), dtype=np.uint64)
    t[:, 1] = 1
    t[-1, 0] = 9
    wl = W.Workload([log_h], widths=[2], aux_widths=[0], programs=[b.serialize()], traces=[t], log_quotient_degrees=[1],
                    num_aux_values=[0])
    got, _ = device_check(sess, wl, W.fast_pcs_params())
    assert got == dict(holds=0, kind=1, instance=0, constraint=0, row=(1 << log_h) - 1, value=(9, 0), failing_rows=1)


@gpu
def test_h100_miden_shape_holds():
    """The benchmark's statement (2^20 x (51, 22, 16), DummyMidenAir, column 0 zero) satisfies its constraint."""
    params = W.miden_pcs_params()
    s = B.Session(params, 0)
    try:
        wl = W.Workload([20, 20, 20])
        ch = W.initial_challenger(params, H.oracle_observe)
        rep, rnd = s.check_constraints(wl.statement, wl.matrices, ch)
        assert report_dict(rep) == dict(NO_FAIL, holds=1, failing_rows=0)
        assert [int(x) for x in rnd] == oracle_challenges(wl, params)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the -m gpu cases above on the kernel emulator (tests/emu)
# ---------------------------------------------------------------------------------------------------------------------
def test_small_gpu_cases_on_the_emulator():
    emu = os.path.join(ROOT, "tests", "emu")
    subprocess.check_call(["make", "-s", "-C", emu])
    env = dict(os.environ, MDN_LIB_PATH=os.path.join(emu, "libmiden_b200_emu.so"), MDN_ALLOW_EMULATOR="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-k", "not h100",
                        "-p", "no:cacheprovider"], env=env, capture_output=True, text=True, timeout=1800, cwd=ROOT)
    assert r.returncode == 0 and " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-3000:] + r.stderr[-1000:]


def _cpp_check_api(target):
    d = os.path.join(ROOT, "tests", "cpp_check")
    if target.endswith("_emu"):
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "tests", "emu")])
    subprocess.check_call(["make", "-s", "-C", d, target])
    r = subprocess.run([os.path.join(d, target)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "CHECK_API_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@gpu
def test_h100_cpp_host_layer_check_constraints():
    """miden::check_constraints / ConstraintViolation (host/miden_prover.hpp) with the reference's panic texts."""
    _cpp_check_api("test_check_api")


def test_cpp_host_layer_check_constraints_on_the_emulator():
    _cpp_check_api("test_check_api_emu")


def test_check_refused_on_a_split_session_on_the_emulator():
    """A session split over 2 ranks (mdn_session_set_shard) refuses the check with MDN_ERR_UNSUPPORTED and checks again
    once the split is removed: tests/run_check_sharded.py under torchrun, one emulated device per rank."""
    emu = os.path.join(ROOT, "tests", "emu")
    subprocess.check_call(["make", "-s", "-C", emu])
    env = dict(os.environ, MDN_LIB_PATH=os.path.join(emu, "libmiden_b200_emu.so"), MDN_ALLOW_EMULATOR="1", MDN_EMU_SHM="1",
               OMP_NUM_THREADS="1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29741", os.path.join(ROOT, "tests", "run_check_sharded.py")],
                       env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.count("CHECK_SHARD_REFUSED_OK") == 2, r.stdout[-2000:] + r.stderr[-3000:]
