"""NVRTC-specialised trace-check kernels (jit.hpp MODE_CHECK: k_jit_check, k_jit_census) against the op-list
interpreter (k_check_rows, k_census_rows).

A session with set_jit(1) specialises every program; one with set_jit(0) interprets every program.  On the same calls
the two must give equal mdn_check_constraints reports (field by field), byte-equal mdn_constraint_census outputs
(truncated and not), and, with the constraint guard on, byte-identical proofs or the same refusal and report.
MDN_INFO_JIT_CHECK (info 11) tells which path ran.  The workloads and fault builders are those of
tests/test_check_constraints.py and tests/test_constraint_census.py; the Miden-size programs are those of
tools/guard_timing.py (every constraint e * z with z a main column that is zero on a holding trace)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import helpers as H
import pkgload
import test_airs as TA
import test_check_constraints as TC
import test_constraint_census as TCC
import test_constraint_guard as TG
import test_device_resident as TDR

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
P = W.P
ROOT = pkgload.ROOT
gpu = pytest.mark.gpu
INFO_JIT_CHECK = 11
sys.path.insert(0, os.path.join(ROOT, "tools"))
import guard_timing as GT  # noqa: E402


def miden_size(log_h, faults=0, seed=7):
    """The three Miden-size AIRs of tools/guard_timing.py at height 2^log_h; `faults` rows per AIR with z != 0."""
    progs = [GT.zero_column_air(AP, P, *spec) for spec in GT.MIDEN_SIZE]
    wl = W.Workload([log_h] * 3, programs=progs)
    rng = np.random.default_rng(seed)
    for i, t in enumerate(wl.traces):
        t[:, wl.widths[i] - 1] = 0
        if faults:
            rows = rng.choice(1 << log_h, faults + i, replace=False)
            t[rows, wl.widths[i] - 1] = rng.integers(1, P, len(rows), dtype=np.uint64)
    return wl


@pytest.fixture(scope="module")
def pair():
    jit, interp = B.Session(W.fast_pcs_params(), 0), B.Session(W.fast_pcs_params(), 0)
    jit.set_jit(1)
    interp.set_jit(0)
    yield jit, interp
    jit.close(); interp.close()


def used(s, k):
    v = [int(x) for x in s.info(INFO_JIT_CHECK)]
    assert len(v) == k
    return v


def both(pair, wl, bld=None, ext=None, layout="host", **kw):
    """device_census (census + check report) on the JIT and the interpreter session: equal, and each took its path."""
    jit, interp = pair
    params = W.fast_pcs_params()
    got = TCC.device_census(jit, wl, params, bld, ext, layout=layout, **kw)
    assert used(jit, wl.k) == [1] * wl.k, jit.jit_status()
    want = TCC.device_census(interp, wl, params, bld, ext, layout=layout, **kw)
    assert used(interp, wl.k) == [0] * wl.k
    assert got == want
    assert "disagreed" not in jit.jit_status()
    return got


CASES = TC.VALID + ["one_cell", "whole_column", "boundary_rows", "two_heights", "more_constraints_than_shared",
                    "external_and_rows", "logup_main_cell", "host_aux_cell"]


@gpu
@pytest.mark.parametrize("name", CASES)
def test_check_and_census_equal_the_interpreter(pair, name):
    wl, bld, _, ext = TCC.any_case(name)
    got, rep, _ = both(pair, wl, bld, ext)
    assert both(pair, wl, bld, ext, max_failures=3, max_tallies=2)[1] == rep     # truncated lists
    if name not in TC.VALID:
        assert got["violations"] > 0
    if name == "external_and_rows":
        assert rep["kind"] == 2 and rep["failing_rows"] > 0


@gpu
@pytest.mark.parametrize("name", ["fib_product", "logup_device", "two_heights", "more_constraints_than_shared", "one_cell"])
def test_trace_layouts(pair, name):
    """Column-major and row-major device traces take the JIT path and give what host traces give."""
    wl, bld, _, ext = TCC.any_case(name)
    host = both(pair, wl, bld, ext)
    assert both(pair, wl, bld, ext, layout="cm") == host
    if bld is None and wl.preprocessed is None and ext is None:
        jit, interp = pair
        params = W.fast_pcs_params()
        assert TCC._row_major_device(jit, wl, params) == TCC._row_major_device(interp, wl, params) == host[0]
        assert used(jit, wl.k) == [1] * wl.k


@gpu
@pytest.mark.parametrize("log_h", [12, 16])
@pytest.mark.parametrize("faults", [0, 40])
def test_miden_size_programs(pair, log_h, faults):
    wl = miden_size(log_h, faults)
    got, rep, _ = both(pair, wl)
    assert both(pair, wl, max_failures=10, max_tallies=7)[1] == rep
    assert (got["violations"] == 0) == (faults == 0)
    if faults:
        assert got["first"]["failing_rows"] == 3 * faults + 3


@gpu
def test_big_program_with_faults_equals_the_oracle(pair):
    jit, _ = pair
    params = W.fast_pcs_params()
    wl = miden_size(12, 25, seed=11)
    got, rep, _ = TCC.device_census(jit, wl, params, max_failures=200, max_tallies=400)
    assert used(jit, wl.k) == [1] * wl.k
    assert rep == TC.oracle_check(wl, params)[0]
    assert got == TCC.oracle_census(wl, params, max_failures=200, max_tallies=400)
    assert got["violations"] > 200


# ---------------------------------------------------------------------------------------------------------------------
# the constraint guard
# ---------------------------------------------------------------------------------------------------------------------
def guard_sessions(hash_kind=B.HASH_POSEIDON2):
    params = W.fast_pcs_params()
    g_jit, g_int, off = (TG.hash_session(params, hash_kind, True), TG.hash_session(params, hash_kind, True),
                         TG.hash_session(params, hash_kind, False))
    g_jit.set_jit(1); g_int.set_jit(0)
    return g_jit, g_int, off


@gpu
@pytest.mark.parametrize("hash_kind", [B.HASH_POSEIDON2, B.HASH_BLAKE3])
@pytest.mark.parametrize("name", ["fib_product", "preprocessed", "logup_device", "big_program", "miden_size"])
def test_guard_identical_proofs(name, hash_kind):
    params = W.fast_pcs_params()
    if name == "miden_size":
        wl, bld = miden_size(10), None
    else:
        wl, bld = TC.valid_case(name)
    g_jit, g_int, off = guard_sessions(hash_kind)
    try:
        a, _ = TG.prove(g_jit, wl, params, bld, hash_kind)
        assert used(g_jit, wl.k) == [1] * wl.k and "disagreed" not in g_jit.jit_status()
        b, _ = TG.prove(g_int, wl, params, bld, hash_kind)
        assert used(g_int, wl.k) == [0] * wl.k
        c, _ = TG.prove(off, wl, params, bld, hash_kind)
        assert TDR.same(a, b) and TDR.same(a, c)
        assert TC.report_dict(g_jit.last_constraint_report()) == TC.report_dict(g_int.last_constraint_report()) == TG.HOLDS
    finally:
        g_jit.close(); g_int.close(); off.close()


@gpu
@pytest.mark.parametrize("name", TG.FAULTS + ["miden_size"])
def test_guard_refusals_equal(name):
    params = W.fast_pcs_params()
    if name == "miden_size":
        wl, bld = miden_size(10, 5), None
    else:
        wl, bld = TG.fault_case(name)
    g_jit, g_int, off = guard_sessions()
    try:
        reps = []
        for s in (g_jit, g_int):
            with pytest.raises(B.ConstraintViolation) as e:
                TG.prove(s, wl, params, bld)
            reps.append((TC.report_dict(e.value.report), TC.report_dict(s.last_constraint_report()), str(e.value)))
        assert reps[0] == reps[1] and reps[0][0]["kind"] == 1
        assert used(g_jit, wl.k) == [1] * wl.k and used(g_int, wl.k) == [0] * wl.k
    finally:
        g_jit.close(); g_int.close(); off.close()


@gpu
def test_guard_staged_api():
    params = W.fast_pcs_params()
    wl, bld = TA.fib_product_workload([5, 6])
    g_jit, g_int, off = guard_sessions()
    try:
        proofs = [TG.staged(s, wl, params, TG.staged_aux(wl, bld)) for s in (g_jit, g_int, off)]
        assert all(rc == 0 for rc, _ in proofs)
        assert TDR.same(proofs[0][1], proofs[1][1]) and TDR.same(proofs[0][1], proofs[2][1])
        assert used(g_jit, wl.k) == [1] * wl.k

        def corrupt(bufs):                                 # instance 0, row 9, the c1 coordinate of its EF aux column
            bufs[0][0][9 * 2 + 1] = (int(bufs[0][0][9 * 2 + 1]) + 1) % P
        reps = []
        for s in (g_jit, g_int):
            assert TG.staged(s, wl, params, TG.staged_aux(wl, bld, corrupt))[0] == B.ERR_CONSTRAINT_VIOLATED
            reps.append(TC.report_dict(s.last_constraint_report()))
        assert reps[0] == reps[1] and reps[0]["kind"] == 1
    finally:
        g_jit.close(); g_int.close(); off.close()


# ---------------------------------------------------------------------------------------------------------------------
# Miden-size programs at the benchmark's height
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("faults", [0, 333])
def test_h100_miden_size_2_20(faults):
    params = W.miden_pcs_params()
    jit, interp = B.Session(params, 0), B.Session(params, 0)
    jit.set_jit(1); interp.set_jit(0)
    try:
        wl = miden_size(20, faults, seed=20)
        ch = W.initial_challenger(params, H.oracle_observe)
        out = []
        for s in (jit, interp):
            c, f, t, _ = s.constraint_census(wl.statement, wl.matrices, ch, max_failures=1 << 12, max_tallies=64)
            rep, _ = s.check_constraints(wl.statement, wl.matrices, ch)
            out.append((TCC.census_dict(c, f, t), TC.report_dict(rep), used(s, 3)))
        assert out[0][:2] == out[1][:2]
        assert out[0][2] == [1, 1, 1] and out[1][2] == [0, 0, 0]
        assert out[0][1]["failing_rows"] == (3 * faults + 3 if faults else 0)
        assert "disagreed" not in jit.jit_status()
    finally:
        jit.close(); interp.close()


@gpu
def test_self_check_with_torch_bundled_nvrtc():
    """tests/run_check_jit_old_nvrtc.py: torch's older NVRTC on the 10 k-node program through check, census and guard."""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "run_check_jit_old_nvrtc.py")], capture_output=True,
                       text=True, timeout=1800, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "SELF-CHECK OK" in r.stdout or "NOTE" in r.stdout or "SKIP" in r.stdout, r.stdout[-3000:]
