"""LogUp aux traces with register columns built on the device (version-2 lookup programs, `mdn_lookup` in
include/miden_b200.h): a stock LogUp trace followed by registers that start at 0 and follow an affine per-row
recurrence, as the precompile uint chiplets' Schwartz-Zippel columns do.

The statement has two AIRs sharing bus 0, modelled on the uint chiplets:
  MUL   (main c0..c15, m; period-8 roles)  LogUp column 0: insert(always, -m, bus 0 [c0, c1, extras...])
        registers id, S:  S' = keep(r) * S + kappa * sum(r)              (keep = 0 on role 0: a reset; kappa an EF constant)
                          id' = id + first(r) * sum(r) + mid(r) * S * sum(r) - last(r) * (S + 1) * q(r)
        with sum(r) = sum_i beta^i c_i and q(r) = c0 + beta * c1
  STORE (main x0, x1, s, v)                LogUp column 0: insert(s, 1, bus 0 [x0, x1, extras...])
        register id:      id' = id + s * v * beta + x0
Every STORE request names a MUL row, so the bus closes across the two AIRs.  The constraint programs tie the LogUp
column to its fractions and each register to its recurrence (`when_first: reg = 0`, `when_transition:
reg_next - U(reg, row) = 0`), so the oracle verifier checks what the device built.

`KCase` is one AIR with k = 1..4 registers that read each other (reg_i' = keep * reg_i + x2 * reg_{i+1 mod k} + beta * x3
+ (i + 1) * x0, keep = 0 on role 0 of 4), a self-closing LogUp column, and optionally a preprocessed column read by an
update only.

Two references, neither reading the op-lists the device reads:
  * `host_builder` restates the chiplets' trace loops on Python integers (roles by r % 8, registers updated in row
    order, a sequential LogUp build); it is the host aux callback of the comparison proofs;
  * `oracle_builder` lowers the version-2 programs a second time on the CPU (tests/oracle_lookup_registers, over the
    oracle's node evaluator, every row evaluated once in row order); the oracle prover proves through it.
tests/test_lookup_registers_oracle.py checks the two references against each other without a GPU."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import helpers as H
import pkgload
import test_check_constraints as TC
import test_device_resident as DR
from test_lookup_preprocessed import ef_add, ef_mul, ef_inv, extras, enc, enc_expr, refused

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
P = W.P
pytestmark = pytest.mark.gpu
EMU = os.environ.get("MDN_ALLOW_EMULATOR") == "1"
CM = B.FLAG_DEVICE_TRACES | B.FLAG_COLUMN_MAJOR
MUL, STORE = 0, 1
RND = [0x1234567890ABCDEF % P, 0x0FEDCBA987654321 % P, 0x7777777711111111 % P, 0x3141592653589793 % P]
KAPPA = (5, 3)                         # the EF multiplier of S
PERIOD = 8
# periodic columns of MUL: first (role 0), keep (S_KEEP: 0 on role 0), mid (roles 1..6), last (role 7), role 3
PER = np.array([[int(r == 0), int(r != 0), int(1 <= r <= 6), int(r == 7), int(r == 3)] for r in range(PERIOD)], dtype=np.uint64)
ID_TRANSITION = 4                      # MUL's constraint index of `id_next - U_id = 0` (after the three LogUp ones)


def ef_sub(x, y):
    return ((x[0] - y[0]) % P, (x[1] - y[1]) % P)


def ef_pow(x, e):
    r = (1, 0)
    for _ in range(e):
        r = ef_mul(r, x)
    return r


class Case:
    def __init__(self, log_mul, log_store, width=3, seed=5, wrong_role3=False):
        rng = random.Random(seed)
        self.log_mul, self.log_store, self.width, self.wrong = log_mul, log_store, width, wrong_role3
        n, ns = 1 << log_mul, 1 << log_store
        t = np.zeros((n, 17), dtype=np.uint64)
        t[:, 0] = np.arange(n, dtype=np.uint64)
        t[:, 1] = (np.arange(n, dtype=np.uint64) * np.uint64(7) + np.uint64(3))
        t[:, 2:16] = np.array([[rng.randrange(1 << 32) for _ in range(14)] for _ in range(n)], dtype=np.uint64).reshape(n, 14)
        st = np.zeros((ns, 4), dtype=np.uint64)
        rows = np.array([rng.randrange(n) for _ in range(ns)], dtype=np.int64)
        s = np.array([rng.randrange(4) != 0 for _ in range(ns)], dtype=np.uint64)
        st[:, 0], st[:, 1], st[:, 2] = rows, rows * 7 + 3, s
        st[:, 3] = [rng.randrange(1 << 40) for _ in range(ns)]
        st[s == 0, 1] += np.uint64(1)                       # flagged-off rows must not be pushed
        t[:, 16] = np.bincount(rows[s == 1], minlength=n)
        self.mul, self.store = t, st

    # ---- the register updates, on any builder: reg(i) is register i's row-r value
    def mul_updates(self, b, reg):
        c = [b.main(0, q) for q in range(16)]
        beta = b.challenge(1)
        bp, sm = None, c[0]
        for q in range(1, 16):
            bp = beta if bp is None else bp * beta
            sm = sm + bp * c[q]
        q_ = c[0] + beta * c[1]
        first, keep, mid, last, role3 = (b.periodic(q) for q in range(5))
        idr, S = reg(0), reg(1)
        u_id = idr + first * sm + mid * (S * sm) - last * ((S + b.const(1)) * q_)
        if self.wrong:
            u_id = u_id + role3 * b.const(1)
        u_s = keep * S + b.ext_const(*KAPPA) * sm
        return [u_id, u_s]

    def store_updates(self, b, reg):
        x0, _, s, v = (b.main(0, q) for q in range(4))
        return [reg(0) + s * v * b.challenge(1) + x0]

    # ---- lookup programs (registers=False: the same interactions without registers)
    def mul_lookup(self, registers=True):
        lb = AP.LookupProgramBuilder(1, 2 if registers else 0)
        c0, c1, m = lb.main(0, 0), lb.main(0, 1), lb.main(0, 16)
        lb.insert(0, None, -m, lb.encode(0, self.width, extras([c0, c1], self.width)))
        if registers:
            for i, u in enumerate(self.mul_updates(lb, lb.register)):
                lb.update(i, u)
        return lb.serialize()

    def store_lookup(self, registers=True):
        lb = AP.LookupProgramBuilder(1, 1 if registers else 0)
        x0, x1, s = lb.main(0, 0), lb.main(0, 1), lb.main(0, 2)
        lb.insert(0, s, lb.const(1), lb.encode(0, self.width, extras([x0, x1], self.width)))
        if registers:
            lb.update(0, self.store_updates(lb, lb.register)[0])
        return lb.serialize()

    # ---- constraint programs
    @staticmethod
    def _logup(b, d, n):
        a0, a0n = b.aux(0, 0), b.aux(1, 0)
        b.assert_zero_ext(((a0n - a0) * d - n) * b.is_transition())
        b.assert_zero_ext(a0 * b.is_first_row())
        b.assert_zero_ext(((b.aux_value(0) - a0) * d - n) * b.is_last_row())

    @staticmethod
    def _registers(b, updates):
        for i in range(len(updates)):
            b.assert_zero_ext(b.aux(0, 1 + i) * b.is_first_row())
            b.assert_zero_ext((b.aux(1, 1 + i) - updates[i]) * b.is_transition())

    def mul_program(self, registers=True):
        b = AP.ProgramBuilder()
        d = enc_expr(b, 0, self.width, extras([b.main(0, 0), b.main(0, 1)], self.width))
        self._logup(b, d, -b.main(0, 16))
        if registers:
            wrong, self.wrong = self.wrong, False             # the AIR states the true recurrence
            self._registers(b, self.mul_updates(b, lambda i: b.aux(0, 1 + i)))
            self.wrong = wrong
        return b.serialize()

    def store_program(self, registers=True):
        b = AP.ProgramBuilder()
        s = b.main(0, 2)
        b.assert_zero(s * (s - b.const(1)))
        d = enc_expr(b, 0, self.width, extras([b.main(0, 0), b.main(0, 1)], self.width))
        self._logup(b, d, s)
        if registers:
            self._registers(b, self.store_updates(b, lambda i: b.aux(0, 1 + i)))
        return b.serialize()

    def wl(self, device=True, registers=True, only=None):
        """device: the AIRs ship their lowered lookup programs; registers=False: the statement without register columns.
        only: MUL or STORE for a one-AIR statement."""
        nr = [2, 1] if registers else [0, 0]
        airs = [MUL, STORE] if only is None else [only]
        traces = [self.mul, self.store]
        progs = [self.mul_program(registers), self.store_program(registers)]
        lks = [(1, self.mul_lookup(registers)), (1, self.store_lookup(registers))]
        return W.Workload([[self.log_mul, self.log_store][i] for i in airs], widths=[[17, 4][i] for i in airs],
                          aux_widths=[1 + nr[i] for i in airs], programs=[progs[i] for i in airs],
                          traces=[traces[i] for i in airs], log_quotient_degrees=[2] * len(airs),
                          periodic=[[PER, None][i] for i in airs], num_aux_values=[1] * len(airs),
                          lookups=[lks[i] if device else None for i in airs])

    # ---- the independent reference: the chiplets' loops on Python integers
    def aux_rows(self, inst, rnd):
        """(rows [(acc, reg...)], final) of AIR `inst`."""
        al, be, wd = (rnd[0], rnd[1]), (rnd[2], rnd[3]), self.width
        acc, out = (0, 0), []
        if inst == MUL:
            idr, S = (0, 0), (0, 0)
            bpow = [ef_pow(be, q) for q in range(16)]
            for r, row in enumerate(self.mul):
                c = [int(v) for v in row]
                out.append((acc, idr, S))
                acc = ef_add(acc, ef_mul(((P - c[16]) % P, 0), ef_inv(enc(rnd, 0, wd, extras([c[0], c[1]], wd)))))
                sm = (0, 0)
                for q in range(16):
                    sm = ef_add(sm, ef_mul(bpow[q], (c[q], 0)))
                role = r % PERIOD
                nid = idr
                if role == 0:
                    nid = ef_add(nid, sm)
                elif role <= 6:
                    nid = ef_add(nid, ef_mul(S, sm))
                else:
                    nid = ef_sub(nid, ef_mul(ef_add(S, (1, 0)), ef_add((c[0], 0), ef_mul(be, (c[1], 0)))))
                if self.wrong and role == 3:
                    nid = ef_add(nid, (1, 0))
                S = ef_add(S if role != 0 else (0, 0), ef_mul(KAPPA, sm))
                idr = nid
        else:
            idr = (0, 0)
            for row in self.store:
                x0, x1, s, v = (int(q) for q in row)
                out.append((acc, idr))
                if s:
                    acc = ef_add(acc, ef_inv(enc(rnd, 0, wd, extras([x0, x1], wd))))
                idr = ef_add(idr, ef_add(ef_mul((s * v % P, 0), be), (x0, 0)))
        del al
        return out, acc

    def host_builder(self):
        return host_builder(self)

    def oracle_airs(self):
        """Per instance: (lookup program, main trace, periodic matrix, preprocessed matrix) for the C++ lowering."""
        return [(self.mul_lookup(), self.mul, PER, None), (self.store_lookup(), self.store, None, None)]

    def oracle_builder(self):
        return oracle_builder(self)


def host_builder(case):
    def fn(ctx, instance, main, randomness, aux_out, aux_values):
        rows, fin = case.aux_rows(instance, [int(randomness[q]) for q in range(4)])
        flat = np.array([w for row in rows for e in row for w in e], dtype=np.uint64)
        np.ctypeslib.as_array(aux_out, shape=(flat.size,))[:] = flat
        aux_values[0], aux_values[1] = fin
        return 0
    return fn


_olib = None


def _oracle_lib():
    global _olib
    if _olib is None:
        L = C.CDLL(os.path.join(pkgload.ROOT, "tests", "oracle_lookup_registers", "liboracle_lookup_registers.so"))
        u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
        L.orc_logup_aux_registers.restype = C.c_int
        L.orc_logup_aux_registers.argtypes = [C.c_uint32, u32p, C.c_size_t, u64p, C.c_uint32, C.c_uint32, u64p, C.c_uint32,
                                              u64p, C.c_uint32, C.c_uint32, u64p, C.c_uint32, u64p, u64p, u64p]
        L.orc_lookup_registers_error.restype = C.c_char_p
        _olib = L
    return _olib


def oracle_aux(program, main, prep, periodic, rnd, num_columns=1):
    """orc_logup_aux_registers: (aux rows, N x 2 * (num_columns + n_registers) u64, final (c0, c1)) of one AIR; raises
    RuntimeError with the library's message on a refused program."""
    L = _oracle_lib()
    u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
    prog = np.ascontiguousarray(program, dtype=np.uint32)
    main = np.ascontiguousarray(main, dtype=np.uint64)
    prep = None if prep is None else np.ascontiguousarray(prep, dtype=np.uint64)
    per = None if periodic is None else np.ascontiguousarray(periodic, dtype=np.uint64)
    rnd = np.array(rnd, dtype=np.uint64)
    n_regs = int(prog[5]) if len(prog) > 5 else 0
    aux = np.zeros((main.shape[0], 2 * (num_columns + n_regs)), dtype=np.uint64)
    fin = np.zeros(2, dtype=np.uint64)
    ptr64 = lambda a: a.ctypes.data_as(u64p) if a is not None else None
    rc = L.orc_logup_aux_registers(num_columns, prog.ctypes.data_as(u32p), len(prog), ptr64(main), main.shape[0].bit_length() - 1,
                                   main.shape[1], ptr64(prep), 0 if prep is None else prep.shape[1], ptr64(per),
                                   0 if per is None else per.shape[1], 0 if per is None else per.shape[0].bit_length() - 1,
                                   None, 0, ptr64(rnd), ptr64(aux), ptr64(fin))
    if rc != 0:
        raise RuntimeError(L.orc_lookup_registers_error().decode())
    return aux, (int(fin[0]), int(fin[1]))


def oracle_builder(case):
    """The oracle prover's aux callback: the C++ lowering on each AIR's version-2 lookup program."""
    airs = case.oracle_airs()

    def fn(ctx, instance, main, randomness, aux_out, aux_values):
        prog, trace, per, prep = airs[instance]
        aux, fin = oracle_aux(prog, trace, prep, per, [int(randomness[q]) for q in range(4)])
        np.ctypeslib.as_array(aux_out, shape=(aux.size,))[:] = aux.reshape(-1)
        aux_values[0], aux_values[1] = fin
        return 0
    return fn


PER4 = np.array([[int(r != 0)] for r in range(4)], dtype=np.uint64)   # keep: 0 on role 0 of 4 (a reset)


class KCase:
    """One AIR with k registers, main (x0 = r, x1 = a permutation of x0, x2, x3): LogUp column 0 inserts +1 on bus 0 [x0]
    and -1 on bus 0 [x1], so it closes within the AIR; reg_i' = keep * reg_i + x2 * reg_{i+1 mod k} + beta * x3 +
    (i + 1) * x0, plus the preprocessed column 0 for register 0 when `prep`."""

    def __init__(self, k, log_n, seed=3, prep=False):
        rng = random.Random(seed)
        self.k, self.log_n = k, log_n
        n = 1 << log_n
        perm = list(range(n))
        rng.shuffle(perm)
        t = np.zeros((n, 4), dtype=np.uint64)
        t[:, 0] = np.arange(n, dtype=np.uint64)
        t[:, 1] = perm
        t[:, 2] = [rng.randrange(1 << 32) for _ in range(n)]
        t[:, 3] = [rng.randrange(1 << 32) for _ in range(n)]
        self.trace = t
        self.prep = np.array([[rng.randrange(P)] for _ in range(n)], dtype=np.uint64) if prep else None

    def updates(self, b, reg):
        x0, x2, x3, keep = b.main(0, 0), b.main(0, 2), b.main(0, 3), b.periodic(0)
        out = []
        for i in range(self.k):
            u = keep * reg(i) + x2 * reg((i + 1) % self.k) + b.challenge(1) * x3 + b.const(i + 1) * x0
            if self.prep is not None and i == 0:
                u = u + b.preprocessed(0, 0)
            out.append(u)
        return out

    def lookup(self, registers=True):
        lb = AP.LookupProgramBuilder(1, self.k if registers else 0)
        lb.insert(0, None, lb.const(1), lb.encode(0, 3, [lb.main(0, 0)]))
        lb.insert(0, None, -lb.const(1), lb.encode(0, 3, [lb.main(0, 1)]))
        if registers:
            for i, u in enumerate(self.updates(lb, lb.register)):
                lb.update(i, u)
        return lb.serialize()

    def program(self, registers=True):
        b = AP.ProgramBuilder()
        d0, d1 = enc_expr(b, 0, 3, [b.main(0, 0)]), enc_expr(b, 0, 3, [b.main(0, 1)])
        dd, num = d0 * d1, d1 - d0
        a0, a0n = b.aux(0, 0), b.aux(1, 0)
        b.assert_zero_ext(((a0n - a0) * dd - num) * b.is_transition())
        b.assert_zero_ext(a0 * b.is_first_row())
        b.assert_zero_ext(((b.aux_value(0) - a0) * dd - num) * b.is_last_row())
        if registers:
            Case._registers(b, self.updates(b, lambda i: b.aux(0, 1 + i)))
        return b.serialize()

    def wl(self, device=True, registers=True):
        return W.Workload([self.log_n], widths=[4], aux_widths=[1 + (self.k if registers else 0)], programs=[self.program(registers)],
                          traces=[self.trace], log_quotient_degrees=[2], periodic=[PER4], num_aux_values=[1],
                          preprocessed=None if self.prep is None else [self.prep],
                          lookups=[(1, self.lookup(registers)) if device else None])

    def aux_rows(self, inst, rnd):
        be = (rnd[2], rnd[3])
        acc, reg, out = (0, 0), [(0, 0)] * self.k, []
        for r, row in enumerate(self.trace):
            x0, x1, x2, x3 = (int(v) for v in row)
            out.append((acc, *reg))
            acc = ef_add(acc, ef_sub(ef_inv(enc(rnd, 0, 3, [x0])), ef_inv(enc(rnd, 0, 3, [x1]))))
            keep = int(PER4[r % 4, 0])
            nxt = []
            for i in range(self.k):
                u = ef_add(ef_mul((keep, 0), reg[i]), ef_mul((x2, 0), reg[(i + 1) % self.k]))
                u = ef_add(u, ef_add(ef_mul(be, (x3, 0)), ((i + 1) * x0 % P, 0)))
                if self.prep is not None and i == 0:
                    u = ef_add(u, (int(self.prep[r, 0]), 0))
                nxt.append(u)
            reg = nxt
        return out, acc

    def host_builder(self):
        return host_builder(self)

    def oracle_airs(self):
        return [(self.lookup(), self.trace, PER4, self.prep)]

    def oracle_builder(self):
        return oracle_builder(self)


def oracle_check(params, case, got, ch):
    """The oracle prover, its aux traces from the C++ lowering, gives the same bytes, and the oracle verifier accepts
    them."""
    owl = case.wl(False)
    _, heights, fields, comms = H.oracle_prove(params, owl, ch, case.oracle_builder())
    assert DR.same(got, (heights, fields, comms)), "the GPU proof differs from the oracle's"
    rc, err = H.oracle_verify(params, owl, ch, *got)
    assert rc == 0, err


@pytest.fixture(scope="module")
def sess():
    s = B.Session(W.fast_pcs_params(), 0)
    yield s
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# proofs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("heights", [(3, 3), (8, 8), (12, 12), (5, 9), (10, 6), (17, 10)], ids=["2_3", "2_8", "2_12", "mixed_5_9", "mixed_10_6", "2_17"])
def test_device_build_equals_host_builder_and_oracle(sess, heights):
    """2^3 is less than one 128-row block; 2^17 scans 1024 block aggregates in the second phase."""
    params = W.fast_pcs_params()
    case = Case(*heights)
    dev, host = case.wl(True), case.wl(False)
    ch = TC.seed(params)
    got = sess.prove(dev.statement, dev.matrices, ch)
    ref = sess.prove(host.statement, host.matrices, ch, B.AUX_BUILDER(case.host_builder()))
    assert DR.same(got, ref), "the device register build differs from the host builder"
    oracle_check(params, case, got, ch)


@pytest.mark.parametrize("k, log_n", [(3, 4), (3, 9), (4, 4), (4, 9), (1, 10), (2, 6)],
                         ids=["k3_2_4", "k3_2_9", "k4_2_4", "k4_2_9", "k1_2_10", "k2_2_6"])
def test_k_registers_equal_host_builder_and_oracle(sess, k, log_n):
    """Every register count: 2^4 is less than one block; 2^9 is four blocks.  k = 4 runs the register kernels above 48 KiB
    of dynamic shared memory per block."""
    params = W.fast_pcs_params()
    case = KCase(k, log_n)
    dev, host = case.wl(True), case.wl(False)
    ch = TC.seed(params)
    got = sess.prove(dev.statement, dev.matrices, ch)
    ref = sess.prove(host.statement, host.matrices, ch, B.AUX_BUILDER(case.host_builder()))
    assert DR.same(got, ref), "the device register build differs from the host builder"
    oracle_check(params, case, got, ch)
    sess.set_constraint_guard(True)
    try:
        assert DR.same(sess.prove(dev.statement, dev.matrices, ch), got)
    finally:
        sess.set_constraint_guard(False)


def test_register_update_reading_a_preprocessed_column(sess):
    """A preprocessed column read only by a register update: the proof reads the installed bundle's rows and equals the
    host builder's and the oracle's; the three lookup checks run the interaction part only and need no bundle."""
    params = W.fast_pcs_params()
    case = KCase(2, 8, prep=True)
    dev, host = case.wl(True), case.wl(False)
    ch = TC.seed(params)
    sess.set_preprocessed(dev.statement, dev.preprocessed_matrices)
    try:
        got = sess.prove(dev.statement, dev.matrices, ch)
        assert DR.same(got, sess.prove(host.statement, host.matrices, ch, B.AUX_BUILDER(case.host_builder())))
        _, heights, fields, comms = H.oracle_prove(params, host, ch, case.oracle_builder())
        assert DR.same(got, (heights, fields, comms)), "the GPU proof differs from the oracle's"
        rc, err = DR.oracle_verify(params, host, B.HASH_POSEIDON2, got, host.oracle_prep_commitment)
        assert rc == 0, err
    finally:
        sess.set_preprocessed(None, None)
    assert sess.check_trace_balance(dev.statement, dev.matrices, RND)["holds"] == 1
    assert sess.check_lookup_folds(dev.statement, dev.matrices, RND)["holds"] == 1
    out, fails, tallies = sess.lookup_fold_census(dev.statement, dev.matrices, RND)
    assert out.first.holds == 1 and fails == []


def test_trace_layouts_staged_api_and_guard(sess):
    """Row-major and column-major device traces, the staged API, and the guard on and off give the same proof bytes."""
    params = W.fast_pcs_params()
    case = Case(9, 7)
    wl = case.wl(True)
    ch = TC.seed(params)
    ref = sess.prove(wl.statement, wl.matrices, ch)
    mats, bufs = DR.row_major_device_traces(wl)
    assert DR.same(sess.prove(wl.statement, mats, ch, None, B.FLAG_DEVICE_TRACES), ref)
    mats, bufs = DR.column_major_traces(wl)
    assert DR.same(sess.prove(wl.statement, mats, ch, None, CM), ref)
    lib, h = B.lib(), sess.handle
    root, rnd = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
    assert lib.mdn_prove_begin(h, C.byref(wl.statement), wl.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0, lib.mdn_last_error(h)
    assert lib.mdn_prove_commit_aux(h, None, None, None) == 0, lib.mdn_last_error(h)
    proof = B.Proof()
    assert lib.mdn_prove_finish(h, C.byref(proof)) == 0, lib.mdn_last_error(h)
    assert DR.same(B.proof_to_numpy(proof), ref)
    sess.set_constraint_guard(True)
    try:
        assert DR.same(sess.prove(wl.statement, wl.matrices, ch), ref)
        assert sess.last_constraint_report().holds == 1
        assert DR.same(sess.prove(wl.statement, mats, ch, None, CM), ref)
    finally:
        sess.set_constraint_guard(False)
    oracle_check(params, case, ref, ch)


def test_wrong_lowering_is_caught(sess):
    """An id update off by one on role 3: the guard refuses at row 3, mdn_check_constraints reports the same constraint
    and row, and the census lists every role-3 row."""
    params = W.fast_pcs_params()
    case = Case(7, 6, wrong_role3=True)
    wl = case.wl(True)
    ch = TC.seed(params)
    sess.set_constraint_guard(True)
    try:
        with pytest.raises(B.ConstraintViolation) as e:
            sess.prove(wl.statement, wl.matrices, ch)
        rep = e.value.report
        assert (rep.holds, rep.instance, rep.row, rep.constraint) == (0, MUL, 3, ID_TRANSITION)
    finally:
        sess.set_constraint_guard(False)
    rep, _ = sess.check_constraints(wl.statement, wl.matrices, ch)
    assert (rep.holds, rep.instance, rep.row, rep.constraint) == (0, MUL, 3, ID_TRANSITION)
    n = 1 << case.log_mul
    out, fails, tallies, _ = sess.constraint_census(wl.statement, wl.matrices, ch, max_failures=n)
    assert [(f.instance, f.row, f.constraint) for f in fails] == [(MUL, r, ID_TRANSITION) for r in range(3, n, PERIOD)]


# ---------------------------------------------------------------------------------------------------------------------
# the three lookup checks: the report of the program with its registers stripped
# ---------------------------------------------------------------------------------------------------------------------
def aux_matrices(case, wl, logup_only):
    bufs, fins, mats = [], [], (B.Matrix * wl.k)()
    for i in range(wl.k):
        rows, fin = case.aux_rows(i, RND)
        a = np.array([[w for e in (row[:1] if logup_only else row) for w in e] for row in rows], dtype=np.uint64)
        bufs.append(np.ascontiguousarray(a))
        mats[i] = B.Matrix(B.ptr(bufs[-1]), wl.log_heights[i], a.shape[1])
        fins.append(fin)
    mats._keep = bufs
    return mats, bufs, fins


def test_lookup_checks_equal_the_stripped_program(sess):
    case = Case(7, 8)
    wl, strip = case.wl(True), case.wl(True, registers=False)
    assert sess.check_trace_balance(wl.statement, wl.matrices, RND) == sess.check_trace_balance(strip.statement, strip.matrices, RND)
    rep = sess.check_lookup_folds(wl.statement, wl.matrices, RND)
    assert rep["holds"] == 1 and rep == sess.check_lookup_folds(strip.statement, strip.matrices, RND)
    out, fails, tallies = sess.lookup_fold_census(wl.statement, wl.matrices, RND)
    assert out.first.holds == 1 and fails == [] and tallies == []
    # given aux traces: a wrong LogUp cell is reported as for the stripped program; wrong register cells are not compared
    full, fb, ffin = aux_matrices(case, wl, False)
    part, pb, pfin = aux_matrices(case, strip, True)
    for b in (fb, pb):
        b[STORE][9, 0] = (int(b[STORE][9, 0]) + 1) % P
    fb[MUL][5, 2] = (int(fb[MUL][5, 2]) + 1) % P                          # MUL's id register
    got = sess.check_lookup_folds(wl.statement, wl.matrices, RND, aux=full, aux_finals=ffin)
    assert got["holds"] == 0 and (got["instance"], got["column"], got["row"]) == (STORE, 0, 8)
    assert got == sess.check_lookup_folds(strip.statement, strip.matrices, RND, aux=part, aux_finals=pfin)
    a, af, at = sess.lookup_fold_census(wl.statement, wl.matrices, RND, aux=full, aux_finals=ffin)
    b, bf, bt = sess.lookup_fold_census(strip.statement, strip.matrices, RND, aux=part, aux_finals=pfin)
    assert B.fold_report_dict(a.first) == B.fold_report_dict(b.first)
    assert [bytes(f) for f in af] == [bytes(f) for f in bf] and [bytes(t) for t in at] == [bytes(t) for t in bt]


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def store_wl(case, program, aux_width=2, nav=1):
    return W.Workload([case.log_store], widths=[4], aux_widths=[aux_width], programs=[case.store_program(aux_width > 1)],
                      traces=[case.store], log_quotient_degrees=[2], num_aux_values=[nav], lookups=[(1, program)])


def test_refusals(sess):
    case = Case(6, 6)
    ch = TC.seed(W.fast_pcs_params())

    def lb_with(update=None, insert_reg=False, n_regs=1):
        lb = AP.LookupProgramBuilder(1, n_regs)
        x0, x1, s = lb.main(0, 0), lb.main(0, 1), lb.main(0, 2)
        d = lb.encode(0, 3, [x0, x1])
        if insert_reg:
            d = d + lb.register(0)
        lb.insert(0, s, lb.const(1), d)
        for i in range(n_regs):
            lb.update(i, update(lb) if update else lb.register(i) + x0)
        return lb

    def bad(words, text, aux_width=2, nav=1):
        wl = store_wl(case, np.asarray(words, dtype=np.uint32), aux_width, nav)
        for fn in (lambda: sess.prove(wl.statement, wl.matrices, ch),
                   lambda: sess.check_trace_balance(wl.statement, wl.matrices, RND)):
            refused(fn, -1, text)

    good = lb_with().serialize()
    sess.prove(store_wl(case, good).statement, store_wl(case, good).matrices, ch)
    bad(good, "aux_width == num_columns + n_registers", aux_width=3)
    bad(good, "num_aux_values == 1", nav=2)
    w = lb_with().serialize().copy(); w[5] = 0
    bad(w, "bad lookup program length")
    bad(lb_with(n_regs=5).serialize(), "1..=4 registers", aux_width=6)
    bad(lb_with(update=lambda lb: lb.register(0) * lb.register(0)).serialize(), "not affine in the registers")
    bad(lb_with(update=lambda lb: lb.register(0) * (lb.register(0) - lb.register(0))).serialize(), "not affine in the registers")
    bad(lb_with(insert_reg=True).serialize(), "a lookup interaction reads a register")
    lb = lb_with(update=lambda lb: lb.aux(1, 1))
    bad(lb.serialize(), "an AUX leaf must read a register column at offset 0")
    lb = lb_with(update=lambda lb: lb.aux(0, 0))
    bad(lb.serialize(), "an AUX leaf must read a register column at offset 0")
    lb = lb_with(update=lambda lb: lb.is_first_row())
    bad(lb.serialize(), "op 5 is not available to a lookup program")
    # version 1 still refuses the AUX leaf
    lb = AP.LookupProgramBuilder(1)
    lb.insert(0, None, lb.const(1), lb.encode(0, 3, [lb.aux(0, 0)]))
    bad(lb.serialize(), "op 1 is not available to a lookup program", aux_width=1)


# ---------------------------------------------------------------------------------------------------------------------
# NVRTC and size
# ---------------------------------------------------------------------------------------------------------------------
def test_jit_interaction_part():
    """Messages of width 20 put the interaction parts above the NVRTC threshold: the LogUp build is specialised, the
    register columns stay interpreted, and the proof equals the interpreter's."""
    if EMU:
        pytest.skip("NVRTC kernels need the GPU")
    params = W.fast_pcs_params()
    case = Case(7, 8, width=20)
    assert int(case.mul_lookup(False)[2]) >= 256 and int(case.store_lookup(False)[2]) >= 256
    assert B.jit_compile_check(case.mul_lookup()) > 0
    wl = case.wl(True)
    jit, interp = B.Session(params, 0), B.Session(params, 0)
    try:
        jit.set_jit(256); interp.set_jit(0)
        ch = TC.seed(params)
        got = jit.prove(wl.statement, wl.matrices, ch)
        assert 1 in [int(v) for v in jit.info(8)], jit.jit_status()
        assert ";" not in jit.jit_status(), jit.jit_status()
        assert DR.same(got, interp.prove(wl.statement, wl.matrices, ch))
        host = case.wl(False)
        assert DR.same(got, interp.prove(host.statement, host.matrices, ch, B.AUX_BUILDER(case.host_builder())))
    finally:
        jit.close(); interp.close()


def test_2_20_mul_against_the_oracle():
    params = W.fast_pcs_params()
    case = Case(20, 12, seed=20)
    wl = case.wl(True)
    s = B.Session(params, 0)
    try:
        ch = TC.seed(params)
        got = s.prove(wl.statement, wl.matrices, ch)
        oracle_check(params, case, got, ch)
    finally:
        s.close()
