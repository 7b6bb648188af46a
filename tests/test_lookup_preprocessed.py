"""LogUp aux traces built on the device for lookup programs that read preprocessed columns (op 15 in `mdn_lookup`), and
the three lookup checks on such programs.

The statement is modelled on a byte-pair lookup table: a table AIR (LUT) whose preprocessed columns are (a, b, c =
f(a, b), tag) and whose main columns are multiplicities, and a requester AIR that looks messages up from its main
columns under 0/1 flags:
  LUT column 0        : insert(always, -m0, bus 0 [prep a, prep b, prep c, extras...])
  LUT column 1        : insert(periodic flag p, -m1, bus 1 [next-row prep c, prep tag, extras...])
                        p is 1 on the odd rows, so row N - 1 reads prep c of row 0 (the wrap, c >= 7); every case gives that
                        row a non-zero m1
  requester column 0  : insert(flag s, 1, bus 0 [x, y, z, extras...])
  requester column 1  : insert(flag g, 1, bus 1 [u, v, extras...])
`extras` pads a message to the bus width W with values computed from its first elements (W = 18 gives the message
width of the precompile relations and a lookup program above the NVRTC threshold).  Constraints tie every aux column
to those fractions, so the oracle verifier checks the built aux traces.

Two references for the aux traces:
  * `host_builder`, independent of the op-lists: Python integers reading the preprocessed table directly;
  * `oracle_builder`, the op-lists lowered a second time on the CPU (tests/oracle_lookup_prep, op 15 included, over the
    oracle's node evaluator).  The oracle prover proves the LUT through it as its aux callback -- the oracle's own
    lookup-program parser does not take op 15 -- and builds the requester from its own lookup program.
tests/test_lookup_preprocessed_oracle.py checks the two references against each other without a GPU."""
import copy
import ctypes as C
import os
import random

import numpy as np
import pytest

import helpers as H
import pkgload
import test_check_constraints as TC
import test_device_resident as DR

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
P = W.P
pytestmark = pytest.mark.gpu
EMU = os.environ.get("MDN_ALLOW_EMULATOR") == "1"
CM = B.FLAG_DEVICE_TRACES | B.FLAG_COLUMN_MAJOR
LUT, REQ = 0, 1                       # instance order of the two-AIR statement
RND = [0x1234567890ABCDEF % P, 0x0FEDCBA987654321 % P, 0x7777777711111111 % P, 0x3141592653589793 % P]


# ---------------------------------------------------------------------------------------------------------------------
# extension-field arithmetic (u^2 = 7), bus encoding, message extras -- on Python integers and on program builders
# ---------------------------------------------------------------------------------------------------------------------
def ef_add(x, y):
    return ((x[0] + y[0]) % P, (x[1] + y[1]) % P)


def ef_mul(x, y):
    return ((x[0] * y[0] + 7 * x[1] * y[1]) % P, (x[0] * y[1] + x[1] * y[0]) % P)


def ef_inv(x):
    n = (x[0] * x[0] - 7 * x[1] * x[1]) % P
    ni = pow(n, P - 2, P)
    return (x[0] * ni % P, (P - x[1]) * ni % P)


def extras(vs, width):
    """The message padded to `width`: element i past the given ones is (v0 + i + 1) * (v1 + 2i + 3) + v_last * (v0 + 3i + 5);
    works on ints (mod P) and on builder expressions alike."""
    out = list(vs)
    for i in range(width - len(vs)):
        e = (vs[0] + (i + 1)) * (vs[1] + (2 * i + 3)) + vs[-1] * (vs[0] + (3 * i + 5))
        out.append(e % P if isinstance(e, int) else e)
    return out


def enc(rnd, bus, width, elems):
    """Challenges::encode: alpha + (bus + 1) * beta^W + sum_i beta^i * elems[i]."""
    al, be = (rnd[0], rnd[1]), (rnd[2], rnd[3])
    g = be
    for _ in range(width - 1):
        g = ef_mul(g, be)
    acc = ef_add(al, ef_mul(g, (bus + 1, 0)))
    bp = (1, 0)
    for i, e in enumerate(elems):
        if i:
            bp = ef_mul(bp, be)
        acc = ef_add(acc, ef_mul(bp, (int(e) % P, 0)))
    return acc


def enc_expr(b, bus, width, elems):
    """The same encoding as an expression of a constraint program (LookupProgramBuilder.encode for lookup programs)."""
    if isinstance(b, AP.LookupProgramBuilder):
        return b.encode(bus, width, elems)
    be = b.challenge(1)
    g = be
    for _ in range(width - 1):
        g = g * be
    acc = b.challenge(0) + g * b.const(bus + 1)
    bp = None
    for i, e in enumerate(elems):
        bp = None if i == 0 else (be if i == 1 else bp * be)
        acc = acc + (e if i == 0 else bp * e)
    return acc


# ---------------------------------------------------------------------------------------------------------------------
# the statement
# ---------------------------------------------------------------------------------------------------------------------
def f_ab(a, b):
    return (a * b + 3 * a + b + 7) % P


class Case:
    """A LUT of 2^log_lut rows and a requester of 2^log_req rows (log_req None: the LUT alone), bus width `width`.
    wl(device): the Workload whose AIRs ship their lowered lookup programs (device=True), or none (host builder);
    oracle_wl(): the requester's lookup program only (the oracle builds the LUT through host_builder)."""

    def __init__(self, log_lut, log_req=None, width=3, seed=7, lqd=2):
        rng = random.Random(seed)
        self.log_lut, self.log_req, self.width, self.lqd = log_lut, log_req, width, lqd
        n = 1 << log_lut
        bits = log_lut // 2
        r = np.arange(n, dtype=np.uint64)
        a, b = r & np.uint64((1 << bits) - 1), r >> np.uint64(bits)
        c = np.array([f_ab(int(x), int(y)) for x, y in zip(a, b)], dtype=np.uint64)
        tag = (a * np.uint64(5) + b * np.uint64(3)) % np.uint64(11)
        self.prep = np.ascontiguousarray(np.stack([a, b, c, tag], axis=1))
        self.per = np.array([[0], [1]], dtype=np.uint64)          # p: the odd LUT rows serve bus 1, N - 1 among them
        m = np.zeros((n, 2), dtype=np.uint64)
        self.req = None
        if log_req is not None:
            nr = 1 << log_req
            t = np.zeros((nr, 7), dtype=np.uint64)
            xs = np.array([rng.randrange(1 << bits) for _ in range(nr)], dtype=np.uint64)
            ys = np.array([rng.randrange(n >> bits) for _ in range(nr)], dtype=np.uint64)
            s = np.array([rng.randrange(4) != 0 for _ in range(nr)], dtype=np.uint64)
            rows = np.array([2 * rng.randrange(n // 2) + 1 for _ in range(nr)], dtype=np.int64)
            g = np.array([rng.randrange(2) for _ in range(nr)], dtype=np.uint64)
            rows[0], g[0] = n - 1, 1                             # a request served by the wrap row
            t[:, 0], t[:, 1], t[:, 3], t[:, 6] = xs, ys, s, g
            t[:, 2] = [f_ab(int(x), int(y)) for x, y in zip(xs, ys)]
            t[:, 4] = c[(rows + 1) % n]
            t[:, 5] = tag[rows]
            m[:, 0] = np.bincount((xs + (ys << np.uint64(bits)))[s == 1].astype(np.int64), minlength=n)
            m[:, 1] = np.bincount(rows[g == 1], minlength=n)
            # flagged-off rows carry other values: they must not be pushed
            off = s == 0
            t[off, 2] = (t[off, 2] + np.uint64(1)) % np.uint64(P)
            self.req = t
        else:
            m[:, 0] = np.array([rng.randrange(3) for _ in range(n)], dtype=np.uint64)
            m[:, 1] = np.array([rng.randrange(3) for _ in range(n)], dtype=np.uint64)
            m[n - 1, 1] = 2
        self.lut = m
        assert int(self.per[(n - 1) % 2, 0]) == 1 and int(m[n - 1, 1]) != 0, "the wrap row must take part" 

    # ---- lookup programs
    def lut_lookup(self):
        lb = AP.LookupProgramBuilder(2)
        pa, pb, pc, ptag, pc1 = lb.preprocessed(0, 0), lb.preprocessed(0, 1), lb.preprocessed(0, 2), lb.preprocessed(0, 3), lb.preprocessed(1, 2)
        lb.insert(0, None, -lb.main(0, 0), lb.encode(0, self.width, extras([pa, pb, pc], self.width)))
        lb.insert(1, lb.periodic(0), -lb.main(0, 1), lb.encode(1, self.width, extras([pc1, ptag], self.width)))
        return lb.serialize()

    def req_lookup(self):
        lb = AP.LookupProgramBuilder(2)
        x, y, z, s, u, v, g = (lb.main(0, q) for q in range(7))
        lb.insert(0, s, lb.const(1), lb.encode(0, self.width, extras([x, y, z], self.width)))
        lb.insert(1, g, lb.const(1), lb.encode(1, self.width, extras([u, v], self.width)))
        return lb.serialize()

    # ---- constraints: the aux columns against the fractions (logup_workload's shape)
    def _logup_constraints(self, b, d0, d1, n0, n1):
        """Column 0 is the exclusive running sum of n0 / d0 + column 1, column 1 = n1 / d1, the aux value the total."""
        a0, a1, a0n = b.aux(0, 0), b.aux(0, 1), b.aux(1, 0)
        b.assert_zero_ext(a1 * d1 - n1)
        b.assert_zero_ext(((a0n - a0 - a1) * d0 - n0) * b.is_transition())
        b.assert_zero_ext(a0 * b.is_first_row())
        b.assert_zero_ext(((b.aux_value(0) - a0 - a1) * d0 - n0) * b.is_last_row())

    def lut_program(self):
        b = AP.ProgramBuilder()
        pa, pb, pc, ptag, pc1 = b.preprocessed(0, 0), b.preprocessed(0, 1), b.preprocessed(0, 2), b.preprocessed(0, 3), b.preprocessed(1, 2)
        d0 = enc_expr(b, 0, self.width, extras([pa, pb, pc], self.width))
        d1 = enc_expr(b, 1, self.width, extras([pc1, ptag], self.width))
        self._logup_constraints(b, d0, d1, -b.main(0, 0), -(b.main(0, 1) * b.periodic(0)))
        return b.serialize()

    def req_program(self):
        b = AP.ProgramBuilder()
        x, y, z, s, u, v, g = (b.main(0, q) for q in range(7))
        b.assert_zero(s * (s - b.const(1)))
        b.assert_zero(g * (g - b.const(1)))
        d0 = enc_expr(b, 0, self.width, extras([x, y, z], self.width))
        d1 = enc_expr(b, 1, self.width, extras([u, v], self.width))
        self._logup_constraints(b, d0, d1, s, g)
        return b.serialize()

    # ---- workloads
    def wl(self, device=True, lut_lookup=None, req_lookup=None, lut_prep=None):
        """lut_lookup / req_lookup: True / False override `device` per AIR; lut_prep: the LUT's preprocessed matrix."""
        lut_lk = device if lut_lookup is None else lut_lookup
        req_lk = device if req_lookup is None else req_lookup
        prep = self.prep if lut_prep is None else lut_prep
        traces, progs, widths, lhs, pers, preps, lks = [self.lut], [self.lut_program()], [2], [self.log_lut], [self.per], [prep], [(2, self.lut_lookup()) if lut_lk else None]
        if self.req is not None:
            traces.append(self.req); progs.append(self.req_program()); widths.append(7); lhs.append(self.log_req)
            pers.append(None); preps.append(None); lks.append((2, self.req_lookup()) if req_lk else None)
        k = len(traces)
        return W.Workload(lhs, widths=widths, aux_widths=[2] * k, programs=progs, traces=traces,
                          log_quotient_degrees=[self.lqd] * k, periodic=pers, num_aux_values=[1] * k,
                          preprocessed=preps, lookups=lks)

    def oracle_wl(self):
        return self.wl(lut_lookup=False, req_lookup=True)

    # ---- the independent reference builder
    def fractions(self, inst, rnd):
        """Per row (f0, f1): the two columns' fractions, from the traces and the preprocessed table (Python integers)."""
        out, wd = [], self.width
        if inst == LUT:
            n = 1 << self.log_lut
            for r in range(n):
                pa, pb, pc, ptag = (int(v) for v in self.prep[r])
                pc1 = int(self.prep[(r + 1) % n, 2])
                m0, m1 = (int(v) for v in self.lut[r])
                i0 = ef_inv(enc(rnd, 0, wd, extras([pa, pb, pc], wd)))
                f0 = ((P - m0) * i0[0] % P, (P - m0) * i0[1] % P)
                f1 = (0, 0)
                if int(self.per[r % 2, 0]):
                    i1 = ef_inv(enc(rnd, 1, wd, extras([pc1, ptag], wd)))
                    f1 = ((P - m1) * i1[0] % P, (P - m1) * i1[1] % P)
                out.append((f0, f1))
        else:
            for row in self.req:
                x, y, z, s, u, v, g = (int(q) for q in row)
                f0 = ef_inv(enc(rnd, 0, wd, extras([x, y, z], wd))) if s else (0, 0)
                f1 = ef_inv(enc(rnd, 1, wd, extras([u, v], wd))) if g else (0, 0)
                out.append((f0, f1))
        return out

    def aux_rows(self, inst, rnd):
        """(aux rows [(acc, f1)], final): build_logup_aux_trace on the fractions."""
        acc, rows = (0, 0), []
        for f0, f1 in self.fractions(inst, rnd):
            rows.append((acc, f1))
            acc = ef_add(acc, ef_add(f0, f1))
        return rows, acc

    def host_builder(self):
        def fn(ctx, instance, main, randomness, aux_out, aux_values):
            rnd = [int(randomness[q]) for q in range(4)]
            rows, fin = self.aux_rows(instance, rnd)
            flat = np.array([w for (acc, f1) in rows for w in (*acc, *f1)], dtype=np.uint64)
            np.ctypeslib.as_array(aux_out, shape=(flat.size,))[:] = flat
            aux_values[0], aux_values[1] = fin
            return 0
        return fn

    def oracle_builder(self):
        """The aux callback of the oracle prover for the LUT: orc_logup_aux_prep on the LUT's lookup program."""
        prog = np.ascontiguousarray(self.lut_lookup(), dtype=np.uint32)

        def fn(ctx, instance, main, randomness, aux_out, aux_values):
            assert instance == LUT
            m = main.contents
            aux, fin = oracle_aux(prog, np.ctypeslib.as_array(m.values, shape=(m.width << m.log_height,)), m.log_height, m.width,
                                  self.prep, self.per, [int(randomness[q]) for q in range(4)])
            np.ctypeslib.as_array(aux_out, shape=(aux.size,))[:] = aux.reshape(-1)
            aux_values[0], aux_values[1] = fin
            return 0
        return fn


_olib = None


def _oracle_lib():
    global _olib
    if _olib is None:
        L = C.CDLL(os.path.join(pkgload.ROOT, "tests", "oracle_lookup_prep", "liboracle_lookup_prep.so"))
        u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
        L.orc_logup_aux_prep.restype = C.c_int
        L.orc_logup_aux_prep.argtypes = [C.c_uint32, u32p, C.c_size_t, u64p, C.c_uint32, C.c_uint32, u64p, C.c_uint32,
                                         u64p, C.c_uint32, C.c_uint32, u64p, C.c_uint32, u64p, u64p, u64p]
        L.orc_lookup_prep_error.restype = C.c_char_p
        _olib = L
    return _olib


def oracle_aux(program, main, log_height, width, prep, periodic, rnd, num_columns=2):
    """orc_logup_aux_prep: (aux rows, 2^log_height x 2 * num_columns u64, final (c0, c1)) of one AIR; raises
    RuntimeError with the library's message on a refused program."""
    L = _oracle_lib()
    u32p, u64p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
    prog = np.ascontiguousarray(program, dtype=np.uint32)
    main = np.ascontiguousarray(main, dtype=np.uint64)
    prep = None if prep is None else np.ascontiguousarray(prep, dtype=np.uint64)
    per = None if periodic is None else np.ascontiguousarray(periodic, dtype=np.uint64)
    rnd = np.array(rnd, dtype=np.uint64)
    aux = np.zeros((1 << log_height, 2 * num_columns), dtype=np.uint64)
    fin = np.zeros(2, dtype=np.uint64)
    ptr64 = lambda a: a.ctypes.data_as(u64p) if a is not None else None
    rc = L.orc_logup_aux_prep(num_columns, prog.ctypes.data_as(u32p), len(prog), ptr64(main), log_height, width,
                              ptr64(prep), 0 if prep is None else prep.shape[1], ptr64(per), 0 if per is None else per.shape[1],
                              0 if per is None else per.shape[0].bit_length() - 1, None, 0, ptr64(rnd), ptr64(aux), ptr64(fin))
    if rc != 0:
        raise RuntimeError(L.orc_lookup_prep_error().decode())
    return aux, (int(fin[0]), int(fin[1]))


def install(s, wl):
    s.set_preprocessed(wl.statement, wl.preprocessed_matrices)


def oracle_proof(params, case, hash_kind=B.HASH_POSEIDON2):
    """The oracle's proof of the case (LUT aux from oracle_builder) and its preprocessed commitment."""
    owl = case.oracle_wl()
    L = TC._orc()
    init = W.initial_hash_challenger(params) if hash_kind in (B.HASH_BLAKE3, B.HASH_KECCAK) else b""
    ch = TC.seed(params, hash_kind) or B.Challenger()
    assert L.orc_set_hash(hash_kind, init or None, len(init)) == 0
    try:
        _, heights, fields, comms = H.oracle_prove(params, owl, ch, case.oracle_builder())
    finally:
        L.orc_set_hash(0, None, 0)
    return owl, (heights, fields, comms)


def assert_oracle(params, case, got, hash_kind=B.HASH_POSEIDON2):
    owl, ref = oracle_proof(params, case, hash_kind)
    assert DR.same(got, ref), "the GPU proof differs from the oracle's"
    rc, err = DR.oracle_verify(params, owl, hash_kind, got, owl.oracle_prep_commitment)
    assert rc == 0, err


@pytest.fixture(scope="module")
def sess():
    s = B.Session(W.fast_pcs_params(), 0)
    yield s
    s.close()


# ---------------------------------------------------------------------------------------------------------------------
# proofs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hash_kind", [B.HASH_POSEIDON2, B.HASH_BLAKE3])
@pytest.mark.parametrize("heights", [(6, 8), (8, 6), (7, 7)])
def test_device_build_equals_host_builder_and_oracle(hash_kind, heights):
    """Host row-major traces: the device LogUp build (both AIRs) gives the host builder's proof bytes and the oracle's;
    (6, 8) puts the LUT below the requester, so the preprocessed tree is shorter than the LDE domain."""
    params = W.fast_pcs_params()
    case = Case(*heights)
    s = DR.session(params, hash_kind)
    try:
        dev, host = case.wl(True), case.wl(False)
        install(s, dev)
        ch = TC.seed(params, hash_kind)
        got = s.prove(dev.statement, dev.matrices, ch)
        ref = s.prove(host.statement, host.matrices, ch, B.AUX_BUILDER(case.host_builder()))
        assert DR.same(got, ref), "the device LogUp build differs from the host builder"
        assert_oracle(params, case, got, hash_kind)
    finally:
        s.close()


def test_device_trace_layouts(sess):
    """Row-major and column-major device traces give the host-trace proof; the caller's traces stay unchanged."""
    params = W.fast_pcs_params()
    case = Case(6, 9)
    wl = case.wl(True)
    install(sess, wl)
    ch = TC.seed(params)
    ref = sess.prove(wl.statement, wl.matrices, ch)
    mats, bufs = DR.row_major_device_traces(wl)
    assert DR.same(sess.prove(wl.statement, mats, ch, None, B.FLAG_DEVICE_TRACES), ref)
    mats, bufs = DR.column_major_traces(wl)
    assert DR.same(sess.prove(wl.statement, mats, ch, None, CM), ref)
    for t, b in zip(wl.traces, bufs):
        assert np.array_equal(DR.from_device(b), t.T)
    assert_oracle(params, case, ref)


def test_staged_api(sess):
    """begin / commit_aux / finish with both aux traces built on the device equals mdn_prove."""
    params = W.fast_pcs_params()
    case = Case(6, 8)
    wl = case.wl(True)
    install(sess, wl)
    ch = TC.seed(params)
    ref = sess.prove(wl.statement, wl.matrices, ch)
    lib, h = B.lib(), sess.handle
    root, rnd = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
    assert lib.mdn_prove_begin(h, C.byref(wl.statement), wl.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0, lib.mdn_last_error(h)
    assert lib.mdn_prove_commit_aux(h, None, None, None) == 0, lib.mdn_last_error(h)
    proof = B.Proof()
    assert lib.mdn_prove_finish(h, C.byref(proof)) == 0, lib.mdn_last_error(h)
    assert DR.same(B.proof_to_numpy(proof), ref)


def test_guard(sess):
    """The guard re-derives the same preprocessed rows as the LogUp build: guarded proofs equal unguarded ones.  One LUT
    multiplicity that disagrees with its (host-built) aux column is refused at that row."""
    params = W.fast_pcs_params()
    case = Case(6, 8)
    wl = case.wl(True)
    install(sess, wl)
    ch = TC.seed(params)
    ref = sess.prove(wl.statement, wl.matrices, ch)
    sess.set_constraint_guard(True)
    try:
        assert DR.same(sess.prove(wl.statement, wl.matrices, ch), ref)
        assert sess.last_constraint_report().holds == 1
        mats, bufs = DR.column_major_traces(wl)
        assert DR.same(sess.prove(wl.statement, mats, ch, None, CM), ref)
        host = case.wl(False)
        builder = B.AUX_BUILDER(copy.deepcopy(case).host_builder())   # the aux trace of the unaltered multiplicities
        case.lut[37, 0] = (int(case.lut[37, 0]) + 1) % P
        with pytest.raises(B.ConstraintViolation) as e:
            sess.prove(host.statement, host.matrices, ch, builder)
        rep = e.value.report
        assert (rep.holds, rep.kind, rep.instance, rep.row, rep.failing_rows) == (0, 1, LUT, 37, 1)
        assert rep.constraint == 1       # the running-sum transition of column 0
    finally:
        sess.set_constraint_guard(False)


def test_jit_lookup_program_reading_preprocessed_columns():
    """Messages of width 18: lookup programs of several hundred nodes, NVRTC-compiled (the LUT's constraint program as
    well, which MDN_INFO_JIT reports); the proof equals the interpreter's and the host builder's."""
    if EMU:
        pytest.skip("NVRTC kernels need the GPU")
    params = W.fast_pcs_params()
    case = Case(6, 7, width=18)
    assert int(case.lut_lookup()[2]) >= 256 and int(case.req_lookup()[2]) >= 256
    wl = case.wl(True)
    jit, interp = B.Session(params, 0), B.Session(params, 0)
    try:
        jit.set_jit(256); interp.set_jit(0)
        for s in (jit, interp):
            install(s, wl)
        ch = TC.seed(params)
        got = jit.prove(wl.statement, wl.matrices, ch)
        assert 1 in [int(v) for v in jit.info(8)], jit.jit_status()
        # no note: both lookup kernels compiled, loaded and agreed with the interpreter on their first use
        assert ";" not in jit.jit_status(), jit.jit_status()
        assert DR.same(got, interp.prove(wl.statement, wl.matrices, ch))
        host = case.wl(False)
        assert DR.same(got, interp.prove(host.statement, host.matrices, ch, B.AUX_BUILDER(case.host_builder())))
        assert_oracle(params, case, got)
    finally:
        jit.close(); interp.close()


def test_2_20_requester_against_a_2_16_lut():
    """A 2^20-row requester against the 2^16-row LUT: GPU = oracle, bit for bit."""
    params = W.fast_pcs_params()
    case = Case(16, 20, seed=20)
    wl = case.wl(True)
    s = B.Session(params, 0)
    try:
        install(s, wl)
        got = s.prove(wl.statement, wl.matrices, TC.seed(params))
        assert_oracle(params, case, got)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# mdn_check_trace_balance
# ---------------------------------------------------------------------------------------------------------------------
def ref_unmatched(case):
    """(denominator, net multiplicity, pushes, (instance, row, interaction) of the least push) of every unbalanced
    denominator, ascending, from the traces and the table (Python integers)."""
    acc = {}
    n, wd = 1 << case.log_lut, case.width

    def push(d, m, key):
        net, cnt, first = acc.get(d, (0, 0, None))
        acc[d] = ((net + m) % P, cnt + 1, key if first is None or key < first else first)
    for r in range(n):
        pa, pb, pc, ptag = (int(v) for v in case.prep[r])
        push(enc(RND, 0, wd, extras([pa, pb, pc], wd)), -int(case.lut[r, 0]), (LUT, r, 0))
        if int(case.per[r % 2, 0]):
            push(enc(RND, 1, wd, extras([int(case.prep[(r + 1) % n, 2]), ptag], wd)), -int(case.lut[r, 1]), (LUT, r, 1))
    for r, row in enumerate(case.req):
        x, y, z, s, u, v, g = (int(q) for q in row)
        if s:
            push(enc(RND, 0, wd, extras([x, y, z], wd)), 1, (REQ, r, 0))
        if g:
            push(enc(RND, 1, wd, extras([u, v], wd)), 1, (REQ, r, 1))
    return sorted((d, net, cnt, first) for d, (net, cnt, first) in acc.items() if net), sum(c for _, c, _ in acc.values()), len(acc)


def test_trace_balance(sess):
    case = Case(6, 9)
    wl = case.wl(True)
    install(sess, wl)
    rep = sess.check_trace_balance(wl.statement, wl.matrices, RND)
    assert rep["holds"] == 1 and rep["n_unmatched"] == 0 and rep["n_skipped_airs"] == 0, rep
    um, pushes, distinct = ref_unmatched(case)
    assert um == [] and (rep["n_pushes"], rep["n_denominators"]) == (pushes, distinct)
    # one wrong LUT multiplicity: that table row's message is unmatched, field for field as the Python balance has it
    case.lut[20, 0] = (int(case.lut[20, 0]) + 2) % P
    wl = case.wl(True)
    rep = sess.check_trace_balance(wl.statement, wl.matrices, RND)
    um, pushes, distinct = ref_unmatched(case)
    assert len(um) == 1 and rep["holds"] == 0
    assert rep["unmatched"] == um and (rep["n_pushes"], rep["n_denominators"]) == (pushes, distinct)
    contrib = sorted(c for c in rep["contributions"])
    assert contrib[0] == (LUT, 20, 0, 0, (P - int(case.lut[20, 0])) % P)


def test_trace_balance_with_the_table_skipped(sess):
    """The LUT given without its lookup program: skipped, so every request it serves is unmatched (what a statement
    without preprocessed lookups had to do)."""
    case = Case(6, 9)
    wl = case.wl(lut_lookup=False, req_lookup=True)
    install(sess, wl)
    rep = sess.check_trace_balance(wl.statement, wl.matrices, RND)
    assert rep["holds"] == 0 and rep["n_skipped_airs"] == 1
    assert rep["n_unmatched"] == rep["n_denominators"] > 0
    assert all(first[0] == REQ for _, _, _, first in rep["unmatched"])


# ---------------------------------------------------------------------------------------------------------------------
# mdn_check_lookup_folds / mdn_lookup_fold_census
# ---------------------------------------------------------------------------------------------------------------------
def aux_matrices(case, wl):
    """The reference aux traces (row-major) and closing values of both AIRs, as the fold checks take them."""
    bufs, fins = [], []
    mats = (B.Matrix * wl.k)()
    for i in range(wl.k):
        rows, fin = case.aux_rows(i, RND)
        bufs.append(np.ascontiguousarray(np.array([[*acc, *f1] for acc, f1 in rows], dtype=np.uint64)))
        mats[i] = B.Matrix(B.ptr(bufs[-1]), wl.log_heights[i], 4)
        fins.append(fin)
    mats._keep = bufs
    return mats, bufs, fins


def test_lookup_folds(sess):
    case = Case(6, 8)
    wl = case.wl(True)
    install(sess, wl)
    rep = sess.check_lookup_folds(wl.statement, wl.matrices, RND)
    assert rep["holds"] == 1 and rep["failing_rows"] == 0, rep
    out, fails, tallies = sess.lookup_fold_census(wl.statement, wl.matrices, RND)
    assert out.first.holds == 1 and out.disagreements == 0 and fails == [] and tallies == []
    mats, bufs, fins = aux_matrices(case, wl)
    assert sess.check_lookup_folds(wl.statement, wl.matrices, RND, aux=mats, aux_finals=fins)["holds"] == 1
    # one faulty fraction cell of LUT column 1 at the wrap row N - 1 (odd: the periodic flag is 1 there; its message reads
    # prep c of row 0): the closed-form fold of that single-interaction column is (V, U) = (-m1, d1), expected V / U
    r = (1 << case.log_lut) - 1
    good = (int(bufs[LUT][r, 2]), int(bufs[LUT][r, 3]))
    bufs[LUT][r, 2] = (good[0] + 5) % P
    m1 = int(case.lut[r, 1])
    d1 = enc(RND, 1, case.width, extras([int(case.prep[0, 2]), int(case.prep[r, 3])], case.width))
    V, U = ((P - m1) % P, 0), d1
    assert ef_mul(V, ef_inv(U)) == good
    want = dict(holds=0, kind=1, instance=LUT, column=1, row=r, fold=(*V, *U), expected=good,
                actual=((good[0] + 5) % P, good[1]), failing_rows=1, zero_u=0, n_skipped_airs=0)
    assert sess.check_lookup_folds(wl.statement, wl.matrices, RND, aux=mats, aux_finals=fins) == want
    out, fails, tallies = sess.lookup_fold_census(wl.statement, wl.matrices, RND, aux=mats, aux_finals=fins)
    assert B.fold_report_dict(out.first) == want
    assert (out.disagreements, out.n_failures, out.failing_columns, out.n_tallies) == (1, 1, 1, 1)
    f = fails[0]
    assert (f.instance, f.column, f.kind, f.row, tuple(f.fold), tuple(f.expected), tuple(f.actual)) == \
        (LUT, 1, 1, r, want["fold"], want["expected"], want["actual"])
    t = tallies[0]
    assert (t.instance, t.column, t.failing_rows, t.zero_u_rows, t.first_row, t.last_row, t.first_kind,
            tuple(t.first_expected), tuple(t.first_actual)) == (LUT, 1, 1, 0, r, r, 1, want["expected"], want["actual"])


# ---------------------------------------------------------------------------------------------------------------------
# mdn_check_constraints / mdn_constraint_census: the call's own preprocessed argument
# ---------------------------------------------------------------------------------------------------------------------
def test_checks_read_the_calls_preprocessed_argument(sess):
    """The LogUp build of the constraint checks reads the call's `preprocessed`, as their row checks do, and not the
    bundle: with a bundle of another table installed the statement holds; were the build reading the bundle, its
    fractions would break the LogUp constraints on the rows where the tables differ."""
    params = W.fast_pcs_params()
    case = Case(6, 8)
    wl = case.wl(True)
    other = case.prep.copy()
    other[:, 2] = (other[:, 2] + np.uint64(1)) % np.uint64(P)
    owl = case.wl(True, lut_prep=other)
    for bundle in (None, owl):
        if bundle is None:
            sess.set_preprocessed(None, None)
        else:
            install(sess, bundle)
        rep, _ = sess.check_constraints(wl.statement, wl.matrices, TC.seed(params), preprocessed=wl.preprocessed_matrices)
        assert rep.holds == 1 and rep.failing_rows == 0
        out, fails, tallies, _ = sess.constraint_census(wl.statement, wl.matrices, TC.seed(params), preprocessed=wl.preprocessed_matrices)
        assert out.first.holds == 1 and fails == []
    # the wrong table as the argument while the proof's table is installed: the constraint rows read it as well, and
    # the device build must agree with them -- it holds, and the bundle is not consulted
    install(sess, wl)
    rep, _ = sess.check_constraints(owl.statement, owl.matrices, TC.seed(params), preprocessed=owl.preprocessed_matrices)
    assert rep.holds == 1


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def refused(fn, code, text):
    with pytest.raises(B.ProverError) as e:
        fn()
    assert f"[{code}]" in str(e.value) and text in str(e.value), str(e.value)


def test_op15_needs_preprocessed_columns(sess):
    case = Case(6, 8)
    wl = case.wl(True)
    # the requester declares no preprocessed columns: a lookup program of its reading op 15 is refused
    lb = AP.LookupProgramBuilder(2)
    lb.insert(0, None, lb.const(1), lb.encode(0, 3, [lb.preprocessed(0, 0)]))
    bad = W.Workload([6], widths=[7], aux_widths=[2], programs=[case.req_program()], traces=[case.req[:64].copy()],
                     log_quotient_degrees=[2], num_aux_values=[1], lookups=[(2, lb.serialize())])
    sess.set_preprocessed(None, None)
    refused(lambda: sess.prove(bad.statement, bad.matrices, TC.seed(W.fast_pcs_params())), -1, "AIR 0: preprocessed column out of range")
    refused(lambda: sess.check_trace_balance(bad.statement, bad.matrices, RND), -1, "AIR 0: preprocessed column out of range")
    # ops a LookupBuilder does not expose are still refused
    lb = AP.LookupProgramBuilder(2)
    lb.insert(0, None, lb.const(1), lb.encode(0, 3, [lb.aux(0, 0)]))
    bad2 = W.Workload([6], widths=[7], aux_widths=[2], programs=[case.req_program()], traces=[case.req[:64].copy()],
                      log_quotient_degrees=[2], num_aux_values=[1], lookups=[(2, lb.serialize())])
    refused(lambda: sess.check_trace_balance(bad2.statement, bad2.matrices, RND), -1, "op 1 is not available to a lookup program")
    # with one, it proves
    install(sess, wl)
    sess.prove(wl.statement, wl.matrices, TC.seed(W.fast_pcs_params()))


def test_lookup_checks_need_the_bundle(sess):
    case = Case(6, 8)
    wl = case.wl(True)
    calls = [lambda: sess.check_trace_balance(wl.statement, wl.matrices, RND),
             lambda: sess.check_lookup_folds(wl.statement, wl.matrices, RND),
             lambda: sess.lookup_fold_census(wl.statement, wl.matrices, RND)]
    sess.set_preprocessed(None, None)
    for fn in calls:
        refused(fn, -1, "AIR 0: its lookup program reads preprocessed columns, but the installed preprocessed bundle does not hold AIR 0")
    short = Case(5, 8)
    install(sess, short.wl(True))
    for fn in calls:
        refused(fn, -1, "AIR 0: the installed preprocessed bundle holds it as 2^5 rows of 4 columns, the call needs 2^6 rows of 4")
    # programs that read no preprocessed column do not consult the bundle
    req_only = W.Workload([8], widths=[7], aux_widths=[2], programs=[case.req_program()], traces=[case.req],
                          log_quotient_degrees=[2], num_aux_values=[1], lookups=[(2, case.req_lookup())])
    assert sess.check_trace_balance(req_only.statement, req_only.matrices, RND)["n_pushes"] > 0
    assert sess.check_lookup_folds(req_only.statement, req_only.matrices, RND)["holds"] == 1
    install(sess, wl)
    rep = calls[0]()
    assert rep["holds"] == 1 and rep["n_skipped_airs"] == 0
    rep = calls[1]()
    assert rep["holds"] == 1 and rep["failing_rows"] == 0 and rep["n_skipped_airs"] == 0
    out, fails, tallies = calls[2]()
    assert out.first.holds == 1 and out.disagreements == 0 and fails == [] and tallies == []
