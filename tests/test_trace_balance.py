"""mdn_check_trace_balance: unbalanced LogUp bus messages, found on the device without proving (the reference's
`check_trace_balance`, air/src/lookup/debug/trace/mod.rs:169-309 with builder.rs).

Two references:
  * `ref_balance` below: run_trace_walk + track_mutex + finalize restated with Python integers on the lowered lookup
    op-list (every node over all rows, then every interaction row by row);
  * the CPU oracle's walk, orc_check_trace_balance (tests/oracle_balance: the oracle's C API plus its restatement, with
    the oracle's node evaluator).
The CPU tests pin `ref_balance` on hand-derived faults and the oracle on `ref_balance`; the -m gpu tests compare every
field of the device report with both, from host row-major, row-major device and column-major device traces.  The small
-m gpu cases also run on the kernel emulator of tests/emu (tests/test_trace_balance_emulated.py)."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import oracle_binding as ob
import pkgload

pkg = pkgload.load_pkg()
W, B, AP = pkg.workload, pkg.binding, pkg.air_program
P = W.P
ROOT = pkgload.ROOT
gpu = pytest.mark.gpu
EMU = os.environ.get("MDN_ALLOW_EMULATOR") == "1"
NONE = 0xFFFFFFFF
MW = 2                                   # max_message_width of the buses below
# challenges (alpha, beta) of the fixed cases: the check takes them as an argument
RND = [0x1234567890ABCDEF % P, 0x0FEDCBA987654321 % P, 0x7777777711111111 % P, 0x3141592653589793 % P]


# ---------------------------------------------------------------------------------------------------------------------
# extension-field arithmetic (u^2 = 7) and the bus encoding of LookupProgramBuilder.encode
# ---------------------------------------------------------------------------------------------------------------------
def ef_add(x, y):
    return ((x[0] + y[0]) % P, (x[1] + y[1]) % P)


def ef_mul(x, y):
    return ((x[0] * y[0] + 7 * x[1] * y[1]) % P, (x[0] * y[1] + x[1] * y[0]) % P)


def ef_inv(x):
    n = (x[0] * x[0] - 7 * x[1] * x[1]) % P
    ni = pow(n, P - 2, P)
    return (x[0] * ni % P, (-x[1]) * ni % P)


def enc(rnd, bus, elems):
    """Challenges::encode: alpha + (bus + 1) * beta^MW + sum_i beta^i * elems[i]."""
    al, be = (rnd[0], rnd[1]), (rnd[2], rnd[3])
    g = be
    for _ in range(MW - 1):
        g = ef_mul(g, be)
    acc = ef_add(al, ef_mul(g, (bus + 1, 0)))
    bp = (1, 0)
    for i, e in enumerate(elems):
        if i:
            bp = ef_mul(bp, be)
        acc = ef_add(acc, ef_mul(bp, (int(e) % P, 0)))
    return acc


# ---------------------------------------------------------------------------------------------------------------------
# reference: run_trace_walk + finalize on the op-list, Python integers
# ---------------------------------------------------------------------------------------------------------------------
def _nodes(words, main, periodic, publics, rnd):
    """Every node of a lookup program over all rows: per node (c0 list, c1 list or None for a base value)."""
    w = [int(x) for x in words]
    nn, ni, nk = w[2], w[3], w[4]
    nodes = [tuple(w[5 + 3 * j: 8 + 3 * j]) for j in range(nn)]
    items = [tuple(w[5 + 3 * nn + 4 * q: 9 + 3 * nn + 4 * q]) for q in range(ni)]
    kw = w[5 + 3 * nn + 4 * ni:]
    consts = [kw[2 * j] | (kw[2 * j + 1] << 32) for j in range(nk)]
    n = main.shape[0]
    cols = [[int(x) for x in main[:, c]] for c in range(main.shape[1])]
    per = [[int(x) for x in periodic[:, c]] for c in range(periodic.shape[1])] if periodic is not None else []
    v = []
    for op, a, b in nodes:
        if op == 0:
            col = cols[b]
            x = (col[1:] + col[:1] if a else col, None)
        elif op == 2: x = ([int(publics[a])] * n, None)
        elif op == 3: x = ([rnd[2 * a]] * n, [rnd[2 * a + 1]] * n)
        elif op == 8: x = ([consts[a]] * n, None)
        elif op == 9: x = ([consts[a]] * n, [consts[a + 1]] * n)
        elif op in (10, 11):
            (p0, p1), (q0, q1) = v[a], v[b]
            s = 1 if op == 10 else -1
            c0 = [(u + s * t) % P for u, t in zip(p0, q0)]
            c1 = None if p1 is None and q1 is None else [(u + s * t) % P for u, t in zip(p1 or [0] * n, q1 or [0] * n)]
            x = (c0, c1)
        elif op == 12:
            (p0, p1), (q0, q1) = v[a], v[b]
            if p1 is None and q1 is None:
                x = ([u * t % P for u, t in zip(p0, q0)], None)
            else:
                p1, q1 = p1 or [0] * n, q1 or [0] * n
                x = ([(u0 * t0 + 7 * u1 * t1) % P for u0, u1, t0, t1 in zip(p0, p1, q0, q1)],
                     [(u0 * t1 + u1 * t0) % P for u0, u1, t0, t1 in zip(p0, p1, q0, q1)])
        elif op == 13:
            p0, p1 = v[a]
            x = ([(-u) % P for u in p0], None if p1 is None else [(-u) % P for u in p1])
        elif op == 14:
            col = per[a]
            x = ([col[r % len(col)] for r in range(n)], None)
        else:
            raise ValueError(op)
        v.append(x)
    return v, items


def ref_balance(airs, rnd, boundary=(), mutex_sites=None, max_contributions=1 << 16):
    """airs: per AIR (instance order) dict(lookup words or None, main (N, w), periodic (maxp, n) or None); publics
    shared.  Returns the report as binding.balance_report_dict gives it."""
    balances, log, mutex, skipped = {}, [], [], 0
    for i, a in enumerate(airs):
        if a["lookup"] is None:
            skipped += 1
            continue
        v, items = _nodes(a["lookup"], a["main"], a["periodic"], a.get("publics", ()), rnd)
        n = a["main"].shape[0]
        ann = mutex_sites[i] if mutex_sites is not None else None
        flags = [None if f == NONE else v[f][0] for (_, f, _, _) in items]
        for r in range(n):
            sites = {}
            for q, (col, f, m, d) in enumerate(items):
                active = flags[q] is None or flags[q][r] != 0
                if ann is not None and int(ann[q]) != NONE and active:
                    sites.setdefault((col, int(ann[q]) >> 16), set()).add(int(ann[q]) & 0xFFFF)
                if not active:
                    continue
                key = (v[d][0][r], v[d][1][r] if v[d][1] is not None else 0)
                mult = v[m][0][r]
                balances[key] = (balances.get(key, 0) + mult) % P
                log.append((key, (i, r, col, q, mult)))
            for (col, g), s in sorted(sites.items()):
                if len(s) > 1:
                    mutex.append((i, r, col, g, len(s)))
    for q, (c0, c1, m) in enumerate(boundary):
        key = (int(c0), int(c1))
        balances[key] = (balances.get(key, 0) + int(m)) % P
        log.append((key, (NONE, 2 ** 64 - 1, NONE, q, int(m))))
    unm = sorted(k for k, net in balances.items() if net)
    pushes = {k: [] for k in unm}
    for key, rec in log:
        if key in pushes:
            pushes[key].append(rec)
    um = [(k, balances[k], len(pushes[k]), (pushes[k][0][0], pushes[k][0][1], pushes[k][0][3])) for k in unm]
    n_contrib = sum(len(p) for p in pushes.values())
    complete = n_contrib <= max_contributions
    return dict(holds=int(not unm and not mutex), contributions_complete=int(complete), n_pushes=len(log),
                n_denominators=len(balances), n_unmatched=len(unm), n_mutex_violations=len(mutex), n_contributions=n_contrib,
                n_skipped_airs=skipped, unmatched=um, contributions=[r for k in unm for r in pushes[k]] if complete else [],
                mutex_violations=mutex[:max_contributions])


# ---------------------------------------------------------------------------------------------------------------------
# the closed bus: a table AIR, a lookup AIR of another height, an AIR without lookup, and boundary emissions
# ---------------------------------------------------------------------------------------------------------------------
def _trivial_program():
    b = AP.ProgramBuilder()
    b.assert_zero(b.const(0))
    return b.serialize()


def table_lookup():
    """Table AIR, main [v0, v1, m]: column 0 pushes m / enc(bus 0, [v0, v1]) on every row."""
    lb = AP.LookupProgramBuilder(1)
    with lb.group(0):
        lb.insert(0, None, lb.main(0, 2), lb.encode(0, MW, [lb.main(0, 0), lb.main(0, 1)]))
    return lb


def sender_lookup():
    """Lookup AIR, main [a0, a1, f, x, y, z, s0, s1, s2, h, q], periodic p (period 4):
      column 0, group 0: insert(flag f, -1, bus 0 [a0, a1])                   interaction 0
      column 0, group 1: batch(flag p) { +1 bus 1 [x]; -1 bus 1 [y] }         interactions 1, 2
      column 1, group 0, cached encoding: insert(s0, +1, bus 2 [z]) site 0;   interaction 3
                                          insert(s1, -1, bus 2 [z]) site 1;   interaction 4
                                          batch(s2) { +1 bus 3 [z]; -1 bus 3 [z] } site 2: interactions 5, 6
      column 2, group 0: insert_encoded(flag h, +1, denominator q)            interaction 7"""
    lb = AP.LookupProgramBuilder(3)
    m = [lb.main(0, c) for c in range(11)]
    with lb.group(0):
        lb.insert(0, m[2], lb.const(P - 1), lb.encode(0, MW, [m[0], m[1]]))
    with lb.group(0):
        p = lb.periodic(0)
        with lb.batch():
            lb.insert(0, p, lb.const(1), lb.encode(1, MW, [m[3]]))
            lb.insert(0, p, lb.const(P - 1), lb.encode(1, MW, [m[4]]))
    with lb.group(1, cached=True):
        lb.insert(1, m[6], lb.const(1), lb.encode(2, MW, [m[5]]))
        lb.insert(1, m[7], lb.const(P - 1), lb.encode(2, MW, [m[5]]))
        with lb.batch():
            lb.insert(1, m[8], lb.const(1), lb.encode(3, MW, [m[5]]))
            lb.insert(1, m[8], lb.const(P - 1), lb.encode(3, MW, [m[5]]))
    with lb.group(2):
        lb.insert(2, m[9], lb.const(1), m[10])
    return lb


PERIOD = np.array([[1], [0], [0], [0]], dtype=np.uint64)      # p = 1 on rows r = 0 mod 4
K_F, K_S0, K_S1, K_S2, K_H = 0, 3, 4, 5, 7


class Bus:
    """The closed two-AIR bus (+ one AIR without lookup) of heights 2^log_t (table) and 2^log_l (lookups)."""

    def __init__(self, log_t=5, log_l=7, seed=11, n_boundary=2, third_air=True):
        rng = random.Random(seed)
        nt, nl = 1 << log_t, 1 << log_l
        self.log_t, self.log_l = log_t, log_l
        t = np.zeros((nt, 3), dtype=np.uint64)
        t[:, 0] = [rng.randrange(1, P) for _ in range(nt)]
        t[:, 1] = [rng.randrange(1, P) for _ in range(nt)]
        s = np.zeros((nl, 11), dtype=np.uint64)
        entry = [rng.randrange(nt) for _ in range(nl)]
        s[:, 0] = t[entry, 0]
        s[:, 1] = t[entry, 1]
        s[:, 2] = [rng.randrange(2) for _ in range(nl)]
        for r in range(nl):
            if s[r, 2]:
                t[entry[r], 2] += 1
        s[:, 3] = [rng.randrange(P) for _ in range(nl)]
        s[:, 4] = [rng.randrange(P) for _ in range(nl)]
        rows_p = list(range(0, nl, 4))
        perm = rows_p[:]
        rng.shuffle(perm)
        for r, r2 in zip(rows_p, perm):
            s[r, 4] = s[r2, 3]                                   # y is a permutation of x over the rows where p = 1
        s[:, 5] = [rng.randrange(P) for _ in range(nl)]
        u = [int(s[r, 5]) for r in rows_p]
        rng.shuffle(u)
        for i, r in enumerate(rows_p):
            s[r + 1, 5] = u[i]                                   # the s1 rows consume the z of the s0 rows
        s[0::4, 6] = 1
        s[1::4, 7] = 1
        s[2::4, 8] = 1
        s[:, 10] = [rng.randrange(1, P) for _ in range(nl)]
        self.boundary_entries = [rng.randrange(nt) for _ in range(n_boundary)]
        for e in self.boundary_entries:
            t[e, 2] += 1
        self.entry = entry
        self.table, self.sender = t, s
        self.third_air = third_air

    def boundary(self, rnd):
        """eval_boundary: one -1 emission per boundary entry of the table."""
        return [(*enc(rnd, 0, [self.table[e, 0], self.table[e, 1]]), P - 1) for e in self.boundary_entries]

    def workload(self, which=(0, 1, 2)):
        """The statement of AIRs `which` (0 table, 1 lookups, 2 without lookup), with the per-AIR mutex annotations."""
        tl, sl = table_lookup(), sender_lookup()
        spec = {0: (self.log_t, self.table, tl, None), 1: (self.log_l, self.sender, sl, PERIOD),
                2: (3, np.zeros((8, 2), dtype=np.uint64), None, None)}
        which = [w for w in which if w != 2 or self.third_air]
        sel = [spec[w] for w in which]
        wl = W.Workload([x[0] for x in sel], widths=[x[1].shape[1] for x in sel],
                        aux_widths=[x[2].num_columns if x[2] else 0 for x in sel],
                        programs=[_trivial_program() for _ in sel], traces=[np.ascontiguousarray(x[1]) for x in sel],
                        log_quotient_degrees=[1] * len(sel), num_aux_values=[1 if x[2] else 0 for x in sel],
                        periodic=[x[3] for x in sel], lookups=[(x[2].num_columns, x[2].serialize()) if x[2] else None for x in sel])
        sites = [x[2].mutex_sites() if x[2] else None for x in sel]
        airs = [dict(lookup=x[2].serialize() if x[2] else None, main=x[1], periodic=x[3]) for x in sel]
        return wl, sites, airs


def one_key(log_n=20):
    """2^log_n pushes of multiplicity p - 1 on one denominator: the net is -2^log_n mod p."""
    lb = AP.LookupProgramBuilder(1)
    with lb.group(0):
        lb.insert(0, None, lb.const(P - 1), lb.ext_const(5, 9))
    main = np.zeros((1 << log_n, 1), dtype=np.uint64)
    wl = W.Workload([log_n], widths=[1], aux_widths=[1], programs=[_trivial_program()], traces=[main],
                    log_quotient_degrees=[1], num_aux_values=[1], lookups=[(1, lb.serialize())])
    return wl, [lb.mutex_sites()], [dict(lookup=lb.serialize(), main=main, periodic=None)]


# ---------------------------------------------------------------------------------------------------------------------
# the cases: the closed bus and one hand-made fault at a time
# ---------------------------------------------------------------------------------------------------------------------
def _rows(bus, e):
    return [r for r in range(bus.sender.shape[0]) if bus.sender[r, 2] and bus.entry[r] == e]


def _entry_with_lookups(bus):
    """A table entry some row looks up and no boundary emission consumes."""
    return next(e for e in range(bus.table.shape[0]) if _rows(bus, e) and e not in bus.boundary_entries)


def case(name, seed=11):
    """(bus, boundary, expected unmatched list or None, expected mutex violations or None); the expected lists are
    derived by hand from the fault."""
    bus = Bus(seed=seed)
    bnd = bus.boundary(RND)
    if name == "closed":
        return bus, bnd, [], []
    if name == "cell":                     # one table cell changed: the old denominator keeps the consumers, the new the table push
        e = _entry_with_lookups(bus)
        m = int(bus.table[e, 2])
        old = enc(RND, 0, bus.table[e, :2])
        bus.table[e, 0] = (int(bus.table[e, 0]) + 12345) % P
        new = enc(RND, 0, bus.table[e, :2])
        exp = sorted([(old, P - m, m, (1, _rows(bus, e)[0], K_F)), (new, m, 1, (0, e, 0))])
        return bus, bnd, exp, []
    if name == "multiplicity":
        e = _entry_with_lookups(bus)
        bus.table[e, 2] += 1
        m = int(bus.table[e, 2])
        return bus, bnd, [(enc(RND, 0, bus.table[e, :2]), 1, m, (0, e, 0))], []
    if name == "flag":
        e = _entry_with_lookups(bus)
        r = _rows(bus, e)[0]
        bus.sender[r, 2] = 0
        return bus, bnd, [(enc(RND, 0, bus.table[e, :2]), 1, int(bus.table[e, 2]), (0, e, 0))], []
    if name == "dropped_boundary":
        e = bus.boundary_entries[0]
        return bus, bnd[1:], [(enc(RND, 0, bus.table[e, :2]), 1, int(bus.table[e, 2]), (0, e, 0))], []
    if name == "zero_denominator":
        r = 9
        bus.sender[r, 9], bus.sender[r, 10] = 1, 0
        return bus, bnd, [((0, 0), 1, 1, (1, r, K_H))], []
    if name == "mutex":
        # row 0: s0 and s1 (two sites; s1's extra -1 unbalances bus 2), row 4: s0 and the batch s2 (one site for its two
        # interactions, so two active sites; the batch cancels itself)
        bus.sender[0, 7] = 1
        bus.sender[4, 8] = 1
        z = int(bus.sender[0, 5])
        return bus, bnd, [(enc(RND, 2, [z]), P - 1, 3, (1, 0, K_S0))], [(1, 0, 1, 0, 2), (1, 4, 1, 0, 2)]
    raise KeyError(name)


CASES = ["closed", "cell", "multiplicity", "flag", "dropped_boundary", "zero_denominator", "mutex"]


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's walk (tests/oracle_balance/liboracle_balance.so)
# ---------------------------------------------------------------------------------------------------------------------
_ob_lib = None


def _obl():
    global _ob_lib
    if _ob_lib is None:
        d = os.path.join(ROOT, "tests", "oracle_balance")
        subprocess.check_call(["make", "-s", "-C", d])
        L = C.CDLL(os.path.join(d, "liboracle_balance.so"))
        L.orc_last_error.restype = C.c_char_p
        L.orc_check_trace_balance.restype = C.c_int
        L.orc_check_trace_balance.argtypes = [C.POINTER(ob.Statement), C.POINTER(ob.Matrix), ob.u64p, ob.u64p, C.c_size_t,
                                              C.POINTER(ob.u32p), C.c_uint64, C.POINTER(B.BalanceReport)]
        _ob_lib = L
    return _ob_lib


def _cast(obj, typ):
    return C.cast(C.pointer(obj) if not isinstance(obj, C.Array) else obj, C.POINTER(typ))


def oracle_balance(wl, rnd, boundary=(), mutex_sites=None, max_contributions=1 << 16):
    L = _obl()
    r = np.array(rnd if len(rnd) else [0], dtype=np.uint64)
    bnd = np.array([[int(x) for x in t] for t in boundary] or [[0, 0, 0]], dtype=np.uint64).reshape(-1)
    keep, sites = [], None
    if mutex_sites is not None:
        sites = (ob.u32p * wl.k)()
        for i, m in enumerate(mutex_sites):
            if m is not None:
                keep.append(np.ascontiguousarray(m, dtype=np.uint32))
                sites[i] = keep[-1].ctypes.data_as(ob.u32p)
    rep = B.BalanceReport()
    rc = L.orc_check_trace_balance(_cast(wl.statement, ob.Statement), _cast(wl.matrices, ob.Matrix), ob.ptr(r), ob.ptr(bnd),
                                   len(boundary), sites, max_contributions, C.byref(rep))
    if rc != 0:
        raise RuntimeError(L.orc_last_error().decode())
    return B.balance_report_dict(rep)


def _norm(d):
    """Plain ints and tuples (the ctypes and Python sides give the same values in different containers)."""
    def n(x):
        if isinstance(x, (list, tuple)):
            return tuple(n(y) for y in x)
        return int(x)
    return {k: n(v) for k, v in d.items()}


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the Python reference on hand-derived faults, the oracle on the Python reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_ref_balance_gives_the_hand_derived_report(name):
    bus, bnd, exp_unm, exp_mutex = case(name)
    wl, sites, airs = bus.workload()
    rep = ref_balance(airs, RND, bnd, sites)
    assert rep["unmatched"] == exp_unm
    assert rep["mutex_violations"] == exp_mutex
    assert rep["holds"] == int(name == "closed") and rep["n_skipped_airs"] == 1
    assert rep["n_contributions"] == sum(u[2] for u in exp_unm) and rep["contributions_complete"] == 1
    if name == "mutex":
        # the batch at row 2 (two interactions, one site) alone is never a violation
        assert all(v[1] % 4 != 2 for v in rep["mutex_violations"])


def test_ref_balance_counts_pushes_of_the_closed_bus():
    bus, bnd, _, _ = case("closed")
    wl, sites, airs = bus.workload()
    rep = ref_balance(airs, RND, bnd, sites)
    s = bus.sender
    n_push = bus.table.shape[0] + int(s[:, 2].sum()) + 2 * (s.shape[0] // 4) + int(s[:, 6].sum() + s[:, 7].sum()) + 2 * int(s[:, 8].sum()) + len(bnd)
    assert rep["n_pushes"] == n_push


def test_one_key_sum_is_exact():
    wl, sites, airs = one_key(20)
    rep = ref_balance(airs, RND, (), sites)
    assert rep["unmatched"] == [((5, 9), (-(1 << 20)) % P, 1 << 20, (0, 0, 0))]
    assert rep["contributions_complete"] == 0 and rep["contributions"] == []


@pytest.mark.parametrize("name", CASES + ["one_key_2_20"])
def test_oracle_equals_ref_balance(name):
    if name == "one_key_2_20":
        wl, sites, airs = one_key(20)
        bnd = ()
    else:
        bus, bnd, _, _ = case(name)
        wl, sites, airs = bus.workload()
    assert _norm(oracle_balance(wl, RND, bnd, sites)) == _norm(ref_balance(airs, RND, bnd, sites))


def test_oracle_truncates_contributions_like_ref_balance():
    bus, bnd, _, _ = case("cell")
    wl, sites, airs = bus.workload()
    full = ref_balance(airs, RND, bnd, sites)
    n = full["n_contributions"] - 1
    assert _norm(oracle_balance(wl, RND, bnd, sites, n)) == _norm(ref_balance(airs, RND, bnd, sites, n))


def test_builder_annotates_groups_and_sites():
    sites = sender_lookup().mutex_sites()
    assert [int(x) for x in sites] == [NONE, NONE, NONE, 0, 1, 2, 2, NONE]
    assert len(sender_lookup().serialize()) == len(sender_lookup().serialize())   # serialize() is unchanged by annotations


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the device report against both references
# ---------------------------------------------------------------------------------------------------------------------
def _to_device(a):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if EMU:
        return a.copy()
    import torch
    return torch.from_numpy(a.view(np.int64)).cuda()


def _addr(buf):
    return buf.ctypes.data if EMU else buf.data_ptr()


def traces_for(wl, mode):
    """(mdn_matrix array, flags, buffers to keep alive) for host row-major, row-major device or column-major device."""
    if mode == "host":
        return wl.matrices, 0, None
    bufs = [_to_device(t if mode == "device_rm" else t.T) for t in wl.traces]
    mats = (B.Matrix * wl.k)()
    for i, b in enumerate(bufs):
        mats[i] = B.Matrix(C.cast(C.c_void_p(_addr(b)), B.u64p), wl.log_heights[i], wl.widths[i])
    flags = B.FLAG_DEVICE_TRACES | (B.FLAG_COLUMN_MAJOR if mode == "device_cm" else 0)
    return mats, flags, bufs


_sess = None


def session():
    global _sess
    if _sess is None:
        _sess = B.Session(W.miden_pcs_params(), 0)
    return _sess


@gpu
@pytest.mark.parametrize("mode", ["host", "device_rm", "device_cm"])
@pytest.mark.parametrize("name", CASES)
def test_device_report_equals_both_references(name, mode):
    bus, bnd, exp_unm, exp_mutex = case(name)
    wl, sites, airs = bus.workload()
    mats, flags, keep = traces_for(wl, mode)
    got = _norm(session().check_trace_balance(wl.statement, mats, RND, bnd, sites, flags=flags))
    assert got == _norm(ref_balance(airs, RND, bnd, sites))
    assert got == _norm(oracle_balance(wl, RND, bnd, sites))
    assert got["unmatched"] == _norm(dict(x=exp_unm))["x"]
    assert got["mutex_violations"] == _norm(dict(x=exp_mutex))["x"]


@gpu
@pytest.mark.parametrize("which", [(0,), (1,), (2,), (1, 2)])
def test_per_air_statements_give_the_per_air_report(which):
    """A one-AIR statement is the reference's per-AIR check_trace_balance (no boundary emissions)."""
    bus, _, _, _ = case("closed")
    wl, sites, airs = bus.workload(which)
    got = _norm(session().check_trace_balance(wl.statement, wl.matrices, RND, (), sites))
    assert got == _norm(ref_balance(airs, RND, (), sites))
    assert got["n_skipped_airs"] == int(2 in which)


@gpu
def test_truncated_contributions_are_reported_and_deterministic():
    bus, bnd, _, _ = case("cell")
    wl, sites, airs = bus.workload()
    full = _norm(session().check_trace_balance(wl.statement, wl.matrices, RND, bnd, sites))
    assert full["contributions_complete"] == 1 and len(full["contributions"]) == full["n_contributions"] > 0
    n = full["n_contributions"] - 1
    a = _norm(session().check_trace_balance(wl.statement, wl.matrices, RND, bnd, sites, max_contributions=n))
    b = _norm(session().check_trace_balance(wl.statement, wl.matrices, RND, bnd, sites, max_contributions=n))
    assert a == b == _norm(ref_balance(airs, RND, bnd, sites, n))
    assert a["contributions_complete"] == 0 and a["contributions"] == () and a["unmatched"] == full["unmatched"]


@gpu
def test_two_calls_give_identical_reports():
    bus, bnd, _, _ = case("mutex")
    wl, sites, _ = bus.workload()
    a = session().check_trace_balance(wl.statement, wl.matrices, RND, bnd, sites)
    b = session().check_trace_balance(wl.statement, wl.matrices, RND, bnd, sites)
    assert _norm(a) == _norm(b)


@gpu
@pytest.mark.parametrize("name", ["closed", "cell", "multiplicity", "flag", "dropped_boundary", "mutex"])
def test_logup_finals_plus_boundary_equal_the_unmatched_fractions(name):
    """Public APIs only: the LogUp finals the device builds in mdn_check_constraints (captured by the external check),
    plus the boundary fractions, equal the sum of net / denominator over the unmatched denominators reported with the
    same challenges -- the balance kernels and k_logup_rows see the same pushes."""
    bus, _, _, _ = case(name)
    wl, sites, _ = bus.workload()
    sess = B.Session(W.miden_pcs_params(), 0)
    finals = []

    def capture(ch, av, lh):          # every assertion holds; the aux values are the device-built LogUp finals
        finals.extend(av)
    sess.set_external_check(capture)
    ch = W.initial_challenger(W.miden_pcs_params(), lambda c, f: B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(f, dtype=np.uint64)), len(f)))
    _, rnd = sess.check_constraints(wl.statement, wl.matrices, ch)
    rnd = [int(x) for x in rnd]
    # the fault's boundary with these challenges
    bnd = bus.boundary(rnd)[1:] if name == "dropped_boundary" else bus.boundary(rnd)
    rep = sess.check_trace_balance(wl.statement, wl.matrices, rnd, bnd, sites)
    lhs = (0, 0)
    for av in finals:
        if len(av):
            lhs = ef_add(lhs, (int(av[0]), int(av[1])))
    for c0, c1, m in bnd:
        lhs = ef_add(lhs, ef_mul((int(m), 0), ef_inv((int(c0), int(c1)))))
    rhs = (0, 0)
    for d, net, _, _ in rep["unmatched"]:
        rhs = ef_add(rhs, ef_mul((int(net), 0), ef_inv(d)))
    assert lhs == rhs
    assert rep["holds"] == int(name == "closed")
    sess.close()


@gpu
def test_one_key_2_20_sums_exactly():
    wl, sites, _ = one_key(20)
    got = _norm(session().check_trace_balance(wl.statement, wl.matrices, RND, (), sites))
    assert got["unmatched"] == (((5, 9), (-(1 << 20)) % P, 1 << 20, (0, 0, 0)),)
    assert got == _norm(oracle_balance(wl, RND, (), sites))


@gpu
def test_lookup_2_20_against_table_2_16_matches_the_oracle():
    bus = Bus(log_t=16, log_l=20, seed=3, n_boundary=4)
    bus.sender[1000, 2] ^= 1            # one flipped flag: something to report
    wl, sites, _ = bus.workload()
    bnd = bus.boundary(RND)
    for mode in ("host", "device_cm"):
        mats, flags, keep = traces_for(wl, mode)
        got = _norm(session().check_trace_balance(wl.statement, mats, RND, bnd, sites, flags=flags))
        assert got == _norm(oracle_balance(wl, RND, bnd, sites))
        assert got["n_unmatched"] == 1


def _expect_error(code, fn, text):
    with pytest.raises(B.ProverError) as e:
        fn()
    assert f"[{code}]" in str(e.value) and text in str(e.value), str(e.value)


@gpu
def test_error_paths_are_refused_and_proofs_still_match():
    bus, bnd, _, _ = case("closed")
    wl, sites, _ = bus.workload()
    sess = B.Session(W.miden_pcs_params(), 0)
    run = lambda **kw: sess.check_trace_balance(wl.statement, wl.matrices, kw.get("rnd", RND), kw.get("bnd", bnd), kw.get("sites", sites))
    _expect_error(-1, lambda: run(rnd=[P] + RND[1:]), "randomness word 0 is not a canonical")
    _expect_error(-1, lambda: run(bnd=[(bnd[0][0], bnd[0][1], P)]), "boundary emission 0")
    bad = [s.copy() if s is not None else None for s in sites]
    bad[1][K_S1] = bad[1][K_S0]                  # two inserts with different flags claimed as one site
    _expect_error(-1, lambda: run(sites=bad), "share mutex site")
    bad = list(sites)
    bad[2] = np.zeros(1, dtype=np.uint32)        # an annotation for the AIR without lookup
    _expect_error(-1, lambda: run(sites=bad), "without a lookup program")
    # inside a staged proof: refused without disturbing it
    pw = W.Workload([10, 9, 8])
    ch = W.initial_challenger(W.miden_pcs_params(), lambda c, f: B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(f, dtype=np.uint64)), len(f)))
    root = np.zeros(4, dtype=np.uint64)
    rnd = np.zeros(8, dtype=np.uint64)
    assert B.lib().mdn_prove_begin(sess.handle, C.byref(pw.statement), pw.matrices, C.byref(ch), 0, B.ptr(root), B.ptr(rnd)) == 0
    _expect_error(-1, run, "inside a proof")
    assert B.lib().mdn_prove_commit_aux(sess.handle, None, None, B.ptr(root)) == 0
    proof = B.Proof()
    assert B.lib().mdn_prove_finish(sess.handle, C.byref(proof)) == 0
    staged = B.proof_to_numpy(proof)
    fresh = B.Session(W.miden_pcs_params(), 0)
    ch2 = W.initial_challenger(W.miden_pcs_params(), lambda c, f: B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(f, dtype=np.uint64)), len(f)))
    ref = fresh.prove(pw.statement, pw.matrices, ch2)
    assert staged[0] == ref[0] and np.array_equal(staged[1], ref[1]) and np.array_equal(staged[2], ref[2])
    sess.close(); fresh.close()


@gpu
def test_proof_after_a_balance_check_is_byte_identical():
    pw = W.Workload([10, 9, 8])
    params = W.miden_pcs_params()
    obs = lambda c, f: B.lib().mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(f, dtype=np.uint64)), len(f))
    a = B.Session(params, 0)
    before = a.prove(pw.statement, pw.matrices, W.initial_challenger(params, obs))
    t_before = (a.timings().total, a.timings().kernel_launches)
    info_before = a.info(0)
    bus, bnd, _, _ = case("cell")
    wl, sites, _ = bus.workload()
    a.check_trace_balance(wl.statement, wl.matrices, RND, bnd, sites)
    assert (a.timings().total, a.timings().kernel_launches) == t_before and np.array_equal(a.info(0), info_before)
    after = a.prove(pw.statement, pw.matrices, W.initial_challenger(params, obs))
    assert before[0] == after[0] and np.array_equal(before[1], after[1]) and np.array_equal(before[2], after[2])
    a.close()
