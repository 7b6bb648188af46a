#!/usr/bin/env python3
"""Cost of the three lookup checks (mdn_check_trace_balance, mdn_check_lookup_folds, mdn_lookup_fold_census) on a
Miden-shaped lookup statement, NVRTC row kernels (set_jit(1): k_jit_balance, k_jit_fold, k_jit_fold_census) against
the interpreter (set_jit(0): k_balance_rows, k_fold_rows, k_fold_census_rows).

The statement is modelled on the reference's MainLookupAir (air/src/constraints/lookup/main_air.rs): a requester AIR with
4 LogUp columns and 40 interactions, whose flags are degree-7 products of bit columns read at row offsets 0 and 1 (as
build_op_flags builds the decoder's op flags, all of them before the first message), whose messages are up to
16 wide (MIDEN_MAX_MESSAGE_WIDTH) through LookupProgramBuilder.encode, in cached-encoding groups (two mutually
exclusive sites, one of them a batch) and plain groups.  The multiplicity is a main column: 1 on the requester's trace.
The responder table AIR runs the same lookup program on a copy of the trace whose multiplicity column is p - 1, so it
receives every message the requester sends and the bus closes.  Both AIRs share one lookup program, hence one cubin.

Arms alternate, after one warm-up call each (--reps timed calls per arm and check).  Whole-call times are host clocks
around calls that end in a stream synchronisation inside the library; kernel times come from torch.profiler traces of
separate calls.  Prints the program's node count and interpreter slot tier, then one JSON line with the card's name
and power limit.  MDN_LIB_PATH selects another build of the library, as for bench.py."""
import argparse, json, os, random, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import pkgload

N_BITS, N_VALUES, WIDTH = 10, 16, 16      # bit columns, value columns, MIDEN_MAX_MESSAGE_WIDTH
COL_M = N_BITS + N_VALUES                 # the multiplicity column
MAIN_WIDTH = COL_M + 1
N_COLUMNS = 4


def requester_lookup(AP, P, seed=5):
    """The requester's lookup program (LookupProgramBuilder).  Per LogUp column: three groups of two exclusive sites
    (site 0 one insert, site 1 a batch of two), the first and third with cached encoding, plus one insert of its own:
    40 interactions."""
    rng = random.Random(seed)
    lb = AP.LookupProgramBuilder(N_COLUMNS)
    bit = lambda off, c: lb.main(off, c)

    def factor(off, c, pol):
        b = bit(off, c)
        return b if pol else lb.const(1) - b

    # the op flags first, as build_op_flags: a degree-6 prefix per group, then the two degree-7 site flags
    flags = []
    for col in range(N_COLUMNS):
        for g in range(4):
            picks = rng.sample([(o, c) for o in (0, 1) for c in range(N_BITS)], 7)
            pref = None
            for (o, c) in picks[:6]:
                f = factor(o, c, rng.randrange(2))
                pref = f if pref is None else pref * f
            zo, zc = picks[6]
            flags.append((pref * bit(zo, zc), pref * (lb.const(1) - bit(zo, zc))))
    m = lb.main(0, COL_M)
    k = 0

    def message(k):
        w = 2 + (k * 7) % (WIDTH - 1)            # 2 .. 16 elements
        elems = [lb.const(k + 1)]
        for i in range(1, w):
            elems.append(lb.main(i % 2, N_BITS + (k + 3 * i) % N_VALUES))
        return lb.encode(k % 8, WIDTH, elems)

    for col in range(N_COLUMNS):
        for g in range(3):
            f0, f1 = flags[4 * col + g]
            with lb.group(col, cached=g != 1):
                lb.insert(col, f0, m, message(k)); k += 1
                with lb.batch():
                    lb.insert(col, f1, m, message(k)); k += 1
                    lb.insert(col, f1, m, message(k)); k += 1
        lb.insert(col, flags[4 * col + 3][0], m, message(k)); k += 1
    return lb


def slot_tier(words):
    """The interpreter's slot count for a version-1 lookup program (session.cu compile_oplist: node definitions in order,
    each interaction emitted once its operands are defined, a slot freed after its last use) and its tier."""
    nn, nc = int(words[2]), int(words[3])
    nodes = [(int(words[5 + 3 * j]), int(words[6 + 3 * j]), int(words[7 + 3 * j])) for j in range(nn)]
    items = [tuple(int(x) for x in words[5 + 3 * nn + 4 * q: 9 + 3 * nn + 4 * q]) for q in range(nc)]
    ops = lambda it: [x for x in it[1:] if x != 0xFFFFFFFF]
    evs, q = [], 0
    for j in range(nn):
        evs.append((0, j))
        while q < nc and max(ops(items[q])) <= j:
            evs.append((1, q)); q += 1
    last = [0] * nn
    for e, (kind, x) in enumerate(evs):
        if kind:
            for o in ops(items[x]):
                last[o] = e
        else:
            last[x] = max(last[x], e)
            op, a, b = nodes[x]
            if 10 <= op <= 12:
                last[a] = last[b] = e
            elif op == 13:
                last[a] = e
    live = peak = 0
    for e, (kind, x) in enumerate(evs):
        if not kind:
            live += 1
            peak = max(peak, live)
        used = set(ops(items[x])) if kind else ({nodes[x][1], nodes[x][2]} if 10 <= nodes[x][0] <= 12 else {nodes[x][1]} if nodes[x][0] == 13 else set())
        live -= sum(1 for o in used if last[o] == e)
        if not kind and last[x] == e:
            live -= 1
    return peak, next(t for t in (16, 64, 256, 1024, 1 << 30) if peak <= t)


def statement(W, AP, P, log_n, fault=None, seed=7):
    """(workload, mutex sites, fold marks) of the two-AIR statement at 2^log_n rows.  fault: None (the bus closes and the
    folds hold), "scattered" (on a few requester rows a value column changes and a bit column becomes 2) or "whole"
    (on every requester row)."""
    lb = requester_lookup(AP, P)
    prog = lb.serialize()
    n = 1 << log_n
    rng = np.random.default_rng(seed)
    req = np.zeros((n, MAIN_WIDTH), dtype=np.uint64)
    req[:, :N_BITS] = rng.integers(0, 2, (n, N_BITS), dtype=np.uint64)
    req[:, N_BITS:COL_M] = rng.integers(0, P, (n, N_VALUES), dtype=np.uint64)
    req[:, COL_M] = 1
    resp = req.copy()
    resp[:, COL_M] = P - 1
    if fault == "scattered":
        rows = rng.choice(n, 24, replace=False)
        req[rows[:12], N_BITS + 5] = (req[rows[:12], N_BITS + 5] + 1) % P
        req[rows[12:], 3] = 2
    elif fault == "whole":
        req[:, N_BITS + 5] = (req[:, N_BITS + 5] + 1) % P
        req[:, 3] = 2
    triv = AP.ProgramBuilder()
    triv.assert_zero(triv.const(0))
    wl = W.Workload([log_n, log_n], widths=[MAIN_WIDTH, MAIN_WIDTH], aux_widths=[N_COLUMNS, N_COLUMNS],
                    programs=[triv.serialize()] * 2, traces=[req, resp], log_quotient_degrees=[1, 1],
                    num_aux_values=[1, 1], lookups=[(N_COLUMNS, prog), (N_COLUMNS, prog)])
    return wl, [lb.mutex_sites()] * 2, [lb.fold_marks()] * 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5, help="timed calls of each arm and check (after one warm-up call each)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    from guard_timing import power_limit_w, stats, kernel_ms
    pkg = pkgload.load_pkg()
    B, W, AP = pkg.binding, pkg.workload, pkg.air_program
    P = W.P
    prog = requester_lookup(AP, P).serialize()
    peak, tier = slot_tier(prog)
    print(f"requester lookup program: {int(prog[2])} nodes, {int(prog[3])} interactions, {peak} live values "
          f"(interpreter slot tier {tier})", flush=True)
    rnd = np.array([0x1234567, 0x89ABCDE, 0x13579BD, 0x2468ACE], dtype=np.uint64)
    wl, sites, marks = statement(W, AP, P, a.log_n, "scattered")
    arms = {"nvrtc": B.Session(W.fast_pcs_params(), 0), "interpreter": B.Session(W.fast_pcs_params(), 0)}
    arms["nvrtc"].set_jit(1)
    arms["interpreter"].set_jit(0)
    calls = {
        "check_trace_balance": lambda s: s.check_trace_balance(wl.statement, wl.matrices, rnd, (), sites, 1 << 12),
        "check_lookup_folds": lambda s: s.check_lookup_folds(wl.statement, wl.matrices, rnd, marks),
        "lookup_fold_census": lambda s: s.lookup_fold_census(wl.statement, wl.matrices, rnd, marks, max_failures=1 << 12,
                                                             max_tallies=64)[0].disagreements,
    }
    kernels = {"check_trace_balance": ["k_jit_balance", "k_balance_rows", "k_balance_compare"],
               "check_lookup_folds": ["k_jit_fold", "k_fold_rows", "k_logup_rows", "k_jit("],
               "lookup_fold_census": ["k_jit_fold_census", "k_fold_census_rows", "k_fold_census_list", "k_logup_rows", "k_jit("]}

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, r

    result = {"statement": f"2 AIRs x 2^{a.log_n} rows, width {MAIN_WIDTH}, {N_COLUMNS} LogUp columns, "
                           f"{int(prog[3])} interactions, scattered faults",
              "program": {"nodes": int(prog[2]), "interactions": int(prog[3]), "live_values": peak, "slot_tier": tier},
              "reps": a.reps, "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()},
              "calls": {}}
    try:
        for name, call in calls.items():
            first = {k: timed(lambda s=s: call(s)) for k, s in arms.items()}   # warm-up: compile, load, self-check
            assert str(first["nvrtc"][1]) == str(first["interpreter"][1]), f"{name}: the arms disagree"
            used = {k: [int(x) for x in s.info(B.INFO_JIT_LOOKUP_CHECK)] for k, s in arms.items()}
            wall = {k: [] for k in arms}
            for _ in range(a.reps):
                for k, s in arms.items():
                    wall[k].append(timed(lambda s=s: call(s))[0])
            km = {k: kernel_ms(lambda s=s: call(s), kernels[name], 2) for k, s in arms.items()}
            result["calls"][name] = {"first_call_ms": {k: round(v[0], 1) for k, v in first.items()},
                                     "call_ms": {k: stats(v) for k, v in wall.items()},
                                     "kernel_ms_per_call": km, "jit_lookup_check_info": used}
            print(name, json.dumps(result["calls"][name]), flush=True)
    finally:
        for s in arms.values():
            s.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
