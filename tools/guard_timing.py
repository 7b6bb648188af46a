#!/usr/bin/env python3
"""Cost of the constraint guard (mdn_session_set_constraint_guard) inside a proof, and of the trace checks
(mdn_check_constraints, mdn_constraint_census), on two 2^20 x (51, 22, 16) statements from host traces:
  * the benchmark statement (DummyMidenAir, 19 nodes: below the JIT threshold, interpreted on every arm);
  * Miden-size constraint programs, about 5.2 k operations per row over the three AIRs, built as in
    tools/realistic_air_probe.py but with every constraint written as e * z, z a main column that is zero on the trace
    (zero_column_air), so that the statement holds and no compiler can fold a constraint away.
Three sessions alternate per statement, after one warm-up proof each (--reps timed proofs each): guard on with the
default JIT threshold (the NVRTC check kernel k_jit_check on the Miden-size programs), guard on with set_jit(0) (the
interpreter's k_check_rows -- and, as set_jit(0) turns off every NVRTC kernel, the interpreted proof constraint
evaluation as well), guard off.  Whole-proof times are host clocks around calls that end in a stream synchronisation
inside the library, next to mdn_timings.total.  The check calls alternate the same way on the JIT and the interpreter
session, on the holding statement and on one with z non-zero on 1000 rows (the census's tallies).  Kernel times
(k_jit_check, k_check_rows, k_jit_census, k_census_rows) and the guard's raw-main copies (device-to-device memcpy) come
from torch.profiler traces of separate runs.  Prints one JSON line with the card's name and power limit, and also writes
it to --out when that is given.  MDN_LIB_PATH selects another build of the library, as for bench.py."""
import argparse, ctypes as C, json, os, random, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import pkgload


def power_limit_w():
    import torch
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def zero_column_air(AP, P, width, aux_width, n_ops, n_constraints, seed):
    """realistic_air_probe.random_air over main columns [0, width - 1) with every constraint e written as e * z, z =
    main column width - 1.  The statement holds where z is zero and fails where it is not; unlike `acc - acc`, no
    compiler can fold the chain away, so the interpreter and the NVRTC check kernel do the same work."""
    rng = random.Random(seed)
    b = AP.ProgramBuilder()
    per = max(2, n_ops // n_constraints)
    cols = width - 1
    for c in range(n_constraints):
        acc = b.main(0, rng.randrange(cols))
        for _ in range(per // 2):
            x = b.main(rng.randrange(2), rng.randrange(cols))
            k = rng.randrange(4)
            acc = acc * x if k == 0 else (acc + x if k == 1 else (acc - x * b.main(0, rng.randrange(cols)) if k == 2 else acc + b.const(rng.randrange(P))))
        z = b.main(0, cols)
        if aux_width and c % 7 == 0:
            b.assert_zero_ext((b.aux(0, rng.randrange(aux_width)) * acc + b.challenge(c % 2)) * z)
        else:
            b.assert_zero(acc * z)
    return b.serialize()


# the three Miden-size AIRs: main width, aux width, operations, constraints (realistic_air_probe.py)
MIDEN_SIZE = [(51, 4, 3400, 120, 1), (22, 3, 1300, 60, 2), (16, 1, 500, 30, 3)]


def stats(xs):
    return {"median": round(float(np.median(xs)), 2), "range": [round(min(xs), 2), round(max(xs), 2)]}


def kernel_ms(fn, names, reps):
    """Device time per call of the kernels whose names contain one of `names`, and of device-to-device copies, from a
    torch.profiler trace of `reps` calls of fn."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names + ["Memcpy DtoD"]}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        for n in out:
            if n in ev.name:
                out[n] += ev.device_time / 1e3 / reps
    return {n: round(v, 3) for n, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=7, help="timed calls of each arm (after one warm-up call of each)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    pkg = pkgload.load_pkg()
    B, W, AP = pkg.binding, pkg.workload, pkg.air_program
    lib = B.lib()
    params = W.miden_pcs_params()

    def observe(c, felts):
        lib.mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))

    ch = W.initial_challenger(params, observe)
    arms = {"guard_jit": B.Session(params, 0), "guard_interpreter": B.Session(params, 0), "guard_off": B.Session(params, 0)}
    arms["guard_jit"].set_constraint_guard(True)
    arms["guard_interpreter"].set_constraint_guard(True)
    arms["guard_interpreter"].set_jit(0)
    lh = a.log_n
    miden = W.Workload([lh] * 3, programs=[zero_column_air(AP, W.P, *spec) for spec in MIDEN_SIZE])
    for i, t in enumerate(miden.traces):
        t[:, miden.widths[i] - 1] = 0
    statements = {"benchmark (DummyMidenAir)": W.Workload([lh] * 3), "Miden-size programs (e * z)": miden}
    result = {"shape": f"2^{lh} x (51, 22, 16), host traces, miden_pcs_params", "reps": a.reps,
              "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()}, "statements": {}}
    check_kernels = ["k_jit_check", "k_check_rows", "k_jit_census", "k_census_rows"]

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, r

    try:
        for name, wl in statements.items():
            prove = {k: (lambda s=s: s.prove(wl.statement, wl.matrices, ch)) for k, s in arms.items()}
            proofs = {k: fn() for k, fn in prove.items()}
            ref = proofs["guard_off"]
            for k, pf in proofs.items():
                assert pf[0] == ref[0] and np.array_equal(pf[1], ref[1]) and np.array_equal(pf[2], ref[2]), f"{k} changed the proof"
            wall = {k: [] for k in arms}
            total = {k: [] for k in arms}
            for _ in range(a.reps):
                for k, fn in prove.items():
                    w, _ = timed(fn)
                    wall[k].append(w); total[k].append(arms[k].timings().total)
            entry = {"nodes_per_air": [int(p[2]) for p in wl.programs], "constraints_per_air": [int(p[3]) for p in wl.programs],
                     "proof_wall_ms": {k: stats(v) for k, v in wall.items()},
                     "proof_timings_total_ms": {k: stats(v) for k, v in total.items()},
                     "jit_check_used": {k: [int(x) for x in arms[k].info(11)] for k in ("guard_jit", "guard_interpreter")},
                     "kernel_class4_ms_last_proof": {k: round(s.timings().kernel_ms[4], 3) for k, s in arms.items()},
                     "commit_aux_ms_last_proof": {k: round(s.timings().commit_aux, 3) for k, s in arms.items()},
                     "kernel_launches": {k: s.timings().kernel_launches for k, s in arms.items()},
                     "guard_kernels_ms_per_proof": {k: kernel_ms(prove[k], check_kernels, a.reps) for k in ("guard_jit", "guard_interpreter")}}
            # the check calls: JIT session against interpreter session, holding and failing statement
            calls = {}
            faulty = W.Workload(wl.log_heights, programs=wl.programs) if name.startswith("Miden") else None
            if faulty is not None:
                rng = np.random.default_rng(20)
                for i, t in enumerate(faulty.traces):
                    t[:, faulty.widths[i] - 1] = 0
                    rows = rng.choice(1 << lh, 333 + i, replace=False)
                    t[rows, faulty.widths[i] - 1] = rng.integers(1, W.P, len(rows), dtype=np.uint64)
            for case, stmt in (("holds", wl), ("1002 failing rows", faulty)):
                if stmt is None:
                    continue
                sess = {"jit": arms["guard_jit"], "interpreter": arms["guard_interpreter"]}
                fns = {}
                for k, s in sess.items():
                    fns[f"check_{k}"] = lambda s=s: s.check_constraints(stmt.statement, stmt.matrices, ch)[0]
                    fns[f"census_{k}"] = lambda s=s: s.constraint_census(stmt.statement, stmt.matrices, ch, max_failures=1 << 12, max_tallies=1 << 10)[0]
                outs = {k: fn() for k, fn in fns.items()}
                assert bytes(outs["check_jit"]) == bytes(outs["check_interpreter"]) and bytes(outs["census_jit"]) == bytes(outs["census_interpreter"])
                times = {k: [] for k in fns}
                for _ in range(a.reps):
                    for k, fn in fns.items():
                        times[k].append(timed(fn)[0])
                calls[case] = {"call_wall_ms": {k: stats(v) for k, v in times.items()},
                               "violations": int(outs["census_jit"].violations),
                               "kernels_ms_per_call": {k: kernel_ms(fn, check_kernels, a.reps) for k, fn in fns.items()}}
            entry["check_calls"] = calls
            result["statements"][name] = entry
    finally:
        for s in arms.values():
            s.close()
    line = json.dumps(result)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
