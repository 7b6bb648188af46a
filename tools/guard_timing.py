#!/usr/bin/env python3
"""Cost of the constraint guard (mdn_session_set_constraint_guard) inside a proof, on two 2^20 x (51, 22, 16) statements
from host traces:
  * the benchmark statement (DummyMidenAir, 19 nodes);
  * Miden-size constraint programs, about 5.2 k operations per row over the three AIRs, built as in
    tools/realistic_air_probe.py but with every constraint written as `acc - acc`, so that the statement holds and the
    guard's interpreter does the same work as on the real AIRs.
Per statement, after one warm-up proof on each, guarded and unguarded proofs alternate (--reps each, two sessions).
Whole-proof times are host clocks around calls that end in a stream synchronisation inside the library, next to
mdn_timings.total.  The guard's kernel time (k_check_rows, plus nothing else on these statements: no preprocessed
columns) and the raw-main copies (device-to-device memcpy, absent without the guard for non-LogUp AIRs) come from a
torch.profiler trace of separate guarded proofs.  Prints one JSON line with the card's name and power limit, and also
writes it to --out when that is given.  MDN_LIB_PATH selects another build of the library, as for bench.py."""
import argparse, ctypes as C, json, os, random, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import pkgload


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def holding_air(AP, P, width, aux_width, n_ops, n_constraints, seed):
    """realistic_air_probe.random_air with every constraint e written as e - e (zero on any trace)."""
    rng = random.Random(seed)
    b = AP.ProgramBuilder()
    per = max(2, n_ops // n_constraints)
    for c in range(n_constraints):
        acc = b.main(0, rng.randrange(width))
        for _ in range(per // 2):
            x = b.main(rng.randrange(2), rng.randrange(width))
            k = rng.randrange(4)
            acc = acc * x if k == 0 else (acc + x if k == 1 else (acc - x * b.main(0, rng.randrange(width)) if k == 2 else acc + b.const(rng.randrange(P))))
        if aux_width and c % 7 == 0:
            e = b.aux(0, rng.randrange(aux_width)) * acc + b.challenge(c % 2)
            b.assert_zero_ext(e - e)
        else:
            b.assert_zero(acc - acc)
    return b.serialize()


def stats(xs):
    return {"median": round(float(np.median(xs)), 2), "range": [round(min(xs), 2), round(max(xs), 2)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=7, help="timed proofs of each (after one warm-up proof of each)")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W, AP = pkg.binding, pkg.workload, pkg.air_program
    lib = B.lib()
    params = W.miden_pcs_params()

    def observe(c, felts):
        lib.mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))

    ch = W.initial_challenger(params, observe)
    on, off = B.Session(params, 0), B.Session(params, 0)
    on.set_constraint_guard(True)
    lh = a.log_n
    statements = {
        "benchmark (DummyMidenAir)": W.Workload([lh] * 3),
        "Miden-size programs (acc - acc)": W.Workload([lh] * 3, programs=[
            holding_air(AP, W.P, 51, 4, 3400, 120, 1), holding_air(AP, W.P, 22, 3, 1300, 60, 2), holding_air(AP, W.P, 16, 1, 500, 30, 3)]),
    }
    result = {"shape": f"2^{lh} x (51, 22, 16), host traces, miden_pcs_params", "reps": a.reps,
              "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()}, "statements": {}}
    try:
        for name, wl in statements.items():
            def run(s):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pf = s.prove(wl.statement, wl.matrices, ch)
                torch.cuda.synchronize()
                return (time.perf_counter() - t0) * 1e3, s.timings().total, pf

            _, _, p_on = run(on)
            _, _, p_off = run(off)
            assert p_on[0] == p_off[0] and np.array_equal(p_on[1], p_off[1]) and np.array_equal(p_on[2], p_off[2]), "the guard changed the proof"
            wall = {"on": [], "off": []}
            total = {"on": [], "off": []}
            for _ in range(a.reps):
                for key, s in (("on", on), ("off", off)):
                    w, t, _ = run(s)
                    wall[key].append(w); total[key].append(t)
            t_on = on.timings()
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    on.prove(wl.statement, wl.matrices, ch)
                torch.cuda.synchronize()
            check_ms, dtod_ms = 0.0, 0.0
            for ev in prof.events():
                if ev.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                if "k_check_rows" in ev.name:
                    check_ms += ev.device_time / 1e3 / a.reps
                elif "Memcpy DtoD" in ev.name:
                    dtod_ms += ev.device_time / 1e3 / a.reps
            result["statements"][name] = {
                "nodes_per_air": [int(p[2]) for p in wl.programs], "constraints_per_air": [int(p[3]) for p in wl.programs],
                "proof_wall_ms": {"guard_on": stats(wall["on"]), "guard_off": stats(wall["off"])},
                "proof_timings_total_ms": {"guard_on": stats(total["on"]), "guard_off": stats(total["off"])},
                "guard_k_check_rows_ms_per_proof": round(check_ms, 3),
                "raw_main_copy_ms_per_proof": round(dtod_ms, 3),
                "kernel_class4_ms_guard_on_last_proof": round(t_on.kernel_ms[4], 3),
                "commit_aux_ms_guard_on_last_proof": round(t_on.commit_aux, 3),
                "kernel_launches": {"guard_on": on.timings().kernel_launches, "guard_off": off.timings().kernel_launches},
            }
    finally:
        on.close(); off.close()
    line = json.dumps(result)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
