#!/usr/bin/env python3
"""Time mdn_constraint_census against mdn_check_constraints on the benchmark statement: 2^20 x (51, 22, 16),
DummyMidenAir, no aux builder, in three cases: valid (column 0 is zero), one constraint broken on every row (instance
1's column 0 set to 1) and about a thousand scattered faults (random rows of column 0 in every AIR).  Per case, after
one warm-up call of each, census and check calls alternate; every call ends in a stream synchronisation inside the
library, so host-clock times around the calls are device-complete.  The kernel times come from a torch.profiler trace
of separate calls.  Prints one JSON line with the card's name and power limit.  MDN_LIB_PATH selects another build of
the library, as for bench.py."""
import argparse, ctypes as C, json, os, subprocess, sys, time
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


def workload(W, P, log_n, case):
    wl = W.Workload([log_n] * 3)
    if case == "column":
        wl.traces[1][:, 0] = 1
    elif case == "scattered":
        rng = np.random.default_rng(20)
        for i, t in enumerate(wl.traces):
            rows = rng.choice(1 << log_n, 333 + i, replace=False)
            t[rows, 0] = rng.integers(1, P, len(rows), dtype=np.uint64)
    return wl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=7, help="timed calls of each (after one warm-up call of each)")
    ap.add_argument("--max-failures", type=int, default=1 << 12)
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    lib = B.lib()
    params = W.miden_pcs_params()

    def observe(c, felts):
        lib.mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))

    ch = W.initial_challenger(params, observe)
    sess = B.Session(params, 0)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    result = {"shape": f"2^{a.log_n} x (51, 22, 16), DummyMidenAir", "max_failures": a.max_failures,
              "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()}, "cases": {}}
    try:
        for case in ("valid", "column", "scattered"):
            wl = workload(W, W.P, a.log_n, case)
            out = {}

            def census():
                c, _, _, _ = sess.constraint_census(wl.statement, wl.matrices, ch, max_failures=a.max_failures, max_tallies=64)
                out["violations"] = c.violations
                out["failing_rows"] = c.first.failing_rows

            def check():
                sess.check_constraints(wl.statement, wl.matrices, ch)

            census(); check()
            census_ms, check_ms = [], []
            for _ in range(a.reps):
                census_ms.append(timed(census))
                check_ms.append(timed(check))
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    census()
                    check()
                torch.cuda.synchronize()
            kern = {}
            for ev in prof.events():
                if ev.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                for name in ("k_census_rows", "k_census_list", "k_count_scan", "k_check_rows"):
                    if name in ev.name:
                        kern[name] = kern.get(name, 0.0) + ev.device_time / 1e3 / a.reps
            result["cases"][case] = {
                "violations": out["violations"], "failing_rows": out["failing_rows"],
                "census_ms_median": round(float(np.median(census_ms)), 2),
                "census_ms_range": [round(min(census_ms), 2), round(max(census_ms), 2)],
                "check_ms_median": round(float(np.median(check_ms)), 2),
                "check_ms_range": [round(min(check_ms), 2), round(max(check_ms), 2)],
                "kernel_ms_per_call": {k: round(v, 3) for k, v in sorted(kern.items())},
            }
    finally:
        sess.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
