#!/usr/bin/env python3
"""Time mdn_lookup_fold_census against mdn_check_lookup_folds on the closed bus of tests/test_trace_balance.py at 2^20
lookup rows (11 main, 3 aux columns) against a 2^16 table (plus one AIR without lookup), with host row-major traces and
an explicit aux trace (the oracle's prover path, tests/oracle_fold_census orc_logup_aux).  Three inputs: the aux trace as
built (the statement holds), aux column 1 wrong on every row (2^20 disagreements), and about 1000 scattered faults in
column 2.  Reported per input: the whole call of each function (median and range over the timed calls after one
warm-up, the two functions alternating), and from a torch.profiler trace taken in a separate pass the census's kernels
(k_fold_census_rows, the count scan, k_fold_census_list) against the fold check's k_fold_rows.  Every library call ends
in a stream synchronisation, so host-clock times around the calls are device-complete.  Prints one JSON line with the
card's name and power limit.  MDN_LIB_PATH selects another build of the library, as for bench.py."""
import argparse, json, os, random, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
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


def stats(xs):
    return {"median": round(statistics.median(xs), 2), "min": round(min(xs), 2), "max": round(max(xs), 2), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-l", type=int, default=20)
    ap.add_argument("--log-t", type=int, default=16)
    ap.add_argument("--reps", type=int, default=7, help="timed calls of each function per input (after one warm-up each)")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    import test_trace_balance as TB
    import test_lookup_folds as TF
    import test_lookup_fold_census as TC
    bus = TB.Bus(log_t=a.log_t, log_l=a.log_l, seed=3, n_boundary=4)
    wl, marks, _ = TF.marked(bus)
    base, finals = TC.oracle_aux(wl, TB.RND)
    P, n = TB.P, 1 << a.log_l
    column = [x.copy() if x is not None else None for x in base]
    column[1][:, 2] = (column[1][:, 2] + np.uint64(1)) % np.uint64(P)
    scattered = [x.copy() if x is not None else None for x in base]
    for r in random.Random(20).sample(range(n), 1000):
        TC._bump(scattered[1], r, 4)
    inputs = {"holds": base, "column": column, "scattered": scattered}
    sess = B.Session(W.miden_pcs_params(), 0)
    result = {}

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    try:
        for name, auxs in inputs.items():
            mats, keep = TF.aux_for(wl, auxs, "host")

            def census():
                out, _, _ = sess.lookup_fold_census(wl.statement, wl.matrices, TB.RND, marks, mats, finals, 0, 1 << 16, 1 << 16)
                assert (out.disagreements == 0) == (name == "holds")

            def check():
                rep = sess.check_lookup_folds(wl.statement, wl.matrices, TB.RND, marks, mats, finals)
                assert rep["holds"] == (name == "holds")

            census(); check()
            t_census, t_check = [], []
            for _ in range(a.reps):
                t_census.append(timed(census))
                t_check.append(timed(check))
            from torch.profiler import profile, ProfilerActivity
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    census(); check()
                torch.cuda.synchronize()
            kern = {"k_fold_census_rows": 0.0, "count_scan": 0.0, "k_fold_census_list": 0.0, "k_fold_rows": 0.0}
            for ev in prof.events():
                if ev.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                for key, pat in (("k_fold_census_rows", "k_fold_census_rows"), ("k_fold_census_list", "k_fold_census_list"),
                                 ("count_scan", "k_count_scan"), ("k_fold_rows", "k_fold_rows")):
                    if pat in ev.name:
                        kern[key] += ev.device_time / 1e3
            per = {k: round(v / a.reps, 3) for k, v in kern.items()}
            per["census_kernels"] = round(per["k_fold_census_rows"] + per["count_scan"] + per["k_fold_census_list"], 3)
            result[name] = {"census_call_ms": stats(t_census), "check_call_ms": stats(t_check), "kernels_ms_per_call": per}
    finally:
        sess.close()
    print(json.dumps({
        "shape": f"lookup AIR 2^{a.log_l} x 11 (3 aux columns) + table AIR 2^{a.log_t} x 3 + one AIR without lookup, host traces and aux",
        "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()},
        **result,
    }))


if __name__ == "__main__":
    main()
