#!/usr/bin/env python3
"""Time mdn_check_lookup_folds on the closed bus of tests/test_trace_balance.py at 2^20 lookup rows against a 2^16 table
(plus one AIR without lookup), with aux == NULL: the call builds the LogUp aux traces on the device and checks them
against the constraint-path folds.  Reported: the whole call (host row-major traces, upload included; median and range
over the timed calls after one warm-up), the k_fold_rows kernels and the device LogUp build (k_logup_rows and the scan)
of the same call from a torch.profiler trace taken in a separate pass, and the CPU oracle's walk
orc_collect_column_folds (tests/oracle_folds, single-threaded like the reference's).  Every library call ends in a stream
synchronisation, so host-clock times around the calls are device-complete.  Prints one JSON line with the card's name and
power limit.  MDN_LIB_PATH selects another build of the library, as for bench.py."""
import argparse, json, os, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import pkgload


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-l", type=int, default=20)
    ap.add_argument("--log-t", type=int, default=16)
    ap.add_argument("--reps", type=int, default=9, help="timed calls (after one warm-up call)")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    import test_trace_balance as TB
    import test_lookup_folds as TF
    bus = TB.Bus(log_t=a.log_t, log_l=a.log_l, seed=3, n_boundary=4)
    wl, marks, _ = TF.marked(bus)
    sess = B.Session(W.miden_pcs_params(), 0)

    def folds():
        rep = sess.check_lookup_folds(wl.statement, wl.matrices, TB.RND, marks)
        assert rep["holds"] == 1

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    try:
        folds()
        call_ms = [timed(folds) for _ in range(a.reps)]
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                folds()
            torch.cuda.synchronize()
        kern = {"folds": 0.0, "logup": 0.0}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            if "k_fold_rows" in ev.name:
                kern["folds"] += ev.device_time / 1e3
            elif "k_logup_rows" in ev.name or "k_scan" in ev.name:
                kern["logup"] += ev.device_time / 1e3
    finally:
        sess.close()
    t0 = time.perf_counter()
    TF.oracle_folds(wl, TB.RND, marks)
    orc_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({
        "shape": f"lookup AIR 2^{a.log_l} x 11 (3 aux columns) + table AIR 2^{a.log_t} x 3 + one AIR without lookup",
        "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()},
        "folds_call_ms": {"median": round(statistics.median(call_ms), 2), "min": round(min(call_ms), 2), "max": round(max(call_ms), 2), "n": len(call_ms)},
        "fold_kernels_ms_per_call": round(kern["folds"] / a.reps, 3),
        "logup_build_kernels_ms_per_call": round(kern["logup"] / a.reps, 3),
        "oracle_walk_ms": round(orc_ms, 1),
    }))


if __name__ == "__main__":
    main()
