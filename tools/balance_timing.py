#!/usr/bin/env python3
"""Time mdn_check_trace_balance on the closed bus of tests/test_trace_balance.py at 2^20 lookup rows against a 2^16 table
(plus one AIR without lookup and four boundary emissions; one flipped flag leaves one denominator unmatched).  Compared
with (a) the device LogUp build of the same traces -- the k_logup_rows and scan kernels of mdn_check_constraints, from a
torch.profiler trace -- and (b) the CPU oracle's walk orc_check_trace_balance (tests/oracle_balance, single-threaded like
the reference's).  Every library call ends in a stream synchronisation, so host-clock times around the calls are
device-complete.  Prints one JSON line with the card's name and power limit.  MDN_LIB_PATH selects another build of the
library, as for bench.py."""
import argparse, ctypes as C, json, os, subprocess, sys, time
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-l", type=int, default=20)
    ap.add_argument("--log-t", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5, help="timed calls (after one warm-up call)")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    import test_trace_balance as TB
    lib = B.lib()
    params = W.miden_pcs_params()
    bus = TB.Bus(log_t=a.log_t, log_l=a.log_l, seed=3, n_boundary=4)
    bus.sender[1000, 2] ^= 1
    wl, sites, _ = bus.workload()
    bnd = bus.boundary(TB.RND)

    def observe(c, felts):
        lib.mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))

    ch = W.initial_challenger(params, observe)
    sess = B.Session(params, 0)

    def balance():
        rep = sess.check_trace_balance(wl.statement, wl.matrices, TB.RND, bnd, sites)
        assert rep["n_unmatched"] == 1

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    try:
        balance()
        sess.check_constraints(wl.statement, wl.matrices, ch)
        bal_ms = [timed(balance) for _ in range(a.reps)]
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                balance()
                sess.check_constraints(wl.statement, wl.matrices, ch)
            torch.cuda.synchronize()
        kern = {"balance": 0.0, "logup": 0.0}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            if "k_balance" in ev.name:
                kern["balance"] += ev.device_time / 1e3
            elif "k_logup_rows" in ev.name or "k_scan" in ev.name:
                kern["logup"] += ev.device_time / 1e3
    finally:
        sess.close()
    t0 = time.perf_counter()
    orc = TB.oracle_balance(wl, TB.RND, bnd, sites)
    orc_ms = (time.perf_counter() - t0) * 1e3
    assert orc["n_unmatched"] == 1
    print(json.dumps({
        "shape": f"lookup AIR 2^{a.log_l} x 11 + table AIR 2^{a.log_t} x 3 + one AIR without lookup, 4 boundary emissions",
        "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()},
        "balance_call_ms": sorted(round(x, 2) for x in bal_ms),
        "balance_kernels_ms_per_call": round(kern["balance"] / a.reps, 3),
        "logup_build_kernels_ms_per_call": round(kern["logup"] / a.reps, 3),
        "oracle_walk_ms": round(orc_ms, 1),
    }))


if __name__ == "__main__":
    main()
