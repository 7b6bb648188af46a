#!/usr/bin/env python3
"""Time mdn_check_constraints against mdn_prove on the benchmark statement: 2^20 x (51, 22, 16), DummyMidenAir, no aux
builder (the traces satisfy the constraint: column 0 is zero).  After one warm-up call of each, checks and proofs
alternate; every call ends in a stream synchronisation inside the library, so host-clock times around the calls are
device-complete.  The check's k_check_rows device time comes from a torch.profiler trace of separate calls.  Prints one
JSON line with the card's name and power limit.  MDN_LIB_PATH selects another build of the library, as for bench.py."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5, help="timed calls of each (after one warm-up call of each)")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    lib = B.lib()
    params = W.miden_pcs_params()
    wl = W.Workload([a.log_n] * 3)

    def observe(c, felts):
        lib.mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))

    ch = W.initial_challenger(params, observe)
    sess = B.Session(params, 0)

    def check():
        rep, _ = sess.check_constraints(wl.statement, wl.matrices, ch)
        assert rep.holds == 1 and rep.failing_rows == 0, (rep.kind, rep.instance, rep.row, rep.failing_rows)

    def prove():
        sess.prove(wl.statement, wl.matrices, ch)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    try:
        check(); prove()
        check_ms, prove_ms = [], []
        for _ in range(a.reps):
            check_ms.append(timed(check))
            prove_ms.append(timed(prove))
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                check()
            torch.cuda.synchronize()
        kern, launches = 0.0, 0
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "k_check_rows" in ev.name:
                kern += ev.device_time / 1e3
                launches += 1
    finally:
        sess.close()
    med_c, med_p = float(np.median(check_ms)), float(np.median(prove_ms))
    print(json.dumps({
        "shape": f"2^{a.log_n} x (51, 22, 16), DummyMidenAir",
        "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()},
        "check_ms": sorted(round(x, 2) for x in check_ms),
        "prove_ms": sorted(round(x, 2) for x in prove_ms),
        "check_over_prove": round(med_c / med_p, 3),
        "k_check_rows_ms_per_call": round(kern / a.reps, 3),
        "k_check_rows_launches_per_call": launches // a.reps,
    }))


if __name__ == "__main__":
    main()
