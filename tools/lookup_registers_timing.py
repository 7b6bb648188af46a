#!/usr/bin/env python3
"""Time proofs of the uint-chiplet statement of tests/test_lookup_registers.py: a 2^20-row MUL-like AIR (two register
columns) and a 2^16-row STORE-like AIR (one register column) on host row-major traces.  Two arms on the same traces,
alternating:
  device: both aux traces -- LogUp and register columns -- built on the device from version-2 lookup programs;
  host:   both aux traces from the Python-integer host aux callback (the AIRs ship no lookup program).
Reported: the whole proof per arm (median and range over the timed proofs after one warm-up each; mdn_prove ends in a
stream synchronisation), and from a torch.profiler trace taken in a separate pass the device arm's register kernels
(k_reg_*) and LogUp row kernel per proof.  The two arms' proofs must be identical.  Prints one JSON line with the
card's name and power limit.  MDN_LIB_PATH selects another build of the library, as for bench.py."""
import argparse, json, os, statistics, subprocess, sys, time
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
    ap.add_argument("--log-mul", type=int, default=20)
    ap.add_argument("--log-store", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5, help="timed proofs per arm (after one warm-up each)")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    import helpers as H
    import test_lookup_registers as T
    params = W.fast_pcs_params()
    case = T.Case(a.log_mul, a.log_store, seed=20)
    arms = {"device": (case.wl(True), None), "host": (case.wl(False), B.AUX_BUILDER(case.host_builder()))}
    ch = W.initial_challenger(params, H.oracle_observe)
    s = B.Session(params, 0)

    def prove(arm):
        wl, cb = arms[arm]
        return s.prove(wl.statement, wl.matrices, ch, cb)

    proofs = {arm: prove(arm) for arm in arms}            # warm-up
    same = all(np.array_equal(x, y) for x, y in zip(proofs["device"][1:], proofs["host"][1:])) and proofs["device"][0] == proofs["host"][0]
    ms = {arm: [] for arm in arms}
    for _ in range(a.reps):
        for arm in arms:
            t0 = time.perf_counter()
            prove(arm)
            ms[arm].append((time.perf_counter() - t0) * 1e3)
            print(f"{arm}: {ms[arm][-1]:.1f} ms", file=sys.stderr, flush=True)

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        prove("device")
        torch.cuda.synchronize()
    tot = {"k_reg_block_maps": 0.0, "k_reg_block_carry": 0.0, "k_reg_apply": 0.0, "k_logup_rows": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        for k in tot:
            if k in e.key:
                tot[k] += us
    kern = {k: round(v / 1e3, 3) for k, v in tot.items()}
    kern["registers_total"] = round(sum(v for k, v in kern.items() if k.startswith("k_reg")), 3)
    print(json.dumps({"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
                      "log_mul": a.log_mul, "log_store": a.log_store, "proofs_identical": bool(same),
                      "proof_ms": {arm: stats(v) for arm, v in ms.items()}, "device_kernel_ms_per_proof": kern}))
    s.close()


if __name__ == "__main__":
    main()
