#!/usr/bin/env python3
"""Time proofs of the byte-pair-table statement of tests/test_lookup_preprocessed.py: a 2^20-row requester against a
2^16-row LUT with 4 preprocessed columns.  Two arms on the same traces, alternating:
  device: both LogUp aux traces built on the device; the LUT's lookup program reads its preprocessed columns (op 15),
          re-derived from the installed bundle's coefficients;
  host:   the LUT without its lookup program, its aux trace from the Python-integer host aux callback (the requester is
          built on the device in both arms).
Reported: the whole proof per arm (median and range over the timed proofs after one warm-up each; mdn_prove ends in a
stream synchronisation), and from a torch.profiler trace taken in a separate pass the device arm's k_logup_rows and the
forward-NTT kernels of each arm -- the device arm's extra forward-NTT time is the re-derivation of the preprocessed rows.
The two arms' proofs must be identical.  Prints one JSON line with the card's name and power limit.  MDN_LIB_PATH
selects another build of the library, as for bench.py."""
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
    ap.add_argument("--log-req", type=int, default=20)
    ap.add_argument("--log-lut", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5, help="timed proofs per arm (after one warm-up each)")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    import helpers as H
    import test_lookup_preprocessed as T
    params = W.fast_pcs_params()
    case = T.Case(a.log_lut, a.log_req, seed=20)
    arms = {"device": (case.wl(True), None), "host": (case.oracle_wl(), B.AUX_BUILDER(case.host_builder()))}
    ch = W.initial_challenger(params, H.oracle_observe)
    s = B.Session(params, 0)
    s.set_preprocessed(arms["device"][0].statement, arms["device"][0].preprocessed_matrices)

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

    kern = {}
    for arm in arms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            prove(arm)
            torch.cuda.synchronize()
        tot = {"k_logup_rows": 0.0, "fwd_ntt": 0.0}
        for e in prof.key_averages():
            name = e.key
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            if "k_logup_rows" in name or name.startswith("k_jit"):
                tot["k_logup_rows"] += us
            elif "fwd" in name:
                tot["fwd_ntt"] += us
        kern[arm] = {k: round(v / 1e3, 3) for k, v in tot.items()}
    rederive = round(kern["device"]["fwd_ntt"] - kern["host"]["fwd_ntt"], 3)
    print(json.dumps({"card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
                      "log_req": a.log_req, "log_lut": a.log_lut, "proofs_identical": bool(same),
                      "proof_ms": {arm: stats(v) for arm, v in ms.items()},
                      "kernel_ms_per_proof": kern, "rederive_fwd_ntt_ms": rederive}))
    s.close()


if __name__ == "__main__":
    main()
