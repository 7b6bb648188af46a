#!/usr/bin/env python3
"""Time the coset LDE: mdn_coset_lde_batch of a 2^log_n x cols matrix with blowup 2^log_blowup (default 2^20 x 89, blowup
8), whole call with CUDA events, and each NTT kernel class inside it (k_intt_strided, k_intt_contig, k_fwd_contig,
k_fwd_strided) from a torch.profiler trace of separate calls.  The whole-call time includes the host -> device upload of
the matrix and the device -> host copy of the LDE; the kernel times are device time per call.  Prints one JSON line with
the card's name and power limit.  MDN_LIB_PATH selects another build of the library, as for bench.py."""
import argparse, ctypes as C, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import pkgload

KERNELS = ("k_intt_strided", "k_intt_contig", "k_fwd_contig", "k_fwd_strided")
P = 0xFFFFFFFF00000001


def power_limit_w():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--cols", type=int, default=89)
    ap.add_argument("--log-blowup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5, help="timed calls (after one warm-up call)")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    lib = B.lib()
    params = W.miden_pcs_params() if a.log_blowup == 3 else B.PcsParams(a.log_blowup, 2, 1, 1, 2, 6, 3)
    rng = np.random.default_rng(1)
    m = rng.integers(0, P, size=(1 << a.log_n, a.cols), dtype=np.uint64)
    lde_log = a.log_n + a.log_blowup
    shift = pow(7, 1 << (32 - lde_log), P)
    out = np.empty(((1 << a.log_n) << a.log_blowup, a.cols), dtype=np.uint64)
    sess = B.Session(params, 0)

    def call():
        rc = lib.mdn_coset_lde_batch(sess.handle, C.byref(B.Matrix(B.ptr(m), a.log_n, a.cols)), a.log_blowup, shift,
                                     B.ptr(out.reshape(-1)))
        assert rc == 0, lib.mdn_last_error(sess.handle)

    try:
        call()
        torch.cuda.synchronize()
        call_ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); call(); e1.record(); torch.cuda.synchronize()
            call_ms.append(e0.elapsed_time(e1))
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                call()
            torch.cuda.synchronize()
        kern = {k: 0.0 for k in KERNELS}
        launches = {k: 0 for k in KERNELS}
        for ev in prof.events():
            if ev.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for k in KERNELS:
                if k + "<" in ev.name:
                    kern[k] += ev.device_time / 1e3
                    launches[k] += 1
    finally:
        sess.close()
    per_call = {k: round(v / a.reps, 3) for k, v in kern.items()}
    print(json.dumps({
        "shape": f"2^{a.log_n} x {a.cols} columns, blowup {1 << a.log_blowup}",
        "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()},
        "call_ms": sorted(round(x, 2) for x in call_ms),
        "kernel_ms_per_call": per_call,
        "ntt_ms_per_call": round(sum(per_call.values()), 3),
        "launches_per_call": {k: v // a.reps for k, v in launches.items()},
    }))


if __name__ == "__main__":
    main()
