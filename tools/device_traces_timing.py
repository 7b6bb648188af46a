#!/usr/bin/env python3
"""Time one proof from three trace sources: host pinned row-major, device row-major (MDN_FLAG_DEVICE_TRACES) and device
column-major (| MDN_FLAG_COLUMN_MAJOR).  Two statements at 2^log_n x (51, 22, 16), DummyMidenAir: the benchmark statement
(no aux builder: zero aux traces) and the same statement with aux traces from a builder.  There, the host sources use a
host builder (the library copies its row-major output up and transposes it), and the column-major source uses a device
builder that copies the same columns from device memory into the aux slot on the session's stream (no host round trip).
The builders' aux columns are prepared before timing, so the times measure the library's side.  The sources alternate
after one warm-up proof each; every proof ends in a stream synchronisation inside the library.  Every proof of a
statement must be byte-identical.  Prints one JSON line with the card's name and power limit."""
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
    ap.add_argument("--reps", type=int, default=5, help="timed proofs of each source (after one warm-up proof each)")
    a = ap.parse_args()
    pkg = pkgload.load_pkg()
    B, W = pkg.binding, pkg.workload
    lib = B.lib()
    params = W.miden_pcs_params()
    wl = W.Workload([a.log_n] * 3)
    n = 1 << a.log_n

    def observe(c, felts):
        lib.mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))

    ch = W.initial_challenger(params, observe)
    pinned = [torch.from_numpy(t.view(np.int64)).pin_memory() for t in wl.traces]
    dev_rm = [t.cuda() for t in pinned]
    dev_cm = [torch.from_numpy(np.ascontiguousarray(t.T).view(np.int64)).cuda() for t in wl.traces]

    def mats(ts):
        m = (B.Matrix * wl.k)()
        for i, t in enumerate(ts):
            m[i] = B.Matrix(C.cast(C.c_void_p(t.data_ptr()), B.u64p), wl.log_heights[i], wl.widths[i])
        return m

    m_pin, m_rm, m_cm = mats(pinned), mats(dev_rm), B.device_matrices(dev_cm)
    # aux columns (canonical, pseudo-random; the dummy AIR does not constrain them), row-major on the host, column-major on the device
    aux_rm = [(W.splitmix64(np.arange(n * 2 * w, dtype=np.uint64) ^ np.uint64(77 + i)) % np.uint64(W.P)).reshape(n, 2 * w)
              for i, w in enumerate(wl.aux_widths)]
    aux_cm = [torch.from_numpy(np.ascontiguousarray(x.T).view(np.int64)).cuda() for x in aux_rm]

    def host_builder(ctx, inst, main, rnd, aux_out, aux_values):
        C.memmove(aux_out, aux_rm[inst].ctypes.data, aux_rm[inst].nbytes)
        for q in range(2 * wl.aux_widths[inst]):
            aux_values[q] = q
        return 0

    class Cai:
        def __init__(self, addr, shape):
            self.__cuda_array_interface__ = {"shape": shape, "typestr": "<i8", "data": (addr, False), "version": 3, "strides": None}

    def device_builder(inst, main, rnd, aux_out, stream):
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            torch.as_tensor(Cai(aux_out, tuple(aux_cm[inst].shape)), device="cuda").copy_(aux_cm[inst], non_blocking=True)
        return list(range(2 * wl.aux_widths[inst]))

    hb = B.AUX_BUILDER(host_builder)
    sess = B.Session(params, 0)

    def from_device_rm():
        host = [t.cpu() for t in dev_rm]          # alive until the proof returns
        return sess.prove(wl.statement, mats(host), ch, hb)
    runs = {
        "bench": {"host_pinned_rm": lambda: sess.prove(wl.statement, m_pin, ch),
                  "device_rm": lambda: sess.prove(wl.statement, m_rm, ch, None, B.FLAG_DEVICE_TRACES),
                  "device_cm": lambda: sess.prove(wl.statement, m_cm, ch, None, B.FLAG_DEVICE_TRACES | B.FLAG_COLUMN_MAJOR)},
        # a host builder is refused with row-major device traces, so that source copies the traces back to the host first
        "aux_builder": {"host_pinned_rm": lambda: sess.prove(wl.statement, m_pin, ch, hb),
                        "device_rm": from_device_rm,
                        "device_cm": lambda: sess.prove(wl.statement, m_cm, ch, None, B.FLAG_DEVICE_TRACES | B.FLAG_COLUMN_MAJOR)},
    }
    out = {"shape": f"2^{a.log_n} x (51, 22, 16), DummyMidenAir",
           "device": {"name": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()}}
    try:
        for stmt, srcs in runs.items():
            if stmt == "aux_builder":
                sess.set_device_aux_builder(device_builder)
            proofs = {k: fn() for k, fn in srcs.items()}        # warm-up, and the byte-identity check
            first = next(iter(proofs.values()))
            for k, p in proofs.items():
                assert p[0] == first[0] and np.array_equal(p[1], first[1]) and np.array_equal(p[2], first[2]), (stmt, k)
            ms = {k: [] for k in srcs}
            for _ in range(a.reps):
                for k, fn in srcs.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    ms[k].append((time.perf_counter() - t0) * 1e3)
            out[stmt] = {k: {"median_ms": round(float(np.median(v)), 2), "ms": sorted(round(x, 2) for x in v),
                             "transpose_or_ingest_ms": None} for k, v in ms.items()}
            for k, fn in srcs.items():
                fn()
                out[stmt][k]["transpose_or_ingest_ms"] = round(sess.timings().kernel_ms[0], 3)
    finally:
        sess.set_device_aux_builder(None)
        sess.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
