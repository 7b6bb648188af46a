#!/usr/bin/env python3
"""What the persistent cubin cache (mdn_jit_set_cache_dir) saves a fresh process, at 2^20 rows.

Each arm is a fresh process on a cache directory: "cold" on an empty one (every NVRTC-specialised kernel is compiled and
written), "warm" on the directory the cold process before it filled (every kernel is read back).  The arms alternate,
cold then warm, --rounds times.  Each process, with the default JIT threshold:
  * builds the statements (host traces; not timed);
  * creates a session (miden_pcs_params) with the constraint guard on and proves the Miden-size statement of
    tools/guard_timing.py (three AIRs, 2^20 x (51, 22, 16), about 5.2 k constraint operations per row): this
    compiles or reads the proof's constraint kernels and the guard's check kernels;
  * then runs mdn_check_trace_balance on the Miden-shaped lookup statement of tools/lookup_check_timing.py (two AIRs
    x 2^20 rows, the 2866-node MainLookupAir-shaped program): the lookup-check kernels.
Reported per arm: wall ms from session creation to the end of the first guarded proof, to the end of the first
mdn_check_trace_balance, and the process's NVRTC compiles and NVRTC wall ms (mdn_get_info(NULL, MDN_INFO_JIT_CACHE)).
Host clocks; both calls end in a stream synchronisation inside the library.  Every arm must give the same proof and
the same balance report.  Prints one JSON line with the card's name and power limit, read in the same run."""
import argparse, hashlib, json, os, subprocess, sys, tempfile, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def child(cache_dir, log_n):
    import ctypes as C
    import numpy as np
    import pkgload
    import guard_timing as GT
    import lookup_check_timing as LT
    pkg = pkgload.load_pkg()
    B, W, AP = pkg.binding, pkg.workload, pkg.air_program
    lib = B.lib()
    B.set_jit_cache_dir(cache_dir)
    params = W.miden_pcs_params()

    def observe(c, felts):
        lib.mdn_challenger_observe(C.byref(c), B.ptr(np.ascontiguousarray(felts, dtype=np.uint64)), len(felts))

    ch = W.initial_challenger(params, observe)
    miden = W.Workload([log_n] * 3, programs=[GT.zero_column_air(AP, W.P, *spec) for spec in GT.MIDEN_SIZE])
    for i, t in enumerate(miden.traces):
        t[:, miden.widths[i] - 1] = 0
    lwl, sites, _ = LT.statement(W, AP, W.P, log_n, "scattered")
    rnd = np.array([0x1234567, 0x89ABCDE, 0x13579BD, 0x2468ACE], dtype=np.uint64)

    t0 = time.perf_counter()
    s = B.Session(params, 0)
    s.set_constraint_guard(True)
    heights, fields, comms = s.prove(miden.statement, miden.matrices, ch)
    t_proof = time.perf_counter()
    after_proof = B.jit_cache_stats()
    rep = s.check_trace_balance(lwl.statement, lwl.matrices, rnd, (), sites, 1 << 12)
    t_balance = time.perf_counter()
    st = B.jit_cache_stats()
    out = {"to_first_guarded_proof_ms": round((t_proof - t0) * 1e3, 1),
           "to_first_balance_ms": round((t_balance - t0) * 1e3, 1),
           "first_balance_call_ms": round((t_balance - t_proof) * 1e3, 1),
           "nvrtc_ms": st["compile_ms"], "nvrtc_ms_in_proof": after_proof["compile_ms"], "cache": st,
           "jit_used": [int(x) for x in s.info(8)], "jit_check_used": [int(x) for x in s.info(11)],
           "jit_lookup_check_used": [int(x) for x in s.info(B.INFO_JIT_LOOKUP_CHECK)],
           "proof_sha256": hashlib.sha256(bytes(heights) + fields.tobytes() + comms.tobytes()).hexdigest(),
           "balance_sha256": hashlib.sha256(repr(rep).encode()).hexdigest()}
    s.close()
    print("ARM " + json.dumps(out), flush=True)


def device():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
    if not q:
        raise SystemExit("no GPU: this measurement runs on the H100 only")
    name, limit = [x.strip() for x in q[0].split(",")]
    return {"name": name, "power_limit_w": float(limit)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3, help="cold / warm pairs, alternated")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child is not None:
        return child(a.child, a.log_n)
    result = {"shape": f"guarded proof 2^{a.log_n} x (51, 22, 16) Miden-size programs, miden_pcs_params; "
                       f"mdn_check_trace_balance 2 x 2^{a.log_n} rows, 2866-node lookup program",
              "device": device(), "arms": {"cold": [], "warm": []}}
    with tempfile.TemporaryDirectory(prefix="mdn_jit_cache_") as tmp:
        for r in range(a.rounds):
            d = os.path.join(tmp, f"round{r}")
            os.mkdir(d)
            for arm in ("cold", "warm"):
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--log-n", str(a.log_n), "--child", d],
                                   capture_output=True, text=True, timeout=3600)
                line = [x for x in p.stdout.splitlines() if x.startswith("ARM ")]
                if p.returncode != 0 or not line:
                    raise SystemExit(f"{arm} arm failed:\n{p.stdout}\n{p.stderr}")
                res = json.loads(line[0][4:])
                res["files"] = len(os.listdir(d))
                result["arms"][arm].append(res)
                print(arm, json.dumps(res), flush=True)
    runs = result["arms"]["cold"] + result["arms"]["warm"]
    assert len({x["proof_sha256"] for x in runs}) == 1 and len({x["balance_sha256"] for x in runs}) == 1, "the arms disagree"
    assert all(x["cache"]["compiles"] == 0 for x in result["arms"]["warm"]), "a warm process compiled"
    for arm, xs in result["arms"].items():
        result[arm + "_median"] = {k: sorted(x[k] for x in xs)[len(xs) // 2]
                                   for k in ("to_first_guarded_proof_ms", "to_first_balance_ms", "first_balance_call_ms", "nvrtc_ms")}
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
