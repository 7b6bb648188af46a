"""Subprocess of tests/test_jit_cache.py: one fresh process on a persistent NVRTC cubin cache (mdn_jit_set_cache_dir).

  run_jit_cache.py compile DIR PROGRAM...   mdn_jit_compile_check on each program (.npy of u32 words), no device
  run_jit_cache.py gpu DIR OUT              the NVRTC row passes of every kind on the H100

DIR "-" leaves the cache off.  Prints one JSON line: the return values or outputs, and the process's
mdn_get_info(NULL, MDN_INFO_JIT_CACHE) counts at the end."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

import pkgload

pkg = pkgload.load_pkg()
W, B = pkg.workload, pkg.binding


def plain(x):
    """outputs as JSON values, byte for byte: arrays and ctypes structs as hex of their bytes"""
    if isinstance(x, np.ndarray):
        return x.dtype.str + ":" + x.tobytes().hex()
    if isinstance(x, (bytes, bytearray)):
        return x.hex()
    if isinstance(x, C.Structure) or isinstance(x, C.Array):
        return bytes(x).hex()
    if isinstance(x, dict):
        return {str(k): plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [plain(v) for v in x]
    if isinstance(x, (np.integer,)):
        return int(x)
    return x


def compile_programs(paths):
    out = []
    for p in paths:
        try:
            out.append(B.jit_compile_check(np.load(p)))
        except B.ProverError as e:
            out.append(str(e))
    return out


def gpu_passes(jit_min_nodes):
    """The row passes a statement can specialise, each on a fresh session with set_jit(jit_min_nodes): a guarded proof
    with the device LogUp build, the same proof unguarded, mdn_constraint_census, mdn_check_trace_balance and
    mdn_lookup_fold_census.  Returns (outputs, info flags, the JIT note after each call)."""
    import test_airs as TA
    import test_constraint_census as TCC
    import test_constraint_guard as TG
    import test_jit_self_check as TJS
    import test_lookup_fold_census as TFC
    import test_trace_balance as TB
    params = W.fast_pcs_params()
    outs, flags, notes = {}, {}, {}
    wl, _ = TA.logup_workload(7, device=True)
    for name, guard in (("guarded_proof", True), ("proof", False)):
        s = TG.hash_session(params, guard=guard)
        s.set_jit(jit_min_nodes)
        aux_note, proof, _ = TJS.staged_proof(s, wl, params)
        outs[name], flags[name] = proof, TJS.flags(s, TJS.INFO_JIT)
        if guard:
            flags[name + "_check"] = TJS.flags(s, TJS.INFO_JIT_CHECK)
        notes[name + "_commit_aux"], notes[name] = aux_note, TJS.note(s)
        s.close()

    s = B.Session(params, 0); s.set_jit(jit_min_nodes)
    cwl, bld, _, _ = TCC.any_case("one_cell")
    outs["census"] = TJS.census_call(s, cwl, params, bld, 1 << 16, 1 << 16)
    flags["census"], notes["census"] = TJS.flags(s, TJS.INFO_JIT_CHECK), TJS.note(s)
    s.close()

    s = B.Session(params, 0); s.set_jit(jit_min_nodes)
    bus, bnd, _, _ = TB.case("mutex")
    bwl, sites, _ = bus.workload()
    mats, fl, keep = TB.traces_for(bwl, "host")
    outs["balance"] = s.check_trace_balance(bwl.statement, mats, TB.RND, bnd, sites, 1 << 16, fl)
    flags["balance"], notes["balance"] = TJS.flags(s, B.INFO_JIT_LOOKUP_CHECK), TJS.note(s)
    flags["balance_lookups"] = [1 if bwl.statement.airs[i].lookup else 0 for i in range(bwl.k)]
    s.close()

    s = B.Session(params, 0); s.set_jit(jit_min_nodes)
    fwl, marks, _, auxs, finals, given = TFC.case("scattered")
    outs["fold_census"] = TFC.run(s, fwl, marks, "host", auxs if given else None, finals if given else None, TFC.ALL, TFC.ALL, raw=True)
    flags["fold_census"], notes["fold_census"] = TJS.flags(s, B.INFO_JIT_LOOKUP_CHECK), TJS.note(s)
    flags["fold_census_lookups"] = [1 if fwl.statement.airs[i].lookup else 0 for i in range(fwl.k)]
    s.close()
    return plain(outs), flags, notes


def main():
    mode, d = sys.argv[1], sys.argv[2]
    B.set_jit_cache_dir(None if d == "-" else d)
    if mode == "compile":
        res = {"results": compile_programs(sys.argv[3:])}
    else:
        outs, flags, notes = gpu_passes(1)
        res = {"outputs": outs, "flags": flags, "notes": notes}
        res["stats"] = B.jit_cache_stats()           # before the interpreter's run, which compiles nothing
        res["interpreter_outputs"] = gpu_passes(0)[0]
        with open(sys.argv[3], "w") as f:
            json.dump(res, f)
    res["stats"] = res.get("stats") or B.jit_cache_stats()
    print(json.dumps({k: v for k, v in res.items() if k in ("results", "stats", "flags", "notes")}))


if __name__ == "__main__":
    main()
