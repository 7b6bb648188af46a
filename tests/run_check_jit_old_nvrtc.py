"""Subprocess of test_check_jit.test_self_check_with_torch_bundled_nvrtc: forces the older NVRTC that torch bundles (a
build of it was seen to miscompile the 10 k-node program) and runs that program's trace checks -- mdn_check_constraints,
mdn_constraint_census and a guarded proof -- on a session that specialises every program.  Every output must equal the
interpreter's.  Prints SELF-CHECK OK when the first-use comparison retired a miscompiled check kernel (MDN_INFO_JIT_CHECK
is then 0 and mdn_jit_status says why), NOTE when this NVRTC build compiled it correctly."""
import glob
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

cands = glob.glob(os.path.join(sys.prefix, "lib", "python*", "site-packages", "nvidia", "cuda_nvrtc", "lib", "libnvrtc.so.12"))
if not cands:
    print("SKIP no bundled nvrtc"); sys.exit(0)
os.environ["MDN_NVRTC_PATH"] = cands[0]
os.environ["MDN_NVRTC_ALLOW_OLD"] = "1"
import test_airs
import test_check_constraints as TC
import test_constraint_census as TCC
import test_constraint_guard as TG
import test_device_resident as TDR
W, B = TC.W, TC.B

params = W.fast_pcs_params()
wl = test_airs.big_program_workload(5, n_terms=300)
wl.traces[0][[3, 17], 4] = 7                          # the program's constraints vanish identically: rows still run
jit, interp = B.Session(params, 0), B.Session(params, 0)
g_jit, g_int = TG.hash_session(params, guard=True), TG.hash_session(params, guard=True)
jit.set_jit(1); g_jit.set_jit(1); interp.set_jit(0); g_int.set_jit(0)
try:
    got = TCC.device_census(jit, wl, params)
    used = [int(v) for v in jit.info(11)]
    status = jit.jit_status()
    assert got == TCC.device_census(interp, wl, params), "the check or the census differs from the interpreter"
    pj, _ = TG.prove(g_jit, wl, params)
    pi, _ = TG.prove(g_int, wl, params)
    assert TDR.same(pj, pi), "the guarded proof differs"
    print("STATUS", status, "JIT_CHECK", used, "GUARD", [int(v) for v in g_jit.info(11)], g_jit.jit_status())
    if "NVRTC check kernel disagreed" not in status:
        assert used == [1]
        print("NOTE this NVRTC build did not miscompile the check kernels; self-check path not exercised")
    else:
        assert used == [0]
        assert TCC.device_census(jit, wl, params) == got and [int(v) for v in jit.info(11)] == [0]   # retired for good
        print("SELF-CHECK OK")
finally:
    jit.close(); interp.close(); g_jit.close(); g_int.close()
