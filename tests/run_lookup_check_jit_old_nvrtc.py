"""Subprocess of test_lookup_check_jit.test_self_check_with_torch_bundled_nvrtc: forces the older NVRTC that torch bundles
(a build of it was seen to miscompile large chunk functions) and runs the three lookup checks of the Miden-shaped
statement (tools/lookup_check_timing.py) on a session that specialises every program.  Every report must equal the
interpreter's.  Prints SELF-CHECK OK when a first-use comparison retired a miscompiled kernel (MDN_INFO_JIT_LOOKUP_CHECK
is then 0 and mdn_jit_status says why), NOTE when this NVRTC build compiled the kernels correctly."""
import glob
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))

cands = glob.glob(os.path.join(sys.prefix, "lib", "python*", "site-packages", "nvidia", "cuda_nvrtc", "lib", "libnvrtc.so.12"))
if not cands:
    print("SKIP no bundled nvrtc"); sys.exit(0)
os.environ["MDN_NVRTC_PATH"] = cands[0]
os.environ["MDN_NVRTC_ALLOW_OLD"] = "1"
import lookup_check_timing as LT
import test_lookup_fold_census as TFC
import test_trace_balance as TB
W, B, AP = TB.W, TB.B, TB.AP
RND = TB.RND

wl, sites, marks = LT.statement(W, AP, W.P, 12, "scattered")
jit, interp = B.Session(W.fast_pcs_params(), 0), B.Session(W.fast_pcs_params(), 0)
jit.set_jit(1); interp.set_jit(0)
calls = {
    "balance": lambda s: s.check_trace_balance(wl.statement, wl.matrices, RND, (), sites),
    "folds": lambda s: s.check_lookup_folds(wl.statement, wl.matrices, RND, marks),
    "census": lambda s: TFC._raw(*s.lookup_fold_census(wl.statement, wl.matrices, RND, marks)),
}
try:
    retired = False
    for name, call in calls.items():
        got = call(jit)
        used = [int(v) for v in jit.info(B.INFO_JIT_LOOKUP_CHECK)]
        assert got == call(interp), f"{name}: the report differs from the interpreter"
        status = jit.jit_status()
        print("CALL", name, "USED", used, "STATUS", status)
        if used == [0, 0]:
            assert "NVRTC lookup-check kernel disagreed with the interpreter on its first use; interpreter kept" in status
            assert call(jit) == got and [int(v) for v in jit.info(B.INFO_JIT_LOOKUP_CHECK)] == [0, 0]   # retired for good
            retired = True
        else:
            assert used == [1, 1]
    print("SELF-CHECK OK" if retired else "NOTE this NVRTC build did not miscompile the lookup-check kernels; self-check path not exercised")
finally:
    jit.close(); interp.close()
